// kr_kernels.cuh — sm_90a (H100) kernels of the batched reconcile engine.
//
// Integer / hash work: no tensor cores.  What matters here (DESIGN.md §4): coalesced SoA column streaming,
// shared-memory staging (hash chunks, per-tile digit counters, per-warp group accumulators), warp-ballot /
// match_any group-by, grids sized in multiples of the SM count.
//
// A FULL pass is one CUDA graph (stream M unless noted), programmatic dependent launch along the chain.  Production configuration
// (kr_flags.fetch_pod_lists == 0, <= KR_SMEM_GROUPS worker groups unless KR_OPT_WIDE_CLUSTERS, <= 256 pods per RayCluster) — the
// BUCKET pipeline (kr_bucket2.cuh):
//   k_clear          per-pass clears (hash tables, workersToDelete resolutions, totals, bucket counters / first-head cells) in one launch
//   k_build_tables   cluster table (ns,name)->{idx, flags, name of worker group 0}, the 128-byte per-cluster input record (cl_in),
//                    workersToDelete-name table + Bloom bitmap, head-aux table; closes the running incremental epoch
//   k_match2         per pod: selector match -> its cluster's fixed-stride bucket at an arrival rank (one returning atomic):
//                    8-byte record {pod idx, group slot | flags}; first head per cluster by a 64-bit atomicMax
//   k_decide2        one warp per RayCluster, bucket in registers, ARRIVAL order: order-free counts, the ordered delete prefix by
//                    min-extraction / counting rank, status roll-up, action list + replica indices placed with one atomic per cluster
//   k_hash3          (stream H, concurrent) SHA-1 + base32hex of every muted-spec JSON: producer warp (staging, padding, W expansion)
//                    + consumer warp (the 80-round chain) per 32 messages, messages ordered by block count   [> 19 k messages: k_hash2<4,1>]
//   k_decide2 ph. 1  the clusters whose Recreate gate needs the digest, in the places phase 0 reserved
//   k_jobs           RayJob -> RayCluster status roll-up join
//   k_large_sort / k_decide_large   KR_OPT_LARGE_CLUSTERS / KR_OPT_WIDE_CLUSTERS only (kr_large.cuh): the RayClusters of
//                    257..KR_LARGE_MAX_PODS pods and those of more than KR_SMEM_GROUPS worker groups, one CTA each — List order by a
//                    shared-memory sort beside the hash, then a decide by every warp of the CTA (a wide one: the sort pipeline's
//                    memory-resident warp decide)
//   k_huge_tiles / k_huge_merge     KR_OPT_HUGE_CLUSTERS only (kr_huge.cuh): the RayClusters of more than KR_LARGE_MAX_PODS pods —
//                    List order by a shared-memory sort per 8 192-rank tile and a rank merge of the tiles, one CTA per tile,
//                    beside the hash; then k_decide_huge (k_decide_large with 512 threads) decides them
//   k_lists_init / k_lists_owner / (radix sort) / k_lists_gather   KR_OPT_BUCKET_POD_LISTS with fetch_pod_lists == 1 only
//                    (kr_lists.cuh): every RayCluster's full pod list in List order from the resident buckets, behind the last decide
// When the caller asks for the full per-cluster pod lists (fetch_pod_lists == 1, without KR_OPT_BUCKET_POD_LISTS) or the snapshot does
// not qualify — the SORT pipeline:
//   k_match -> k_place_fused -> k_decide_small (+ k_decide on a side stream) -> [phase 1] -> k_creates_fused
//   (buckets restored to List order by an in-register bitonic sort), and for RayClusters with > 1024 pods the RADIX pipeline
//   (k_match<radix>, k_hist, k_scan_rows, k_scatter: stable LSD sort) with the unfused scan kernels.
// INCREMENTAL epochs (kr_incr.cuh, included by kr_engine.cu): after a full bucket pass everything stays resident; pod-row commits
// run k_inc_retire on the rows' old values, object commits are diffed on the device (k_inc_objects, then k_inc_refresh for the input
// records of the RayClusters that changed), and the pass is
//   k_inc_admit -> k_decide2<K, inc> over the dirty RayClusters (each warp also packs its changed records for the host).
//   k_patch_pods / k_patch_pod_values (copy stream): rewritten pod rows pulled from the mapped pinned arena / scattered from a staged copy.
//
// Reference semantics restated here are cited per function (paths relative to
// ray-operator/controllers/ray/ in ray-project/kuberay).
#pragma once

#include "kr_common.cuh"
#include "kr_match.cuh"
#include "kr_bucket.cuh"
#include "kr_decide.cuh"
#include "kr_emit.cuh"
#include "kr_bucket2.cuh"
#include "kr_hash.cuh"

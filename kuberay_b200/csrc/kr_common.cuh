// kr_common.cuh — device views of the arenas, layout constants and the small device helpers shared by every kernel.
// Part of the sm_90a kernel set of the batched reconcile engine; see kr_kernels.cuh for the pipeline overview.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/kr_engine.h"

namespace kr {

// ------------------------------------------------------------------------------------------------ device views

struct SnapDev {  // device mirror of kr_snapshot_bufs
  const uint32_t *c_ns_id, *c_name_id;
  const uint64_t *c_uid_hash;
  const uint32_t *c_flags;
  const uint8_t *c_suspend_status, *c_ext_err_kind;
  const uint32_t *c_ext_err_msg_id, *c_group_off, *c_group_cnt;
  const uint64_t *c_json_off;
  const uint32_t *c_json_len;
  const uint8_t *c_old_state;
  const int32_t *c_old_counts;
  const uint8_t *c_old_cond_status, *c_old_cond_variant;
  const uint32_t *c_old_cond_reason_id, *c_old_cond_msg_id, *c_old_head_ids;
  const uint8_t *c_svc_count, *c_svc_ip_kind;
  const uint32_t *c_svc_ip_id, *c_svc_name_id;
  const uint32_t *g_cluster_idx, *g_name_id;
  const int32_t *g_replicas, *g_min, *g_max, *g_num_hosts;
  const uint32_t *g_flags, *g_wtd_off, *g_wtd_cnt;
  const uint32_t *w_name_id;
  const uint32_t *p_ns_id, *p_cluster_name_id, *p_group_name_id, *p_name_id, *p_packed;
  const int32_t *p_replica_index;
  const uint32_t *p_replica_name_id;
  const uint32_t *h_pod_idx;
  const uint8_t *h_ready_status;
  const uint32_t *h_ready_reason_id, *h_ready_msg_id, *h_pod_ip_id;
  const uint8_t *h_annot_state, *h_version_state, *h_annot_hash;
  const uint32_t *j_ns_id, *j_cluster_name_id, *j_summary_id, *c_summary_id;
  const uint8_t *json;
};

struct ResDev {  // device results arena
  kr_cluster_result *clusters;
  char *hash;
  kr_group_result *groups;
  uint32_t *wtd_pod_idx;  // unsigned for atomicMin; 0xFFFFFFFF == -1 == NotFound
  uint32_t *sorted_pod_idx;
  uint8_t *sorted_action;
  int32_t *create_idx;
  kr_job_result *jobs;
  uint32_t *act_start;    // [n_clusters + 1]
  uint32_t *act_cnt;      // [n_clusters]
  uint32_t *act_pod_idx;  // [n_pods] capacity; n_actions used
  uint8_t *act_code;
  // [0]=extent of create_idx [1]=n_orphans [2]=n_actions [3]=error flags [4]=clusters deferred to decide phase 1
  // bucket pipeline: [6]=pods to create, [8]/[9]=the two arena cursors as ONE 64-bit word (low: extent of the action list, >= [2]
  // because deferred clusters reserve their whole bucket; high: extent of create_idx)
  uint32_t *totals;
};

struct ScratchDev {
  // cluster table, one 16-byte slot per entry: {name id, ns id, name id of worker group 0, cluster idx << 2 | flags}
  // (flags: bit 0 = some worker group has numOfHosts > 1, bit 1 = more than one worker group).  The common case — one worker
  // group — resolves pod -> cluster -> group slot with this single load.
  uint4 *cl_slots; uint32_t cl_mask;
  uint4 *cl_rec;                                               // [n_clusters] {group_off, group_cnt, name id of group 0, bit0 = has a multi-host group}
  uint64_t *wt_keys; uint32_t *wt_head; uint32_t *wt_next; uint32_t wt_mask;  // workersToDelete-name table
  uint32_t *aux_keys; uint32_t *aux_vals; uint32_t aux_mask;   // pod idx -> head-aux row
  uint4 *rows;                                                 // 16-byte pod rows, original order
  uint32_t *keys[2]; uint32_t *vals[2];                        // radix ping-pong
  uint32_t *hist;                                              // [256 * ntiles] digit-major
  uint32_t *row_total;                                         // [256] per-digit totals of the current pass
  uint32_t *gcreate;                                           // [n_groups] dense n_create (input of the creates scan)
  uint32_t *cact;                                              // [n_clusters] pods with an action per cluster (input of the action-list scan)
  uint32_t *mh_rep, *mh_name, *mh_meta, *mh_cnt, *mh_flg;      // multi-host scratch, indexed by sorted position
  uint8_t *mh_act, *mh_head;                                   // per position: action of a multi-host pod / first pod of a valid replica
  uint32_t *act_tmp_idx; uint8_t *act_tmp_code;                // per cluster, from its pod_start: the pods it acts on (compacted by the decide warp)
  uint32_t *tile_orph;                                         // fast pipeline: orphans per k_match tile -> exclusive prefix
  uint32_t *chain;                                             // chained-scan hand-off cells {ready, carry} (zeroed with ccount)
  uint32_t *ccount, *cstart;                                   // fast pipeline: pods per cluster bucket [n_clusters+1], bucket starts [n_clusters+2]
  uint32_t *deferred_list;                                     // clusters left for decide phase 1 (count in totals[4])
  int32_t *gacc;                                               // [4 * n_groups] spill accumulators (clusters with > KR_SMEM_GROUPS groups)
  // bucket pipeline (kr_bucket2.cuh)
  uint2 *bucket; uint32_t bucket_stride;                       // [n_clusters * stride] {pod idx, slot << 16 | flags}, arrival order (the replica index and
                                                               // the name are read from the Pod columns where they are used)
  uint32_t *wt_bits; uint32_t wt_bits_mask;                    // Bloom bitmap over the workersToDelete (ns, name) keys (power-of-two bit count)
  uint32_t *cl_in;                                             // [32 * n_clusters] every per-cluster input of the decide kernel as ONE 128-byte record (KR_CI_*)
  uint4 *cl_dyn;                                               // [n_clusters] {pods bucketed so far, incremental epoch in which the cluster LOST a row (its bucket must be
                                                               // compacted), ~(first head's pod idx << 32 | head-aux row + 1)}, zeroed every full pass
  // device-side incremental epochs (kr_incr.cuh): the buckets, cl_dyn, cl_in, the tables and the results stay resident between passes
  uint32_t *stamp;                                             // [n_pods] epoch in which the row was last touched (retired) by a pod commit
  uint32_t *touched;                                           // [n_pods] rows touched since the last pass (each once), count in inc[KR_INC_TOUCHED]
  uint32_t *touched_old;                                       // [n_pods] per touched entry: the RayCluster the row was in before the commit (KR_EMPTY32: none)
  uint32_t *pos;                                               // [n_pods] where the row's record sits in its RayCluster's bucket (k_match2, k_inc_admit, phase-2 compaction)
  uint32_t *dirty_flag;                                        // [n_clusters] epoch in which the RayCluster was last marked dirty
  uint32_t *obj_flag;                                          // [n_clusters] epoch in which an object commit changed one of its rows (its input record is rewritten)
  uint32_t *dirty_list;                                        // [n_clusters] RayClusters to decide again, count in inc[KR_INC_DIRTY]
  uint32_t *act_res, *cre_res;                                 // [n_clusters] places the cluster holds in the action list / create arena (reused while they suffice)
  uint32_t *inc;                                               // [16] counters / flags of the running epoch (KR_INC_*)
  // large RayClusters (KR_OPT_LARGE_CLUSTERS, kr_large.cuh): records of arrival rank >= bucket_stride go to the cluster's region
  uint4 *lg;                                                   // [n_clusters] {region offset, region capacity (0: not large), scratch segment, kept pods | KR_LG_OWNED}; nullptr: none
  uint2 *region;                                               // large-cluster record arena (8-byte bucket records)
};
enum {
  KR_INC_TOUCHED = 0, KR_INC_DIRTY = 1,
  KR_INC_STRUCTURAL = 2,   // an object commit changed a table key / CSR offset: the resident tables are stale, take a full pass (KR_FULL_STRUCTURAL)
  KR_INC_EPOCH = 3,        // epochs completed; stamps / dirty flags of the running epoch carry this + 1
  KR_INC_HEADS = 4,        // the pod idx -> head-aux row table must be rebuilt
  KR_INC_VOID = 5,         // the incremental attempt is void (a bucket or an arena overflowed): take a full pass.  Both words hold the
                           // KR_FULL_* bits of their causes (atomicOr; readers test them for non-zero) for kr_last_pass
  KR_INC_GROUPS = 6,       // gather: group records staged so far
  KR_INC_LSEG = 7,         // large RayClusters: scratch positions handed out so far (k_large_sort)
  KR_INC_GROW = 8,         // KR_OPT_LARGE_GROWTH: RayClusters k_inc_admit put on the grow list (k_inc_grow, kr_incr.cuh)
  KR_INC_SPILL = 9,        // ... records it spilled for them
  KR_INC_GROWN = 10,       // ... entries of k_inc_grow's result (0: nothing grew, or the epoch is void)
};
// words of a cl_in record (built by k_build_tables; k_decide2 loads it with one coalesced 128-byte access, lane i = word i)
enum {
  KR_CI_FLAGS = 0, KR_CI_GOFF = 1, KR_CI_GCNT = 2,
  KR_CI_B0 = 3,   // bytes: suspend_status, ext_err_kind, old_state, svc_count
  KR_CI_B1 = 4,   // bytes: svc_ip_kind, old_cond_status[0..2]
  KR_CI_B2 = 5,   // bytes: old_cond_status[3..4], old_cond_variant[0..1]
  KR_CI_B3 = 6,   // bytes: old_cond_variant[2..4], -
  KR_CI_EXT_MSG = 7, KR_CI_CNT = 8 /* ..12 */, KR_CI_REASON = 13, KR_CI_MSG = 14 /* ..15 */, KR_CI_HEAD = 16 /* ..19 */,
  KR_CI_SVC_IP = 20, KR_CI_SVC_NAME = 21,
  KR_CI_G0_FLAGS = 22, KR_CI_G0_REP = 23, KR_CI_G0_MIN = 24, KR_CI_G0_MAX = 25, KR_CI_G0_HOSTS = 26  // worker group 0 (when group_cnt >= 1)
};
#define KR_CL_MH 1u      // cl_slots[].w flag bits
#define KR_CL_MULTI 2u

struct Sizes { uint32_t n_clusters, n_groups, n_wtd, n_pods, n_heads, n_jobs; };

// row.w layout: low 16 bits = p_packed low bits (+ KR_ROW_WTD_OWN), high 16 bits = group slot inside the cluster
#define KR_ROW_WTD_OWN (1u << 11)   // named by its own group's scaleStrategy.workersToDelete
#define KR_ROW_NO_GROUP 0xFFFFu
// Fast pipeline only: once a bucket too large for the in-warp sort was met (k_place_fused / k_scan_counts set the flag), the
// rest of this attempt is void — its buckets are not in List order and sorted_pod_idx is not written for the big ones — and the
// engine reruns the pass on the radix pipeline.  Every later kernel of the attempt leaves at once instead of chasing
// uninitialised indices.
// (load the word early with KR_ATTEMPT_WORD so it travels with the kernel's first real loads, test it with KR_WORD_VOID)
// The word read here sits 128 bytes into the totals block, away from the counters the decide warps update with atomics (reading
// totals[3] itself from every warp serialised on that hot sector and slowed k_decide_small).
#define KR_TOTALS_VOID_WORD 32
#define KR_ATTEMPT_WORD(totals) __ldcg(&(totals)[KR_TOTALS_VOID_WORD])
#define KR_WORD_VOID(w) ((w) != 0)
#define KR_MARK_ATTEMPT_VOID(totals) do { atomicOr(&(totals)[3], KR_TOTALS_BIG_BUCKET); (totals)[KR_TOTALS_VOID_WORD] = 1u; } while (0)
#define KR_ATTEMPT_VOID(totals) KR_WORD_VOID(KR_ATTEMPT_WORD(totals))
#define KR_TOTALS_BIG_BUCKET 2u        // fast pipeline only: some cluster (or the orphan bucket) holds more pods than the in-warp sort takes
#define KR_TOTALS_HASH_WAIT 4u         // bucket pipeline: a decide warp gave up waiting for a digest of the concurrently running hash kernel
                                       // (the engine reruns the pass with the two-phase schedule)


static constexpr int kSortThreads = 256;
static constexpr int kSortItems = 8;
static constexpr int kSortTile = kSortThreads * kSortItems;  // 2048 keys per tile
static constexpr int kMatchItems = 2;                        // fast pipeline: pods per thread in k_match (tile = 512 pods; occupancy beats per-thread ILP here)
static constexpr int kMatchTile = kSortThreads * kMatchItems;
static constexpr int kRadixBits = 8;
static constexpr int kRadix = 1 << kRadixBits;

// ------------------------------------------------------------------------------------------------ small helpers
#ifdef KR_TIMELINE
// Development aid (tools/timeline.py, built with -DKR_TIMELINE into a separate library): every kernel stamps the earliest
// block start and the latest block end it sees (%globaltimer, ns) so the gaps between the kernels of one graph replay show.
__device__ unsigned long long g_tl[64];
struct TlScope {
  int id;
  __device__ __forceinline__ static unsigned long long now() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
  __device__ __forceinline__ explicit TlScope(int i) : id(i) { if (threadIdx.x == 0) atomicMin(&g_tl[2 * id], now()); }
  __device__ __forceinline__ ~TlScope() { if (threadIdx.x == 0) atomicMax(&g_tl[2 * id + 1], now()); }
};
#define KR_TL(id) TlScope tl_scope_(id)
#define KR_TL_POINT(id) do { if (threadIdx.x == 0) { unsigned long long t_ = TlScope::now(); atomicMin(&g_tl[2 * (id)], t_); atomicMax(&g_tl[2 * (id) + 1], t_); } } while (0)
#else
#define KR_TL(id)
#define KR_TL_POINT(id)
#endif

__device__ __forceinline__ uint64_t mix64(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
  return x;
}
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}
__device__ __forceinline__ uint64_t key2(uint32_t a, uint32_t b) { return ((uint64_t)a << 32) | b; }
// slot hash of an (a, b) id pair: two 32-bit multiplies + one finalizer (the tables are small and 2x over-provisioned)
__device__ __forceinline__ uint32_t hash_pair(uint32_t a, uint32_t b) { return mix32(a * 0x9E3779B1u ^ (b * 0x85EBCA77u + 0x165667B1u)); }
// second Bloom position of a workersToDelete key (k = 2: with 64 bits per name the false-positive rate drops from 2.3 % to 0.2 %, and a
// false positive costs a warp two dependent L2 round trips in the name table)
__device__ __forceinline__ uint32_t bloom2(uint32_t hk) { return (hk * 0x9E3779B1u) >> 9; }
#define KR_EMPTY64 0xFFFFFFFFFFFFFFFFull
#define KR_EMPTY32 0xFFFFFFFFu

// Programmatic dependent launch (PDL): a kernel launched with the programmatic-serialization attribute may be scheduled while
// its stream predecessor is still running; it must not touch the predecessor's outputs before pdl_wait().  Both are no-ops
// for ordinary launches.  pdl_trigger() lets the NEXT kernel in the chain be scheduled early.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ uint32_t lanemask_lt() { uint32_t m; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m; }

__device__ __forceinline__ uint32_t pp_node_type(uint32_t f) { return (f >> KR_PP_NODE_TYPE_SHIFT) & 3u; }
__device__ __forceinline__ uint32_t pp_phase(uint32_t f) { return (f >> KR_PP_PHASE_SHIFT) & 7u; }
__device__ __forceinline__ uint32_t pp_ready(uint32_t f) { return (f >> KR_PP_READY_SHIFT) & 3u; }

// shouldDeletePod (raycluster_controller.go:1181-1231)
__device__ __forceinline__ bool should_delete(uint32_t f) {
  uint32_t ph = pp_phase(f);
  return ph == KR_PHASE_FAILED || ph == KR_PHASE_SUCCEEDED ||
         (ph == KR_PHASE_RUNNING && (f & KR_PP_RAY_TERMINATED) && (f & KR_PP_RESTART_NEVER));
}

// utils.GetWorkerGroupDesiredReplicas (utils/util.go:386-404); int32 multiply wraps like Go's
__device__ __forceinline__ int32_t desired_replicas(int32_t replicas, int32_t mn, int32_t mx, int32_t hosts, uint32_t gf) {
  int32_t minr = (gf & KR_GF_MIN_NIL) ? 0 : mn;
  int32_t maxr = (gf & KR_GF_MAX_NIL) ? INT32_MAX : mx;
  if (gf & KR_GF_SUSPEND) return 0;
  int32_t w;
  if ((gf & KR_GF_REPLICAS_NIL) || replicas < minr) w = minr;
  else if (replicas > maxr) w = maxr;
  else w = replicas;
  return (int32_t)((uint32_t)w * (uint32_t)hosts);
}

__device__ __forceinline__ bool cl_lookup(const ScratchDev &sc, uint32_t ns, uint32_t name, uint32_t &out) {
  if (name == 0) return false;
  uint32_t i = hash_pair(ns, name) & sc.cl_mask;
  while (true) {
    uint4 sl = __ldg(&sc.cl_slots[i]);  // one 16-byte load: key and value together
    if (sl.x == name && sl.y == ns) { out = sl.w >> 2; return true; }
    if (sl.x == KR_EMPTY32 && sl.y == KR_EMPTY32) return false;
    i = (i + 1) & sc.cl_mask;
  }
}

}  // namespace kr

// kr_bucket2.cuh — the bucket pipeline: k_match2 + k_decide2, the production path of a pass whose caller does not ask for the
// full per-cluster pod lists (kr_flags.fetch_pod_lists == 0).
// Part of the sm_90a kernel set of the batched reconcile engine; see kr_kernels.cuh for the pipeline overview.
//
// The sort pipeline (k_match -> k_place_fused -> k_decide_small -> k_creates_fused) spends most of its time restoring informer
// List order inside every RayCluster's bucket — a scan + placement kernel, a 16-byte row gather and an in-register bitonic sort
// per cluster — although the reference only looks at that order in three places: the head pod is the FIRST head listed
// (common/association.go:184-196), a scale-down deletes the first -diff running pods (raycluster_controller.go:916-919), and
// the Delete calls are issued in List order.  Everything else (selectors, counts, the unhealthy / workersToDelete sets, the
// lowest free replica indices, the status roll-up) is a set computation.  So here
//   k_match2   drops each pod's 8-byte record {pod idx, group slot | flags} straight into its
//              cluster's fixed-stride bucket at the arrival rank a returning atomic hands out: no scan, no placement pass, no
//              row array — three scattered accesses per pod (table probe, atomic, record store) instead of four plus a gather;
//   k_decide2  (one warp per RayCluster, bucket in registers, ARRIVAL order) takes the first head as a warp minimum over pod
//              indices, the ordered delete prefix by extracting the -diff smallest indices (warp min-reduce per victim; a
//              counting rank for long prefixes) and orders only the handful of pods that carry an action; it also allocates the
//              replica indices from the registers and reserves its places in the action list / create arena with one returning
//              atomic, so nothing follows it: no scan, no creates kernel, no compaction kernel.
// A bucket stride too small for some cluster voids the attempt (the engine widens the stride or falls back to the sort
// pipeline).  k_decide2 leaves every RayCluster of more than KR_SMEM_GROUPS worker groups alone: with KR_OPT_WIDE_CLUSTERS the
// per-cluster kernels of kr_large.cuh decide them, without it the host routes such a snapshot to the sort pipeline before the
// pass.  Multi-host worker groups (numOfHosts > 1 under the RayMultiHostIndexing gate) are decided here too, by the
// k_decide2<K, kInc, true> instantiations the engine launches only when the snapshot has such a group (decide_multihost2).
#pragma once

#include "kr_decide.cuh"

namespace kr {

__device__ __forceinline__ uint32_t inc_epoch_of(const ScratchDev &sc) { return __ldcg(&sc.inc[KR_INC_EPOCH]) + 1u; }  // stamp value of the running incremental epoch (kr_incr.cuh)

#ifndef KR_D2WARPS
#define KR_D2WARPS 8
#endif
static constexpr int kD2Warps = KR_D2WARPS;  // RayClusters per k_decide2 CTA
#define KR_ROW_UNHEALTHY (1u << 13)  // bucket record word: shouldDeletePod(pod) (k_match2 evaluates it once per pod)
#define KR_ROW_FRESH (1u << 14)      // bucket record word: appended by k_inc_admit in the running incremental epoch (cleared by the decide warp)
#define KR_LG_OWNED (1u << 31)       // lg[c].w: k_large_sort took the RayCluster this pass (the low bits are its kept pod count)

// Where the record of arrival rank `rank` >= bucket_stride of RayCluster c goes: its region of the large-cluster arena
// (KR_OPT_LARGE_CLUSTERS, kr_large.cuh), which holds ranks [stride, stride + capacity).  nullptr: no room (an ordinary RayCluster,
// or a large one that outgrew its region): the attempt is void.  Ranks below the stride stay in the cluster's bucket, so an
// ordinary pod never reaches this lookup.
__device__ __forceinline__ uint2 *large_slot(const ScratchDev &sc, uint32_t c, uint32_t rank) {
  if (!sc.lg) return nullptr;
  const uint4 l = __ldcg(&sc.lg[c]);
  const uint32_t j = rank - sc.bucket_stride;
  return j < l.y ? sc.region + l.x + j : nullptr;
}
__device__ __forceinline__ uint2 *rec_slot(const ScratchDev &sc, uint32_t c, uint32_t rank) {
  return rank < sc.bucket_stride ? sc.bucket + (size_t)c * sc.bucket_stride + rank : large_slot(sc, c, rank);
}
// Region capacity of a RayCluster of `count` pods at this stride: 1.25x its pods rounded up to 32, capped at KR_LARGE_MAX_PODS unless
// the cluster is huge, less the stride (the full pass's reclassification and k_inc_grow both size regions by it)
__host__ __device__ __forceinline__ uint32_t large_region_cap(uint32_t count, uint32_t stride) {
  const uint32_t want = ((count + count / 4 + 31) / 32) * 32;
  return (count > KR_LARGE_MAX_PODS ? want : (want < KR_LARGE_MAX_PODS ? want : (uint32_t)KR_LARGE_MAX_PODS)) - stride;
}


// ------------------------------------------------------------------------------------------------ k_match2
// The selector match (common/association.go:83-130) + bucketing.  5 coalesced column loads per pod (issued before the
// programmatic-launch wait: they do not depend on the table build), one 16-byte probe of the cluster table (which also
// carries the name of worker group 0, so a single-group RayCluster needs no second lookup), a shared-memory Bloom test
// for the workersToDelete names, one returning atomic and one 8-byte record store.  The record leaves out the replica index and the
// name: k_decide2 reads them from the Pod columns for the few pods that need them (the head's name, the replica indices in use of a
// RayCluster that creates), and the bucket arena is half the size (C3: 8 MB written and read back instead of 16 MB).
template <int kItems>
__global__ void __launch_bounds__(kSortThreads) k_match2(SnapDev s, ScratchDev sc, ResDev r, Sizes n, int has_wtd) {
  KR_TL(1);
  extern __shared__ uint32_t sm_bits[];  // copy of the workersToDelete Bloom bitmap
  __shared__ uint32_t s_orph[kSortThreads / 32];
  const uint32_t tile = blockIdx.x;
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t base = tile * (kSortThreads * kItems) + warp * (32 * kItems) + lane;
  uint32_t ns[kItems], cn[kItems], gn[kItems], nm[kItems], pk[kItems];
#pragma unroll
  for (int it = 0; it < kItems; it++) {
    const uint32_t p = base + it * 32;
    const bool v = p < n.n_pods;
    ns[it] = v ? __ldg(&s.p_ns_id[p]) : 0u; cn[it] = v ? __ldg(&s.p_cluster_name_id[p]) : 0u;
    gn[it] = v ? __ldg(&s.p_group_name_id[p]) : 0u; nm[it] = v ? __ldg(&s.p_name_id[p]) : 0u;
    pk[it] = v ? __ldg(&s.p_packed[p]) : 0u;
  }
  pdl_wait(); pdl_trigger();
  // (Keep this wait unconditional and in straight-line code: the table probes below use __ldg, i.e. loads the compiler treats as
  //  invariant, and the tables are being written by the predecessor grid until the wait returns.  A persistent-CTA variant with the
  //  wait inside `if (first tile)` had its probes hoisted above it and matched nothing; peeling the first tile fixed that but was
  //  slower in the graph than this one-tile-per-CTA form, so it was dropped.)
  // hash-join probe (namespace, ray.io/cluster) -> slot; the first probe of every pod goes out before anything waits
  uint32_t pi[kItems];
  uint4 sl[kItems];
#pragma unroll
  for (int it = 0; it < kItems; it++) {
    pi[it] = hash_pair(ns[it], cn[it]) & sc.cl_mask;
    sl[it] = __ldg(&sc.cl_slots[pi[it]]);
  }
  if (has_wtd) {
    const uint32_t words = (sc.wt_bits_mask + 1) >> 5;
    for (uint32_t i = threadIdx.x; i < words; i += kSortThreads) sm_bits[i] = __ldcg(&sc.wt_bits[i]);
    __syncthreads();
  }
  uint32_t orphans = 0;
  uint32_t cidx[kItems], roww[kItems];  // cluster idx (n_clusters: none) and the record word (slot << 16 | flags) of every pod
#pragma unroll
  for (int it = 0; it < kItems; it++) {
    const uint32_t p = base + it * 32;
    const bool v = p < n.n_pods;
    uint32_t c = n.n_clusters, cflags = 0, gname0 = 0;
    if (cn[it] != 0) {
      uint4 q = sl[it];
      uint32_t i = pi[it];
      while (true) {
        if (q.x == cn[it] && q.y == ns[it]) { c = q.w >> 2; cflags = q.w & 3u; gname0 = q.z; break; }
        if (q.x == KR_EMPTY32 && q.y == KR_EMPTY32) break;
        i = (i + 1) & sc.cl_mask;
        q = __ldg(&sc.cl_slots[i]);
      }
    }
    const bool matched = v && c < n.n_clusters;
    // ray.io/group against the cluster's worker groups (group names are unique: pkg/webhooks/v1/raycluster_webhook.go:74)
    uint32_t slot = KR_ROW_NO_GROUP, g0 = 0xFFFFFFFFu;
    if (matched && gn[it] != 0) {
      if (gname0 == gn[it]) slot = 0;
      else if (cflags & KR_CL_MULTI) {
        const uint4 rec = __ldg(&sc.cl_rec[c]);
        g0 = rec.x;
        for (uint32_t gi = 1; gi < rec.y; gi++)
          if (__ldg(&s.g_name_id[g0 + gi]) == gn[it]) { slot = gi; break; }
      }
    }
    uint32_t flags = pk[it] & (0x7FFu | KR_PP_TOMBSTONE);  // bit 11 of the record word is KR_ROW_WTD_OWN
    if (should_delete(pk[it])) flags |= KR_ROW_UNHEALTHY;  // shouldDeletePod (raycluster_controller.go:1181-1231), once per pod, here
    if (has_wtd && v) {  // scaleStrategy.workersToDelete: Delete(ns, name) (raycluster_controller.go:817-822)
      const uint32_t hk = hash_pair(ns[it], nm[it]);
      const uint32_t h2 = bloom2(hk);
      if ((sm_bits[(hk & sc.wt_bits_mask) >> 5] & (1u << (hk & 31))) && (sm_bits[(h2 & sc.wt_bits_mask) >> 5] & (1u << (h2 & 31)))) {
        const uint64_t k = key2(ns[it], nm[it]);
        uint32_t i = hk & sc.wt_mask;
        uint64_t kk = __ldg(&sc.wt_keys[i]);
        while (kk != KR_EMPTY64) {
          if (kk == k) {
            for (uint32_t e = sc.wt_head[i]; e != KR_EMPTY32; e = sc.wt_next[e]) {
              atomicMin(&r.wtd_pod_idx[e], p);
              if (slot != KR_ROW_NO_GROUP) {  // is e one of this pod's own group's names?
                if (g0 == 0xFFFFFFFFu) g0 = __ldg(&s.c_group_off[c]);
                const uint32_t g = g0 + slot, off = __ldg(&s.g_wtd_off[g]);
                if (e >= off && e < off + __ldg(&s.g_wtd_cnt[g])) flags |= KR_ROW_WTD_OWN;
              }
            }
            break;
          }
          i = (i + 1) & sc.wt_mask;
          kk = __ldg(&sc.wt_keys[i]);
        }
      }
    }
    if (matched && pp_node_type(pk[it]) == KR_NT_HEAD) {
      // the cluster's FIRST head in List order (common/association.go:184-196) and its head-aux row, as one 64-bit maximum of
      // ~(pod idx << 32 | row + 1): the decide warp reads it together with the pod count
      const int32_t aux = aux_lookup(sc, p);
      const unsigned long long key = ((unsigned long long)p << 32) | (uint32_t)(aux + 1);
      atomicMax(reinterpret_cast<unsigned long long *>(&sc.cl_dyn[c].z), ~key);
    }
    cidx[it] = matched ? c : n.n_clusters;
    roww[it] = (slot << 16) | flags;
    orphans += __popc(__ballot_sync(0xFFFFFFFFu, v && !matched && !(pk[it] & KR_PP_TOMBSTONE)));
  }
  // arrival rank inside the cluster's bucket: every atomic of the thread in flight before the first record store needs its rank
  uint32_t rank[kItems];
#pragma unroll
  for (int it = 0; it < kItems; it++) rank[it] = cidx[it] < n.n_clusters ? atomicAdd(&sc.cl_dyn[cidx[it]].x, 1u) : 0u;
#pragma unroll
  for (int it = 0; it < kItems; it++) {
    if (cidx[it] >= n.n_clusters) continue;
    if (rank[it] < sc.bucket_stride) {
      sc.bucket[(size_t)cidx[it] * sc.bucket_stride + rank[it]] = make_uint2(base + it * 32, roww[it]);
      sc.pos[base + it * 32] = rank[it];  // (coalesced; incremental epochs rewrite a row's record in place)
    } else if (uint2 *slot = large_slot(sc, cidx[it], rank[it])) {
      *slot = make_uint2(base + it * 32, roww[it]);
      sc.pos[base + it * 32] = rank[it];
    } else KR_MARK_ATTEMPT_VOID(r.totals);  // the engine reruns the pass with a wider stride / large regions / on the sort pipeline
  }
  // pods that match no RayCluster of the snapshot (free rows of an incrementally maintained arena are not orphans)
  if (lane == 0) s_orph[warp] = orphans;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
#pragma unroll
    for (int w = 0; w < kSortThreads / 32; w++) t += s_orph[w];
    if (t) atomicAdd(&r.totals[1], t);
  }
}

// ------------------------------------------------------------------------------------------------ k_decide2

// Incremental epochs: the changed records, packed for one small D2H copy — per dirty cluster {idx, act_start, act_cnt, group_off,
// group_cnt, first staged group record}, its kr_cluster_result, and its groups' kr_group_result records back to back.  Entry i belongs
// to dirty_list[i]; the decide warp of that cluster writes it when it is done (k_decide2<K, true>).
struct IncStage { uint32_t *meta; kr_cluster_result *clusters; kr_group_result *groups; uint32_t cap_clusters, cap_groups; };

struct Decide2Args {
  SnapDev s; ScratchDev sc; ResDev r; Sizes n; kr_flags f;
  IncStage st;  // phase 2 only
  uint32_t create_cap;
  int spin_hash;  // phase 0: a cluster whose Recreate gate reads a digest waits for the concurrently running hash kernel (no phase 1)
  int phase;  // 0: every RayCluster; 1: only the clusters phase 0 deferred (Recreate gate waiting for the hash kernel);
              // 2: only the clusters an incremental epoch marked dirty (kr_incr.cuh) — digests resident, places reused while they suffice
};

// Incremental epochs: the records of RayCluster c (entry i of the dirty list) as they now stand in the result arrays, packed at its
// place in the staging buffer by one warp (the host copies the whole arrays instead when the list outgrew the staging area).
__device__ __forceinline__ void stage_cluster(const Decide2Args &a, uint32_t i, uint32_t c, uint32_t act_off, uint32_t n_act, uint32_t g0, uint32_t G, uint32_t lane) {
  const uint32_t n_dirty = __ldcg(&a.sc.inc[KR_INC_DIRTY]);
  if (n_dirty > a.st.cap_clusters) return;
  uint32_t at = 0;
  if (lane == 0) at = atomicAdd(&a.sc.inc[KR_INC_GROUPS], G);
  at = __shfl_sync(0xFFFFFFFFu, at, 0);
  if (lane == 0) {
    uint32_t *m = a.st.meta + 8 * (size_t)i;
    m[0] = c; m[1] = act_off; m[2] = n_act; m[3] = g0; m[4] = G; m[5] = at; m[6] = 0; m[7] = 0;
  }
  static_assert(sizeof(kr_cluster_result) % 4 == 0 && sizeof(kr_cluster_result) / 4 <= 32 && sizeof(kr_group_result) % 4 == 0, "record sizes");
  const uint32_t *csrc = reinterpret_cast<const uint32_t *>(&a.r.clusters[c]);
  uint32_t *cdst = reinterpret_cast<uint32_t *>(&a.st.clusters[i]);
  if (lane < sizeof(kr_cluster_result) / 4) cdst[lane] = __ldcg(csrc + lane);
  if ((uint64_t)at + G <= a.st.cap_groups) {
    const uint32_t words = G * (uint32_t)(sizeof(kr_group_result) / 4);
    const uint32_t *gsrc = reinterpret_cast<const uint32_t *>(&a.r.groups[g0]);
    uint32_t *gdst = reinterpret_cast<uint32_t *>(&a.st.groups[at]);
    for (uint32_t w = lane; w < words; w += 32) gdst[w] = __ldcg(gsrc + w);
  }
}

// reconcileMultiHostWorkerGroup (raycluster_controller.go:963-1125) for worker group `gi` of the warp's RayCluster, from the
// registers of k_decide2 — the decisions of decide_multihost (kr_decide.cuh), which the sort pipeline takes, bit for bit.
// A replica is the set of the group's pods sharing a ray.io/worker-group-replica-name; it is identified by its smallest pod index,
// so ascending identity is "first appearance in List order" (the stand-in for the reference's Go-map iteration) although the
// bucket is in arrival order.  Replicas are peeled off in that order (a warp minimum over the unassigned members, then a compare
// of its name against the K registers): O(replicas x K) warp steps.  The replica-name id is not in the 8-byte bucket record; it
// is read from the pod column here, for the group's members only (an incremental epoch patches that column before this kernel).
// The group's per-pod actions go straight into act[]; mh_head gets bit k for every pod that is the first pod of a healthy
// replica (its replica index is "in use" for the creates); s_rep (>= 32*K words of the warp's shared memory) holds the
// per-replica flags.  Returns the KR_ERR_* kind (0 = nil).
template <int K>
__device__ __forceinline__ int decide_multihost2(const SnapDev &s, uint32_t gi, int32_t expected, int32_t H, bool delete_allowed, uint32_t wtd_cnt,
                                                 const uint32_t (&pidx)[K], const uint32_t (&pw)[K], uint32_t (&act)[K], uint32_t &mh_head,
                                                 uint32_t *s_rep, kr_group_result &gr, int32_t &err_arg, uint32_t lane) {
  const uint32_t lt = lanemask_lt();
  uint32_t rep[K];  // the pod's replica-name id until its replica is identified, then the replica's ordinal (identity order)
  uint32_t todo = 0, noname = 0;  // bit k: member with the label whose replica is not identified yet / member without the label
#pragma unroll
  for (int k = 0; k < K; k++) {
    const bool member = (pw[k] >> 16) == gi;  // (an empty register has no group)
    rep[k] = member ? __ldg(&s.p_replica_name_id[pidx[k]]) : 0u;
    if (member) { if (rep[k]) todo |= 1u << k; else noname |= 1u << k; }
  }
  const uint32_t labelled = todo;
  // 1. replicaMap (:967-972); 2. the first incomplete replica in identity order aborts the group (:975-984)
  uint32_t n_rep = 0, r_empty = KR_MH_NONE, heads = 0;
  while (__any_sync(0xFFFFFFFFu, todo)) {
    uint32_t m = 0xFFFFFFFFu, mname = 0;
#pragma unroll
    for (int k = 0; k < K; k++) if (((todo >> k) & 1u) && pidx[k] < m) { m = pidx[k]; mname = rep[k]; }
    const uint32_t wm = __reduce_min_sync(0xFFFFFFFFu, m);
    const uint32_t name = __shfl_sync(0xFFFFFFFFu, mname, __ffs(__ballot_sync(0xFFFFFFFFu, m == wm)) - 1);
    uint32_t count = 0, mine = 0;
#pragma unroll
    for (int k = 0; k < K; k++) {
      const bool hit = ((todo >> k) & 1u) && rep[k] == name;
      if (hit) { rep[k] = n_rep; mine |= 1u << k; if (pidx[k] == wm) heads |= 1u << k; }
      count += __popc(__ballot_sync(0xFFFFFFFFu, hit));
    }
    todo &= ~mine;
    if ((int64_t)count < (int64_t)H) {
#pragma unroll
      for (int k = 0; k < K; k++) if ((mine >> k) & 1u) act[k] = KR_ACT_DELETE_MH_INCOMPLETE;
      gr.flags |= KR_GR_ABORTED; err_arg = (int32_t)count;
      return KR_ERR_MH_INCOMPLETE;
    }
    if (name == KR_ID_EMPTY_STRING) r_empty = n_rep;
    n_rep++;
  }
  for (uint32_t r = lane; r < n_rep; r += 32) s_rep[r] = 0;
  __syncwarp();
  // 3. unhealthy replicas (:987-1007): a pod marks its replica; unlabelled pods resolve to the "" replica if one exists
#pragma unroll
  for (int k = 0; k < K; k++) {
    if ((((labelled | noname) >> k) & 1u) && (pw[k] & KR_ROW_UNHEALTHY)) {
      const uint32_t r = ((noname >> k) & 1u) ? r_empty : rep[k];
      if (r != KR_MH_NONE) atomicOr(&s_rep[r], KR_MHF_DELETED);
    }
  }
  __syncwarp();
  int32_t n_unh = 0;
#pragma unroll
  for (int k = 0; k < K; k++) {
    const bool hit = ((labelled >> k) & 1u) && (s_rep[rep[k]] & KR_MHF_DELETED);
    if (hit) act[k] = KR_ACT_DELETE_MH_UNHEALTHY;
    n_unh += __popc(__ballot_sync(0xFFFFFFFFu, hit));
  }
  gr.n_unhealthy = n_unh;
  // 4. explicit deletions from the autoscaler (:1010-1038): whole replicas
  if (wtd_cnt > 0) {
#pragma unroll
    for (int k = 0; k < K; k++) {
      if ((((labelled | noname) >> k) & 1u) && (pw[k] & KR_ROW_WTD_OWN)) {
        const uint32_t r = ((noname >> k) & 1u) ? r_empty : rep[k];
        if (r != KR_MH_NONE) atomicOr(&s_rep[r], KR_MHF_WTD);
      }
    }
    __syncwarp();
    int32_t n_del = 0;
#pragma unroll
    for (int k = 0; k < K; k++) {
      const bool hit = ((labelled >> k) & 1u) && (s_rep[rep[k]] & KR_MHF_WTD);
      if (hit && act[k] == KR_ACT_KEEP) act[k] = KR_ACT_DELETE_MH_WTD;
      n_del += __popc(__ballot_sync(0xFFFFFFFFu, hit));
    }
    gr.flags |= KR_GR_WTD_EXECUTED;
    if (n_del > 0) { gr.flags |= KR_GR_ABORTED; err_arg = n_del; return KR_ERR_MH_WTD; }
  }
  // 5. diff by replica (:1042-1064): healthy (complete) replicas are running
  int32_t running = 0;
  for (uint32_t r = lane; r < n_rep; r += 32) running += (s_rep[r] & KR_MHF_DELETED) ? 0 : 1;
  running = __reduce_add_sync(0xFFFFFFFFu, running);
#pragma unroll
  for (int k = 0; k < K; k++) if (((heads >> k) & 1u) && !(s_rep[rep[k]] & KR_MHF_DELETED)) mh_head |= 1u << k;
  gr.n_running = running;
  if (expected % H != 0) { gr.flags |= KR_GR_ABORTED; err_arg = expected; return KR_ERR_MH_NOT_MULTIPLE; }
  const int32_t to_create = expected / H - running;
  gr.diff = to_create;
  if (to_create > 0) gr.n_create = (uint32_t)to_create;  // replica groups; the creates below allocate one replica index each
  else if (to_create < 0) {
    if (delete_allowed) {  // :1104-1118 — the first -to_create healthy replicas in identity order
      const int32_t remove = -to_create;
      int32_t seen = 0;
      for (uint32_t b = 0; b < n_rep && seen < remove; b += 32) {
        const uint32_t r = b + lane;
        const bool ok = r < n_rep && !(s_rep[r] & KR_MHF_DELETED);
        const uint32_t bal = __ballot_sync(0xFFFFFFFFu, ok);
        if (ok && seen + (int32_t)__popc(bal & lt) < remove) s_rep[r] |= KR_MHF_SCALE;
        seen += __popc(bal);
      }
      __syncwarp();
#pragma unroll
      for (int k = 0; k < K; k++) if (((labelled >> k) & 1u) && (s_rep[rep[k]] & KR_MHF_SCALE)) act[k] = KR_ACT_DELETE_MH_SCALE_DOWN;
    } else gr.flags |= KR_GR_RANDOM_DELETE_OFF;
  }
  return KR_ERR_NONE;
}

// reconcilePods (raycluster_controller.go:619-935) + calculateStatus (:1552-1719) for one RayCluster whose bucket (<= 32*K pods,
// arrival order) sits in registers.
// kInc: the instantiation an incremental epoch launches (phase 2 only); the instantiation of the full pass carries none of its code.
// kMH: the snapshot has a multi-host worker group and the RayMultiHostIndexing gate is on — only these instantiations carry the
// multi-host branch (decide_multihost2), so the common path keeps its register budget.  They run at half the occupancy of the
// K <= 4 common path: with the replica peel in the 64-register budget the compiler spills.
template <int K, bool kInc = false, bool kMH = false>
__global__ void __launch_bounds__(kD2Warps * 32, (K <= 4 && !kMH ? 32 : 16) / kD2Warps) k_decide2(Decide2Args a) {
  const int phase = kInc ? 2 : a.phase;
  KR_TL(phase ? 12 : 3);
  __shared__ int32_t s_acc[kD2Warps][3][KR_SMEM_GROUPS];   // n_list, n_unhealthy, n_wtd_own per group
  __shared__ int32_t s_mode[kD2Warps][kMH ? 4 : 3][KR_SMEM_GROUPS];  // mode, delete-prefix length, n_create (, n_running of a multi-host group)
  __shared__ uint32_t s_list[kD2Warps][32 * K];            // pod indices being ranked (delete candidates / acted pods); per-replica flags
                                                           // of the multi-host group being decided
  __shared__ uint32_t s_bits[kD2Warps][32];                // 1024-bit window of replica indices in use
  // Per-cluster state that is uniform across the warp sits in the warp's shared memory, not in every lane's registers: the input
  // record (each field one broadcast load), the result record, and two scalars the placement needs.  With that, and with the
  // replica indices and the head's name read from the Pod columns where they are used and the roll-up ahead of the action list,
  // the K <= 4 instantiations fit their 64-register cap (32 warps per SM) without spilling.
  __shared__ uint32_t s_in[kD2Warps][32];                  // the cluster's cl_in record (RecordCI)
  __shared__ kr_cluster_result s_cr[kD2Warps];             // the cluster's kr_cluster_result, built in place
  // two scalars the placement reads, kept out of registers through the decisions
  __shared__ uint32_t s_deferred[kD2Warps];                // phase 0: the Recreate gate waits for phase 1
  __shared__ uint32_t s_old_create[kInc ? kD2Warps : 1];   // phase 2: pods the cluster asked for in the resident results
  const SnapDev &s = a.s;
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t lt = lanemask_lt();
  const uint32_t S = a.sc.bucket_stride;
  uint32_t c = blockIdx.x * kD2Warps + warp;
  // the cluster's inputs: one 128-byte record (lane i = word i), written by k_build_tables — not by the kernel this one waits for
  bool mine = phase == 0 && c < a.n.n_clusters;
  uint32_t in_word = mine ? __ldg(&a.sc.cl_in[32 * (size_t)c + lane]) : 0u;
  pdl_wait(); pdl_trigger();
  if (phase == 1) {  // compact list of the clusters phase 0 deferred
    mine = c < a.r.totals[4];
    if (mine) { c = a.sc.deferred_list[c]; in_word = __ldg(&a.sc.cl_in[32 * (size_t)c + lane]); }
  } else if (kInc) {  // the dirty list of an incremental epoch (input records rewritten by k_inc_prepare: no read-only path)
    mine = c < __ldcg(&a.sc.inc[KR_INC_DIRTY]) && !__ldcg(&a.sc.inc[KR_INC_VOID]) && !__ldcg(&a.sc.inc[KR_INC_STRUCTURAL]);
    if (mine) {
      c = a.sc.dirty_list[c];
      in_word = __ldcg(&a.sc.cl_in[32 * (size_t)c + lane]);  // (rewritten by k_inc_refresh if an object row of the cluster changed)
    }
  }
  s_in[warp][lane] = in_word;
  __syncwarp();
  const RecordCI ci{s_in[warp]};
  if (KR_ATTEMPT_VOID(a.r.totals)) mine = false;
  // A RayCluster of more than KR_SMEM_GROUPS worker groups is k_large_sort / k_decide_large's (KR_OPT_WIDE_CLUSTERS, kr_large.cuh):
  // the lane-per-group arrays below hold 32 groups.  Left before the Recreate deferral, the digest wait and the epoch's compaction.
  if (ci.group_cnt() > KR_SMEM_GROUPS) mine = false;
  // An incremental epoch launches one warp per RayCluster of the snapshot but only the first n_dirty have work: the others leave here
  // (the kernel has no CTA-wide barrier, and `mine` is uniform across a warp) instead of walking the whole decision path predicated off —
  // that walk was 4 M of the 13.8 M warp instructions of a 63 %-dirty epoch and nearly all of a 1 %-dirty one.
  if (kInc && !mine) return;
  // pod count + first head, and the whole bucket beside them (stale records past the count are masked once it is here)
  uint2 *bucket = a.sc.bucket + (size_t)(mine ? c : 0) * S;
  uint4 dyn = make_uint4(0, 0, 0, 0);
  uint2 recs[K] = {};
  if (mine) {
    dyn = __ldcg(&a.sc.cl_dyn[c]);
#pragma unroll
    for (int k = 0; k < K; k++) if ((uint32_t)(k * 32) + lane < S) recs[k] = __ldcg(&bucket[k * 32 + lane]);
  }
  uint32_t P = dyn.x;
  if (P > S) { mine = false; P = 0; }  // k_match2 voided the attempt
  if (kInc) {
    // Incremental epoch: k_inc_admit rewrote the records of rows that stayed in this cluster in place and appended the records of
    // rows that joined it (KR_ROW_FRESH).  Only if the cluster LOST a row (deleted, or now in another cluster: cl_dyn.y carries the
    // epoch) some records are stale — the ones whose row is still stamped: drop them and store the bucket back compacted (arrival
    // order kept, pos[] follows the records that move).  Then take the cluster's first head from what is left.
    const uint32_t epoch = inc_epoch_of(a.sc);
    const bool lost = dyn.y == epoch;
    uint32_t kept = 0, head_min = 0xFFFFFFFFu;
#pragma unroll
    for (int k = 0; k < K; k++) {
      const uint32_t j = k * 32 + lane;
      bool keep = mine && j < P;
      const bool fresh = keep && (recs[k].y & KR_ROW_FRESH);
      if (keep && lost && !fresh) keep = __ldcg(&a.sc.stamp[recs[k].x]) != epoch;
      const uint32_t bal = __ballot_sync(0xFFFFFFFFu, keep);
      if (keep) {
        uint2 rec = recs[k];
        rec.y &= ~KR_ROW_FRESH;
        const uint32_t to = kept + __popc(bal & lt);
        if (fresh || to != j) { bucket[to] = rec; if (to != j) a.sc.pos[rec.x] = to; }
        if (pp_node_type(rec.y & 0xFFFFu) == KR_NT_HEAD) head_min = min(head_min, rec.x);
      }
      kept += __popc(bal);
    }
    head_min = __reduce_min_sync(0xFFFFFFFFu, head_min);
    __syncwarp();
    unsigned long long raw = 0;
    if (mine) {
      if (lane == 0 && head_min != 0xFFFFFFFFu) raw = ~(((unsigned long long)head_min << 32) | (uint32_t)(aux_lookup(a.sc, head_min) + 1));
      raw = __shfl_sync(0xFFFFFFFFu, raw, 0);
      P = kept;
      dyn = make_uint4(kept, 0u, (uint32_t)raw, (uint32_t)(raw >> 32));
      if (lane == 0) a.sc.cl_dyn[c] = dyn;
    }
    // the compacted bucket (every register rewritten, so none of the records read before the compaction stays live past it)
#pragma unroll
    for (int k = 0; k < K; k++) recs[k] = mine && (uint32_t)(k * 32) + lane < kept ? __ldcg(&bucket[k * 32 + lane]) : make_uint2(0, 0);
  }
  const uint32_t cf = ci.flags(), G = ci.group_cnt(), g0 = ci.group_off();
  const uint8_t suspend_status = ci.suspend_status(), ext_err = ci.ext_err_kind(), old_prov = ci.cond_status(KR_COND_PROVISIONED);
  const bool gate = a.f.gate_status_conditions != 0;
  if (kInc && mine) {  // phase 2: pods this cluster asked for in the resident results (they leave the running total)
    uint32_t old_create = 0;
    for (uint32_t gi = lane; gi < G; gi += 32) old_create += a.r.groups[g0 + gi].n_create;
    s_old_create[warp] = __reduce_add_sync(0xFFFFFFFFu, old_create);  // (read by the placement, after the group loop rewrote the records)
  }
  // first head in List order = the smallest pod index among the heads (k_match2), with its head-aux row
  uint32_t head_pod = 0xFFFFFFFFu;
  int32_t head_aux = -1;
  {
    const unsigned long long raw = ((unsigned long long)dyn.w << 32) | dyn.z;
    if (mine && raw != 0) { const unsigned long long key = ~raw; head_pod = (uint32_t)(key >> 32); head_aux = (int32_t)(uint32_t)key - 1; }
  }
  // what the decisions need from the head-aux table goes out now, beside the bucket
  uint8_t h_ver = KR_VER_EMPTY, h_ast = KR_ANNOT_EMPTY;
  if (head_aux >= 0 && (cf & KR_CF_UPGRADE_RECREATE)) { h_ver = s.h_version_state[head_aux]; h_ast = s.h_annot_state[head_aux]; }
  uint32_t pidx[K], pw[K], act[K];
  uint32_t head_pos = 0xFFFFFFFFu, head_flags = 0;  // (the head's name is read from its bucket record by the roll-up)
#pragma unroll
  for (int k = 0; k < K; k++) {
    const uint32_t i = k * 32 + lane;
    const bool valid = i < P;
    pidx[k] = valid ? recs[k].x : 0xFFFFFFFFu; pw[k] = valid ? recs[k].y : (KR_ROW_NO_GROUP << 16); act[k] = KR_ACT_KEEP;
    const uint32_t hit = __ballot_sync(0xFFFFFFFFu, valid && recs[k].x == head_pod);
    if (hit) {
      const int src = __ffs(hit) - 1;
      head_pos = k * 32 + src;
      head_flags = __shfl_sync(0xFFFFFFFFu, recs[k].y, src) & 0xFFFFu;
    }
  }
  int32_t *acc_list = s_acc[warp][0], *acc_unh = s_acc[warp][1], *acc_wtd = s_acc[warp][2];
  int32_t *g_mode = s_mode[warp][0], *g_prefix = s_mode[warp][1], *g_ncreate = s_mode[warp][2], *g_mh_running = s_mode[warp][kMH ? 3 : 2];
  uint32_t mh_head = 0;  // kMH: bit k = this lane's pod of chunk k is the first pod of a healthy replica of a multi-host group
  if (lane < KR_SMEM_GROUPS) { acc_list[lane] = 0; acc_unh[lane] = 0; acc_wtd[lane] = 0; g_mode[lane] = GM_UNPROCESSED; g_prefix[lane] = 0; g_ncreate[lane] = 0; }
  __syncwarp();

  // ---------------- scan 1: counts over the cluster's pods (order-free)
  int32_t ready = 0, available = 0, n_heads = 0, n0_list = 0, n0_unh = 0, n0_wtd = 0;
  bool all_running = P > 0;       // CheckAllPodsRunning (utils/util.go:584-603)
  const uint32_t nchunks = (P + 31) / 32;
#pragma unroll
  for (int k = 0; k < K; k++) {
    if ((uint32_t)k >= nchunks) break;
    const bool valid = (uint32_t)(k * 32) + lane < P;
    const uint32_t w = pw[k], fl = w & 0xFFFFu, slot = valid ? (w >> 16) : KR_ROW_NO_GROUP;
    const uint32_t nt = pp_node_type(fl), ph = pp_phase(fl), rd = pp_ready(fl);
    const bool w_run = valid && nt == KR_NT_WORKER && ph == KR_PHASE_RUNNING;
    available += __popc(__ballot_sync(0xFFFFFFFFu, w_run));
    ready += __popc(__ballot_sync(0xFFFFFFFFu, w_run && rd == KR_COND_TRUE));
    const bool not_ok = valid && (ph != KR_PHASE_RUNNING || rd == KR_COND_FALSE || rd == KR_COND_UNKNOWN);
    if (__any_sync(0xFFFFFFFFu, not_ok)) all_running = false;
    n_heads += __popc(__ballot_sync(0xFFFFFFFFu, valid && nt == KR_NT_HEAD));
    if (G == 1) {  // the common case: one worker group — three ballots instead of the match_any group-by
      const bool in0 = slot == 0;
      n0_list += __popc(__ballot_sync(0xFFFFFFFFu, in0));
      n0_unh += __popc(__ballot_sync(0xFFFFFFFFu, in0 && (fl & KR_ROW_UNHEALTHY)));
      n0_wtd += __popc(__ballot_sync(0xFFFFFFFFu, in0 && (fl & KR_ROW_WTD_OWN)));
      continue;
    }
    const uint32_t gkey = (slot < G) ? slot : KR_ROW_NO_GROUP;
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, gkey);
    if (gkey != KR_ROW_NO_GROUP) {
      const uint32_t ub = __ballot_sync(peers, (fl & KR_ROW_UNHEALTHY) != 0);
      const uint32_t wb = __ballot_sync(peers, (fl & KR_ROW_WTD_OWN) != 0);
      if ((peers & lt) == 0) {  // leader of its group in this chunk
        acc_list[gkey] += __popc(peers);
        acc_unh[gkey] += __popc(ub & peers);
        acc_wtd[gkey] += __popc(wb & peers);
      }
    }
    __syncwarp();
  }
  if (G == 1) { if (lane == 0) { acc_list[0] = n0_list; acc_unh[0] = n0_unh; acc_wtd[0] = n0_wtd; } __syncwarp(); }

  // ---------------- scalar decisions (uniform across the warp) — same order as decide_cluster / the reference
  // Every lane stores the same value to each field of cr.  A field stored twice with different values (stop_after_group) has a
  // __syncwarp between the stores, so no lane's earlier store can land after another lane's later one.  (volatile: each field is
  // stored where it is decided and loaded where it is read, instead of being carried in registers to a merged store.)
  volatile kr_cluster_result &cr = s_cr[warp];
  static_assert(sizeof(kr_cluster_result) % 4 == 0 && sizeof(kr_cluster_result) / 4 <= 32, "one word of the result record per lane");
  if (lane < sizeof(kr_cluster_result) / 4) {  // all zero but head_pod_idx = stop_after_group = -1
    const bool neg = lane == offsetof(kr_cluster_result, head_pod_idx) / 4 || lane == offsetof(kr_cluster_result, stop_after_group) / 4;
    reinterpret_cast<volatile uint32_t *>(&cr)[lane] = neg ? 0xFFFFFFFFu : 0u;
  }
  if (lane == 0) s_deferred[warp] = 0;
  __syncwarp();
  uint8_t all_action = KR_ACT_KEEP;
  bool head_delete = false, run_groups = false, any_prefix = false;
  uint32_t n_create_cluster = 0;
  if (mine) {
    if (cf & KR_CF_SKIP) {
      cr.path = KR_PATH_SKIPPED;
    } else if (ext_err != KR_EXT_ERR_NONE) {
      cr.path = KR_PATH_SKIPPED;  // :308-314
      cr.err_kind = ext_err == KR_EXT_ERR_STATUS_ONLY_NIL ? KR_ERR_NONE : KR_ERR_EXTERNAL;
    } else if (suspend_status == KR_SUSPEND_SUSPENDING || (!gate && (cf & KR_CF_SUSPEND))) {
      cr.path = KR_PATH_SUSPENDING_DELETE_ALL; all_action = KR_ACT_DELETE_ALL_SUSPEND;  // :629-644
    } else if (gate && (suspend_status == KR_SUSPEND_SUSPENDED || (cf & KR_CF_SUSPEND))) {
      cr.path = KR_PATH_SUSPENDED_NOOP;  // :646-654
    } else {
      bool recreate = false;
      if ((cf & KR_CF_UPGRADE_RECREATE) && n_heads > 0) {  // shouldRecreatePodsForUpgrade :1132-1171
        const int32_t aux = head_aux;
        const uint8_t ver = h_ver, ast = h_ast;
        if (ver == KR_VER_DIFFERENT) cr.head_update_annotations = 1;
        else if (ast == KR_ANNOT_OTHER) recreate = true;
        else if (ast == KR_ANNOT_HASH32 && !a.f.skip_hash) {
          if (phase == 0 && !a.spin_hash) {
            // The hash kernel is still running on its own stream.  Decide the cluster as if the digests matched, reserve the
            // whole bucket in the action list (a Recreate deletes every pod) and let phase 1 redo it once the digest is there.
            s_deferred[warp] = 1;
            if (lane == 0) a.sc.deferred_list[atomicAdd(&a.r.totals[4], 1u)] = c;
          } else {
            const uint8_t *ah = s.h_annot_hash + 32 * (size_t)aux;
            const uint32_t *hw = reinterpret_cast<const uint32_t *>(a.r.hash + 32 * (size_t)c);
            if (phase == 0) {
              // The hash kernel runs beside this one (its CTAs were resident before the chain started, and it takes the
              // digests these gates read FIRST: kr_engine.cu builds the hash order that way), so the digest is normally there
              // already; if not, wait for its last word — zeroed on the hash stream in front of the hash kernel, stored last by the hash lane.  Bounded: a warp that
              // gives up flags the pass and the engine reruns it on the two-phase schedule.
              if (lane == 0) {
                const volatile uint32_t *w7 = hw + 7;
                uint32_t it = 0;
                while (*w7 == 0u && it < 40000u) { __nanosleep(100); it++; }
                if (*w7 == 0u) atomicOr(&a.r.totals[3], KR_TOTALS_HASH_WAIT);
              }
              __syncwarp();
              __threadfence();
            }
            const uint32_t word = __ldcg(&hw[lane >> 2]);
            recreate = __any_sync(0xFFFFFFFFu, ah[lane] != (uint8_t)(word >> (8 * (lane & 3))));
          }
        }
      }
      if (recreate) {
        cr.path = KR_PATH_RECREATE_DELETE_ALL; all_action = KR_ACT_DELETE_ALL_RECREATE;  // :657-670
      } else {
        cr.path = KR_PATH_NORMAL;
        if (!(cf & KR_CF_HEAD_EXPECT_OK)) { cr.head_action = KR_HEAD_EXPECT_PENDING; run_groups = true; }  // head (:673-748)
        else if (n_heads == 1) {
          if (head_flags & KR_ROW_UNHEALTHY) { cr.head_action = KR_HEAD_DELETE; cr.err_kind = KR_ERR_HEAD_DELETED; head_delete = true; }
          else run_groups = true;
        } else if (n_heads == 0) {
          if (old_prov == KR_COND_TRUE && (cf & KR_CF_SKIP_HEAD_RESTART)) cr.head_action = KR_HEAD_SKIP_RESTART;
          else { cr.head_action = KR_HEAD_CREATE; run_groups = true; }
        } else {
          cr.head_action = KR_HEAD_MULTIPLE; cr.err_kind = KR_ERR_MULTIPLE_HEADS; cr.err_arg = n_heads;
        }
      }
    }
    // worker groups in spec order (:751-933): O(1) per group from the scan-1 counters
    if (run_groups) {
      const bool autoscaling = (cf & KR_CF_AUTOSCALING) != 0;
      cr.stop_after_group = (int32_t)G;
      for (uint32_t gi = 0; gi < G; gi++) {
        const uint32_t g = g0 + gi;
        const bool rec0 = gi == 0;  // worker group 0 came with the cluster's record
        const uint32_t gf = rec0 ? ci.g0_flags() : LDG(s.g_flags[g]);
        const int32_t hosts = rec0 ? ci.g0_hosts() : LDG(s.g_num_hosts[g]), g_rep = rec0 ? ci.g0_rep() : LDG(s.g_replicas[g]);
        const int32_t g_mn = rec0 ? ci.g0_min() : LDG(s.g_min[g]), g_mx = rec0 ? ci.g0_max() : LDG(s.g_max[g]);
        kr_group_result gr;
        gr.expected = 0; gr.n_list = 0; gr.n_unhealthy = 0; gr.n_running = 0; gr.diff = 0; gr.n_create = 0; gr.create_off = 0;
        gr.flags = KR_GR_PROCESSED;
        int32_t mode = GM_SKIP, prefix = 0;
        bool abort_here = false;
        if (!(gf & KR_GF_EXPECT_OK)) {
          gr.flags |= KR_GR_EXPECT_PENDING;
        } else {
          const int32_t expected = desired_replicas(g_rep, g_mn, g_mx, hosts, gf);
          const int32_t n_list = acc_list[gi], n_unh = acc_unh[gi], n_wtd = acc_wtd[gi];
          gr.expected = expected; gr.n_list = n_list;
          if (gf & KR_GF_SUSPEND) { gr.flags |= KR_GR_SUSPENDED; mode = GM_SUSPENDED; }
          else if (kMH && hosts > 1 && a.f.gate_multihost_indexing) {  // :777-784 (numOfHosts from the group row, never from the table's bit)
            gr.flags |= KR_GR_MULTIHOST; mode = GM_MULTIHOST;
            int32_t earg = 0;
            const int ek = decide_multihost2<K>(s, gi, expected, hosts, !autoscaling || a.f.env_random_pod_delete, LDG(s.g_wtd_cnt[g]), pidx, pw, act, mh_head,
                                                s_list[warp], gr, earg, lane);
            if (ek != KR_ERR_NONE) { cr.err_kind = (uint8_t)ek; cr.err_arg = earg; abort_here = true; }
            if (lane == 0) g_mh_running[gi] = gr.n_running;
          }
          else if (n_unh > 0) {  // :786-812
            gr.n_unhealthy = n_unh; gr.flags |= KR_GR_ABORTED; mode = GM_UNHEALTHY;
            cr.err_kind = KR_ERR_UNHEALTHY_WORKERS; cr.err_arg = n_unh; abort_here = true;
          } else {
            gr.flags |= KR_GR_WTD_EXECUTED; mode = GM_NORMAL;  // :814-849
            const int32_t running = n_list - n_wtd;
            const long long diff = (long long)expected - running;  // Go int (:757, :849): no int32 wrap below -2^31
            gr.n_running = running; gr.diff = diff < INT32_MIN ? INT32_MIN : (int32_t)diff;  // (saturated in the record)
            if (diff > 0) gr.n_create = (uint32_t)diff;
            else if (diff < 0) {
              if (!autoscaling || a.f.env_random_pod_delete) {  // :898-928
                const long long remove = -diff;
                if (remove > running) {  // expected < 0: the Go loop would index past runningPods (:917)
                  prefix = running; gr.flags |= KR_GR_ABORTED;
                  cr.err_kind = KR_ERR_NEGATIVE_EXPECTED; cr.err_arg = expected; abort_here = true;
                } else prefix = (int32_t)remove;
              } else gr.flags |= KR_GR_RANDOM_DELETE_OFF;
            }
          }
        }
        any_prefix |= prefix > 0;
        n_create_cluster += gr.n_create;
        __syncwarp();
        if (lane == 0) {
          g_mode[gi] = mode; g_prefix[gi] = prefix; g_ncreate[gi] = (int32_t)gr.n_create;
          a.r.groups[g] = gr;  // create_off follows once the look-back has placed this cluster
        }
        if (abort_here) { cr.stop_after_group = (int32_t)gi; break; }
      }
    }
    // groups never reached keep an all-zero record
    {
      const int32_t reached = ((cf & KR_CF_SKIP) || !run_groups) ? 0 : (cr.stop_after_group == (int32_t)G ? (int32_t)G : cr.stop_after_group + 1);
      for (uint32_t gi = reached + lane; gi < G; gi += 32) {
        kr_group_result z; z.expected = 0; z.n_list = 0; z.n_unhealthy = 0; z.n_running = 0; z.diff = 0; z.n_create = 0; z.create_off = 0; z.flags = 0;
        a.r.groups[g0 + gi] = z;
      }
    }
  }
  __syncwarp();

  // ---------------- scan 2: per-pod actions (set computations first, then the two ordered pieces)
  uint32_t cand = 0;  // bit k: this lane's pod of chunk k is a running pod of a group in normal mode (subject to the ordered delete prefix)
  if (mine) {
#pragma unroll
    for (int k = 0; k < K; k++) {
      if ((uint32_t)k >= nchunks) break;
      const bool valid = (uint32_t)(k * 32) + lane < P;
      const uint32_t w = pw[k], fl = w & 0xFFFFu;
      const uint32_t gkey = (valid && run_groups && (w >> 16) < G) ? (w >> 16) : KR_ROW_NO_GROUP;
      const int32_t mode = (gkey != KR_ROW_NO_GROUP) ? g_mode[gkey] : GM_UNPROCESSED;
      uint32_t ac = KR_ACT_KEEP;
      if (all_action != KR_ACT_KEEP) ac = valid ? all_action : (uint32_t)KR_ACT_KEEP;
      else if (head_delete) { if (valid && pidx[k] == head_pod) ac = KR_ACT_DELETE_HEAD; }
      else if (mode == GM_SUSPENDED) ac = KR_ACT_DELETE_GROUP_SUSPEND;
      else if (kMH && mode == GM_MULTIHOST) ac = act[k];  // decided with its group (decide_multihost2)
      else if (mode == GM_UNHEALTHY) { if (fl & KR_ROW_UNHEALTHY) ac = KR_ACT_DELETE_UNHEALTHY; }
      else if (mode == GM_NORMAL) {
        if (fl & KR_ROW_WTD_OWN) ac = KR_ACT_DELETE_WTD;
        else cand |= 1u << k;
      }
      act[k] = ac;
    }
    // runningPods.Items[0 .. -diff) (:916-919): the -diff smallest pod indices among the group's running pods
    if (any_prefix) {
      for (uint32_t gi = 0; gi < G; gi++) {
        const int32_t pre = g_prefix[gi];
        if (pre <= 0) continue;
        if (pre <= 8) {  // a few victims: extract the minimum pre times
          for (int32_t it = 0; it < pre; it++) {
            uint32_t m = 0xFFFFFFFFu;
#pragma unroll
            for (int k = 0; k < K; k++)
              if (((cand >> k) & 1u) && (pw[k] >> 16) == gi && act[k] == KR_ACT_KEEP) m = min(m, pidx[k]);
            const uint32_t wm = __reduce_min_sync(0xFFFFFFFFu, m);
            if (wm == 0xFFFFFFFFu) break;
#pragma unroll
            for (int k = 0; k < K; k++)
              if (((cand >> k) & 1u) && pidx[k] == wm) act[k] = KR_ACT_DELETE_RANDOM;
          }
        } else {  // a long prefix: rank every candidate among the group's candidates by counting
          uint32_t nc = 0;
#pragma unroll
          for (int k = 0; k < K; k++) {
            const bool isc = ((cand >> k) & 1u) && (pw[k] >> 16) == gi;
            const uint32_t bal = __ballot_sync(0xFFFFFFFFu, isc);
            if (isc) s_list[warp][nc + __popc(bal & lt)] = pidx[k];
            nc += __popc(bal);
          }
          __syncwarp();
#pragma unroll
          for (int k = 0; k < K; k++) {
            const bool isc = ((cand >> k) & 1u) && (pw[k] >> 16) == gi;
            if (!__any_sync(0xFFFFFFFFu, isc)) continue;
            uint32_t rank = 0;
            for (uint32_t i = 0; i < nc; i++) rank += s_list[warp][i] < pidx[k] ? 1u : 0u;
            if (isc && (int32_t)rank < pre) act[k] = KR_ACT_DELETE_RANDOM;
          }
          __syncwarp();
        }
      }
    }
  }
  // ---------------- status roll-up + record (needs nothing from the action list and the placement below: it comes first, so no
  // register of theirs is live through it)
  if (!(cf & KR_CF_SKIP)) {  // (every lane runs it, uniformly: the inputs are one broadcast load away in the record)
    const uint32_t head_name = (n_heads == 1 && head_pos != 0xFFFFFFFFu) ? __ldg(&s.p_name_id[head_pod]) : 0u;
    status_rollup(a.s, a.f, ci, cr, P, (uint32_t)n_heads, n_heads > 0 ? (int32_t)head_pod : -1, head_aux, head_name, ready, available, all_running);
  }
  __syncwarp();
  if (mine && lane < sizeof(kr_cluster_result) / 4)  // one coalesced store: lane i = word i
    reinterpret_cast<uint32_t *>(&a.r.clusters[c])[lane] = reinterpret_cast<const volatile uint32_t *>(&cr)[lane];

  // the cluster's action list in List order: stage the acted pods, rank each by counting the smaller pod indices
  uint32_t n_act = 0;
  uint32_t arank[K];
#pragma unroll
  for (int k = 0; k < K; k++) {
    arank[k] = 0;
    const bool isa = act[k] != KR_ACT_KEEP;
    const uint32_t bal = __ballot_sync(0xFFFFFFFFu, isa);
    if (isa) s_list[warp][n_act + __popc(bal & lt)] = pidx[k];
    n_act += __popc(bal);
  }
  __syncwarp();
  if (n_act > 1) {
#pragma unroll
    for (int k = 0; k < K; k++) {
      const bool isa = act[k] != KR_ACT_KEEP;
      if (!__any_sync(0xFFFFFFFFu, isa)) continue;
      uint32_t rank = 0;
      for (uint32_t i = 0; i < n_act; i++) rank += s_list[warp][i] < pidx[k] ? 1u : 0u;
      arank[k] = rank;
    }
  }

  // ---------------- placement: where this cluster's action list and replica indices go.  One returning 64-bit atomic per
  // RayCluster on the two arena cursors (pods to create << 32 | action slots), issued by lane 0 and needed only for the stores
  // below.  (A decoupled look-back over the CTAs was built first: placement in cluster order, but the prefix crosses the grid in
  // 32-CTA hops — 39 hops on the critical path of a 10 k-cluster pass, with the kernel's stalls gathered at the barrier
  // in front of it.  The owners' ORDER inside the arenas is therefore unspecified; every owner
  // finds its place through (act_start, act_cnt) / (create_off, n_create), which is what the shim reads anyway.)
  const bool deferred = s_deferred[warp] != 0;
  const uint32_t slots = deferred ? P : n_act;  // a deferred cluster may still turn into "delete every pod"
  uint32_t act_off = 0, create_off = 0;
  if (phase == 0) {
    unsigned long long base = 0;
    if (mine && lane == 0) {
      if (slots | n_create_cluster) base = atomicAdd(reinterpret_cast<unsigned long long *>(&a.r.totals[8]), ((unsigned long long)n_create_cluster << 32) | slots);
      if (n_act) atomicAdd(&a.r.totals[2], n_act);  // pods acted on (the extent of the list also counts reserved slots)
      if (n_create_cluster) atomicAdd(&a.r.totals[6], n_create_cluster);
    }
    base = __shfl_sync(0xFFFFFFFFu, base, 0);
    act_off = (uint32_t)base; create_off = (uint32_t)(base >> 32);
    if (mine && lane == 0) {
      a.r.act_start[c] = act_off; a.r.act_cnt[c] = n_act;
      if (deferred) a.sc.cact[c] = n_create_cluster;  // phase 1 corrects the count of pods to create if the cluster turns into a Recreate
      a.sc.act_res[c] = slots; a.sc.cre_res[c] = n_create_cluster;  // what an incremental epoch may reuse
    }
  } else if (kInc) {  // incremental epoch: keep the cluster's places while they suffice, else take new ones at the cursors
    unsigned long long base = 0;
    uint32_t need = 0;  // bit 0: new action slots, bit 1: new create slots
    if (mine && lane == 0) {
      const uint32_t old_act = a.r.act_cnt[c], old_create = s_old_create[warp];
      need = (n_act > a.sc.act_res[c] ? 1u : 0u) | (n_create_cluster > a.sc.cre_res[c] ? 2u : 0u);
      if (need) base = atomicAdd(reinterpret_cast<unsigned long long *>(&a.r.totals[8]), ((unsigned long long)((need & 2u) ? n_create_cluster : 0u) << 32) | ((need & 1u) ? n_act : 0u));
      if ((need & 1u) && (uint64_t)(uint32_t)base + n_act > a.n.n_pods) atomicOr(&a.sc.inc[KR_INC_VOID], KR_FULL_ARENA);         // the action list is full of abandoned runs:
      if ((need & 2u) && (uint64_t)(uint32_t)(base >> 32) + n_create_cluster > a.create_cap) atomicOr(&a.sc.inc[KR_INC_VOID], KR_FULL_ARENA);  // a full pass packs it again
      if (n_act != old_act) atomicAdd(&a.r.totals[2], n_act - old_act);
      if (n_create_cluster != old_create) atomicAdd(&a.r.totals[6], n_create_cluster - old_create);
    }
    base = __shfl_sync(0xFFFFFFFFu, base, 0); need = __shfl_sync(0xFFFFFFFFu, need, 0);
    if (mine) {
      act_off = (need & 1u) ? (uint32_t)base : a.r.act_start[c];
      create_off = (need & 2u) ? (uint32_t)(base >> 32) : (G ? a.sc.gcreate[g0] : 0u);
      if ((need & 1u) && (uint64_t)act_off + n_act > a.n.n_pods) mine = false;
      if ((need & 2u) && (uint64_t)create_off + n_create_cluster > a.create_cap) mine = false;
      if (mine && lane == 0) {
        a.r.act_start[c] = act_off; a.r.act_cnt[c] = n_act;
        if (need & 1u) a.sc.act_res[c] = n_act;
        if (need & 2u) a.sc.cre_res[c] = n_create_cluster;
      }
    }
  } else if (mine) {  // phase 1: the places phase 0 reserved
    act_off = a.r.act_start[c];
    if (lane == 0) {
      const uint32_t old_act = a.r.act_cnt[c], old_create = a.sc.cact[c];
      a.r.act_cnt[c] = n_act;
      if (n_act != old_act) atomicAdd(&a.r.totals[2], n_act - old_act);
      if (n_create_cluster != old_create) atomicAdd(&a.r.totals[6], n_create_cluster - old_create);
    }
  }
  if (!mine) return;
  // action list, List order
#pragma unroll
  for (int k = 0; k < K; k++)
    if (act[k] != KR_ACT_KEEP) { a.r.act_pod_idx[act_off + arank[k]] = pidx[k]; a.r.act_code[act_off + arank[k]] = (uint8_t)act[k]; }
  // create offsets + lowest free ray.io/worker-group-replica-index values (:854-881), from the registers
  if (phase == 1 || n_create_cluster) {
    uint32_t off = create_off;
    for (uint32_t gi = 0; gi < G; gi++) {
      const uint32_t g = g0 + gi;
      const uint32_t want = (uint32_t)g_ncreate[gi];
      if (phase == 1) {
        // keep the arena position phase 0 gave this group (a Recreate leaves a gap: n_create is now 0)
        off = a.sc.gcreate[g];
      }
      if (lane == 0) { a.r.groups[g].create_off = off; if (phase != 1) a.sc.gcreate[g] = off; }
      if (want == 0) continue;
      if ((uint64_t)off + want > a.create_cap) { off += want; continue; }  // the host reports KR_E_CAPACITY from totals[0]
      int32_t *out = a.r.create_idx + off;
      if (!a.f.gate_multihost_indexing) {  // createWorkerPod without an index (:884-889)
        for (uint32_t k2 = lane; k2 < want; k2 += 32) out[k2] = -1;
      } else {
        // multi-host (:1067-1077): in use = the label of the first pod of every healthy replica, and n_create counts replicas
        const bool mh = kMH && g_mode[gi] == GM_MULTIHOST;
        const uint64_t bound = (uint64_t)(mh ? g_mh_running[gi] : acc_list[gi] - acc_wtd[gi]) + want;  // the `want` lowest free indices all lie below n_running + want
        uint32_t written = 0;
        for (uint64_t w0 = 0; w0 < bound && written < want; w0 += 1024) {
          s_bits[warp][lane] = 0;
          __syncwarp();
#pragma unroll
          for (int k = 0; k < K; k++) {
            // runningPods of this group: listed, not deleted by name, label present and numeric
            if ((pw[k] >> 16) == gi && (pw[k] & KR_PP_HAS_REPLICA_IDX) && (mh ? ((mh_head >> k) & 1u) != 0 : (act[k] == KR_ACT_KEEP && pidx[k] != 0xFFFFFFFFu))) {
              // (read from the Pod column: the bucket record does not carry it, and no register holds it through the decisions)
              const int32_t idx = __ldg(&s.p_replica_index[pidx[k]]);
              if (idx >= 0 && (uint64_t)idx >= w0 && (uint64_t)idx < w0 + 1024 && (uint64_t)idx < bound)
                atomicOr(&s_bits[warp][(idx - w0) >> 5], 1u << ((idx - w0) & 31));
            }
          }
          __syncwarp();
          const uint32_t word = s_bits[warp][lane];
          const uint64_t wbase = w0 + 32ull * lane;
          uint32_t freeb = ~word;
          if (wbase >= bound) freeb = 0;
          else if (bound - wbase < 32) freeb &= (1u << (uint32_t)(bound - wbase)) - 1;
          const uint32_t cnt = __popc(freeb);
          uint32_t x = cnt;
#pragma unroll
          for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, d); if (lane >= (uint32_t)d) x += y; }
          uint32_t pos = written + x - cnt;
          while (freeb && pos < want) {
            const uint32_t bit = __ffs(freeb) - 1;
            freeb &= freeb - 1;
            out[pos++] = (int32_t)(wbase + bit);
          }
          written += __shfl_sync(0xFFFFFFFFu, x, 31);
          __syncwarp();
        }
      }
      off += want;
    }
  } else if (G) {
    // no pod to create: every group of the cluster still gets its (empty) place in the arena
    for (uint32_t gi = lane; gi < G; gi += 32) { a.r.groups[g0 + gi].create_off = create_off; a.sc.gcreate[g0 + gi] = create_off; }
  }
  if (kInc) {
    __syncwarp();  // this warp's own stores to r.clusters / r.groups above are ordered before the loads of the staging copy
    stage_cluster(a, blockIdx.x * kD2Warps + warp, c, act_off, n_act, g0, G, lane);
  }
}

}  // namespace kr

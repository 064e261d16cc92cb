// kr_match.cuh — k_clear, k_build_tables, k_match: per-pass clears, the join tables and the per-pod label / selector match.
// Part of the sm_90a kernel set of the batched reconcile engine; see kr_kernels.cuh for the pipeline overview.
#pragma once

#include "kr_common.cuh"

namespace kr {

// ------------------------------------------------------------------------------------------------ k_clear
// One launch for the per-pass clears (hash tables to 0xFF, workersToDelete resolutions to -1, totals and bucket counters
// to 0) instead of four memset nodes at the head of the graph.
struct ClearArgs { uint32_t *ptr[4]; uint32_t words[4]; uint32_t value[4]; };
__global__ void __launch_bounds__(256) k_clear(ClearArgs a) {
  KR_TL(9);
  const uint32_t stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
#pragma unroll
  for (int r = 0; r < 4; r++) {
    uint32_t *p = a.ptr[r];
    const uint32_t v = a.value[r], nw = a.words[r];
    uint4 *p4 = reinterpret_cast<uint4 *>(p);  // every region starts 256-byte aligned
    for (uint32_t i = t0; i < nw / 4; i += stride) p4[i] = make_uint4(v, v, v, v);
    for (uint32_t i = (nw & ~3u) + t0; i < nw; i += stride) p[i] = v;
  }
}

// The decide kernel's per-cluster inputs, gathered from ~25 columns into one 128-byte record (KR_CI_*).  Written by k_build_tables
// in a full pass and again by k_inc_prepare for the RayClusters an incremental epoch found changed.
__device__ __forceinline__ void write_cl_in(const SnapDev &s, const ScratchDev &sc, uint32_t t, uint32_t g0, uint32_t G) {
  uint32_t *ci = sc.cl_in + 32 * (size_t)t;
  const uint8_t *cs = s.c_old_cond_status + 5 * (size_t)t, *cv = s.c_old_cond_variant + 5 * (size_t)t;
  uint4 w0, w1;
  w0.x = s.c_flags[t]; w0.y = g0; w0.z = G;
  w0.w = s.c_suspend_status[t] | ((uint32_t)s.c_ext_err_kind[t] << 8) | ((uint32_t)s.c_old_state[t] << 16) | ((uint32_t)s.c_svc_count[t] << 24);
  w1.x = s.c_svc_ip_kind[t] | ((uint32_t)cs[0] << 8) | ((uint32_t)cs[1] << 16) | ((uint32_t)cs[2] << 24);
  w1.y = cs[3] | ((uint32_t)cs[4] << 8) | ((uint32_t)cv[0] << 16) | ((uint32_t)cv[1] << 24);
  w1.z = cv[2] | ((uint32_t)cv[3] << 8) | ((uint32_t)cv[4] << 16);
  w1.w = s.c_ext_err_msg_id[t];
  uint4 *o = reinterpret_cast<uint4 *>(ci);
  o[0] = w0; o[1] = w1;
  const int32_t *oc = s.c_old_counts + 5 * (size_t)t;
  o[2] = make_uint4((uint32_t)oc[0], (uint32_t)oc[1], (uint32_t)oc[2], (uint32_t)oc[3]);
  o[3] = make_uint4((uint32_t)oc[4], s.c_old_cond_reason_id[t], s.c_old_cond_msg_id[2 * (size_t)t], s.c_old_cond_msg_id[2 * (size_t)t + 1]);
  const uint32_t *oh = s.c_old_head_ids + 4 * (size_t)t;
  o[4] = make_uint4(oh[0], oh[1], oh[2], oh[3]);
  uint4 w5 = make_uint4(s.c_svc_ip_id[t], s.c_svc_name_id[t], 0, 0), w6 = make_uint4(0, 0, 0, 0);
  if (G) { w5.z = s.g_flags[g0]; w5.w = (uint32_t)s.g_replicas[g0]; w6.x = (uint32_t)s.g_min[g0]; w6.y = (uint32_t)s.g_max[g0]; w6.z = (uint32_t)s.g_num_hosts[g0]; }
  o[5] = w5; o[6] = w6; o[7] = make_uint4(0, 0, 0, 0);
}

// every workersToDelete name of group t: Delete(ns of the cluster, name) (raycluster_controller.go:817-822), into the name table
// and its Bloom bitmap (cleared beforehand: keys and chain heads to 0xFF, bits to 0).  k_build_tables, and k_inc_wtd_insert when
// an incremental epoch rebuilds the table.
__device__ __forceinline__ void wt_insert_group(const SnapDev &s, const ScratchDev &sc, uint32_t t) {
  uint32_t c = s.g_cluster_idx[t];
  uint32_t ns = s.c_ns_id[c];
  uint32_t off = s.g_wtd_off[t], cnt = s.g_wtd_cnt[t];
  for (uint32_t w = 0; w < cnt; w++) {
    uint32_t e = off + w;
    uint64_t k = key2(ns, s.w_name_id[e]);
    const uint32_t hk = hash_pair(ns, s.w_name_id[e]);
    atomicOr(&sc.wt_bits[(hk & sc.wt_bits_mask) >> 5], 1u << (hk & 31));  // Bloom bits: k_match2 probes the table only for pods whose two bits are set
    { const uint32_t h2 = bloom2(hk); atomicOr(&sc.wt_bits[(h2 & sc.wt_bits_mask) >> 5], 1u << (h2 & 31)); }
    uint32_t i = hk & sc.wt_mask;
    while (true) {
      unsigned long long prev = atomicCAS((unsigned long long *)&sc.wt_keys[i], KR_EMPTY64, k);
      if (prev == KR_EMPTY64 || prev == k) {
        // push e on the slot's chain
        uint32_t old = atomicExch(&sc.wt_head[i], e);
        sc.wt_next[e] = old;  // KR_EMPTY32 terminates (wt_head memset to 0xFF)
        break;
      }
      i = (i + 1) & sc.wt_mask;
    }
  }
}

// RayCluster t into the cluster table (namespace, name) -> {idx, flags, name of worker group 0}, and its cl_rec and cl_in records.
// k_build_tables, and k_inc_clusters_insert for the RayClusters an incremental epoch appended.
__device__ __forceinline__ void cl_insert_cluster(const SnapDev &s, const ScratchDev &sc, uint32_t t) {
  uint32_t ns = s.c_ns_id[t], name = s.c_name_id[t];
  uint32_t i = hash_pair(ns, name) & sc.cl_mask;
  unsigned long long *slots = reinterpret_cast<unsigned long long *>(sc.cl_slots);  // [2*i] = key (x = name, y = ns), [2*i+1] = payload
  const unsigned long long kk = ((unsigned long long)ns << 32) | name;
  uint32_t g0 = s.c_group_off[t], G = s.c_group_cnt[t], mh = 0;
  for (uint32_t gi = 0; gi < G; gi++) mh |= (s.g_num_hosts[g0 + gi] > 1) ? 1u : 0u;
  const uint32_t gname0 = G ? s.g_name_id[g0] : 0u;
  // payload = {z: name id of group 0, w: idx << 2 | flags} as one 64-bit word whose high half orders by cluster index
  const unsigned long long payload = ((unsigned long long)((t << 2) | (G > 1 ? KR_CL_MULTI : 0u) | mh) << 32) | gname0;
  while (true) {
    unsigned long long prev = atomicCAS(&slots[2 * (size_t)i], KR_EMPTY64, kk);
    if (prev == KR_EMPTY64 || prev == kk) { atomicMin(&slots[2 * (size_t)i + 1], payload); break; }  // duplicate (ns,name): lowest index wins, with its own payload
    i = (i + 1) & sc.cl_mask;
  }
  sc.cl_rec[t] = make_uint4(g0, G, gname0, mh);  // .w bit 0: some worker group has numOfHosts > 1
  write_cl_in(s, sc, t, g0, G);
}

// ------------------------------------------------------------------------------------------------ k_build_tables
// One thread per cluster / workersToDelete entry / head-aux row.  Tables were memset to 0xFF.

__global__ void __launch_bounds__(256) k_build_tables(SnapDev s, ScratchDev sc, ResDev r, Sizes n) {
  KR_TL(0);
  pdl_trigger();  // the match kernel's CTAs may be scheduled now: they load their pod columns, then wait for this grid to finish
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t == 0) {
    // A full pass closes the running incremental epoch (kr_incr.cuh): whatever the commits queued for an incremental pass is void,
    // and the next epoch's stamps must differ from every stamp written so far.  (Every commit kernel of this epoch has finished:
    // the pass waits for the commit stream before this kernel.)
    sc.inc[KR_INC_TOUCHED] = 0; sc.inc[KR_INC_DIRTY] = 0; sc.inc[KR_INC_STRUCTURAL] = 0; sc.inc[KR_INC_HEADS] = 0; sc.inc[KR_INC_VOID] = 0; sc.inc[KR_INC_GROUPS] = 0; sc.inc[KR_INC_LSEG] = 0;
    sc.inc[KR_INC_GROW] = 0; sc.inc[KR_INC_SPILL] = 0; sc.inc[KR_INC_GROWN] = 0;
    sc.inc[KR_INC_EPOCH] += 1u;
  }
  if (t < n.n_clusters) {
    cl_insert_cluster(s, sc, t);
    return;
  }
  t -= n.n_clusters;
  if (t < n.n_groups) {
    wt_insert_group(s, sc, t);
    return;
  }
  t -= n.n_groups;
  if (t < n.n_heads) {
    uint32_t p = s.h_pod_idx[t];
    uint32_t i = mix32(p) & sc.aux_mask;
    while (true) {
      uint32_t prev = atomicCAS(&sc.aux_keys[i], KR_EMPTY32, p);
      if (prev == KR_EMPTY32 || prev == p) { atomicMin(&sc.aux_vals[i], t); break; }
      i = (i + 1) & sc.aux_mask;
    }
  }
}

__device__ __forceinline__ int32_t aux_lookup(const ScratchDev &sc, uint32_t p) {
  uint32_t i = mix32(p) & sc.aux_mask;
  while (true) {
    uint32_t k = sc.aux_keys[i];
    if (k == p) return (int32_t)sc.aux_vals[i];
    if (k == KR_EMPTY32) return -1;
    i = (i + 1) & sc.aux_mask;
  }
}

// ------------------------------------------------------------------------------------------------ k_match
// The selector match (common/association.go:83-130): pod -> RayCluster by (namespace, ray.io/cluster), then
// ray.io/group against the cluster's worker groups.  Streams 7 coalesced columns (28 B/pod), writes one 16-byte row
// + 4-byte sort key per pod, and the pass-0 digit histogram of its tile.

// kFast: the count/place/sort-in-warp pipeline (per-cluster arrival rank by a returning atomic, no radix histogram).
// The loop is phased — all column loads, then all table probes, then all record loads — so that each thread keeps
// 8 independent memory requests in flight per phase instead of walking one pod's dependent chain at a time.
template <bool kFast, int kItems>
__global__ void __launch_bounds__(kSortThreads) k_match(SnapDev s, ScratchDev sc, ResDev r, Sizes n, int has_wtd) {
  KR_TL(1);
  __shared__ uint32_t s_hist[kRadix];
  pdl_wait(); pdl_trigger();
  const uint32_t tile = blockIdx.x, ntiles = gridDim.x;
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (!kFast) { s_hist[threadIdx.x] = 0; __syncthreads(); }
  const uint32_t base = tile * (kSortThreads * kItems) + warp * (32 * kItems) + lane;
  uint32_t ns[kItems], cn[kItems], gn[kItems], nm[kItems], pk[kItems], rn[kItems], ri[kItems];
  // phase A: 7 coalesced column loads per pod
#pragma unroll
  for (int it = 0; it < kItems; it++) {
    uint32_t p = base + it * 32;
    bool v = p < n.n_pods;
    ns[it] = v ? __ldg(&s.p_ns_id[p]) : 0u; cn[it] = v ? __ldg(&s.p_cluster_name_id[p]) : 0u;
    gn[it] = v ? __ldg(&s.p_group_name_id[p]) : 0u; nm[it] = v ? __ldg(&s.p_name_id[p]) : 0u;
    pk[it] = v ? __ldg(&s.p_packed[p]) : 0u; ri[it] = v ? (uint32_t)__ldg(&s.p_replica_index[p]) : 0u;
    rn[it] = v ? __ldg(&s.p_replica_name_id[p]) : 0u;
  }
  // phase B: hash-join probe (namespace, ray.io/cluster) -> cluster idx; first slot of every pod in flight together
  uint32_t c[kItems], pi[kItems];
  uint4 sl[kItems];
#pragma unroll
  for (int it = 0; it < kItems; it++) {
    pi[it] = hash_pair(ns[it], cn[it]) & sc.cl_mask;
    sl[it] = __ldg(&sc.cl_slots[pi[it]]);
  }
#pragma unroll
  for (int it = 0; it < kItems; it++) {
    c[it] = n.n_clusters;
    if (cn[it] != 0) {
      uint4 q = sl[it];
      uint32_t i = pi[it];
      while (true) {
        if (q.x == cn[it] && q.y == ns[it]) { c[it] = q.w >> 2; break; }
        if (q.x == KR_EMPTY32 && q.y == KR_EMPTY32) break;
        i = (i + 1) & sc.cl_mask;
        q = __ldg(&sc.cl_slots[i]);
      }
    }
  }
  // phase C: the cluster's group record
  uint4 rec[kItems];
#pragma unroll
  for (int it = 0; it < kItems; it++) rec[it] = (c[it] < n.n_clusters) ? __ldg(&sc.cl_rec[c[it]]) : make_uint4(0, 0, 0, 0);
  // phase C': first probe of the (tiny, cache-resident) workersToDelete-name table for every pod, and the bucket ranks
  uint32_t wi[kItems];
  uint64_t wk[kItems];
  if (has_wtd) {
#pragma unroll
    for (int it = 0; it < kItems; it++) { wi[it] = hash_pair(ns[it], nm[it]) & sc.wt_mask; wk[it] = __ldg(&sc.wt_keys[wi[it]]); }
  }
  uint32_t rank[kItems], orank[kItems], woff = 0;
  if (kFast) {
#pragma unroll
    for (int it = 0; it < kItems; it++)  // arrival rank inside the cluster's bucket; 8 atomics in flight
      rank[it] = (base + it * 32 < n.n_pods && c[it] < n.n_clusters) ? atomicAdd(&sc.ccount[c[it]], 1u) : 0u;
    // Orphans (no RayCluster) need no decision, only List order, and their bucket has no size bound: give them a STABLE rank
    // right here — thread order inside a tile is pod order (warp, then item, then lane) — plus the tile's orphan count, which
    // k_scan_counts turns into a per-tile prefix.  No atomics, no sort.
    __shared__ uint32_t s_worph[kSortThreads / 32];
    uint32_t wcount = 0;
    const uint32_t ltm = lanemask_lt();
#pragma unroll
    for (int it = 0; it < kItems; it++) {  // (kept apart from rank[]: nothing here may wait for the atomics above)
      bool orph = (base + it * 32 < n.n_pods) && c[it] == n.n_clusters;
      uint32_t bal = __ballot_sync(0xFFFFFFFFu, orph);
      orank[it] = wcount + __popc(bal & ltm);
      wcount += __popc(bal);
    }
    if (lane == 0) s_worph[warp] = wcount;
    __syncthreads();
    uint32_t ttot = 0;
#pragma unroll
    for (int w2 = 0; w2 < kSortThreads / 32; w2++) { uint32_t v = s_worph[w2]; if (w2 < (int)warp) woff += v; ttot += v; }
    if (threadIdx.x == 0) { sc.tile_orph[tile] = ttot; if (ttot) atomicAdd(&sc.ccount[n.n_clusters], ttot); }
  }
  // phase D: ray.io/group against the cluster's worker groups, workersToDelete-name intersection, outputs
#pragma unroll
  for (int it = 0; it < kItems; it++) {
    uint32_t p = base + it * 32;
    if (p >= n.n_pods) continue;
    uint32_t slot = KR_ROW_NO_GROUP, g0 = rec[it].x;
    if (c[it] < n.n_clusters && gn[it] != 0) {
      if (rec[it].y && rec[it].z == gn[it]) slot = 0;
      else
        for (uint32_t gi = 1; gi < rec[it].y; gi++)
          if (__ldg(&s.g_name_id[g0 + gi]) == gn[it]) { slot = gi; break; }  // group names are unique (pkg/webhooks/v1/raycluster_webhook.go:74)
    }
    uint32_t flags = pk[it] & (0x7FFu | KR_PP_TOMBSTONE);  // bit 11 of the row word is KR_ROW_WTD_OWN
    if (has_wtd) {
      const uint64_t k = key2(ns[it], nm[it]);
      uint32_t i = wi[it];
      uint64_t kk = wk[it];
      while (kk != KR_EMPTY64) {
        if (kk == k) {
          for (uint32_t e = sc.wt_head[i]; e != KR_EMPTY32; e = sc.wt_next[e]) {
            atomicMin(&r.wtd_pod_idx[e], p);
            if (slot != KR_ROW_NO_GROUP) {  // is e one of this pod's own group's names?
              uint32_t g = g0 + slot;
              uint32_t off = __ldg(&s.g_wtd_off[g]);
              if (e >= off && e < off + __ldg(&s.g_wtd_cnt[g])) flags |= KR_ROW_WTD_OWN;
            }
          }
          break;
        }
        i = (i + 1) & sc.wt_mask;
        kk = __ldg(&sc.wt_keys[i]);
      }
    }
    sc.rows[p] = make_uint4(nm[it], rn[it], ri[it], (slot << 16) | flags);
    sc.keys[0][p] = c[it];
    if (kFast) sc.keys[1][p] = (c[it] == n.n_clusters) ? orank[it] + woff : rank[it];
    else atomicAdd(&s_hist[c[it] & (kRadix - 1)], 1u);
  }
  if (!kFast) {
    __syncthreads();
    sc.hist[threadIdx.x * ntiles + tile] = s_hist[threadIdx.x];
  }
}

}  // namespace kr

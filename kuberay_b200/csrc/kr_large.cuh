// kr_large.cuh — RayClusters the bucket pipeline decides one CTA per cluster: large ones (KR_OPT_LARGE_CLUSTERS: more than 256 and
// at most KR_LARGE_MAX_PODS pods) and wide ones (KR_OPT_WIDE_CLUSTERS: more than KR_SMEM_GROUPS worker groups).
// Part of the sm_90a kernel set of the batched reconcile engine; see kr_kernels.cuh for the pipeline overview.
//
// The engine classifies large clusters on the host after a bucket attempt that voided (k_match2 counts every cluster's pods past
// the stride) and gives each one a region of the large-cluster record arena: k_match2 and k_inc_admit put the records of arrival
// rank >= bucket_stride there (rec_slot, kr_bucket2.cuh), so the rest of the fleet keeps its stride and an ordinary pod never looks
// at the region table.  Wide clusters are known at commit (their group counts); one without a region keeps its pods in its bucket,
// and an overflow past the stride voids the attempt as for any cluster.  Both kinds share one cluster table and one list (lg,
// lg_list).  k_decide2 leaves every cluster whose count exceeds the stride, and every wide one, alone; these two kernels, one CTA per
// listed RayCluster, decide them instead:
//   k_large_sort    (beside the hash) loads the cluster's records, drops the stale ones of an incremental epoch and stores the rest
//                   back compacted, writes each pod's 16-byte row (what the memory-resident decide reads), sorts the pod indices
//                   into List order in shared memory and publishes them at a scratch segment (sorted_pod_idx);
//   k_decide_large  (after the join with the hash stream: a Recreate gate reads a finished digest) decides the cluster with every
//                   warp of the CTA (decide_cluster_block, kr_decide.cuh; a wide one with warp 0 alone: decide_cluster<0, true>, which
//                   spills the accumulators to gacc, as the sort pipeline does), reserves its action run and create run at the bucket
//                   pipeline's cursors, moves the actions into place and fills the replica indices.  Its 512-thread instantiation,
//                   k_decide_huge, decides the huge RayClusters (kr_huge.cuh).
// Two kernels, because the decide reads sorted_pod_idx and the rows through the read-only cache, which is only coherent with
// stores of an earlier grid.
#pragma once

#include "kr_incr.cuh"

namespace kr {

static constexpr int kLargeSortThreads = 512;
static constexpr int kLargeDecideThreads = 128;
static constexpr int kHugeDecideThreads = 512;  // (k_decide_huge: the most threads that keep its registers free of spills)
static constexpr int kHugeTile = KR_LARGE_MAX_PODS;  // arrival ranks per tile of a huge RayCluster (kr_huge.cuh)

// Ascending bitonic sort of s[0, total) in shared memory, padded to the next power of two (at least 2) with 0xFFFFFFFF: s must
// hold that many words.  Every thread of the CTA calls it; the stores of s[0, total) are ordered before by its first barrier.
template <int kThreads>
__device__ __forceinline__ void block_sort_asc(uint32_t *s, uint32_t total, uint32_t tid) {
  uint32_t n2 = 2;
  while (n2 < total) n2 <<= 1;
  for (uint32_t k = total + tid; k < n2; k += kThreads) s[k] = 0xFFFFFFFFu;
  __syncthreads();
  for (uint32_t size = 2; size <= n2; size <<= 1) {
    for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
      for (uint32_t t = tid; t < n2 / 2; t += kThreads) {
        const uint32_t lo = 2 * stride * (t / stride) + (t % stride), hi = lo + stride;
        const bool asc = (lo & size) == 0;
        const uint32_t u = s[lo], v = s[hi];
        if ((u > v) == asc) { s[lo] = v; s[hi] = u; }
      }
      __syncthreads();
    }
  }
}

// ------------------------------------------------------------------------------------------------ k_inc_grow
// KR_OPT_LARGE_GROWTH: regions for the RayClusters k_inc_admit put on the grow list (kr_incr.cuh: grow_spill), in one launch.  Every
// CTA reads the list and reaches the same allocation: the entries by row, each final count (cl_dyn.x) sized by large_region_cap, one
// prefix from the region cursor past every region in use.  The epoch is void (every CTA decides so alike) when a count passes
// KR_LARGE_MAX_PODS (a huge RayCluster needs tiles) without kHuge, the arena has no room, or newly listed RayClusters would take the
// per-cluster list past list_cap (a regrowth adds no one: it is never held back by the cap).  Else the
// CTAs copy each regrown RayCluster's old region into its new one and place the spilled records; CTA 0 writes the region table and
// the result the host and the per-cluster kernels read (a RayCluster is newly listed when it had no region and is not wide: a wide
// one is on the list already).  No other kernel reads the table between k_inc_admit and this one, and the list kept the old regions.
// kHuge (KR_OPT_HUGE_GROWTH): a RayCluster whose new region reaches past KR_LARGE_MAX_PODS ranks is huge.  CTA 0 appends its tiles
// (kr_huge.cuh) to the KR_HUGE_GROW_TILES reserve entries at tiles[n_tiles, ...) and retires a huge one's old tiles among the
// n_tiles resident ones (cluster word KR_EMPTY32: k_huge_tiles and k_huge_merge pass over them); the epoch is also void when the
// appended tiles pass the reserve or the resident tiles would pass tile_cap.  A huge old region (up to about 25 000 records) is
// copied by every CTA of the launch.
template <bool kHuge>
__global__ void __launch_bounds__(256) k_inc_grow(SnapDev s, ScratchDev sc, uint4 *grow, uint32_t cursor, uint32_t arena, uint32_t n_list,
                                                  uint32_t list_cap, int wide, uint4 *tiles, uint32_t n_tiles, uint32_t tile_cap) {
  __shared__ uint4 s_e[KR_GROW_MAX];  // {cluster, old offset, old capacity, count}, ascending rows
  __shared__ uint32_t s_off[KR_GROW_MAX], s_cap[KR_GROW_MAX], s_new[KR_GROW_MAX];
  __shared__ uint32_t s_ok;
  const uint32_t tid = threadIdx.x;
  const uint32_t n = __ldcg(&sc.inc[KR_INC_GROW]);
  if (n == 0 || n > KR_GROW_MAX || __ldcg(&sc.inc[KR_INC_VOID]) || __ldcg(&sc.inc[KR_INC_STRUCTURAL])) return;  // (nothing grew, or void)
  const uint32_t S = sc.bucket_stride;
  uint4 mine = make_uint4(0u, 0u, 0u, 0u);
  if (tid < n) { mine = __ldcg(&grow[tid]); mine.w = __ldcg(&sc.cl_dyn[mine.x].x); }
  uint32_t rank = 0;  // (rows are distinct: one entry per cluster)
  for (uint32_t k = 0; k < n; k++) rank += __ldcg(&grow[k].x) < mine.x ? 1u : 0u;
  if (tid < n) s_e[rank] = mine;
  __syncthreads();
  if (tid == 0) {
    uint64_t off = cursor;
    uint32_t listed = 0, added = 0, retired = 0;
    bool ok = true;
    for (uint32_t i = 0; i < n; i++) {
      const uint4 e = s_e[i];
      ok = ok && (kHuge || e.w <= KR_LARGE_MAX_PODS);
      const uint32_t cap = ok ? large_region_cap(e.w, S) : 0u;
      s_off[i] = (uint32_t)off; s_cap[i] = cap;
      off += cap;
      s_new[i] = e.z == 0 && !(wide && s.c_group_cnt[e.x] > KR_SMEM_GROUPS);
      listed += s_new[i];
      if (kHuge && S + cap > KR_LARGE_MAX_PODS) added += (S + cap + kHugeTile - 1) / kHugeTile;
      if (kHuge && S + e.z > KR_LARGE_MAX_PODS) retired += (S + e.z + kHugeTile - 1) / kHugeTile;  // (upload_lg cut them alike)
    }
    ok = ok && (!kHuge || (added <= KR_HUGE_GROW_TILES && n_tiles + added <= tile_cap + retired));
    s_ok = ok && off <= arena && (listed == 0 || n_list + listed <= list_cap);  // (a pure regrowth lists no one)
  }
  __syncthreads();
  if (!s_ok) {
    if (blockIdx.x == 0 && tid == 0) atomicOr(&sc.inc[KR_INC_VOID], KR_FULL_GROW_LIMIT);
    return;
  }
  for (uint32_t i = blockIdx.x; i < n; i += gridDim.x)  // a regrown RayCluster's records of ranks [stride, stride + old capacity)
    if (!kHuge || s_e[i].z <= KR_LARGE_MAX_PODS)
      for (uint32_t j = tid; j < s_e[i].z; j += blockDim.x) sc.region[s_off[i] + j] = __ldcg(&sc.region[s_e[i].y + j]);
  if (kHuge)  // ... a huge old region over the whole launch
    for (uint32_t i = 0; i < n; i++)
      if (s_e[i].z > KR_LARGE_MAX_PODS)
        for (uint32_t j = blockIdx.x * blockDim.x + tid; j < s_e[i].z; j += gridDim.x * blockDim.x) sc.region[s_off[i] + j] = __ldcg(&sc.region[s_e[i].y + j]);
  const uint32_t n_spill = __ldcg(&sc.inc[KR_INC_SPILL]);  // (at most KR_GROW_SPILL: k_inc_admit voided the attempt otherwise)
  for (uint32_t k = blockIdx.x * blockDim.x + tid; k < n_spill && k < KR_GROW_SPILL; k += gridDim.x * blockDim.x) {
    const uint4 at = __ldcg(&grow[kGrowSpill + 2 * k]);
    uint32_t lo = 0, hi = n - 1;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (s_e[mid].x < at.z) lo = mid + 1; else hi = mid; }
    // (a record whose RayCluster is not on the list, or whose rank the new region does not hold, cannot be placed: void rather than
    // write into another region; the full pass that follows rebuilds every bucket and region)
    if (s_e[lo].x != at.z || at.y < S + s_e[lo].z || at.y - S >= s_cap[lo]) { atomicOr(&sc.inc[KR_INC_VOID], KR_FULL_GROW_LIMIT); continue; }
    const uint4 rec = __ldcg(&grow[kGrowSpill + 2 * k + 1]);
    sc.region[s_off[lo] + at.y - S] = make_uint2(rec.x, rec.y);
  }
  if (blockIdx.x == 0) {
    if (tid < n) {
      sc.lg[s_e[tid].x] = make_uint4(s_off[tid], s_cap[tid], 0u, 0u);
      grow[kGrowResult + tid] = make_uint4(s_e[tid].x, s_off[tid], s_cap[tid], s_new[tid]);
    }
    if (tid == 0) sc.inc[KR_INC_GROWN] = n;
    if (kHuge) {
      for (uint32_t t = tid; t < n_tiles; t += blockDim.x) {  // the regrown huge RayClusters' resident tiles
        const uint32_t c = tiles[t].x;
        uint32_t lo = 0, hi = n - 1;
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (s_e[mid].x < c) lo = mid + 1; else hi = mid; }
        if (s_e[lo].x == c) tiles[t].x = KR_EMPTY32;
      }
      if (tid == 0) {
        uint32_t k = n_tiles;
        for (uint32_t i = 0; i < n; i++) {
          const uint32_t span = S + s_cap[i];
          if (span <= KR_LARGE_MAX_PODS) continue;
          const uint32_t nt = (span + kHugeTile - 1) / kHugeTile, first = k;
          for (uint32_t t = 0; t < nt; t++) tiles[k++] = make_uint4(s_e[i].x, t * kHugeTile, first, nt);
        }
      }
    }
  }
}

// The k-th RayCluster of k_inc_grow's result that was newly listed (KR_EMPTY32: fewer were).  The per-cluster kernels give each such
// RayCluster one of their KR_GROW_MAX CTAs past the list.
__device__ __forceinline__ uint32_t grown_row(const ScratchDev &sc, const uint4 *grown, uint32_t k) {
  const uint32_t n = __ldcg(&sc.inc[KR_INC_GROWN]);
  for (uint32_t i = 0; i < n; i++) {
    const uint4 g = __ldcg(&grown[i]);
    if (g.w && k-- == 0) return g.x;
  }
  return KR_EMPTY32;
}

// One CTA per large RayCluster (lg_list, n_list entries).  kInc: only the ones the epoch marked dirty.  grown (KR_OPT_LARGE_GROWTH:
// k_inc_grow's result): the CTAs past the list take the newly listed RayClusters.
template <bool kInc>
__global__ void __launch_bounds__(kLargeSortThreads) k_large_sort(Decide2Args a, const uint32_t *__restrict__ lg_list, uint32_t n_list, const uint4 *grown) {
  __shared__ uint32_t s_idx[KR_LARGE_MAX_PODS];
  __shared__ uint32_t s_warp[kLargeSortThreads / 32];
  __shared__ uint32_t s_seg;
  const ScratchDev &sc = a.sc;
  const uint32_t c = !kInc || blockIdx.x < n_list ? lg_list[blockIdx.x] : grown_row(sc, grown, blockIdx.x - n_list);
  if (kInc && c == KR_EMPTY32) return;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t S = sc.bucket_stride;
  const uint32_t epoch = kInc ? inc_epoch_of(sc) : 0u;
  const uint4 dyn = __ldcg(&sc.cl_dyn[c]);
  const uint32_t P = dyn.x;
  if (tid == 0) {  // (decided once for the CTA: other CTAs may flag the attempt void meanwhile)
    const uint32_t cap = __ldcg(&sc.lg[c].y);
    sc.lg[c].w = 0;  // not taken (yet) this pass
    bool go = !KR_ATTEMPT_VOID(a.r.totals);
    if (kInc) go = go && !__ldcg(&sc.inc[KR_INC_VOID]) && !__ldcg(&sc.inc[KR_INC_STRUCTURAL]) && __ldcg(&sc.dirty_flag[c]) == epoch;
    // a large cluster past the stride, within its region; a wide one (k_decide2 leaves it alone) also with every pod in its bucket.
    // Else k_decide2 decides it, or the attempt is void (k_match2 / k_inc_admit flagged it: a wide cluster without a region has cap 0)
    const bool wide = a.s.c_group_cnt[c] > KR_SMEM_GROUPS;
    // (and never one that k_inc_grow made huge this pass, KR_OPT_HUGE_GROWTH: s_idx holds KR_LARGE_MAX_PODS ranks, its tiles sort it)
    s_seg = go && (P > S ? P - S <= cap : wide) && S + cap <= KR_LARGE_MAX_PODS;
  }
  __syncthreads();
  if (!s_seg) return;
  const bool lost = kInc && dyn.y == epoch;  // the cluster lost a row this epoch: the records of stamped rows are stale
  // each thread owns a contiguous run of ranks, so the kept records keep their arrival order
  const uint32_t per = (P + kLargeSortThreads - 1) / kLargeSortThreads;
  const uint32_t j0 = min(tid * per, P), j1 = min(j0 + per, P);
  uint32_t kept = 0;
  for (uint32_t j = j0; j < j1; j++) {
    const uint2 rec = __ldcg(rec_slot(sc, c, j));
    const bool keep = !lost || (rec.y & KR_ROW_FRESH) || __ldcg(&sc.stamp[rec.x]) != epoch;
    if (keep) {  // (the name and the replica index come from the Pod columns: the 8-byte record does not carry them)
      sc.rows[rec.x] = make_uint4(a.s.p_name_id[rec.x], a.s.p_replica_name_id[rec.x], (uint32_t)a.s.p_replica_index[rec.x], rec.y & ~KR_ROW_FRESH);
      kept++;
    }
  }
  // exclusive prefix of the kept counts over the CTA
  uint32_t x = kept;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, d); if (lane >= (uint32_t)d) x += y; }
  if (lane == 31) s_warp[warp] = x;
  __syncthreads();
  uint32_t before = 0, total = 0;
  for (uint32_t w = 0; w < kLargeSortThreads / 32; w++) { const uint32_t v = s_warp[w]; before += w < warp ? v : 0u; total += v; }
  uint32_t o = before + x - kept;
  for (uint32_t j = j0; j < j1; j++) {
    const uint2 rec = __ldcg(rec_slot(sc, c, j));
    const bool keep = !lost || (rec.y & KR_ROW_FRESH) || __ldcg(&sc.stamp[rec.x]) != epoch;
    if (keep) s_idx[o++] = rec.x;
  }
  if (tid == 0) {
    s_seg = atomicAdd(&sc.inc[KR_INC_LSEG], total);
    if ((uint64_t)s_seg + total > a.n.n_pods) {  // cannot happen while the regions hold distinct live rows; void rather than overrun
      if (kInc) atomicOr(&sc.inc[KR_INC_VOID], KR_FULL_ARENA); else KR_MARK_ATTEMPT_VOID(a.r.totals);
    }
  }
  __syncthreads();  // (also orders every rows[] store of the CTA before the record rewrite below)
  const uint32_t seg = s_seg;
  if ((uint64_t)seg + total > a.n.n_pods) return;
  if (kInc) {
    // the region (and bucket) compacted in arrival order, FRESH marks cleared; pos[] follows the records that moved
    for (uint32_t k = tid; k < total; k += kLargeSortThreads) {
      const uint32_t p = s_idx[k];
      const uint4 row = sc.rows[p];
      *rec_slot(sc, c, k) = make_uint2(p, row.w);
      sc.pos[p] = k;
    }
    if (tid == 0) { sc.cl_dyn[c].x = total; sc.cl_dyn[c].y = 0u; }
  }
  // informer List order = ascending pod index
  block_sort_asc<kLargeSortThreads>(s_idx, total, tid);
  for (uint32_t k = tid; k < total; k += kLargeSortThreads) a.r.sorted_pod_idx[seg + k] = s_idx[k];
  if (tid == 0) { sc.lg[c].z = seg; sc.lg[c].w = total | KR_LG_OWNED; }
}

// One CTA per RayCluster of the list that k_large_sort or k_huge_tiles took: every warp decides it (decide_cluster_block) but for a
// wide one, whose accumulators live in gacc (warp 0 alone: decide_cluster<0, true>); warp 0 reserves its action and create runs;
// every warp fills replica indices.  Two instantiations split the list (in profiles, k_decide_large and k_decide_huge):
//   kThreads = kLargeDecideThreads  the list, the grown CTAs past it, and the wide RayClusters of its huge part [n_lsort, n_list);
//   kThreads = kHugeDecideThreads   the rest of the huge part (launched on lg_list + n_lsort, with n_lsort = 0 and no grown CTAs).
template <bool kInc, int kThreads>
__global__ void __launch_bounds__(kThreads, 1) k_decide_large(Decide2Args a, const uint32_t *__restrict__ lg_list, uint32_t n_list, uint32_t n_lsort,
                                                           const uint4 *grown) {
  constexpr int kWarps = kThreads / 32;
  constexpr bool kHugePart = kThreads != kLargeDecideThreads;
  __shared__ int32_t s_acc[4][KR_SMEM_GROUPS];  // (a wide RayCluster's warp decide)
  __shared__ int32_t s_mode[2][KR_SMEM_GROUPS];
  __shared__ BlockDecideSmem<kWarps> s_dec;
  __shared__ uint32_t s_bits[kWarps][32];
  __shared__ uint32_t s_place[4];  // act_off, n_act, stage index, go on
  const ScratchDev &sc = a.sc;
  const ResDev &r = a.r;
  const uint32_t c = !kInc || blockIdx.x < n_list ? lg_list[blockIdx.x] : grown_row(sc, grown, blockIdx.x - n_list);
  if (kInc && c == KR_EMPTY32) return;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint4 l = __ldcg(&sc.lg[c]);  // (written by k_large_sort: an earlier grid)
  if (!(l.w & KR_LG_OWNED)) return;
  const uint32_t seg = l.z, P = l.w & ~KR_LG_OWNED;
  const uint32_t G = a.s.c_group_cnt[c], g0 = a.s.c_group_off[c];
  const bool wide = G > KR_SMEM_GROUPS;
  if (kHugePart ? wide : (blockIdx.x >= n_lsort && blockIdx.x < n_list && !wide)) return;  // the other instantiation's
  if (kInc) {  // this cluster's place in the dirty list (= its entry of the staging buffer)
    if (tid == 0) s_place[2] = 0xFFFFFFFFu;
    __syncthreads();
    const uint32_t n_dirty = __ldcg(&sc.inc[KR_INC_DIRTY]);
    for (uint32_t i = tid; i < n_dirty; i += kThreads) if (__ldcg(&sc.dirty_list[i]) == c) s_place[2] = i;
  }
  // what the cluster holds in the resident results (an incremental epoch keeps its places while they suffice), read before the
  // decide rewrites them
  uint32_t old_create = 0, old_act = 0, old_create_off = 0;
  if (kInc && warp == 0) {
    for (uint32_t gi = lane; gi < G; gi += 32) old_create += r.groups[g0 + gi].n_create;
    old_create = __reduce_add_sync(0xFFFFFFFFu, old_create);
    old_act = r.act_cnt[c];
    old_create_off = G ? sc.gcreate[g0] : 0u;
  }
  __syncwarp();
  DecideArgs da{a.s, a.sc, a.r, a.n, a.f, nullptr, nullptr, 0, 1};  // phase 1: the digests are final
  if (!kHugePart && wide) {
    if (warp == 0) {
      uint32_t d0[1] = {0}, d1[1] = {0};
      decide_cluster<0, true>(da, c, seg, seg + P, d0, d1, s_acc, s_mode, lane);
    }
  } else decide_cluster_block<kWarps>(da, c, seg, seg + P, s_dec, warp, lane);
  if (warp == 0) {
    __syncwarp();
    // the decide left n_create per group in gcreate[] and the action count in cact[]
    uint32_t n_create = 0;
    for (uint32_t gi = lane; gi < G; gi += 32) n_create += sc.gcreate[g0 + gi];
    n_create = __reduce_add_sync(0xFFFFFFFFu, n_create);
    const uint32_t n_act = sc.cact[c];
    if (lane == 0) {
      uint32_t act_off, create_off;
      if (!kInc) {
        const unsigned long long base = (n_act | n_create) ? atomicAdd(reinterpret_cast<unsigned long long *>(&r.totals[8]), ((unsigned long long)n_create << 32) | n_act) : 0ull;
        act_off = (uint32_t)base; create_off = (uint32_t)(base >> 32);
        if (n_create) atomicAdd(&r.totals[6], n_create);
      } else {
        const uint32_t need = (n_act > sc.act_res[c] ? 1u : 0u) | (n_create > sc.cre_res[c] ? 2u : 0u);
        unsigned long long base = 0;
        if (need) base = atomicAdd(reinterpret_cast<unsigned long long *>(&r.totals[8]), ((unsigned long long)((need & 2u) ? n_create : 0u) << 32) | ((need & 1u) ? n_act : 0u));
        act_off = (need & 1u) ? (uint32_t)base : r.act_start[c];
        create_off = (need & 2u) ? (uint32_t)(base >> 32) : old_create_off;
        if ((need & 1u) && (uint64_t)act_off + n_act > a.n.n_pods) atomicOr(&sc.inc[KR_INC_VOID], KR_FULL_ARENA);            // the action list is full of abandoned runs:
        if ((need & 2u) && (uint64_t)create_off + n_create > a.create_cap) atomicOr(&sc.inc[KR_INC_VOID], KR_FULL_ARENA);  // a full pass packs it again
        if (need & 1u) sc.act_res[c] = n_act;
        if (need & 2u) sc.cre_res[c] = n_create;
        if (old_act) atomicSub(&r.totals[2], old_act);  // (the decide added this pass's n_act)
        if (n_create != old_create) atomicAdd(&r.totals[6], n_create - old_create);
      }
      if (!kInc) { sc.act_res[c] = n_act; sc.cre_res[c] = n_create; }
      r.act_start[c] = act_off; r.act_cnt[c] = n_act;
      // create runs per group, in spec order (gcreate[] keeps the offsets afterwards, as k_decide2 leaves them)
      uint32_t off = create_off;
      for (uint32_t gi = 0; gi < G; gi++) {
        const uint32_t want = sc.gcreate[g0 + gi];
        r.groups[g0 + gi].create_off = off; sc.gcreate[g0 + gi] = off;
        off += want;
      }
      s_place[0] = act_off; s_place[1] = n_act;
      s_place[3] = !kInc || !__ldcg(&sc.inc[KR_INC_VOID]);  // (a void epoch is redone by a full pass: nothing more to write)
    }
  }
  __syncthreads();
  if (!s_place[3]) return;
  for (uint32_t gi = warp; gi < G; gi += kWarps)
    create_fill_group(a.s, sc, r, a.f, g0 + gi, r.groups[g0 + gi].create_off, a.create_cap, s_bits[warp], lane);
  if (warp == 0) compact_cluster_actions(r, sc, c, s_place[0], s_place[1], lane);
  __syncthreads();  // both read the cluster's pod_start
  if (tid == 0) r.clusters[c].pod_start = 0;  // as everywhere on the bucket pipeline (kr_flags.fetch_pod_lists = 0)
  if (kInc && warp == 0 && s_place[2] != 0xFFFFFFFFu) {
    __syncwarp();
    stage_cluster(a, s_place[2], c, s_place[0], s_place[1], g0, G, lane);
  }
}

}  // namespace kr

// kr_huge.cuh — RayClusters of more than KR_LARGE_MAX_PODS pods on the bucket pipeline (KR_OPT_HUGE_CLUSTERS, with
// KR_OPT_LARGE_CLUSTERS).  Part of the sm_90a kernel set of the batched reconcile engine; see kr_kernels.cuh for the overview.
//
// Such a "huge" RayCluster gets a region of the large-cluster arena like a large one (kr_large.cuh) and is decided by the same
// block decide, in k_decide_large's 512-thread instantiation (k_decide_huge); only its List-order sort differs, because k_large_sort sorts a whole cluster in one CTA's shared memory.  The
// engine cuts the arrival ranks a huge cluster's bucket and region can hold, [0, stride + region capacity), into tiles of
// kHugeTile ranks (a table {cluster, first rank, the cluster's first tile, its tile count}, uploaded with the cluster list):
//   k_huge_tiles   one CTA per tile: drops the stale records of an incremental epoch (k_large_sort's rule), writes each kept pod's
//                  16-byte row, sorts the kept pod indices in shared memory and stores the sorted run and the same indices in
//                  arrival order (the stash) in the tile's scratch slots.  The last CTA of a cluster (fenced tile counts, one
//                  counting atomic) reserves the cluster's sorted_pod_idx segment at KR_INC_LSEG and publishes it in lg[c].z / .w
//                  as k_large_sort does, so k_decide_huge (k_decide_large's 512-thread instantiation) decides the cluster;
//   k_huge_merge   one CTA per tile: a pod's place in List order is its rank in its own run plus, for every other tile of the
//                  cluster, how many of that tile's pods precede it (the keys are distinct pod indices).  Each other run is staged
//                  in shared memory in turn; a thread owns kHugePer consecutive keys and finds their places by galloping from the
//                  previous one.  In an incremental epoch it also rewrites the bucket and region compacted in arrival order from
//                  the stash (pos[] follows, cl_dyn[c].x takes the kept count): a tile's compacted ranks overlap its predecessors'
//                  records, so this waits for the grid after the one that read them.
// Both run on stream M between k_large_sort and the join with the hash stream; their grids are the tile count (in an incremental
// pass with KR_OPT_HUGE_GROWTH, also the KR_HUGE_GROW_TILES reserve entries past it, where k_inc_grow appends the tiles of the
// RayClusters it makes huge or regrows; a free entry, and a resident tile it retired, has the cluster word KR_EMPTY32).
#pragma once

#include "kr_large.cuh"

namespace kr {

static constexpr int kHugeThreads = 1024;
static constexpr int kHugePer = kHugeTile / kHugeThreads;  // keys per thread in k_huge_merge

struct HugeDev {
  const uint4 *tiles;  // [n_tiles] {cluster, first arrival rank, the cluster's first tile, the cluster's tile count}
  uint32_t *cnt;       // [n_tiles] kept pods of the tile this pass
  uint32_t *done;      // [n_tiles] at a cluster's first tile: its tiles finished this pass (the last one sets it back to 0)
  uint32_t *runs;      // [n_tiles][kHugeTile] the tile's kept pod indices, ascending
  uint32_t *stash;     // [n_tiles][kHugeTile] ... in arrival order
};

// first i in [lo, n) with s[i] >= x, given s ascending and s[lo - 1] < x: galloping, then binary search in the last step
__device__ __forceinline__ uint32_t gallop_lower_bound(const uint32_t *s, uint32_t lo, uint32_t n, uint32_t x) {
  uint32_t hi = lo, step = 1;
  while (hi < n && s[hi] < x) { lo = hi + 1; hi += step; step <<= 1; }
  hi = min(hi, n);
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (s[mid] < x) lo = mid + 1; else hi = mid; }
  return lo;
}

// One CTA per tile of the huge RayClusters.  kInc: only the dirty ones.
template <bool kInc>
__global__ void __launch_bounds__(kHugeThreads) k_huge_tiles(Decide2Args a, HugeDev h) {
  __shared__ uint32_t s_idx[kHugeTile];
  __shared__ uint32_t s_warp[kHugeThreads / 32];
  __shared__ uint32_t s_go;
  const ScratchDev &sc = a.sc;
  const uint4 t = h.tiles[blockIdx.x];
  if (t.x == KR_EMPTY32) return;  // a free reserve entry, or a tile k_inc_grow retired (KR_OPT_HUGE_GROWTH)
  const uint32_t c = t.x, r0 = t.y;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t S = sc.bucket_stride;
  const uint32_t epoch = kInc ? inc_epoch_of(sc) : 0u;
  const uint4 dyn = __ldcg(&sc.cl_dyn[c]);
  const uint32_t P = dyn.x;
  if (tid == 0) {
    // k_large_sort's choice, from state only earlier grids write (this grid flags nothing void): every tile of the cluster makes
    // the same one, so either all of them count themselves in below or none does
    const uint32_t cap = __ldcg(&sc.lg[c].y);
    bool go = !KR_ATTEMPT_VOID(a.r.totals);
    if (kInc) go = go && !__ldcg(&sc.inc[KR_INC_VOID]) && !__ldcg(&sc.inc[KR_INC_STRUCTURAL]) && __ldcg(&sc.dirty_flag[c]) == epoch;
    const bool wide = a.s.c_group_cnt[c] > KR_SMEM_GROUPS;
    s_go = go && (P > S ? P - S <= cap : wide);
    if (!s_go && r0 == 0) sc.lg[c].w = 0;  // not taken this pass: k_huge_merge and the decide leave it alone
  }
  __syncthreads();
  if (!s_go) return;
  const bool lost = kInc && dyn.y == epoch;  // the cluster lost a row this epoch: the records of stamped rows are stale
  // ranks [r0, r1); each thread owns a contiguous run of them, so the kept records keep their arrival order
  const uint32_t r1 = min(P, r0 + (uint32_t)kHugeTile), n = r1 > r0 ? r1 - r0 : 0u;
  const uint32_t per = (n + kHugeThreads - 1) / kHugeThreads;
  const uint32_t j0 = r0 + min(tid * per, n), j1 = min(j0 + per, r1);
  uint32_t kept = 0;
  for (uint32_t j = j0; j < j1; j++) {
    const uint2 rec = __ldcg(rec_slot(sc, c, j));
    const bool keep = !lost || (rec.y & KR_ROW_FRESH) || __ldcg(&sc.stamp[rec.x]) != epoch;
    if (keep) {  // (the name and the replica index come from the Pod columns, as in k_large_sort)
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
  for (uint32_t w = 0; w < kHugeThreads / 32; w++) { const uint32_t v = s_warp[w]; before += w < warp ? v : 0u; total += v; }
  uint32_t o = before + x - kept;
  uint32_t *stash = h.stash + (size_t)blockIdx.x * kHugeTile;
  for (uint32_t j = j0; j < j1; j++) {
    const uint2 rec = __ldcg(rec_slot(sc, c, j));
    const bool keep = !lost || (rec.y & KR_ROW_FRESH) || __ldcg(&sc.stamp[rec.x]) != epoch;
    if (keep) { s_idx[o] = rec.x; stash[o] = rec.x; o++; }
  }
  block_sort_asc<kHugeThreads>(s_idx, total, tid);
  uint32_t *run = h.runs + (size_t)blockIdx.x * kHugeTile;
  for (uint32_t k = tid; k < total; k += kHugeThreads) run[k] = s_idx[k];
  if (tid == 0) {
    h.cnt[blockIdx.x] = total;
    __threadfence();  // the count is visible before this tile is counted in
    if (atomicAdd(&h.done[t.z], 1u) == t.w - 1) {  // the cluster's last tile: every count of the cluster is in
      __threadfence();
      uint32_t sum = 0;
      for (uint32_t i = t.z; i < t.z + t.w; i++) sum += __ldcg(&h.cnt[i]);
      const uint32_t seg = atomicAdd(&sc.inc[KR_INC_LSEG], sum);
      sc.lg[c].z = seg; sc.lg[c].w = sum | KR_LG_OWNED;  // (k_huge_merge checks the segment against the pod count)
      h.done[t.z] = 0;
    }
  }
}

// One CTA per tile of the huge RayClusters that k_huge_tiles took: the tile's pods into their places of the List-order segment.
template <bool kInc>
__global__ void __launch_bounds__(kHugeThreads) k_huge_merge(Decide2Args a, HugeDev h) {
  __shared__ uint32_t s_run[kHugeTile];  // another tile's run
  const ScratchDev &sc = a.sc;
  const uint4 t = h.tiles[blockIdx.x];
  if (t.x == KR_EMPTY32) return;  // (as in k_huge_tiles)
  const uint32_t c = t.x, me = blockIdx.x, tid = threadIdx.x;
  const uint4 l = __ldcg(&sc.lg[c]);  // (written by k_huge_tiles: an earlier grid)
  if (!(l.w & KR_LG_OWNED)) return;
  const uint32_t seg = l.z, total = l.w & ~KR_LG_OWNED;
  if ((uint64_t)seg + total > a.n.n_pods) {  // cannot happen while the regions hold distinct live rows; void rather than overrun
    if (me == t.z && tid == 0) {
      sc.lg[c].w = 0;  // (the cluster's other CTAs return here too, whichever value they read)
      if (kInc) atomicOr(&sc.inc[KR_INC_VOID], KR_FULL_ARENA); else KR_MARK_ATTEMPT_VOID(a.r.totals);
    }
    return;
  }
  const uint32_t n_me = __ldcg(&h.cnt[me]);
  const uint32_t *mine = h.runs + (size_t)me * kHugeTile;
  const uint32_t k0 = tid * kHugePer;
  uint32_t v[kHugePer], at[kHugePer];
#pragma unroll
  for (int i = 0; i < kHugePer; i++) { v[i] = k0 + i < n_me ? __ldcg(mine + k0 + i) : 0xFFFFFFFFu; at[i] = k0 + i; }
  uint32_t base = 0;  // kept pods of the cluster's earlier tiles: they precede this tile's in arrival order
  for (uint32_t u = t.z; u < t.z + t.w; u++) {
    const uint32_t n_u = __ldcg(&h.cnt[u]);
    if (u < me) base += n_u;
    if (u == me || n_u == 0) continue;  // (the same for the whole CTA)
    __syncthreads();  // the previous run is no longer read
    const uint32_t *run = h.runs + (size_t)u * kHugeTile;
    for (uint32_t k = tid; k < n_u; k += kHugeThreads) s_run[k] = __ldcg(run + k);
    __syncthreads();
    if (k0 >= n_me) continue;
    uint32_t lo = 0;
#pragma unroll
    for (int i = 0; i < kHugePer; i++) { lo = gallop_lower_bound(s_run, lo, n_u, v[i]); at[i] += lo; }
  }
#pragma unroll
  for (int i = 0; i < kHugePer; i++) if (k0 + i < n_me) a.r.sorted_pod_idx[seg + at[i]] = v[i];
  if (kInc) {
    // the bucket and region compacted in arrival order, FRESH marks cleared; pos[] follows the records that moved
    const uint32_t *stash = h.stash + (size_t)me * kHugeTile;
    for (uint32_t k = tid; k < n_me; k += kHugeThreads) {
      const uint32_t p = __ldcg(stash + k);
      const uint4 row = __ldcg(&sc.rows[p]);
      *rec_slot(sc, c, base + k) = make_uint2(p, row.w);
      sc.pos[p] = base + k;
    }
    if (me == t.z && tid == 0) { sc.cl_dyn[c].x = total; sc.cl_dyn[c].y = 0u; }
  }
}

}  // namespace kr

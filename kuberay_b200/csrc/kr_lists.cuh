// kr_lists.cuh — every RayCluster's full pod list on the bucket pipeline (KR_OPT_BUCKET_POD_LISTS with kr_flags.fetch_pod_lists = 1).
// Part of the sm_90a kernel set of the batched reconcile engine; see kr_kernels.cuh for the pipeline overview.
//
// The bucket pipeline decides in arrival order and never lays the pods out in List order, but after the last decide kernel of a
// pass, full or incremental, every RayCluster's bucket (and region) holds exactly its live pods at ranks [0, cl_dyn.x) (an incremental
// decide stores its bucket back compacted) and its action run is final.  So the lists are built from that resident state, on stream M
// behind the decides, without touching them:
//   k_lists_init    per pod row: owner = n_clusters (in no bucket), action = KEEP;
//   k_lists_owner   one warp per RayCluster: owner = c for every record of its bucket and region (rec_slot), and the codes of its
//                   action run [act_start, act_start + act_cnt) scattered to their pods;
//   k_hist / k_scan_rows / k_scatter   the radix pipeline's stable LSD sort (kr_bucket.cuh) by owner, pod index as the value:
//                   RayClusters in row order, Pods in List (row) order inside each, then the orphans and free rows;
//   k_lists_gather  per list position: sorted_action along sorted_pod_idx, and pod_start as the first position of each owner.
// The result is byte for byte the sort pipeline's sorted_pod_idx, sorted_action and pod_start.  pod_start goes to its own array
// ([n_clusters + 1] in the results arena): the cluster records keep 0 there, as everywhere on the bucket pipeline, and the fetch
// patches the host's records, since an incremental epoch shifts the start of RayClusters it did not re-decide.
// Scratch: owner in keys[0] (the sort ping-pongs through keys / vals / hist / row_total, all of them the sort pipeline's only), the
// per-pod action in act_tmp_code (the decides' per-pass staging, dead once they are done).  sorted_pod_idx and sorted_action are
// also the per-cluster kernels' scratch segments (kr_large.cuh, kr_huge.cuh), but each pass reads only segments it wrote itself:
// k_decide_large reads a segment only once k_large_sort or k_huge_tiles of the same pass marked it KR_LG_OWNED, and both clear that
// mark first for every RayCluster they take.  So the lists, written last, are what the fetch copies, and the next pass overwrites
// them freely.
#pragma once

#include "kr_incr.cuh"

namespace kr {

struct ListsArgs {
  SnapDev s; ScratchDev sc; ResDev r; Sizes n;
  uint32_t *owner;      // [n_pods] RayCluster of each pod row, n_clusters for none: the sort's keys
  uint8_t *act;         // [n_pods] KR_ACT_* of each pod row in a RayCluster
  uint32_t *pod_start;  // [n_clusters + 1] first list position of each RayCluster; [n_clusters]: of the orphans
  int inc;              // an incremental pass (a void attempt is flagged in sc.inc, not in the totals)
};

// The attempt is void: its buckets and action runs may point anywhere, and the pass that follows builds the lists again.
__device__ __forceinline__ bool lists_void(const ListsArgs &a) {
  return a.inc ? (__ldcg(&a.sc.inc[KR_INC_VOID]) | __ldcg(&a.sc.inc[KR_INC_STRUCTURAL])) != 0u : KR_ATTEMPT_VOID(a.r.totals);
}

// One thread per pod row.
__global__ void __launch_bounds__(256) k_lists_init(ListsArgs a) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.n.n_pods) return;
  a.owner[p] = a.n.n_clusters;
  a.act[p] = KR_ACT_KEEP;
}

// One warp per RayCluster.
__global__ void __launch_bounds__(256) k_lists_owner(ListsArgs a) {
  const uint32_t c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, Np = a.n.n_pods;
  if (c >= a.n.n_clusters || lists_void(a)) return;
  const uint32_t P = a.sc.cl_dyn[c].x;
  for (uint32_t j = lane; j < P; j += 32) {
    const uint2 *rec = rec_slot(a.sc, c, j);
    const uint32_t p = rec ? rec->x : Np;
    if (p < Np) a.owner[p] = c;
  }
  const uint32_t a0 = a.r.act_start[c], na = a.r.act_cnt[c];
  if ((uint64_t)a0 + na > Np) return;  // (cannot happen in an attempt that stands: the decide voids it)
  for (uint32_t i = lane; i < na; i += 32) {
    const uint32_t p = a.r.act_pod_idx[a0 + i];
    if (p < Np) a.act[p] = a.r.act_code[a0 + i];
  }
}

// One thread per list position i in [0, n_pods]; keys: the owners in list order (the sort's last output).
__global__ void __launch_bounds__(256) k_lists_gather(ListsArgs a, const uint32_t *__restrict__ keys) {
  const uint32_t Np = a.n.n_pods, Nc = a.n.n_clusters, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > Np) return;
  // position i starts the lists of the owners after the previous position's, up to its own (Np: up to the orphans' segment)
  const uint32_t k = i < Np ? keys[i] : Nc;
  for (uint32_t c = i ? keys[i - 1] + 1 : 0u; c <= k; c++) a.pod_start[c] = i;
  if (i < Np) {
    const uint32_t p = a.r.sorted_pod_idx[i];
    a.r.sorted_action[i] = k < Nc ? a.act[p] : (a.s.p_packed[p] & KR_PP_TOMBSTONE) ? (uint8_t)KR_ACT_TOMBSTONE : (uint8_t)KR_ACT_ORPHAN;
  }
}

}  // namespace kr

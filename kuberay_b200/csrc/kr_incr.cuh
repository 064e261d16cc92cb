// kr_incr.cuh — device-side incremental epochs on top of the bucket pipeline (kr_bucket2.cuh).
// Part of the sm_90a kernel set of the batched reconcile engine; see kr_kernels.cuh for the pipeline overview.
//
// A full pass leaves everything a later pass needs resident on the device: the join tables, every RayCluster's bucket of pod
// records and its {count, first head} cell, the 128-byte input records, the digests and the result records.  The informer
// events of an epoch (raycluster_controller.go:1525-1533 watches RayClusters and the Pods they own) then arrive as
//   * pod rows     kr_snapshot_commit_pod_rows / _values   -> k_inc_retire runs on the rows' OLD values before the patch lands:
//                                                             it takes each row out of the orphan count / workersToDelete
//                                                             resolutions, stamps it and marks the RayCluster it was in dirty;
//   * object rows  kr_snapshot_commit_parts(KR_PART_OBJECTS) -> uploaded beside the resident tables and diffed by k_inc_objects:
//                                                             changed RayCluster / group / head-aux rows mark their cluster
//                                                             dirty, a changed table key or CSR offset makes the epoch
//                                                             "structural" (the next pass is a full one).
// The pass then touches only what changed:
//   k_inc_admit    (one thread per touched row) runs the selector match of k_match2 on the row's NEW values and appends the
//                  record (marked KR_ROW_FRESH) to its RayCluster's bucket — marking that RayCluster dirty as well;
//   k_inc_refresh  (launched by the object commit itself, behind its diff kernel) rewrites the 128-byte input record of the RayClusters whose
//                  RayCluster / group rows changed;
//   k_decide2<K>   phase 2: the decide kernel over the dirty list.  Each warp first drops the records of stamped rows from its bucket (stored back compacted, arrival order
//                  kept) and recomputes the first head; then decides as in a full pass (digests are resident, so the Recreate
//                  gate is decided in place); a cluster keeps its places in the action list / create arena while they suffice;
//                  and packs the cluster's changed records for one small D2H copy (IncStage).
// Results are bit-identical to a full pass over the same state (tests/test_live_arena.py, tests/test_packer.py run every epoch
// against the oracle); anything the resident state cannot absorb — structural object changes, a bucket or arena overflow — voids
// the attempt and the engine takes the full pass instead.
#pragma once

#include "kr_bucket2.cuh"

namespace kr {

__device__ __forceinline__ uint32_t inc_epoch(const ScratchDev &sc) { return inc_epoch_of(sc); }

__device__ __forceinline__ void mark_dirty(const ScratchDev &sc, uint32_t c, uint32_t epoch) {
  if (atomicExch(&sc.dirty_flag[c], epoch) != epoch) sc.dirty_list[atomicAdd(&sc.inc[KR_INC_DIRTY], 1u)] = c;
}

// (namespace, ray.io/cluster) -> cluster idx, table flags and the name of worker group 0 (the probe of k_match2)
__device__ __forceinline__ bool cl_probe(const ScratchDev &sc, uint32_t ns, uint32_t name, uint32_t &c, uint32_t &cflags, uint32_t &gname0) {
  if (name == 0) return false;
  uint32_t i = hash_pair(ns, name) & sc.cl_mask;
  while (true) {
    const uint4 q = __ldcg(&sc.cl_slots[i]);
    if (q.x == name && q.y == ns) { c = q.w >> 2; cflags = q.w & 3u; gname0 = q.z; return true; }
    if (q.x == KR_EMPTY32 && q.y == KR_EMPTY32) return false;
    i = (i + 1) & sc.cl_mask;
  }
}

// Touches pod row p once per epoch: stamps it and appends it to the touched list (k_inc_admit re-matches it), then marks the
// RayCluster its current device columns probe to dirty, or takes it out of the orphan count.  Those columns must still hold the
// values its resident record was built from.  Returns false when p was touched already this epoch or was appended since the last
// pass (n_resident rows existed then: a newer row holds nothing resident); else ns / nm are its namespace and name.
__device__ __forceinline__ bool inc_touch(const SnapDev &s, const ScratchDev &sc, const ResDev &r, uint32_t p, uint32_t epoch, uint32_t n_resident, uint32_t &ns, uint32_t &nm) {
  if (atomicExch(&sc.stamp[p], epoch) == epoch) return false;  // touched twice since the last pass: retired already
  const uint32_t ti = atomicAdd(&sc.inc[KR_INC_TOUCHED], 1u);
  sc.touched[ti] = p; sc.touched_old[ti] = KR_EMPTY32;
  if (p >= n_resident) return false;
  ns = s.p_ns_id[p];
  const uint32_t cn = s.p_cluster_name_id[p];
  nm = s.p_name_id[p];
  const uint32_t pk = s.p_packed[p];
  uint32_t c = 0, cflags, gname0;
  if (cl_probe(sc, ns, cn, c, cflags, gname0)) { mark_dirty(sc, c, epoch); sc.touched_old[ti] = c; }  // (k_inc_admit rewrites the record in place if the row stays)
  else if (!(pk & KR_PP_TOMBSTONE)) atomicSub(&r.totals[1], 1u);  // it was an orphan
  return true;
}

// ------------------------------------------------------------------------------------------------ k_inc_retire
// One thread per committed row, launched in front of the patch kernel: the device columns still hold the row's previous
// values.  n_resident = pod rows that existed at the last pass (rows appended since hold nothing to retire).
__global__ void __launch_bounds__(256) k_inc_retire(const uint32_t *rows, uint32_t n_rows, SnapDev s, ScratchDev sc, ResDev r, Sizes n, uint32_t n_resident, int has_wtd) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rows) return;
  const uint32_t p = rows[i];
  uint32_t ns, nm;
  if (!inc_touch(s, sc, r, p, inc_epoch(sc), n_resident, ns, nm)) return;
  if (has_wtd) {  // names that resolved to this row: (namespace, name) is unique among live Pods, so nothing else holds them
    const uint32_t hk = hash_pair(ns, nm);
    if ((__ldcg(&sc.wt_bits[(hk & sc.wt_bits_mask) >> 5]) & (1u << (hk & 31))) && (__ldcg(&sc.wt_bits[(bloom2(hk) & sc.wt_bits_mask) >> 5]) & (1u << (bloom2(hk) & 31)))) {
      const uint64_t k = key2(ns, nm);
      uint32_t j = hk & sc.wt_mask;
      uint64_t kk = __ldcg(&sc.wt_keys[j]);
      while (kk != KR_EMPTY64) {
        if (kk == k) {
          for (uint32_t e = sc.wt_head[j]; e != KR_EMPTY32; e = sc.wt_next[e]) atomicCAS(&r.wtd_pod_idx[e], p, 0xFFFFFFFFu);
          break;
        }
        j = (j + 1) & sc.wt_mask;
        kk = __ldcg(&sc.wt_keys[j]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ workersToDelete edits
// KR_OPT_WTD_EDITS: an epoch whose object commits changed a workersToDelete list (a name, a length, an offset) rebuilds the name
// table in front of k_inc_admit, after every commit of the epoch has landed:
//   k_inc_wtd_release  touches every row a name of the OLD table resolved to (wtd_pod_idx as the last pass left it);
//   k_inc_wtd_clear    empties the table and its Bloom bitmap and sets the new resolutions to -1;
//   k_inc_wtd_insert   inserts the new names (k_build_tables' group part);
//   k_inc_wtd_resolve  probes every pod row against them, resolves wtd_pod_idx as k_match2 does and touches each row that hits.
// k_inc_admit then rewrites each touched record with KR_ROW_WTD_OWN from the new table, and the decide kernels re-decide the
// RayClusters those rows sit in.  k_inc_retire of this epoch's committed rows ran against the old table: its writes to wtd_pod_idx
// are cleared here, and a committed row is stamped already, so the touches below skip it.
__global__ void __launch_bounds__(256) k_inc_wtd_release(SnapDev s, ScratchDev sc, ResDev r, uint32_t n_wtd_old, uint32_t n_resident) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_wtd_old) return;
  const uint32_t p = r.wtd_pod_idx[e];
  uint32_t ns, nm;
  if (p != 0xFFFFFFFFu) inc_touch(s, sc, r, p, inc_epoch(sc), n_resident, ns, nm);
}

__global__ void __launch_bounds__(256) k_inc_wtd_clear(ScratchDev sc, ResDev r, uint32_t n_wtd) {
  const uint32_t stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t i = t0; i <= sc.wt_mask; i += stride) { sc.wt_keys[i] = KR_EMPTY64; sc.wt_head[i] = KR_EMPTY32; }
  for (uint32_t i = t0; i < (sc.wt_bits_mask + 1) >> 5; i += stride) sc.wt_bits[i] = 0u;
  for (uint32_t i = t0; i < n_wtd; i += stride) r.wtd_pod_idx[i] = 0xFFFFFFFFu;
}

__global__ void __launch_bounds__(256) k_inc_wtd_insert(SnapDev s, ScratchDev sc, Sizes n) {
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n.n_groups; t += gridDim.x * blockDim.x) wt_insert_group(s, sc, t);
}

// grid-stride over the pod rows: 8 bytes per row and a Bloom test in shared memory (the bitmap copied per CTA, as k_match2 does).
// Only names from entry `first_name` on are resolved, and only rows that hit one of them are touched (0: every name, the rebuild;
// the first new name: the names of RayClusters an epoch appended, KR_OPT_CLUSTER_CREATES).
__global__ void __launch_bounds__(256) k_inc_wtd_resolve(SnapDev s, ScratchDev sc, ResDev r, Sizes n, uint32_t n_resident, uint32_t first_name) {
  extern __shared__ uint32_t sm_bits[];
  const uint32_t words = (sc.wt_bits_mask + 1) >> 5;
  for (uint32_t i = threadIdx.x; i < words; i += blockDim.x) sm_bits[i] = __ldcg(&sc.wt_bits[i]);
  __syncthreads();
  const uint32_t epoch = inc_epoch(sc);
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n.n_pods; p += gridDim.x * blockDim.x) {
    const uint32_t ns = __ldg(&s.p_ns_id[p]), nm = __ldg(&s.p_name_id[p]);
    const uint32_t hk = hash_pair(ns, nm), h2 = bloom2(hk);
    if (!(sm_bits[(hk & sc.wt_bits_mask) >> 5] & (1u << (hk & 31))) || !(sm_bits[(h2 & sc.wt_bits_mask) >> 5] & (1u << (h2 & 31)))) continue;
    const uint64_t k = key2(ns, nm);
    uint32_t j = hk & sc.wt_mask;
    uint64_t kk = __ldcg(&sc.wt_keys[j]);
    while (kk != KR_EMPTY64) {
      if (kk == k) {
        bool hit = false;
        for (uint32_t e = __ldcg(&sc.wt_head[j]); e != KR_EMPTY32; e = __ldcg(&sc.wt_next[e]))
          if (e >= first_name) { atomicMin(&r.wtd_pod_idx[e], p); hit = true; }
        uint32_t ns2, nm2;
        if (hit) inc_touch(s, sc, r, p, epoch, n_resident, ns2, nm2);
        break;
      }
      j = (j + 1) & sc.wt_mask;
      kk = __ldcg(&sc.wt_keys[j]);
    }
  }
}

// ------------------------------------------------------------------------------------------------ k_inc_objects
// Diff of a KR_PART_OBJECTS upload (staged beside the resident tables) against the resident copy, then the copy into place.
enum { KR_OC_COPY = 0, KR_OC_STRUCT = 1, KR_OC_CLUSTER = 2, KR_OC_GROUP = 3, KR_OC_HEAD = 4, KR_OC_HEADKEY = 5 };
enum { KR_MAP_CLUSTER = 1, KR_MAP_GROUP = 2, KR_MAP_NAME = 3 };

// x among the n ascending values of v
__device__ __forceinline__ bool sorted_has(const uint32_t *v, uint32_t n, uint32_t x) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (__ldg(&v[mid]) < x) lo = mid + 1; else hi = mid; }
  return lo < n && __ldg(&v[lo]) == x;
}
static constexpr int kMaxObjCols = 48;
struct ObjDiffArgs {
  const uint8_t *src[kMaxObjCols];   // staged (new) column
  const uint32_t *rowlist[kMaxObjCols];  // NULL: staged row k is resident row k (a whole-table upload); else staged row k is resident row rowlist[k]
                                         // (kr_snapshot_commit_object_rows: only the rewritten rows travel, packed)
  uint8_t *dst[kMaxObjCols];         // resident column
  uint32_t first[kMaxObjCols + 1];   // flat index of the column's first row (prefix sums of the new row counts)
  uint32_t rows_old[kMaxObjCols];    // rows the resident column held
  uint16_t row_bytes[kMaxObjCols];
  uint8_t cls[kMaxObjCols];
  uint8_t cls_new[kMaxObjCols];      // class of a row at or past rows_old (KR_OPT_CLUSTER_CREATES: a row of an appended RayCluster)
  // KR_OPT_CLUSTER_DELETES, an object commit that renumbered RayClusters (a row map): per column 0, or KR_MAP_CLUSTER (the rows of
  // init are new RayCluster rows, classed like rows past rows_old), KR_MAP_GROUP / KR_MAP_NAME (rows from shift_from on were
  // shifted: row k compares against the resident row src[k - shift_from], KR_EMPTY32: a row of a moved or created RayCluster, classed
  // like a row past rows_old).  A map commit launches the diff twice, because a shifted row reads a resident row another thread
  // overwrites: map_pass 1 diffs only the shifted rows and copies nothing, map_pass 2 copies them without a diff and diffs the rest.
  uint8_t map_kind[kMaxObjCols];
  uint32_t shift_from[kMaxObjCols];
  const uint32_t *init; uint32_t n_init;
  const uint32_t *gsrc, *wsrc;
  int map_pass;
  int n_cols;
  const uint32_t *g_cluster_idx_new;  // staged g_cluster_idx (group row -> RayCluster)
  const uint32_t *h_pod_idx_new;      // staged h_pod_idx
  const uint32_t *h_pod_idx_old;      // resident h_pod_idx (read before this launch's copy of that column: it is diffed LAST)
  uint32_t n_heads_old;
};

__device__ __forceinline__ void mark_pod_cluster_dirty(const SnapDev &s, const ScratchDev &sc, const Sizes &n, uint32_t p, uint32_t epoch) {
  if (p >= n.n_pods) return;
  uint32_t c = 0, cflags, gname0;
  if (cl_probe(sc, s.p_ns_id[p], s.p_cluster_name_id[p], c, cflags, gname0)) mark_dirty(sc, c, epoch);
}

__global__ void __launch_bounds__(256) k_inc_objects(ObjDiffArgs a, SnapDev s, ScratchDev sc, Sizes n) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.first[a.n_cols]) return;
  int lo = 0, hi = a.n_cols - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (a.first[mid] <= t) lo = mid; else hi = mid - 1; }
  const int col = lo;
  const uint32_t k_st = t - a.first[col], rb = a.row_bytes[col];
  const uint32_t row = a.rowlist[col] ? a.rowlist[col][k_st] : k_st;
  const uint8_t *src = a.src[col] + (size_t)k_st * rb;
  uint8_t *dst = a.dst[col] + (size_t)row * rb;
  const uint8_t *old = dst;  // the resident row this one is diffed against
  bool past = row >= a.rows_old[col];
  if (a.map_pass) {
    const uint8_t mk = a.map_kind[col];
    const bool shifted = mk >= KR_MAP_GROUP && row >= a.shift_from[col];
    if (shifted && a.map_pass == 2) { for (uint32_t k = 0; k < rb; k++) dst[k] = src[k]; return; }  // (diffed by the first launch)
    if (!shifted && a.map_pass == 1) return;
    if (shifted) {  // (a kept RayCluster's row may land past the old count when groups or names were added before it)
      const uint32_t o = (mk == KR_MAP_GROUP ? a.gsrc : a.wsrc)[row - a.shift_from[col]];
      past = o == KR_EMPTY32;
      if (!past) old = a.dst[col] + (size_t)o * rb;
    } else if (mk == KR_MAP_CLUSTER && !past) past = sorted_has(a.init, a.n_init, row);
  }
  const uint8_t cls = past ? a.cls_new[col] : a.cls[col];
  bool differ = past;
  if (!differ) {
    if ((rb & 3u) == 0) { for (uint32_t k = 0; k < rb; k += 4) differ |= *reinterpret_cast<const uint32_t *>(src + k) != *reinterpret_cast<const uint32_t *>(old + k); }
    else for (uint32_t k = 0; k < rb; k++) differ |= src[k] != old[k];
  }
  if (!differ) return;
  const uint32_t epoch = inc_epoch(sc);
  switch (cls) {
    case KR_OC_STRUCT: atomicOr(&sc.inc[KR_INC_STRUCTURAL], KR_FULL_STRUCTURAL); break;
    case KR_OC_CLUSTER: if (row < n.n_clusters) { sc.obj_flag[row] = epoch; mark_dirty(sc, row, epoch); } break;
    case KR_OC_GROUP: { const uint32_t c = a.g_cluster_idx_new[k_st]; if (c < n.n_clusters) { sc.obj_flag[c] = epoch; mark_dirty(sc, c, epoch); } break; }
    case KR_OC_HEADKEY:  // (the host compared the keys as well and rebuilds the pod -> row table); both pods' clusters see a different head-aux row now
    case KR_OC_HEAD:
      mark_pod_cluster_dirty(s, sc, n, a.h_pod_idx_new[k_st], epoch);
      if (row < a.n_heads_old) mark_pod_cluster_dirty(s, sc, n, a.h_pod_idx_old[row], epoch);
      break;
    default: break;
  }
  if (cls == KR_OC_HEADKEY || a.map_pass == 1) return;  // (copied by k_inc_objects_keys once every head row has read the old key)
  if ((rb & 3u) == 0) { for (uint32_t k = 0; k < rb; k += 4) *reinterpret_cast<uint32_t *>(dst + k) = *reinterpret_cast<const uint32_t *>(src + k); }
  else for (uint32_t k = 0; k < rb; k++) dst[k] = src[k];
}

// second step of the object diff: h_pod_idx into place (every head row of k_inc_objects read the old keys first)
__global__ void __launch_bounds__(256) k_inc_objects_keys(const uint32_t *src, uint32_t *dst, uint32_t n, const uint32_t *rowlist) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) dst[rowlist ? rowlist[t] : t] = src[t];
}

// ------------------------------------------------------------------------------------------------ head-aux table rebuild
// pod idx -> head-aux row, when an epoch changed h_pod_idx (a head Pod came or went): clear, then insert (k_build_tables' third part)
__global__ void __launch_bounds__(256) k_inc_aux_clear(ScratchDev sc) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= sc.aux_mask; i += gridDim.x * blockDim.x) { sc.aux_keys[i] = KR_EMPTY32; sc.aux_vals[i] = KR_EMPTY32; }
}
__global__ void __launch_bounds__(256) k_inc_aux_insert(SnapDev s, ScratchDev sc, Sizes n) {
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n.n_heads; t += gridDim.x * blockDim.x) {
    const uint32_t p = s.h_pod_idx[t];
    uint32_t i = mix32(p) & sc.aux_mask;
    while (true) {
      const uint32_t prev = atomicCAS(&sc.aux_keys[i], KR_EMPTY32, p);
      if (prev == KR_EMPTY32 || prev == p) { atomicMin(&sc.aux_vals[i], t); break; }
      i = (i + 1) & sc.aux_mask;
    }
  }
}

// every RayCluster whose Recreate gate reads a digest, when the spec JSON was committed again (the digests are being recomputed)
__global__ void __launch_bounds__(256) k_inc_mark_recreate(SnapDev s, ScratchDev sc, Sizes n) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < n.n_clusters && (s.c_flags[c] & KR_CF_UPGRADE_RECREATE)) mark_dirty(sc, c, inc_epoch(sc));
}

// ------------------------------------------------------------------------------------------------ spec rows
// kr_snapshot_commit_spec_rows: the device pulls the rewritten muted-spec JSON ranges out of the mapped pinned arena (one CTA per
// row, 16-byte loads over PCIe) and sets the rows' c_json_off / c_json_len from the uploaded list; the next pass hashes only the
// listed messages (the hash kernels take the list as their order), marks the listed Recreate-gated RayClusters dirty and gathers
// the new digests for the fetch.
__global__ void __launch_bounds__(128) k_spec_pull(const uint32_t *__restrict__ rows, const uint64_t *__restrict__ offs, const uint32_t *__restrict__ lens,
                                                   const uint8_t *__restrict__ h_json, uint8_t *__restrict__ d_json, uint64_t *c_json_off, uint32_t *c_json_len) {
  const uint32_t i = blockIdx.x;
  const uint64_t off = offs[i];
  const uint32_t len = lens[i];
  const uint4 *src = reinterpret_cast<const uint4 *>(h_json + off);
  uint4 *dst = reinterpret_cast<uint4 *>(d_json + off);
  for (uint32_t k = threadIdx.x; k < (len + 15) / 16; k += blockDim.x) dst[k] = src[k];
  if (threadIdx.x == 0) { c_json_off[rows[i]] = off; c_json_len[rows[i]] = len; }
}

// kr_snapshot_commit_json_moves: the listed RayClusters' unchanged muted-spec JSON moves inside the device arena, from the range the
// record holds (src) to the host's new one (dst).  Sources and destinations may overlap in any direction (a compaction re-places the
// blobs in row order), so the copy goes out of place: k_json_move_gather copies every listed range into the scratch at its
// destination offset, then k_json_move_scatter copies the destination ranges back and sets the rows' c_json_off / c_json_len.  One
// CTA per row, 16-byte loads; the padded destinations are disjoint, so no two CTAs write the same bytes.
__global__ void __launch_bounds__(128) k_json_move_gather(const uint64_t *__restrict__ src, const uint64_t *__restrict__ dst, const uint32_t *__restrict__ lens,
                                                          const uint8_t *__restrict__ d_json, uint8_t *__restrict__ scratch) {
  const uint32_t i = blockIdx.x;
  const uint4 *from = reinterpret_cast<const uint4 *>(d_json + src[i]);
  uint4 *to = reinterpret_cast<uint4 *>(scratch + dst[i]);
  for (uint32_t k = threadIdx.x; k < (lens[i] + 15) / 16; k += blockDim.x) to[k] = from[k];
}
__global__ void __launch_bounds__(128) k_json_move_scatter(const uint32_t *__restrict__ rows, const uint64_t *__restrict__ dst, const uint32_t *__restrict__ lens,
                                                           const uint8_t *__restrict__ scratch, uint8_t *__restrict__ d_json, uint64_t *c_json_off, uint32_t *c_json_len) {
  const uint32_t i = blockIdx.x;
  const uint64_t off = dst[i];
  const uint32_t len = lens[i];
  const uint4 *from = reinterpret_cast<const uint4 *>(scratch + off);
  uint4 *to = reinterpret_cast<uint4 *>(d_json + off);
  for (uint32_t k = threadIdx.x; k < (len + 15) / 16; k += blockDim.x) to[k] = from[k];
  if (threadIdx.x == 0) { c_json_off[rows[i]] = off; c_json_len[rows[i]] = len; }
}

// the listed RayClusters whose Recreate gate reads the digest (k_inc_mark_recreate's test, for the listed rows only)
__global__ void __launch_bounds__(256) k_inc_mark_rows(SnapDev s, ScratchDev sc, const uint32_t *__restrict__ rows, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && (s.c_flags[rows[i]] & KR_CF_UPGRADE_RECREATE)) mark_dirty(sc, rows[i], inc_epoch(sc));
}

// the listed digests, packed in list order (two 16-byte pieces per digest)
__global__ void __launch_bounds__(256) k_inc_digest_gather(const uint32_t *__restrict__ rows, uint32_t n, const char *__restrict__ hash, char *__restrict__ out) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 2 * n) return;
  reinterpret_cast<uint4 *>(out)[t] = reinterpret_cast<const uint4 *>(hash + 32 * (size_t)rows[t >> 1])[t & 1];
}

// ------------------------------------------------------------------------------------------------ k_inc_refresh
// Input records (cl_in) of the RayClusters one of whose RayCluster / group rows an object commit changed (grid-stride over the
// dirty list as the commits left it; clusters k_inc_admit adds later had no object change).
__global__ void __launch_bounds__(256) k_inc_refresh(SnapDev s, ScratchDev sc) {
  const uint32_t n_dirty = __ldcg(&sc.inc[KR_INC_DIRTY]);
  const uint32_t epoch = inc_epoch(sc);
  if (__ldcg(&sc.inc[KR_INC_STRUCTURAL])) return;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_dirty; i += gridDim.x * blockDim.x) {
    const uint32_t c = sc.dirty_list[i];
    if (__ldcg(&sc.obj_flag[c]) == epoch) write_cl_in(s, sc, c, s.c_group_off[c], s.c_group_cnt[c]);
  }
}

// ------------------------------------------------------------------------------------------------ k_inc_admit
// KR_OPT_LARGE_GROWTH: the grow buffer (16-byte words) holds the grow list {cluster, old region offset, old capacity, -} at
// [0, KR_GROW_MAX), k_inc_grow's result {cluster, offset, capacity, newly listed} at [KR_GROW_MAX, 2 KR_GROW_MAX), then the spill:
// per record a pair {pod, rank, cluster, -}, {pod, slot << 16 | flags, -, -} (the 8-byte record).
static constexpr uint32_t kGrowResult = KR_GROW_MAX, kGrowSpill = 2 * KR_GROW_MAX;
static constexpr size_t kGrowBytes = 16 * ((size_t)kGrowSpill + 2 * (size_t)KR_GROW_SPILL);

// A record of arrival rank `rank` that has no slot in RayCluster c's bucket or region waits in the spill for the region k_inc_grow
// gives c.  The thread that meets the first rank past the room (exactly one per cluster and epoch: every record before the epoch fit)
// puts c on the grow list, with the region it has now.  false: the list or the spill is full (the attempt is void).
// Out of line, and given the few scratch fields it uses by value: k_inc_admit's loop keeps its registers, and no kernel parameter
// has its address taken (that would copy the whole parameter block to local memory in every thread of the launch).
__device__ __noinline__ bool grow_spill(const uint4 *lg, uint32_t *inc, uint32_t *pos, uint32_t stride, uint4 *grow, uint32_t c,
                                        uint32_t rank, uint2 rec) {
  const uint4 l = __ldcg(&lg[c]);  // (bound whenever the pass grows: 0 for an ordinary cluster)
  if (rank == stride + l.y) {
    const uint32_t j = atomicAdd(&inc[KR_INC_GROW], 1u);
    if (j >= KR_GROW_MAX) return false;
    grow[j] = make_uint4(c, l.x, l.y, 0u);
  }
  const uint32_t k = atomicAdd(&inc[KR_INC_SPILL], 1u);
  if (k >= KR_GROW_SPILL) return false;
  grow[kGrowSpill + 2 * k] = make_uint4(rec.x, rank, c, 0u);
  grow[kGrowSpill + 2 * k + 1] = make_uint4(rec.x, rec.y, 0u, 0u);
  pos[rec.x] = rank;
  return true;
}

// The selector match of k_match2 for the touched rows' new values (grid-stride over the touched list).  grow: the grow buffer
// (KR_OPT_LARGE_GROWTH), nullptr: a record without a slot voids the attempt.
__global__ void __launch_bounds__(256) k_inc_admit(SnapDev s, ScratchDev sc, ResDev r, Sizes n, int has_wtd, uint4 *grow) {
  const uint32_t n_touched = __ldcg(&sc.inc[KR_INC_TOUCHED]);
  const uint32_t epoch = inc_epoch(sc);
  if (__ldcg(&sc.inc[KR_INC_STRUCTURAL])) return;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_touched; i += gridDim.x * blockDim.x) {
    const uint32_t p = sc.touched[i], c_old = sc.touched_old[i];
    if (p >= n.n_pods) continue;
    const uint32_t ns = s.p_ns_id[p], cn = s.p_cluster_name_id[p], gn = s.p_group_name_id[p], nm = s.p_name_id[p], pk = s.p_packed[p];
    uint32_t c = n.n_clusters, cflags = 0, gname0 = 0;
    const bool matched = cl_probe(sc, ns, cn, c, cflags, gname0);
    uint32_t slot = KR_ROW_NO_GROUP, g0 = 0xFFFFFFFFu;
    if (matched && gn != 0) {
      if (gname0 == gn) slot = 0;
      else if (cflags & KR_CL_MULTI) {
        const uint4 rec = sc.cl_rec[c];
        g0 = rec.x;
        for (uint32_t gi = 1; gi < rec.y; gi++)
          if (s.g_name_id[g0 + gi] == gn) { slot = gi; break; }
      }
    }
    uint32_t flags = pk & (0x7FFu | KR_PP_TOMBSTONE);
    if (should_delete(pk)) flags |= KR_ROW_UNHEALTHY;
    if (has_wtd) {
      const uint32_t hk = hash_pair(ns, nm);
      if ((__ldcg(&sc.wt_bits[(hk & sc.wt_bits_mask) >> 5]) & (1u << (hk & 31))) && (__ldcg(&sc.wt_bits[(bloom2(hk) & sc.wt_bits_mask) >> 5]) & (1u << (bloom2(hk) & 31)))) {
        const uint64_t k = key2(ns, nm);
        uint32_t j = hk & sc.wt_mask;
        uint64_t kk = __ldcg(&sc.wt_keys[j]);
        while (kk != KR_EMPTY64) {
          if (kk == k) {
            for (uint32_t e = sc.wt_head[j]; e != KR_EMPTY32; e = sc.wt_next[e]) {
              atomicMin(&r.wtd_pod_idx[e], p);
              if (slot != KR_ROW_NO_GROUP) {
                if (g0 == 0xFFFFFFFFu) g0 = s.c_group_off[c];
                const uint32_t g = g0 + slot, off = s.g_wtd_off[g];
                if (e >= off && e < off + s.g_wtd_cnt[g]) flags |= KR_ROW_WTD_OWN;
              }
            }
            break;
          }
          j = (j + 1) & sc.wt_mask;
          kk = __ldcg(&sc.wt_keys[j]);
        }
      }
    }
    if (matched && c == c_old) {
      // the usual event — a status update: the row stays in its RayCluster, its record is rewritten where it sits and the row's
      // stamp is lifted (nothing of this cluster has to be dropped on its account)
      uint2 *at = rec_slot(sc, c, sc.pos[p]);  // (a record of a large RayCluster may sit in its region)
      if (!at) { sc.inc[KR_INC_VOID] = KR_FULL_OVERFLOW; continue; }
      *at = make_uint2(p, (slot << 16) | flags);
      sc.stamp[p] = 0u;
      continue;  // (k_inc_retire marked the cluster dirty)
    }
    if (c_old != KR_EMPTY32) sc.cl_dyn[c_old].y = epoch;  // the old cluster lost this row: its decide warp drops the stale record (the row stays stamped)
    if (!matched) {
      if (!(pk & KR_PP_TOMBSTONE)) atomicAdd(&r.totals[1], 1u);
      continue;
    }
    mark_dirty(sc, c, epoch);  // the row joined this cluster: a fresh record at the end of its bucket
    const uint32_t rank = atomicAdd(&sc.cl_dyn[c].x, 1u);
    const uint2 rec = make_uint2(p, (slot << 16) | flags | KR_ROW_FRESH);
    if (uint2 *at = rec_slot(sc, c, rank)) { *at = rec; sc.pos[p] = rank; }
    // (an ordinary RayCluster outgrew its bucket, a large one its region: k_inc_grow gives it a new one, or the full pass reclassifies.
    // Here and for a rewritten record without a slot above, a plain store of one constant keeps this kernel's registers (an atomicOr
    // of a selected bit cost three).  It is right only because k_inc_admit is the first kernel of an attempt that writes
    // KR_INC_VOID: a void site launched before it must not be added without making these stores atomicOr.  The host reads the
    // constant as KR_FULL_GROW_LIMIT when the pass could grow, the rewritten-record case included, which cannot happen while every
    // resident record has its slot.)
    else if (!grow || !grow_spill(sc.lg, sc.inc, sc.pos, sc.bucket_stride, grow, c, rank, rec)) sc.inc[KR_INC_VOID] = KR_FULL_OVERFLOW;
  }
}

// ------------------------------------------------------------------------------------------------ RayCluster creation and deletion
// KR_OPT_CLUSTER_CREATES / KR_OPT_CLUSTER_DELETES: an epoch whose object commit brought RayClusters into the fleet or renumbered
// them by swap-remove carries the commit's row map: the old rows `gone` that no RayCluster keeps (deleted, or moved to a row a
// deleted one vacated) and the new rows `init` that were created or moved (k_inc_objects copied them into place and marked them
// dirty).  RayClusters appended after the last resident row are the map without gone rows: every resident RayCluster, group and
// workersToDelete name kept its row, and only the steps that read `init` run.  KR_OPT_GROUP_EDITS adds regrouped RayClusters (same
// key and row, another list of worker groups): such a row is listed in both `gone` and `init`, so it is released with the old group
// table, stays on the dirty list at its index, is rekeyed with its new group 0 and offset, and starts again from an empty bucket;
// k_inc_admit then matches its Pods against the new group names (a Pod of a removed group stays among its Pods, in no group).  In
// front of k_inc_admit, each step launched only when its list is not empty:
//   k_inc_digest_move          first, ahead of the hash stream: the digests of moved RayClusters whose spec range stayed;
//   k_inc_clusters_release     one warp per gone row, while the cluster table still holds the old rows: touches every Pod in its
//                              bucket (k_inc_admit re-matches it against the new table: a Pod of a deleted RayCluster becomes an
//                              orphan, one of a moved RayCluster joins its new bucket) and takes the row's share out of the running
//                              totals, the way the incremental decide counts it (its act_cnt, its groups' n_create);
//   (the rebuild of the workersToDelete name table, when a resident name shifted, vanished or changed)
//   k_inc_orphan_adopt         touches every resident Pod row labelled for an `init` RayCluster — an orphan until now, or a Pod of an
//                              older RayCluster of the same key (the lowest row keeps such a key) — while the cluster table does not
//                              hold them yet: inc_touch takes an orphan out of the orphan count, and k_inc_admit appends it to its new
//                              bucket.  The host launches it only when RayClusters were created and the last pass counted orphans;
//   k_inc_clusters_translate   one CTA: a touched row whose old RayCluster is gone had no RayCluster (its stale record went with the
//                              bucket), and the dirty list drops the old rows at or past the new count (every entry below it names a
//                              RayCluster of the new numbering: a kept one, or one that k_inc_clusters_insert marks anyway);
//   k_inc_clusters_rekey       the cluster table cleared and rebuilt from every new row (cl_slots, cl_rec and cl_in: the offsets of
//                              the shifted groups), the lowest row keeping a duplicate key;
//   k_inc_groups_gather        the kept RayClusters' group records and create offsets from the first shifted group on, out of a
//                              copy of the old ones (the ranges overlap);
//   k_inc_clusters_insert      inserts the `init` RayClusters into the cluster table (k_build_tables' per-cluster part) and
//                              initialises every per-cluster cell a decide warp or k_decide_large reads: a moved or created
//                              RayCluster starts from an empty bucket, and rows past the previous count may hold values of an earlier,
//                              larger fleet.  With `names` (new names after the resident ones, the name table not rebuilt), it also
//                              inserts their groups' workersToDelete names into the name table and its Bloom bitmap (k_build_tables'
//                              group part) and sets their resolutions to -1;
//   k_inc_wtd_resolve          (first_name = the first new name; only with `names`) then probes every pod row once: a new name may
//                              name any resident Pod.  It resolves the new names and touches the rows that hit one.  A row of a new
//                              RayCluster was an orphan and k_inc_orphan_adopt touched it already; any other resident row still
//                              probes to the RayCluster that holds it (the lowest row keeps a duplicate key).
// (KR_OPT_LARGE_MOVES adds two steps for gone rows that have a region: k_inc_large_release beside k_inc_clusters_release, and
// k_inc_large_carry right behind k_inc_clusters_insert; see there.)
// Places in the action list and create arena that a gone RayCluster held are abandoned until the next full pass.
// k_inc_clusters_insert and k_inc_orphan_adopt take the `init` RayClusters as the ascending row list `rows` of n entries.
__global__ void __launch_bounds__(256) k_inc_clusters_insert(SnapDev s, ScratchDev sc, ResDev r, const uint32_t *rows, uint32_t n, int names) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || __ldcg(&sc.inc[KR_INC_STRUCTURAL])) return;
  const uint32_t c = rows[i];
  cl_insert_cluster(s, sc, c);
  sc.cl_dyn[c] = make_uint4(0u, 0u, 0u, 0u);  // no pod yet (k_inc_admit appends them), no first head, not "lost a row"
  sc.act_res[c] = 0u; sc.cre_res[c] = 0u;     // no reserved places: the decide takes new ones at the cursors
  r.act_start[c] = 0u; r.act_cnt[c] = 0u;
  if (sc.lg) sc.lg[c] = make_uint4(0u, 0u, 0u, 0u);  // no region (a RayCluster that outgrows its bucket voids the epoch)
  const uint32_t g0 = s.c_group_off[c], G = s.c_group_cnt[c];
  for (uint32_t g = g0; g < g0 + G; g++) {  // no pods asked for in the resident results
    kr_group_result z; z.expected = 0; z.n_list = 0; z.n_unhealthy = 0; z.n_running = 0; z.diff = 0; z.n_create = 0; z.create_off = 0; z.flags = 0;
    r.groups[g] = z;
    sc.gcreate[g] = 0u;
    if (names) {
      for (uint32_t e = s.g_wtd_off[g]; e < s.g_wtd_off[g] + s.g_wtd_cnt[g]; e++) r.wtd_pod_idx[e] = 0xFFFFFFFFu;
      wt_insert_group(s, sc, g);
    }
  }
  mark_dirty(sc, c, inc_epoch(sc));
}

// Grid-stride over the resident pod rows, 8 bytes per row (namespace, ray.io/cluster), against a Bloom bitmap of the new RayClusters'
// keys and, behind it, an open-addressed table of their rows (both built per CTA in shared memory: 4 * (slot_mask + 1) bytes of slots
// after (bloom_mask + 1) / 8 bytes of bits).
__global__ void __launch_bounds__(256) k_inc_orphan_adopt(SnapDev s, ScratchDev sc, ResDev r, const uint32_t *rows, uint32_t n, uint32_t bloom_mask,
                                                          uint32_t slot_mask, uint32_t n_resident) {
  extern __shared__ uint32_t sm_adopt[];
  uint32_t *bits = sm_adopt, *slots = sm_adopt + ((bloom_mask + 1) >> 5);
  for (uint32_t i = threadIdx.x; i < (bloom_mask + 1) >> 5; i += blockDim.x) bits[i] = 0u;
  for (uint32_t i = threadIdx.x; i <= slot_mask; i += blockDim.x) slots[i] = KR_EMPTY32;
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    const uint32_t c = rows[i];
    const uint32_t ns = s.c_ns_id[c], nm = s.c_name_id[c];
    if (nm == 0) continue;  // (cl_probe matches no pod against an absent name)
    const uint32_t hk = hash_pair(ns, nm), h2 = bloom2(hk);
    atomicOr(&bits[(hk & bloom_mask) >> 5], 1u << (hk & 31));
    atomicOr(&bits[(h2 & bloom_mask) >> 5], 1u << (h2 & 31));
    uint32_t j = hk & slot_mask;
    while (atomicCAS(&slots[j], KR_EMPTY32, c) != KR_EMPTY32) j = (j + 1) & slot_mask;
  }
  __syncthreads();
  const uint32_t epoch = inc_epoch(sc);
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n_resident; p += gridDim.x * blockDim.x) {
    const uint32_t ns = __ldg(&s.p_ns_id[p]), cn = __ldg(&s.p_cluster_name_id[p]);
    if (cn == 0) continue;
    const uint32_t hk = hash_pair(ns, cn), h2 = bloom2(hk);
    if (!(bits[(hk & bloom_mask) >> 5] & (1u << (hk & 31))) || !(bits[(h2 & bloom_mask) >> 5] & (1u << (h2 & 31)))) continue;
    for (uint32_t j = hk & slot_mask, c; (c = slots[j]) != KR_EMPTY32; j = (j + 1) & slot_mask) {
      if (s.c_ns_id[c] == ns && s.c_name_id[c] == cn) {
        uint32_t ns2, nm2;
        inc_touch(s, sc, r, p, epoch, n_resident, ns2, nm2);
        break;
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_inc_digest_move(const uint32_t *__restrict__ pairs, uint32_t n, char *hash) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 2 * n) return;
  const uint32_t from = pairs[2 * (t >> 1)], to = pairs[2 * (t >> 1) + 1];  // (sources sit at or past the new count, targets below it)
  reinterpret_cast<uint4 *>(hash + 32 * (size_t)to)[t & 1] = reinterpret_cast<const uint4 *>(hash + 32 * (size_t)from)[t & 1];
}

__global__ void __launch_bounds__(256) k_inc_clusters_release(SnapDev s, ScratchDev sc, ResDev r, const uint32_t *gone, uint32_t n_gone, uint32_t n_resident) {
  const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= n_gone) return;
  const uint32_t o = gone[w], epoch = inc_epoch(sc);
  const uint4 rec = sc.cl_rec[o];  // {group_off, group_cnt} of the old row
  const uint32_t P = sc.cl_dyn[o].x;
  for (uint32_t k = lane; k < P; k += 32) {
    const uint2 *at = rec_slot(sc, o, k);
    uint32_t ns, nm;
    if (at) inc_touch(s, sc, r, at->x, epoch, n_resident, ns, nm);
  }
  uint32_t cre = 0;
  for (uint32_t g = rec.x + lane; g < rec.x + rec.y; g += 32) cre += r.groups[g].n_create;
  cre = __reduce_add_sync(0xFFFFFFFFu, cre);
  if (lane == 0) {
    if (r.act_cnt[o]) atomicSub(&r.totals[2], r.act_cnt[o]);
    if (cre) atomicSub(&r.totals[6], cre);
  }
}

// KR_OPT_LARGE_MOVES: the gone rows that have a region (large RayClusters deleted, moved or regrouped) are listed apart, as
// {old row, region offset, region capacity, new row or KR_EMPTY32}, and k_inc_clusters_release takes only the others.  The host
// uploaded the region table in the new numbering at the start of the pass, so the old regions come from the list:
//   k_inc_large_release  one CTA per listed row (a 2 000-Pod row is 8 iterations per thread, not 63 per lane of one warp): the work of
//                        k_inc_clusters_release for ranks [0, stride) in the bucket and [stride, stride + capacity) in the region;
//   k_inc_large_carry    behind k_inc_clusters_insert, which cleared the entry of every init row: a moved or regrouped RayCluster's
//                        region back into the table at its new row ({offset, capacity}, no sorted segment yet), so k_inc_admit
//                        brings its Pods into the bucket and then the carried region.  Every record before the epoch fits it, so
//                        with KR_OPT_LARGE_GROWTH exactly one record meets the first rank past it (grow_spill).
__global__ void __launch_bounds__(256) k_inc_large_release(SnapDev s, ScratchDev sc, ResDev r, const uint4 *gone, uint32_t n_resident) {
  __shared__ uint32_t s_cre[8];
  const uint4 g = gone[blockIdx.x];
  const uint32_t o = g.x, S = sc.bucket_stride, epoch = inc_epoch(sc), tid = threadIdx.x;
  const uint32_t P = min(__ldcg(&sc.cl_dyn[o].x), S + g.z);
  for (uint32_t k = tid; k < P; k += blockDim.x) {
    const uint2 *at = k < S ? sc.bucket + (size_t)o * S + k : sc.region + g.y + (k - S);
    uint32_t ns, nm;
    inc_touch(s, sc, r, at->x, epoch, n_resident, ns, nm);
  }
  const uint4 rec = sc.cl_rec[o];  // {group_off, group_cnt} of the old row
  uint32_t cre = 0;
  for (uint32_t gi = rec.x + tid; gi < rec.x + rec.y; gi += blockDim.x) cre += r.groups[gi].n_create;
  cre = __reduce_add_sync(0xFFFFFFFFu, cre);
  if ((tid & 31) == 0) s_cre[tid >> 5] = cre;
  __syncthreads();
  if (tid == 0) {
    cre = 0;
    for (uint32_t w = 0; w < blockDim.x / 32; w++) cre += s_cre[w];
    if (r.act_cnt[o]) atomicSub(&r.totals[2], r.act_cnt[o]);
    if (cre) atomicSub(&r.totals[6], cre);
  }
}

__global__ void __launch_bounds__(256) k_inc_large_carry(ScratchDev sc, const uint4 *gone, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint4 g = gone[i];
  if (g.w != KR_EMPTY32) sc.lg[g.w] = make_uint4(g.y, g.z, 0u, 0u);
}

__global__ void __launch_bounds__(1024) k_inc_clusters_translate(ScratchDev sc, const uint32_t *gone, uint32_t n_gone, uint32_t n_clusters) {
  __shared__ uint32_t s_warp[32];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t n_touched = __ldcg(&sc.inc[KR_INC_TOUCHED]), n_dirty = __ldcg(&sc.inc[KR_INC_DIRTY]);
  for (uint32_t i = tid; i < n_touched; i += blockDim.x) {
    const uint32_t c = sc.touched_old[i];
    if (c != KR_EMPTY32 && sorted_has(gone, n_gone, c)) sc.touched_old[i] = KR_EMPTY32;
  }
  uint32_t kept = 0;  // entries of the dirty list kept so far (compacted in place: an entry never moves up)
  for (uint32_t i0 = 0; i0 < n_dirty; i0 += blockDim.x) {
    const uint32_t i = i0 + tid;
    const uint32_t c = i < n_dirty ? sc.dirty_list[i] : KR_EMPTY32;
    const bool keep = c < n_clusters;
    const uint32_t b = __ballot_sync(0xFFFFFFFFu, keep);
    if (lane == 0) s_warp[warp] = __popc(b);
    __syncthreads();
    uint32_t before = 0, total = 0;
    for (uint32_t k = 0; k < blockDim.x / 32; k++) { const uint32_t v = s_warp[k]; before += k < warp ? v : 0u; total += v; }
    if (keep) sc.dirty_list[kept + before + __popc(b & lanemask_lt())] = c;
    kept += total;
    __syncthreads();
  }
  if (tid == 0) sc.inc[KR_INC_DIRTY] = kept;
}

__global__ void __launch_bounds__(256) k_inc_clusters_rekey(SnapDev s, ScratchDev sc, uint32_t n_clusters) {
  for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n_clusters; c += gridDim.x * blockDim.x) cl_insert_cluster(s, sc, c);
}

// new group gs0 + k takes old group gsrc[k] (KR_EMPTY32: a group of a moved or created RayCluster, which k_inc_clusters_insert
// clears); old_groups / old_gcreate hold the old groups from g_lo on
__global__ void __launch_bounds__(256) k_inc_groups_gather(ResDev r, ScratchDev sc, const uint32_t *__restrict__ gsrc, uint32_t gs0, uint32_t n_shifted,
                                                           const kr_group_result *__restrict__ old_groups, const uint32_t *__restrict__ old_gcreate, uint32_t g_lo) {
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n_shifted; k += gridDim.x * blockDim.x) {
    const uint32_t o = gsrc[k];
    if (o == KR_EMPTY32) continue;
    r.groups[gs0 + k] = old_groups[o - g_lo];
    sc.gcreate[gs0 + k] = old_gcreate[o - g_lo];
  }
}

// ------------------------------------------------------------------------------------------------ k_inc_finish
// (The changed records are packed for the host by the decide warps themselves: IncStage in kr_bucket2.cuh.)

// closes the epoch (after the host's copy of the counters was enqueued): next epoch's stamps differ from every stamp written so far
__global__ void k_inc_finish(ScratchDev sc) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    sc.inc[KR_INC_TOUCHED] = 0; sc.inc[KR_INC_DIRTY] = 0; sc.inc[KR_INC_STRUCTURAL] = 0; sc.inc[KR_INC_HEADS] = 0; sc.inc[KR_INC_VOID] = 0; sc.inc[KR_INC_GROUPS] = 0; sc.inc[KR_INC_LSEG] = 0;
    sc.inc[KR_INC_GROW] = 0; sc.inc[KR_INC_SPILL] = 0; sc.inc[KR_INC_GROWN] = 0;
    sc.inc[KR_INC_EPOCH] += 1u;
  }
}

}  // namespace kr

// kr_engine.cu — C ABI (include/kr_engine.h) of the batched reconcile engine: arenas, streams, kernel schedule.
//
// One engine = one device and four streams: M (the pass's main chain), H (the hash beside it), G (the general decide kernel beside
// k_decide_small) and a copy stream for the commits.  Inputs live in ONE pinned host arena and ONE device arena with identical
// layouts computed per snapshot from kr_sizes.  PassCtx, launch_hash, launch_decide2 and launch_large_sort are the launch helpers of
// the full pass (launch_pass, replayed as a CUDA graph by run_pass_once) and the incremental one (run_pass_inc); run_pass drives both
// for every reconcile call, profiled or not.  fetch_results copies the results back with the exact sizes of the totals words the
// pass left, behind one host wait.  Every commit checks its whole input first (check_cluster_row, check_head_row),
// then moves the host's record of what the device holds (CommitRecord) through that record's update functions, then uploads on the
// copy stream between begin_commit and finish_commit: an invalid call commits nothing.  The two object commits diff their rows
// against the resident tables on the device (object_diff_args, launch_object_diff).
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "kr_kernels.cuh"
#include "kr_incr.cuh"
#include "kr_large.cuh"
#include "kr_huge.cuh"
#include "kr_lists.cuh"

using namespace kr;

// kr_specjson.cpp
int kr_specjson_emit_string(const uint8_t *spec_json, uint64_t len, bool muted, long max_groups, std::string &out, long *n_groups);

namespace {

constexpr size_t kAlign = 256;
// most RayClusters one incremental epoch brings in while there are orphans (k_inc_orphan_adopt: 16 Bloom bits and two 4-byte table
// slots per RayCluster in shared memory, 40 KB); more take the full pass
constexpr uint32_t kAdoptMax = 4096;
// most RayClusters one incremental epoch that renumbers them (KR_OPT_CLUSTER_DELETES) or regroups them (KR_OPT_GROUP_EDITS) deletes,
// moves, creates and regroups together; more take the full pass
constexpr uint32_t kMapMax = 4096;

// Attempts of one full pass: bucket pipeline -> wider stride -> sort pipeline -> radix pipeline, or a rerun on the two-phase hash
// schedule.  Each closes an epoch of the device counter (k_build_tables), and a void incremental attempt before them one more
// (k_inc_finish).  A counter past 2^32 - 1 - kEpochMargin before a pass is zeroed again, so none reaches 2^32 - 1: no epoch stamps
// with 0, the value of the zeroed stamps and of "not this epoch", and no stamp written since the zeroing comes round again.
constexpr int kFullAttempts = 5;
constexpr uint32_t kEpochMargin = 8;
static_assert(kEpochMargin > kFullAttempts + 1, "one pass may close kFullAttempts + 1 epochs");

enum MapList { MP_GONE, MP_INIT, MP_DIGESTS, MP_GSRC, MP_WSRC, MP_SGONE, MP_LARGE, MP_LISTS };  // the lists of a row map on the device, in this order
inline size_t align_up(size_t x, size_t a = kAlign) { return (x + a - 1) / a * a; }
inline uint32_t pow2_at_least(uint64_t x) { uint32_t p = 16; while (p < x) p <<= 1; return p; }
// staging of an incremental pass's changed records, for up to a quarter of the RayClusters (beyond that the whole record arrays are
// as cheap to move): meta 32 B x capc, cluster records x capc, group records x capg, then the re-hashed digests of a spec-row epoch
// (32 B x capc)
struct IncStageLayout { uint32_t capc, capg; size_t clusters, groups, digests, total; };
IncStageLayout inc_stage_layout(uint32_t n_clusters, uint32_t n_groups) {
  IncStageLayout L;
  L.capc = std::max<uint32_t>(64, n_clusters / 4);
  L.capg = (uint32_t)std::min<uint64_t>((uint64_t)L.capc * KR_SMEM_GROUPS, (uint64_t)n_groups + 1);
  L.clusters = align_up(32 * (size_t)L.capc);
  L.groups = L.clusters + align_up(sizeof(kr_cluster_result) * (size_t)L.capc);
  L.digests = L.groups + align_up(sizeof(kr_group_result) * (size_t)L.capg);
  L.total = L.digests + 32 * (size_t)L.capc + 1024;
  return L;
}

// bucket stride of a new layout: a power of two with 25 % head room over the mean cluster size (a cluster that outgrows it voids the
// attempt; the pass then widens the stride, up to 256, or leaves the bucket pipeline for this layout)
uint32_t first_stride(const kr_sizes &n) {
  uint32_t st = 64;
  const uint64_t want = n.n_clusters ? ((uint64_t)n.n_pods * 5 / 4 + n.n_clusters - 1) / n.n_clusters : 0;
  while (st < want && st < 512) st <<= 1;
  return st <= 256 ? st : 0;
}

struct InLayout {  // offsets of every input column inside the snapshot arena
  size_t off[64];
  size_t total;
};

// (element size, per-row multiplicity, dimension index) in the order of kr_snapshot_bufs
enum { D_CLUSTERS, D_GROUPS, D_WTD, D_PODS, D_HEADS, D_JOBS, D_JSON };
struct ColDesc { uint8_t elem, mult, dim; };
constexpr ColDesc kCols[] = {
    {4, 1, D_CLUSTERS}, {4, 1, D_CLUSTERS}, {8, 1, D_CLUSTERS}, {4, 1, D_CLUSTERS}, {1, 1, D_CLUSTERS}, {1, 1, D_CLUSTERS},
    {4, 1, D_CLUSTERS}, {4, 1, D_CLUSTERS}, {4, 1, D_CLUSTERS}, {8, 1, D_CLUSTERS}, {4, 1, D_CLUSTERS},
    {1, 1, D_CLUSTERS}, {4, 5, D_CLUSTERS}, {1, 5, D_CLUSTERS}, {1, 5, D_CLUSTERS}, {4, 1, D_CLUSTERS}, {4, 2, D_CLUSTERS},
    {4, 4, D_CLUSTERS}, {1, 1, D_CLUSTERS}, {1, 1, D_CLUSTERS}, {4, 1, D_CLUSTERS}, {4, 1, D_CLUSTERS},
    {4, 1, D_GROUPS}, {4, 1, D_GROUPS}, {4, 1, D_GROUPS}, {4, 1, D_GROUPS}, {4, 1, D_GROUPS}, {4, 1, D_GROUPS},
    {4, 1, D_GROUPS}, {4, 1, D_GROUPS}, {4, 1, D_GROUPS},
    {4, 1, D_WTD},
    {4, 1, D_PODS}, {4, 1, D_PODS}, {4, 1, D_PODS}, {4, 1, D_PODS}, {4, 1, D_PODS}, {4, 1, D_PODS}, {4, 1, D_PODS},
    {4, 1, D_HEADS}, {1, 1, D_HEADS}, {4, 1, D_HEADS}, {4, 1, D_HEADS}, {4, 1, D_HEADS}, {1, 1, D_HEADS}, {1, 1, D_HEADS}, {1, 32, D_HEADS},
    {4, 1, D_JOBS}, {4, 1, D_JOBS}, {4, 1, D_JOBS}, {4, 1, D_CLUSTERS},
    {1, 1, D_JSON},
};
constexpr int kNumCols = sizeof(kCols) / sizeof(kCols[0]);
constexpr int kFirstPodCol = 32;  // p_ns_id ... p_replica_name_id are columns 32..38
static_assert(kCols[kFirstPodCol].dim == D_PODS && kCols[kFirstPodCol - 1].dim != D_PODS && kCols[kFirstPodCol + 6].dim == D_PODS && kCols[kFirstPodCol + 7].dim != D_PODS,
              "kFirstPodCol must point at the seven per-pod columns");
static_assert(sizeof(kr_snapshot_bufs) == kNumCols * sizeof(void *), "kCols must mirror kr_snapshot_bufs");
static_assert(sizeof(SnapDev) == kNumCols * sizeof(void *), "SnapDev must mirror kr_snapshot_bufs");
static_assert(sizeof(kr_cluster_result) == 96 && sizeof(kr_group_result) == 32 && sizeof(kr_job_result) == 8, "result record sizes");

// how a changed row of each object column is treated by the on-device diff of an object commit (kr_incr.cuh, KR_OC_*).
// (g_num_hosts is an ordinary group column: k_decide2 reads numOfHosts from the group rows / the refreshed input record, never from
// the multi-host bit of the resident cluster table, which only the sort pipeline reads and a full pass rebuilds.)
static const uint8_t kObjClass[kNumCols] = {
        KR_OC_STRUCT, KR_OC_STRUCT, KR_OC_COPY, KR_OC_CLUSTER, KR_OC_CLUSTER, KR_OC_CLUSTER, KR_OC_CLUSTER, KR_OC_STRUCT, KR_OC_STRUCT, KR_OC_COPY, KR_OC_COPY,
        KR_OC_CLUSTER, KR_OC_CLUSTER, KR_OC_CLUSTER, KR_OC_CLUSTER, KR_OC_CLUSTER, KR_OC_CLUSTER, KR_OC_CLUSTER, KR_OC_CLUSTER, KR_OC_CLUSTER, KR_OC_CLUSTER, KR_OC_CLUSTER,
        KR_OC_STRUCT, KR_OC_STRUCT, KR_OC_GROUP, KR_OC_GROUP, KR_OC_GROUP, KR_OC_GROUP, KR_OC_GROUP, KR_OC_STRUCT, KR_OC_STRUCT,
        KR_OC_STRUCT,
        0, 0, 0, 0, 0, 0, 0,
        KR_OC_HEADKEY, KR_OC_HEAD, KR_OC_HEAD, KR_OC_HEAD, KR_OC_HEAD, KR_OC_HEAD, KR_OC_HEAD, KR_OC_HEAD,
        KR_OC_COPY, KR_OC_COPY, KR_OC_COPY, KR_OC_COPY,
        0};
constexpr int kHeadKeyCol = 39, kGroupClusterCol = 22, kJsonOffCol = 9;
static_assert(kCols[kJsonOffCol].elem == 8 && kCols[kJsonOffCol + 1].elem == 4 && kCols[kJsonOffCol + 1].dim == D_CLUSTERS, "c_json_off / c_json_len column indices");
static_assert(kCols[kHeadKeyCol].dim == D_HEADS && kCols[kHeadKeyCol - 1].dim == D_PODS && kCols[kGroupClusterCol].dim == D_GROUPS && kCols[kGroupClusterCol - 1].dim == D_CLUSTERS, "column indices of the object diff");
// g_wtd_off, g_wtd_cnt, w_name_id.  With KR_OPT_WTD_EDITS a staged object commit classifies them as copy / group / copy instead:
// the next pass rebuilds the name table and recomputes KR_ROW_WTD_OWN (the only use of the offsets), and the multi-host decide
// reads the count.
constexpr int kWtdOffCol = 29, kWtdCntCol = 30, kWtdNameCol = 31, kGroupOffCol = 7;
static_assert(kCols[kGroupOffCol].dim == D_CLUSTERS && kCols[kGroupOffCol + 1].dim == D_CLUSTERS && kCols[kGroupOffCol + 2].elem == 8, "c_group_off column index");
static_assert(kCols[kWtdCntCol].dim == D_GROUPS && kCols[kWtdNameCol].dim == D_WTD && kCols[kWtdNameCol + 1].dim == D_PODS, "workersToDelete column indices");
// With KR_OPT_CLUSTER_CREATES a row past the resident rows of a RayCluster / group / workersToDelete column belongs to a RayCluster
// the epoch appended (`appended`): it marks that RayCluster dirty and refreshes its input record (a group row: its RayCluster's) instead
// of making the epoch structural.  A row map (KR_OPT_CLUSTER_DELETES, KR_OPT_GROUP_EDITS) classes the rows of its moved, created and
// regrouped RayClusters the same way.
uint8_t obj_class(int col, bool wtd_edits, bool appended = false) {
  if (appended && kObjClass[col] == KR_OC_STRUCT)
    return kCols[col].dim == D_CLUSTERS ? KR_OC_CLUSTER : kCols[col].dim == D_GROUPS ? KR_OC_GROUP : KR_OC_COPY;
  if (wtd_edits && (col == kWtdOffCol || col == kWtdNameCol)) return KR_OC_COPY;
  if (wtd_edits && col == kWtdCntCol) return KR_OC_GROUP;
  return kObjClass[col];
}

// The host's record of what the device's object columns, JSON ranges and hash order were last committed from, and of what the next
// pass owes them.  Only its four update functions change it, each after its commit has checked the whole input and before the
// commit uploads anything: commit_whole (kr_snapshot_commit_parts, any parts), commit_rows (the row path of
// kr_snapshot_commit_object_rows), commit_spec_rows (kr_snapshot_commit_spec_rows) and commit_json_moves
// (kr_snapshot_commit_json_moves).  The passes clear the four flags at the end.
struct CommitRecord {
  struct Row {
    uint64_t json_off;             // the JSON range the digests and the hash order were computed from: whole, spec rows
    uint32_t json_len, group_off, group_cnt;  // (groups: whole)
    uint8_t recreate, mh;          // KR_CF_UPGRADE_RECREATE: whole with the object part; some worker group has numOfHosts > 1: whole, rows
    uint32_t ns, name, wtd_off;    // key and first workersToDelete name: whole with the object part
  };
  std::vector<Row> rows;             // per RayCluster row (sized, zero-filled, by every whole commit)
  // KR_OPT_CLUSTER_CREATES / KR_OPT_CLUSTER_DELETES / KR_OPT_GROUP_EDITS: the RayCluster rows that entered the fleet since the last
  // pass, how the last object commit renumbered the others (swap-remove) and which ones changed their list of worker groups, for the
  // next pass.  Without gone rows: RayClusters appended after the resident ones.  A regrouped RayCluster (same key and row, another
  // ordered list of group names) is gone and initialised again in its own row: listed in both `gone` and `init`.
  struct RowMap {
    std::vector<uint32_t> gone;      // old rows no RayCluster keeps (deleted, moved away, or regrouped), ascending
    std::vector<uint32_t> init;      // new rows of a moved, created or regrouped RayCluster, ascending
    std::vector<uint32_t> created;   // ... those whose specs are hashed (created, or moved / regrouped with a new spec range)
    std::vector<uint32_t> digests;   // (old row, new row) of the moved RayClusters whose spec range stayed: the digest moves
    std::vector<uint32_t> moved_to;  // per gone row: its new row (itself when regrouped), or KR_EMPTY32 (deleted)
    uint32_t gs0 = 0, ws0 = 0;       // groups / names from these on were shifted
    std::vector<uint32_t> gsrc, wsrc;  // ... and came from these old ones (KR_EMPTY32: of a moved or created RayCluster)
    uint32_t g_lo = 0, g_hi = 0;     // the old groups gsrc reads
    bool names_moved = false;        // a resident workersToDelete name shifted or vanished, or a map with gone rows brought new ones
    // KR_OPT_LARGE_MOVES, filled by commit_map when some gone row has a region: the gone rows without one, and per gone row with one
    // {old row, region offset, region capacity, new row or KR_EMPTY32} (kr_incr.cuh: k_inc_large_release, k_inc_large_carry)
    std::vector<uint32_t> small_gone, large;
  };
  RowMap map;
  uint32_t n_recreate = 0;           // RayClusters with KR_CF_UPGRADE_RECREATE (decide phase 1 needed): whole
  uint64_t recreate_sig = 0;         // which ones (their messages lead the hash order): whole, when it rebuilds the order
  uint32_t n_mh = 0;                 // rows with a multi-host group: whole, rows
  uint32_t snap_max_groups = 0;      // most worker groups in one RayCluster: whole
  std::vector<uint32_t> wide_rows;   // RayClusters of more than KR_SMEM_GROUPS worker groups, ascending: whole
  // rows whose range a JSON-only whole commit recorded while the device's c_json_off / c_json_len kept the old one (sorted,
  // distinct): the row path takes them only all together; any object commit clears the list
  std::vector<uint32_t> json_cols_behind;
  // rows whose device JSON bytes a move overwrote (sorted, distinct): no pass runs until each is re-committed (a spec row of it, or the
  // whole JSON part) or an object commit leaves it gone.  Through a row map the mark goes with its RayCluster while the range stays.
  std::vector<uint32_t> overwritten;
  uint32_t res_n_heads = 0;              // head-aux rows the resident device columns hold: whole with the object part
  uint32_t res_clusters = 0, res_groups = 0, res_wtd = 0;  // ... and RayCluster / group / workersToDelete rows: whole with the object part
  std::vector<uint32_t> prev_h_pod_idx;  // ... and their keys: whole with the object part, rows
  std::vector<uint32_t> prev_wtd;        // KR_OPT_WTD_EDITS: {n_groups, g_wtd_off, g_wtd_cnt, w_name_id} (empty while it is off): whole with the object part
  std::vector<uint32_t> prev_gnames;     // KR_OPT_GROUP_EDITS: g_name_id of the resident groups (empty while it is off): whole with the object part, rows
  bool hash_dirty = false;        // spec JSON or a JSON range committed since the digests were computed: whole
  bool heads_rebuild = false;     // a head key changed: the pod -> head-aux row table is rebuilt: whole, rows
  bool wtd_rebuild = false;       // a workersToDelete list changed: the name table is rebuilt (kr_incr.cuh): whole
  bool spec_order_stale = false;  // a spec commit changed a block count the full-pass hash order (d_order) was built from: spec rows (whole clears it)

  // the snapshot's workersToDelete lists are the recorded ones
  bool wtd_same(const kr_snapshot_bufs &hb, const kr_sizes &n) const {
    const size_t G = n.n_groups, W = n.n_wtd;
    return prev_wtd.size() == 1 + 2 * G + W && prev_wtd[0] == G && memcmp(prev_wtd.data() + 1, hb.g_wtd_off, 4 * G) == 0 &&
           memcmp(prev_wtd.data() + 1 + G, hb.g_wtd_cnt, 4 * G) == 0 && memcmp(prev_wtd.data() + 1 + 2 * G, hb.w_name_id, 4 * W) == 0;
  }
  // The resident object columns can take the named RayCluster rows as they are: the same row and head-aux counts, per named row the
  // same Recreate bit (hash order), JSON range (digests) and groups (the pipeline, the widest RayCluster and the wide set follow the
  // counts), with KR_OPT_WTD_EDITS the same workersToDelete lists, and every row a JSON-only commit left behind among the named ones.
  bool takes_rows(const kr_snapshot_bufs &hb, const kr_sizes &n, const uint32_t *cl, uint32_t n_cl, bool wtd_edits) const {
    if (rows.size() != n.n_clusters || res_n_heads != n.n_heads || (wtd_edits && !wtd_same(hb, n))) return false;
    for (const uint32_t *c = cl; c < cl + n_cl; c++) {
      const Row &r = rows[*c];
      if (r.recreate != ((hb.c_flags[*c] & KR_CF_UPGRADE_RECREATE) ? 1 : 0) || r.json_off != hb.c_json_off[*c] || r.json_len != hb.c_json_len[*c] ||
          r.group_off != hb.c_group_off[*c] || r.group_cnt != hb.c_group_cnt[*c])
        return false;
    }
    if (json_cols_behind.empty()) return true;
    std::vector<uint32_t> given(cl, cl + n_cl);
    std::sort(given.begin(), given.end());
    return std::includes(given.begin(), given.end(), json_cols_behind.begin(), json_cols_behind.end());
  }

  // The row map of an object part that brought RayClusters into the recorded fleet, renumbered it or regrouped some of it (into
  // `map`).  With `deletes` (KR_OPT_CLUSTER_DELETES) the rows whose key changed and the old rows at or past the new count are looked
  // at, with `regroups` (KR_OPT_GROUP_EDITS) the rows whose key stayed and whose ordered group names did not; otherwise only the rows
  // past the recorded ones are (a changed key or group is the device diff's to find).  -> 0: nothing entered, left, moved or
  // regrouped, 1: a map the resident state follows, -1: a renumbering it does not follow (the next pass is a full one).
  // `creates`: KR_OPT_CLUSTER_CREATES; `resident`: the RayCluster rows the device tables hold.
  int derive_map(const kr_snapshot_bufs &hb, const kr_sizes &n, bool creates, bool deletes, bool regroups, uint32_t resident,
                 uint32_t res_groups_old, uint32_t res_wtd_old) {
    const uint32_t had = (uint32_t)rows.size(), nn = n.n_clusters, lo = std::min(had, nn);
    auto key = [](uint32_t ns, uint32_t name) { return (uint64_t)ns << 32 | name; };
    regroups = regroups && prev_gnames.size() == res_groups_old;  // (the names are recorded from the object commit after the option came on)
    std::vector<uint32_t> old_ch, new_ch;
    uint32_t n_regrouped = 0;
    for (uint32_t c = 0; c < lo && (deletes || regroups); c++) {
      const Row &r = rows[c];
      const bool same_key = r.ns == hb.c_ns_id[c] && r.name == hb.c_name_id[c];
      const bool regrouped = regroups && same_key &&
                             (r.group_cnt != hb.c_group_cnt[c] || r.group_off + r.group_cnt > prev_gnames.size() || memcmp(prev_gnames.data() + r.group_off, hb.g_name_id + hb.c_group_off[c], 4 * (size_t)r.group_cnt) != 0);
      if ((deletes && !same_key) || regrouped) old_ch.push_back(c), new_ch.push_back(c);
      n_regrouped += regrouped;
    }
    if (deletes) for (uint32_t c = nn; c < had; c++) old_ch.push_back(c);
    if (old_ch.empty()) {
      // No recorded row left or moved: the rows past the resident ones, if this part added any, are created RayClusters, any number of
      // them, with their groups and names after the resident ones.  Counted from the resident rows (all of them recorded), not from
      // the recorded ones: the map of a second such commit in one epoch stands for both.
      if (!creates || nn <= had || had < resident) return 0;
      RowMap m;
      for (uint32_t c = resident; c < nn; c++) m.init.push_back(c);
      m.created = m.init;
      m.gs0 = n.n_groups; m.ws0 = n.n_wtd;
      map = std::move(m);
      return 1;
    }
    if (had != resident) return -1;  // (an earlier object commit of this epoch added rows the device tables do not hold yet)
    for (uint32_t c = had; c < nn; c++) new_ch.push_back(c);
    if (old_ch.size() > kMapMax || new_ch.size() > kMapMax) return -1;
    std::unordered_map<uint64_t, uint32_t> old_key;  // key of a gone row -> that row
    for (uint32_t o : old_ch) if (!old_key.emplace(key(rows[o].ns, rows[o].name), o).second) return -1;
    for (uint32_t c = 0; c < lo; c++)  // a kept row holding a gone row's key: the table's lowest-row rule would move it
      if (rows[c].ns == hb.c_ns_id[c] && rows[c].name == hb.c_name_id[c] && !std::binary_search(new_ch.begin(), new_ch.end(), c) &&
          old_key.count(key(rows[c].ns, rows[c].name)))
        return -1;
    RowMap m;
    m.gone = old_ch;
    m.moved_to.assign(old_ch.size(), KR_EMPTY32);
    std::unordered_set<uint64_t> new_keys;
    for (uint32_t c : new_ch) {
      const uint64_t k = key(hb.c_ns_id[c], hb.c_name_id[c]);
      if (!new_keys.insert(k).second) return -1;
      const auto it = old_key.find(k);
      // regrouped in its own row, or moved by swap-remove (with KR_OPT_GROUP_EDITS its group count may have changed as well: it
      // starts from an empty bucket either way); a digest stays or moves with an unchanged spec range, else it is hashed anew
      const bool regrouped = it != old_key.end() && it->second == c;
      if (regrouped || (it != old_key.end() && it->second >= nn && (regroups || rows[it->second].group_cnt == hb.c_group_cnt[c]))) {
        const uint32_t o = it->second;
        m.moved_to[std::lower_bound(m.gone.begin(), m.gone.end(), o) - m.gone.begin()] = c;
        if (rows[o].json_off != hb.c_json_off[c] || rows[o].json_len != hb.c_json_len[c]) m.created.push_back(c);
        else if (!regrouped) { m.digests.push_back(o); m.digests.push_back(c); }
      } else if (creates) m.created.push_back(c);
      else return -1;
    }
    if (old_ch.size() - m.digests.size() / 2 + new_ch.size() - n_regrouped > kMapMax) return -1;  // deleted + moved + created + regrouped
    m.init = new_ch;
    std::sort(m.created.begin(), m.created.end());
    // groups and names from the first renumbered row on: a kept RayCluster's come from its old ones, the others' are new
    const uint32_t c_min = new_ch.empty() ? nn : new_ch.front();
    m.gs0 = c_min < nn ? hb.c_group_off[c_min] : n.n_groups;
    m.ws0 = m.gs0 < n.n_groups ? hb.g_wtd_off[m.gs0] : n.n_wtd;
    m.g_lo = res_groups_old; m.g_hi = 0;
    for (uint32_t c = c_min; c < nn; c++) {
      const bool fresh = std::binary_search(new_ch.begin(), new_ch.end(), c);
      const uint32_t g0 = hb.c_group_off[c], G = hb.c_group_cnt[c];
      for (uint32_t gi = 0; gi < G; gi++) {
        const uint32_t og = fresh || gi >= rows[c].group_cnt ? KR_EMPTY32 : rows[c].group_off + gi;
        const bool ok = og < res_groups_old;
        m.gsrc.push_back(ok ? og : KR_EMPTY32);
        if (ok) { m.g_lo = std::min(m.g_lo, og); m.g_hi = std::max(m.g_hi, og + 1); }
        const uint32_t g = g0 + gi, w0 = hb.g_wtd_off[g];
        for (uint32_t w = w0; w < w0 + hb.g_wtd_cnt[g]; w++) {
          const uint32_t ow = ok ? rows[c].wtd_off + (w - hb.g_wtd_off[g0]) : KR_EMPTY32;
          m.wsrc.push_back(ow < res_wtd_old ? ow : KR_EMPTY32);
        }
      }
    }
    if (m.g_hi < m.g_lo) m.g_lo = m.g_hi = 0;
    m.names_moved = m.ws0 < n.n_wtd || n.n_wtd != res_wtd_old;
    map = std::move(m);
    return 1;
  }

  // what a whole commit moved: the launch shape / pipeline, the wide set, the hash order; `map`: derive_map's verdict (1: the created
  // RayClusters of `map`, whose specs the caller commits as spec rows, are hashed by the next pass)
  struct Moved { bool shape, wide, order; int map; };
  // (`creates`, `deletes`, `regroups`, `resident`: KR_OPT_CLUSTER_CREATES, KR_OPT_CLUSTER_DELETES, KR_OPT_GROUP_EDITS, the RayCluster
  // rows the device tables hold)
  Moved commit_whole(const kr_snapshot_bufs &hb, const kr_sizes &n, uint32_t parts, bool wtd_edits, bool creates, bool deletes, bool regroups,
                     uint32_t resident) {
    const bool objects = parts & (KR_PART_COLUMNS | KR_PART_OBJECTS);
    const size_t had = rows.size();
    const int mapped = (creates || deletes || regroups) && objects && had ? derive_map(hb, n, creates, deletes, regroups, resident, res_groups, res_wtd) : 0;
    bool ranges_moved = had != n.n_clusters && mapped != 1;  // some RayCluster's JSON range differs from the one the digests / the hash order were computed from
    if (parts & KR_PART_JSON) overwritten.clear();
    else if (objects && !overwritten.empty()) {
      std::vector<uint32_t> kept;
      for (uint32_t o : overwritten) {
        const auto it = mapped == 1 ? std::lower_bound(map.gone.begin(), map.gone.end(), o) : map.gone.end();
        if (it == map.gone.end() || *it != o) { if (o < n.n_clusters) kept.push_back(o); continue; }
        const uint32_t c = map.moved_to[it - map.gone.begin()];
        if (c != KR_EMPTY32 && rows[o].json_off == hb.c_json_off[c] && rows[o].json_len == hb.c_json_len[c]) kept.push_back(c);
      }
      std::sort(kept.begin(), kept.end());
      kept.erase(std::unique(kept.begin(), kept.end()), kept.end());
      overwritten.swap(kept);
    }
    uint32_t n_rc = 0, n_mh_now = 0, max_groups = 0;
    std::vector<uint32_t> wide;
    rows.resize(n.n_clusters);
    uint32_t woff = 0;
    for (uint32_t c = 0; c < n.n_clusters; c++) {
      Row &r = rows[c];
      const bool fresh = mapped == 1 && std::binary_search(map.init.begin(), map.init.end(), c);  // (its digest moves with it or is computed anew)
      const bool moved = !fresh && (c >= had || r.json_off != hb.c_json_off[c] || r.json_len != hb.c_json_len[c]);
      if (moved && !objects) json_cols_behind.push_back(c);  // (the device's range columns keep the old range)
      ranges_moved |= moved;
      r.json_off = hb.c_json_off[c]; r.json_len = hb.c_json_len[c];
      r.group_off = hb.c_group_off[c]; r.group_cnt = hb.c_group_cnt[c];
      if (objects) { r.ns = hb.c_ns_id[c]; r.name = hb.c_name_id[c]; r.wtd_off = woff; }
      for (uint32_t g = r.group_off; g < r.group_off + r.group_cnt; g++) woff += hb.g_wtd_cnt[g];
      r.mh = 0;
      for (uint32_t g = r.group_off; g < r.group_off + r.group_cnt; g++) r.mh |= hb.g_num_hosts[g] > 1 ? 1 : 0;
      n_mh_now += r.mh;
      max_groups = std::max(max_groups, r.group_cnt);
      if (r.group_cnt > KR_SMEM_GROUPS) wide.push_back(c);
      if (hb.c_flags[c] & KR_CF_UPGRADE_RECREATE) n_rc++;
      if (objects) r.recreate = (hb.c_flags[c] & KR_CF_UPGRADE_RECREATE) ? 1 : 0;
    }
    if (objects) json_cols_behind.clear();
    std::sort(json_cols_behind.begin(), json_cols_behind.end());
    json_cols_behind.erase(std::unique(json_cols_behind.begin(), json_cols_behind.end()), json_cols_behind.end());
    const bool shape = n_rc != n_recreate || (n_mh_now > 0) != (n_mh > 0) || (max_groups > KR_SMEM_GROUPS) != (snap_max_groups > KR_SMEM_GROUPS);
    n_recreate = n_rc; n_mh = n_mh_now; snap_max_groups = max_groups;
    const bool wide_moved = wide != wide_rows;
    wide_rows.swap(wide);
    uint64_t rsig = 0x9E3779B97F4A7C15ull * (n_rc + 1);
    for (uint32_t c = 0; c < n.n_clusters; c++) if (hb.c_flags[c] & KR_CF_UPGRADE_RECREATE) rsig = (rsig ^ c) * 0x100000001B3ull;
    // (a spec-row commit updates the recorded ranges itself: its own flag says the order no longer follows them)
    bool order = ranges_moved || rsig != recreate_sig || spec_order_stale;
    if (mapped == 1 && !ranges_moved) { spec_order_stale = true; order = false; }  // (the order lacks the new rows: the next pass that hashes every message rebuilds it)
    if (order) spec_order_stale = false;  // (the new order travels with this commit)
    recreate_sig = rsig;
    if ((parts & KR_PART_JSON) || ranges_moved) hash_dirty = true;
    if (objects) {
      if (prev_h_pod_idx.size() != n.n_heads || (n.n_heads && memcmp(prev_h_pod_idx.data(), hb.h_pod_idx, 4 * (size_t)n.n_heads) != 0)) {
        heads_rebuild = true;
        prev_h_pod_idx.assign(hb.h_pod_idx, hb.h_pod_idx + n.n_heads);
      }
      res_n_heads = n.n_heads; res_clusters = n.n_clusters; res_groups = n.n_groups; res_wtd = n.n_wtd;
      if (!wtd_edits) prev_wtd.clear();  // (the first commit after the option is turned on rebuilds the name table once)
      else if (!wtd_same(hb, n)) {
        wtd_rebuild = true;
        prev_wtd.assign(1, n.n_groups);
        prev_wtd.insert(prev_wtd.end(), hb.g_wtd_off, hb.g_wtd_off + n.n_groups);
        prev_wtd.insert(prev_wtd.end(), hb.g_wtd_cnt, hb.g_wtd_cnt + n.n_groups);
        prev_wtd.insert(prev_wtd.end(), hb.w_name_id, hb.w_name_id + n.n_wtd);
      }
      if (regroups) prev_gnames.assign(hb.g_name_id, hb.g_name_id + n.n_groups);
      else prev_gnames.clear();
    }
    return {shape, wide_moved, order, mapped};
  }
  // -> the snapshot's first multi-host group came or its last went (a numOfHosts edit)
  bool commit_rows(const kr_snapshot_bufs &hb, const uint32_t *cl, uint32_t n_cl, const uint32_t *hd, uint32_t n_hd) {
    const bool had_mh = n_mh > 0;
    for (uint32_t i = 0; i < n_cl; i++) {
      Row &r = rows[cl[i]];
      uint8_t bit = 0;
      for (uint32_t g = r.group_off; g < r.group_off + r.group_cnt; g++) bit |= hb.g_num_hosts[g] > 1 ? 1 : 0;
      n_mh += bit - r.mh; r.mh = bit;
      if (r.group_off + r.group_cnt <= prev_gnames.size())  // (a renamed group here is the diff's structural change: the full pass follows)
        std::copy(hb.g_name_id + r.group_off, hb.g_name_id + r.group_off + r.group_cnt, prev_gnames.begin() + r.group_off);
    }
    for (uint32_t i = 0; i < n_hd; i++)  // the pod -> head-aux row table follows the keys
      if (prev_h_pod_idx[hd[i]] != hb.h_pod_idx[hd[i]]) { heads_rebuild = true; prev_h_pod_idx[hd[i]] = hb.h_pod_idx[hd[i]]; }
    json_cols_behind.clear();  // (every recorded row is among the named ones)
    return (n_mh > 0) != had_mh;
  }
  // the m pulled rows' new ranges: a later object commit does not re-hash everything on their account; the full-pass hash order
  // does not follow them (spec_order_stale when a block count moved)
  // (rows past the recorded ones: the next object commit records them as created, or sees every range as moved)
  void commit_spec_rows(const uint32_t *cl, const uint64_t *off, const uint32_t *len, uint32_t m) {
    for (uint32_t i = 0; i < m; i++) {
      if (cl[i] >= rows.size()) continue;
      Row &r = rows[cl[i]];
      if ((r.json_len + 8) / 64 != (len[i] + 8) / 64) spec_order_stale = true;
      r.json_off = off[i]; r.json_len = len[i];
    }
    if (overwritten.empty()) return;
    std::vector<uint32_t> pulled(cl, cl + m);
    std::sort(pulled.begin(), pulled.end());
    overwritten.erase(std::remove_if(overwritten.begin(), overwritten.end(), [&](uint32_t c) { return std::binary_search(pulled.begin(), pulled.end(), c); }),
                      overwritten.end());
  }
  // the moved rows' new ranges (`to`: {destination, row} by destination, distinct recorded rows of unchanged lengths whose padded
  // destinations are disjoint; `listed`: per recorded row, whether it is among them): their bytes moved on the device, so the digests
  // and the hash order still hold and the device's range columns follow; every other recorded row whose range a destination
  // overlaps has lost its bytes (`overwritten`).  -> the rows it newly marked.
  std::vector<uint32_t> commit_json_moves(const std::vector<std::pair<uint64_t, uint32_t>> &to, const std::vector<uint8_t> &listed) {
    std::vector<uint64_t> lo, hi;  // the padded destination ranges that hold bytes, ascending
    for (const auto &t : to) {
      Row &r = rows[t.second];
      r.json_off = t.first;
      if (r.json_len) { lo.push_back(t.first); hi.push_back(t.first + ((r.json_len + 15ull) & ~15ull)); }
    }
    json_cols_behind.erase(std::remove_if(json_cols_behind.begin(), json_cols_behind.end(), [&](uint32_t c) { return listed[c] != 0; }), json_cols_behind.end());
    std::vector<uint32_t> hit;
    for (uint32_t c = 0; c < rows.size() && !lo.empty(); c++) {
      const Row &r = rows[c];
      if (!r.json_len || listed[c]) continue;
      const size_t k = std::lower_bound(lo.begin(), lo.end(), r.json_off + r.json_len) - lo.begin();  // (destinations starting before its end)
      if (k && hi[k - 1] > r.json_off) hit.push_back(c);
    }
    if (!hit.empty()) {
      std::vector<uint32_t> all;
      std::set_union(overwritten.begin(), overwritten.end(), hit.begin(), hit.end(), std::back_inserter(all));
      overwritten.swap(all);
    }
    return hit;
  }
};


void dims_of(const kr_sizes &n, uint64_t d[7]) {
  d[D_CLUSTERS] = n.n_clusters; d[D_GROUPS] = n.n_groups; d[D_WTD] = n.n_wtd; d[D_PODS] = n.n_pods;
  d[D_HEADS] = n.n_heads; d[D_JOBS] = n.n_jobs; d[D_JSON] = n.json_bytes;
}
Sizes sizes_of(const kr_sizes &n) { return Sizes{n.n_clusters, n.n_groups, n.n_wtd, n.n_pods, n.n_heads, n.n_jobs}; }

InLayout in_layout(const kr_sizes &n) {
  InLayout L;
  uint64_t d[7];
  dims_of(n, d);
  size_t o = 0;
  for (int i = 0; i < kNumCols; i++) {
    L.off[i] = o;
    o = align_up(o + (size_t)kCols[i].elem * kCols[i].mult * d[kCols[i].dim]);
  }
  L.total = o;
  return L;
}

struct OutLayout {  // results arena: [small fixed part | full pod lists | variable-length lists]
  size_t totals, clusters, hash, groups, wtd, jobs, act_start, act_cnt, small_total, sorted_idx, sorted_act, act_idx, act_code, create, pod_start, total;
};
OutLayout out_layout(const kr_sizes &n, uint32_t create_cap) {
  OutLayout L;
  size_t o = 0;
  L.totals = o; o = align_up(o + 256);  // 8 counters + (128 bytes in) the void-attempt word
  L.clusters = o; o = align_up(o + sizeof(kr_cluster_result) * (size_t)n.n_clusters);
  L.hash = o; o = align_up(o + 32 * (size_t)n.n_clusters);
  L.groups = o; o = align_up(o + sizeof(kr_group_result) * (size_t)n.n_groups);
  L.wtd = o; o = align_up(o + 4 * (size_t)n.n_wtd);
  L.jobs = o; o = align_up(o + sizeof(kr_job_result) * (size_t)n.n_jobs);
  L.act_start = o; o = align_up(o + 4 * ((size_t)n.n_clusters + 1));
  L.act_cnt = o; o = align_up(o + 4 * (size_t)n.n_clusters);
  L.small_total = o;  // everything above comes back in ONE copy
  L.sorted_idx = o; o = align_up(o + 4 * (size_t)n.n_pods);
  L.sorted_act = o; o = align_up(o + (size_t)n.n_pods);
  L.act_idx = o; o = align_up(o + 4 * (size_t)n.n_pods);
  L.act_code = o; o = align_up(o + (size_t)n.n_pods);
  L.create = o; o = align_up(o + 4 * (size_t)create_cap);
  L.pod_start = o; o = align_up(o + 4 * ((size_t)n.n_clusters + 1));  // the bucket pipeline's list starts (kr_lists.cuh)
  L.total = o;
  return L;
}

struct ScratchLayout {
  // 0xFF-initialised region first
  size_t cl_slots_off, wt_keys, wt_head, aux_keys, aux_vals, ff_total;
  size_t cl_rec, wt_next, rows, keys0, keys1, vals0, vals1, hist, row_total, gacc, gcreate, deferred_list, cact, ccount, chain, wt_bits, cl_dyn, cstart, tile_orph, mh_rep, mh_name, mh_meta, mh_cnt, mh_flg, mh_act, mh_head, act_tmp_idx, act_tmp_code, cl_in, bucket, inc_zero, stamp, dirty_flag, obj_flag, inc, inc_zero_end, touched, touched_old, pos, dirty_list, act_res, cre_res, total;
  uint32_t cl_slots, wt_slots, aux_slots, ntiles, mtiles;  // radix tiles (2048 keys) / k_match tiles of the fast pipeline
  uint32_t wt_bits_n;      // bits of the workersToDelete Bloom bitmap
  size_t bucket_entries;   // capacity of the bucket arena of the bucket pipeline (0: that pipeline is off for this engine)
};
ScratchLayout scratch_layout(const kr_sizes &n) {
  ScratchLayout L;
  L.cl_slots = pow2_at_least(2ull * n.n_clusters);
  L.wt_slots = pow2_at_least(2ull * n.n_wtd);
  L.aux_slots = pow2_at_least(2ull * n.n_heads);
  L.ntiles = (uint32_t)((n.n_pods + kSortTile - 1) / kSortTile);
  if (L.ntiles == 0) L.ntiles = 1;
  L.mtiles = (uint32_t)((n.n_pods + kMatchTile - 1) / kMatchTile);
  if (L.mtiles == 0) L.mtiles = 1;
  size_t o = 0;
  L.cl_slots_off = o; o = align_up(o + 16 * (size_t)L.cl_slots);
  L.wt_keys = o; o = align_up(o + 8 * (size_t)L.wt_slots);
  L.wt_head = o; o = align_up(o + 4 * (size_t)L.wt_slots);
  L.aux_keys = o; o = align_up(o + 4 * (size_t)L.aux_slots);
  L.aux_vals = o; o = align_up(o + 4 * (size_t)L.aux_slots);
  L.ff_total = o;
  L.cl_rec = o; o = align_up(o + 16 * (size_t)n.n_clusters);
  L.wt_next = o; o = align_up(o + 4 * (size_t)n.n_wtd);
  L.rows = o; o = align_up(o + 16 * (size_t)n.n_pods);
  L.keys0 = o; o = align_up(o + 4 * (size_t)n.n_pods);
  L.keys1 = o; o = align_up(o + 4 * (size_t)n.n_pods);
  L.vals0 = o; o = align_up(o + 4 * (size_t)n.n_pods);
  L.vals1 = o; o = align_up(o + 4 * (size_t)n.n_pods);
  L.hist = o; o = align_up(o + 4 * (size_t)kRadix * L.ntiles);
  L.row_total = o; o = align_up(o + 4 * (size_t)kRadix);
  L.gacc = o; o = align_up(o + 16 * (size_t)n.n_groups);
  L.gcreate = o; o = align_up(o + 4 * (size_t)n.n_groups + 32);
  L.deferred_list = o; o = align_up(o + 4 * (size_t)n.n_clusters);
  L.cact = o; o = align_up(o + 4 * ((size_t)n.n_clusters + 8));
  L.ccount = o; o = align_up(o + 4 * ((size_t)n.n_clusters + 2));
  L.chain = o;  // directly after ccount: k_clear zeroes both as one region
  o = align_up(o + 8 * (((size_t)n.n_clusters + 2) / 8192 + (size_t)L.mtiles / 8192 + (size_t)n.n_groups / 8192 + (size_t)n.n_clusters / 8192 + 10));
  {
    static const uint64_t per_name = [] { const char *g = getenv("KR_BLOOM_BITS"); return g && atoi(g) > 0 ? (uint64_t)atoi(g) : 64ull; }();
    uint64_t bits = 1024;
    while (bits < per_name * n.n_wtd && bits < (1ull << 17)) bits <<= 1;  // 64 bits per name up to 16 KB (shared-memory copy per k_match2 CTA)
    L.wt_bits_n = (uint32_t)bits;
  }
  L.wt_bits = o; o = align_up(o + L.wt_bits_n / 8);   // zeroed with ccount and chain (one region up to cstart)
  L.cl_dyn = o; o = align_up(o + 16 * (size_t)n.n_clusters);
  L.cstart = o; o = align_up(o + 4 * ((size_t)n.n_clusters + 2));
  L.tile_orph = o; o = align_up(o + 4 * ((size_t)L.mtiles + 8));
  L.mh_rep = o; o = align_up(o + 4 * (size_t)n.n_pods);
  L.mh_name = o; o = align_up(o + 4 * (size_t)n.n_pods);
  L.mh_meta = o; o = align_up(o + 4 * (size_t)n.n_pods);
  L.mh_cnt = o; o = align_up(o + 4 * (size_t)n.n_pods);
  L.mh_flg = o; o = align_up(o + 4 * (size_t)n.n_pods);
  L.mh_act = o; o = align_up(o + (size_t)n.n_pods);
  L.mh_head = o; o = align_up(o + (size_t)n.n_pods);
  L.act_tmp_idx = o; o = align_up(o + 4 * (size_t)n.n_pods);
  L.act_tmp_code = o; o = align_up(o + (size_t)n.n_pods);
  // bucket pipeline: fixed-stride buckets of 8-byte records.  Room for a stride of >= 4x the mean cluster size, at least 64
  // records per cluster; snapshots of very many tiny clusters (64 records per cluster would dwarf the pods) do without.
  L.bucket_entries = std::max<size_t>(4 * (size_t)n.n_pods, 64 * (size_t)n.n_clusters);
  L.bucket_entries = std::max<size_t>(L.bucket_entries, std::min<size_t>(256 * (size_t)n.n_clusters, (size_t)4 << 20));  // small snapshots: room for the widest stride
  if (64 * (size_t)n.n_clusters > 8 * (size_t)n.n_pods + (4u << 20)) L.bucket_entries = 0;
  L.cl_in = o; o = align_up(o + 128 * (size_t)n.n_clusters);
  L.bucket = o; o = align_up(o + sizeof(uint2) * L.bucket_entries);
  // incremental epochs (kr_incr.cuh): [stamps | dirty flags | counters] start out zero (one memset when the layout moves)
  L.inc_zero = o;
  L.stamp = o; o = align_up(o + 4 * (size_t)n.n_pods);
  L.dirty_flag = o; o = align_up(o + 4 * (size_t)n.n_clusters);
  L.obj_flag = o; o = align_up(o + 4 * (size_t)n.n_clusters);
  L.inc = o; o = align_up(o + 64);
  L.inc_zero_end = o;
  L.touched = o; o = align_up(o + 4 * (size_t)n.n_pods);
  L.touched_old = o; o = align_up(o + 4 * (size_t)n.n_pods);
  L.pos = o; o = align_up(o + 4 * (size_t)n.n_pods);
  L.dirty_list = o; o = align_up(o + 4 * (size_t)n.n_clusters);
  L.act_res = o; o = align_up(o + 4 * (size_t)n.n_clusters);
  L.cre_res = o; o = align_up(o + 4 * (size_t)n.n_clusters);
  L.total = o;
  return L;
}

// A pinned staging buffer and its device twin.  A caller whose upload may still be reading `h` when it returns records `ev` on the
// copy stream and sets `busy`; wait() is the next call's wait for it.
struct Staging {
  uint8_t *h = nullptr, *d = nullptr; size_t cap = 0;
  cudaEvent_t ev = nullptr; bool busy = false;
  // room for `need` bytes; a buffer that has to grow takes `slack` bytes more
  cudaError_t reserve(size_t need, size_t slack) {
    if (need <= cap) return cudaSuccess;
    if (h) cudaFreeHost(h);
    if (d) cudaFree(d);
    h = nullptr; d = nullptr; cap = 0;
    cudaError_t rc = cudaHostAlloc((void **)&h, need + slack, cudaHostAllocDefault);
    if (rc == cudaSuccess && (rc = cudaMalloc((void **)&d, need + slack)) == cudaSuccess) cap = need + slack;
    return rc;
  }
  cudaError_t wait() {
    const cudaError_t rc = busy ? cudaEventSynchronize(ev) : cudaSuccess;
    if (rc == cudaSuccess) busy = false;
    return rc;
  }
  void release() { if (h) cudaFreeHost(h); if (d) cudaFree(d); if (ev) cudaEventDestroy(ev); }
};

}  // namespace

struct kr_engine {
  kr_config cfg{};
  cudaStream_t sm = nullptr, sh = nullptr, sg = nullptr, scopy = nullptr;
  cudaEvent_t ev_h2d0 = nullptr, ev_h2d1 = nullptr, ev_cols = nullptr, ev_json = nullptr;  // commit: copy start, columns landed, JSON landed
  cudaEvent_t ev_fork2 = nullptr, ev_join2 = nullptr, ev_fork3 = nullptr, ev_join3 = nullptr;
  cudaEvent_t ev_inc = nullptr;  // an incremental pass's counters have reached the host
  cudaEvent_t ev_fork = nullptr, ev_hash = nullptr, ev_a = nullptr, ev_b = nullptr, ev_c = nullptr;
  cudaEvent_t ev_k[KR_MAX_KERNEL_TIMES + 1]{};
  uint8_t *h_in = nullptr, *d_in = nullptr, *d_scratch = nullptr, *d_out = nullptr, *h_out = nullptr;
  size_t in_cap = 0, scratch_cap = 0, out_cap = 0;
  kr_sizes sizes{};
  InLayout il{};
  OutLayout ol{};
  ScratchLayout sl{};
  bool begun = false, committed = false, ran = false;
  kr_flags last_flags{};      // flags of the last pass (kr_results_fetch honours fetch_pod_lists)
  bool committed_full = false;  // every part of the current layout has been uploaded at least once
  bool fixed_layout = false;    // KR_OPT_FIXED_LAYOUT: arenas laid out for the capacities, live counts in `sizes`
  CommitRecord rec;            // what the device's object columns, JSON ranges and hash order were last committed from
  kr_profile prof{};
  std::string err;
  Staging hb;                  // kr_hash_batch
  Staging pr;                  // incremental pod commits
  Staging orow;                // kr_snapshot_commit_object_rows
  Staging mp;                  // the row map of an object commit (rec.map), for its diff and the next pass
  bool map_pending = false;    // ... uploaded and not yet applied by a pass
  kr_sizes map_sizes{};        // ... the live counts of that object commit
  size_t mp_at[MP_LISTS]{};     // offsets in mp of its lists (MapList)
  uint8_t *h_in_dev = nullptr;  // device-side address of h_in
  int sm_count = 148;         // SMs the SM-sized grids are laid out for: the device's count, or fewer with KR_SM_COUNT
  // the whole pass (both streams) captured once per (layout, flags, n_recreate) and replayed
  cudaGraphExec_t gexec = nullptr;
  kr_flags gflags{};
  bool gvalid = false;
  bool use_graph = true;
  bool use_pdl = true;        // KR_NO_PDL=1 disables programmatic dependent launch
  int hash_ctas_per_sm = 2;   // KR_HASH_CTAS: resident hash CTAs per SM in the throughput regime
  int place_ctas = 1;         // k_place_fused CTAs per SM (KR_PLACE_CTAS; a second CTA per SM competes with the hash)
  // pipeline choice: fast = count/place/in-warp sort (every bucket <= 1024 pods); radix = general stable LSD sort.
  bool force_radix = false;   // sticky per layout: set when a pass met a bucket the fast pipeline cannot sort
  bool ran_fast = false;
  bool h2d_timed = true;      // h2d_ms of the last commit has been read back from its events
  bool no_fuse = false;       // KR_NO_FUSE=1: always take the separate scan kernels (tests; large snapshots take them anyway)
  bool env_radix = false;     // KR_FORCE_RADIX=1: always take the general pipeline (tests)
  uint32_t *h_totals = nullptr;  // pinned copy of the device totals (pipeline fallback check)
  // bucket pipeline (kr_bucket2.cuh): taken when the caller does not fetch the full pod lists and the snapshot qualifies
  bool no_bucket = false;       // KR_NO_BUCKET=1: never take it (tests of the sort pipeline)
  bool hash_spin = true;        // bucket pipeline: Recreate gates wait for their digest inside k_decide2 instead of a second decide phase
                                // (KR_NO_HASH_SPIN=1, or a pass in which a warp gave up waiting, turns it off)
  uint32_t bstride = 0;         // bucket stride of this layout (64 / 128 / 256); 0 = the layout does not qualify (a cluster outgrew 256 pods, ...)
  bool large_on = false;        // KR_OPT_LARGE_CLUSTERS
  bool wide_on = false;         // KR_OPT_WIDE_CLUSTERS
  bool huge_on = false;         // KR_OPT_HUGE_CLUSTERS (only with KR_OPT_LARGE_CLUSTERS)
  // The per-cluster kernels (kr_large.cuh) take the RayClusters of one list: the large half (rows and regions {offset, capacity}
  // from the last bucket attempt that voided, sticky like bstride) and, with KR_OPT_WIDE_CLUSTERS, the wide ones of the last commit.
  std::vector<uint32_t> large_rows; std::vector<uint2> large_reg;
  bool lg_stale = false;        // the device table / list do not reflect the two halves yet (upload_lg at the next pass)
  bool lg_moved = false;        // KR_OPT_LARGE_MOVES: an object commit renumbered the large half: the next upload writes the table
  uint32_t n_large = 0;         // RayClusters in the device list
  uint32_t n_lsort = 0;         // ... of which the first n_lsort are k_large_sort's; the huge ones after them go to k_huge_tiles / k_huge_merge
  uint32_t n_tiles = 0;         // tiles of the huge RayClusters in the device tile table
  // Sized for the capacities so that they never grow, allocated when an option first needs them (an engine without either pays
  // nothing): [lg: 16 B x max_clusters | lg_list: 4 B x max_clusters] for both options, regions (8 B x large_entries) for large ones
  uint8_t *d_lg = nullptr;
  uint2 *d_region = nullptr;
  size_t large_entries = 0;
  std::vector<uint4> h_lg; std::vector<uint32_t> h_lg_list;  // host side of the last upload (kept alive while it is in flight)
  // KR_OPT_HUGE_CLUSTERS, allocated when first turned on, for the capacities: the tile table {cluster, first rank, first tile, tiles}
  // and per-tile count / counter words (24 B x huge_tiles), then each tile's sorted run and arrival-order stash (2 x 4 B x kHugeTile)
  uint8_t *d_huge = nullptr;
  size_t huge_tiles = 0;
  std::vector<uint4> h_tiles;
  // KR_OPT_HUGE_GROWTH: the tile scratch holds huge_reserve (KR_HUGE_GROW_TILES once the option was first turned on) more tiles
  // past the huge_tiles resident ones, where k_inc_grow appends the tiles of the RayClusters it makes huge or regrows
  bool huge_growth = false;
  size_t huge_reserve = 0;
  // KR_OPT_LARGE_GROWTH, allocated when first turned on: the grow buffer of the incremental pass (kGrowBytes: list, result, spill)
  // and a pinned copy of its result; lg_cursor is the region arena's first entry past every region in use (after_bucket_void lays
  // them out from 0, each growth allocates past it)
  bool large_growth = false;
  uint4 *d_grow = nullptr; uint4 *h_grow = nullptr;
  size_t lg_cursor = 0;
  bool ran_bucket = false;
  bool bucket_lists = false;    // KR_OPT_BUCKET_POD_LISTS: fetch_pod_lists asks the bucket pipeline for the lists (kr_lists.cuh)
  bool host_starts = false;     // ... and the host's cluster records hold the list starts the last fetch patched in
  uint64_t h2d_accum = 0;       // bytes uploaded by the commits since the last pass (kr_profile.h2d_bytes)
  // hash order: message ids by descending SHA-1 block count, rebuilt at every commit from c_json_len
  uint32_t *h_order = nullptr, *d_order = nullptr;
  cudaEvent_t ev_order = nullptr;  // the upload of h_order has left the pinned buffer
  bool order_pending = false;
  std::vector<uint32_t> row_stamp;  // kr_snapshot_commit_pod_values: duplicate-row detection (epoch-stamped)
  uint32_t row_epoch = 0;
  // device-side incremental epochs (kr_incr.cuh)
  bool no_incr = false;          // KR_NO_INCR=1: every pass is a full pass (tests)
  bool inc_valid = false;        // the resident buckets / tables / results describe the committed snapshot up to the commits since the last pass
  bool inc_zero_needed = true;   // the stamp / dirty-flag / counter region of this layout has not been zeroed yet
  uint32_t dev_epoch = 0;        // the device's epoch counter (sc.inc[KR_INC_EPOCH]) as of the last pass
  uint32_t epoch_seed = 0;       // KR_EPOCH_BASE: the counter's value after the engine's first zeroing (later zeroings start from 0)
  kr_flags inc_flags{};          // flags of the pass that left the resident state
  uint32_t inc_n_pods = 0, inc_n_heads = 0;  // rows resident at the last pass
  bool wtd_edits = false;        // KR_OPT_WTD_EDITS
  bool cluster_creates = false;  // KR_OPT_CLUSTER_CREATES
  bool cluster_deletes = false;  // KR_OPT_CLUSTER_DELETES
  bool group_edits = false;      // KR_OPT_GROUP_EDITS
  bool large_moves = false;      // KR_OPT_LARGE_MOVES
  uint32_t inc_n_clusters = 0;   // RayClusters in the resident tables
  uint32_t res_n_wtd = 0;        // names in the resident name table and its resolutions (wtd_pod_idx)
  bool ran_inc = false;          // the last pass was an incremental one
  bool host_results_stale = false;  // an incremental pass went unfetched: the host copy misses its records, the next fetch copies everything
  bool fetched = true;              // the last pass's results have been copied to the host arena
  uint32_t inc_n_dirty = 0;      // changed RayClusters of the last incremental pass
  bool inc_gathered = false;     // ... and their records sit packed in the staging buffer
  bool inc_hash_ran = false;
  // kr_snapshot_commit_spec_rows, pinned mirror and device copy of {pull rows u32 | lens u32 | offs u64 | hash order u32}[max_clusters]:
  // each call appends the rows it pulls to the pull lists; the pass that hashes them sorts the pending rows once and uploads them as
  // the hash order
  Staging spec;
  uint32_t n_pull = 0;                // pull-list entries since the last pass
  std::vector<uint32_t> spec_pending;  // rows listed since the last pass that hashed (each once)
  std::vector<uint32_t> spec_stamp;    // cluster row -> spec_epoch that listed it (the union of the calls until they are hashed)
  uint32_t spec_epoch = 1;
  std::vector<uint32_t> pull_stamp;    // cluster row -> pull_epoch that pulled it: a pass in between lets the caller rewrite the arena,
  uint32_t pull_epoch = 1;             // so a row listed again after a pass (skip_hash leaves it pending) is pulled again
  bool spec_rows_opt = false;          // KR_OPT_SPEC_ROWS (read by kr_packer_flush)
  bool json_moves_opt = false;         // KR_OPT_JSON_MOVES (read by kr_packer_flush)
  // kr_snapshot_commit_json_moves, allocated at the first move commit: pinned mirror and device copy of {rows u32 | lens u32 | dst u64 |
  // src u64}[max_clusters], and the out-of-place copy's scratch, as large as the JSON arena's capacity
  Staging mv;
  uint8_t *d_json_scratch = nullptr;
  uint32_t inc_spec_n = 0;             // rows the last incremental pass re-hashed ...
  bool inc_spec_gathered = false;      // ... and their digests sit packed in the staging buffer
  std::vector<uint32_t> spec_hashed;   // ... which rows (the fetch scatters the digests)
  uint8_t *d_obj_stage = nullptr; size_t obj_stage_cap = 0;   // KR_PART_OBJECTS uploads land here while the state is resident
  Staging inc_stage;             // an incremental pass's changed records, sized for the capacities
  IncStageLayout inc_layout{};   // ... as the last incremental pass laid them out
  uint32_t *h_inc = nullptr;     // pinned copy of the epoch counters (16 words) + the changed-cluster list
  uint32_t *h_changed = nullptr; size_t h_changed_cap = 0;
  // kr_last_pass: the KR_FULL_* causes recorded since the last pass (a full pass that leaves nothing resident starts the next
  // pass's with its own), whether a commit of this epoch dropped the resident state (the later ones then record theirs too), the
  // report run_pass made of its pass and the one the last call that returned KR_OK published
  uint32_t why_full = KR_FULL_FIRST;
  bool epoch_dropped = false;
  kr_pass_report pass_made{}, pass_last{};
  bool has_pass = false;
};

namespace {

int fail(kr_engine *e, int code, const char *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (e) e->err = buf;
  return code;
}

#define CK(call)                                                                                          \
  do {                                                                                                    \
    cudaError_t _e = (call);                                                                              \
    if (_e != cudaSuccess) return fail(e, KR_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

kr_sizes cap_sizes(const kr_config &c) {
  kr_sizes n;
  n.n_clusters = c.max_clusters; n.n_groups = c.max_groups; n.n_wtd = c.max_wtd; n.n_pods = c.max_pods;
  n.n_heads = c.max_heads; n.n_jobs = c.max_jobs; n.json_bytes = c.max_json_bytes;
  return n;
}

void bind_in(const InLayout &L, uint8_t *base, void *struct_of_ptrs) {
  void **p = reinterpret_cast<void **>(struct_of_ptrs);
  for (int i = 0; i < kNumCols; i++) p[i] = base + L.off[i];
}

ResDev bind_out(const OutLayout &L, uint8_t *base) {
  ResDev r;
  r.totals = reinterpret_cast<uint32_t *>(base + L.totals);
  r.clusters = reinterpret_cast<kr_cluster_result *>(base + L.clusters);
  r.hash = reinterpret_cast<char *>(base + L.hash);
  r.groups = reinterpret_cast<kr_group_result *>(base + L.groups);
  r.wtd_pod_idx = reinterpret_cast<uint32_t *>(base + L.wtd);
  r.sorted_pod_idx = reinterpret_cast<uint32_t *>(base + L.sorted_idx);
  r.sorted_action = base + L.sorted_act;
  r.jobs = reinterpret_cast<kr_job_result *>(base + L.jobs);
  r.act_start = reinterpret_cast<uint32_t *>(base + L.act_start);
  r.act_cnt = reinterpret_cast<uint32_t *>(base + L.act_cnt);
  r.act_pod_idx = reinterpret_cast<uint32_t *>(base + L.act_idx);
  r.act_code = base + L.act_code;
  r.create_idx = reinterpret_cast<int32_t *>(base + L.create);
  return r;
}

ScratchDev bind_scratch(const ScratchLayout &L, uint8_t *b) {
  ScratchDev s;
  s.cl_slots = reinterpret_cast<uint4 *>(b + L.cl_slots_off); s.cl_mask = L.cl_slots - 1;
  s.cl_rec = reinterpret_cast<uint4 *>(b + L.cl_rec);
  s.wt_keys = reinterpret_cast<uint64_t *>(b + L.wt_keys); s.wt_head = reinterpret_cast<uint32_t *>(b + L.wt_head);
  s.wt_next = reinterpret_cast<uint32_t *>(b + L.wt_next); s.wt_mask = L.wt_slots - 1;
  s.aux_keys = reinterpret_cast<uint32_t *>(b + L.aux_keys); s.aux_vals = reinterpret_cast<uint32_t *>(b + L.aux_vals); s.aux_mask = L.aux_slots - 1;
  s.rows = reinterpret_cast<uint4 *>(b + L.rows);
  s.keys[0] = reinterpret_cast<uint32_t *>(b + L.keys0); s.keys[1] = reinterpret_cast<uint32_t *>(b + L.keys1);
  s.vals[0] = reinterpret_cast<uint32_t *>(b + L.vals0); s.vals[1] = reinterpret_cast<uint32_t *>(b + L.vals1);
  s.hist = reinterpret_cast<uint32_t *>(b + L.hist);
  s.row_total = reinterpret_cast<uint32_t *>(b + L.row_total);
  s.gacc = reinterpret_cast<int32_t *>(b + L.gacc);
  s.gcreate = reinterpret_cast<uint32_t *>(b + L.gcreate);
  s.deferred_list = reinterpret_cast<uint32_t *>(b + L.deferred_list);
  s.cact = reinterpret_cast<uint32_t *>(b + L.cact);
  s.ccount = reinterpret_cast<uint32_t *>(b + L.ccount);
  s.chain = reinterpret_cast<uint32_t *>(b + L.chain);
  s.cstart = reinterpret_cast<uint32_t *>(b + L.cstart);
  s.tile_orph = reinterpret_cast<uint32_t *>(b + L.tile_orph);
  s.mh_rep = reinterpret_cast<uint32_t *>(b + L.mh_rep); s.mh_name = reinterpret_cast<uint32_t *>(b + L.mh_name);
  s.mh_meta = reinterpret_cast<uint32_t *>(b + L.mh_meta); s.mh_cnt = reinterpret_cast<uint32_t *>(b + L.mh_cnt);
  s.mh_flg = reinterpret_cast<uint32_t *>(b + L.mh_flg); s.mh_act = b + L.mh_act; s.mh_head = b + L.mh_head;
  s.act_tmp_idx = reinterpret_cast<uint32_t *>(b + L.act_tmp_idx); s.act_tmp_code = b + L.act_tmp_code;
  s.bucket = reinterpret_cast<uint2 *>(b + L.bucket); s.bucket_stride = 0;
  s.wt_bits = reinterpret_cast<uint32_t *>(b + L.wt_bits); s.wt_bits_mask = L.wt_bits_n - 1;
  s.cl_in = reinterpret_cast<uint32_t *>(b + L.cl_in);
  s.cl_dyn = reinterpret_cast<uint4 *>(b + L.cl_dyn);
  s.stamp = reinterpret_cast<uint32_t *>(b + L.stamp); s.touched = reinterpret_cast<uint32_t *>(b + L.touched);
  s.touched_old = reinterpret_cast<uint32_t *>(b + L.touched_old); s.pos = reinterpret_cast<uint32_t *>(b + L.pos);
  s.obj_flag = reinterpret_cast<uint32_t *>(b + L.obj_flag);
  s.dirty_flag = reinterpret_cast<uint32_t *>(b + L.dirty_flag); s.dirty_list = reinterpret_cast<uint32_t *>(b + L.dirty_list);
  s.act_res = reinterpret_cast<uint32_t *>(b + L.act_res); s.cre_res = reinterpret_cast<uint32_t *>(b + L.cre_res);
  s.inc = reinterpret_cast<uint32_t *>(b + L.inc);
  s.lg = nullptr; s.region = nullptr;  // (set by the pass when the layout has large RayClusters: bind_large)
  return s;
}

// Kernel launch with the programmatic-dependent-launch attribute (see pdl_wait / pdl_trigger in kr_common.cuh).
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

// An incremental pass may give RayClusters regions (KR_OPT_LARGE_GROWTH): the engine's bucket layout has a region arena and table.
bool grows(const kr_engine *e) { return e->large_growth && e->large_on && e->d_grow && e->d_region && e->d_lg; }
// ... and make RayClusters huge, with tiles in the reserve entries of the tile table (KR_OPT_HUGE_GROWTH).
bool huge_grows(const kr_engine *e) { return e->huge_growth && e->huge_on && e->huge_reserve && grows(e); }

// Points the pass at the cluster table of the per-cluster kernels when their list is not empty, or the pass may grow regions
// (`grow`); returns the device list.
const uint32_t *bind_large(const kr_engine *e, ScratchDev &sc, bool grow) {
  if (!e->n_large && !grow) return nullptr;
  sc.lg = reinterpret_cast<uint4 *>(e->d_lg);
  sc.region = e->d_region;  // (nullptr without KR_OPT_LARGE_CLUSTERS: every capacity is then 0)
  return reinterpret_cast<const uint32_t *>(e->d_lg + align_up(16 * (size_t)e->cfg.max_clusters));
}

// The tile scratch of KR_OPT_HUGE_CLUSTERS (layout: kr_engine::d_huge).
HugeDev bind_huge(const kr_engine *e) {
  HugeDev h{};
  if (!e->d_huge) return h;
  const size_t T = e->huge_tiles + e->huge_reserve;
  uint8_t *b = e->d_huge;
  h.tiles = reinterpret_cast<const uint4 *>(b); b += align_up(16 * T);
  h.cnt = reinterpret_cast<uint32_t *>(b); b += align_up(4 * T);
  h.done = reinterpret_cast<uint32_t *>(b); b += align_up(4 * T);
  h.runs = reinterpret_cast<uint32_t *>(b); b += align_up(4 * (size_t)kHugeTile * T);
  h.stash = reinterpret_cast<uint32_t *>(b);
  return h;
}
size_t huge_bytes(size_t T) { return align_up(16 * T) + 2 * align_up(4 * T) + 2 * align_up(4 * (size_t)kHugeTile * T); }
// Tiles a huge RayCluster's bucket and region take: its arrival ranks [0, stride + region capacity) in kHugeTile-rank tiles.
uint32_t huge_tile_count(uint32_t stride, uint32_t cap) { return (stride + cap + kHugeTile - 1) / kHugeTile; }
// Resident tiles of the tile scratch: a huge cluster's tiles cover about 1.25x its pods rounded up to 32, plus at most one partial
// tile, and it lists more than KR_LARGE_MAX_PODS pods: this many tiles hold those of any snapshot within the capacities.
size_t resident_tiles(const kr_config &cfg) {
  const size_t Np = cfg.max_pods, n_huge = Np / (KR_LARGE_MAX_PODS + 1);
  return (Np * 5 / 4 + 32 * (n_huge + 1)) / kHugeTile + n_huge + 2;
}
// Allocates the tile scratch for huge_tiles resident tiles and `reserve` more, zeroed (the per-cluster tile counters start at 0;
// every pass leaves them there).  A scratch allocated before goes once the new one is in place (between passes: the captured graph
// and the table go with it); when the allocation fails, the engine keeps the old scratch and its reserve.
int alloc_huge(kr_engine *e, size_t reserve) {
  const size_t T = e->huge_tiles + reserve;
  uint8_t *d = nullptr;
  CK(cudaMalloc((void **)&d, huge_bytes(T)));
  if (cudaMemset(d, 0, huge_bytes(T)) != cudaSuccess) { cudaFree(d); return fail(e, KR_E_CUDA, "tile scratch of %zu tiles", T); }
  if (e->d_huge) {
    CK(cudaStreamSynchronize(e->sm));
    CK(cudaFree(e->d_huge));
  }
  e->d_huge = d;
  e->huge_reserve = reserve;
  e->lg_stale = true; e->gvalid = false;
  return KR_OK;
}
// A RayCluster of the large half is huge when its region reaches past KR_LARGE_MAX_PODS ranks (it listed more than that many pods):
// k_large_sort's shared memory could not hold it.
bool is_huge(uint32_t stride, uint32_t cap) { return stride + cap > KR_LARGE_MAX_PODS; }

// Drops the large half's entries from `from` on (its rows ascending), in the device table too, and marks the list for upload.  The
// device table holds a region for the rows of the large half only (every other entry is zero): a RayCluster created later in a row the
// half no longer lists starts without a region, whatever the row held before.  (One span: the rows between hold zero already.)
int drop_regions(kr_engine *e, size_t from) {
  if (from >= e->large_rows.size()) return KR_OK;
  const size_t r0 = e->large_rows[from], r1 = e->large_rows.back();
  CK(cudaMemsetAsync(e->d_lg + 16 * r0, 0, 16 * (r1 - r0 + 1), e->sm));
  e->large_rows.resize(from); e->large_reg.resize(from);
  e->lg_stale = true;
  return KR_OK;
}

// Rebuilds the cluster table and the list of the per-cluster kernels from the large half and, with KR_OPT_WIDE_CLUSTERS, the wide
// RayClusters, and uploads them on stream M, ahead of the next pass.  The huge RayClusters go last, after the ones k_large_sort
// takes, and their tiles into the tile table.  A new list length, split or tile count is a new grid of the captured graph.
int upload_lg(kr_engine *e) {
  e->lg_stale = false;
  std::vector<uint32_t> list, huge;  // (both halves ascending: a wide cluster with a region is listed once)
  std::vector<uint4> tiles;
  const uint32_t Nc = e->sizes.n_clusters;
  for (size_t i = 0; i < e->large_rows.size(); i++) {
    const uint32_t c = e->large_rows[i], cap = e->large_reg[i].y;
    if (c >= Nc) return fail(e, KR_E_STATE, "internal: region of RayCluster row %u, past the %u live rows", c, Nc);
    if (!is_huge(e->bstride, cap)) { list.push_back(c); continue; }
    huge.push_back(c);
    const uint32_t nt = huge_tile_count(e->bstride, cap), first = (uint32_t)tiles.size();
    for (uint32_t t = 0; t < nt; t++) tiles.push_back(make_uint4(c, t * kHugeTile, first, nt));
  }
  if (e->wide_on)
    for (uint32_t c : e->rec.wide_rows) if (!std::binary_search(e->large_rows.begin(), e->large_rows.end(), c)) list.push_back(c);
  const uint32_t n_lsort = (uint32_t)list.size();
  list.insert(list.end(), huge.begin(), huge.end());
  if (tiles.size() > e->huge_tiles) return fail(e, KR_E_STATE, "internal: %zu huge-cluster tiles, room for %zu", tiles.size(), e->huge_tiles);
  if ((uint32_t)list.size() != e->n_large || n_lsort != e->n_lsort || (uint32_t)tiles.size() != e->n_tiles) e->gvalid = false;
  e->n_large = (uint32_t)list.size(); e->n_lsort = n_lsort; e->n_tiles = (uint32_t)tiles.size();
  // (KR_OPT_HUGE_GROWTH: the reserve entries past the resident tiles free again, whatever the last incremental pass appended)
  if (huge_grows(e)) tiles.resize(tiles.size() + e->huge_reserve, make_uint4(KR_EMPTY32, 0, 0, 0));
  // (an incremental pass that grows regions reads the table even then: all zero; and so does one that follows a renumbered large
  // half, KR_OPT_LARGE_MOVES, whose vacated rows must read zero)
  if (list.empty() && !grows(e) && !e->lg_moved) return KR_OK;
  e->lg_moved = false;
  std::vector<uint4> lg(Nc, make_uint4(0, 0, 0, 0));  // a wide cluster without a region: capacity 0
  for (size_t i = 0; i < e->large_rows.size(); i++) lg[e->large_rows[i]] = make_uint4(e->large_reg[i].x, e->large_reg[i].y, 0, 0);
  CK(cudaStreamSynchronize(e->sm));  // the previous upload has left the host copies
  e->h_lg.swap(lg); e->h_lg_list.swap(list); e->h_tiles.swap(tiles);
  CK(cudaMemcpyAsync(e->d_lg, e->h_lg.data(), 16 * (size_t)Nc, cudaMemcpyHostToDevice, e->sm));
  if (!e->h_lg_list.empty())
    CK(cudaMemcpyAsync(e->d_lg + align_up(16 * (size_t)e->cfg.max_clusters), e->h_lg_list.data(), 4 * e->h_lg_list.size(), cudaMemcpyHostToDevice, e->sm));
  if (!e->h_tiles.empty()) CK(cudaMemcpyAsync(e->d_huge, e->h_tiles.data(), 16 * e->h_tiles.size(), cudaMemcpyHostToDevice, e->sm));
  return KR_OK;
}

// hash order: message ids by descending SHA-1 block count (counting sort; the kernels run length-homogeneous warps, longest first).
// The RayClusters whose Recreate gate compares a digest lead the order: their digests are ready when the decide kernel, running
// beside the hash, gets to them (k_decide2 waits for a digest's last word otherwise).  Fills h_order (no upload still reading it).
void build_order(kr_engine *e, const kr_snapshot_bufs &hb) {
  const kr_sizes &n = e->sizes;
  uint32_t maxb = 0;
  for (uint32_t c = 0; c < n.n_clusters; c++) maxb = std::max(maxb, (hb.c_json_len[c] + 8) / 64 + 1);
  auto blocks_of = [&](uint32_t c) { return (hb.c_json_len[c] + 8) / 64 + 1; };
  auto lead = [&](uint32_t c) { return (hb.c_flags[c] & KR_CF_UPGRADE_RECREATE) ? 0u : 1u; };
  if (maxb <= (1u << 20)) {  // counting sort on (not Recreate, descending block count): bucket 0 = the longest Recreate message
    std::vector<uint32_t> start(2 * ((size_t)maxb + 1) + 1, 0);
    auto key = [&](uint32_t c) { return lead(c) * (maxb + 1) + (maxb - blocks_of(c)); };
    for (uint32_t c = 0; c < n.n_clusters; c++) start[key(c) + 1]++;
    for (size_t b = 0; b + 1 < start.size(); b++) start[b + 1] += start[b];
    for (uint32_t c = 0; c < n.n_clusters; c++) e->h_order[start[key(c)]++] = c;
  } else {
    for (uint32_t c = 0; c < n.n_clusters; c++) e->h_order[c] = c;
    std::stable_sort(e->h_order, e->h_order + n.n_clusters, [&](uint32_t a, uint32_t b) { return lead(a) != lead(b) ? lead(a) < lead(b) : blocks_of(a) > blocks_of(b); });
  }
}

// Spec-row commits keep the full-pass hash order as it was; a pass that hashes every message rebuilds it first when their block
// counts moved (uploaded on stream M, ahead of the pass).
int refresh_order(kr_engine *e) {
  e->rec.spec_order_stale = false;
  if (!e->sizes.n_clusters) return KR_OK;
  if (e->order_pending) { CK(cudaEventSynchronize(e->ev_order)); e->order_pending = false; }
  kr_snapshot_bufs hb;
  bind_in(e->il, e->h_in, &hb);
  build_order(e, hb);
  CK(cudaMemcpyAsync(e->d_order, e->h_order, 4 * (size_t)e->sizes.n_clusters, cudaMemcpyHostToDevice, e->sm));
  CK(cudaEventRecord(e->ev_order, e->sm));
  e->order_pending = true;
  e->prof.h2d_bytes = (e->h2d_accum += 4 * (uint64_t)e->sizes.n_clusters);  // (as when a commit uploads the order)
  return KR_OK;
}

// the spec rows were hashed (or every message was): a new epoch of the row stamps
void clear_spec_rows(kr_engine *e) {
  e->spec_pending.clear();
  if (++e->spec_epoch == 0) { std::fill(e->spec_stamp.begin(), e->spec_stamp.end(), 0u); e->spec_epoch = 1; }
}

// every pass: the caller may rewrite the arenas once it returns, so the next spec commit pulls its rows again (the pass waits for
// the pulls enqueued so far: their pinned list entries are free again)
void new_pull_epoch(kr_engine *e) {
  e->n_pull = 0;
  if (++e->pull_epoch == 0) { std::fill(e->pull_stamp.begin(), e->pull_stamp.end(), 0u); e->pull_epoch = 1; }
}

// The hash order of the pending spec rows (descending SHA-1 block count, so warps are length-homogeneous), uploaded on stream M ahead
// of the pass that hashes them; returns its device address.
const uint32_t *upload_spec_order(kr_engine *e) {
  const size_t cap = (size_t)e->cfg.max_clusters + 1;
  kr_snapshot_bufs hb;
  bind_in(e->il, e->h_in, &hb);
  uint32_t *h = reinterpret_cast<uint32_t *>(e->spec.h + 16 * cap);
  const uint32_t n = (uint32_t)e->spec_pending.size();
  std::copy(e->spec_pending.begin(), e->spec_pending.end(), h);
  std::stable_sort(h, h + n, [&](uint32_t a, uint32_t b) { return (hb.c_json_len[a] + 8) / 64 > (hb.c_json_len[b] + 8) / 64; });
  uint32_t *d = reinterpret_cast<uint32_t *>(e->spec.d + 16 * cap);
  if (cudaMemcpyAsync(d, h, 4 * (size_t)n, cudaMemcpyHostToDevice, e->sm) != cudaSuccess) return nullptr;
  e->prof.h2d_bytes = (e->h2d_accum += 4 * (uint64_t)n);  // (the pass's own upload: reported with the commits that fed it)
  return d;
}

// What the launches of a pass share: the arenas and the per-cluster kernels' tables bound for this layout, stream M and the hash
// stream H (M as well when profiling).  mark() counts a kernel in kr_profile.n_kernels and, profiling, names it and records its
// start event on M; close() records the last kernel's end event and stores the count.
struct PassCtx {
  kr_engine *e; bool profile;
  SnapDev s; ResDev r; ScratchDev sc; const uint32_t *lg_list; HugeDev hd; Sizes z;
  cudaStream_t M, H;
  int k = 0;
  PassCtx(kr_engine *e_, bool profile_, bool grow = false)
      : e(e_), profile(profile_), r(bind_out(e->ol, e->d_out)), sc(bind_scratch(e->sl, e->d_scratch)), lg_list(bind_large(e, sc, grow)),
        hd(bind_huge(e)), z(sizes_of(e->sizes)), M(e->sm), H(profile ? e->sm : e->sh) {
    bind_in(e->il, e->d_in, &s);
    sc.bucket_stride = e->bstride;
    e->prof.n_kernels = 0;
  }
  void mark(const char *name) {
    if (profile && k < KR_MAX_KERNEL_TIMES) { e->prof.kernel_name[k] = name; cudaEventRecord(e->ev_k[k], M); }
    k++;
  }
  void close() {
    if (profile && k <= KR_MAX_KERNEL_TIMES) cudaEventRecord(e->ev_k[k], M);
    e->prof.n_kernels = (uint32_t)k;
  }
};

// SHA-1 digests of the n messages (json + off[i], len[i]) taken in `order` (descending block count: length-homogeneous warps,
// longest first).  Latency regime (C3: 313 groups of 32): the caller waits for the longest message's serial chain — warp-specialised
// pairs, two per SM so that every hash warp has a scheduler to itself.  Throughput regime: up to ctas_per_sm resident CTAs per SM of
// four one-lane-per-message warps walk the groups, round adds on the FMA pipe.
void launch_hash(const kr_engine *e, cudaStream_t st, const uint8_t *json, const uint64_t *off, const uint32_t *len, const uint32_t *order,
                 uint32_t n, char *out, int ctas_per_sm) {
  const uint32_t ngroups = (n + 31) / 32;
  if (ngroups <= (uint32_t)e->sm_count * 4)
    k_hash3<1, 0><<<std::min<uint32_t>(ngroups, (uint32_t)e->sm_count * 2), 64, sizeof(H3Smem), st>>>(json, off, len, order, n, out);
  else
    k_hash2<4, 1><<<std::min<uint32_t>((n + 127) / 128, (uint32_t)e->sm_count * ctas_per_sm), 128, 0, st>>>(json, off, len, order, n, out, 1u);
}

// k_decide2 for this layout's bucket stride; the instantiation with the multi-host branch when the snapshot has a multi-host
// group and the gate is on, and the incremental epoch's one (phase 2) when `inc`.
cudaError_t launch_decide2(const PassCtx &c, const Decide2Args &da, dim3 grid, bool inc, bool pdl) {
  using Kernel = void (*)(Decide2Args);
  static const Kernel kern[3][2][2] = {  // [stride 64 / 128 / 256][inc][multi-host]
      {{k_decide2<2>, k_decide2<2, false, true>}, {k_decide2<2, true>, k_decide2<2, true, true>}},
      {{k_decide2<4>, k_decide2<4, false, true>}, {k_decide2<4, true>, k_decide2<4, true, true>}},
      {{k_decide2<8>, k_decide2<8, false, true>}, {k_decide2<8, true>, k_decide2<8, true, true>}}};
  const int st = c.e->bstride <= 64 ? 0 : c.e->bstride <= 128 ? 1 : 2;
  const bool mh = c.e->rec.n_mh > 0 && da.f.gate_multihost_indexing;
  return launch_pdl(kern[st][inc][mh], grid, dim3(kD2Warps * 32), 0, c.M, pdl, da);
}

// The sorts of the per-cluster kernels' RayClusters (kr_large.cuh): k_large_sort for the first n_lsort of the list (and, with `grown`,
// k_inc_grow's result, for the RayClusters it listed), the huge ones after them tile by tile, then merged (kr_huge.cuh).  reserve:
// the tile table's reserve entries too (KR_OPT_HUGE_GROWTH, incremental: k_inc_grow may have appended tiles there).
template <bool kInc>
void launch_large_sort(PassCtx &c, const Decide2Args &da, const uint4 *grown = nullptr, uint32_t reserve = 0) {
  const kr_engine *e = c.e;
  const uint32_t n = e->n_lsort + (grown ? KR_GROW_MAX : 0), nt = e->n_tiles + reserve;
  if (n) { c.mark("k_large_sort"); k_large_sort<kInc><<<n, kLargeSortThreads, 0, c.M>>>(da, c.lg_list, e->n_lsort, grown); }
  if (nt) {
    c.mark("k_huge_tiles"); k_huge_tiles<kInc><<<nt, kHugeThreads, 0, c.M>>>(da, c.hd);
    c.mark("k_huge_merge"); k_huge_merge<kInc><<<nt, kHugeThreads, 0, c.M>>>(da, c.hd);
  }
}

// The decides of the per-cluster kernels' RayClusters (kr_large.cuh): k_decide_large over the list (and, with `grown`, one CTA per
// RayCluster k_inc_grow listed), then k_decide_huge over its huge part, but for the wide RayClusters there, which k_decide_large keeps.
template <bool kInc>
void launch_large_decide(PassCtx &c, const Decide2Args &da, const uint4 *grown = nullptr) {
  const kr_engine *e = c.e;
  c.mark("k_decide_large");
  k_decide_large<kInc, kLargeDecideThreads><<<e->n_large + (grown ? KR_GROW_MAX : 0), kLargeDecideThreads, 0, c.M>>>(da, c.lg_list, e->n_large, e->n_lsort, grown);
  if (const uint32_t n_huge = e->n_large - e->n_lsort) {
    c.mark("k_decide_huge");
    k_decide_large<kInc, kHugeDecideThreads><<<n_huge, kHugeDecideThreads, 0, c.M>>>(da, c.lg_list + e->n_lsort, n_huge, 0u, nullptr);
  }
}

// Every RayCluster's full pod list from the bucket pipeline's resident state (kr_lists.cuh), behind the pass's last decide kernel on
// stream M: owners, the radix pipeline's stable sort by owner, then the actions along the list and the starts.
void launch_lists(PassCtx &c, bool inc) {
  const kr_engine *e = c.e;
  const ScratchDev &sc = c.sc;
  const uint32_t Np = c.z.n_pods, Nc = c.z.n_clusters;
  const ListsArgs la{c.s, sc, c.r, c.z, sc.keys[0], sc.act_tmp_code, reinterpret_cast<uint32_t *>(e->d_out + e->ol.pod_start), inc ? 1 : 0};
  int cur = 0;
  if (Np) {
    c.mark("k_lists_init");
    k_lists_init<<<(Np + 255) / 256, 256, 0, c.M>>>(la);
    if (Nc) { c.mark("k_lists_owner"); k_lists_owner<<<(Nc + 7) / 8, 256, 0, c.M>>>(la); }  // (a warp per RayCluster)
    uint32_t bits = 1;
    while ((1ull << bits) <= Nc) bits++;  // keys are in [0, n_clusters]
    const uint32_t nt = (Np + kSortTile - 1) / kSortTile;  // (the live rows: at most the layout's tiles)
    for (uint32_t shift = 0; shift < bits; shift += kRadixBits) {
      c.mark("k_hist"); k_hist<<<nt, kSortThreads, 0, c.M>>>(sc.keys[cur], sc.hist, Np, (int)shift);
      c.mark("k_scan_rows"); k_scan_rows<<<kRadix, kRowScanThreads, 0, c.M>>>(sc.hist, sc.row_total, nt);
      c.mark("k_scatter");
      uint32_t *vout = shift + kRadixBits >= bits ? c.r.sorted_pod_idx : sc.vals[cur ^ 1];
      k_scatter<<<nt, kSortThreads, 0, c.M>>>(sc.keys[cur], sc.vals[cur], sc.keys[cur ^ 1], vout, sc.hist, sc.row_total, Np, (int)shift, shift == 0);
      cur ^= 1;
    }
  }
  c.mark("k_lists_gather");
  k_lists_gather<<<Np / 256 + 1, 256, 0, c.M>>>(la, sc.keys[cur]);  // (a thread per list position and one past the end)
}

// Launches the whole pass.  profile: serialise everything on stream M and bracket each kernel with events.
int launch_pass(kr_engine *e, const kr_flags &f, bool profile, bool capturing = false) {
  PassCtx c(e, profile);
  const kr_sizes &n = e->sizes;
  const SnapDev &s = c.s; const ResDev &r = c.r; const ScratchDev &sc = c.sc; const Sizes &z = c.z;
  const cudaStream_t M = c.M, H = c.H;

  // --- stream H: hash (only needs the committed snapshot)
  const bool do_hash = !f.skip_hash && n.n_clusters > 0;
  // the committed snapshot: columns gate stream M, the JSON arena gates the hash
  const unsigned wflag = capturing ? cudaEventWaitExternal : cudaEventWaitDefault;
  // (the fork comes first so the hash can start while the columns are still landing — an incremental pod-row epoch leaves the JSON untouched)
  // bucket pipeline (kr_bucket2.cuh): the caller does not fetch the full pod lists (or KR_OPT_BUCKET_POD_LISTS builds them there),
  // every RayCluster has few worker groups (or KR_OPT_WIDE_CLUSTERS lists the others for the per-cluster kernels) and (checked on the
  // device) at most `bstride` pods
  const bool bucket = !e->no_bucket && (!f.fetch_pod_lists || e->bucket_lists) && e->bstride != 0 && !e->force_radix && (e->rec.snap_max_groups <= KR_SMEM_GROUPS || e->wide_on) &&
                      (size_t)n.n_clusters * e->bstride <= e->sl.bucket_entries;
  // ... and there the clusters whose Recreate gate reads a digest wait for it inside the decide kernel (the hash runs beside it)
  const bool spin = bucket && !profile && do_hash && e->hash_spin && e->rec.n_recreate > 0;
  // the digests, messages taken in e->d_order (built at commit), or zeros when the pass skips the hash
  auto hash_or_zero = [&]() -> int {
    if (do_hash) { c.mark("k_hash"); launch_hash(e, H, s.json, s.c_json_off, s.c_json_len, e->d_order, n.n_clusters, r.hash, e->hash_ctas_per_sm); }
    else if (n.n_clusters) CK(cudaMemsetAsync(r.hash, 0, 32 * (size_t)n.n_clusters, H));
    return KR_OK;
  };
  // where stream M needs the digests: it joins the hash stream (profiled, it runs the hash itself there, once the JSON arena and
  // the hash order have landed: the commit sends both after ev_cols, the only upload stream M waited for so far)
  auto join_hash = [&]() -> int {
    if (profile) {
      CK(cudaStreamWaitEvent(M, e->ev_json, 0));
      return hash_or_zero();
    }
    CK(cudaStreamWaitEvent(M, e->ev_hash, 0));
    return KR_OK;
  };
  // The hash goes first: its 313 one-warp CTAs must be resident before the main chain fills the SMs (launched after
  // k_build_tables instead, they queue behind the chain's blocks and the hash takes more than twice as long).
  if (!profile) {
    CK(cudaEventRecord(e->ev_fork, M)); CK(cudaStreamWaitEvent(H, e->ev_fork, 0));
    CK(cudaStreamWaitEvent(H, e->ev_json, wflag));
    if (spin) CK(cudaMemsetAsync(r.hash, 0, 32 * (size_t)n.n_clusters, H));  // the digests' last words are "ready" marks (k_decide2)
    if (int rc = hash_or_zero()) return rc;  // (the hash counts among the pass's kernels: kr_profile.n_kernels)
    CK(cudaEventRecord(e->ev_hash, H));
  }

  // --- stream M
  e->ran_bucket = bucket;
  const bool pdl = !profile && e->use_pdl;
  bool fuse_place_done = false;    // k_decide_small directly follows k_place_fused on stream M
  bool creates_after_kernel = false;  // k_creates_fused directly follows a kernel on stream M (no event wait in between)
  {
    ClearArgs ca{};
    ca.ptr[0] = reinterpret_cast<uint32_t *>(e->d_scratch); ca.words[0] = (uint32_t)(e->sl.ff_total / 4); ca.value[0] = 0xFFFFFFFFu;
    ca.ptr[1] = r.wtd_pod_idx; ca.words[1] = n.n_wtd; ca.value[1] = 0xFFFFFFFFu;
    ca.ptr[2] = r.totals; ca.words[2] = 64; ca.value[2] = 0;  // the 8 counters and, 128 bytes in, the void-attempt word (the block is 256 bytes)
    // per-cluster counts + the chained-scan cells + the workersToDelete Bloom bitmap + the bucket fill counters / first-head
    // cells (one region)
    ca.ptr[3] = sc.ccount; ca.words[3] = (uint32_t)((e->sl.cstart - e->sl.ccount) / 4); ca.value[3] = 0;
    c.mark("k_clear");
    k_clear<<<e->sm_count * 2, 256, 0, M>>>(ca);
  }
  CK(cudaStreamWaitEvent(M, e->ev_cols, wflag));  // the scratch clears above overlap the tail of the upload
  {
    uint32_t items = n.n_clusters + n.n_groups + n.n_heads;
    if (items) { c.mark("k_build_tables"); k_build_tables<<<(items + 255) / 256, 256, 0, M>>>(s, sc, r, z); }
  }
  if (bucket) {
    e->ran_fast = false;
    const uint32_t mtiles = e->sl.mtiles;
    if (n.n_pods) {
      c.mark("k_match2");
      CK(launch_pdl(k_match2<kMatchItems>, dim3(mtiles), dim3(kSortThreads), n.n_wtd ? e->sl.wt_bits_n / 8 : 0, M, pdl, s, sc, r, z, n.n_wtd ? 1 : 0));
    }
    Decide2Args da{s, sc, r, z, f, IncStage{}, e->cfg.max_creates, spin ? 1 : 0, 0};
    if (n.n_clusters) {
      c.mark("k_decide2");
      CK(launch_decide2(c, da, dim3((n.n_clusters + kD2Warps - 1) / kD2Warps), false, pdl && n.n_pods != 0));
    } else CK(cudaMemsetAsync(r.act_start, 0, 4, M));
    if (n.n_jobs) { c.mark("k_jobs"); k_jobs<<<(n.n_jobs + 255) / 256, 256, 0, M>>>(s, sc, r, z); }
    const bool large = e->n_large && sc.lg && n.n_clusters;  // large RayClusters (kr_large.cuh): sorted beside the hash, decided after it
    if (large) launch_large_sort<false>(c, da);
    if (int rc = join_hash()) return rc;
    if (large) launch_large_decide<false>(c, da);
    if (e->rec.n_recreate > 0 && do_hash && !spin) {  // clusters whose Recreate gate needs the digest: decided again, in the places phase 0 reserved
      da.phase = 1;
      c.mark("k_decide2_phase1");
      CK(launch_decide2(c, da, dim3((e->rec.n_recreate + kD2Warps - 1) / kD2Warps), false, false));
    }
    if (f.fetch_pod_lists) launch_lists(c, false);  // (KR_OPT_BUCKET_POD_LISTS: behind the last decide)
  } else {
  const uint32_t ntiles = e->sl.ntiles;
  const bool fast = !e->force_radix;
  e->ran_fast = fast;
  const uint32_t *sorted_keys = sc.keys[0];
  if (n.n_pods && fast) {
    c.mark("k_match");
    const uint32_t mtiles = e->sl.mtiles;
    CK(launch_pdl(k_match<true, kMatchItems>, dim3(mtiles), dim3(kSortThreads), 0, M, pdl, s, sc, r, z, n.n_wtd ? 1 : 0));
    const bool fuse_place = !e->no_fuse && (uint64_t)n.n_clusters + 2 + mtiles <= kFusedMaxCounters;
    if (fuse_place) {
      fuse_place_done = true;
      c.mark("k_place_fused");
      size_t smem = 4 * ((size_t)n.n_clusters + 2 + mtiles);
      CK(launch_pdl(k_place_fused, dim3(e->sm_count * e->place_ctas), dim3(1024), smem, M, pdl, (const uint32_t *)sc.keys[0], (const uint32_t *)sc.keys[1], (const uint32_t *)sc.ccount, sc.cstart,
                    (const uint32_t *)sc.tile_orph, sc.vals[0], n.n_pods, n.n_clusters, mtiles, r.totals));
    } else {
    c.mark("k_scan_counts");
    const uint32_t nch_c = (n.n_clusters + 1 + kScanChunk - 1) / kScanChunk, nch_t = (mtiles + kScanChunk - 1) / kScanChunk;
    k_scan_counts<<<nch_c + nch_t, 1024, 0, M>>>(sc.ccount, sc.cstart, n.n_clusters + 1, nch_c, sc.tile_orph, mtiles, sc.chain, r.totals);
    c.mark("k_place");
    k_place<<<(n.n_pods + 1023) / 1024, 256, 0, M>>>(sc.keys[0], sc.keys[1], sc.cstart, sc.tile_orph, sc.vals[0], n.n_pods, n.n_clusters);
    }
  } else if (n.n_pods) {
    uint32_t bits = 1;
    while ((1ull << bits) <= n.n_clusters) bits++;  // keys are in [0, n_clusters]
    const int passes = (int)((bits + kRadixBits - 1) / kRadixBits);
    c.mark("k_match");
    k_match<false, kSortItems><<<ntiles, kSortThreads, 0, M>>>(s, sc, r, z, n.n_wtd ? 1 : 0);
    int cur = 0;
    for (int p = 0; p < passes; p++) {
      if (p > 0) { c.mark("k_hist"); k_hist<<<ntiles, kSortThreads, 0, M>>>(sc.keys[cur], sc.hist, n.n_pods, p * kRadixBits); }
      c.mark("k_scan_rows");
      k_scan_rows<<<kRadix, kRowScanThreads, 0, M>>>(sc.hist, sc.row_total, ntiles);
      c.mark("k_scatter");
      uint32_t *vout = (p == passes - 1) ? r.sorted_pod_idx : sc.vals[cur ^ 1];
      k_scatter<<<ntiles, kSortThreads, 0, M>>>(sc.keys[cur], sc.vals[cur], sc.keys[cur ^ 1], vout, sc.hist, sc.row_total, n.n_pods, p * kRadixBits, p == 0);
      cur ^= 1;
    }
    sorted_keys = sc.keys[cur];
  } else if (fast) {
    CK(cudaMemsetAsync(sc.cstart, 0, 4 * ((size_t)n.n_clusters + 2), M));
  }
  DecideArgs da{s, sc, r, z, f, sorted_keys, sc.vals[0], fast ? 1 : 0, 0};
  {
    // fast pipeline: k_decide_small (buckets kept in registers) and the general k_decide run side by side
    cudaStream_t G2 = (fast && !profile) ? e->sg : M;
    if (fast && !profile) { CK(cudaEventRecord(e->ev_fork2, M)); CK(cudaStreamWaitEvent(G2, e->ev_fork2, 0)); }
    uint32_t warps = n.n_clusters + 1;
    c.mark("k_decide");
    k_decide<<<(warps + kDecideWarps - 1) / kDecideWarps, kDecideWarps * 32, 0, G2>>>(da);
    if (fast && n.n_clusters) {
      c.mark("k_decide_small");
      CK(launch_pdl(k_decide_small, dim3((n.n_clusters + kDecideWarps - 1) / kDecideWarps), dim3(kDecideWarps * 32), 0, M, pdl && fuse_place_done, da));
    }
    if (fast && !profile) { CK(cudaEventRecord(e->ev_join2, G2)); CK(cudaStreamWaitEvent(M, e->ev_join2, 0)); }
  }
  if (n.n_jobs) { c.mark("k_jobs"); k_jobs<<<(n.n_jobs + 255) / 256, 256, 0, M>>>(s, sc, r, z); }
  if (int rc = join_hash()) return rc;
  if (e->rec.n_recreate > 0 && do_hash) {
    da.phase = 1;
    uint32_t warps = e->rec.n_recreate;  // upper bound on the deferred list
    const dim3 grid1((warps + kDecideWarps - 1) / kDecideWarps), block1(kDecideWarps * 32);
    // like phase 0: the register-resident kernel on M for the small clusters, the general one beside it on G for the rest
    cudaStream_t G1 = (fast && !profile) ? e->sg : M;
    if (fast && !profile) { CK(cudaEventRecord(e->ev_fork3, M)); CK(cudaStreamWaitEvent(G1, e->ev_fork3, 0)); }
    c.mark("k_decide_phase1");
    k_decide<<<grid1, block1, 0, G1>>>(da);
    if (fast) { c.mark("k_decide_small_phase1"); k_decide_small<<<grid1, block1, 0, M>>>(da); }
    if (fast && !profile) { CK(cudaEventRecord(e->ev_join3, G1)); CK(cudaStreamWaitEvent(M, e->ev_join3, 0)); }
    creates_after_kernel = !(fast && !profile);
  }
  if (!e->no_fuse && (uint64_t)n.n_groups + n.n_clusters + 1 <= kFusedMaxCounters) {
    c.mark("k_creates_fused");
    CK(launch_pdl(k_creates_fused, dim3(e->sm_count), dim3(1024), 4 * ((size_t)n.n_groups + n.n_clusters + 1), M, pdl && creates_after_kernel, s, sc, r, z, f, e->cfg.max_creates));
  } else {
    const uint32_t nch_a = (n.n_clusters + kScanChunk - 1) / kScanChunk;
    uint32_t *achain = sc.chain + 2 * ((size_t)(n.n_clusters + 1 + kScanChunk - 1) / kScanChunk + (e->sl.mtiles + kScanChunk - 1) / kScanChunk + (n.n_groups + kScanChunk - 1) / kScanChunk + 1);
    if (n.n_clusters) {
      if (e->force_radix) CK(cudaMemsetAsync(achain, 0, 8 * (size_t)nch_a, M));
      c.mark("k_scan_actions");
      k_scan_actions<<<nch_a, 1024, 0, M>>>(r, sc.cact, n.n_clusters, achain);
      c.mark("k_compact_actions");
      k_compact_actions<<<(n.n_clusters + 3) / 4, 128, 0, M>>>(r, sc, n.n_clusters);
    } else CK(cudaMemsetAsync(r.act_start, 0, 4, M));
  }
  if (e->no_fuse || (uint64_t)n.n_groups + n.n_clusters + 1 > kFusedMaxCounters) if (n.n_groups) {
    c.mark("k_scan_creates");
    const uint32_t nch_g = (n.n_groups + kScanChunk - 1) / kScanChunk;
    uint32_t *gchain = sc.chain + 2 * ((size_t)(n.n_clusters + 1 + kScanChunk - 1) / kScanChunk + (e->sl.mtiles + kScanChunk - 1) / kScanChunk);
    if (e->force_radix) CK(cudaMemsetAsync(gchain, 0, 8 * (size_t)nch_g, M));  // (the fast pipeline cleared the cells together with ccount)
    k_scan_creates<<<nch_g, 1024, 0, M>>>(r, sc.gcreate, n.n_groups, gchain);
    c.mark("k_create_fill");
    k_create_fill<<<(n.n_groups + 3) / 4, 128, 0, M>>>(s, sc, r, z, f, e->cfg.max_creates);
  }
  }  // sort / radix pipelines
  c.close();
  CK(cudaGetLastError());
  return KR_OK;
}

// Replays the captured CUDA graph of the pass (captures it first when the layout / flags changed).
int run_pass_once(kr_engine *e, const kr_flags &f) {
  if (!e->use_graph) return launch_pass(e, f, false);
  kr_flags fk = f;  // (fetch_pod_lists selects the pipeline, or the list builder on the bucket pipeline: part of the key)
  if (!e->gvalid || memcmp(&e->gflags, &fk, sizeof fk) != 0) {
    e->gvalid = false;
    CK(cudaStreamBeginCapture(e->sm, cudaStreamCaptureModeThreadLocal));
    int rc = launch_pass(e, f, false, true);
    cudaGraph_t g = nullptr;
    cudaError_t ce = cudaStreamEndCapture(e->sm, &g);
    if (rc != KR_OK) { if (g) cudaGraphDestroy(g); cudaGetLastError(); return rc; }
    if (ce != cudaSuccess) return fail(e, KR_E_CUDA, "graph capture failed: %s", cudaGetErrorString(ce));
    // New row counts / pointers with the same kernel chain are a parameter update of the instantiated graph (cheap);
    // a different chain (fast <-> radix, fused <-> unfused, phase 1 or RayJobs appearing) is instantiated afresh.
    bool updated = false;
    if (e->gexec) {
      cudaGraphExecUpdateResultInfo info;
      updated = cudaGraphExecUpdate(e->gexec, g, &info) == cudaSuccess;
      if (!updated) { cudaGetLastError(); cudaGraphExecDestroy(e->gexec); e->gexec = nullptr; }
    }
    if (!updated) ce = cudaGraphInstantiate(&e->gexec, g, 0);
    cudaGraphDestroy(g);
    if (ce != cudaSuccess) return fail(e, KR_E_CUDA, "graph instantiate failed: %s", cudaGetErrorString(ce));
    e->gflags = fk;
    e->gvalid = true;
  }
#ifdef KR_TIMELINE
  {
    unsigned long long init[64];
    for (int i = 0; i < 64; i++) init[i] = (i & 1) ? 0ull : ~0ull;
    CK(cudaMemcpyToSymbolAsync(g_tl, init, sizeof init, 0, cudaMemcpyHostToDevice, e->sm));
  }
#endif
  CK(cudaGraphLaunch(e->gexec, e->sm));
  return KR_OK;
}


// A bucket attempt voided: some RayCluster listed more pods than the stride holds (k_match2 counted them all in cl_dyn[].x) or
// outgrew its region.  Widen the stride (64 -> 128 -> 256) or leave the bucket pipeline for this layout; with KR_OPT_LARGE_CLUSTERS
// the RayClusters of more than 256 (and at most KR_LARGE_MAX_PODS, or any number with KR_OPT_HUGE_CLUSTERS) pods get regions
// instead, and only the others widen the stride.
// A void rebuilds only the large half of the per-cluster kernels' list: the wide RayClusters stay on it.
int after_bucket_void(kr_engine *e) {
  const uint32_t Nc = e->sizes.n_clusters;
  auto fits = [&](uint32_t st) { return st <= 256 && (size_t)Nc * st <= e->sl.bucket_entries; };
  if (!e->large_on) { e->bstride = fits(e->bstride * 2) ? e->bstride * 2 : 0; return KR_OK; }  // (no large half)
  std::vector<uint4> dyn(Nc);
  CK(cudaMemcpyAsync(dyn.data(), e->d_scratch + e->sl.cl_dyn, 16 * (size_t)Nc, cudaMemcpyDeviceToHost, e->sm));
  CK(cudaStreamSynchronize(e->sm));
  if (int rc = drop_regions(e, 0)) return rc;  // (rebuilt below from this attempt's counts; a layout that leaves the bucket pipeline
  e->lg_cursor = 0;                             // uploads nothing it would read)
  uint32_t st = e->bstride, n_big = 0, most = 0;
  for (const uint4 &d : dyn) { if (d.x > 256) n_big++; if (d.x <= 256) most = std::max(most, d.x); }
  if (!e->huge_on)
    for (const uint4 &d : dyn) if (d.x > KR_LARGE_MAX_PODS) { e->bstride = 0; return KR_OK; }  // the sort / radix pipelines take it, as before
  if (n_big == 0) {
    e->bstride = fits(st * 2) ? st * 2 : 0;
    return e->bstride ? upload_lg(e) : KR_OK;
  }
  while (st < most && fits(st * 2)) st <<= 1;
  if (st < most) { e->bstride = 0; return KR_OK; }
  // regions: ranks [st, st + cap) of every large cluster, cap = 1.25x its pods rounded up to 32 (at most KR_LARGE_MAX_PODS unless
  // the cluster is huge), less the stride
  size_t off = 0, tiles = 0;
  for (uint32_t c = 0; c < Nc; c++) {
    if (dyn[c].x <= 256) continue;
    const uint32_t cap = large_region_cap(dyn[c].x, st);
    e->large_rows.push_back(c); e->large_reg.push_back(make_uint2((uint32_t)off, cap));
    off += cap;
    if (is_huge(st, cap)) tiles += huge_tile_count(st, cap);
  }
  if (off > e->large_entries || tiles > e->huge_tiles) { e->bstride = 0; return drop_regions(e, 0); }
  e->bstride = st;
  e->lg_cursor = off;
  return upload_lg(e);  // (on the pass's stream: ordered before the rerun)
}
// A commit drops the resident state: its cause goes to the next pass's report (and so do the causes of the epoch's later commits).
void drop_state(kr_engine *e, uint32_t why) {
  if (e->inc_valid || e->epoch_dropped) { e->why_full |= why; e->epoch_dropped = true; }
  e->inc_valid = false;
}
// Why a full pass left nothing resident (KR_FULL_*; 0: it did): every term of run_pass_once's bucket-pipeline test, and of
// after_full_pass's, that failed.
uint32_t why_not_resident(const kr_engine *e, const kr_flags &f) {
  if (e->inc_valid) return 0;
  uint32_t why = 0;
  if (e->no_incr || e->no_bucket || e->env_radix) why |= KR_FULL_DISABLED;
  if (e->ran_bucket) return e->h_totals[9] > e->cfg.max_creates ? why | KR_FULL_CAPACITY : why;  // (totals[9]: the bucket pipeline's create extent)
  if (f.fetch_pod_lists && !e->bucket_lists) why |= KR_FULL_POD_LISTS;
  if (e->bstride == 0 || (e->force_radix && !e->env_radix) || (size_t)e->sizes.n_clusters * e->bstride > e->sl.bucket_entries) why |= KR_FULL_LARGE;
  if (e->rec.snap_max_groups > KR_SMEM_GROUPS && !e->wide_on) why |= KR_FULL_WIDE;
  return why;
}
// The pass's results stand: run_pass makes its report (the call publishes it when it returns KR_OK), and the causes recorded for
// it make way for those the pass leaves for the next one.
void make_report(kr_engine *e, bool inc, uint32_t attempts, bool hash_wait, uint32_t why_next) {
  kr_pass_report &p = e->pass_made;
  p = kr_pass_report{};
  p.kind = inc ? KR_PASSK_INCREMENTAL : KR_PASSK_FULL;
  p.pipeline = e->ran_bucket ? KR_PIPE_BUCKET : e->ran_fast ? KR_PIPE_SORT : KR_PIPE_RADIX;
  p.attempts = (uint8_t)attempts;
  p.hash_wait = hash_wait ? 1 : 0;
  p.stride = e->ran_bucket ? e->bstride : 0;
  p.why_full = e->why_full;
  e->why_full = why_next;
  e->epoch_dropped = false;
}
// a bucket-pipeline pass leaves everything an incremental epoch needs on the device
void after_full_pass(kr_engine *e, const kr_flags &f) {
  // (a pass whose create runs overran kr_config.max_creates is reported as KR_E_CAPACITY and left groups' runs unwritten: an
  // incremental epoch would inherit that cursor and fail the same way, so the next pass starts over)
  e->inc_valid = e->ran_bucket && !e->no_incr && e->h_totals[9] <= e->cfg.max_creates;
  // (without fetch_pod_lists: a pass that left the state resident took the bucket pipeline, so it did not fetch them or
  // KR_OPT_BUCKET_POD_LISTS made them output only)
  e->inc_flags = f; e->inc_flags.fetch_pod_lists = 0; e->inc_n_pods = e->sizes.n_pods; e->inc_n_heads = e->sizes.n_heads; e->inc_n_clusters = e->sizes.n_clusters;
  e->host_results_stale = false; e->inc_n_dirty = 0; e->fetched = false; e->ran_inc = false; e->rec.heads_rebuild = false;
  e->rec.wtd_rebuild = false; e->res_n_wtd = e->sizes.n_wtd; e->map_pending = false;
  if (!f.skip_hash) { e->rec.hash_dirty = false; clear_spec_rows(e); }
}

// A pass has read what the commits since the previous one uploaded: the pinned hash order is free again, and kr_profile keeps the
// commits' bytes (h2d_bytes) and copy time (h2d_ms).
void commits_read(kr_engine *e) {
  e->order_pending = false;
  e->h2d_accum = 0;  // (kr_profile.h2d_bytes keeps the sum of the commits that fed this pass)
  if (!e->h2d_timed) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, e->ev_h2d0, e->ev_h2d1) == cudaSuccess) e->prof.h2d_ms = ms;
    e->h2d_timed = true;
  }
}

// One incremental pass over the resident state (kr_incr.cuh).  Returns KR_OK with *done_inc = true when its results stand;
// *done_inc = false means the attempt was void (structural object change, bucket / arena overflow) and a full pass must follow.
int run_pass_inc(kr_engine *e, const kr_flags &f, cudaEvent_t done, bool profile, bool *done_inc) {
  *done_inc = false;
  const kr_sizes &n = e->sizes;
  // An object commit created or renumbered RayClusters (rec.map, uploaded to mp; none: no list of it holds a row): its RayCluster and
  // group rows must be the committed ones, the bucket arena must hold the RayClusters at this stride, a wide one needs
  // KR_OPT_WIDE_CLUSTERS, and the orphan scan's shared-memory table holds kAdoptMax new RayClusters.  A RayCluster count that
  // kr_snapshot_begin moved without an object commit behind it takes the full pass.
  static const CommitRecord::RowMap no_map;
  const CommitRecord::RowMap &m = e->map_pending ? e->rec.map : no_map;
  const uint32_t n_gone = (uint32_t)m.gone.size(), n_init = (uint32_t)m.init.size();
  const bool adopt = !m.created.empty() && e->h_totals[1] != 0;  // (the last pass counted orphans: some of them may be the new RayClusters' Pods)
  if (e->map_pending ? e->rec.res_clusters != n.n_clusters || e->rec.res_groups != n.n_groups || e->map_sizes.n_clusters != n.n_clusters ||
                           e->map_sizes.n_groups != n.n_groups || (size_t)n.n_clusters * e->bstride > e->sl.bucket_entries ||
                           (e->rec.snap_max_groups > KR_SMEM_GROUPS && !e->wide_on) || (adopt && n_init > kAdoptMax)
                     : n.n_clusters != e->inc_n_clusters) {
    e->why_full |= e->map_pending ? KR_FULL_ROW_MAP : KR_FULL_SIZES;
    return KR_OK;
  }
  const bool grow = grows(e) && e->bstride;  // (KR_OPT_LARGE_GROWTH: a RayCluster that outgrows its room gets a region in this pass)
  const bool huge_grow = grow && huge_grows(e);  // (KR_OPT_HUGE_GROWTH: ... past KR_LARGE_MAX_PODS Pods too, with tiles)
  const uint32_t n_large_gone = (uint32_t)m.large.size() / 4;  // (KR_OPT_LARGE_MOVES: gone rows with a region)
  PassCtx c(e, profile, grow || n_large_gone);
  const SnapDev &s = c.s; const ResDev &r = c.r; const ScratchDev &sc = c.sc; const Sizes &z = c.z;
  const cudaStream_t M = c.M, H = c.H;
  CK(cudaStreamWaitEvent(M, e->ev_cols, 0));
  const bool do_hash = e->rec.hash_dirty && !f.skip_hash && n.n_clusters > 0;
  auto map_dev = [&](MapList i) { return reinterpret_cast<const uint32_t *>(e->mp.d + e->mp_at[i]); };
  if (!do_hash && !m.digests.empty()) {  // (ahead of the hash stream's fork: a re-hashed row's digest lands after it)
    const uint32_t nd = (uint32_t)m.digests.size() / 2;
    c.mark("k_inc_digest_move");
    k_inc_digest_move<<<(2 * nd + 255) / 256, 256, 0, M>>>(map_dev(MP_DIGESTS), nd, r.hash);
  }
  // ... or only the messages kr_snapshot_commit_spec_rows listed (a whole-arena commit wins; a skip_hash pass leaves them pending)
  const uint32_t n_rows = (!e->rec.hash_dirty && !f.skip_hash) ? (uint32_t)e->spec_pending.size() : 0;
  const uint32_t *spec_rows = n_rows ? upload_spec_order(e) : nullptr;
  if (n_rows && !spec_rows) return fail(e, KR_E_CUDA, "upload of the spec rows' hash order failed");
  if (do_hash && e->rec.spec_order_stale) if (int rc = refresh_order(e)) return rc;
  if (do_hash || n_rows) {  // the spec JSON was committed again: the digests are recomputed (on their own stream), the Recreate gates re-read
    const uint32_t *order = do_hash ? e->d_order : spec_rows;
    const uint32_t nm = do_hash ? n.n_clusters : n_rows;
    if (!profile) { CK(cudaEventRecord(e->ev_fork, M)); CK(cudaStreamWaitEvent(H, e->ev_fork, 0)); }
    CK(cudaStreamWaitEvent(H, e->ev_json, 0));
    if (profile) c.mark(do_hash ? "k_hash" : "k_hash_rows");  // (unprofiled, an incremental pass does not count its hash)
    launch_hash(e, H, s.json, s.c_json_off, s.c_json_len, order, nm, r.hash, e->hash_ctas_per_sm);
    if (!profile) CK(cudaEventRecord(e->ev_hash, H));
    if (e->rec.n_recreate && do_hash) { c.mark("k_inc_mark_recreate"); k_inc_mark_recreate<<<(n.n_clusters + 255) / 256, 256, 0, M>>>(s, sc, z); }
    if (e->rec.n_recreate && !do_hash) { c.mark("k_inc_mark_rows"); k_inc_mark_rows<<<(n_rows + 255) / 256, 256, 0, M>>>(s, sc, spec_rows, n_rows); }
  }
  const int grid = e->sm_count * 2;
  // RayClusters created or renumbered (kr_incr.cuh), each step when its list of the map holds a row
  const uint32_t n_small_gone = n_large_gone ? (uint32_t)m.small_gone.size() : n_gone;
  if (n_small_gone) {  // the gone rows' Pods touched while the table holds the old rows
    c.mark("k_inc_clusters_release");
    k_inc_clusters_release<<<(32 * n_small_gone + 255) / 256, 256, 0, M>>>(s, sc, r, map_dev(n_large_gone ? MP_SGONE : MP_GONE), n_small_gone, e->inc_n_pods);
  }
  if (n_large_gone) {  // ... those with a region a CTA each, their old regions from the map (the table is in the new numbering)
    c.mark("k_inc_large_release");
    k_inc_large_release<<<n_large_gone, 256, 0, M>>>(s, sc, r, reinterpret_cast<const uint4 *>(map_dev(MP_LARGE)), e->inc_n_pods);
  }
  if (e->rec.heads_rebuild) {  // a head Pod came or went since the table was built (the commit compared the keys on the host)
    c.mark("k_inc_aux_rebuild");
    k_inc_aux_clear<<<std::min<uint32_t>(grid, (e->sl.aux_slots + 255) / 256), 256, 0, M>>>(sc);
    k_inc_aux_insert<<<std::min<uint32_t>(grid, (n.n_heads + 255) / 256 + 1), 256, 0, M>>>(s, sc, z);
  }
  if (e->rec.wtd_rebuild) {  // a workersToDelete list changed since the name table was built (KR_OPT_WTD_EDITS; the commit compared them on the host)
    if (e->res_n_wtd) { c.mark("k_inc_wtd_release"); k_inc_wtd_release<<<(e->res_n_wtd + 255) / 256, 256, 0, M>>>(s, sc, r, e->res_n_wtd, e->inc_n_pods); }
    c.mark("k_inc_wtd_clear");
    k_inc_wtd_clear<<<std::min<uint32_t>(grid, (e->sl.wt_slots + 255) / 256), 256, 0, M>>>(sc, r, n.n_wtd);
    if (n.n_wtd) {
      c.mark("k_inc_wtd_insert");
      k_inc_wtd_insert<<<std::min<uint32_t>(grid, (n.n_groups + 255) / 256 + 1), 256, 0, M>>>(s, sc, z);
      c.mark("k_inc_wtd_resolve");
      k_inc_wtd_resolve<<<std::min<uint32_t>((uint32_t)e->sm_count * 4, (n.n_pods + 255) / 256 + 1), 256, e->sl.wt_bits_n / 8, M>>>(s, sc, r, z, e->inc_n_pods, 0u);
    }
    e->res_n_wtd = n.n_wtd;
    e->rec.wtd_rebuild = false;
  }
  if (adopt) {  // the created RayClusters' orphans touched while the table does not hold them
    uint32_t bloom_bits = 1024, slots = 64;
    while (bloom_bits < 16 * n_init) bloom_bits <<= 1;
    while (slots < 2 * n_init) slots <<= 1;
    c.mark("k_inc_orphan_adopt");
    k_inc_orphan_adopt<<<std::min<uint32_t>((uint32_t)e->sm_count * 4, (e->inc_n_pods + 255) / 256 + 1), 256, bloom_bits / 8 + 4 * (size_t)slots, M>>>(
        s, sc, r, map_dev(MP_INIT), n_init, bloom_bits - 1, slots - 1, e->inc_n_pods);
  }
  if (n_gone) {  // ... then the resident state in the new numbering
    c.mark("k_inc_clusters_translate");
    k_inc_clusters_translate<<<1, 1024, 0, M>>>(sc, map_dev(MP_GONE), n_gone, n.n_clusters);
    c.mark("k_inc_clusters_rekey");
    CK(cudaMemsetAsync(sc.cl_slots, 0xFF, 16 * (size_t)e->sl.cl_slots, M));
    k_inc_clusters_rekey<<<std::min<uint32_t>(grid, (n.n_clusters + 255) / 256 + 1), 256, 0, M>>>(s, sc, n.n_clusters);
    if (m.gs0 < n.n_groups && m.g_hi > m.g_lo) {  // the old group records and create offsets the gather reads, staged first
      const size_t ng = m.g_hi - m.g_lo;
      kr_group_result *og = reinterpret_cast<kr_group_result *>(e->inc_stage.d);
      uint32_t *oc = reinterpret_cast<uint32_t *>(e->inc_stage.d + sizeof(kr_group_result) * ng);
      CK(cudaMemcpyAsync(og, r.groups + m.g_lo, sizeof(kr_group_result) * ng, cudaMemcpyDeviceToDevice, M));
      CK(cudaMemcpyAsync(oc, sc.gcreate + m.g_lo, 4 * ng, cudaMemcpyDeviceToDevice, M));
      c.mark("k_inc_groups_gather");
      k_inc_groups_gather<<<std::min<uint32_t>(grid, (n.n_groups - m.gs0 + 255) / 256 + 1), 256, 0, M>>>(r, sc, map_dev(MP_GSRC), m.gs0, n.n_groups - m.gs0, og, oc, m.g_lo);
    }
  }
  if (n_init) {  // ... and the moved and created RayClusters enter the table as new ones
    // their workersToDelete names after the resident ones: inserted here and resolved against every pod row (a map that moved a
    // resident name had the whole table rebuilt above, the new names with it)
    const bool names = n.n_wtd > e->res_n_wtd;
    c.mark("k_inc_clusters_insert");
    k_inc_clusters_insert<<<(n_init + 255) / 256, 256, 0, M>>>(s, sc, r, map_dev(MP_INIT), n_init, names ? 1 : 0);
    if (n_large_gone) {  // (the insert cleared their entries)
      c.mark("k_inc_large_carry");
      k_inc_large_carry<<<(n_large_gone + 255) / 256, 256, 0, M>>>(sc, reinterpret_cast<const uint4 *>(map_dev(MP_LARGE)), n_large_gone);
    }
    if (names) {
      c.mark("k_inc_wtd_resolve");
      k_inc_wtd_resolve<<<std::min<uint32_t>((uint32_t)e->sm_count * 4, (n.n_pods + 255) / 256 + 1), 256, e->sl.wt_bits_n / 8, M>>>(s, sc, r, z, e->inc_n_pods, e->res_n_wtd);
      e->res_n_wtd = n.n_wtd;  // (a void attempt is followed by the full pass, which sets it again)
    }
  }
  // (k_inc_refresh ran behind the object commits' diff kernels: the input records are current)
  c.mark("k_inc_admit");
  k_inc_admit<<<grid, 256, 0, M>>>(s, sc, r, z, n.n_wtd ? 1 : 0, grow ? e->d_grow : nullptr);
  if (grow) {  // regions for the RayClusters that outgrew their room (most launches find the grow list empty and leave at once)
    c.mark("k_inc_grow");
    const uint32_t list_cap = std::max<uint32_t>(KR_GROW_LIST_MIN, n.n_clusters / KR_GROW_LIST_DIV);
    if (huge_grow)
      k_inc_grow<true><<<e->sm_count, 256, 0, M>>>(s, sc, e->d_grow, (uint32_t)e->lg_cursor, (uint32_t)e->large_entries, e->n_large, list_cap,
                                                    e->wide_on ? 1 : 0, const_cast<uint4 *>(c.hd.tiles), e->n_tiles, (uint32_t)e->huge_tiles);
    else
      k_inc_grow<false><<<e->sm_count, 256, 0, M>>>(s, sc, e->d_grow, (uint32_t)e->lg_cursor, (uint32_t)e->large_entries, e->n_large, list_cap,
                                                     e->wide_on ? 1 : 0, nullptr, 0u, 0u);
  }
  if ((do_hash || n_rows) && !profile) CK(cudaStreamWaitEvent(M, e->ev_hash, 0));
  const IncStageLayout sl = e->inc_layout = inc_stage_layout(n.n_clusters, n.n_groups);  // staging for the changed records
  if (sl.total > e->inc_stage.cap) return fail(e, KR_E_STATE, "internal: incremental staging of %zu bytes, room for %zu", sl.total, e->inc_stage.cap);
  const IncStage st{reinterpret_cast<uint32_t *>(e->inc_stage.d), reinterpret_cast<kr_cluster_result *>(e->inc_stage.d + sl.clusters),
                    reinterpret_cast<kr_group_result *>(e->inc_stage.d + sl.groups), sl.capc, sl.capg};
  const bool gather_rows = n_rows && n_rows <= sl.capc;  // (more re-hashed digests than that: the fetch copies them all)
  if (gather_rows) {
    c.mark("k_inc_digest_gather");
    k_inc_digest_gather<<<(2 * n_rows + 255) / 256, 256, 0, M>>>(spec_rows, n_rows, r.hash, reinterpret_cast<char *>(e->inc_stage.d + sl.digests));
  }
  if (n.n_clusters) {
    Decide2Args da{s, sc, r, z, f, st, e->cfg.max_creates, 0, 2};
    c.mark("k_decide2_dirty");
    // (the multi-host rows as of the latest commit: an object commit may have brought the snapshot's first multi-host group or taken its last)
    CK(launch_decide2(c, da, dim3((n.n_clusters + kD2Warps - 1) / kD2Warps), true, false));
    if (e->n_large || grow) {  // the dirty large RayClusters (k_decide2 left every cluster past the stride alone), and those k_inc_grow listed
      const uint4 *grown = grow ? e->d_grow + kGrowResult : nullptr;
      CK(cudaMemsetAsync(sc.inc + KR_INC_LSEG, 0, 4, M));
      launch_large_sort<true>(c, da, grown, huge_grow ? (uint32_t)e->huge_reserve : 0u);
      launch_large_decide<true>(c, da, grown);
    }
  }
  if (n.n_jobs) { c.mark("k_jobs"); k_jobs<<<(n.n_jobs + 255) / 256, 256, 0, M>>>(s, sc, r, z); }
  if (f.fetch_pod_lists) launch_lists(c, true);  // (only with KR_OPT_BUCKET_POD_LISTS: the flags of the resident pass leave it out)
  c.close();
  if (done) CK(cudaEventRecord(done, M));
  CK(cudaMemcpyAsync(e->h_totals, e->d_out + e->ol.totals, 48, cudaMemcpyDeviceToHost, M));
  CK(cudaMemcpyAsync(e->h_inc, sc.inc, 64, cudaMemcpyDeviceToHost, M));
  if (grow) CK(cudaMemcpyAsync(e->h_grow, e->d_grow + kGrowResult, 16 * KR_GROW_MAX, cudaMemcpyDeviceToHost, M));
  CK(cudaEventRecord(e->ev_inc, M));
  k_inc_finish<<<1, 32, 0, M>>>(sc);  // (the host does not wait for it: whatever comes next is ordered behind it on this stream)
  CK(cudaGetLastError());
  CK(cudaEventSynchronize(e->ev_inc));
  e->dev_epoch = e->h_inc[KR_INC_EPOCH] + 1u;  // (k_inc_finish closes the epoch, void or not)
  commits_read(e);
  e->rec.heads_rebuild = false;  // (rebuilt here, or about to be rebuilt by the full pass)
  if (e->h_inc[KR_INC_VOID] || e->h_inc[KR_INC_STRUCTURAL]) {  // the caller takes the full pass
    // (the device's KR_FULL_* bits; k_inc_admit reports every record without room as an overflow, which growth refused when it could grow)
    const uint32_t why = e->h_inc[KR_INC_VOID] | e->h_inc[KR_INC_STRUCTURAL];
    e->why_full |= grow && (why & KR_FULL_OVERFLOW) ? (why & ~KR_FULL_OVERFLOW) | KR_FULL_GROW_LIMIT : why;
    if (grow) e->lg_stale = true;  // (k_inc_grow may have written regions of this attempt into the device table: the full pass reads the host's)
    return KR_OK;
  }
  // the regions k_inc_grow gave, into the large half (rows ascending: commit_map and upload_lg search it); the next pass's upload
  // lists the newly listed RayClusters
  for (uint32_t i = 0; grow && i < e->h_inc[KR_INC_GROWN]; i++) {
    const uint4 g = e->h_grow[i];
    const size_t at = std::lower_bound(e->large_rows.begin(), e->large_rows.end(), g.x) - e->large_rows.begin();
    if (at == e->large_rows.size() || e->large_rows[at] != g.x) { e->large_rows.insert(e->large_rows.begin() + at, g.x); e->large_reg.insert(e->large_reg.begin() + at, make_uint2(g.y, g.z)); }
    else e->large_reg[at] = make_uint2(g.y, g.z);
    e->lg_cursor = std::max<size_t>(e->lg_cursor, (size_t)g.y + g.z);
    e->lg_stale = true;
  }
  if (!e->fetched) e->host_results_stale = true;  // the previous pass's records never reached the host copy
  e->fetched = false;
  e->inc_n_dirty = e->h_inc[KR_INC_DIRTY];
  e->inc_gathered = e->inc_n_dirty <= sl.capc && e->h_inc[KR_INC_GROUPS] <= sl.capg;
  e->inc_hash_ran = do_hash;
  if (do_hash) e->rec.hash_dirty = false;
  e->inc_spec_n = n_rows; e->inc_spec_gathered = gather_rows;
  if (n_rows) {
    const uint32_t *h = reinterpret_cast<const uint32_t *>(e->spec.h + 16 * ((size_t)e->cfg.max_clusters + 1));
    e->spec_hashed.assign(h, h + n_rows);
  }
  if (do_hash || n_rows) clear_spec_rows(e);
  // the host copy in the new numbering as well: moved digests, shifted group records (re-decided RayClusters come with the fetch)
  ResDev hr = bind_out(e->ol, e->h_out);
  if (!do_hash)
    for (size_t i = 0; i < m.digests.size(); i += 2) memcpy(hr.hash + 32 * (size_t)m.digests[i + 1], hr.hash + 32 * (size_t)m.digests[i], 32);
  if (m.gs0 < n.n_groups && m.g_hi > m.g_lo) {
    const std::vector<kr_group_result> old(hr.groups + m.g_lo, hr.groups + m.g_hi);
    for (uint32_t k = 0; k < n.n_groups - m.gs0; k++)
      if (m.gsrc[k] != KR_EMPTY32) hr.groups[m.gs0 + k] = old[m.gsrc[k] - m.g_lo];
  }
  e->map_pending = false;
  e->ran_inc = true;
  *done_inc = true;
  return KR_OK;
}

// The pass's results stand: kernels_ms is the time from ev_a to `done`.
int pass_done(kr_engine *e, cudaEvent_t done) {
  float ms = 0;
  if (cudaEventElapsedTime(&ms, e->ev_a, done) == cudaSuccess) e->prof.kernels_ms = ms;
  e->ran = true;
  return KR_OK;
}

// Runs the pass: an incremental epoch when the resident state allows one, else the full pass, which runs again on the next pipeline
// of its ladder while it meets a RayCluster its pipeline cannot hold.  Records `done` behind the kernels and leaves the stream
// synchronised (after an incremental pass only its one-thread epoch-closing kernel may still be in flight: it touches the epoch
// counters, nothing a reader of the results sees).  ev_a is recorded once, first; profile: each kernel between events, no graph,
// and ev_a recorded again before each attempt, so that kernels_ms covers the last one.
int run_pass(kr_engine *e, const kr_flags &f, cudaEvent_t done, bool profile) {
  if (!e->committed) return fail(e, KR_E_STATE, "no committed snapshot");
  if (!e->rec.overwritten.empty())  // (a pass would hash bytes a move overwrote)
    return fail(e, KR_E_STATE, "cluster %u: a JSON move overwrote its spec bytes on the device; commit its spec row or the JSON part first", e->rec.overwritten.front());
  CK(cudaSetDevice(e->cfg.device));
  if (!profile) CK(cudaEventRecord(e->ev_a, e->sm));
  e->last_flags = f;
  new_pull_epoch(e);
  // Regions of rows past the live count (a deleted large RayCluster in the last rows, whose row map voided the epoch) go: the full
  // pass that follows would list a row it does not hold.  (Large rows at or past the count are gone rows of the map, and a map with a
  // large gone row is followed incrementally only with KR_OPT_LARGE_MOVES, whose commit renumbered the large half: nothing is left
  // past the count then.)  A deleted large RayCluster's row below the count keeps its region for the RayCluster that took the row
  // when the map was not followed.
  if (int rc = drop_regions(e, std::lower_bound(e->large_rows.begin(), e->large_rows.end(), e->sizes.n_clusters) - e->large_rows.begin())) return rc;
  // (the list moves with a group count, an option or a new layout, when a full pass follows, and with the RayClusters an incremental
  // epoch created)
  if (e->lg_stale) if (int rc = upload_lg(e)) return rc;
  // The running epoch stamps with the counter + 1, and 0 means "not this epoch": before the counter can reach 2^32 - 1 the region is
  // zeroed again and a full pass runs (kEpochMargin).
  const bool wrap = e->dev_epoch > 0xFFFFFFFFu - kEpochMargin;
  if (wrap) { e->why_full |= KR_FULL_EPOCH_WRAP; e->inc_zero_needed = true; e->epoch_seed = 0; }
  kr_flags fk = f;  // (KR_OPT_BUCKET_POD_LISTS: fetching the lists keeps the epoch incremental)
  if (e->bucket_lists) fk.fetch_pod_lists = 0;
  const bool same_flags = memcmp(&e->inc_flags, &fk, sizeof fk) == 0;
  if (e->inc_valid && !e->no_incr && same_flags && !wrap) {
    if (profile) CK(cudaEventRecord(e->ev_a, e->sm));
    bool ok = false;
    if (int rc = run_pass_inc(e, f, done, profile, &ok)) return rc;
    if (ok) {
      e->inc_n_pods = e->sizes.n_pods; e->inc_n_heads = e->sizes.n_heads; e->inc_n_clusters = e->sizes.n_clusters;
      make_report(e, true, 0, false, 0);
      return pass_done(e, done);
    }
    if (e->lg_stale) if (int rc = upload_lg(e)) return rc;  // (a void attempt that grew regions left them in the device table)
  } else if (e->inc_valid && !e->no_incr && !same_flags) e->why_full |= KR_FULL_FLAGS;
  e->inc_valid = false; e->ran_inc = false;
  if (e->inc_zero_needed) {  // first pass on this layout, or the counter's wrap: stamps, dirty flags and epoch counters start from zero
    CK(cudaMemsetAsync(e->d_scratch + e->sl.inc_zero, 0, e->sl.inc_zero_end - e->sl.inc_zero, e->sm));
    if (e->epoch_seed) CK(cudaMemcpyAsync(e->d_scratch + e->sl.inc + 4 * KR_INC_EPOCH, &e->epoch_seed, 4, cudaMemcpyHostToDevice, e->sm));
    e->dev_epoch = e->epoch_seed;
    e->epoch_seed = 0;
    e->inc_zero_needed = false;
  }
  if (e->rec.spec_order_stale && !f.skip_hash) if (int rc = refresh_order(e)) return rc;
  uint32_t voided = 0;
  bool hash_wait = false;
  for (int attempt = 0; attempt < kFullAttempts; attempt++) {
    if (profile) CK(cudaEventRecord(e->ev_a, e->sm));
    if (int rc = profile ? launch_pass(e, f, true) : run_pass_once(e, f)) return rc;
    if (e->sizes.n_clusters + e->sizes.n_groups + e->sizes.n_heads) e->dev_epoch++;  // (k_build_tables closed an epoch)
    if (done) CK(cudaEventRecord(done, e->sm));
    CK(cudaMemcpyAsync(e->h_totals, e->d_out + e->ol.totals, 48, cudaMemcpyDeviceToHost, e->sm));
    CK(cudaStreamSynchronize(e->sm));
    // A profiled full pass frees the pinned hash order but leaves the commits' h2d_accum and h2d_ms alone: h2d_bytes then keeps
    // adding up until an unprofiled pass or an incremental one reads the commits.
    if (!profile) commits_read(e);
    else e->order_pending = false;
    if (e->h_totals[3] & KR_TOTALS_HASH_WAIT) {  // a decide warp gave up waiting for its digest (a profiled pass never waits): rerun on the two-phase schedule
      e->hash_spin = false; e->gvalid = false;
      hash_wait = true;
      continue;
    }
    if (!(e->h_totals[3] & KR_TOTALS_BIG_BUCKET)) {
      after_full_pass(e, f);
      make_report(e, false, voided, hash_wait, why_not_resident(e, f));
      return pass_done(e, done);
    }
    voided++;
    // some RayCluster outgrew what this pipeline holds per bucket: bucket pipeline -> wider stride -> sort pipeline -> radix pipeline
    if (e->ran_bucket) {
      if (int rc = after_bucket_void(e)) return rc;
    } else if (e->ran_fast) e->force_radix = true;
    else break;
    e->gvalid = false;
  }
  return fail(e, KR_E_STATE, "internal: radix pipeline flagged a big bucket");
}

// Results back to the pinned host arena.  run_pass already brought the totals words over, so every copy is issued with its
// exact size up front and the host waits once: [small fixed part] (+ the full pod lists when asked for) + the compact action
// list + the replica-index arena.
int fetch_results(kr_engine *e, kr_results_view *out) {
  const kr_sizes &n = e->sizes;
  const uint32_t *tot = e->h_totals;
  // bucket pipeline: the two arenas can hold reserved-but-unused places (totals[9] / totals[8] are their extents, [6] / [2] the counts)
  const uint32_t n_create = e->ran_bucket ? tot[9] : tot[0], n_actions = e->ran_bucket ? tot[8] : tot[2];
  const bool full = e->last_flags.fetch_pod_lists != 0;
  const bool starts = full && e->ran_bucket;  // (KR_OPT_BUCKET_POD_LISTS: the lists' starts travel apart from the cluster records)
  CK(cudaEventRecord(e->ev_b, e->sm));
  if (n_create > e->cfg.max_creates) {
    CK(cudaEventRecord(e->ev_c, e->sm));
    return fail(e, KR_E_CAPACITY, "pods to create (%u) exceed kr_config.max_creates (%u)", n_create, e->cfg.max_creates);
  }
  const bool inc = e->ran_inc && !e->host_results_stale;
  const bool packed = inc && e->inc_gathered;
  uint64_t bytes = 0;
  const uint32_t nd = e->inc_n_dirty, ngr = inc ? e->h_inc[KR_INC_GROUPS] : 0;
  const size_t st_cl = e->inc_layout.clusters, st_gr = e->inc_layout.groups, st_dig = e->inc_layout.digests;
  const bool spec_packed = packed && e->inc_spec_n && e->inc_spec_gathered && !e->inc_hash_ran;
  if (packed) {
    // incremental pass: the changed cluster / group records come back packed (k_inc_gather) and are scattered into the host
    // arena below; the flat arrays an epoch can touch anywhere (name resolutions, RayJob rows, digests when they were
    // recomputed) are small and come back whole
    if (nd) {
      CK(cudaMemcpyAsync(e->inc_stage.h, e->inc_stage.d, 32 * (size_t)nd, cudaMemcpyDeviceToHost, e->sm));
      CK(cudaMemcpyAsync(e->inc_stage.h + st_cl, e->inc_stage.d + st_cl, sizeof(kr_cluster_result) * (size_t)nd, cudaMemcpyDeviceToHost, e->sm));
      if (ngr) CK(cudaMemcpyAsync(e->inc_stage.h + st_gr, e->inc_stage.d + st_gr, sizeof(kr_group_result) * (size_t)ngr, cudaMemcpyDeviceToHost, e->sm));
      bytes += (32 + sizeof(kr_cluster_result)) * (uint64_t)nd + sizeof(kr_group_result) * (uint64_t)ngr;
    }
    CK(cudaMemcpyAsync(e->h_out + e->ol.totals, e->d_out + e->ol.totals, 256, cudaMemcpyDeviceToHost, e->sm));
    if (n.n_wtd) { CK(cudaMemcpyAsync(e->h_out + e->ol.wtd, e->d_out + e->ol.wtd, 4 * (size_t)n.n_wtd, cudaMemcpyDeviceToHost, e->sm)); bytes += 4ull * n.n_wtd; }
    if (n.n_jobs) { CK(cudaMemcpyAsync(e->h_out + e->ol.jobs, e->d_out + e->ol.jobs, sizeof(kr_job_result) * (size_t)n.n_jobs, cudaMemcpyDeviceToHost, e->sm)); bytes += sizeof(kr_job_result) * (uint64_t)n.n_jobs; }
    if ((e->inc_hash_ran || (e->inc_spec_n && !e->inc_spec_gathered)) && n.n_clusters) { CK(cudaMemcpyAsync(e->h_out + e->ol.hash, e->d_out + e->ol.hash, 32 * (size_t)n.n_clusters, cudaMemcpyDeviceToHost, e->sm)); bytes += 32ull * n.n_clusters; }
    else if (e->inc_spec_n) {  // the digests of the spec rows, packed by k_inc_digest_gather
      CK(cudaMemcpyAsync(e->inc_stage.h + st_dig, e->inc_stage.d + st_dig, 32 * (size_t)e->inc_spec_n, cudaMemcpyDeviceToHost, e->sm));
      bytes += 32ull * e->inc_spec_n;
    }
  } else {
    bytes = e->ol.small_total;
    CK(cudaMemcpyAsync(e->h_out, e->d_out, e->ol.small_total, cudaMemcpyDeviceToHost, e->sm));
  }
  if (inc && nd) {  // the changed-cluster list itself
    if ((size_t)nd > e->h_changed_cap) return fail(e, KR_E_STATE, "internal: %u changed RayClusters, room for %zu", nd, e->h_changed_cap);
    CK(cudaMemcpyAsync(e->h_changed, e->d_scratch + e->sl.dirty_list, 4 * (size_t)nd, cudaMemcpyDeviceToHost, e->sm));
    bytes += 4ull * nd;
  }
  if (full && n.n_pods) {
    if (!e->fixed_layout) {
      size_t span = e->ol.act_idx - e->ol.sorted_idx;  // sorted_pod_idx + sorted_action, contiguous
      CK(cudaMemcpyAsync(e->h_out + e->ol.sorted_idx, e->d_out + e->ol.sorted_idx, span, cudaMemcpyDeviceToHost, e->sm));
      bytes += span;
    } else {  // capacity slack between the two arrays: copy the live prefixes
      CK(cudaMemcpyAsync(e->h_out + e->ol.sorted_idx, e->d_out + e->ol.sorted_idx, 4 * (size_t)n.n_pods, cudaMemcpyDeviceToHost, e->sm));
      CK(cudaMemcpyAsync(e->h_out + e->ol.sorted_act, e->d_out + e->ol.sorted_act, (size_t)n.n_pods, cudaMemcpyDeviceToHost, e->sm));
      bytes += 5 * (size_t)n.n_pods;
    }
  }
  if (starts && n.n_clusters) {
    CK(cudaMemcpyAsync(e->h_out + e->ol.pod_start, e->d_out + e->ol.pod_start, 4 * (size_t)n.n_clusters, cudaMemcpyDeviceToHost, e->sm));
    bytes += 4ull * n.n_clusters;
  }
  if (n_actions) {
    CK(cudaMemcpyAsync(e->h_out + e->ol.act_idx, e->d_out + e->ol.act_idx, 4 * (size_t)n_actions, cudaMemcpyDeviceToHost, e->sm));
    CK(cudaMemcpyAsync(e->h_out + e->ol.act_code, e->d_out + e->ol.act_code, (size_t)n_actions, cudaMemcpyDeviceToHost, e->sm));
    bytes += 5ull * n_actions;
  }
  if (n_create) {
    CK(cudaMemcpyAsync(e->h_out + e->ol.create, e->d_out + e->ol.create, 4 * (size_t)n_create, cudaMemcpyDeviceToHost, e->sm));
    bytes += 4ull * n_create;
  }
  CK(cudaEventRecord(e->ev_c, e->sm));
  CK(cudaStreamSynchronize(e->sm));
  if (packed && nd) {  // scatter the packed records into the host arena
    ResDev hr = bind_out(e->ol, e->h_out);
    const uint32_t *meta = reinterpret_cast<const uint32_t *>(e->inc_stage.h);
    const kr_cluster_result *scl = reinterpret_cast<const kr_cluster_result *>(e->inc_stage.h + st_cl);
    const kr_group_result *sgr = reinterpret_cast<const kr_group_result *>(e->inc_stage.h + st_gr);
    for (uint32_t i = 0; i < nd; i++) {
      const uint32_t *m = meta + 8 * (size_t)i;
      const uint32_t c = m[0];
      hr.clusters[c] = scl[i]; hr.act_start[c] = m[1]; hr.act_cnt[c] = m[2];
      if (m[4]) memcpy(&hr.groups[m[3]], &sgr[m[5]], sizeof(kr_group_result) * (size_t)m[4]);
    }
  }
  if (spec_packed) {  // ... and the re-hashed digests
    char *hh = reinterpret_cast<char *>(e->h_out + e->ol.hash);
    for (uint32_t i = 0; i < e->inc_spec_n; i++) memcpy(hh + 32 * (size_t)e->spec_hashed[i], e->inc_stage.h + st_dig + 32 * (size_t)i, 32);
  }
  // The list starts into the host's cluster records, and out again on a fetch without the lists: the records a packed incremental
  // fetch leaves alone still hold the starts of an earlier one (on the device they are 0, as the bucket pipeline leaves them).
  if (starts || (packed && e->host_starts)) {
    kr_cluster_result *hc = bind_out(e->ol, e->h_out).clusters;
    const uint32_t *st = reinterpret_cast<const uint32_t *>(e->h_out + e->ol.pod_start);
    for (uint32_t c = 0; c < n.n_clusters; c++) hc[c].pod_start = starts ? st[c] : 0u;
  }
  e->host_starts = starts;
  e->fetched = true; e->host_results_stale = false;
  if (out) {
    ResDev hr = bind_out(e->ol, e->h_out);
    out->clusters = hr.clusters; out->hash = hr.hash; out->groups = hr.groups;
    out->wtd_pod_idx = reinterpret_cast<const int32_t *>(hr.wtd_pod_idx);
    out->sorted_pod_idx = full ? hr.sorted_pod_idx : nullptr; out->sorted_action = full ? hr.sorted_action : nullptr;
    out->create_idx = hr.create_idx; out->jobs = hr.jobs;
    out->act_start = hr.act_start; out->act_cnt = hr.act_cnt; out->act_pod_idx = hr.act_pod_idx; out->act_code = hr.act_code;
    out->n_create_total = e->ran_bucket ? tot[6] : n_create; out->n_orphans = tot[1]; out->n_actions = tot[2];
    out->create_extent = n_create; out->act_extent = n_actions;
    out->n_changed = inc ? nd : n.n_clusters;
    out->changed_clusters = (inc && nd) ? e->h_changed : nullptr;
  }
  float ms = 0;
  if (cudaEventElapsedTime(&ms, e->ev_b, e->ev_c) == cudaSuccess) e->prof.d2h_ms = ms;
  e->prof.d2h_bytes = bytes;
  return KR_OK;
}

// The checks every commit makes of the rows it takes, before anything moves (an invalid call commits nothing).  The kernels trust
// these indices: a shim bug must come back as KR_E_INVALID, not as out-of-bounds device reads and writes.  (Inlined: the whole
// commit runs them on every row.)
// A RayCluster row: its JSON range 16-byte aligned and inside json_bytes; unless json_only, fewer worker groups than the limit, its
// groups inside n_groups and naming it in g_cluster_idx, and their workersToDelete names inside n_wtd.
__attribute__((always_inline)) inline int check_cluster_row(kr_engine *e, const kr_snapshot_bufs &hb, const kr_sizes &n, uint32_t c, bool json_only = false) {
  if (c >= n.n_clusters) return fail(e, KR_E_INVALID, "cluster row %u out of range", c);
  if (hb.c_json_off[c] & 15) return fail(e, KR_E_INVALID, "cluster %u: json offset not 16-byte aligned", c);
  if (hb.c_json_off[c] + hb.c_json_len[c] > n.json_bytes) return fail(e, KR_E_INVALID, "cluster %u: json range outside arena", c);
  if (json_only) return KR_OK;
  const uint64_t g0 = hb.c_group_off[c], cnt = hb.c_group_cnt[c];
  if (cnt >= 0xFFFFu) return fail(e, KR_E_CAPACITY, "cluster %u has %u worker groups (limit 65534)", c, hb.c_group_cnt[c]);
  if (g0 + cnt > n.n_groups) return fail(e, KR_E_INVALID, "cluster %u: groups run past n_groups", c);
  for (uint64_t g = g0; g < g0 + cnt; g++) {
    if (hb.g_cluster_idx[g] != c) return fail(e, KR_E_INVALID, "group %llu: g_cluster_idx %u != owning cluster %u", (unsigned long long)g, hb.g_cluster_idx[g], c);
    if ((uint64_t)hb.g_wtd_off[g] + hb.g_wtd_cnt[g] > n.n_wtd) return fail(e, KR_E_INVALID, "group %llu: workersToDelete names run past n_wtd", (unsigned long long)g);
  }
  return KR_OK;
}
__attribute__((always_inline)) inline int check_head_row(kr_engine *e, const kr_snapshot_bufs &hb, const kr_sizes &n, uint32_t h) {
  if (h >= n.n_heads) return fail(e, KR_E_INVALID, "head-aux row %u out of range", h);
  if (hb.h_pod_idx[h] >= n.n_pods) return fail(e, KR_E_INVALID, "head-aux row %u: h_pod_idx %u >= n_pods %u", h, hb.h_pod_idx[h], n.n_pods);
  return KR_OK;
}

// The start of every commit: a pass still reading what it overwrites must finish first; ev_h2d0 opens its copy time.
int begin_commit(kr_engine *e) {
  CK(cudaStreamSynchronize(e->sm));
  CK(cudaEventRecord(e->ev_h2d0, e->scopy));
  return KR_OK;
}

// KR_OPT_CLUSTER_CREATES has an effect (the tables are sized for the capacities)
bool creates_on(const kr_engine *e) { return e->cluster_creates && e->fixed_layout; }
// KR_OPT_CLUSTER_DELETES has an effect
bool deletes_on(const kr_engine *e) { return e->cluster_deletes && e->fixed_layout; }
// KR_OPT_GROUP_EDITS has an effect
bool regroups_on(const kr_engine *e) { return e->group_edits && e->fixed_layout; }

// KR_OPT_LARGE_MOVES has an effect
bool large_moves_on(const kr_engine *e) { return e->large_moves && e->large_on && e->fixed_layout && e->d_lg && e->d_region; }

// KR_OPT_LARGE_MOVES: a row map the pass follows takes the large half into the new numbering (rows ascending: upload_lg, drop_regions
// and commit_map search it).  A deleted RayCluster's region is abandoned until the next full pass that reclassifies; a moved or
// regrouped one's goes with it to its new row.  The map lists the gone rows with a region apart (RowMap::large), since the release
// reads their old regions after the pass's upload wrote the table in the new numbering, which leaves zero in the rows a deleted one
// vacated.  Rows left past the count are cleared here, on stream M ahead of the pass: nothing uploads them.
int renumber_large(kr_engine *e, CommitRecord::RowMap &m) {
  m.small_gone.clear(); m.large.clear();
  std::vector<std::pair<uint32_t, uint2>> half;
  for (size_t i = 0; i < e->large_rows.size(); i++) {
    const uint32_t o = e->large_rows[i];
    const uint2 reg = e->large_reg[i];
    const auto it = std::lower_bound(m.gone.begin(), m.gone.end(), o);
    if (it == m.gone.end() || *it != o) { half.push_back({o, reg}); continue; }
    const uint32_t to = m.moved_to[it - m.gone.begin()];
    m.large.insert(m.large.end(), {o, reg.x, reg.y, to});
    if (to != KR_EMPTY32) half.push_back({to, reg});
    if (o >= e->sizes.n_clusters) CK(cudaMemsetAsync(e->d_lg + 16 * (size_t)o, 0, 16, e->sm));
  }
  if (m.large.empty()) return KR_OK;
  for (uint32_t o : m.gone) if (!std::binary_search(e->large_rows.begin(), e->large_rows.end(), o)) m.small_gone.push_back(o);
  std::sort(half.begin(), half.end(), [](const std::pair<uint32_t, uint2> &a, const std::pair<uint32_t, uint2> &b) { return a.first < b.first; });
  e->large_rows.clear(); e->large_reg.clear();
  for (const auto &h : half) { e->large_rows.push_back(h.first); e->large_reg.push_back(h.second); }
  e->lg_stale = true; e->lg_moved = true;
  return KR_OK;
}

// The column table of an object commit's diff: every object column i, staged at stage + at[i] with cnt[d] rows of its dimension d,
// against the resident one as the record last left it.  Without row lists, staged row k is resident row k; with them (the row path)
// it is the k-th row of the list of dimension d at stage + list_at[d], and a dimension without staged rows is left out.
ObjDiffArgs object_diff_args(const kr_engine *e, const uint8_t *stage, const size_t *at, const uint32_t cnt[7], const size_t *list_at) {
  uint64_t dn[7];
  dims_of(e->sizes, dn);
  ObjDiffArgs oa{};
  for (int i = 0; i < kNumCols - 1; i++) {
    const int d = kCols[i].dim;
    if (d == D_PODS || (list_at && !cnt[d])) continue;
    const int k = oa.n_cols++;
    oa.src[k] = stage + at[i];
    oa.rowlist[k] = list_at ? reinterpret_cast<const uint32_t *>(stage + list_at[d]) : nullptr;
    oa.dst[k] = e->d_in + e->il.off[i];
    oa.first[k + 1] = oa.first[k] + cnt[d];
    oa.rows_old[k] = d == D_HEADS ? e->rec.res_n_heads : d == D_CLUSTERS ? e->rec.res_clusters : d == D_GROUPS ? e->rec.res_groups : d == D_WTD ? e->rec.res_wtd : (uint32_t)dn[d];
    oa.row_bytes[k] = (uint16_t)(kCols[i].elem * kCols[i].mult);
    oa.cls[k] = obj_class(i, e->wtd_edits);
    oa.cls_new[k] = obj_class(i, e->wtd_edits, creates_on(e) || deletes_on(e) || regroups_on(e));
    if (i == kGroupClusterCol) oa.g_cluster_idx_new = reinterpret_cast<const uint32_t *>(stage + at[i]);
    if (i == kHeadKeyCol) oa.h_pod_idx_new = reinterpret_cast<const uint32_t *>(stage + at[i]);
  }
  oa.h_pod_idx_old = reinterpret_cast<const uint32_t *>(e->d_in + e->il.off[kHeadKeyCol]);
  oa.n_heads_old = e->rec.res_n_heads;
  return oa;
}

// An object commit whose part created or renumbered RayClusters, or moved a row count after a renumbering of the same epoch (on the
// copy stream, before its diff): a row map the resident state follows (`ok`, rec.map) is checked against what the pass can move,
// queues the created RayClusters' specs and renumbers the pending spec rows, travels to the device and, when rows were renumbered,
// sets up the diff (oa).  Otherwise `voided`: the resident state does not follow this epoch, and the caller drops it once the diff
// has copied the object part into place (the next pass is a full one, which re-hashes every spec).
int commit_map(kr_engine *e, bool ok, ObjDiffArgs &oa, bool &voided) {
  CommitRecord::RowMap &m = e->rec.map;
  const kr_sizes &n = e->sizes;
  // (a large RayCluster's region and tiles move with it only with KR_OPT_LARGE_MOVES; the old groups the gather reads are staged in
  // the incremental staging buffer, which the pass fills only later)
  ok = ok && 36 * (size_t)(m.g_hi - m.g_lo) <= e->inc_stage.cap;
  if (!large_moves_on(e)) for (uint32_t o : m.gone) ok = ok && !std::binary_search(e->large_rows.begin(), e->large_rows.end(), o);
  if (!ok) {  // (the record took the new rows' ranges as the digests' ones)
    e->rec.hash_dirty = true;
    e->map_pending = false;
    voided = true;
    return KR_OK;
  }
  if (int rc = renumber_large(e, m)) return rc;
  // the digests the next pass computes: the created RayClusters', and the pending spec rows in the new numbering
  std::vector<uint32_t> pending;
  for (uint32_t r : e->spec_pending) {
    const auto it = std::lower_bound(m.gone.begin(), m.gone.end(), r);
    if (it == m.gone.end() || *it != r) pending.push_back(r);
    else if (m.moved_to[it - m.gone.begin()] != KR_EMPTY32) pending.push_back(m.moved_to[it - m.gone.begin()]);
  }
  pending.insert(pending.end(), m.created.begin(), m.created.end());
  clear_spec_rows(e);
  if (e->spec_stamp.size() < n.n_clusters) e->spec_stamp.resize(n.n_clusters, 0u);
  for (uint32_t c : pending)
    if (e->spec_stamp[c] != e->spec_epoch) { e->spec_stamp[c] = e->spec_epoch; e->spec_pending.push_back(c); }
  const std::vector<uint32_t> *lists[MP_LISTS] = {&m.gone, &m.init, &m.digests, &m.gsrc, &m.wsrc, &m.small_gone, &m.large};
  size_t bytes = 0;
  for (int i = 0; i < MP_LISTS; i++) { e->mp_at[i] = bytes; bytes += align_up(4 * lists[i]->size(), 16); }
  CK(e->mp.wait());
  CK(e->mp.reserve(bytes, bytes / 2 + 4096));  // (reserved at create for the largest map: no pinned allocation here)
  for (int i = 0; i < MP_LISTS; i++) if (!lists[i]->empty()) memcpy(e->mp.h + e->mp_at[i], lists[i]->data(), 4 * lists[i]->size());
  CK(cudaMemcpyAsync(e->mp.d, e->mp.h, bytes, cudaMemcpyHostToDevice, e->scopy));
  CK(cudaEventRecord(e->mp.ev, e->scopy));
  e->mp.busy = true;
  e->h2d_accum += bytes;
  if (!m.gone.empty()) {  // (without gone rows no resident row shifted: the diff classes the rows past the resident ones as new by itself)
    auto dev = [&](MapList i) { return reinterpret_cast<const uint32_t *>(e->mp.d + e->mp_at[i]); };
    oa.map_pass = 1;
    oa.init = dev(MP_INIT); oa.n_init = (uint32_t)m.init.size();
    oa.gsrc = dev(MP_GSRC); oa.wsrc = dev(MP_WSRC);
    for (int k = 0, i = 0; i < kNumCols - 1; i++) {
      const int d = kCols[i].dim;
      if (d == D_PODS) continue;
      oa.map_kind[k] = d == D_CLUSTERS ? KR_MAP_CLUSTER : d == D_GROUPS ? KR_MAP_GROUP : d == D_WTD ? KR_MAP_NAME : 0;
      oa.shift_from[k] = d == D_GROUPS ? m.gs0 : d == D_WTD ? m.ws0 : 0u;
      if (i == kGroupOffCol || i == kWtdOffCol) oa.cls[k] = KR_OC_COPY;  // (the offsets follow from the counts: groups and names stay in row order)
      k++;
    }
  }
  if (m.names_moved) e->rec.wtd_rebuild = true;
  e->map_pending = true;
  e->map_sizes = n;
  return KR_OK;
}

// The on-device diff of an object commit (kr_incr.cuh), on the copy stream: the staged rows of oa's columns against the resident
// ones (changed rows mark their RayCluster dirty, a changed key makes the next pass a full one), the head-aux keys of the n_hd rows
// head_rows (device list; nullptr: rows 0 .. n_hd - 1), then with `refresh` the input records (cl_in) of the RayClusters the diff
// found changed, now that every column of theirs is in place.
int launch_object_diff(kr_engine *e, const ObjDiffArgs &oa, uint32_t n_hd, const uint32_t *head_rows, bool refresh) {
  SnapDev sd;
  bind_in(e->il, e->d_in, &sd);
  ScratchDev scd = bind_scratch(e->sl, e->d_scratch);
  const uint32_t rows = oa.first[oa.n_cols];
  if (rows) k_inc_objects<<<(rows + 255) / 256, 256, 0, e->scopy>>>(oa, sd, scd, sizes_of(e->sizes));
  if (rows && oa.map_pass) {  // (a row map: the shifted rows were diffed by the launch above, this one copies them and diffs the rest)
    ObjDiffArgs copy = oa;
    copy.map_pass = 2;
    k_inc_objects<<<(rows + 255) / 256, 256, 0, e->scopy>>>(copy, sd, scd, sizes_of(e->sizes));
  }
  if (n_hd) k_inc_objects_keys<<<(n_hd + 255) / 256, 256, 0, e->scopy>>>(oa.h_pod_idx_new, const_cast<uint32_t *>(sd.h_pod_idx), n_hd, head_rows);
  if (refresh) k_inc_refresh<<<std::min<uint32_t>((uint32_t)e->sm_count * 2, (e->sizes.n_clusters + 255) / 256 + 1), 256, 0, e->scopy>>>(sd, scd);
  CK(cudaGetLastError());
  return KR_OK;
}

// The end of every commit on the copy stream: ev_h2d1 closes its copy time (kr_profile.h2d_ms), ev_cols (cols; else the caller
// recorded it ahead of its JSON copy) gates stream M of the next pass, and ev_json (json) its hash, which need not wait for commits
// that leave the JSON alone.
int finish_commit(kr_engine *e, uint64_t bytes, bool cols, bool json) {
  CK(cudaEventRecord(e->ev_h2d1, e->scopy));
  if (cols) CK(cudaEventRecord(e->ev_cols, e->scopy));
  if (json) CK(cudaEventRecord(e->ev_json, e->scopy));
  e->h2d_timed = false;
  e->prof.h2d_bytes = (e->h2d_accum += bytes);
  e->committed = true;
  return KR_OK;
}

}  // namespace

// =================================================================================================== C ABI

extern "C" {

#ifdef KR_TIMELINE
// development aid: (first block start, last block end) in ns of %globaltimer for kernel ids 0..31 of the last graph replay
int kr_debug_timeline(kr_engine *e, unsigned long long *out64) {
  CK(cudaStreamSynchronize(e->sm));
  CK(cudaMemcpyFromSymbol(out64, g_tl, 64 * sizeof(unsigned long long)));
  return KR_OK;
}
#endif

int kr_engine_set_option(kr_engine *e, uint32_t option, uint64_t value) {
  if (!e) return KR_E_INVALID;
  if (option == KR_OPT_FIXED_LAYOUT) {
    if (e->begun) return fail(e, KR_E_STATE, "KR_OPT_FIXED_LAYOUT must be set before the first kr_snapshot_begin");
    e->fixed_layout = value != 0;
    return KR_OK;
  }
  if (option == KR_OPT_INCREMENTAL) {
    e->no_incr = value == 0;
    if (e->no_incr) drop_state(e, KR_FULL_DISABLED);
    return KR_OK;
  }
  if (option == KR_OPT_WTD_EDITS) {  // (read at each object commit: nothing resident depends on it)
    e->wtd_edits = value != 0;
    return KR_OK;
  }
  if (option == KR_OPT_SPEC_ROWS) {  // (read by kr_packer_flush only)
    e->spec_rows_opt = value != 0;
    return KR_OK;
  }
  if (option == KR_OPT_JSON_MOVES) {  // (read by kr_packer_flush only)
    e->json_moves_opt = value != 0;
    return KR_OK;
  }
  if (option == KR_OPT_CLUSTER_CREATES) {  // (read at each kr_snapshot_begin and object commit)
    e->cluster_creates = value != 0;
    return KR_OK;
  }
  if (option == KR_OPT_CLUSTER_DELETES) {  // (read at each kr_snapshot_begin and object commit)
    e->cluster_deletes = value != 0;
    return KR_OK;
  }
  if (option == KR_OPT_GROUP_EDITS) {  // (read at each kr_snapshot_begin and object commit, and by kr_packer_cluster_upsert)
    e->group_edits = value != 0;
    return KR_OK;
  }
  if (option == KR_OPT_BUCKET_POD_LISTS) {  // (read at each pass; a fetching pass's captured graph follows it)
    if (e->bucket_lists != (value != 0)) e->gvalid = false;
    e->bucket_lists = value != 0;
    return KR_OK;
  }
  if (option == KR_OPT_LARGE_MOVES) {  // (read at each object commit)
    e->large_moves = value != 0;
    return KR_OK;
  }
  if (option == KR_OPT_HUGE_GROWTH) {  // (read at each incremental pass)
    if (value && e->huge_reserve < KR_HUGE_GROW_TILES) {
      CK(cudaSetDevice(e->cfg.device));
      if (!e->d_huge) e->huge_tiles = resident_tiles(e->cfg);  // (KR_OPT_HUGE_CLUSTERS then finds the scratch allocated)
      if (int rc = alloc_huge(e, KR_HUGE_GROW_TILES)) return rc;
    }
    e->huge_growth = value != 0;
    e->lg_stale = true;  // (the next pass uploads the reserve entries free)
    return KR_OK;
  }
  if (option == KR_OPT_LARGE_GROWTH) {  // (read at each incremental pass)
    if (value && !e->d_grow) {
      CK(cudaSetDevice(e->cfg.device));
      CK(cudaMalloc((void **)&e->d_grow, kGrowBytes));
      CK(cudaHostAlloc((void **)&e->h_grow, 16 * KR_GROW_MAX, cudaHostAllocDefault));
    }
    e->large_growth = value != 0;
    e->lg_stale = true;  // (the next pass uploads the region table, all zero while no RayCluster has a region)
    return KR_OK;
  }
  if (option == KR_OPT_LARGE_CLUSTERS || option == KR_OPT_WIDE_CLUSTERS || option == KR_OPT_HUGE_CLUSTERS) {
    bool &on = option == KR_OPT_LARGE_CLUSTERS ? e->large_on : option == KR_OPT_WIDE_CLUSTERS ? e->wide_on : e->huge_on;
    if (on == (value != 0)) return KR_OK;
    if (value) CK(cudaSetDevice(e->cfg.device));
    if (value && option != KR_OPT_HUGE_CLUSTERS && !e->d_lg) {  // the cluster table and list of the per-cluster kernels
      const size_t Nc = e->cfg.max_clusters;
      CK(cudaMalloc((void **)&e->d_lg, align_up(16 * Nc) + 4 * Nc));
      CK(cudaMemset(e->d_lg, 0, align_up(16 * Nc)));  // (no region anywhere: see drop_regions)
    }
    if (value && option == KR_OPT_LARGE_CLUSTERS && !e->d_region) {
      // every region holds about 1.25x its cluster's pods rounded up to 32 records, and a large cluster lists more than 256 pods:
      // this many records hold the regions of any snapshot within the capacities
      const size_t Np = e->cfg.max_pods;
      const size_t entries = Np * 5 / 4 + 32 * (Np / 257 + 1);
      CK(cudaMalloc((void **)&e->d_region, sizeof(uint2) * entries));
      e->large_entries = entries;
    }
    if (value && option == KR_OPT_HUGE_CLUSTERS && !e->d_huge) {
      e->huge_tiles = resident_tiles(e->cfg);
      if (int rc = alloc_huge(e, 0)) return rc;
    }
    on = value != 0;
    // the next full pass starts again from the layout's first stride and the fast sort pipeline: a pass with the option off may
    // have left the bucket pipeline (and the fast pipeline, for a cluster above 1024 pods) for this layout
    if (int rc = drop_regions(e, 0)) return rc;
    e->lg_cursor = 0; e->lg_stale = true; e->gvalid = false;
    drop_state(e, KR_FULL_OPTION);
    e->force_radix = e->env_radix;
    if (e->begun) e->bstride = first_stride(e->sizes);
    return KR_OK;
  }
  if (option == KR_OPT_BUCKET_STRIDE) return fail(e, KR_E_INVALID, "KR_OPT_BUCKET_STRIDE can only be read");
  if (option == KR_OPT_SM_COUNT) return fail(e, KR_E_INVALID, "KR_OPT_SM_COUNT can only be read");
  return fail(e, KR_E_INVALID, "unknown option %u", option);
}

int kr_engine_get_option(kr_engine *e, uint32_t option, uint64_t *value) {
  if (!e || !value) return KR_E_INVALID;
  switch (option) {
    case KR_OPT_FIXED_LAYOUT: *value = e->fixed_layout; return KR_OK;
    case KR_OPT_INCREMENTAL: *value = !e->no_incr; return KR_OK;
    case KR_OPT_LARGE_CLUSTERS: *value = e->large_on; return KR_OK;
    case KR_OPT_WIDE_CLUSTERS: *value = e->wide_on; return KR_OK;
    case KR_OPT_HUGE_CLUSTERS: *value = e->huge_on; return KR_OK;
    case KR_OPT_WTD_EDITS: *value = e->wtd_edits; return KR_OK;
    case KR_OPT_SPEC_ROWS: *value = e->spec_rows_opt; return KR_OK;
    case KR_OPT_CLUSTER_CREATES: *value = e->cluster_creates; return KR_OK;
    case KR_OPT_CLUSTER_DELETES: *value = e->cluster_deletes; return KR_OK;
    case KR_OPT_GROUP_EDITS: *value = e->group_edits; return KR_OK;
    case KR_OPT_LARGE_GROWTH: *value = e->large_growth; return KR_OK;
    case KR_OPT_LARGE_MOVES: *value = e->large_moves; return KR_OK;
    case KR_OPT_HUGE_GROWTH: *value = e->huge_growth; return KR_OK;
    case KR_OPT_BUCKET_POD_LISTS: *value = e->bucket_lists; return KR_OK;
    case KR_OPT_JSON_MOVES: *value = e->json_moves_opt; return KR_OK;
    case KR_OPT_BUCKET_STRIDE: *value = e->bstride; return KR_OK;
    case KR_OPT_SM_COUNT: *value = (uint64_t)e->sm_count; return KR_OK;
    default: return fail(e, KR_E_INVALID, "unknown option %u", option);
  }
}

int kr_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return KR_E_NO_DEVICE; }
  return n;
}

int kr_engine_create(const kr_config *cfg, kr_engine **out) {
  if (!cfg || !out) return KR_E_INVALID;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return KR_E_NO_DEVICE; }
  if (cfg->device < 0 || cfg->device >= ndev) return KR_E_INVALID;
  kr_engine *e = new kr_engine();
  e->cfg = *cfg;
  auto bail = [&](int code) { kr_engine_destroy(e); return code; };
  if (cudaSetDevice(cfg->device) != cudaSuccess) return bail(KR_E_CUDA);
  cudaDeviceGetAttribute(&e->sm_count, cudaDevAttrMultiProcessorCount, cfg->device);
  kr_sizes cap = cap_sizes(*cfg);
  e->in_cap = in_layout(cap).total;
  e->scratch_cap = scratch_layout(cap).total;
  e->out_cap = out_layout(cap, cfg->max_creates).total;
  // Block-scheduling priorities (kept by the captured graph nodes): the short general-decide kernel on G goes ahead of the
  // k_decide_small blocks still queued on M, and both go ahead of the hash, which is never on the critical path of the chain.
  int prio_least = 0, prio_greatest = 0;
  cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest);
  const int prio_m = prio_greatest < prio_least ? prio_greatest + 1 : prio_greatest;
  if (cudaStreamCreateWithPriority(&e->sm, cudaStreamNonBlocking, prio_m) != cudaSuccess) return bail(KR_E_CUDA);
  if (cudaStreamCreateWithPriority(&e->sh, cudaStreamNonBlocking, prio_least) != cudaSuccess) return bail(KR_E_CUDA);
  if (cudaStreamCreateWithPriority(&e->sg, cudaStreamNonBlocking, prio_greatest) != cudaSuccess) return bail(KR_E_CUDA);
  if (cudaStreamCreateWithFlags(&e->scopy, cudaStreamNonBlocking) != cudaSuccess) return bail(KR_E_CUDA);
  cudaEventCreate(&e->ev_h2d0); cudaEventCreate(&e->ev_h2d1); cudaEventCreate(&e->ev_cols); cudaEventCreate(&e->ev_json);
  for (cudaEvent_t *ev : {&e->pr.ev, &e->orow.ev, &e->mp.ev, &e->mv.ev, &e->ev_inc, &e->ev_order, &e->ev_fork2, &e->ev_join2, &e->ev_fork3, &e->ev_join3, &e->ev_fork, &e->ev_hash})
    cudaEventCreateWithFlags(ev, cudaEventDisableTiming);
  cudaEventCreate(&e->ev_a); cudaEventCreate(&e->ev_b); cudaEventCreate(&e->ev_c);
  for (auto &ev : e->ev_k) cudaEventCreate(&ev);
  if (cudaHostAlloc((void **)&e->h_in, e->in_cap, cudaHostAllocDefault) != cudaSuccess) return bail(KR_E_CUDA);
  if (cudaHostGetDevicePointer((void **)&e->h_in_dev, e->h_in, 0) != cudaSuccess) return bail(KR_E_CUDA);  // (mapped under UVA)
  if (cudaHostAlloc((void **)&e->h_out, e->out_cap, cudaHostAllocDefault) != cudaSuccess) return bail(KR_E_CUDA);
  if (cudaMalloc((void **)&e->d_in, e->in_cap) != cudaSuccess) return bail(KR_E_CUDA);
  if (cudaMalloc((void **)&e->d_scratch, e->scratch_cap) != cudaSuccess) return bail(KR_E_CUDA);
  if (cudaMalloc((void **)&e->d_out, e->out_cap) != cudaSuccess) return bail(KR_E_CUDA);
  cudaMemset(e->d_out, 0, e->out_cap);  // the alignment padding between the result arrays travels with the single D2H copy
  cudaMemset(e->d_scratch, 0, e->scratch_cap);  // bucket records past a cluster's count are loaded speculatively (and masked): never garbage
  cudaFuncSetAttribute(k_place_fused, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * (int)kFusedMaxCounters);
  cudaFuncSetAttribute(k_creates_fused, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * (int)kFusedMaxCounters);
  {
    // One shared-memory carveout for every kernel of the pass.  An SM can only change its L1 / shared-memory split while it is
    // idle, and the hash kernel keeps every SM busy for the first half of the pass: with per-kernel defaults the main chain
    // either inherits whatever split the previous pass left behind (k_match then runs with a minimal L1) or waits for the
    // hash to drain (split 0 / 25: k_place_fused starts late).  50 % holds the largest
    // shared-memory user (k_creates_fused, 80 KB) and leaves about 114 KB of L1 for the table probes (an SM has
    // 256 KB of L1 / shared memory).  tools/timeline.py shows the effect on the pass; KR_CARVEOUT=<percent> overrides.
    int pct = 50;
    if (const char *g = getenv("KR_CARVEOUT")) pct = atoi(g);
    const void *ks[] = {(const void *)k_build_tables, (const void *)k_match<true, kMatchItems>, (const void *)k_place_fused, (const void *)k_decide_small,
                        (const void *)k_decide, (const void *)k_creates_fused, (const void *)k_jobs, (const void *)k_hash2<1, 0>, (const void *)k_hash2<4, 1>,
                        (const void *)k_clear, (const void *)k_match<false, kSortItems>, (const void *)k_hist, (const void *)k_scan_rows, (const void *)k_scatter,
                        (const void *)k_scan_counts, (const void *)k_place, (const void *)k_scan_creates, (const void *)k_create_fill, (const void *)k_scan_actions,
                        (const void *)k_compact_actions, (const void *)k_patch_pods, (const void *)k_patch_pod_values,
                        (const void *)k_match2<kMatchItems>, (const void *)k_decide2<2>, (const void *)k_decide2<4>, (const void *)k_decide2<8>, (const void *)k_hash3<1, 0>,
                        (const void *)k_inc_retire, (const void *)k_inc_objects, (const void *)k_inc_objects_keys, (const void *)k_inc_aux_clear, (const void *)k_inc_aux_insert,
                        (const void *)k_inc_mark_recreate, (const void *)k_decide2<2, true>, (const void *)k_decide2<4, true>, (const void *)k_decide2<8, true>, (const void *)k_inc_refresh, (const void *)k_inc_admit,
                        (const void *)k_inc_finish, (const void *)k_decide2<2, false, true>, (const void *)k_decide2<4, false, true>, (const void *)k_decide2<8, false, true>,
                        (const void *)k_decide2<2, true, true>, (const void *)k_decide2<4, true, true>, (const void *)k_decide2<8, true, true>,
                        (const void *)k_large_sort<false>, (const void *)k_large_sort<true>, (const void *)k_decide_large<false, kLargeDecideThreads>, (const void *)k_decide_large<true, kLargeDecideThreads>,
                        (const void *)k_decide_large<false, kHugeDecideThreads>, (const void *)k_decide_large<true, kHugeDecideThreads>, (const void *)k_inc_grow<false>, (const void *)k_inc_grow<true>,
                        (const void *)k_huge_tiles<false>, (const void *)k_huge_tiles<true>, (const void *)k_huge_merge<false>, (const void *)k_huge_merge<true>};
    for (const void *k : ks) cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, pct);
  }
  if (const char *g = getenv("KR_NO_GRAPH")) e->use_graph = !(g[0] == '1');
  if (const char *g = getenv("KR_FORCE_RADIX")) e->env_radix = (g[0] == '1');
  if (const char *g = getenv("KR_NO_FUSE")) e->no_fuse = (g[0] == '1');
  if (const char *g = getenv("KR_NO_PDL")) e->use_pdl = !(g[0] == '1');
  if (const char *g = getenv("KR_HASH_CTAS")) e->hash_ctas_per_sm = atoi(g) > 0 ? atoi(g) : 2;
  if (const char *g = getenv("KR_PLACE_CTAS")) e->place_ctas = atoi(g) > 0 ? atoi(g) : 1;
  // (tests: the grids of a part with fewer SMs; never more than the device has, so no persistent or spinning CTA waits for a slot;
  // a value that is not a positive number is ignored, like the two knobs above)
  if (const char *g = getenv("KR_SM_COUNT")) if (atoi(g) > 0) e->sm_count = std::min(e->sm_count, atoi(g));
  e->force_radix = e->env_radix;
  if (cudaHostAlloc((void **)&e->h_totals, 64, cudaHostAllocDefault) != cudaSuccess) return bail(KR_E_CUDA);
  if (const char *g = getenv("KR_NO_BUCKET")) e->no_bucket = (g[0] == '1');
  if (const char *g = getenv("KR_NO_INCR")) e->no_incr = (g[0] == '1');
  if (const char *g = getenv("KR_NO_HASH_SPIN")) e->hash_spin = !(g[0] == '1');
  if (const char *g = getenv("KR_EPOCH_BASE")) {  // (tests: the device's and the host's stamp counters start near their wrap)
    const uint32_t base = (uint32_t)strtoul(g, nullptr, 0);
    if (base) e->epoch_seed = e->dev_epoch = e->row_epoch = e->spec_epoch = e->pull_epoch = base;
  }
  if (cudaHostAlloc((void **)&e->h_inc, 64, cudaHostAllocDefault) != cudaSuccess) return bail(KR_E_CUDA);
  {  // buffers of the incremental path, sized for the capacities up front (a pinned allocation inside an epoch costs milliseconds)
    const InLayout capl = in_layout(cap);
    const size_t objs = capl.off[kFirstPodCol] + (capl.off[kNumCols - 1] - capl.off[kFirstPodCol + 7]);
    if (cudaMalloc((void **)&e->d_obj_stage, objs) != cudaSuccess) return bail(KR_E_CUDA);
    e->obj_stage_cap = objs;
    if (e->inc_stage.reserve(inc_stage_layout(cfg->max_clusters, cfg->max_groups).total, 0) != cudaSuccess) return bail(KR_E_CUDA);
    // the largest row map: gone / digests of kMapMax rows, every RayCluster created, every group and name shifted, and with
    // KR_OPT_LARGE_MOVES the gone rows once more and four words per gone row
    if (e->mp.reserve(4 * (8 * (size_t)kMapMax + cfg->max_clusters + cfg->max_groups + cfg->max_wtd) + MP_LISTS * 16, 0) != cudaSuccess) return bail(KR_E_CUDA);
    const size_t chg = std::max<size_t>(1024, (size_t)cfg->max_clusters);
    if (cudaHostAlloc((void **)&e->h_changed, 4 * chg, cudaHostAllocDefault) != cudaSuccess) return bail(KR_E_CUDA);
    e->h_changed_cap = chg;
  }
  if (cudaHostAlloc((void **)&e->h_order, 4 * ((size_t)cfg->max_clusters + 1), cudaHostAllocDefault) != cudaSuccess) return bail(KR_E_CUDA);
  if (cudaMalloc((void **)&e->d_order, 4 * ((size_t)cfg->max_clusters + 1)) != cudaSuccess) return bail(KR_E_CUDA);
  if (e->spec.reserve(20 * ((size_t)cfg->max_clusters + 1), 0) != cudaSuccess) return bail(KR_E_CUDA);
  cudaFuncSetAttribute(k_hash3<1, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(H3Smem));
  *out = e;
  return KR_OK;
}

void kr_engine_destroy(kr_engine *e) {
  if (!e) return;
  cudaSetDevice(e->cfg.device);
  if (e->sm) cudaStreamSynchronize(e->sm);
  if (e->sh) cudaStreamSynchronize(e->sh);
  if (e->h_in) cudaFreeHost(e->h_in);
  if (e->h_out) cudaFreeHost(e->h_out);
  e->hb.release(); e->pr.release(); e->orow.release(); e->mp.release(); e->inc_stage.release(); e->spec.release(); e->mv.release();
  if (e->d_json_scratch) cudaFree(e->d_json_scratch);
  if (e->h_totals) cudaFreeHost(e->h_totals);
  if (e->h_order) cudaFreeHost(e->h_order);
  if (e->h_inc) cudaFreeHost(e->h_inc);
  if (e->h_grow) cudaFreeHost(e->h_grow);
  if (e->h_changed) cudaFreeHost(e->h_changed);
  if (e->d_obj_stage) cudaFree(e->d_obj_stage);
  if (e->d_lg) cudaFree(e->d_lg);
  if (e->d_region) cudaFree(e->d_region);
  if (e->d_grow) cudaFree(e->d_grow);
  if (e->d_huge) cudaFree(e->d_huge);
  if (e->d_order) cudaFree(e->d_order);
  if (e->d_in) cudaFree(e->d_in);
  if (e->d_scratch) cudaFree(e->d_scratch);
  if (e->d_out) cudaFree(e->d_out);
  if (e->gexec) cudaGraphExecDestroy(e->gexec);
  for (auto ev : {e->ev_fork, e->ev_hash, e->ev_a, e->ev_b, e->ev_c}) if (ev) cudaEventDestroy(ev);
  for (auto ev : e->ev_k) if (ev) cudaEventDestroy(ev);
  if (e->sm) cudaStreamDestroy(e->sm);
  if (e->sh) cudaStreamDestroy(e->sh);
  if (e->sg) cudaStreamDestroy(e->sg);
  if (e->scopy) { cudaStreamSynchronize(e->scopy); cudaStreamDestroy(e->scopy); }
  for (auto ev : {e->ev_h2d0, e->ev_h2d1, e->ev_cols, e->ev_json, e->ev_inc, e->ev_order, e->ev_fork2, e->ev_join2, e->ev_fork3, e->ev_join3}) if (ev) cudaEventDestroy(ev);
  delete e;
}

int kr_snapshot_begin(kr_engine *e, const kr_sizes *sizes, kr_snapshot_bufs *out) {
  if (!e || !sizes || !out) return KR_E_INVALID;
  const kr_config &c = e->cfg;
  if (sizes->n_clusters > c.max_clusters || sizes->n_groups > c.max_groups || sizes->n_wtd > c.max_wtd || sizes->n_pods > c.max_pods ||
      sizes->n_heads > c.max_heads || sizes->n_jobs > c.max_jobs || sizes->json_bytes > c.max_json_bytes)
    return fail(e, KR_E_CAPACITY, "snapshot exceeds the engine capacities given to kr_engine_create");
  if (sizes->n_clusters >= 0xFFFFFFF0u || sizes->n_pods >= 0xFFFFFFF0u) return fail(e, KR_E_CAPACITY, "too many rows");
  CK(cudaSetDevice(c.device));
  CK(cudaStreamSynchronize(e->scopy));
  CK(cudaStreamSynchronize(e->sm));  // previous results are invalidated from here on
  if (memcmp(&e->sizes, sizes, sizeof *sizes) != 0) {  // row counts (and, without KR_OPT_FIXED_LAYOUT, every column address) change
    e->gvalid = false;
    // The resident state of the incremental path survives new live counts under a fixed layout as long as the object tables keep
    // their shape: pod rows appended (they arrive as committed rows), head-aux rows come and go, the JSON arena grows; with
    // KR_OPT_WTD_EDITS workersToDelete lists grow and shrink as well while the RayClusters and groups stay (the name table is sized
    // for the capacity).  The RayCluster, group and name counts may each grow with KR_OPT_CLUSTER_CREATES (RayClusters created, with
    // their groups and names) while the bucket arena holds the RayClusters at the current stride, with which RayJobs come and go as
    // well, and shrink with KR_OPT_CLUSTER_DELETES (RayClusters deleted by swap-remove); with KR_OPT_GROUP_EDITS the group and name
    // counts may move either way (RayClusters that gained or lost worker groups); the object commit's row map checks the rest.
    const bool fits = (size_t)sizes->n_clusters * e->bstride <= e->sl.bucket_entries;
    const bool same_groups = sizes->n_clusters == e->sizes.n_clusters && sizes->n_groups == e->sizes.n_groups;
    auto keeps = [&](bool room) {
      auto moves_ok = [&](uint32_t now, uint32_t was) { return now == was || (now < was ? deletes_on(e) : creates_on(e) && room); };
      return e->inc_valid && e->fixed_layout && moves_ok(sizes->n_clusters, e->sizes.n_clusters) &&
             (moves_ok(sizes->n_groups, e->sizes.n_groups) || regroups_on(e)) &&
             (moves_ok(sizes->n_wtd, e->sizes.n_wtd) || (e->wtd_edits && same_groups) || regroups_on(e)) &&
             (sizes->n_jobs == e->sizes.n_jobs || creates_on(e)) && sizes->n_pods >= e->sizes.n_pods;
    };
    const bool keep = keeps(fits);
    if (!e->fixed_layout) { e->committed_full = false; e->inc_zero_needed = true; }
    // (the next pass is a full one, which hashes every message: listed rows may not exist any more)
    if (sizes->n_clusters != e->sizes.n_clusters && !keep) clear_spec_rows(e);
    if (!keep) {
      // (KR_OPT_CLUSTER_CREATES follows these counts, but the bucket arena does not hold the new RayClusters at this stride)
      drop_state(e, keeps(true) ? KR_FULL_ROW_MAP : KR_FULL_SIZES);
      e->force_radix = e->env_radix;
      e->bstride = first_stride(*sizes);
      if (int rc = drop_regions(e, 0)) return rc;
      e->lg_cursor = 0; e->lg_stale = true;
    }
  }
  e->sizes = *sizes;
  const kr_sizes lay = e->fixed_layout ? cap_sizes(c) : *sizes;
  e->il = in_layout(lay);
  e->ol = out_layout(lay, c.max_creates);
  e->sl = scratch_layout(lay);
  if (e->fixed_layout) {  // offsets and table sizes from the capacities, tile counts (grid sizes) from the live pod count
    const ScratchLayout live = scratch_layout(*sizes);
    e->sl.ntiles = live.ntiles; e->sl.mtiles = live.mtiles;
  }
  if (e->il.total > e->in_cap || e->ol.total > e->out_cap || e->sl.total > e->scratch_cap)
    return fail(e, KR_E_CAPACITY, "internal: layout exceeds arena");
  bind_in(e->il, e->h_in, out);
  e->begun = true; e->committed = false; e->ran = false;
  return KR_OK;
}

int kr_snapshot_commit(kr_engine *e) { return kr_snapshot_commit_parts(e, KR_PART_ALL); }

int kr_snapshot_commit_parts(kr_engine *e, uint32_t parts) {
  if (!e || !e->begun) return e ? fail(e, KR_E_STATE, "kr_snapshot_commit before kr_snapshot_begin") : KR_E_INVALID;
  CK(cudaSetDevice(e->cfg.device));
  // every row checked, the groups stored in cluster order and their workersToDelete names in group order
  kr_snapshot_bufs hb;
  bind_in(e->il, e->h_in, &hb);
  const kr_sizes &n = e->sizes;
  uint64_t goff = 0, woff = 0;
  for (uint32_t c = 0; c < n.n_clusters; c++) {
    if (hb.c_group_off[c] != goff) return fail(e, KR_E_INVALID, "cluster %u: groups must be stored in cluster order (group_off %u != %llu)", c, hb.c_group_off[c], (unsigned long long)goff);
    if (int rc = check_cluster_row(e, hb, n, c)) return rc;
    for (uint64_t g = goff; g < goff + hb.c_group_cnt[c]; g++) {
      if (hb.g_wtd_off[g] != woff) return fail(e, KR_E_INVALID, "group %llu: workersToDelete names must be stored in group order (wtd_off %u != %llu)", (unsigned long long)g, hb.g_wtd_off[g], (unsigned long long)woff);
      woff += hb.g_wtd_cnt[g];
    }
    goff += hb.c_group_cnt[c];
  }
  if (goff != n.n_groups) return fail(e, KR_E_INVALID, "sum of group_cnt (%llu) != n_groups (%u)", (unsigned long long)goff, n.n_groups);
  if (woff != n.n_wtd) return fail(e, KR_E_INVALID, "sum of g_wtd_cnt (%llu) != n_wtd (%u)", (unsigned long long)woff, n.n_wtd);
  for (uint32_t h = 0; h < n.n_heads; h++)
    if (int rc = check_head_row(e, hb, n, h)) return rc;
  if ((parts & KR_PART_ALL) != KR_PART_ALL && !e->committed_full)
    return fail(e, KR_E_STATE, "a partial commit needs a full commit of this layout first");
  const size_t a1 = e->il.off[kFirstPodCol], b0 = e->il.off[kFirstPodCol + 7], json_off = e->il.off[kNumCols - 1];
  // While the incremental state is resident, an object commit lands beside the resident tables and is diffed against them on
  // the device (k_inc_objects): changed rows mark their RayCluster dirty, a changed key makes the next pass a full one.
  const bool stage_objects = e->inc_valid && !e->no_incr && (parts & KR_PART_OBJECTS) && !(parts & KR_PART_COLUMNS);
  if (stage_objects && a1 + (json_off - b0) > e->obj_stage_cap)
    return fail(e, KR_E_STATE, "internal: object part of %zu bytes, staging room for %zu", a1 + (json_off - b0), e->obj_stage_cap);
  auto stage_of = [&](size_t off) { return off < a1 ? off : a1 + (off - b0); };
  size_t at[kNumCols];
  for (int i = 0; i < kNumCols; i++) at[i] = stage_of(e->il.off[i]);
  const uint32_t cnt[7] = {n.n_clusters, n.n_groups, n.n_wtd, n.n_pods, n.n_heads, n.n_jobs, 0};
  ObjDiffArgs oa = object_diff_args(e, e->d_obj_stage, at, cnt, nullptr);  // (before the record moves on)
  if (e->order_pending) { CK(cudaEventSynchronize(e->ev_order)); e->order_pending = false; }  // a previous upload may still be reading h_order
  if (int rc = begin_commit(e)) return rc;
  const bool renumbered = e->map_pending && !e->rec.map.gone.empty();  // (by an earlier object commit of this epoch)
  const CommitRecord::Moved moved = e->rec.commit_whole(hb, n, parts, e->wtd_edits, creates_on(e), deletes_on(e), regroups_on(e), e->inc_n_clusters);
  if (moved.shape) e->gvalid = false;  // launch shape / pipeline depend on it
  // The object part created or renumbered RayClusters, or moved a row count after a renumbering of this epoch.  A pending renumbering
  // is not composed with either: its map would no longer describe the rows.  (Created RayClusters after created ones: the new map
  // lists them all.)
  bool voided = false;
  const bool recounted = renumbered && (parts & KR_PART_OBJECTS) &&
                         (n.n_clusters != e->map_sizes.n_clusters || n.n_groups != e->map_sizes.n_groups || n.n_wtd != e->map_sizes.n_wtd);
  if (moved.map != 0 || recounted) {
    if (int rc = commit_map(e, moved.map == 1 && stage_objects && !renumbered, oa, voided)) return rc;
  }
  if (moved.wide && e->wide_on) e->lg_stale = true;  // a different wide set is a different list, and grid, of the per-cluster kernels
  if (parts & KR_PART_COLUMNS) drop_state(e, KR_FULL_COLUMNS);  // pod columns uploaded wholesale: the resident buckets no longer describe them
  if (moved.order) build_order(e, hb);  // (unchanged lengths and gates: the resident order stands — an object / pod epoch does not pay for it)
  // Asynchronous, in two parts on the copy stream: every column first, the spec-JSON arena (the larger half) second.
  // The pass waits on the two events, so match/place/decide run while the JSON is still crossing PCIe and only the hash
  // (and what depends on it) waits for the second part.  Nothing here blocks the host.
  size_t bytes = 0;
  auto up = [&](size_t off, size_t len) -> int {
    if (!len) return KR_OK;
    uint8_t *dst = (stage_objects && off < json_off) ? e->d_obj_stage + stage_of(off) : e->d_in + off;
    CK(cudaMemcpyAsync(dst, e->h_in + off, len, cudaMemcpyHostToDevice, e->scopy));
    bytes += len;
    return KR_OK;
  };
  if ((parts & KR_PART_COLUMNS) && !e->fixed_layout) { if (int rc = up(0, json_off)) return rc; }
  else if (parts & (KR_PART_COLUMNS | KR_PART_OBJECTS)) {
    // the (small) columns on either side of the seven per-pod ones; then, for KR_PART_COLUMNS under a fixed layout, the live
    // prefix of each per-pod column (the capacity slack between the columns is not worth moving)
    if (int rc = up(0, a1)) return rc;
    if (int rc = up(b0, json_off - b0)) return rc;
    if (parts & KR_PART_COLUMNS)
      for (int k = 0; k < 7; k++)
        if (int rc = up(e->il.off[kFirstPodCol + k], 4 * (size_t)n.n_pods)) return rc;
  }
  if (stage_objects) { if (int rc = launch_object_diff(e, oa, n.n_heads, nullptr, n.n_clusters != 0)) return rc; }
  if (voided) drop_state(e, KR_FULL_ROW_MAP);  // (the diff above copied the object part into place: the full pass reads it)
  CK(cudaEventRecord(e->ev_cols, e->scopy));
  if (moved.order && n.n_clusters) {  // the new order travels with this commit
    CK(cudaMemcpyAsync(e->d_order, e->h_order, 4 * (size_t)n.n_clusters, cudaMemcpyHostToDevice, e->scopy)); bytes += 4 * (size_t)n.n_clusters;
    CK(cudaEventRecord(e->ev_order, e->scopy));
    e->order_pending = true;
  }
  if (parts & KR_PART_JSON) { if (int rc = up(json_off, e->fixed_layout ? (size_t)n.json_bytes : e->il.total - json_off)) return rc; }
  if ((parts & KR_PART_ALL) == KR_PART_ALL) e->committed_full = true;
  return finish_commit(e, bytes, false, true);
}

// Shared by the two incremental pod commits: stage the row list (and, journal style, the 7 values per row), upload, scatter.
static int commit_pod_patch(kr_engine *e, const uint32_t *rows, const uint32_t *values, uint32_t n, bool rows_known_distinct = false) {
  if (!e || (!rows && n)) return KR_E_INVALID;
  if (!e->committed_full) return fail(e, KR_E_STATE, "an incremental pod commit needs a full commit of this layout first");
  if (n == 0) return KR_OK;
  CK(cudaSetDevice(e->cfg.device));
  const size_t bytes = (values ? 32 : 4) * (size_t)n;  // row list (+ 7 values per row); kr_snapshot_commit_pod_rows lets the device pull the rows
  CK(e->pr.wait());  // a previous patch may still be reading the staging buffer
  CK(e->pr.reserve(bytes, bytes / 2 + 4096));
  for (uint32_t i = 0; i < n; i++)
    if (rows[i] >= e->sizes.n_pods) return fail(e, KR_E_INVALID, "pod row %u out of range", rows[i]);
  if (values && !rows_known_distinct) {  // the scatter kernel writes one thread per entry: two entries for one row would race
    if (e->row_stamp.size() < e->sizes.n_pods) e->row_stamp.assign(e->sizes.n_pods, 0);
    if (++e->row_epoch == 0) { std::fill(e->row_stamp.begin(), e->row_stamp.end(), 0u); e->row_epoch = 1; }
    for (uint32_t i = 0; i < n; i++) {
      if (e->row_stamp[rows[i]] == e->row_epoch) return fail(e, KR_E_INVALID, "kr_snapshot_commit_pod_values: pod row %u appears twice", rows[i]);
      e->row_stamp[rows[i]] = e->row_epoch;
    }
  }
  memcpy(e->pr.h, rows, 4 * (size_t)n);
  if (values) memcpy(e->pr.h + 4 * (size_t)n, values, 28 * (size_t)n);
  kr_snapshot_bufs hb;
  bind_in(e->il, e->h_in, &hb);
  SnapDev s;
  bind_in(e->il, e->d_in, &s);
  PodCols hc, dc;
  const void *hsrc[7] = {hb.p_ns_id, hb.p_cluster_name_id, hb.p_group_name_id, hb.p_name_id, hb.p_packed, hb.p_replica_index, hb.p_replica_name_id};
  const void *dsrc[7] = {s.p_ns_id, s.p_cluster_name_id, s.p_group_name_id, s.p_name_id, s.p_packed, s.p_replica_index, s.p_replica_name_id};
  for (int k = 0; k < 7; k++) {
    hc.c[k] = reinterpret_cast<uint32_t *>(e->h_in_dev + (static_cast<const uint8_t *>(hsrc[k]) - e->h_in));
    dc.c[k] = static_cast<uint32_t *>(const_cast<void *>(dsrc[k]));
  }
  if (int rc = begin_commit(e)) return rc;
  CK(cudaMemcpyAsync(e->pr.d, e->pr.h, bytes, cudaMemcpyHostToDevice, e->scopy));
  CK(cudaEventRecord(e->pr.ev, e->scopy));
  e->pr.busy = true;
  const uint32_t *drows = reinterpret_cast<const uint32_t *>(e->pr.d);
  if (e->inc_valid && !e->no_incr) {  // the rows' previous values leave the resident state before the new ones land
    ScratchDev scd = bind_scratch(e->sl, e->d_scratch);
    ResDev rd = bind_out(e->ol, e->d_out);
    k_inc_retire<<<(n + 255) / 256, 256, 0, e->scopy>>>(drows, n, s, scd, rd, sizes_of(e->sizes), e->inc_n_pods, e->sizes.n_wtd ? 1 : 0);
  }
  if (values) k_patch_pod_values<<<(n + 255) / 256, 256, 0, e->scopy>>>(drows, n, dc);
  else k_patch_pods<<<(n + 255) / 256, 256, 0, e->scopy>>>(drows, n, hc, dc);
  CK(cudaGetLastError());
  // row list + the 28-byte row payload (pulled one 32-byte sector per value in the rows-only variant); the JSON is untouched
  return finish_commit(e, 32 * (uint64_t)n, true, false);
}


int kr_snapshot_commit_object_rows(kr_engine *e, const uint32_t *cluster_rows, uint32_t n_cl, const uint32_t *head_rows, uint32_t n_hd) {
  if (!e || (!cluster_rows && n_cl) || (!head_rows && n_hd)) return KR_E_INVALID;
  if (!e->begun) return fail(e, KR_E_STATE, "kr_snapshot_commit_object_rows before kr_snapshot_begin");
  if (n_cl == 0 && n_hd == 0) return KR_OK;
  const kr_sizes &n = e->sizes;
  kr_snapshot_bufs hb;
  bind_in(e->il, e->h_in, &hb);
  // the named rows are checked as the whole commit checks them, whichever path follows
  for (uint32_t i = 0; i < n_cl; i++)
    if (int rc = check_cluster_row(e, hb, n, cluster_rows[i])) return rc;
  for (uint32_t i = 0; i < n_hd; i++)
    if (int rc = check_head_row(e, hb, n, head_rows[i])) return rc;
  // Only an optimisation of kr_snapshot_commit_parts(KR_PART_OBJECTS): whenever the resident state cannot take the rows as they
  // are, the whole object part is committed instead (which checks the layout around them as well).
  if (!e->inc_valid || e->no_incr || !e->committed_full || !e->rec.takes_rows(hb, n, cluster_rows, n_cl, e->wtd_edits))
    return kr_snapshot_commit_parts(e, KR_PART_OBJECTS);
  CK(cudaSetDevice(e->cfg.device));
  // group rows of the named clusters
  std::vector<uint32_t> grows;
  for (uint32_t i = 0; i < n_cl; i++) for (uint32_t g = 0; g < hb.c_group_cnt[cluster_rows[i]]; g++) grows.push_back(hb.c_group_off[cluster_rows[i]] + g);
  const uint32_t cnt[7] = {n_cl, (uint32_t)grows.size(), 0, 0, n_hd, 0, 0};
  const uint32_t *lists[7] = {cluster_rows, grows.data(), nullptr, nullptr, head_rows, nullptr, nullptr};
  // staging: the three row lists, then every object column's rows packed in list order
  size_t need = 0, list_off[7] = {0};
  for (int d = 0; d < 7; d++) { list_off[d] = need; need = align_up(need + 4 * (size_t)cnt[d]); }
  size_t col_off[kNumCols] = {0};
  for (int i = 0; i < kNumCols - 1; i++) {
    const int d = kCols[i].dim;
    if (d == D_PODS || !cnt[d]) continue;
    col_off[i] = need; need = align_up(need + (size_t)kCols[i].elem * kCols[i].mult * cnt[d]);
  }
  CK(e->orow.wait());
  CK(e->orow.reserve(need, need / 2 + 65536));
  for (int d = 0; d < 7; d++) if (cnt[d]) memcpy(e->orow.h + list_off[d], lists[d], 4 * (size_t)cnt[d]);
  for (int i = 0; i < kNumCols - 1; i++) {
    const int d = kCols[i].dim;
    if (d == D_PODS || !cnt[d]) continue;
    const size_t rb = (size_t)kCols[i].elem * kCols[i].mult;
    const uint8_t *col = e->h_in + e->il.off[i];
    uint8_t *dst = e->orow.h + col_off[i];
    // (row sizes are 1, 4 or 8 bytes for almost every column: fixed-size copies instead of ~10 k variable-length memcpy calls per epoch)
    const uint32_t *rl = lists[d];
    if (rb == 4) { const uint32_t *c4 = reinterpret_cast<const uint32_t *>(col); uint32_t *d4 = reinterpret_cast<uint32_t *>(dst); for (uint32_t k = 0; k < cnt[d]; k++) d4[k] = c4[rl[k]]; }
    else if (rb == 1) { for (uint32_t k = 0; k < cnt[d]; k++) dst[k] = col[rl[k]]; }
    else if (rb == 8) { const uint64_t *c8 = reinterpret_cast<const uint64_t *>(col); uint64_t *d8 = reinterpret_cast<uint64_t *>(dst); for (uint32_t k = 0; k < cnt[d]; k++) d8[k] = c8[rl[k]]; }
    else for (uint32_t k = 0; k < cnt[d]; k++) memcpy(dst + k * rb, col + (size_t)rl[k] * rb, rb);
  }
  const ObjDiffArgs oa = object_diff_args(e, e->orow.d, col_off, cnt, list_off);
  if (int rc = begin_commit(e)) return rc;
  if (e->rec.commit_rows(hb, cluster_rows, n_cl, head_rows, n_hd)) e->gvalid = false;  // (the captured full pass launches the other k_decide2 instantiation)
  CK(cudaMemcpyAsync(e->orow.d, e->orow.h, need, cudaMemcpyHostToDevice, e->scopy));
  CK(cudaEventRecord(e->orow.ev, e->scopy));
  e->orow.busy = true;
  if (int rc = launch_object_diff(e, oa, n_hd, reinterpret_cast<const uint32_t *>(e->orow.d + list_off[D_HEADS]), n_cl != 0)) return rc;
  return finish_commit(e, need, true, false);
}

int kr_snapshot_commit_spec_rows(kr_engine *e, const uint32_t *rows, uint32_t n) {
  if (!e || (!rows && n)) return KR_E_INVALID;
  if (!e->begun || !e->committed_full) return fail(e, KR_E_STATE, "a spec-row commit needs a full commit of this layout first");
  if (n == 0) return KR_OK;
  const kr_sizes &z = e->sizes;
  kr_snapshot_bufs hb;
  bind_in(e->il, e->h_in, &hb);
  for (uint32_t i = 0; i < n; i++)
    if (int rc = check_cluster_row(e, hb, z, rows[i], true)) return rc;
  CK(cudaSetDevice(e->cfg.device));
  if (e->spec_stamp.size() < z.n_clusters) e->spec_stamp.resize(z.n_clusters, 0u);
  if (e->pull_stamp.size() < z.n_clusters) e->pull_stamp.resize(z.n_clusters, 0u);
  if (e->n_pull == 0) CK(cudaStreamSynchronize(e->scopy));  // (the pinned pull list is rewritten from its start)
  // the rows this call pulls, appended to the pull list: a row pulled since the last pass is in the device arena already (the caller
  // may not rewrite the arenas before the next pass returns); a row listed before that pass, still pending, is pulled again
  const size_t cap = (size_t)e->cfg.max_clusters + 1, base = e->n_pull;
  uint32_t *lr = reinterpret_cast<uint32_t *>(e->spec.h) + base;
  uint32_t *ll = reinterpret_cast<uint32_t *>(e->spec.h + 4 * cap) + base;
  uint64_t *lo = reinterpret_cast<uint64_t *>(e->spec.h + 8 * cap) + base;
  uint32_t m = 0;
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t c = rows[i];
    if (e->pull_stamp[c] == e->pull_epoch) continue;
    e->pull_stamp[c] = e->pull_epoch;
    lr[m++] = c;
    if (e->spec_stamp[c] != e->spec_epoch) { e->spec_stamp[c] = e->spec_epoch; e->spec_pending.push_back(c); }  // (hashed once)
  }
  if (m == 0) return KR_OK;
  size_t bytes = 16 * (size_t)m;
  for (uint32_t i = 0; i < m; i++) {
    ll[i] = hb.c_json_len[lr[i]]; lo[i] = hb.c_json_off[lr[i]];
    bytes += ((size_t)ll[i] + 15) & ~(size_t)15;
  }
  e->rec.commit_spec_rows(lr, lo, ll, m);
  if (int rc = begin_commit(e)) return rc;
  uint32_t *dr = reinterpret_cast<uint32_t *>(e->spec.d) + base;
  uint32_t *dl = reinterpret_cast<uint32_t *>(e->spec.d + 4 * cap) + base;
  uint64_t *dof = reinterpret_cast<uint64_t *>(e->spec.d + 8 * cap) + base;
  CK(cudaMemcpyAsync(dr, lr, 4 * (size_t)m, cudaMemcpyHostToDevice, e->scopy));
  CK(cudaMemcpyAsync(dl, ll, 4 * (size_t)m, cudaMemcpyHostToDevice, e->scopy));
  CK(cudaMemcpyAsync(dof, lo, 8 * (size_t)m, cudaMemcpyHostToDevice, e->scopy));
  const size_t json_off = e->il.off[kNumCols - 1];
  k_spec_pull<<<m, 128, 0, e->scopy>>>(dr, dof, dl, e->h_in_dev + json_off, e->d_in + json_off, reinterpret_cast<uint64_t *>(e->d_in + e->il.off[kJsonOffCol]),
                                       reinterpret_cast<uint32_t *>(e->d_in + e->il.off[kJsonOffCol + 1]));
  CK(cudaGetLastError());
  e->n_pull += m;
  return finish_commit(e, bytes, true, true);  // (k_spec_pull wrote the columns' ranges as well as the JSON)
}

int kr_snapshot_commit_json_moves(kr_engine *e, const uint32_t *rows, uint32_t n) {
  if (!e || (!rows && n)) return KR_E_INVALID;
  if (!e->begun || !e->committed_full) return fail(e, KR_E_STATE, "a JSON move commit needs a full commit of this layout first");
  if (n == 0) return KR_OK;
  const kr_sizes &z = e->sizes;
  kr_snapshot_bufs hb;
  bind_in(e->il, e->h_in, &hb);
  const std::vector<CommitRecord::Row> &rec = e->rec.rows;
  std::vector<uint8_t> seen(rec.size(), 0);
  std::vector<std::pair<uint64_t, uint32_t>> to(n);  // (destination, row) for the overlap check
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t c = rows[i];
    if (c >= rec.size() || c >= z.n_clusters) return fail(e, KR_E_INVALID, "cluster row %u: not a recorded row", c);
    if (seen[c]) return fail(e, KR_E_INVALID, "cluster row %u appears twice", c);
    seen[c] = 1;
    if (hb.c_json_len[c] != rec[c].json_len) return fail(e, KR_E_INVALID, "cluster %u: json length %u, recorded %u (a move keeps the bytes)", c, hb.c_json_len[c], rec[c].json_len);
    if (int rc = check_cluster_row(e, hb, z, c, true)) return rc;
    to[i] = {hb.c_json_off[c], c};
  }
  if (!std::is_sorted(to.begin(), to.end())) std::sort(to.begin(), to.end());  // (a compaction in row order lists them sorted)
  uint64_t end = 0;
  uint32_t last = KR_EMPTY32;  // (the listed row with a non-empty destination that ends last so far)
  for (const auto &t : to) {
    if (!hb.c_json_len[t.second]) continue;
    if (last != KR_EMPTY32 && t.first < end) return fail(e, KR_E_INVALID, "clusters %u and %u: json destinations overlap", last, t.second);
    end = t.first + ((hb.c_json_len[t.second] + 15ull) & ~15ull); last = t.second;
  }
  CK(cudaSetDevice(e->cfg.device));
  const size_t cap = (size_t)e->cfg.max_clusters + 1;
  if (!e->d_json_scratch) {  // (an engine that never moves pays nothing)
    if (e->mv.reserve(24 * cap, 0) != cudaSuccess) return fail(e, KR_E_CUDA, "allocation of the JSON move list failed");
    if (cudaMalloc((void **)&e->d_json_scratch, align_up((size_t)e->cfg.max_json_bytes + 16)) != cudaSuccess) {
      e->d_json_scratch = nullptr;
      return fail(e, KR_E_CUDA, "allocation of the JSON move scratch failed");
    }
  }
  CK(e->mv.wait());  // a previous move list may still be crossing
  uint32_t *lr = reinterpret_cast<uint32_t *>(e->mv.h), *ll = reinterpret_cast<uint32_t *>(e->mv.h + 4 * cap);
  uint64_t *ld = reinterpret_cast<uint64_t *>(e->mv.h + 8 * cap), *ls = reinterpret_cast<uint64_t *>(e->mv.h + 16 * cap);
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t c = rows[i];
    lr[i] = c; ll[i] = rec[c].json_len; ld[i] = hb.c_json_off[c]; ls[i] = rec[c].json_off;
  }
  if (int rc = begin_commit(e)) return rc;
  // a row whose bytes went is pulled again by its next spec-row commit, even within this epoch
  for (uint32_t c : e->rec.commit_json_moves(to, seen)) if (c < e->pull_stamp.size()) e->pull_stamp[c] = 0;
  uint32_t *dr = reinterpret_cast<uint32_t *>(e->mv.d), *dl = reinterpret_cast<uint32_t *>(e->mv.d + 4 * cap);
  uint64_t *dd = reinterpret_cast<uint64_t *>(e->mv.d + 8 * cap), *ds = reinterpret_cast<uint64_t *>(e->mv.d + 16 * cap);
  CK(cudaMemcpyAsync(dr, lr, 4 * (size_t)n, cudaMemcpyHostToDevice, e->scopy));
  CK(cudaMemcpyAsync(dl, ll, 4 * (size_t)n, cudaMemcpyHostToDevice, e->scopy));
  CK(cudaMemcpyAsync(dd, ld, 8 * (size_t)n, cudaMemcpyHostToDevice, e->scopy));
  CK(cudaMemcpyAsync(ds, ls, 8 * (size_t)n, cudaMemcpyHostToDevice, e->scopy));
  CK(cudaEventRecord(e->mv.ev, e->scopy));
  e->mv.busy = true;
  uint8_t *d_json = e->d_in + e->il.off[kNumCols - 1];
  k_json_move_gather<<<n, 128, 0, e->scopy>>>(ds, dd, dl, d_json, e->d_json_scratch);
  k_json_move_scatter<<<n, 128, 0, e->scopy>>>(dr, dd, dl, e->d_json_scratch, d_json, reinterpret_cast<uint64_t *>(e->d_in + e->il.off[kJsonOffCol]),
                                               reinterpret_cast<uint32_t *>(e->d_in + e->il.off[kJsonOffCol + 1]));
  CK(cudaGetLastError());
  return finish_commit(e, 24 * (uint64_t)n, true, true);  // (the move list only: no spec byte crosses PCIe)
}

int kr_snapshot_commit_pod_rows(kr_engine *e, const uint32_t *rows, uint32_t n) { return commit_pod_patch(e, rows, nullptr, n); }

// for kr_packer.cpp: its journal holds every row once (row_dirty), so the duplicate scan is skipped
int kr_internal_commit_pod_values_distinct(kr_engine *e, const uint32_t *rows, const uint32_t *values, uint32_t n) {
  if (!values && n) return KR_E_INVALID;
  return commit_pod_patch(e, rows, values, n, true);
}

int kr_snapshot_commit_pod_values(kr_engine *e, const uint32_t *rows, const uint32_t *values, uint32_t n) {
  if (!values && n) return KR_E_INVALID;
  return commit_pod_patch(e, rows, values, n);
}

// the report of the pass a call that returns KR_OK made (kr_last_pass)
static int published(kr_engine *e, int rc) {
  if (rc == KR_OK) { e->pass_last = e->pass_made; e->has_pass = true; }
  return rc;
}

int kr_reconcile_device_only(kr_engine *e, const kr_flags *flags) {
  if (!e || !flags) return KR_E_INVALID;
  return published(e, run_pass(e, *flags, e->ev_b, false));
}

int kr_reconcile_batch(kr_engine *e, const kr_flags *flags, kr_results_view *out) {
  if (!e || !flags || !out) return KR_E_INVALID;
  static const bool trace = getenv("KR_ENGINE_TRACE") != nullptr;  // development aid: host time of the two halves of a call (stderr)
  const auto t0 = std::chrono::steady_clock::now();
  if (int rc = run_pass(e, *flags, e->ev_k[KR_MAX_KERNEL_TIMES], false)) return rc;
  const auto t1 = std::chrono::steady_clock::now();
  const int rc = fetch_results(e, out);  // d2h_ms = ev_b..ev_c
  if (trace) {
    const auto t2 = std::chrono::steady_clock::now();
    auto us = [](auto a, auto b) { return std::chrono::duration<double, std::micro>(b - a).count(); };
    fprintf(stderr, "kr_reconcile_batch: pass %.0f us (device %.0f us), fetch %.0f us (device copy %.0f us, %llu bytes)%s\n", us(t0, t1), e->prof.kernels_ms * 1e3, us(t1, t2),
            e->prof.d2h_ms * 1e3, (unsigned long long)e->prof.d2h_bytes, e->ran_inc ? " [incremental]" : "");
  }
  return published(e, rc);
}

int kr_reconcile_batch_profiled(kr_engine *e, const kr_flags *flags, kr_profile *prof) {
  if (!e || !flags) return KR_E_INVALID;
  if (int rc = run_pass(e, *flags, e->ev_b, true)) return rc;
  uint32_t k = e->prof.n_kernels < KR_MAX_KERNEL_TIMES ? e->prof.n_kernels : KR_MAX_KERNEL_TIMES;
  for (uint32_t i = 0; i < k; i++) {
    float t = 0;
    cudaEventElapsedTime(&t, e->ev_k[i], e->ev_k[i + 1]);
    e->prof.kernel_ms[i] = t;
  }
  if (prof) *prof = e->prof;
  return published(e, KR_OK);
}

int kr_results_fetch(kr_engine *e, kr_results_view *out) {
  if (!e || !out) return KR_E_INVALID;
  if (!e->ran) return fail(e, KR_E_STATE, "no pass has run on the committed snapshot");
  CK(cudaSetDevice(e->cfg.device));
  return fetch_results(e, out);
}

// Digests of n messages given as (pointer, length) pieces: staged 16-byte aligned in pinned memory (the copies run on `threads` host
// threads when the batch is large), one upload, one SHA-1 launch, digests back.
static int hash_pieces(kr_engine *e, const uint8_t *const *ptr, const uint64_t *len, uint32_t n, char *out32xN, uint32_t threads) {
  if (n == 0) return KR_OK;
  CK(cudaSetDevice(e->cfg.device));
  // staging layout: [aligned offsets (n+0) u64 | lens u32 | order u32 | bytes, each message 16-byte aligned | out 32n]
  size_t data = 0;
  for (uint32_t i = 0; i < n; i++) {
    if (len[i] > 0xFFFFFFFFull) return fail(e, KR_E_CAPACITY, "message %u longer than 4 GiB", i);
    data += align_up(len[i], 16);
  }
  size_t o_off = 0, o_len = align_up(8 * (size_t)n), o_ord = align_up(o_len + 4 * (size_t)n), o_data = align_up(o_ord + 4 * (size_t)n), o_out = align_up(o_data + data + 16), total = o_out + 32 * (size_t)n;
  CK(e->hb.reserve(total, total / 4));
  uint64_t *so = reinterpret_cast<uint64_t *>(e->hb.h + o_off);
  uint32_t *sl = reinterpret_cast<uint32_t *>(e->hb.h + o_len);
  size_t cur = 0;
  for (uint32_t i = 0; i < n; i++) { so[i] = cur; sl[i] = (uint32_t)len[i]; cur += align_up(len[i], 16); }
  auto fill = [&](uint32_t lo, uint32_t hi) {
    for (uint32_t i = lo; i < hi; i++) {
      uint8_t *dst = e->hb.h + o_data + so[i];
      if (len[i]) memcpy(dst, ptr[i], len[i]);
      const size_t pad = align_up(len[i], 16) - len[i];
      if (pad) memset(dst + len[i], 0, pad);
    }
  };
  threads = std::min<uint32_t>(threads, (uint32_t)(data >> 20) + 1);  // a thread per MiB at most
  if (threads <= 1) fill(0, n);
  else {
    std::vector<std::thread> pool;
    const uint32_t per = (n + threads - 1) / threads;
    for (uint32_t t = 0; t < threads; t++) { const uint32_t lo = t * per, hi = std::min(n, lo + per); if (lo < hi) pool.emplace_back(fill, lo, hi); }
    for (auto &th : pool) th.join();
  }
  // message ids by descending block count, staged behind the lengths
  uint32_t *ord = reinterpret_cast<uint32_t *>(e->hb.h + o_ord);
  for (uint32_t i = 0; i < n; i++) ord[i] = i;
  std::stable_sort(ord, ord + n, [&](uint32_t a, uint32_t b) { return (sl[a] + 8) / 64 > (sl[b] + 8) / 64; });
  CK(cudaMemcpyAsync(e->hb.d, e->hb.h, o_data + data, cudaMemcpyHostToDevice, e->sh));
  const uint64_t *doff = reinterpret_cast<const uint64_t *>(e->hb.d + o_off);
  const uint32_t *dlen = reinterpret_cast<const uint32_t *>(e->hb.d + o_len);
  const uint32_t *dord = reinterpret_cast<const uint32_t *>(e->hb.d + o_ord);
  char *dout = reinterpret_cast<char *>(e->hb.d + o_out);
  launch_hash(e, e->sh, e->hb.d + o_data, doff, dlen, dord, n, dout, 4);  // (a batch takes up to sm_count * 4 CTAs of k_hash2, a pass hash_ctas_per_sm per SM)
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(e->hb.h + o_out, dout, 32 * (size_t)n, cudaMemcpyDeviceToHost, e->sh));
  CK(cudaStreamSynchronize(e->sh));
  memcpy(out32xN, e->hb.h + o_out, 32 * (size_t)n);
  return KR_OK;
}

int kr_hash_batch(kr_engine *e, const uint8_t *bytes, const uint64_t *offsets, uint32_t n, char *out32xN) {
  if (!e || (!bytes && n) || !offsets || (!out32xN && n)) return KR_E_INVALID;
  if (n == 0) return KR_OK;
  std::vector<const uint8_t *> ptr(n);
  std::vector<uint64_t> len(n);
  for (uint32_t i = 0; i < n; i++) {
    if (offsets[i + 1] < offsets[i]) return fail(e, KR_E_INVALID, "offsets must be non-decreasing");
    ptr[i] = bytes + offsets[i]; len[i] = offsets[i + 1] - offsets[i];
  }
  return hash_pieces(e, ptr.data(), len.data(), n, out32xN, 1);
}

// strconv.Atoi: optional sign, decimal digits only, no spaces / underscores, must fit an int
static bool go_atoi(const char *t, uint32_t len, long long &v) {
  if (!t || len == 0 || len > 19) return false;
  uint32_t i = 0;
  bool neg = false;
  if (t[0] == '+' || t[0] == '-') { neg = t[0] == '-'; i = 1; }
  if (i >= len) return false;
  v = 0;
  for (; i < len; i++) { if (t[i] < '0' || t[i] > '9') return false; v = v * 10 + (t[i] - '0'); }
  if (neg) v = -v;
  return true;
}

int kr_hash_compare_batch(kr_engine *e, const kr_hash_compare_row *rows, uint32_t n, uint8_t *equal_out, char *goal_hash_out32xN) {
  if (!e || (!rows && n) || (!equal_out && n)) return KR_E_INVALID;
  if (goal_hash_out32xN) memset(goal_hash_out32xN, 0, 32 * (size_t)n);
  // 1. goal specs -> canonical muted JSON (host), rows that need no hash are settled here
  std::vector<int32_t> msg_of(n, -1);  // row -> message index, -1 = goal hash is ""
  std::vector<std::string> emitted(n);
  std::vector<uint8_t> has_msg(n, 0);
  auto emit_rows = [&](uint32_t lo, uint32_t hi) {  // rows are independent: mute + marshal on as many host threads as the batch is worth
    for (uint32_t i = lo; i < hi; i++) {
      const kr_hash_compare_row &r = rows[i];
      equal_out[i] = 2;  // undecided
      long max_groups = -1;
      if (r.partial) {
        long long ng = 0;
        if (!go_atoi(r.num_worker_groups, r.num_worker_groups_len, ng) || ng < 0 || ng > 0x7FFFFFFF) { equal_out[i] = 1; continue; }  // :1140-1142
        max_groups = (long)ng;
      }
      const int rc = kr_specjson_emit_string(r.goal_spec_json, r.goal_spec_len, true, max_groups, emitted[i], nullptr);
      if (rc == KR_E_STATE) continue;                                   // fewer goal groups than the cluster has: goal hash stays ""
      if (rc != KR_OK) { if (r.partial) equal_out[i] = 1; continue; }   // :1151-1153 / the dropped error of :1135
      has_msg[i] = 1;
    }
  };
  uint32_t emit_threads = 1;
  {
    const uint32_t hw = std::max(1u, std::thread::hardware_concurrency());
    const uint32_t nthreads = std::min<uint32_t>(std::min<uint32_t>(hw, 32u), n / 64u);  // a thread is worth ~64 rows (~2 ms of emitting)
    emit_threads = std::max(1u, nthreads);
    if (nthreads <= 1) emit_rows(0, n);
    else {
      std::vector<std::thread> pool;
      const uint32_t per = (n + nthreads - 1) / nthreads;
      for (uint32_t t = 0; t < nthreads; t++) { const uint32_t lo = t * per, hi = std::min(n, lo + per); if (lo < hi) pool.emplace_back(emit_rows, lo, hi); }
      for (auto &th : pool) th.join();
    }
  }
  std::vector<const uint8_t *> mptr;
  std::vector<uint64_t> mlen;
  for (uint32_t i = 0; i < n; i++) {
    if (!has_msg[i]) continue;
    msg_of[i] = (int32_t)mptr.size();
    mptr.push_back(reinterpret_cast<const uint8_t *>(emitted[i].data()));
    mlen.push_back(emitted[i].size());
  }
  // 2. one GPU batch for every digest (the emitted strings go straight into the pinned staging area)
  const uint32_t nmsg = (uint32_t)mptr.size();
  std::vector<char> digests(32 * (size_t)nmsg);
  if (nmsg) {
    int rc = hash_pieces(e, mptr.data(), mlen.data(), nmsg, digests.data(), emit_threads);
    if (rc) return rc;
  }
  // 3. compare with the annotation
  for (uint32_t i = 0; i < n; i++) {
    if (equal_out[i] != 2) continue;
    const kr_hash_compare_row &r = rows[i];
    const uint32_t clen = r.cluster_hash ? r.cluster_hash_len : 0;
    if (msg_of[i] < 0) { equal_out[i] = clen == 0; continue; }
    const char *d = &digests[32 * (size_t)msg_of[i]];
    if (goal_hash_out32xN) memcpy(goal_hash_out32xN + 32 * (size_t)i, d, 32);
    equal_out[i] = clen == 32 && memcmp(r.cluster_hash, d, 32) == 0;
  }
  return KR_OK;
}

int kr_last_profile(kr_engine *e, kr_profile *prof) {
  if (!e || !prof) return KR_E_INVALID;
  *prof = e->prof;
  return KR_OK;
}

int kr_last_pass(kr_engine *e, kr_pass_report *out) {
  if (!e || !out) return KR_E_INVALID;
  if (!e->has_pass) return fail(e, KR_E_STATE, "no pass has returned KR_OK on this engine");
  *out = e->pass_last;
  return KR_OK;
}

int kr_group_results_device(kr_engine *e, const void **dev_ptr, uint64_t *bytes) {
  if (!e || !dev_ptr || !bytes) return KR_E_INVALID;
  if (!e->ran) return fail(e, KR_E_STATE, "no pass has run");
  *dev_ptr = e->d_out + e->ol.groups;
  *bytes = sizeof(kr_group_result) * (uint64_t)e->sizes.n_groups;
  return KR_OK;
}

int kr_group_results_copy(kr_engine *e, void *dst_device, uint64_t dst_capacity_bytes) {
  if (!e || !dst_device) return KR_E_INVALID;
  if (!e->ran) return fail(e, KR_E_STATE, "no pass has run");
  uint64_t bytes = sizeof(kr_group_result) * (uint64_t)e->sizes.n_groups;
  if (bytes > dst_capacity_bytes) return fail(e, KR_E_CAPACITY, "destination too small (%llu < %llu)", (unsigned long long)dst_capacity_bytes, (unsigned long long)bytes);
  CK(cudaSetDevice(e->cfg.device));
  if (bytes) CK(cudaMemcpyAsync(dst_device, e->d_out + e->ol.groups, bytes, cudaMemcpyDeviceToDevice, e->sm));
  CK(cudaStreamSynchronize(e->sm));
  return KR_OK;
}

const char *kr_last_error(kr_engine *e) { return e ? e->err.c_str() : "null engine"; }

int kr_algorithmic_bytes(kr_engine *e, uint64_t *pass_bytes, uint64_t *hash_bytes, uint64_t *match_bytes) {
  if (!e || !e->begun) return KR_E_INVALID;
  const kr_sizes &n = e->sizes;
  // SURVEY.md §8(d): compulsory traffic only — every input column read once, every output written once
  uint64_t json = 0;
  if (e->committed) {
    kr_snapshot_bufs hb;
    bind_in(e->il, e->h_in, &hb);
    for (uint32_t c = 0; c < n.n_clusters; c++) json += hb.c_json_len[c];
  } else json = n.json_bytes;
  uint64_t hashb = json + 32ull * n.n_clusters;
  uint64_t matchb = 144ull * n.n_clusters - 32ull * n.n_clusters + 56ull * n.n_groups + 4ull * n.n_wtd + 33ull * n.n_pods;
  if (pass_bytes) *pass_bytes = hashb + matchb;
  if (hash_bytes) *hash_bytes = hashb;
  if (match_bytes) *match_bytes = matchb;
  return KR_OK;
}

}  // extern "C"

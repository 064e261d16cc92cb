// kr_packer.cpp — native, event-driven snapshot packer / interner (include/kr_engine.h kr_packer_*; SURVEY §8(f) rank 1: the step
// BEFORE the path).  Host code on top of the single-device C ABI.
//
// The shim's informer handlers (watch set raycluster_controller.go:1525-1533; cache universe internal/managercache/cache.go:16-36)
// call kr_packer_{pod,cluster,job}_{upsert,delete} as events arrive; kr_packer_flush() brings the device copy up to date before an
// epoch.  The packer
//   * interns every string to the u32 ids the engine compares (0 = absent, 1 = ""), and hands them back for the results
//     (kr_packer_string);
//   * keeps the pod table IN the engine's pinned arenas (KR_OPT_FIXED_LAYOUT: columns never move): an Update rewrites the pod's
//     row, a Delete turns it into a free row (KR_PP_TOMBSTONE), an Add takes the lowest free row or appends — and remembers the
//     touched rows, so an epoch uploads exactly those (kr_snapshot_commit_pod_values);
//   * keeps RayCluster scalars in place as well, and rebuilds the small CSR tables (worker groups, workersToDelete names) and
//     the head-aux / RayJob tables only when an event changed them (KR_PART_OBJECTS, ~2 MB at 10 k RayClusters);
//   * re-emits a RayCluster's muted-spec JSON through the native emitter (kr_spec_json_emit) only when metadata.generation
//     moved, compacting the JSON arena when more than half of it is dead (KR_PART_JSON);
//   * stamps every epoch: kr_packer_epoch() / kr_packer_cluster_epoch() give the (podset version, resourceVersion) pair a
//     Reconcile(req) compares before it trusts a record (SURVEY §8(b): "... epoch matches, else fall back").
// Everything an epoch needs beyond the changed rows is already resident in HBM: no per-epoch repack, no per-epoch full upload.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <queue>
#include <string>
#include <string_view>
#include <unordered_map>
#include <vector>

#include "../../include/kr_engine.h"

// kr_specjson.cpp
int kr_specjson_emit_string(const uint8_t *spec_json, uint64_t len, bool muted, long max_groups, std::string &out, long *n_groups);

extern "C" int kr_internal_commit_pod_values_distinct(kr_engine *e, const uint32_t *rows, const uint32_t *values, uint32_t n);  // kr_engine.cu (not in the public header)

namespace {

struct Key { uint32_t a, b; bool operator==(const Key &o) const { return a == o.a && b == o.b; } };
struct KeyHash { size_t operator()(const Key &k) const { return (size_t)(((uint64_t)k.a << 32 | k.b) * 0x9E3779B97F4A7C15ull >> 16); } };

struct GroupRec { uint32_t name_id; int32_t replicas, mn, mx, hosts; uint32_t flags; std::vector<uint32_t> wtd; };
struct ClusterRec {
  uint32_t ns_id, name_id, row;
  uint64_t generation = ~0ull, resource_version = 0;
  std::vector<GroupRec> groups;
  std::string json;     // muted-spec JSON of `generation`
  uint64_t json_off = 0;  // where it sits in the arena
  bool json_placed = false;
};
struct HeadRec { uint32_t ready_reason_id, ready_msg_id, pod_ip_id; uint8_t ready_status, annot_state, version_state; char hash[32]; uint32_t slot; /* its head-aux row */ };

bool go_atoi32(const kr_str &t, int32_t &v) {  // strconv.Atoi on the replica-index label (raycluster_controller.go:857-860)
  if (!t.p || t.n == 0 || t.n > 11) return false;
  uint32_t i = 0;
  bool neg = false;
  if (t.p[0] == '+' || t.p[0] == '-') { neg = t.p[0] == '-'; i = 1; }
  if (i >= t.n) return false;
  long long x = 0;
  for (; i < t.n; i++) { if (t.p[i] < '0' || t.p[i] > '9') return false; x = x * 10 + (t.p[i] - '0'); }
  if (neg) x = -x;
  if (x > 2147483647LL || x < -2147483648LL) return false;
  v = (int32_t)x;
  return true;
}

}  // namespace

struct kr_packer {
  kr_engine *e = nullptr;
  kr_config cap{};
  std::string kuberay_version = "nightly";  // utils.KUBERAY_VERSION (utils/constant.go:281)
  kr_sizes sizes{};
  kr_snapshot_bufs b{};
  std::string err;
  // interner
  std::unordered_map<std::string_view, uint32_t> ids;   // views into `strs` (a deque: elements never move)
  std::deque<std::string> strs;
  // pods
  std::unordered_map<Key, uint32_t, KeyHash> pod_row;     // (ns id, name id) -> row
  std::vector<Key> row_key;                                // row -> key ({0,0}: free)
  std::priority_queue<uint32_t, std::vector<uint32_t>, std::greater<uint32_t>> free_rows;
  std::vector<uint32_t> dirty_rows;
  std::vector<uint8_t> row_dirty;
  std::unordered_map<uint32_t, HeadRec> heads;            // pod row -> head-aux fields
  // clusters (rows in insertion order; a delete moves the last row into the hole)
  std::unordered_map<Key, uint32_t, KeyHash> cluster_row;
  std::vector<ClusterRec> clusters;
  struct JobRec { uint32_t ns_id, name_id, cluster_name_id, summary_id; };
  std::unordered_map<Key, uint32_t, KeyHash> job_row;
  std::vector<JobRec> jobs;
  // what the next flush has to do
  bool first = true, objects_dirty = false, tables_dirty = false, heads_dirty = false, jobs_dirty = false, json_dirty = false;
  uint64_t json_cursor = 0, json_dead = 0;
  uint64_t podset_version = 0, epoch = 0;
  uint32_t last_mode = 0;
  std::vector<uint32_t> stage_vals;   // the epoch's journal: 7 values per entry of dirty_rows
  std::vector<uint32_t> row_slot;     // pod row -> its journal entry (valid while row_dirty)
  uint32_t n_heads_live = 0;          // head-aux rows in use (sizes.n_heads follows at flush)
  kr_sizes engine_sizes{};            // the live counts the engine was last told (kr_snapshot_begin)
  // object rows rewritten in place since the last flush (kr_snapshot_commit_object_rows when no table changed shape)
  std::vector<uint32_t> dirty_cl, dirty_hd;
  std::vector<uint8_t> cl_flag, hd_flag;
  bool wtd_changed = false;           // a workersToDelete name was rewritten in place (same count): the whole object part travels
  // RayClusters whose muted-spec JSON was re-emitted since the last flush (kr_snapshot_commit_spec_rows with KR_OPT_SPEC_ROWS, unless
  // the arena was compacted without KR_OPT_JSON_MOVES or, without KR_OPT_CLUSTER_DELETES, a RayCluster row moved); a deletion moves a
  // row's flag with the row.  A compaction re-places every blob without flagging it.
  std::vector<uint32_t> json_rows;
  std::vector<uint8_t> json_flag;
  bool json_compacted = false, clusters_moved = false;
  // per row, the blob's offset before the first compaction since the last flush (valid while json_compacted): for a RayCluster that
  // kept its row and was not re-emitted, the range the engine holds (KR_OPT_JSON_MOVES moves it from there)
  std::vector<uint64_t> pre_compact_off;
  bool reshaped = false;              // a RayCluster the engine holds changed its group count or a workersToDelete list length (with
                                      // KR_OPT_GROUP_EDITS: a list length, unless KR_OPT_WTD_EDITS as well)
  bool regrouped = false;             // KR_OPT_GROUP_EDITS: a RayCluster the engine holds changed its list of worker groups
  // per row: a RayCluster created in, moved into or (KR_OPT_GROUP_EDITS) regrouped in this row since the last flush (its spec travels
  // after the object part, whose row map tells the engine about it); `fresh_any`: some row is set
  std::vector<uint8_t> fresh;
  bool fresh_any = false;
  void set_fresh(uint32_t row, uint8_t v) {
    if (row >= fresh.size()) fresh.resize((size_t)row + 256, 0);
    fresh[row] = v; fresh_any |= v != 0;
  }
  bool is_fresh(uint32_t row) const { return row < fresh.size() && fresh[row]; }

  uint32_t intern(const kr_str &s) {
    if (!s.p) return KR_ID_ABSENT;
    auto it = ids.find(std::string_view(s.p, s.n));  // no allocation on the hit path
    if (it != ids.end()) return it->second;
    uint32_t id = (uint32_t)strs.size();
    strs.emplace_back(s.p, s.n);
    ids.emplace(std::string_view(strs.back()), id);
    return id;
  }
  uint32_t intern0(const kr_str &s) { return (s.p && s.n) ? intern(s) : 0u; }  // HeadInfo-like fields: "" is encoded as 0
};

namespace {

int pfail(kr_packer *p, int code, const std::string &m) { p->err = m; return code; }

// A touched row gets a slot in the epoch's journal (row list + 7 values per row, what kr_snapshot_commit_pod_values takes): the
// handler has the values in hand, so the flush gathers nothing from the arenas (70 k scattered reads per 10 k rows: 0.3 ms).
uint32_t mark_row(kr_packer *p, uint32_t row) {
  if (row >= p->row_dirty.size()) { p->row_dirty.resize((size_t)row + 1024, 0); p->row_slot.resize(p->row_dirty.size(), 0); }
  if (!p->row_dirty[row]) {
    p->row_dirty[row] = 1; p->row_slot[row] = (uint32_t)p->dirty_rows.size();
    p->dirty_rows.push_back(row); p->stage_vals.resize(7 * p->dirty_rows.size());
  }
  p->podset_version++;
  return p->row_slot[row];
}

void write_pod_row(kr_packer *p, uint32_t row, uint32_t ns, uint32_t cl, uint32_t gr, uint32_t nm, uint32_t packed, int32_t ridx, uint32_t rname) {
  p->b.p_ns_id[row] = ns; p->b.p_cluster_name_id[row] = cl; p->b.p_group_name_id[row] = gr; p->b.p_name_id[row] = nm;
  p->b.p_packed[row] = packed; p->b.p_replica_index[row] = ridx; p->b.p_replica_name_id[row] = rname;
  uint32_t *v = &p->stage_vals[7 * (size_t)mark_row(p, row)];  // (the last write of an epoch wins)
  v[0] = ns; v[1] = cl; v[2] = gr; v[3] = nm; v[4] = packed; v[5] = (uint32_t)ridx; v[6] = rname;
}

// Head-aux rows are dense and STABLE: a head Pod keeps its row while it lives, a new one is appended, a removed one is replaced by
// the last row.  An update rewrites one row in place — nothing is rebuilt at flush, and the engine's on-device diff of the object
// tables sees exactly the rows that changed.
void write_head_row(kr_packer *p, uint32_t h, uint32_t pod_row, const HeadRec &r) {
  if (h >= p->hd_flag.size()) p->hd_flag.resize((size_t)h + 256, 0);
  if (!p->hd_flag[h]) { p->hd_flag[h] = 1; p->dirty_hd.push_back(h); }
  p->b.h_pod_idx[h] = pod_row; p->b.h_ready_status[h] = r.ready_status; p->b.h_ready_reason_id[h] = r.ready_reason_id; p->b.h_ready_msg_id[h] = r.ready_msg_id;
  p->b.h_pod_ip_id[h] = r.pod_ip_id; p->b.h_annot_state[h] = r.annot_state; p->b.h_version_state[h] = r.version_state;
  memcpy(p->b.h_annot_hash + 32 * (size_t)h, r.hash, 32);
}
void remove_head(kr_packer *p, uint32_t pod_row) {
  auto it = p->heads.find(pod_row);
  if (it == p->heads.end()) return;
  const uint32_t h = it->second.slot, last = p->n_heads_live - 1;
  p->heads.erase(it);
  if (h != last) {  // the last row moves into the hole
    const uint32_t moved_pod = p->b.h_pod_idx[last];
    HeadRec &m = p->heads[moved_pod];
    m.slot = h;
    write_head_row(p, h, moved_pod, m);
  }
  p->n_heads_live = last;
  p->heads_dirty = true;
}

// group / workersToDelete CSR + per-cluster offsets, from the cluster records (only when an event changed a group or a name list)
int rebuild_tables(kr_packer *p) {
  uint64_t ng = 0, nw = 0;
  for (auto &c : p->clusters) { ng += c.groups.size(); for (auto &g : c.groups) nw += g.wtd.size(); }
  if (ng > p->cap.max_groups || nw > p->cap.max_wtd) return pfail(p, KR_E_CAPACITY, "kr_packer: worker groups / workersToDelete names exceed the engine capacities");
  uint32_t g = 0, w = 0;
  for (auto &c : p->clusters) {
    p->b.c_group_off[c.row] = g; p->b.c_group_cnt[c.row] = (uint32_t)c.groups.size();
    for (auto &gr : c.groups) {
      p->b.g_cluster_idx[g] = c.row; p->b.g_name_id[g] = gr.name_id; p->b.g_replicas[g] = gr.replicas; p->b.g_min[g] = gr.mn; p->b.g_max[g] = gr.mx;
      p->b.g_num_hosts[g] = gr.hosts; p->b.g_flags[g] = gr.flags; p->b.g_wtd_off[g] = w; p->b.g_wtd_cnt[g] = (uint32_t)gr.wtd.size();
      for (uint32_t id : gr.wtd) p->b.w_name_id[w++] = id;
      g++;
    }
  }
  p->sizes.n_groups = g; p->sizes.n_wtd = w;
  return KR_OK;
}

void mark_emitted(kr_packer *p, uint32_t row) {
  if (row >= p->json_flag.size()) p->json_flag.resize((size_t)row + 256, 0);
  if (!p->json_flag[row]) { p->json_flag[row] = 1; p->json_rows.push_back(row); }
}

// put the cluster's blob at the arena's cursor (16-byte aligned, zero padded); `emitted`: a new blob, not a compaction's
int place_json(kr_packer *p, ClusterRec &c, bool emitted = true) {
  const uint64_t padded = (c.json.size() + 15) & ~15ull;
  if (p->json_cursor + padded > p->cap.max_json_bytes) return KR_E_CAPACITY;
  memcpy(p->b.json + p->json_cursor, c.json.data(), c.json.size());
  memset(p->b.json + p->json_cursor + c.json.size(), 0, padded - c.json.size());
  c.json_off = p->json_cursor; c.json_placed = true;
  p->b.c_json_off[c.row] = c.json_off; p->b.c_json_len[c.row] = (uint32_t)c.json.size();
  p->json_cursor += padded;
  if (emitted) mark_emitted(p, c.row);
  return KR_OK;
}

int compact_json(kr_packer *p) {
  if (!p->json_compacted) {
    p->pre_compact_off.resize(p->clusters.size());
    for (size_t r = 0; r < p->clusters.size(); r++) p->pre_compact_off[r] = p->clusters[r].json_off;
  }
  p->json_cursor = 0; p->json_dead = 0; p->json_compacted = true;
  for (auto &c : p->clusters) if (int rc = place_json(p, c, false)) return pfail(p, rc, "kr_packer: muted-spec JSON exceeds kr_config.max_json_bytes");
  return KR_OK;
}

void rebuild_jobs(kr_packer *p) {
  for (size_t j = 0; j < p->jobs.size(); j++) { p->b.j_ns_id[j] = p->jobs[j].ns_id; p->b.j_cluster_name_id[j] = p->jobs[j].cluster_name_id; p->b.j_summary_id[j] = p->jobs[j].summary_id; }
  p->sizes.n_jobs = (uint32_t)p->jobs.size();
}

}  // namespace

extern "C" {

int kr_packer_create(const kr_config *capacities, kr_packer **out) {
  if (!capacities || !out) return KR_E_INVALID;
  *out = nullptr;
  kr_packer *p = new kr_packer();
  p->cap = *capacities;
  int rc = kr_engine_create(capacities, &p->e);
  if (rc) { delete p; return rc; }
  kr_engine_set_option(p->e, KR_OPT_FIXED_LAYOUT, 1);
  memset(&p->sizes, 0, sizeof p->sizes);
  rc = kr_snapshot_begin(p->e, &p->sizes, &p->b);  // fixed layout: these pointers stay valid for the packer's lifetime
  if (rc) { kr_engine_destroy(p->e); delete p; return rc; }
  p->strs.emplace_back("<absent>"); p->strs.emplace_back("");
  p->ids.emplace(std::string_view(p->strs[1]), 1u);
  *out = p;
  return KR_OK;
}

void kr_packer_destroy(kr_packer *p) { if (!p) return; kr_engine_destroy(p->e); delete p; }
kr_engine *kr_packer_engine(kr_packer *p) { return p ? p->e : nullptr; }
const char *kr_packer_last_error(kr_packer *p) { return p ? (p->err.empty() ? kr_last_error(p->e) : p->err.c_str()) : "null packer"; }
uint32_t kr_packer_intern(kr_packer *p, kr_str s) { return p ? p->intern(s) : 0; }
int kr_packer_string(kr_packer *p, uint32_t id, kr_str *out) {
  if (!p || !out || id >= p->strs.size()) return KR_E_INVALID;
  if (id == KR_ID_ABSENT) { out->p = nullptr; out->n = 0; return KR_OK; }
  out->p = p->strs[id].data(); out->n = (uint32_t)p->strs[id].size();
  return KR_OK;
}
int kr_packer_set_kuberay_version(kr_packer *p, kr_str v) { if (!p || !v.p) return KR_E_INVALID; p->kuberay_version.assign(v.p, v.n); return KR_OK; }

// ---- Pods: Add / Update (the same call) and Delete
int kr_packer_pod_upsert(kr_packer *p, const kr_pod_obj *o) {
  if (!p || !o || !o->ns.p || !o->name.p) return KR_E_INVALID;
  const uint32_t ns = p->intern(o->ns), nm = p->intern(o->name);
  uint32_t row;
  auto it = p->pod_row.find(Key{ns, nm});
  if (it != p->pod_row.end()) row = it->second;
  else {
    if (!p->free_rows.empty()) { row = p->free_rows.top(); p->free_rows.pop(); }
    else {
      if (p->row_key.size() >= p->cap.max_pods) return pfail(p, KR_E_CAPACITY, "kr_packer: more Pods than kr_config.max_pods");
      row = (uint32_t)p->row_key.size(); p->row_key.push_back(Key{0, 0});
    }
    p->pod_row.emplace(Key{ns, nm}, row);
    p->row_key[row] = Key{ns, nm};
  }
  uint32_t packed = ((uint32_t)(o->node_type & 3) << KR_PP_NODE_TYPE_SHIFT) | ((uint32_t)(o->phase & 7) << KR_PP_PHASE_SHIFT) | ((uint32_t)(o->ready_cond & 3) << KR_PP_READY_SHIFT);
  if (o->restart_never) packed |= KR_PP_RESTART_NEVER;
  if (o->ray_terminated) packed |= KR_PP_RAY_TERMINATED;
  if (o->has_deletion_ts) packed |= KR_PP_HAS_DELETION_TS;
  int32_t ridx = 0;
  if (go_atoi32(o->replica_index, ridx)) packed |= KR_PP_HAS_REPLICA_IDX; else ridx = 0;
  write_pod_row(p, row, ns, p->intern(o->cluster), p->intern(o->group), nm, packed, ridx, p->intern(o->replica_name));
  auto hit = p->heads.find(row);
  const bool was_head = hit != p->heads.end();
  if (o->node_type == KR_NT_HEAD) {
    HeadRec h{};
    h.ready_status = o->head_ready_status; h.ready_reason_id = p->intern(o->head_ready_reason); h.ready_msg_id = p->intern(o->head_ready_msg);
    h.pod_ip_id = p->intern0(o->pod_ip);
    if (!o->recreate_hash.p || o->recreate_hash.n == 0) h.annot_state = KR_ANNOT_EMPTY;
    else if (o->recreate_hash.n == 32) { h.annot_state = KR_ANNOT_HASH32; memcpy(h.hash, o->recreate_hash.p, 32); }
    else h.annot_state = KR_ANNOT_OTHER;
    if (!o->kuberay_version.p || o->kuberay_version.n == 0) h.version_state = KR_VER_EMPTY;
    else h.version_state = (o->kuberay_version.n == p->kuberay_version.size() && !memcmp(o->kuberay_version.p, p->kuberay_version.data(), o->kuberay_version.n)) ? KR_VER_CURRENT : KR_VER_DIFFERENT;
    if (!was_head && p->heads.size() >= p->cap.max_heads) return pfail(p, KR_E_CAPACITY, "kr_packer: more head Pods than kr_config.max_heads");
    if (was_head) h.slot = hit->second.slot;
    else h.slot = p->n_heads_live++;
    p->heads[row] = h;
    write_head_row(p, h.slot, row, h);
    p->heads_dirty = true;
  } else if (was_head) remove_head(p, row);
  return KR_OK;
}

int kr_packer_pod_delete(kr_packer *p, kr_str ns, kr_str name) {
  if (!p || !ns.p || !name.p) return KR_E_INVALID;
  auto it = p->pod_row.find(Key{p->intern(ns), p->intern(name)});
  if (it == p->pod_row.end()) return KR_OK;  // not in the cache: nothing to do
  const uint32_t row = it->second;
  p->pod_row.erase(it);
  p->row_key[row] = Key{0, 0};
  write_pod_row(p, row, 0, 0, 0, 0, KR_PP_TOMBSTONE, 0, 0);  // a free row: matches no RayCluster
  p->free_rows.push(row);
  remove_head(p, row);
  return KR_OK;
}

// ---- RayClusters
int kr_packer_cluster_upsert(kr_packer *p, const kr_cluster_obj *o) {
  if (!p || !o || !o->ns.p || !o->name.p) return KR_E_INVALID;
  const uint32_t ns = p->intern(o->ns), nm = p->intern(o->name);
  auto it = p->cluster_row.find(Key{ns, nm});
  uint32_t row;
  if (it == p->cluster_row.end()) {
    if (p->clusters.size() >= p->cap.max_clusters) return pfail(p, KR_E_CAPACITY, "kr_packer: more RayClusters than kr_config.max_clusters");
    row = (uint32_t)p->clusters.size();
    p->clusters.emplace_back();
    p->clusters[row].ns_id = ns; p->clusters[row].name_id = nm; p->clusters[row].row = row;
    p->cluster_row.emplace(Key{ns, nm}, row);
    p->tables_dirty = true;
    p->set_fresh(row, 1);
  } else row = it->second;
  ClusterRec &c = p->clusters[row];
  kr_snapshot_bufs &b = p->b;
  b.c_ns_id[row] = ns; b.c_name_id[row] = nm;
  {  // FNV-1a 64 over the UID (the sharding key, SURVEY §8(e)); without a UID: over "ns/name"
    uint64_t h = 0xCBF29CE484222325ull;
    auto feed = [&](const char *s, uint32_t n) { for (uint32_t i = 0; i < n; i++) { h ^= (uint8_t)s[i]; h *= 0x100000001B3ull; } };
    if (o->uid.p && o->uid.n) feed(o->uid.p, o->uid.n); else { feed(o->ns.p, o->ns.n); feed("/", 1); feed(o->name.p, o->name.n); }
    b.c_uid_hash[row] = h;
  }
  b.c_flags[row] = o->flags; b.c_suspend_status[row] = o->suspend_status; b.c_ext_err_kind[row] = o->ext_err_kind; b.c_ext_err_msg_id[row] = p->intern(o->ext_err_msg);
  b.c_old_state[row] = o->old_state;
  for (int k = 0; k < 5; k++) { b.c_old_counts[5 * (size_t)row + k] = o->old_counts[k]; b.c_old_cond_status[5 * (size_t)row + k] = o->old_cond_status[k]; b.c_old_cond_variant[5 * (size_t)row + k] = o->old_cond_variant[k]; }
  b.c_old_cond_reason_id[row] = p->intern(o->old_head_ready_reason);
  b.c_old_cond_msg_id[2 * (size_t)row] = p->intern(o->old_head_ready_msg); b.c_old_cond_msg_id[2 * (size_t)row + 1] = p->intern(o->old_replica_failure_msg);
  for (int k = 0; k < 4; k++) b.c_old_head_ids[4 * (size_t)row + k] = p->intern0(o->old_head[k]);
  b.c_svc_count[row] = o->svc_count; b.c_svc_ip_kind[row] = o->svc_ip_kind; b.c_svc_ip_id[row] = p->intern0(o->svc_ip); b.c_svc_name_id[row] = p->intern0(o->svc_name);
  b.c_summary_id[row] = p->intern(o->status_summary);
  c.resource_version = o->resource_version;
  p->objects_dirty = true;
  if (row >= p->cl_flag.size()) p->cl_flag.resize((size_t)row + 256, 0);
  if (!p->cl_flag[row]) { p->cl_flag[row] = 1; p->dirty_cl.push_back(row); }
  // worker groups (replicas / expectations / workersToDelete move every few seconds under the autoscaler)
  bool shape = c.groups.size() != o->n_groups, wtd_len = false;
  bool regroup = shape;  // the ordered list of group names changed
  c.groups.resize(o->n_groups);
  for (uint32_t gi = 0; gi < o->n_groups; gi++) {
    const kr_group_obj &g = o->groups[gi];
    GroupRec &r = c.groups[gi];
    const uint32_t name_id = p->intern(g.name);
    regroup |= r.name_id != name_id;
    r.name_id = name_id; r.replicas = g.replicas; r.mn = g.min_replicas; r.mx = g.max_replicas; r.hosts = g.num_hosts; r.flags = g.flags;
    if (r.wtd.size() != g.n_workers_to_delete) wtd_len = true;
    r.wtd.resize(g.n_workers_to_delete);
    for (uint32_t k = 0; k < g.n_workers_to_delete; k++) r.wtd[k] = p->intern(g.workers_to_delete[k]);
  }
  shape |= wtd_len;
  // KR_OPT_GROUP_EDITS: the engine initialises a regrouped RayCluster again in its row (its spec travels after the object part, which
  // always goes whole: the row path takes a renamed group as structural), and with KR_OPT_WTD_EDITS as well it follows list lengths
  uint64_t group_edits = 0, wtd_edits = 0;
  kr_engine_get_option(p->e, KR_OPT_GROUP_EDITS, &group_edits);
  if (group_edits) kr_engine_get_option(p->e, KR_OPT_WTD_EDITS, &wtd_edits);
  if (row < p->engine_sizes.n_clusters && !p->is_fresh(row)) {
    if (group_edits && regroup) { p->set_fresh(row, 1); p->regrouped = true; p->tables_dirty = true; }
    else if (shape && !(group_edits && wtd_edits && !regroup)) p->reshaped = true;
  }
  if (shape || p->tables_dirty) p->tables_dirty = true;
  else {  // same shape: the group rows are rewritten in place
    const uint32_t g0 = b.c_group_off[row];
    for (uint32_t gi = 0; gi < o->n_groups; gi++) {
      const GroupRec &r = c.groups[gi];
      const uint32_t g = g0 + gi;
      b.g_name_id[g] = r.name_id; b.g_replicas[g] = r.replicas; b.g_min[g] = r.mn; b.g_max[g] = r.mx; b.g_num_hosts[g] = r.hosts; b.g_flags[g] = r.flags;
      for (size_t k = 0; k < r.wtd.size(); k++) {
        if (b.w_name_id[b.g_wtd_off[g] + k] != r.wtd[k]) { b.w_name_id[b.g_wtd_off[g] + k] = r.wtd[k]; p->wtd_changed = true; }
      }
    }
  }
  // muted-spec JSON: re-emitted only when metadata.generation moved
  if (c.generation != o->generation || !c.json_placed) {
    std::string js;
    if (o->spec_json_verbatim) js.assign(reinterpret_cast<const char *>(o->spec_json), o->spec_json_len);
    else if (int rc = kr_specjson_emit_string(o->spec_json, o->spec_json_len, true, -1, js, nullptr)) return pfail(p, rc, std::string("kr_packer: ") + kr_spec_json_last_error());
    if (!c.json_placed || js != c.json) {
      if (c.json_placed) p->json_dead += (c.json.size() + 15) & ~15ull;
      c.json.swap(js);
      if (place_json(p, c) != KR_OK) {  // arena full: compact once, then give up
        p->json_dead = 0;
        if (int rc2 = compact_json(p)) return rc2;
        mark_emitted(p, row);  // (the compaction placed the new blob)
      }
      p->json_dirty = true;
    }
    c.generation = o->generation;
  }
  return KR_OK;
}

int kr_packer_cluster_delete(kr_packer *p, kr_str ns, kr_str name) {
  if (!p || !ns.p || !name.p) return KR_E_INVALID;
  auto it = p->cluster_row.find(Key{p->intern(ns), p->intern(name)});
  if (it == p->cluster_row.end()) return KR_OK;
  const uint32_t row = it->second, last = (uint32_t)p->clusters.size() - 1;
  p->json_dead += (p->clusters[row].json.size() + 15) & ~15ull;
  p->cluster_row.erase(it);
  p->clusters_moved = true;
  // the placed-spec flag goes with the RayCluster: the deleted one's is dropped, the moved one's moves to its new row, which is fresh
  auto unplace = [&](uint32_t r) {
    if (r >= p->json_flag.size() || !p->json_flag[r]) return false;
    p->json_flag[r] = 0;
    p->json_rows.erase(std::find(p->json_rows.begin(), p->json_rows.end(), r));
    return true;
  };
  unplace(row);
  if (row != last) {
    if (unplace(last)) { p->json_flag[row] = 1; p->json_rows.push_back(row); }
    p->set_fresh(row, 1);
  }
  p->set_fresh(last, 0);
  if (row != last) {  // the last RayCluster moves into the hole: copy its scalar columns
    ClusterRec moved = std::move(p->clusters[last]);
    moved.row = row;
    p->cluster_row[Key{moved.ns_id, moved.name_id}] = row;
    kr_snapshot_bufs &b = p->b;
#define MV1(f) b.f[row] = b.f[last]
#define MVN(f, k) memcpy(&b.f[(size_t)(k) * row], &b.f[(size_t)(k) * last], sizeof(b.f[0]) * (k))
    MV1(c_ns_id); MV1(c_name_id); MV1(c_uid_hash); MV1(c_flags); MV1(c_suspend_status); MV1(c_ext_err_kind); MV1(c_ext_err_msg_id); MV1(c_json_off); MV1(c_json_len);
    MV1(c_old_state); MVN(c_old_counts, 5); MVN(c_old_cond_status, 5); MVN(c_old_cond_variant, 5); MV1(c_old_cond_reason_id); MVN(c_old_cond_msg_id, 2);
    MVN(c_old_head_ids, 4); MV1(c_svc_count); MV1(c_svc_ip_kind); MV1(c_svc_ip_id); MV1(c_svc_name_id); MV1(c_summary_id);
#undef MV1
#undef MVN
    p->clusters[row] = std::move(moved);
  }
  p->clusters.pop_back();
  p->objects_dirty = p->tables_dirty = true;
  return KR_OK;
}

// ---- RayJobs (roll-up rows: rayjob_controller.go:203-216,343,880-905)
int kr_packer_job_upsert(kr_packer *p, const kr_job_obj *o) {
  if (!p || !o || !o->ns.p || !o->name.p) return KR_E_INVALID;
  const uint32_t ns = p->intern(o->ns), nm = p->intern(o->name);
  auto it = p->job_row.find(Key{ns, nm});
  uint32_t row;
  if (it == p->job_row.end()) {
    if (p->jobs.size() >= p->cap.max_jobs) return pfail(p, KR_E_CAPACITY, "kr_packer: more RayJobs than kr_config.max_jobs");
    row = (uint32_t)p->jobs.size(); p->jobs.emplace_back(); p->job_row.emplace(Key{ns, nm}, row);
  } else row = it->second;
  p->jobs[row] = {ns, nm, (o->cluster_name.p && o->cluster_name.n) ? p->intern(o->cluster_name) : 0u, p->intern(o->status_summary)};
  p->jobs_dirty = true;
  return KR_OK;
}
int kr_packer_job_delete(kr_packer *p, kr_str ns, kr_str name) {
  if (!p || !ns.p || !name.p) return KR_E_INVALID;
  auto it = p->job_row.find(Key{p->intern(ns), p->intern(name)});
  if (it == p->job_row.end()) return KR_OK;
  const uint32_t row = it->second, last = (uint32_t)p->jobs.size() - 1;
  p->job_row.erase(it);
  if (row != last) { p->jobs[row] = p->jobs[last]; p->job_row[Key{p->jobs[row].ns_id, p->jobs[row].name_id}] = row; }
  p->jobs.pop_back();
  p->jobs_dirty = true;
  return KR_OK;
}

// ---- epoch: bring the device copy up to date.  *mode_out: KR_PACK_FULL (everything uploaded: first epoch) or a mask of what moved.
int kr_packer_flush(kr_packer *p, uint32_t *mode_out) {
  if (!p) return KR_E_INVALID;
  p->err.clear();
  static const bool trace = getenv("KR_PACKER_TRACE") != nullptr;  // development aid: where a flush spends its time (stderr)
  auto now = [] { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  const double t0 = trace ? now() : 0;
  double t1 = 0, t2 = 0, t3 = 0;
  if (p->json_dead * 2 > p->json_cursor && p->json_dead > (1u << 20)) { if (int rc = compact_json(p)) return rc; p->json_dirty = true; }
  // Row-granular object commit when nothing changed shape: only the rewritten RayCluster / group / head-aux rows travel.
  bool rows_ok = p->objects_dirty && !p->first && !p->tables_dirty && !p->jobs_dirty && !p->wtd_changed && p->n_heads_live == p->engine_sizes.n_heads;
  if (p->tables_dirty) { if (int rc = rebuild_tables(p)) return rc; p->objects_dirty = true; }
  if (p->heads_dirty) { p->sizes.n_heads = p->n_heads_live; p->objects_dirty = true; }  // (rows were written in place by the handlers)
  if (p->jobs_dirty) { rebuild_jobs(p); p->objects_dirty = true; }
  if (trace) t1 = now();
  kr_sizes want = p->sizes;
  want.n_clusters = (uint32_t)p->clusters.size(); want.n_pods = (uint32_t)p->row_key.size(); want.json_bytes = p->json_cursor;
  kr_snapshot_bufs same;
  p->sizes = want;
  if (want.n_clusters != p->engine_sizes.n_clusters || want.n_groups != p->engine_sizes.n_groups || want.n_wtd != p->engine_sizes.n_wtd || want.n_jobs != p->engine_sizes.n_jobs) rows_ok = false;
  // KR_OPT_CLUSTER_CREATES: RayClusters only appended after the engine's rows (none deleted, none it holds reshaped, the JSON arena
  // not compacted) keep the incremental epoch: the object part, then the new RayClusters' specs as spec rows (no KR_PART_JSON on
  // their account)
  uint64_t creates_opt = 0;
  kr_engine_get_option(p->e, KR_OPT_CLUSTER_CREATES, &creates_opt);
  const uint32_t old_nc = p->engine_sizes.n_clusters;
  // KR_OPT_JSON_MOVES (with KR_OPT_SPEC_ROWS): a compaction travels as moves inside the device arena and keeps every row path below;
  // without it, a compacted arena goes whole
  uint64_t spec_opt = 0, moves_opt = 0;
  kr_engine_get_option(p->e, KR_OPT_SPEC_ROWS, &spec_opt);
  kr_engine_get_option(p->e, KR_OPT_JSON_MOVES, &moves_opt);
  const bool compacted = p->json_compacted && !(moves_opt && spec_opt && !p->first);
  const bool appends = creates_opt && !p->first && !p->clusters_moved && !p->reshaped && !compacted && want.n_clusters > old_nc;
  // KR_OPT_CLUSTER_DELETES: RayClusters deleted by swap-remove (none the engine holds reshaped, the arena not compacted) keep the
  // incremental epoch as well: the kept RayClusters' edited specs as spec rows before the object part, the moved and created ones'
  // after it
  uint64_t deletes_opt = 0;
  kr_engine_get_option(p->e, KR_OPT_CLUSTER_DELETES, &deletes_opt);
  const bool renumbered = deletes_opt && !p->first && p->clusters_moved && !p->reshaped && !compacted;
  // KR_OPT_GROUP_EDITS: RayClusters that changed their worker groups (none reshaped, the arena not compacted, any creation or deletion
  // of the flush on the path above) keep the incremental epoch too: the object part, then their specs as spec rows
  const bool regroups = p->regrouped && !p->first && !p->reshaped && !compacted &&
                        ((want.n_clusters == old_nc && !p->clusters_moved) || appends || renumbered);
  // Row-granular spec commit (KR_OPT_SPEC_ROWS): only the re-emitted blobs travel, while every other one stays where it was.
  const bool spec_ok = spec_opt && p->json_dirty && !p->first && !compacted && !p->clusters_moved && (want.n_clusters == old_nc || appends);
  std::vector<uint32_t> new_rows, old_rows;  // blobs placed this flush: of appended, moved or created RayClusters / of the others
  for (uint32_t r : p->json_rows) (r >= old_nc || p->is_fresh(r) ? new_rows : old_rows).push_back(r);
  // every placed blob travels as a spec row
  const bool json_rows_ok = spec_ok || ((appends || renumbered || regroups) && (old_rows.empty() || spec_opt));
  // A compaction under KR_OPT_JSON_MOVES: the RayClusters the engine holds in the same row, not re-emitted, move where the compaction
  // put them; every created, moved or regrouped RayCluster's spec follows the object part as a spec row (its range changed too)
  const bool moves = p->json_compacted && !compacted && json_rows_ok;
  std::vector<uint32_t> move_rows;
  if (moves) {
    const uint32_t kept = std::min<uint32_t>(old_nc, want.n_clusters);
    for (uint32_t r = 0; r < kept && r < p->pre_compact_off.size(); r++)
      if (!p->is_fresh(r) && !(r < p->json_flag.size() && p->json_flag[r]) && p->pre_compact_off[r] != p->clusters[r].json_off) move_rows.push_back(r);
    new_rows.clear();
    for (uint32_t r = 0; r < want.n_clusters; r++) if (r >= old_nc || p->is_fresh(r)) new_rows.push_back(r);
  }
  if (memcmp(&want, &p->engine_sizes, sizeof want) != 0 || p->first) {
    if (int rc = kr_snapshot_begin(p->e, &p->sizes, &same)) return rc;  // fixed layout: new live counts, same addresses, resident data kept
    p->engine_sizes = want;
  }
  uint32_t mode = 0;
  if (p->first) {
    if (int rc = kr_snapshot_commit(p->e)) return rc;
    mode = KR_PACK_FULL;
  } else {
    if (trace) t2 = now();
    if (moves) {  // (first: the spec-row and object commits below then find the ranges where the host has them)
      if (int rc = kr_snapshot_commit_json_moves(p->e, move_rows.data(), (uint32_t)move_rows.size())) return rc;
      mode |= KR_PACK_JSON_MOVES;
    }
    if (json_rows_ok && !old_rows.empty()) {  // (before the object commit, which would otherwise see the moved ranges and re-hash every RayCluster)
      if (int rc = kr_snapshot_commit_spec_rows(p->e, old_rows.data(), (uint32_t)old_rows.size())) return rc;
      mode |= KR_PACK_SPEC_ROWS;
    }
    uint32_t parts = ((p->objects_dirty && !rows_ok) ? KR_PART_OBJECTS : 0u) | ((p->json_dirty && !json_rows_ok) ? KR_PART_JSON : 0u);
    if (parts) { if (int rc = kr_snapshot_commit_parts(p->e, parts)) return rc; mode |= parts; }
    if (rows_ok) {
      if (int rc = kr_snapshot_commit_object_rows(p->e, p->dirty_cl.data(), (uint32_t)p->dirty_cl.size(), p->dirty_hd.data(), (uint32_t)p->dirty_hd.size())) return rc;
      mode |= KR_PACK_OBJECT_ROWS;
    }
    if (json_rows_ok && !new_rows.empty()) {  // the new RayClusters' specs, once the object part has recorded them as new rows
      if (int rc = kr_snapshot_commit_spec_rows(p->e, new_rows.data(), (uint32_t)new_rows.size())) return rc;
      mode |= KR_PACK_SPEC_ROWS;
    }
    if (trace) t3 = now();
    if (!p->dirty_rows.empty()) {  // the epoch's journal, as the handlers wrote it
      if (int rc = kr_internal_commit_pod_values_distinct(p->e, p->dirty_rows.data(), p->stage_vals.data(), (uint32_t)p->dirty_rows.size())) return rc;
      mode |= KR_PACK_POD_ROWS;
    }
  }
  if (trace) fprintf(stderr, "kr_packer_flush: rebuilds %.0f us, begin %.0f us, commit_parts %.0f us, pod rows (%zu) %.0f us\n", t1 - t0, t2 - t1, t3 - t2, p->dirty_rows.size(), now() - t3);
  for (uint32_t r : p->dirty_rows) p->row_dirty[r] = 0;
  p->dirty_rows.clear(); p->stage_vals.clear();
  for (uint32_t r : p->dirty_cl) p->cl_flag[r] = 0;
  for (uint32_t r : p->dirty_hd) if (r < p->hd_flag.size()) p->hd_flag[r] = 0;
  p->dirty_cl.clear(); p->dirty_hd.clear(); p->wtd_changed = false;
  for (uint32_t r : p->json_rows) p->json_flag[r] = 0;
  p->json_rows.clear(); p->json_compacted = p->clusters_moved = p->reshaped = p->regrouped = false;
  if (p->fresh_any) { std::fill(p->fresh.begin(), p->fresh.end(), 0); p->fresh_any = false; }
  p->first = p->objects_dirty = p->tables_dirty = p->heads_dirty = p->jobs_dirty = p->json_dirty = false;
  p->epoch++;
  p->last_mode = mode;
  if (mode_out) *mode_out = mode;
  return KR_OK;
}

int kr_packer_bufs(kr_packer *p, kr_snapshot_bufs *out) { if (!p || !out) return KR_E_INVALID; *out = p->b; return KR_OK; }
int kr_packer_sizes(kr_packer *p, kr_sizes *out) { if (!p || !out) return KR_E_INVALID; *out = p->sizes; out->n_clusters = (uint32_t)p->clusters.size(); out->n_pods = (uint32_t)p->row_key.size(); out->n_heads = p->n_heads_live; return KR_OK; }
int64_t kr_packer_cluster_row(kr_packer *p, kr_str ns, kr_str name) {
  if (!p || !ns.p || !name.p) return -1;
  auto it = p->cluster_row.find(Key{p->intern(ns), p->intern(name)});
  return it == p->cluster_row.end() ? -1 : (int64_t)it->second;
}
int64_t kr_packer_pod_row(kr_packer *p, kr_str ns, kr_str name) {
  if (!p || !ns.p || !name.p) return -1;
  auto it = p->pod_row.find(Key{p->intern(ns), p->intern(name)});
  return it == p->pod_row.end() ? -1 : (int64_t)it->second;
}
// kr_packer_pod_row without interning the key (kr_group_packer.cpp asks every shard for a Pod that lives on at most one of them:
// the others must not collect its strings).
int64_t kr_internal_packer_find_pod(kr_packer *p, kr_str ns, kr_str name) {
  if (!p || !ns.p || !name.p) return -1;
  auto a = p->ids.find(std::string_view(ns.p, ns.n)), b = p->ids.find(std::string_view(name.p, name.n));
  if (a == p->ids.end() || b == p->ids.end()) return -1;
  auto it = p->pod_row.find(Key{a->second, b->second});
  return it == p->pod_row.end() ? -1 : (int64_t)it->second;
}
int kr_packer_pod_key(kr_packer *p, uint32_t row, kr_str *ns, kr_str *name) {
  if (!p || row >= p->row_key.size() || !ns || !name) return KR_E_INVALID;
  const Key k = p->row_key[row];
  if (k.a == 0 && k.b == 0) { ns->p = name->p = nullptr; ns->n = name->n = 0; return KR_OK; }  // a free row
  ns->p = p->strs[k.a].data(); ns->n = (uint32_t)p->strs[k.a].size(); name->p = p->strs[k.b].data(); name->n = (uint32_t)p->strs[k.b].size();
  return KR_OK;
}
// The epoch a record belongs to: Reconcile(req) trusts the record of `req` only if the RayCluster's resourceVersion in ITS cache
// read equals the one packed here and no Pod event arrived since the flush (podset version) — else it takes the per-object path.
int kr_packer_epoch(kr_packer *p, uint64_t *epoch, uint64_t *podset_version) {
  if (!p) return KR_E_INVALID;
  if (epoch) *epoch = p->epoch;
  if (podset_version) *podset_version = p->podset_version;
  return KR_OK;
}
int kr_packer_cluster_epoch(kr_packer *p, uint32_t cluster_row, uint64_t *resource_version, uint64_t *generation) {
  if (!p || cluster_row >= p->clusters.size()) return KR_E_INVALID;
  if (resource_version) *resource_version = p->clusters[cluster_row].resource_version;
  if (generation) *generation = p->clusters[cluster_row].generation;
  return KR_OK;
}

}  // extern "C"

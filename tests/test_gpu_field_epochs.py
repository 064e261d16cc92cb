"""Incremental epochs one input field at a time: every snapshot column, written alone, on one RayCluster of every class.

Each epoch writes one (field, value) pair into one RayCluster of every class the fleet holds (or into a Pod, group or head-aux row
of it), commits it through one of the entry points that applies, runs the pass against the oracle, and the next epoch reverts the
edit through another entry point.  The field table below states, independently of the engine's own column classes (kObjClass in
kr_engine.cu), which columns force a full pass (the table keys and CSR offsets of DESIGN §4.3; with KR_OPT_WTD_EDITS the
workersToDelete lists no longer do) and which RayClusters an edit may re-decide.  So a wrong entry in the engine's positional
class table, a byte of a 5-byte row the diff misses or a Pod bit k_inc_admit derives differently from k_match2 shows up as a
record that differs from the oracle, as an epoch that was full or incremental against the table, or as a record recomputed that
the table says no input of changed.

Per epoch: the results equal the oracle; the pass is incremental exactly when the table says so; a row commit stays a few KB
unless the header says it falls back to the whole object part (a Recreate bit, a head-aux row count, a workersToDelete list);
the recomputed records lie among the ones the table allows (none for a copy-only column); after the revert every record equals
the one from before the edit.  After each column one more incremental epoch re-matches every Pod of the roles and their partners
and moves a Pod between them; it must equal a fresh engine's full pass, so that what the column's epochs left in the resident
state and no record shows (bucket positions, orphan counts, workersToDelete resolutions) has to be right too.  Every
column must change the oracle's results with at least one of its values, except c_uid_hash, which must change nothing.

On an H100 80GB HBM3 (700 W power limit) the two matrices took 48 s and 52 s of wall time, and this file with
test_gpu_packer_fields.py 104 s."""
import collections
import time

import numpy as np
import pytest

from harness import OBJ_COLS, POD_COLS, Driver, b32, group_pods, head_row, members, run, scale_to, spec_bytes
from kuberay_b200 import abi, synthetic
from kuberay_b200.snapshot import Snapshot

pytestmark = pytest.mark.gpu

N_CLUSTERS = 720
ORD, RC_TRUE, RC_BAD, SUSP, AUTO, MH, LARGE, HUGE, WIDE = range(700, 709)
SMALL_ROLES = (ORD, RC_TRUE, RC_BAD, SUSP, AUTO, MH)
BIG_ROLES = (LARGE, HUGE, WIDE)
LARGE_PODS, HUGE_PODS, WIDE_PODS, WIDE_GROUPS = 600, 8300, 200, 40
MAX_CREATES = 1 << 18
ROW_PATH_BYTES = 40_000  # a row commit of a few RayClusters and head-aux rows; the whole object part of this fleet is ~190 KB
I32_MAX, I32_MIN = 2 ** 31 - 1, -2 ** 31
HEAD_COLS = tuple(name for name, _dt, _m, dim in abi.COLUMNS if dim == "heads")


def partner(r):
    """The ordinary RayCluster (same namespace) an edit of role r may move a Pod, a head-aux key or a workersToDelete name to."""
    return r - 50


# ------------------------------------------------------------------------------------------------ the fleet
class Fleet:
    """The base snapshot, its flags, the roles present and the rows each edit writes: wp (a Running, Ready worker of group 0 with
    a replica index), tp (a worker of group 0 whose ray container terminated, under restartPolicy Always), w0 (the worker group
    0's workersToDelete list names) and the fresh ids no row holds.  The suspended RayCluster carries an external error."""

    def __init__(self, big, oracle):
        snap, flags = synthetic.generate(synthetic.SynthParams(
            n_clusters=N_CLUSTERS, pods_per_cluster=20, groups=3, clusters_per_namespace=N_CLUSTERS, jobs=True, shuffle=False,
            recreate_frac=0.0, suspended_frac=0.0, multihost_frac=0.0, wtd_group_frac=0.0, seed=4242))
        self.roles = SMALL_ROLES + (BIG_ROLES if big else ())
        if big:  # (the donors are the fleet's first rows: clusters 0 .. ~470, far from the roles and their partners)
            synthetic.grow_clusters(snap, [HUGE], HUGE_PODS)
            synthetic.grow_clusters(snap, [HUGE, LARGE], LARGE_PODS)
            synthetic.grow_clusters(snap, [HUGE, LARGE, WIDE], WIDE_PODS)
            snap = synthetic.widen_clusters(snap, [WIDE], WIDE_GROUPS)
        self.next_id = max(int(snap.cols[c].max()) for c in synthetic._ID_COLUMNS if snap.cols[c].size) + 1000
        s = snap
        for r in self.roles + tuple(partner(r) for r in self.roles):
            s.c_flags[r] = (s.c_flags[r] & ~np.uint32(abi.CF_SKIP | abi.CF_SUSPEND | abi.CF_UPGRADE_RECREATE)) | np.uint32(abi.CF_HEAD_EXPECT_OK)
            for gi in range(int(s.c_group_cnt[r])):
                g = int(s.c_group_off[r]) + gi
                n = group_pods(s, r, gi).size
                scale_to(s, g, n + (gi == 0))  # (group 0 creates one Pod: at the lowest free replica index)
                s.g_max[g] = n + 40
                s.g_num_hosts[g] = 1
        self.wp, self.tp, self.w0 = {}, {}, {}
        lists = [[] for _ in range(s.dims["groups"])]
        for r in self.roles:
            rows = group_pods(s, r, 0)
            self.w0[r], self.wp[r], self.tp[r] = int(rows[0]), int(rows[1]), int(rows[2])
            pk = s.p_packed
            for p in (self.wp[r], self.tp[r]):
                pk[p] = np.uint32((abi.NT_WORKER << abi.PP_NODE_TYPE_SHIFT) | (abi.PHASE_RUNNING << abi.PP_PHASE_SHIFT)
                                  | (abi.COND_TRUE << abi.PP_READY_SHIFT) | abi.PP_HAS_REPLICA_IDX)
            pk[self.tp[r]] |= np.uint32(abi.PP_RAY_TERMINATED)  # (healthy under restartPolicy Always; Never makes it one to delete)
            # wp holds the lowest replica index no other Pod of the group holds: the Pod group 0 creates takes it when wp lets go of it
            held = rows[((s.p_packed[rows] & abi.PP_HAS_REPLICA_IDX) != 0) & (rows != self.wp[r]) & (rows != self.tp[r])]
            used = set(s.p_replica_index[held].tolist()) | {1}
            s.p_replica_index[self.wp[r]], s.p_replica_index[self.tp[r]] = min(set(range(len(rows) + 2)) - used), 1
            g0 = int(s.c_group_off[r])
            lists[g0] = [int(s.p_name_id[self.w0[r]]), self.fresh()]   # an own worker and a name no Pod has
            lists[g0 + 1] = [int(s.p_name_id[group_pods(s, r, 1)[0]]), self.fresh()]
            lists[int(s.c_group_off[partner(r)])] = [self.fresh()]
        s = self.snap = snap = _with_lists(s, lists)
        s.c_flags[AUTO] |= np.uint32(abi.CF_AUTOSCALING)
        s.c_flags[SUSP] |= np.uint32(abi.CF_SUSPEND)
        s.c_ext_err_kind[SUSP], s.c_ext_err_msg_id[SUSP] = abi.EXT_ERR_FAILED_CREATE_WORKER_POD, self.fresh()
        for r, true in ((RC_TRUE, True), (RC_BAD, False)):  # Recreate gates: the head carries the spec's digest, or not
            s.c_flags[r] |= np.uint32(abi.CF_UPGRADE_RECREATE)
            h = head_row(s, r)
            d = b32(spec_bytes(s, r))
            s.h_version_state[h], s.h_annot_state[h] = abi.VER_CURRENT, abi.ANNOT_HASH32
            s.h_annot_hash.reshape(-1, 32)[h] = np.frombuffer(d if true else d[::-1], dtype=np.uint8)
        for gi, hosts in ((0, 2), (1, 4)):  # multi-host groups: replicas of `hosts` Pods, each with its replica name and index
            g = int(s.c_group_off[MH]) + gi
            rows = group_pods(s, MH, gi)
            rows = rows[:rows.size // hosts * hosts]
            k = np.arange(rows.size) // hosts
            s.g_num_hosts[g], s.g_replicas[g], s.g_max[g] = hosts, rows.size // hosts + (gi == 0), 6  # (group 0 creates a replica)
            s.p_replica_name_id[rows] = self.next_id + k
            s.p_replica_index[rows] = k
            s.p_packed[rows] |= np.uint32(abi.PP_HAS_REPLICA_IDX)
            self.next_id += int(k.max()) + 1
        self.mh_names = {gi: s.p_replica_name_id[group_pods(s, MH, gi)] for gi in (0, 1)}
        self.owner = np.full(s.dims["pods"], -1, dtype=np.int64)  # the RayCluster each Pod row belongs to in the base snapshot
        for c in range(N_CLUSTERS):
            self.owner[members(s, c)] = c
        flags.fetch_pod_lists = 0
        self.flags = flags
        # the roles' old status is the one this pass computes (a converged RayCluster): an edit of any old-status field shows
        want = oracle.run(s, flags)
        for r in self.roles + tuple(partner(r) for r in self.roles):
            w = want.clusters[r]
            s.c_old_state[r] = w["new_state"]
            s.c_old_counts.reshape(-1, 5)[r] = w["counts"]
            s.c_old_cond_status.reshape(-1, 5)[r] = w["cond_status"][:5]
            s.c_old_cond_variant.reshape(-1, 5)[r] = w["cond_variant"][:5]
            s.c_old_cond_reason_id[r], s.c_old_cond_msg_id[2 * r] = w["head_ready_reason_id"], w["head_ready_msg_id"]
            s.c_old_head_ids.reshape(-1, 4)[r] = w["head_ids"]
        s.c_old_cond_msg_id[2 * SUSP + 1] = s.c_ext_err_msg_id[SUSP]  # (the ReplicaFailure message the error wrote)
        snap.validate()

    def fresh(self):
        self.next_id += 1
        return self.next_id


def _with_lists(snap, lists):
    """`snap` with the workersToDelete lists `lists` (one list of name ids per group row)."""
    d = snap.dims
    cnt = np.array([len(x) for x in lists], dtype=np.uint32)
    out = Snapshot(d["clusters"], d["groups"], int(cnt.sum()), d["pods"], d["heads"], d["jobs"], d["json"])
    for name, _dt, _m, dim in abi.COLUMNS:
        if dim != "wtd":
            out.cols[name][:] = snap.cols[name]
    out.g_wtd_cnt[:] = cnt
    out.g_wtd_off[:] = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.uint32)
    out.w_name_id[:] = np.array([x for lst in lists for x in lst], dtype=np.uint32)
    return out.validate()


def copy_snap(snap):
    d = snap.dims
    out = Snapshot(d["clusters"], d["groups"], d["wtd"], d["pods"], d["heads"], d["jobs"], d["json"])
    for name in snap.cols:
        out.cols[name][:] = snap.cols[name]
    return out


def with_heads(snap, add=(), drop=()):
    """A copy of `snap` whose head-aux table gains a row (a copy of row 0) for each pod of `add` and loses the rows of `drop`."""
    d = snap.dims
    keep = np.setdiff1d(np.arange(d["heads"]), np.asarray(drop, dtype=np.int64))
    out = Snapshot(d["clusters"], d["groups"], d["wtd"], d["pods"], keep.size + len(add), d["jobs"], d["json"])
    for name, _dt, m, dim in abi.COLUMNS:
        a = snap.cols[name]
        if dim == "heads":
            a = a.reshape(d["heads"], m)
            a = np.concatenate([a[keep]] + [a[:1]] * len(add)).reshape(-1)
        out.cols[name][:] = a
    if len(add):
        out.h_pod_idx[keep.size:] = np.asarray(add, dtype=np.uint32)
        out.h_annot_state[keep.size:] = abi.ANNOT_EMPTY
        out.h_annot_hash.reshape(-1, 32)[keep.size:] = 0
    return out.validate()


# ------------------------------------------------------------------------------------------------ the field table
# Case: (column, label, edit(fleet, snap, role) -> snap, may re-decide, columns written besides `column`)
#   may re-decide: "self" the role's RayCluster, "pair" it and partner(role), "prev" it and the RayCluster before it in the table,
#   "none" no record (a copy-only column)
# Expected pass: FULL columns are table keys or CSR offsets (DESIGN §4.3: c_name_id, c_group_off, g_name_id, w_name_id ...); the
# workersToDelete columns are full without KR_OPT_WTD_EDITS and incremental with it; every other column is incremental.
FULL = {"c_ns_id", "c_name_id", "g_name_id"}
WTD = {"g_wtd_off", "g_wtd_cnt", "w_name_id"}
# columns no edit of this file writes alone, and why
NOT_ALONE = {
    "c_group_off": "a CSR offset: moved alone it breaks the group table, which every commit refuses (test_gpu_commit_checks.py)",
    "c_group_cnt": "a CSR count: changed alone it breaks the group table, which every commit refuses (test_gpu_commit_checks.py)",
    "g_cluster_idx": "must name the RayCluster that owns the group row; every commit refuses anything else (test_gpu_commit_checks.py)",
    "c_json_off": "a spec JSON range: test_gpu_spec_rows.py and test_gpu_packer_arena.py edit the ranges and the arena",
    "c_json_len": "a spec JSON range: test_gpu_spec_rows.py and test_gpu_packer_arena.py edit the ranges and the arena",
    "json": "the spec JSON arena: test_gpu_spec_rows.py and test_gpu_packer_arena.py",
    "g_wtd_off": "moves only together with g_wtd_cnt (the lists are stored in group order): the g_wtd_cnt cases write both",
}


def _set(col, value, row_of, elem=None):
    """An edit writing `value` (or value(fleet, snap, role)) into row row_of(fleet, snap, role) of `col` (element `elem` of a
    multi-element row, else every element)."""
    mult = {name: m for name, _dt, m, _d in abi.COLUMNS}[col]

    def edit(f, s, r):
        v = value(f, s, r) if callable(value) else value
        row = row_of(f, s, r)
        a = s.cols[col].reshape(-1, mult)
        if elem is None:
            a[row] = v
        else:
            a[row, elem] = v
        return s
    return edit


def _xor(col, bits, row_of):
    def edit(f, s, r):
        s.cols[col][row_of(f, s, r)] ^= s.cols[col].dtype.type(bits)
        return s
    return edit


cl = lambda f, s, r: r                                            # noqa: E731  the RayCluster row
g0 = lambda f, s, r: int(s.c_group_off[r])                        # noqa: E731  its worker group 0
glast = lambda f, s, r: int(s.c_group_off[r] + s.c_group_cnt[r]) - 1  # noqa: E731  its last group (a slot above 31 when wide)
hd = lambda f, s, r: head_row(s, r)                               # noqa: E731  its head-aux row
job = lambda f, s, r: r                                           # noqa: E731  its RayJob (the fleet's RayJob c points at RayCluster c)
wp = lambda f, s, r: f.wp[r]                                      # noqa: E731
tp = lambda f, s, r: f.tp[r]                                      # noqa: E731
fresh = lambda f, s, r: f.fresh()                                 # noqa: E731


def _other(col, row, elem=None):
    """The value the partner's row holds in `col` (element `elem`, else the first)."""
    mult = {name: m for name, _dt, m, _d in abi.COLUMNS}[col]
    return lambda f, s, r: int(s.cols[col].reshape(-1, mult)[row(f, s, partner(r)), elem or 0])


def _id_values(col, row, elem=None):
    """An id another RayCluster's row holds (already interned), a fresh id, absent (0) and the empty string (1)."""
    at = "" if elem is None else f"[{elem}] "
    return [(at + "other", _set(col, _other(col, row, elem), row, elem)), (at + "fresh", _set(col, fresh, row, elem)),
            (at + "0", _set(col, 0, row, elem)), (at + "1", _set(col, 1, row, elem))]


def _packed(field_shift, width, value):
    def edit(f, s, r):
        p = f.wp[r]
        s.p_packed[p] = (s.p_packed[p] & ~np.uint32(((1 << width) - 1) << field_shift)) | np.uint32(value << field_shift)
        return s
    return edit


def _node_type(frm, to):
    """Pod wp (a worker) or the head Pod becomes node type `to`; a Pod that becomes a head gets a head-aux row, a head Pod that
    stops being one loses its row (as snapshot.pack_objects would lay them out)."""
    def edit(f, s, r):
        p = f.wp[r] if frm == abi.NT_WORKER else int(s.h_pod_idx[head_row(s, r)])
        drop = [head_row(s, r)] if frm == abi.NT_HEAD else []
        s.p_packed[p] = (s.p_packed[p] & ~np.uint32(3)) | np.uint32(to)
        return with_heads(s, add=[p] if to == abi.NT_HEAD else [], drop=drop)
    return edit


def _tombstone(f, s, r):
    p = f.wp[r]
    for c in POD_COLS:
        s.cols[c][p] = 0
    s.p_packed[p] = abi.PP_TOMBSTONE
    return s


def _head_swap(f, s, r):
    """The head-aux keys of the role's head and its partner's trade places (both heads now carry the other's status)."""
    a, b = head_row(s, r), head_row(s, partner(r))
    s.h_pod_idx[a], s.h_pod_idx[b] = s.h_pod_idx[b], s.h_pod_idx[a]
    return s


def _wtd_move(into_next, across=False):
    """The boundary between group 0's and group 1's workersToDelete lists (`across`: the previous RayCluster's last group's and
    group 0's) moves by one name: g_wtd_cnt of both groups and g_wtd_off of the second change together, or the list table
    breaks."""
    def edit(f, s, r):
        g = int(s.c_group_off[r]) - (1 if across else 0)
        d = 1 if into_next else -1  # names that change lists: the last of the first group's, or the first of the second's
        s.g_wtd_cnt[g], s.g_wtd_cnt[g + 1] = int(s.g_wtd_cnt[g]) - d, int(s.g_wtd_cnt[g + 1]) + d
        s.g_wtd_off[g + 1] = int(s.g_wtd_off[g + 1]) - d
        return s
    return edit


def _wtd_name(which):
    def value(f, s, r):
        if which == "own":
            return int(s.p_name_id[f.wp[r]])
        if which == "other group":
            return int(s.p_name_id[group_pods(s, r, 1)[0]])
        if which == "other cluster":
            return int(s.p_name_id[group_pods(s, partner(r), 0)[0]])
        return f.fresh()
    return _set("w_name_id", value, lambda f, s, r: int(s.g_wtd_off[int(s.c_group_off[r])]))


def _pod_name(which):
    """Pod wp takes a name a workersToDelete list holds (and no live Pod has): its own group's, its cluster's group 1's, the
    partner's."""
    def value(f, s, r):
        g = int(s.c_group_off[r if which != "other cluster" else partner(r)]) + (1 if which == "other group" else 0)
        off, cnt = int(s.g_wtd_off[g]), int(s.g_wtd_cnt[g])
        return int(s.w_name_id[off + cnt - 1])
    return _set("p_name_id", value, wp)


def _replica_name(join):
    def value(f, s, r):
        if r == MH:
            names = f.mh_names[0]
            return int(names[-1]) if join else f.fresh()
        return int(s.p_replica_name_id[f.tp[r]]) if join else f.fresh()
    return _set("p_replica_name_id", value, wp)


def _svc_kind(kind):
    def edit(f, s, r):
        s.c_svc_ip_kind[r] = kind
        if kind != abi.SVCIP_NORMAL:
            s.c_svc_ip_id[r] = 0
        return s
    return edit


def _annot(state, digest):
    def edit(f, s, r):
        h = head_row(s, r)
        s.h_annot_state[h] = state
        d = b32(spec_bytes(s, r)) if digest == "true" else (b32(b"other") if digest == "wrong" else b"\0" * 32)
        s.h_annot_hash.reshape(-1, 32)[h] = np.frombuffer(d, dtype=np.uint8)
        return s
    return edit


def _table():
    T = collections.OrderedDict()

    def add(col, cases, dirty="self", also=()):
        T[col] = dict(cases=cases, dirty=dirty, also=also)

    add("c_ns_id", [("other", _set("c_ns_id", lambda f, s, r: int(s.c_ns_id[0]) + 1, cl)), ("fresh", _set("c_ns_id", fresh, cl))])
    add("c_name_id", [("other", _set("c_name_id", _other("c_name_id", cl), cl)), ("fresh", _set("c_name_id", fresh, cl))])
    add("c_uid_hash", [("0", _set("c_uid_hash", 0, cl)), ("max", _set("c_uid_hash", 2 ** 64 - 1, cl)),
                       ("other", _set("c_uid_hash", lambda f, s, r: int(s.c_uid_hash[partner(r)]), cl))], dirty="none")
    add("c_flags", [(f"bit {b}", _xor("c_flags", 1 << b, cl)) for b in range(9)] + [("nil", _set("c_flags", 0, cl))])
    add("c_suspend_status", [(str(v), _set("c_suspend_status", v, cl)) for v in (abi.SUSPEND_NONE, abi.SUSPEND_SUSPENDING, abi.SUSPEND_SUSPENDED)])
    add("c_ext_err_kind", [(str(v), _set("c_ext_err_kind", v, cl)) for v in range(8)])
    add("c_ext_err_msg_id", _id_values("c_ext_err_msg_id", cl))
    add("c_old_state", [(str(v), _set("c_old_state", v, cl)) for v in range(5)])
    add("c_old_counts", [(f"[{k}]={v}", _set("c_old_counts", v, cl, k)) for k in range(5) for v in (-1, 7)] + [("max", _set("c_old_counts", I32_MAX, cl, 4))])
    add("c_old_cond_status", [(f"[{k}]={v}", _set("c_old_cond_status", v, cl, k)) for k in range(abi.NUM_CONDS) for v in range(4)])
    add("c_old_cond_variant", [(f"[{k}]={v}", _set("c_old_cond_variant", v, cl, k)) for k in range(abi.NUM_CONDS)
                               for v in (abi.CV_NONE, abi.CV_PROV_ALL_READY, abi.CV_PROV_PROVISIONING, abi.CV_PROV_SUSPENDED, abi.CV_CANONICAL,
                                         abi.CV_HEAD_FROM_POD, abi.CV_HEAD_NOT_FOUND, abi.CV_OTHER)])
    add("c_old_cond_reason_id", _id_values("c_old_cond_reason_id", cl))
    add("c_old_cond_msg_id", _id_values("c_old_cond_msg_id", cl, 0) + _id_values("c_old_cond_msg_id", cl, 1))
    add("c_old_head_ids", [v for k in range(4) for v in _id_values("c_old_head_ids", cl, k)])
    add("c_svc_count", [(str(v), _set("c_svc_count", v, cl)) for v in (0, 1, 2)])
    add("c_svc_ip_kind", [(str(v), _svc_kind(v)) for v in (abi.SVCIP_NORMAL, abi.SVCIP_EMPTY, abi.SVCIP_NONE)], also=("c_svc_ip_id",))
    add("c_svc_ip_id", _id_values("c_svc_ip_id", cl))
    add("c_svc_name_id", _id_values("c_svc_name_id", cl))
    add("c_summary_id", _id_values("c_summary_id", cl), dirty="none")
    add("g_name_id", [("interned", _set("g_name_id", lambda f, s, r: int(s.c_name_id[partner(r)]), glast)), ("fresh", _set("g_name_id", fresh, g0))])
    add("g_replicas", [(str(v), _set("g_replicas", v, g0)) for v in (0, 3, -1, -7, I32_MAX, I32_MIN, 2 ** 30 + 1)]
        + [("nil", _xor("g_flags", abi.GF_REPLICAS_NIL, g0)), ("last group", _set("g_replicas", 0, glast))], also=("g_flags",))
    add("g_min", [(str(v), _set("g_min", v, g0)) for v in (-1, 0, 5, 250)] + [("nil", _xor("g_flags", abi.GF_MIN_NIL, g0))], also=("g_flags",))
    add("g_max", [(str(v), _set("g_max", v, g0)) for v in (0, 3, -1, 250)] + [("nil", _xor("g_flags", abi.GF_MAX_NIL, g0))], also=("g_flags",))
    add("g_num_hosts", [("2", _set("g_num_hosts", 2, g0)), ("1", _set("g_num_hosts", 1, g0)), ("0", _set("g_num_hosts", 0, g0)),
                        ("-1", _set("g_num_hosts", -1, g0)), ("4", _set("g_num_hosts", 4, glast))])
    add("g_flags", [(f"bit {b}", _xor("g_flags", 1 << b, g0)) for b in range(5)] + [("nil", _set("g_flags", 0, g0)),
                                                                                    ("last group suspended", _xor("g_flags", abi.GF_SUSPEND, glast))])
    add("g_wtd_cnt", [("name to group 1", _wtd_move(True)), ("name to group 0", _wtd_move(False)),
                      ("name to the previous RayCluster", _wtd_move(False, across=True))], dirty="prev", also=("g_wtd_off",))
    add("w_name_id", [(w, _wtd_name(w)) for w in ("own", "other group", "other cluster", "fresh")], dirty="pair")
    add("p_ns_id", [("fresh", _set("p_ns_id", fresh, wp)), ("0", _set("p_ns_id", 0, wp))])
    add("p_cluster_name_id", [("partner", _set("p_cluster_name_id", lambda f, s, r: int(s.c_name_id[partner(r)]), wp)),
                              ("unknown", _set("p_cluster_name_id", fresh, wp)), ("orphan", _set("p_cluster_name_id", 0, wp))], dirty="pair")
    add("p_group_name_id", [("last group", _set("p_group_name_id", lambda f, s, r: int(s.g_name_id[glast(f, s, r)]), wp)),
                            ("unknown", _set("p_group_name_id", fresh, wp)), ("0", _set("p_group_name_id", 0, wp))])
    add("p_name_id", [(w, _pod_name(w)) for w in ("own group", "other group", "other cluster")], dirty="pair")
    add("p_packed", [(f"worker->{t}", _node_type(abi.NT_WORKER, t)) for t in (abi.NT_NONE, abi.NT_HEAD, abi.NT_REDIS)]
        + [(f"head->{t}", _node_type(abi.NT_HEAD, t)) for t in (abi.NT_NONE, abi.NT_WORKER, abi.NT_REDIS)]
        + [(f"phase {v}", _packed(abi.PP_PHASE_SHIFT, 3, v)) for v in range(6)]
        + [(f"ready {v}", _packed(abi.PP_READY_SHIFT, 2, v)) for v in range(4)]
        + [("restart-never", _xor("p_packed", abi.PP_RESTART_NEVER, tp)), ("ray-terminated", _xor("p_packed", abi.PP_RAY_TERMINATED, tp)),
           ("deletion timestamp", _xor("p_packed", abi.PP_HAS_DELETION_TS, wp)), ("has-replica-index", _xor("p_packed", abi.PP_HAS_REPLICA_IDX, wp)),
           ("tombstone", _tombstone)], also=tuple(c for c in POD_COLS if c != "p_packed") + HEAD_COLS)
    add("p_replica_index", [(str(v), _set("p_replica_index", v, wp)) for v in (-1, 1023, 1024, 1025)]
        + [("duplicate", _set("p_replica_index", lambda f, s, r: int(s.p_replica_index[f.tp[r]]), wp))])
    add("p_replica_name_id", [("join", _replica_name(True)), ("new", _replica_name(False))])
    add("h_pod_idx", [("swap with partner", _head_swap)], dirty="pair")
    add("h_ready_status", [(str(v), _set("h_ready_status", v, hd)) for v in range(4)])
    add("h_ready_reason_id", _id_values("h_ready_reason_id", hd))
    add("h_ready_msg_id", _id_values("h_ready_msg_id", hd))
    add("h_pod_ip_id", _id_values("h_pod_ip_id", hd))
    add("h_annot_state", [(f"{st} {d}", _annot(st, d)) for st, d in ((abi.ANNOT_EMPTY, "zero"), (abi.ANNOT_HASH32, "true"),
                                                                     (abi.ANNOT_HASH32, "wrong"), (abi.ANNOT_OTHER, "zero"))], also=("h_annot_hash",))
    add("h_version_state", [(str(v), _set("h_version_state", v, hd)) for v in (abi.VER_EMPTY, abi.VER_CURRENT, abi.VER_DIFFERENT)])
    add("h_annot_hash", [("true", _annot(abi.ANNOT_HASH32, "true")), ("wrong", _annot(abi.ANNOT_HASH32, "wrong")),
                         ("last byte", _xor_byte(31))], also=("h_annot_state",))
    add("j_ns_id", [("fresh", _set("j_ns_id", fresh, job)), ("0", _set("j_ns_id", 0, job))], dirty="none")
    add("j_cluster_name_id", [("other", _set("j_cluster_name_id", lambda f, s, r: int(s.c_name_id[partner(r)]), job)),
                              ("unknown", _set("j_cluster_name_id", fresh, job)), ("0", _set("j_cluster_name_id", 0, job))], dirty="none")
    add("j_summary_id", [("cluster's", _set("j_summary_id", lambda f, s, r: int(s.c_summary_id[r]), job)),
                         ("other", _set("j_summary_id", lambda f, s, r: int(s.c_summary_id[partner(r)]), job)),
                         ("fresh", _set("j_summary_id", fresh, job))], dirty="none")
    return T


def _xor_byte(k):
    def edit(f, s, r):
        h = head_row(s, r)
        s.h_annot_hash.reshape(-1, 32)[h, k] ^= 1
        return s
    return edit


TABLE = _table()


def test_the_field_table_covers_every_column():
    """Not a GPU test in substance (it runs with the file): every column of abi.COLUMNS has cases or a written reason, never both."""
    cols = [name for name, _dt, _m, _d in abi.COLUMNS]
    assert set(TABLE) | set(NOT_ALONE) == set(cols), sorted(set(cols) - set(TABLE) - set(NOT_ALONE))
    assert not set(TABLE) & set(NOT_ALONE)
    assert all(T["cases"] for T in TABLE.values())


# ------------------------------------------------------------------------------------------------ the epochs
ENTRY_OBJECTS, ENTRY_ROWS, ENTRY_POD_ROWS, ENTRY_POD_VALUES = "objects", "object rows", "pod rows", "pod values"


def _diff_rows(a, b):
    """-> (pod rows, RayCluster rows (their own or a group's), head-aux rows) in which b differs from a; dims equal."""
    pods = np.zeros(a.dims["pods"], dtype=bool)
    for c in POD_COLS:
        pods |= a.cols[c] != b.cols[c]
    cls, hds = set(), set()
    for name, _dt, m, dim in abi.COLUMNS:
        if dim not in ("clusters", "groups", "heads"):
            continue
        d = np.flatnonzero((a.cols[name] != b.cols[name]).reshape(-1, m).any(axis=1))
        if dim == "clusters":
            cls.update(d.tolist())
        elif dim == "groups":
            cls.update(int(a.g_cluster_idx[g]) for g in d)
        else:
            hds.update(d.tolist())
    return np.flatnonzero(pods), sorted(cls), sorted(hds)


class Matrix(Driver):
    def __init__(self, fleet, options):
        self.fleet, self.options = fleet, options
        super().__init__(copy_snap(fleet.snap), fleet.flags, slack=1.1, max_creates=MAX_CREATES, **options)
        self.stats = collections.Counter()
        self.live = collections.defaultdict(bool)

    def go(self, new, entry, pod_entry):
        """Move to snapshot `new`, committing the object part through `entry` and the pod rows through `pod_entry`.
        -> whether a row commit had to fall back to the whole object part (a head-aux row count or a Recreate bit moved)."""
        old = self.snap
        fallback = False
        self.shifted = set()
        if new.dims != old.dims:  # a head-aux row came or went: the object part is laid out again
            rows = np.flatnonzero(np.logical_or.reduce([old.cols[c] != new.cols[c] for c in POD_COLS]))
            # the rows behind a dropped or re-inserted one hold another head now: their Pods' RayClusters are re-decided as well
            n = min(old.dims["heads"], new.dims["heads"])
            moved = np.flatnonzero(old.h_pod_idx[:n] != new.h_pod_idx[:n])
            self.shifted = {int(self.fleet.owner[int(p)]) for p in np.concatenate([old.h_pod_idx[moved], new.h_pod_idx[moved]])}
            self.use(new)
            self.commit_objects()
            fallback = True
        else:
            rows, cls, hds = _diff_rows(old, new)
            wtd_moved = any(not np.array_equal(old.cols[c], new.cols[c]) for c in ("w_name_id", "g_wtd_off", "g_wtd_cnt"))
            job_moved = any(not np.array_equal(old.cols[c], new.cols[c]) for c in ("j_ns_id", "j_cluster_name_id", "j_summary_id"))
            self.snap = new
            if entry == ENTRY_ROWS and (cls or hds) and not job_moved and (not wtd_moved or self.options.get("wtd_edits")):
                for c in OBJ_COLS:
                    np.copyto(self.views[c], new.cols[c])
                self.eng.commit_object_rows(cls, hds)
                rc = abi.CF_UPGRADE_RECREATE
                fallback = bool(((old.c_flags & rc) != (new.c_flags & rc)).any()) or wtd_moved
                self.stats["object rows"] += 1
            elif cls or hds or wtd_moved or job_moved:
                self.commit_objects()
                fallback = True
                self.stats["objects"] += 1
        if len(rows):
            self.commit_rows(rows, journal=pod_entry == ENTRY_POD_VALUES)
            self.stats[pod_entry] += 1
        return fallback

    def epoch(self, oracle, new, entry, pod_entry, full, allowed):
        fallback = self.go(new, entry, pod_entry)
        got, _ = self.check(oracle, expect_incremental=not full)
        if not full:
            if entry == ENTRY_ROWS and not fallback:
                assert self.eng.last_profile()["h2d_bytes"] < ROW_PATH_BYTES, self.eng.last_profile()["h2d_bytes"]
            changed = set(got.changed_clusters.tolist()) if got.changed_clusters is not None else set(range(N_CLUSTERS)) if got.n_changed else set()
            allowed = allowed | self.shifted
            assert changed <= allowed, ("records recomputed that no edited input reaches", sorted(changed - allowed))
            if not allowed:
                assert got.n_changed == 0
        self.stats["full" if full else "incremental"] += 1
        return got


def _run_matrix(oracle, big, flag_sets, options):
    t0 = time.time()
    fleet = Fleet(big, oracle)
    dr = Matrix(fleet, options)
    wtd_on = bool(options.get("wtd_edits"))
    try:
        for fs in flag_sets:
            for k, v in fs.items():
                setattr(dr.flags, k, v)
            base = fleet.snap
            dr.go(copy_snap(base), ENTRY_OBJECTS, ENTRY_POD_ROWS)
            base_got, _ = dr.check(oracle, expect_incremental=False)  # (new flags: a full pass)
            n = 0
            for col, T in TABLE.items():
                full = col in FULL or (col in WTD and not wtd_on)
                for label, edit in T["cases"]:
                    new = copy_snap(base)
                    allowed = set()
                    for r in fleet.roles:
                        new = edit(fleet, new, r)
                        allowed |= {"self": {r}, "pair": {r, partner(r)}, "prev": {r, r - 1}, "none": set()}[T["dirty"]]
                    written = {c for c in new.cols if new.cols[c].shape != base.cols[c].shape or not np.array_equal(new.cols[c], base.cols[c])}
                    assert written <= {col, *T["also"]}, (col, label, written)
                    if not written:  # (the value every role holds already)
                        continue
                    _valid(new, fleet)
                    obj = col not in POD_COLS
                    entry, back = (ENTRY_OBJECTS, ENTRY_ROWS) if n % 2 == 0 else (ENTRY_ROWS, ENTRY_OBJECTS)
                    pe, pb = (ENTRY_POD_ROWS, ENTRY_POD_VALUES) if n % 2 == 0 else (ENTRY_POD_VALUES, ENTRY_POD_ROWS)
                    n += 1
                    got = dr.epoch(oracle, new, entry if obj else ENTRY_ROWS, pe, full, allowed)
                    changed_any = bool(base_got.diff(got))
                    dr.live[col] |= changed_any
                    if col == "c_uid_hash":
                        assert not changed_any, (label, base_got.diff(got)[:4])
                    got = dr.epoch(oracle, copy_snap(base), back if obj else ENTRY_ROWS, pb, full, allowed)
                    d = base_got.diff(got)
                    assert not d, (col, label, "the revert left records that differ from the ones before the edit", d[:4])
                # what the column's epochs left in the resident state and no record shows (bucket positions, bucket order, orphan
                # counts, workersToDelete resolutions) is read by one more incremental epoch that re-matches every Pod of every role
                # and partner and moves a Pod from each role to its partner; it must equal a fresh engine's full pass
                probe = _probe(fleet, base)
                near = set(fleet.roles) | {partner(r) for r in fleet.roles}
                got = dr.epoch(oracle, probe, ENTRY_OBJECTS, ENTRY_POD_VALUES, False, near)
                fresh_got, _, _ = run(probe, dr.flags, max_creates=MAX_CREATES, **options)
                d = fresh_got.diff(got)
                assert not d, (col, "a fresh engine's full pass differs", d[:4])
                d = base_got.diff(dr.epoch(oracle, copy_snap(base), ENTRY_OBJECTS, ENTRY_POD_ROWS, False, near))
                assert not d, (col, "the revert of the probe epoch left records that differ", d[:4])
        quiet = {"c_uid_hash"}
        dead = [c for c in TABLE if c not in quiet and not dr.live[c]]
        assert not dead, ("columns none of whose values changed a result", dead)
        print("field epochs", dict(big=big, **options), dict(dr.stats), f"{time.time() - t0:.1f} s")
        for e in (ENTRY_OBJECTS, ENTRY_ROWS, ENTRY_POD_ROWS, ENTRY_POD_VALUES):
            assert dr.stats[e] >= 10, (e, dict(dr.stats))
    finally:
        dr.close()


def _probe(fleet, base):
    """`base` with every Pod of every role and partner flipped to the other Ready status and Pod wp of each role moved into its
    partner (the same worker group name)."""
    s = copy_snap(base)
    for r in fleet.roles:
        for c in (r, partner(r)):
            s.p_packed[members(base, c)] ^= np.uint32(1 << abi.PP_READY_SHIFT)
    for r in fleet.roles:
        s.p_cluster_name_id[fleet.wp[r]] = s.c_name_id[partner(r)]
    _valid(s, fleet)
    return s


def _valid(s, fleet):
    """The edited snapshot is one snapshot.pack_objects could produce: (namespace, name) unique among live Pods, group names unique
    per RayCluster, one head-aux row per head Pod and none for another Pod.  (fuzz_objects also keeps every worker group's
    |expected| at 300 or less, which keeps its create lists small.  That rule is not enforced here: the large and huge RayClusters
    expect more than 300 Pods in the base fleet, and an edit such as numOfHosts 4 on the huge one's last group asks for more; the
    engines have MAX_CREATES room for every create list the table makes.)"""
    live = (s.p_packed & abi.PP_TOMBSTONE) == 0
    key = (s.p_ns_id[live].astype(np.uint64) << np.uint64(32)) | s.p_name_id[live].astype(np.uint64)
    assert np.unique(key).size == key.size, "two live Pods share a namespace and name"
    gk = (s.g_cluster_idx.astype(np.uint64) << np.uint64(32)) | s.g_name_id.astype(np.uint64)
    assert np.unique(gk).size == gk.size, "two worker groups of one RayCluster share a name"
    heads = np.flatnonzero(live & (((s.p_packed >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_HEAD))
    assert np.array_equal(np.sort(s.h_pod_idx), heads), "head-aux rows and head Pods differ"
    s.validate()


GATES_ON = dict(gate_status_conditions=1, gate_multihost_indexing=1, env_random_pod_delete=0)
GATES_OFF = dict(gate_status_conditions=0, gate_multihost_indexing=0, env_random_pod_delete=1)


def test_field_epochs_with_every_option_off(oracle_mod):
    """The ordinary classes only (no large, huge or wide RayCluster): the bucket pipeline with every opt-in option off."""
    _run_matrix(oracle_mod, False, [GATES_ON, GATES_OFF], {})


def test_field_epochs_with_every_option_on(oracle_mod):
    """Every class, large (600 Pods), huge (8 300 Pods) and wide (40 worker groups) among them, with KR_OPT_LARGE_CLUSTERS,
    _HUGE_CLUSTERS, _WIDE_CLUSTERS and _WTD_EDITS on."""
    _run_matrix(oracle_mod, True, [GATES_ON, GATES_OFF], dict(large_clusters=True, huge_clusters=True, wide_clusters=True, wtd_edits=True))

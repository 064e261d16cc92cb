"""Helpers the test files share (no test_ prefix: pytest does not collect it).  Imports nothing that needs a GPU.

  * snapshot edits: rows of a RayCluster or group, pod status, workersToDelete lists, the JSON arena, digests;
  * full passes: one engine per pass (`run`), the engine against the oracle with the full pod lists and with compact results
    (`parity`), and an opt-in option on against off (`parity_on_off`);
  * `Driver`: one engine on a fixed layout through incremental epochs, every pass checked against the oracle and the records the
    pass did not name checked against the previous epoch's; `SpecDriver` adds a twin engine that takes spec edits as KR_PART_JSON;
  * object streams: fuzz objects, the native packer's `Mirror` and its oracle check, informer events, and the epoch loops of the
    native packer and of LiveArena."""
import base64
import collections
import copy
import hashlib

import numpy as np

import fuzz_objects
from kuberay_b200 import abi, synthetic
from kuberay_b200 import snapshot as snp
from kuberay_b200.engine import Engine
from kuberay_b200.packer import Packer
from kuberay_b200.snapshot import Snapshot

POD_COLS = [name for name, _dt, _m, dim in abi.COLUMNS if dim == "pods"]
OBJ_COLS = [name for name, _dt, _m, dim in abi.COLUMNS if dim not in ("pods", "json")]
SORT_KERNELS = {"k_match", "k_place_fused", "k_decide_small", "k_decide"}
BUCKET_KERNELS = {"k_match2", "k_decide2", "k_large_sort", "k_decide_large"}
REBUILD = ("k_inc_wtd_release", "k_inc_wtd_clear", "k_inc_wtd_insert", "k_inc_wtd_resolve")  # the name table rebuilt after a list edit
L_TYPE, L_GROUP, L_CLUSTER = "ray.io/node-type", "ray.io/group", "ray.io/cluster"


# ------------------------------------------------------------------------------------------------ snapshot edits
def members(snap, c):
    """Pod rows of RayCluster c."""
    return np.flatnonzero((snap.p_ns_id == snap.c_ns_id[c]) & (snap.p_cluster_name_id == snap.c_name_id[c]))


def workers(snap, c):
    m = members(snap, c)
    return m[((snap.p_packed[m] >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER]


def group_pods(snap, c, gi):
    """Worker rows of RayCluster c's worker group gi."""
    w = workers(snap, c)
    return w[snap.p_group_name_id[w] == snap.g_name_id[int(snap.c_group_off[c]) + gi]]


def workers_of(snap, g, running=False):
    """Live worker rows of group row g (running: in phase Running only)."""
    c = int(snap.g_cluster_idx[g])
    pk = snap.p_packed
    m = ((pk & abi.PP_TOMBSTONE) == 0) & (((pk >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER) & (snap.p_ns_id == snap.c_ns_id[c]) & \
        (snap.p_cluster_name_id == snap.c_name_id[c]) & (snap.p_group_name_id == snap.g_name_id[g])
    if running:
        m &= ((pk >> abi.PP_PHASE_SHIFT) & 7) == abi.PHASE_RUNNING
    return np.flatnonzero(m)


def head_row(snap, c):
    """The head-aux row of RayCluster c (it must have exactly one)."""
    rows = np.flatnonzero(np.isin(snap.h_pod_idx, members(snap, c)))
    assert rows.size == 1
    return int(rows[0])


def set_phase(snap, rows, phase):
    pk = snap.p_packed
    pk[rows] = (pk[rows] & ~np.uint32(7 << abi.PP_PHASE_SHIFT)) | np.uint32(phase << abi.PP_PHASE_SHIFT)


def flip_ready(snap, rows):
    snap.p_packed[rows] ^= np.uint32(1 << abi.PP_READY_SHIFT)


def move(snap, rows, c):
    """Pods move into RayCluster c's first worker group."""
    snap.p_ns_id[rows], snap.p_cluster_name_id[rows] = snap.c_ns_id[c], snap.c_name_id[c]
    snap.p_group_name_id[rows] = snap.g_name_id[snap.c_group_off[c]]


def scale_to(snap, g, replicas):
    """Group row g asks for `replicas` and nothing else limits it: no minimum or maximum, not suspended, expectations met."""
    snap.g_replicas[g] = replicas
    snap.g_max[g] = 2 ** 31 - 1
    snap.g_min[g] = 0
    snap.g_flags[g] &= ~np.uint32(abi.GF_REPLICAS_NIL | abi.GF_MAX_NIL | abi.GF_MIN_NIL | abi.GF_SUSPEND)
    snap.g_flags[g] |= np.uint32(abi.GF_EXPECT_OK)


def lists_of(snap):
    """The workersToDelete name ids of every group row."""
    off, cnt, w = snap.g_wtd_off, snap.g_wtd_cnt, snap.w_name_id
    return [w[int(off[g]):int(off[g]) + int(cnt[g])].tolist() for g in range(snap.dims["groups"])]


def with_wtd_lists(snap, lists):
    """A copy of `snap` whose workersToDelete lists are `lists` (one list of name ids per group row)."""
    d = snap.dims
    cnt = np.array([len(x) for x in lists], dtype=np.uint32)
    out = Snapshot(d["clusters"], d["groups"], int(cnt.sum()), d["pods"], d["heads"], d["jobs"], d["json"])
    for name, _dt, _m, dim in abi.COLUMNS:
        if dim != "wtd":
            out.cols[name][:] = snap.cols[name]
    out.g_wtd_cnt[:] = cnt
    out.g_wtd_off[:] = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.uint32) if cnt.size else 0
    out.w_name_id[:] = np.array([x for lst in lists for x in lst], dtype=np.uint32)
    return out.validate()


def with_json(snap, json_bytes):
    """A copy of `snap` whose JSON arena holds json_bytes bytes (the old bytes first)."""
    d = snap.dims
    out = Snapshot(d["clusters"], d["groups"], d["wtd"], d["pods"], d["heads"], d["jobs"], json_bytes)
    for name, _dt, _m, dim in abi.COLUMNS:
        if dim != "json":
            out.cols[name][:] = snap.cols[name]
    n = min(json_bytes, d["json"])
    out.json[:n] = snap.json[:n]
    return out


def spec_bytes(snap, c):
    """RayCluster c's muted spec JSON."""
    off, ln = int(snap.c_json_off[c]), int(snap.c_json_len[c])
    return snap.json[off:off + ln].tobytes()


def b32(data: bytes) -> bytes:
    """The base32hex SHA-1 digest KubeRay annotates head Pods with (and the engine returns per RayCluster)."""
    return base64.b32hexencode(hashlib.sha1(data).digest())


# ------------------------------------------------------------------------------------------------ full passes
def compact(flags):
    """A copy of `flags` with kr_flags.fetch_pod_lists = 0: the pass takes the bucket pipeline (kr_bucket2.cuh) when the snapshot
    qualifies and the sort / radix pipeline otherwise; only the compact results come back."""
    f = abi.kr_flags.from_buffer_copy(flags)
    f.fetch_pod_lists = 0
    return f


def grown_fleet(size, n_clusters=300, seed=12):
    """RayClusters of 20 pods (the 64-pod stride); worker pods of the others move into cluster 0 until it lists `size` pods.
    -> (snapshot, compact flags)."""
    n_clusters = max(n_clusters, (size * 3 // 2) // 20 + 1)
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=n_clusters, pods_per_cluster=20, groups=1, seed=seed))
    synthetic.grow_clusters(snap, [0], size)
    assert members(snap, 0).size == size
    return snap, compact(flags)


def kernels(snap, flags, **kw):
    """The kernel names of one profiled pass of a fresh engine (Engine.for_snapshot(snap, **kw)) over `snap`."""
    eng = Engine.for_snapshot(snap, **kw)
    try:
        eng.load(snap)
        return [k for k, _ in eng.reconcile_profiled(flags)["kernels"]]
    finally:
        eng.close()


def parity(snap, flags, oracle, both=False, **kw):
    """Engine vs oracle, twice: with the full pod lists (sort / radix pipeline) and without (bucket pipeline).
    -> the first run's results, or both runs' with `both`."""
    eng = Engine.for_snapshot(snap, **kw)
    try:
        eng.load(snap)
        got = eng.reconcile(flags)
        lean = eng.reconcile(compact(flags))
    finally:
        eng.close()
    want = oracle.run(snap, flags, threads=8)
    d = want.diff(got)
    assert not d, "\n".join(d[:20])
    d = want.diff(lean)
    assert not d, "compact results (fetch_pod_lists = 0):\n" + "\n".join(d[:20])
    assert lean.sorted_pod_idx.size == 0
    return (got, lean) if both else got


def run(snap, flags, profiled=False, max_creates=1 << 16, **options):
    """One fresh engine with `options` (Engine.for_snapshot keywords): a profiled pass first when asked, then a pass.
    -> (results, kernel names of the profiled pass or None, bucket stride).  (The default max_creates holds what drained donor
    RayClusters ask for.)"""
    eng = Engine.for_snapshot(snap, max_creates=max_creates, **options)
    try:
        eng.load(snap)
        names = [k for k, _ in eng.reconcile_profiled(flags)["kernels"]] if profiled else None
        got = eng.reconcile(flags)
        stride = eng.get_option(abi.OPT_BUCKET_STRIDE)
    finally:
        eng.close()
    return got, names, stride


def parity_on_off(snap, flags, oracle, option, **others):
    """Engine with `option` on == oracle == engine with it off (`others` for both); Results.diff covers every result array except
    the run order inside the two arenas and pod_start.  -> (results, kernel names, stride) of the option-on run."""
    on, names, stride = run(snap, flags, profiled=True, **{option: True}, **others)
    off, _, _ = run(snap, flags, **{option: False}, **others)
    d = oracle.run(snap, flags).diff(on)
    assert not d, d[:6]
    d = off.diff(on)
    assert not d, d[:6]
    return on, names, stride


# ------------------------------------------------------------------------------------------------ incremental epochs
def incremental(got, n_clusters):
    """Whether a pass was incremental on the device: it named the records it recomputed, or recomputed fewer than all."""
    return got.changed_clusters is not None or got.n_changed < n_clusters


def room_caps(snap, wtd_room=None, json_room=None):
    """Engine capacities with room to grow: 1.25 x + 16 rows of every table, 4 creates per Pod; the workersToDelete and JSON
    arenas `wtd_room` names / `json_room` bytes past today's size when given."""
    d = snap.dims
    up = lambda x: int(x * 1.25) + 16  # noqa: E731
    return dict(max_clusters=up(d["clusters"]), max_groups=up(d["groups"]),
                max_wtd=up(d["wtd"]) if wtd_room is None else d["wtd"] + wtd_room, max_pods=up(d["pods"]), max_heads=up(d["heads"]),
                max_jobs=up(d["jobs"]), max_creates=4 * d["pods"] + 4096,
                max_json_bytes=up(d["json"]) if json_room is None else d["json"] + json_room)


class Driver:
    """One engine on a fixed layout, committed through the incremental entry points epoch by epoch.

    Capacities: Engine.for_snapshot(snap, slack, max_creates), or room_caps(snap, wtd_room, json_room) when either room is given
    (the layout, and so the bucket stride, follows from the capacities).  `options` are Engine set_* options, set before the
    layout is laid out.  Sets kr_flags.fetch_pod_lists = 0 on `flags`: the bucket pipeline, the one with incremental epochs."""

    def __init__(self, snap, flags, slack=1.0, max_creates=None, wtd_room=None, json_room=None, **options):
        self.snap, self.flags = snap, flags
        flags.fetch_pod_lists = 0
        if wtd_room is None and json_room is None:
            self.eng = Engine.for_snapshot(snap, slack=slack, max_creates=max_creates)
        else:
            self.eng = Engine(0, **room_caps(snap, wtd_room, json_room))
        for k, v in options.items():
            getattr(self.eng, f"set_{k}")(v)
        self.eng.set_fixed_layout(True)
        self.views = self.eng.begin(snap.sizes())
        self.eng.fill(self.views, snap)
        self.eng.commit()
        self.prev = None

    def use(self, new):
        """Make `new` the snapshot (nothing is committed); a layout of other row counts is begun."""
        if new.dims != self.snap.dims:
            self.views = self.eng.begin(new.sizes())
        self.snap = new

    def commit_rows(self, rows, journal=True):
        """The pod rows `rows`: their values (kr_snapshot_commit_pod_values) with `journal`, else the rows of the views."""
        rows = np.unique(np.asarray(rows, dtype=np.uint32))
        for c in POD_COLS:
            self.views[c][rows] = self.snap.cols[c][rows]
        if not rows.size:
            return
        if journal:
            self.eng.commit_pod_values(rows, np.stack([self.snap.cols[c][rows].view(np.uint32) for c in POD_COLS], axis=1))
        else:
            self.eng.commit_pod_rows(rows)

    def commit_objects(self, parts=abi.PART_OBJECTS):
        for c in OBJ_COLS:
            np.copyto(self.views[c], self.snap.cols[c])
        self.eng.commit(parts)

    def set_wtd_lists(self, lists, commit=True):
        """New workersToDelete lists (one per group row), committed with the object part unless told otherwise."""
        self.use(with_wtd_lists(self.snap, lists))
        if commit:
            self.commit_objects()

    def switch(self, new, commit=True):
        """Move to snapshot `new` (same row counts): its object part (unless told otherwise); -> the pod rows that differ."""
        changed = np.zeros(new.dims["pods"], dtype=bool)
        for col in POD_COLS:
            changed |= self.snap.cols[col] != new.cols[col]
        self.snap = new
        if commit:
            self.commit_objects()
        return np.flatnonzero(changed)

    def check(self, oracle, expect_incremental=None, profiled=False, device_only=False):
        """One pass (profiled: kr_reconcile_batch_profiled; device_only: kr_reconcile_device_only; either then kr_results_fetch)
        compared with the oracle.  When it was incremental, the cluster records, action counts and group records of every RayCluster
        it did not name must equal the previous epoch's; with the full pod lists fetched, but for pod_start, which moves with every
        earlier RayCluster's Pod count (the oracle's diff checks it).  -> (results, kernel names of a profiled pass, else [])."""
        names = []
        if profiled:
            names = [k for k, _ in self.eng.reconcile_profiled(self.flags)["kernels"]]
            got = self.eng.fetch()
        elif device_only:
            self.eng.reconcile_device_only(self.flags)
            got = self.eng.fetch()
        else:
            got = self.eng.reconcile(self.flags)
        d = oracle.run(self.snap, self.flags).diff(got)
        assert not d, (d[:6], got.n_changed)
        nc = self.snap.dims["clusters"]
        inc = incremental(got, nc)
        if expect_incremental is not None:
            assert inc == expect_incremental, (inc, got.n_changed, names)
        if inc and self.prev is not None:
            same = np.ones(nc, dtype=bool)
            if got.changed_clusters is not None:
                same[got.changed_clusters] = False
            now, was = got.clusters[same].copy(), self.prev.clusters[same].copy()
            if self.flags.fetch_pod_lists:
                now["pod_start"] = was["pod_start"] = 0
            assert np.array_equal(now, was)
            assert np.array_equal(got.act_cnt[same], self.prev.act_cnt[same])
            gs = same[self.snap.g_cluster_idx]
            assert np.array_equal(got.groups[gs], self.prev.groups[gs])
        self.prev = got
        return got, names

    def close(self):
        self.eng.close()


class SpecDriver(Driver):
    """A Driver committing spec edits row by row (kr_snapshot_commit_spec_rows) and a twin Driver on the same capacities and
    options committing them as KR_PART_JSON; every pass of the first must equal the twin's as well."""

    def __init__(self, snap, flags, json_room=1 << 20, **options):
        super().__init__(snap, flags, json_room=json_room, **options)
        self.twin = Driver(snap, flags, json_room=json_room, **options)
        self.pending, self.edits = set(), {}

    def use(self, new):
        super().use(new)
        self.twin.use(new)

    def edit(self, c, body: bytes, move=False):
        """Rewrite cluster c's muted spec with `body` (applied by apply()): in place when the padded size stays and `move` is not
        asked for, else at a new range at the arena's end."""
        self.edits[int(c)] = (body, move or (len(body) + 15) // 16 != (int(self.snap.c_json_len[c]) + 15) // 16)

    def apply(self):
        if not self.edits:
            return
        end = (self.snap.dims["json"] + 15) // 16 * 16
        grow = sum((len(b) + 15) // 16 * 16 for b, mv in self.edits.values() if mv)
        if grow:
            self.use(with_json(self.snap, end + grow))
        s = self.snap
        for c, (body, mv) in self.edits.items():
            if mv:
                off, end = end, end + (len(body) + 15) // 16 * 16
            else:
                off = int(s.c_json_off[c])
            s.json[off:off + (len(body) + 15) // 16 * 16] = 0
            s.json[off:off + len(body)] = np.frombuffer(body, dtype=np.uint8)
            s.c_json_off[c], s.c_json_len[c] = off, len(body)
            self.pending.add(c)
        self.edits = {}

    def commit_specs(self, rows=None, calls=1):
        """The edited specs: row by row on the first engine (`rows` as given, possibly split over several calls), the whole arena
        plus the object part on the twin."""
        self.apply()
        rows = sorted(self.pending) if rows is None else rows
        np.copyto(self.views["json"], self.snap.json)
        for name in ("c_json_off", "c_json_len"):
            self.views[name][:] = self.snap.cols[name]
        for part in np.array_split(np.asarray(rows, dtype=np.uint32), calls):
            self.eng.commit_spec_rows(part)
        np.copyto(self.twin.views["json"], self.snap.json)
        self.twin.commit_objects(abi.PART_OBJECTS | abi.PART_JSON)
        self.pending.clear()

    def commit_objects(self, parts=abi.PART_OBJECTS, twin=True):
        super().commit_objects(parts)
        if twin:
            self.twin.commit_objects(parts)

    def commit_rows(self, rows):
        super().commit_rows(rows, journal=False)
        self.twin.commit_rows(rows, journal=False)

    def check(self, oracle, expect_incremental=True, profiled=False, h2d=None, h2d_after=None):
        """h2d: the commits' counted bytes before the pass; h2d_after: with the hash order the pass uploaded."""
        if h2d is not None:
            assert self.eng.last_profile()["h2d_bytes"] == h2d
        got, names = super().check(oracle, expect_incremental, profiled)
        if h2d_after is not None:
            assert self.eng.last_profile()["h2d_bytes"] == h2d_after
        d = self.twin.eng.reconcile(self.flags).diff(got)
        assert not d, d[:6]
        return got, names

    def body(self, c):
        return spec_bytes(self.snap, c)

    def close(self):
        super().close()
        self.twin.close()


# ------------------------------------------------------------------------------------------------ object streams
PACKER_CAPS = dict(max_clusters=64, max_groups=512, max_wtd=512, max_pods=4096, max_heads=256, max_jobs=64, max_creates=1 << 16,
                   max_json_bytes=4 << 20)


def stamp(clusters, pods, jobs):
    """Object metadata the informer would carry: generation and resourceVersion of every RayCluster, a name for every RayJob."""
    for i, c in enumerate(clusters):
        c["generation"], c["resourceVersion"] = 1, 100 + i
    for i, j in enumerate(jobs):
        j.setdefault("name", f"rayjob-{i}")
    return clusters, pods, jobs


def objects(seed, **fuzz_kw):
    """fuzz_objects.generate(seed, **fuzz_kw), stamped."""
    return stamp(*fuzz_objects.generate(seed, **fuzz_kw))


class Mirror:
    """The objects behind a native packer, held the way LiveArena holds them (so `events` drives both), every event passed on."""

    def __init__(self, clusters, pods, jobs, packer: Packer):
        self.clusters = {(c.get("namespace", "default"), c["name"]): c for c in clusters}
        self.rows = list(pods)
        self.row_of = {(p.get("namespace", "default"), p["name"]): i for i, p in enumerate(self.rows)}
        self.jobs = list(jobs)
        self.pk = packer
        for c in clusters:
            packer.upsert_cluster(c)
        for p in pods:
            packer.upsert_pod(p)
        for j in jobs:
            packer.upsert_job(j)

    def upsert_pod(self, pod):
        key = (pod.get("namespace", "default"), pod["name"])
        if key in self.row_of:
            self.rows[self.row_of[key]] = pod
        else:  # like the native packer: the lowest free row, else append — so both sides see the same List order
            free = [i for i, p in enumerate(self.rows) if p is None]
            if free:
                self.row_of[key] = free[0]; self.rows[free[0]] = pod
            else:
                self.row_of[key] = len(self.rows); self.rows.append(pod)
        self.pk.upsert_pod(pod)
        assert self.pk.pod_row(*key) == self.row_of[key]

    def delete_pod(self, ns, name):
        i = self.row_of.pop((ns, name), None)
        if i is not None:
            self.rows[i] = None
        self.pk.delete_pod(ns, name)

    def upsert_cluster(self, c):
        self.clusters[(c.get("namespace", "default"), c["name"])] = c
        self.pk.upsert_cluster(c)

    def delete_cluster(self, ns, name):
        self.clusters.pop((ns, name), None)
        self.pk.delete_cluster(ns, name)

    def upsert_job(self, j):
        key = (j.get("namespace", "default"), j["name"])
        keys = [(x.get("namespace", "default"), x["name"]) for x in self.jobs]
        self.jobs = [j if k == key else x for k, x in zip(keys, self.jobs)] + ([] if key in keys else [j])
        self.pk.upsert_job(j)

    def delete_job(self, ns, name):
        self.jobs = [x for x in self.jobs if (x.get("namespace", "default"), x["name"]) != (ns, name)]
        self.pk.delete_job(ns, name)

    def live_pods(self):
        return [p for p in self.rows if p is not None]


ID_FIELDS = ("head_ready_reason_id", "head_ready_msg_id")
PLAIN_FIELDS = ("path", "head_action", "err_kind", "status_err", "new_state", "state_changed", "needs_status_write", "head_update_annotations",
                "stop_after_group", "err_arg", "n_pods", "n_heads", "counts", "cond_status", "cond_variant", "status_flags")


def packer_check(m: Mirror, oracle, lean: bool, run=None):
    """The packer's pass against the oracle on the same objects packed by the Python packer.  Ids and row numbers differ between the
    two (different interning order, free rows), so the records are compared through the strings and Pod keys they stand for.
    `run(flags) -> Results` takes the packer's pass another way than kr_reconcile_batch (default: pk.engine.reconcile).
    -> (oracle results, packer results)."""
    pk = m.pk
    clusters = [m.clusters[k] for k in sorted(m.clusters)]
    pods = m.live_pods()
    snap, meta = snp.pack_objects(clusters, pods, m.jobs)
    flags = meta.flags
    flags.fetch_pod_lists = 0 if lean else 1
    want = oracle.run(snap, flags)
    f2 = pk.flags(fetch_pod_lists=flags.fetch_pod_lists)
    got = (run or pk.engine.reconcile)(f2)
    it = meta.interner
    assert got.n_orphans == want.n_orphans and got.n_actions == want.n_actions and got.n_create_total == want.n_create_total
    for ci, key in enumerate(meta.cluster_keys):
        r = pk.cluster_row(*key)
        assert r >= 0, key
        a, b = want.clusters[ci], got.clusters[r]
        for f in PLAIN_FIELDS:
            assert np.array_equal(a[f], b[f]), (key, f, a[f], b[f])
        for f in ID_FIELDS:
            assert (it.str(int(a[f])) or "") == (pk.string(int(b[f])) or ""), (key, f)
        assert [it.str(int(x)) or "" for x in a["head_ids"]] == [pk.string(int(x)) or "" for x in b["head_ids"]], key
        hp = int(a["head_pod_idx"])
        assert (meta.pod_keys[hp] if hp >= 0 else (None, None)) == (pk.pod_key(int(b["head_pod_idx"])) if int(b["head_pod_idx"]) >= 0 else (None, None))
        assert bytes(want.hash[ci]) == bytes(got.hash[r]), key
        # actions: (pod key, code) in List order (the mirror reuses the lowest free row exactly like the native packer)
        wa = [(meta.pod_keys[int(p)], int(c)) for p, c in zip(*want.actions_of(ci))]
        ga = [(pk.pod_key(int(p)), int(c)) for p, c in zip(*got.actions_of(r))]
        assert wa == ga, (key, wa, ga)
        # worker groups: the native side's group rows follow ITS cluster order, found through the record's group offset
        g0w, g0g = int(snap.c_group_off[ci]), int(pk.column("c_group_off")[r])
        for gi in range(int(snap.c_group_cnt[ci])):
            wg, gg = want.groups[g0w + gi], got.groups[g0g + gi]
            for f in ("expected", "n_list", "n_unhealthy", "n_running", "diff", "n_create", "flags"):
                assert wg[f] == gg[f], (key, gi, f, wg[f], gg[f])
            assert sorted(want.creates_of(g0w + gi).tolist()) == sorted(got.creates_of(g0g + gi).tolist())
    return want, got


def events(rng, live, counter: list, structural: bool):
    """A handful of informer events on a LiveArena or Mirror; `structural` allows the ones that move a table's row count."""
    pods = [p for p in live.rows if p is not None]
    for _ in range(int(rng.integers(1, 8))):
        kind = rng.random()
        workers = [p for p in pods if (p.get("labels") or {}).get(L_TYPE) != "head" and (p["namespace"], p["name"]) in live.row_of]
        if kind < 0.35 and pods:  # status update
            p = copy.deepcopy(pods[int(rng.integers(len(pods)))])
            if (p["namespace"], p["name"]) not in live.row_of:
                continue
            p["phase"] = ["Running", "Pending", "Failed", "Succeeded"][int(rng.integers(4))]
            p["conditions"] = [{"type": "Ready", "status": ["True", "False"][int(rng.integers(2))]}]
            live.upsert_pod(p)
        elif kind < 0.55 and workers:  # pod deleted
            p = workers[int(rng.integers(len(workers)))]
            live.delete_pod(p["namespace"], p["name"])
        elif kind < 0.8 and workers:  # pod created (same labels as an existing worker)
            src = workers[int(rng.integers(len(workers)))]
            counter[0] += 1
            live.upsert_pod({"namespace": src["namespace"], "name": f"new{counter[0]}", "labels": dict(src["labels"]), "phase": "Pending",
                             "restartPolicy": "Always"})
        elif kind < 0.95:  # RayCluster spec / status change that keeps every table's row count
            key = sorted(live.clusters)[int(rng.integers(len(live.clusters)))]
            c = copy.deepcopy(live.clusters[key])
            groups = c["spec"].get("workerGroupSpecs") or []
            if groups:
                g = groups[int(rng.integers(len(groups)))]
                g["replicas"] = int(rng.integers(0, 7))
            c.setdefault("status", {})["readyWorkerReplicas"] = int(rng.integers(0, 5))
            c["expectations"] = {k: bool(rng.random() < 0.9) for k in (c.get("expectations") or {"head": True})}
            live.upsert_cluster(c)
        elif structural:
            heads = [p for p in pods if (p.get("labels") or {}).get(L_TYPE) == "head" and (p["namespace"], p["name"]) in live.row_of]
            if heads and rng.random() < 0.5:
                h = heads[int(rng.integers(len(heads)))]
                live.delete_pod(h["namespace"], h["name"])
            else:
                key = sorted(live.clusters)[int(rng.integers(len(live.clusters)))]
                counter[0] += 1
                live.upsert_pod({"namespace": key[0], "name": f"head{counter[0]}", "labels": {L_CLUSTER: key[1], L_TYPE: "head", L_GROUP: "headgroup"},
                                 "phase": "Running", "conditions": [{"type": "Ready", "status": "True"}], "podIP": "10.9.9.9"})


def autoscale_objects(rng, side, pending):
    """Autoscaler traffic on informer objects (native packer / LiveArena): delete last epoch's named Pods and clear the lists, then
    name 1-3 own workers of one or two groups and lower their replicas."""
    for key, (gname, names) in list(pending.items()):
        for nm in names:
            side.delete_pod(key[0], nm)
        c = copy.deepcopy(side.clusters[key])
        for g in c["spec"].get("workerGroupSpecs") or []:
            if g["groupName"] == gname:
                g["workersToDelete"] = []
        side.upsert_cluster(c)
    pending.clear()
    keys = sorted(side.clusters)
    for _ in range(int(rng.integers(1, 3))):
        key = keys[int(rng.integers(len(keys)))]
        c = copy.deepcopy(side.clusters[key])
        groups = c["spec"].get("workerGroupSpecs") or []
        if not groups:
            continue
        g = groups[int(rng.integers(len(groups)))]
        mine = [p["name"] for p in side.rows if p is not None and p.get("namespace", "default") == key[0] and (p.get("labels") or {}).get(L_CLUSTER) == key[1]
                and (p.get("labels") or {}).get(L_GROUP) == g["groupName"] and (p.get("labels") or {}).get(L_TYPE) != "head"]
        if not mine:
            continue
        names = [mine[i] for i in rng.choice(len(mine), min(len(mine), int(rng.integers(1, 4))), replace=False)]
        g["workersToDelete"] = names
        if isinstance(g.get("replicas"), int):
            g["replicas"] = max(0, g["replicas"] - len(names))
        side.upsert_cluster(c)
        pending[key] = (g["groupName"], names)


def spec_edits(rng, side, gen, k):
    """k RayClusters' specs edited (rayVersion), each with the next generation `gen[0]`; the spec JSON is emitted from then on."""
    keys = sorted(side.clusters)
    for i in rng.choice(len(keys), min(k, len(keys)), replace=False):
        c = copy.deepcopy(side.clusters[keys[int(i)]])
        c.pop("specJson", None)
        c["spec"]["rayVersion"] = "v" + "9" * int(rng.integers(1, 90))
        gen[0] += 1
        c["generation"] = gen[0]
        c["resourceVersion"] = 10_000 + gen[0]
        side.upsert_cluster(c)


def huge_objects(seed, size, n_clusters=80):
    """fuzz_objects' RayClusters copied under new names (with their pods) until there are n_clusters of them (a fleet of a few
    RayClusters with one huge one has a mean size no bucket stride holds), then the workers of the one that has the most cloned
    until it lists `size` pods."""
    clusters, pods, jobs = fuzz_objects.generate(seed, max_clusters=16)
    base, k = list(clusters), 0
    while len(clusters) < n_clusters:
        k += 1
        for c in base:
            q = copy.deepcopy(c)
            q["name"] = f"{c['name']}-x{k}"
            clusters.append(q)
            for p in [p for p in pods if p.get("namespace", "default") == c.get("namespace", "default") and p["labels"].get("ray.io/cluster") == c["name"]]:
                r = copy.deepcopy(p)
                r["name"], r["labels"]["ray.io/cluster"] = f"{p['name']}-x{k}", q["name"]
                pods.append(r)
    owner = most_workers(pods)
    src = [p for p in pods if (p.get("namespace"), p["labels"].get("ray.io/cluster")) == owner and p["labels"].get("ray.io/node-type") == "worker"]
    n_now = sum((p.get("namespace"), p["labels"].get("ray.io/cluster")) == owner for p in pods)
    for i in range(size - n_now):
        q = copy.deepcopy(src[i % len(src)])
        q["name"] = f"{q['name']}-huge-{i}"
        pods.append(q)
    return stamp(clusters, pods, jobs)


def most_workers(pods):
    """(namespace, ray.io/cluster) of the RayCluster with the most worker Pods."""
    return collections.Counter((p.get("namespace"), p["labels"].get("ray.io/cluster")) for p in pods
                               if p["labels"].get("ray.io/node-type") == "worker").most_common(1)[0][0]


def device_incremental(got):
    """Whether a packer's or LiveArena's pass was incremental on the device: it named the records it recomputed, or none changed."""
    return got.changed_clusters is not None or got.n_changed == 0


def packer_stream(m: Mirror, oracle, epochs, step, lean=True):
    """`epochs` epochs through Mirror m's native packer: step(epoch) applies the epoch's events to m, the packer flushes and
    packer_check compares its pass with the oracle (lean: compact results; a callable: by epoch).
    -> (each epoch's results, each flush's mode)."""
    gots, modes = [], []
    for epoch in range(epochs):
        step(epoch)
        modes.append(m.pk.flush())
        _, got = packer_check(m, oracle, lean=lean(epoch) if callable(lean) else lean)
        gots.append(got)
    return gots, modes


def arena_stream(arena, oracle, epochs, step):
    """`epochs` epochs through a LiveArena: step(epoch) applies the epoch's events, the arena flushes and a pass with compact
    results must equal the oracle on the arena's snapshot.  -> each epoch's results."""
    gots = []
    for epoch in range(epochs):
        step(epoch)
        arena.flush()
        flags = arena.meta.flags
        flags.fetch_pod_lists = 0
        got = arena.reconcile(flags)
        d = oracle.run(arena.snap, flags).diff(got)
        assert not d, (epoch, d[:6])
        gots.append(got)
    return gots

"""RayCluster creation, deletion, regrouping and growth together, with every engine option on (KR_OPT_LARGE_CLUSTERS, _WIDE_CLUSTERS,
_HUGE_CLUSTERS, _WTD_EDITS, _SPEC_ROWS, _CLUSTER_CREATES, _CLUSTER_DELETES, _GROUP_EDITS, _LARGE_GROWTH), in the sequences the RayJob
and RayService lifecycles produce: a RayCluster created, scaled past its bucket and its region, regrouped, and deleted while its
neighbours do the same.

A fleet is a "universe" snapshot holding every RayCluster that will ever exist plus the list of live universe rows in row order;
each epoch's snapshot is synthetic.select_clusters(universe, order) (creation appends to the order, deletion is swap-remove), and
the Pods of RayClusters that are not live are orphans.  Every epoch is compared with the oracle; tests/class_model.py's Model
predicts which epochs are incremental (and why the others take the full pass), the stride, every decided RayCluster's Pod count
and, every few epochs, the per-cluster kernels' list; and every RayCluster the pass did not name keeps its records, read through
the epoch's composed row map (new row -> old row, group records at their shifted indices).

Directed cases pin the lifecycles one epoch at a time, among them a deleted large RayCluster in the last row: its region used to
stay on the host's large list past the live rows (the next upload of the region table wrote past its end, and a large and wide one
was decided by the per-cluster kernels with another RayCluster's groups); run_pass now drops such regions before the pass.
The native packer runs the nine options against an all-off twin on one informer stream of creates, deletes, group edits and growth.
On an H100 80GB HBM3 (700 W power limit) the file took 21 s of wall time."""
import collections
import copy
import json

import numpy as np
import pytest

from class_model import Model, counts, owners, region_arena
from harness import (PACKER_CAPS, POD_COLS, SORT_KERNELS, Driver, Mirror, events, incremental, lists_of, members, objects, packer_check,
                     scale_to, with_wtd_lists)
from kuberay_b200 import abi, synthetic
from kuberay_b200.packer import GroupPacker, Packer
from kuberay_b200.snapshot import Snapshot

pytestmark = pytest.mark.gpu

ALL = dict(large_clusters=True, wide_clusters=True, huge_clusters=True, wtd_edits=True, spec_rows=True, cluster_creates=True,
           cluster_deletes=True, group_edits=True, large_growth=True)


def _with_pods(snap, n):
    """A copy of `snap` with n pod rows: rows cut off must be free (KR_PP_TOMBSTONE), rows added are free."""
    d = snap.dims
    assert (snap.p_packed[n:] == abi.PP_TOMBSTONE).all()
    out = Snapshot(d["clusters"], d["groups"], d["wtd"], n, d["heads"], d["jobs"], d["json"])
    k = min(n, d["pods"])
    for name, _dt, _m, dim in abi.COLUMNS:
        if dim == "pods":
            out.cols[name][:k] = snap.cols[name][:k]
            out.cols[name][k:] = abi.PP_TOMBSTONE if name == "p_packed" else 0
        else:
            out.cols[name][:] = snap.cols[name]
    return out.validate()


def _universe(n, live, pods_per_cluster=24, seed=0, wide=(), wtd=0.2, spare_pods=0):
    """n RayClusters of 2 worker groups (healthy, able to scale), the first `live` of them live; `wide`: universe rows of 40 groups;
    `spare_pods` free pod rows at the end."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=n, pods_per_cluster=pods_per_cluster, groups=2, seed=seed, healthy=True,
                                                           wtd_group_frac=wtd, autoscaling_frac=0.3, shuffle=False))
    snap.c_flags[:] &= ~np.uint32(abi.CF_SKIP | abi.CF_SUSPEND)
    for g in range(snap.dims["groups"]):
        scale_to(snap, g, int(snap.g_replicas[g]))
    if wide:
        snap = synthetic.widen_clusters(snap, list(wide), 40)
    if spare_pods:
        snap = _with_pods(snap, snap.dims["pods"] + spare_pods)
    return snap, flags


class Fleet(Driver):
    """One engine with every option on, over a universe and its live order; each epoch is built by edits to the universe (pods,
    groups) and to the order, then committed and checked."""

    def __init__(self, universe, flags, live, oracle, seed, slack=1.4):
        self.uni, self.order, self.oracle = universe, list(live), oracle
        self.rng = np.random.default_rng(seed)
        super().__init__(universe, flags, slack=slack, max_creates=1 << 21, **ALL)
        snap = synthetic.select_clusters(universe, self.order)
        self.use(snap)
        self.commit_objects(abi.PART_ALL)
        for c in POD_COLS:
            self.views[c][:] = snap.cols[c]
        self.eng.commit(abi.PART_ALL)
        self.model = Model(len(self.order), snap.dims["pods"], True, True, huge=True, arena=region_arena(self.eng.cfg.max_pods))
        self.stats, self.seen = collections.Counter(), set()
        self.prev = None
        self.begin()
        self.finish(expect="first pass")

    # ------------------------------------------------------------------------------------------------ edits of one epoch
    def begin(self):
        self.touched, self.regrouped, self.created, self.forced = set(), set(), [], None
        self.reset_layout = self.twice = False
        self.old_order, self.old_snap = list(self.order), self.snap
        self.tags = set()

    def uown(self):
        """Universe row of every pod row's RayCluster (-1: none), live or not."""
        return owners(self.uni)

    def relabel(self, rows, u):
        """Pods move into universe RayCluster u (its first worker group)."""
        s = self.uni
        rows = np.asarray(rows, dtype=np.int64)
        s.p_ns_id[rows], s.p_cluster_name_id[rows] = s.c_ns_id[u], s.c_name_id[u]
        s.p_group_name_id[rows] = s.g_name_id[int(s.c_group_off[u])] if s.c_group_cnt[u] else 0
        self.touched.update(rows.tolist())

    def workers(self, u, own=None):
        s = self.uni
        own = self.uown() if own is None else own
        w = ((s.p_packed >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER
        rows = np.flatnonzero(w & (own == u) & ((s.p_packed & abi.PP_TOMBSTONE) == 0))
        return rows[~np.isin(rows, list(self.touched))]

    def set_count(self, u, target, donors):
        """Universe RayCluster u gains workers of the `donors` (live ordinary RayClusters; as many as they have left) or gives some
        to them.  -> whether it now lists more Pods than its row's bucket and region held (the model's limits before the epoch)."""
        own = self.uown()
        cur = int((own == u).sum())
        if target > cur:
            w = ((self.uni.p_packed >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER
            src = np.flatnonzero(w & np.isin(own, donors) & (own != u))
            src = src[~np.isin(src, list(self.touched))]
            target = min(target, cur + src.size)
            self.relabel(self.rng.choice(src, target - cur, replace=False), u)
        elif target < cur:
            out = self.rng.choice(self.workers(u, own), cur - target, replace=False)
            sinks = [int(d) for d in donors if d != u][:4]
            for i, part in enumerate(np.array_split(out, 4)):
                if part.size:
                    self.relabel(part, sinks[i])
        assert int((self.uown() == u).sum()) == target
        if u not in self.order:
            return False
        row = self.order.index(u)
        return target > (self.model.limits()[row] if row < self.model.nc else self.model.stride)

    def flip(self, k):
        """k readiness flips on random live workers."""
        own = self.uown()
        live = np.flatnonzero(np.isin(own, self.order))
        rows = self.rng.choice(live, min(k, live.size), replace=False)
        self.uni.p_packed[rows] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        self.touched.update(rows.tolist())

    def create(self, u):
        assert u not in self.order
        self.order.append(u)
        self.created.append(u)

    def delete(self, u):
        i = self.order.index(u)
        self.order = [self.order[j] for j in synthetic.swap_remove_order(len(self.order), [i])]

    def shrink_pods(self, k):
        """The last k pod rows (free) leave the pod table: fewer pod rows than the resident state holds, so kr_snapshot_begin lays
        the layout out again (first stride, no region)."""
        self.uni = _with_pods(self.uni, self.uni.dims["pods"] - k)
        self.reset_layout = True

    def regroup(self, u, pairs):
        """Universe RayCluster u has the worker groups `pairs` ((source group row, name id or None), regroup_clusters)."""
        self.uni = synthetic.regroup_clusters(self.uni, {u: pairs})
        self.regrouped.add(u)

    def groups(self, u):
        g0 = int(self.uni.c_group_off[u])
        return [(g, None) for g in range(g0, g0 + int(self.uni.c_group_cnt[u]))]

    def fresh_id(self, k=0):
        cols = ("g_name_id", "p_group_name_id", "p_name_id", "w_name_id", "c_name_id", "p_cluster_name_id")
        return max(int(self.uni.cols[c].max()) for c in cols if self.uni.cols[c].size) + 1 + k

    # ------------------------------------------------------------------------------------------------ commit and check
    def finish(self, expect=None, profiled=False, device_only=False):
        """Commit the epoch (object part and created RayClusters' specs when the order or a group list changed, then the touched pod
        rows), predict it with the model, run and check it.  expect: a cause of a full pass the caller knows of (an option, flags).
        -> (results, whether it was incremental, the model's cause)."""
        old, m = self.old_snap, self.model
        new = synthetic.select_clusters(self.uni, self.order)
        n = len(self.order)
        pos_old = {u: i for i, u in enumerate(self.old_order)}
        # the composed row map: new row -> old row (-1: created, or regrouped: initialised again in its row)
        old_rows = np.array([pos_old.get(u, -1) if u not in self.regrouped and u not in self.created else -1 for u in self.order], dtype=np.int64)
        structural = self.order != self.old_order or bool(self.regrouped)
        self.use(new)
        if structural:
            self.commit_objects()
            if self.twice:  # a second object commit of the same part (no further row map: the epoch stays as it was)
                self.commit_objects()
                self.tags.add("two object commits")
            rows = [self.order.index(u) for u in self.created]
            if rows:
                np.copyto(self.views["json"][:new.dims["json"]], new.json)
                self.eng.commit_spec_rows(np.asarray(sorted(rows), dtype=np.uint32))
        self.commit_rows(sorted(self.touched), journal=bool(self.rng.integers(2)))
        own, own_old = owners(new), owners(old)
        cnt, groups = counts(new, own), new.c_group_cnt.astype(np.int64)
        # the model's cause of a full pass, most certain first
        cause = expect
        if self.reset_layout:
            m.nc, m.n_pods = n, new.dims["pods"]
            m.reset()
            cause = "layout reset"
        if cause is None and not m.valid:
            cause = "sort pipeline"
        if cause is None and structural:
            kept = [i for i, u in enumerate(self.order) if old_rows[i] == i]
            gone = sorted(set(range(len(self.old_order))) - set(kept))
            init = [i for i in range(n) if old_rows[i] != i]
            adopt = bool(self.created) and self.prev is not None and self.prev.n_orphans > 0
            cause = m.row_map(gone, len(gone) + len(init), len(self.created), adopt)
        if cause is None:
            # peak records: a kept row's records of the last pass plus the Pods that joined it; an initialised row admits every Pod
            t = np.asarray(sorted(self.touched), dtype=np.int64)
            to_new = np.full(max(len(self.old_order), 1), -1, dtype=np.int64)
            for i in range(n):
                if old_rows[i] >= 0:
                    to_new[old_rows[i]] = i
            was = np.where(own_old[t] >= 0, to_new[np.maximum(own_old[t], 0)], -1) if t.size else t
            arrive = t[(own[t] >= 0) & (own[t] != was)] if t.size else t
            prev_cnt = counts(old, own_old)
            peak = np.where(old_rows >= 0, prev_cnt[np.maximum(old_rows, 0)], 0) + np.bincount(own[arrive], minlength=n)
            peak = np.where(old_rows >= 0, peak, cnt)
            m.nc = n
            cause = m.grow(peak, groups)
        got, _ = self.run(profiled, device_only)
        inc = incremental(got, n)
        assert inc == (cause is None), (cause, inc, self.tags, dict(self.stats))
        decided = got.clusters["path"] != abi.PATH_SKIPPED
        assert np.array_equal(got.clusters["n_pods"][decided], cnt[decided])
        if inc and self.prev is not None:
            self.kept_records(got, old, new, old_rows)
        if not inc:
            m.n_pods = new.dims["pods"]
            m.full_pass(cnt, groups)
        assert self.eng.get_option(abi.OPT_BUCKET_STRIDE) == m.stride, (self.eng.get_option(abi.OPT_BUCKET_STRIDE), m.stride, cause)
        self.stats["epochs"] += 1
        self.stats["incremental" if inc else f"full: {cause}"] += 1
        for tag in self.tags:
            self.seen.add(tag)
        self.prev = got
        return got, inc, cause

    def run(self, profiled, device_only):
        self.prev, prev = None, self.prev  # (Driver.check compares rows in place: kept_records reads them through the map instead)
        got, names = self.check(self.oracle, profiled=profiled, device_only=device_only)
        self.prev = prev
        return got, names

    def kept_records(self, got, old, new, old_rows):
        """Every RayCluster the pass did not name keeps its previous records: cluster record, action count and digest from its old row,
        group records from its old group indices.  One rule for rows kept in place, moved and shifted by a regroup before them."""
        prev = self.prev
        ch = set(got.changed_clusters.tolist()) if got.changed_clusters is not None else set()
        for c in range(new.dims["clusters"]):
            o = int(old_rows[c])
            if o < 0 or c in ch:
                continue
            assert got.clusters[c].tobytes() == prev.clusters[o].tobytes(), (c, o)
            assert got.act_cnt[c] == prev.act_cnt[o], (c, o)
            assert bytes(got.hash[c]) == bytes(prev.hash[o]), (c, o)
            g_new, g_old, G = int(new.c_group_off[c]), int(old.c_group_off[o]), int(new.c_group_cnt[c])
            assert G == int(old.c_group_cnt[o]), (c, o)
            assert got.groups[g_new:g_new + G].tobytes() == prev.groups[g_old:g_old + G].tobytes(), (c, o)

    def kernels(self):
        """A profiled pass without changes: which pipeline ran, and the per-cluster kernels when the model lists any."""
        names = {k for k, _ in self.eng.reconcile_profiled(self.flags)["kernels"]}
        self.prev = self.eng.fetch()
        m, groups = self.model, self.snap.c_group_cnt.astype(np.int64)
        if m.valid:
            assert not SORT_KERNELS & names, names
            per = m.per_cluster_list(groups)
            huge = {c for c in m.caps if m.stride + m.caps[c] > abi.LARGE_MAX_PODS}
            assert ("k_large_sort" in names) == bool(per - huge), (names, per)
            assert ("k_huge_tiles" in names) == bool(huge), (names, huge)
        assert self.eng.get_option(abi.OPT_BUCKET_STRIDE) == m.stride
        self.stats["kernel checks"] += 1

    def epoch(self, **kw):
        got = self.finish(**kw)
        self.begin()
        return got


# ------------------------------------------------------------------------------------------------ directed cases
def _fleet(seed, n=420, live=360, wide=(), pods_per_cluster=24, spare_pods=0):
    snap, flags = _universe(n, live, pods_per_cluster, seed=seed, wide=wide, spare_pods=spare_pods)
    return snap, flags, list(range(live))


@pytest.fixture
def fleet_of(oracle_mod):
    made = []

    def make(seed, **kw):
        snap, flags, live = _fleet(seed, **kw)
        f = Fleet(snap, flags, live, oracle_mod, seed)
        made.append(f)
        return f
    yield make
    for f in made:
        f.close()


def test_rayjob_lifecycle(fleet_of):
    """A RayJob's RayCluster: created, grown 20 -> 300 -> 1 200 Pods over three epochs, deleted while in the last row (the full pass),
    then another RayCluster grows, then a new one is created into that row, then an ordinary epoch."""
    f = fleet_of(1)
    donors = np.arange(0, 200)
    job = 360
    f.create(job)
    f.epoch()
    assert f.order[-1] == job
    for size in (300, 1200):
        f.set_count(job, size, donors)
        got, inc, _ = f.epoch()
        assert inc and got.clusters["n_pods"][len(f.order) - 1] == size
    assert len(f.order) - 1 in f.model.caps
    f.delete(job)  # the last row, with a region
    _, inc, cause = f.epoch()
    assert not inc and cause == "large gone row"
    f.set_count(250, 400, donors)  # a growth merge: the next pass uploads the region table
    _, inc, _ = f.epoch()
    assert inc
    f.flip(20)
    _, inc, _ = f.epoch()
    assert inc
    f.create(361)  # into the row the RayJob's RayCluster held
    f.flip(20)
    _, inc, _ = f.epoch()
    assert inc
    f.flip(20)
    _, inc, _ = f.epoch()
    assert inc


def test_large_and_wide_in_the_last_row_deleted(fleet_of):
    """A RayCluster both large (a region) and wide (40 groups) in the last row, deleted: the full pass that follows must not decide
    it with the groups of the RayClusters laid out after the relayout, and the epochs after it stay incremental."""
    f = fleet_of(2, wide=(359,))
    donors = np.arange(0, 200)
    f.set_count(359, 700, donors)
    _, inc, _ = f.epoch()
    assert inc and 359 in f.model.caps
    f.delete(359)
    _, inc, cause = f.epoch()
    assert not inc and cause == "large gone row"
    for k in range(3):
        f.flip(30)
        if k == 1:
            f.set_count(100, 300, donors[donors != 100])
        _, inc, _ = f.epoch()
        assert inc


def test_layout_reset_past_a_large_row(fleet_of):
    """A layout reset (fewer pod rows: kr_snapshot_begin lays the arenas out again) in the epoch that deletes a large RayCluster in the
    last row forgets every region.  The next RayCluster to grow gets its region at the start of the arena, where the forgotten one
    lay; then the deleted key is created again in its old row and adopts its 700 orphaned Pods, more than its bucket holds: it must
    start without a region (its row's entry of the device table is zero) and grow one of its own."""
    f = fleet_of(5, spare_pods=64)
    donors = np.arange(0, 200)
    f.set_count(359, 700, donors)
    _, inc, _ = f.epoch()
    assert inc and 359 in f.model.caps
    f.delete(359)
    f.shrink_pods(64)
    _, inc, cause = f.epoch()
    assert not inc and cause == "layout reset" and not f.model.caps
    f.set_count(100, 700, donors)
    _, inc, _ = f.epoch()
    assert inc and f.model.offs[100] == 0
    f.flip(30)  # (the growth's upload of the region table, of 359 rows, comes with this epoch's pass: none with the next one)
    _, inc, _ = f.epoch()
    assert inc
    f.create(359)
    got, inc, _ = f.epoch()
    assert inc and got.clusters["n_pods"][359] == 700 and f.model.offs[359] == f.model.caps[100]
    f.flip(30)
    _, inc, _ = f.epoch()
    assert inc


def test_rayservice_update(fleet_of):
    """RayService in place: A gains a worker group and B is created; then A is deleted (the last row moves into its hole) while B
    outgrows its bucket in the same epoch."""
    f = fleet_of(3)
    donors = np.arange(0, 150)
    a, b = 200, 360
    g0 = int(f.uni.c_group_off[a])
    f.regroup(a, f.groups(a) + [(g0, f.fresh_id())])
    f.create(b)
    _, inc, _ = f.epoch()
    assert inc
    f.delete(a)
    f.set_count(b, 150, donors)
    got, inc, _ = f.epoch()
    assert inc and got.clusters["n_pods"][f.order.index(b)] == 150
    f.flip(25)
    _, inc, _ = f.epoch()
    assert inc


def test_recreated_key_adopts_past_its_bucket(fleet_of):
    """X deleted; in the next epoch X is created again and adopts more of its orphaned Pods than its bucket holds."""
    f = fleet_of(4)
    donors = np.arange(0, 150)
    x = 300
    f.set_count(x, 120, donors)
    _, inc, _ = f.epoch()
    assert inc and f.order.index(x) in f.model.caps
    f.delete(x)  # (a middle row with a region: the full pass, and the RayCluster moved into the row keeps the region)
    _, inc, cause = f.epoch()
    assert not inc and cause == "large gone row"
    f.create(x)
    got, inc, _ = f.epoch()
    assert inc and got.clusters["n_pods"][f.order.index(x)] == 120


# ------------------------------------------------------------------------------------------------ randomised streams
NEED_EVENTS = {"create", "create wide", "create adopting", "re-create", "delete last", "delete middle", "delete wide", "delete large",
               "regroup append", "regroup remove", "regroup rename", "regroup reorder", "regroup 0-1", "regroup 32-33", "grow stride",
               "grow region", "grow created", "grow moved", "grow regrouped", "grow many", "promote past the list cap", "scale down",
               "create with workersToDelete", "two object commits"}


def _stream_epoch(f, rng, donors, deleted, pool, wide_pool):
    """Several structural events on top of Pod traffic."""
    m = f.model
    f.flip(int(rng.integers(5, 40)))
    n_events = int(rng.integers(1, 4))
    for _ in range(n_events):
        live = [u for u in f.order if u not in donors and u != wide_pool]
        kind = rng.choice(["create", "delete", "regroup", "grow", "shrink"], p=[0.25, 0.2, 0.2, 0.25, 0.1])
        if kind == "create":
            cands = [u for u in pool if u not in f.order and u not in deleted]
            if deleted and rng.random() < 0.3:
                u = deleted.pop(int(rng.integers(len(deleted))))
                f.tags.add("re-create")
            elif cands:
                u = cands[int(rng.integers(len(cands)))]
            else:
                continue
            f.create(u)
            f.tags.add("create")
            g0 = int(f.uni.c_group_off[u])
            if f.uni.g_wtd_cnt[g0:g0 + int(f.uni.c_group_cnt[u])].sum():
                f.tags.add("create with workersToDelete")
            if f.uni.c_group_cnt[u] > 32:
                f.tags.add("create wide")
            if (f.uown() == u).any():
                f.tags.add("create adopting")
            if rng.random() < 0.4 and f.set_count(u, max(int((f.uown() == u).sum()), m.stride) + int(rng.integers(1, 60)), donors):
                f.tags.add("grow created")  # (it grows past its bucket in the epoch that creates it)
        elif kind == "delete" and len(live) > 20:
            row = {"last": len(f.order) - 1, "middle": int(rng.integers(len(f.order) // 2, len(f.order) - 1))}[rng.choice(["last", "middle"])]
            u = f.order[row]
            if u in donors or u in f.created or u in f.regrouped:
                continue
            f.tags.add("delete last" if row == len(f.order) - 1 else "delete middle")
            if f.uni.c_group_cnt[u] > 32:
                f.tags.add("delete wide")
            if row in m.caps:
                f.tags.add("delete large")
            moved = f.order[-1]
            f.delete(u)
            deleted.append(u)
            if moved != u and rng.random() < 0.5 and moved not in donors and moved != wide_pool:  # the RayCluster moved into the hole grows
                if f.set_count(moved, max(int((f.uown() == moved).sum()), m.stride) + int(rng.integers(1, 60)), donors):
                    f.tags.add("grow moved")
        elif kind == "regroup":
            u = live[int(rng.integers(len(live)))]
            if u in f.regrouped or u in f.created:
                continue
            gs = f.groups(u)
            how = rng.choice(["append", "remove", "rename", "reorder", "zero", "wide"])
            if how == "append" or (how in ("remove", "reorder") and len(gs) < 2):
                gs = gs + [(gs[0][0], f.fresh_id())] if gs else [(int(f.uni.c_group_off[0]), f.fresh_id())]
                f.tags.add("regroup append")
            elif how == "remove":
                gs = gs[:-1]
                f.tags.add("regroup remove")
            elif how == "rename":
                gs = [(gs[0][0], f.fresh_id())] + gs[1:]
                f.tags.add("regroup rename")
            elif how == "reorder":
                gs = gs[::-1]
                f.tags.add("regroup reorder")
            elif how == "zero":
                gs = [] if len(gs) == 1 else gs[:1] if gs else [(int(f.uni.c_group_off[donors[0]]), f.fresh_id())]
                f.tags.add("regroup 0-1")
            else:  # 32 <-> 33 on the cluster kept at 32 groups
                u = wide_pool
                if u not in f.order or u in f.regrouped:
                    continue
                gs = f.groups(u)
                gs = gs[:32] if len(gs) == 33 else gs + [(gs[0][0], f.fresh_id())]
                f.tags.add("regroup 32-33")
            f.regroup(u, gs)
            if rng.random() < 0.3 and u in f.order and f.order.index(u) not in m.caps:
                if f.set_count(u, max(int((f.uown() == u).sum()), m.stride) + int(rng.integers(1, 60)), donors):
                    f.tags.add("grow regrouped")
        elif kind == "grow":
            u = live[int(rng.integers(len(live)))]
            cur = int((f.uown() == u).sum())
            row = f.order.index(u)
            region = row in m.caps and rng.random() < 0.5
            tgt = m.stride + m.caps[row] + int(rng.integers(1, 60)) if region else max(cur, m.stride) + int(rng.integers(1, 60))
            if tgt < 1500 and f.set_count(u, tgt, donors):
                f.tags.add("grow region" if region else "grow stride")
        else:
            big = [u for u in live if f.order.index(u) in m.caps]
            if big:
                u = big[int(rng.integers(len(big)))]
                f.set_count(u, int(rng.integers(40, 200)), donors)
                f.tags.add("scale down")


WIDE32 = 300  # the universe RayCluster that goes between 32 and 33 worker groups


def _scheduled(f, e, donors, deleted):
    """Events a stream must reach whatever its dice say, on top of the epoch's random ones."""
    m = f.model
    quiet = [u for u in f.order if u not in donors and u != WIDE32 and u not in f.created and u not in f.regrouped]
    fresh = [u for u in (401, 450, 500) if u not in f.order and u not in deleted]
    if e == 3 and fresh:
        f.create(fresh[0])  # 40 worker groups
        f.tags.add("create wide")
    if e == 20 and deleted:
        f.create(deleted.pop(0))
        f.tags.add("re-create")
    big = [u for u in quiet if f.order.index(u) in m.caps and int((f.uown() == u).sum()) < 900]
    if e in (5, 15, 25) and big:
        u = big[0]
        if f.set_count(u, m.stride + m.caps[f.order.index(u)] + 20, donors):
            f.tags.add("grow region")
    wide = [u for u in quiet if f.uni.c_group_cnt[u] > 32]
    if e == 8 and wide:
        u = wide[-1]
        f.tags.add("delete wide")
        f.tags.add("delete large" if f.order.index(u) in m.caps else "delete last" if u == f.order[-1] else "delete middle")
        f.delete(u)
        deleted.append(u)
    multi = [u for u in quiet if 2 <= f.uni.c_group_cnt[u] <= 32]
    if e in (10, 12, 14) and multi:
        u, gs = multi[0], f.groups(multi[0])
        f.regroup(u, {10: gs[::-1], 12: gs[:-1], 14: [(gs[0][0], f.fresh_id())] + gs[1:]}[e])
        f.tags.add({10: "regroup reorder", 12: "regroup remove", 14: "regroup rename"}[e])
    if e == 16 and WIDE32 in f.order and WIDE32 not in f.regrouped:
        gs = f.groups(WIDE32)
        f.regroup(WIDE32, gs[:32] if len(gs) == 33 else gs + [(gs[0][0], f.fresh_id())])
        f.tags.add("regroup 32-33")
    if e == 19 and len(multi) > 1 and multi[1] not in f.regrouped:
        f.regroup(multi[1], f.groups(multi[1])[:1])
        f.tags.add("regroup 0-1")
    if e == 22 and len(quiet) > 2 and f.order[-1] in quiet and f.order[-1] != quiet[0]:
        moved = f.order[-1]
        f.delete(quiet[0])
        deleted.append(quiet[0])
        f.tags.add("delete middle")
        if f.set_count(moved, max(int((f.uown() == moved).sum()), m.stride) + 20, donors):
            f.tags.add("grow moved")
    if e in (13, 27) and big and big[-1] in f.order and big[-1] not in f.regrouped:
        u = big[-1]
        f.tags.add("delete large")
        f.delete(u)
        deleted.append(u)


def _run_stream(seed, oracle_mod, epochs=40):
    snap, flags = _universe(640, 480, 32, seed=9000 + seed, wide=(401, 501, 550, 600))
    snap = synthetic.widen_clusters(snap, [WIDE32], 32)
    lists = lists_of(snap)  # every third RayCluster yet to be created names one of its own Pods in workersToDelete
    for u in range(480, 640, 3):
        lists[int(snap.c_group_off[u])].append(int(snap.p_name_id[members(snap, u)[-1]]))
    snap = with_wtd_lists(snap, lists)
    f = Fleet(snap, flags, list(range(480)), oracle_mod, seed)
    try:
        rng = f.rng
        donors = np.arange(0, 320)
        pool = list(range(480, 640))
        deleted = []
        promoted = []
        for e in range(epochs):
            expect = None
            if e in (1, 2):
                # 64 RayClusters just past the stride: every one newly listed, so the per-cluster list (the wide RayClusters are on it)
                # would pass max(KR_GROW_LIST_MIN, n / KR_GROW_LIST_DIV); then those 64 and one more past the wider stride the full
                # pass left: more than KR_GROW_MAX at once
                if not promoted:
                    promoted = [u for i, u in enumerate(f.order) if u >= 320 and i not in f.model.caps and u != WIDE32 and f.uni.c_group_cnt[u] <= 32]
                grown = sum(f.set_count(u, max(f.model.stride + 1, int((f.uown() == u).sum()) + 1), donors) for u in promoted[:64 + e - 1])
                if grown == 64 + e - 1:
                    f.tags.add("promote past the list cap" if e == 1 else "grow many")
            else:
                _stream_epoch(f, rng, donors, deleted, pool, WIDE32)
                _scheduled(f, e, donors, deleted)
                f.twice = e % 5 == 4
            if e in (17, 18):  # the process flags change, and change back
                f.flags.env_random_pod_delete ^= 1
                expect = "process flags"
            f.epoch(expect=expect, profiled=e % 7 == 3, device_only=e % 7 == 5)
            if e % 4 == 3:
                f.kernels()
        report = dict(seed=seed, **f.stats, events=sorted(f.seen))
        print("structural stream", json.dumps(report))
        missing = NEED_EVENTS - f.seen
        assert not missing, (missing, report)
        for cause in ("large gone row", "grow list", "list cap", "process flags"):
            assert f.stats[f"full: {cause}"] >= 1, (cause, report)
        assert f.stats["incremental"] >= 0.6 * f.stats["epochs"], report
    finally:
        f.close()


@pytest.mark.parametrize("seed", range(4))
def test_structural_streams(seed, oracle_mod):
    _run_stream(seed, oracle_mod)


# ------------------------------------------------------------------------------------------------ the native packer, nine options
def _packer_events(m, rng, counter, deleted):
    """Informer events plus creates, deletes (their Pods stay), group appends and removals, and scale-ups past a bucket."""
    events(rng, m, counter, structural=False)
    keys = sorted(m.clusters)
    u = rng.random()
    tag = ""
    if u < 0.2 and len(keys) > 8:
        key = keys[int(rng.integers(len(keys)))]
        deleted[key] = m.clusters[key]
        m.delete_cluster(*key)
        tag = "delete"
    elif u < 0.3 and deleted:
        key = sorted(deleted)[int(rng.integers(len(deleted)))]
        counter[0] += 1
        m.upsert_cluster(dict(deleted.pop(key), resourceVersion=90_000 + counter[0]))
        tag = "create"
    elif u < 0.4:
        src = copy.deepcopy(m.clusters[keys[int(rng.integers(len(keys)))]])
        counter[0] += 1
        src["name"], src["generation"], src["resourceVersion"] = f"{src['name']}-c{counter[0]}", 1, 50_000 + counter[0]
        m.upsert_cluster(src)
        tag = "create"
    elif u < 0.6:
        key = keys[int(rng.integers(len(keys)))]
        c = copy.deepcopy(m.clusters[key])
        gs = c["spec"].setdefault("workerGroupSpecs", [])
        counter[0] += 1
        if gs and rng.random() < 0.4:
            gs.pop()
        else:
            gs.append({"groupName": f"added-{counter[0]}", "replicas": 1, "minReplicas": 0, "maxReplicas": 4, "numOfHosts": 1})
        c["generation"] = c.get("generation", 1) + 1
        c["resourceVersion"] = 70_000 + counter[0]
        m.upsert_cluster(c)
        tag = "regroup"
    elif u < 0.75:
        key = keys[int(rng.integers(len(keys)))]
        for _ in range(int(rng.integers(40, 160))):
            counter[0] += 1
            w = next((p for p in m.rows if p is not None and p.get("namespace", "default") == key[0] and p["labels"].get("ray.io/cluster") == key[1]), None)
            if w is None:
                break
            m.upsert_pod({"namespace": key[0], "name": f"scale{counter[0]}", "labels": dict(w["labels"], **{"ray.io/node-type": "worker"}),
                          "phase": "Running", "conditions": [{"type": "Ready", "status": "True"}], "restartPolicy": "Always"})
        tag = "grow"
    return tag


def _live_counts(m):
    """Pods per (namespace, RayCluster) among the Mirror's live Pods."""
    return collections.Counter((p.get("namespace", "default"), (p.get("labels") or {}).get("ray.io/cluster")) for p in m.live_pods())


def _json_offsets(m):
    col = m.pk.column("c_json_off")
    return {k: (int(col[m.pk.cluster_row(*k)]), m.clusters[k].get("generation")) for k in m.clusters}


def test_native_packer_nine_options(oracle_mod):
    """Every epoch both packers equal the oracle and each other; the all-on flush sends no KR_PART_JSON unless it compacted the JSON
    arena (specs go row by row); and the all-on pass is incremental unless the epoch deleted, regrouped or moved (the last row, into
    a deleted one's hole) a RayCluster that has listed more Pods than the stride since the stream began: such a RayCluster may hold a
    region, and a gone row with a region takes the full pass.  Regions belong to rows: a RayCluster moved into a row that held one
    takes the region over, so the exemption follows every row a big RayCluster has held."""
    caps = dict(PACKER_CAPS, max_clusters=256, max_groups=2048, max_wtd=1024, max_pods=16384, max_jobs=256, max_creates=1 << 20)
    on, off = Packer(**caps, **ALL), Packer(**caps)
    try:
        for o in (abi.OPT_LARGE_CLUSTERS, abi.OPT_WIDE_CLUSTERS, abi.OPT_HUGE_CLUSTERS, abi.OPT_WTD_EDITS, abi.OPT_SPEC_ROWS,
                  abi.OPT_CLUSTER_CREATES, abi.OPT_CLUSTER_DELETES, abi.OPT_GROUP_EDITS, abi.OPT_LARGE_GROWTH):
            assert on.engine.get_option(o) == 1 and off.engine.get_option(o) == 0, o
        objs = objects(5)
        ms = [Mirror(*copy.deepcopy(objs), pk) for pk in (on, off)]
        for pk, m in zip((on, off), ms):
            pk.flush()
            packer_check(m, oracle_mod, lean=True)
        state = [([0], {}), ([0], {})]
        kinds, full = collections.Counter(), collections.Counter()
        big_rows = set()  # rows a RayCluster listing more Pods than the stride has held (a region may be theirs)
        for epoch in range(120):
            m_on = ms[0]
            stride = on.engine.get_option(abi.OPT_BUCKET_STRIDE)
            row_of = {k: on.cluster_row(*k) for k in m_on.clusters}
            big_rows |= {row_of[k] for k, n in _live_counts(m_on).items() if n > stride and k in row_of}
            last = max(m_on.clusters, key=row_of.get)
            before_keys, before_off = set(m_on.clusters), _json_offsets(m_on)
            regrouped_before = {k: len(c["spec"].get("workerGroupSpecs") or []) for k, c in m_on.clusters.items()}
            outs = []
            for (counter, deleted), m, pk in zip(state, ms, (on, off)):
                rng = np.random.default_rng(5000 + epoch)
                tag = _packer_events(m, rng, counter, deleted) if len(m.clusters) < caps["max_clusters"] - 8 else ""
                mode = pk.flush()
                _, got = packer_check(m, oracle_mod, lean=True)
                outs.append((tag, mode, got))
            (tag, mode, got), (_, _, twin) = outs
            d = twin.diff(got)
            assert not d, (epoch, d[:6])
            kinds[tag] += 1
            after_off = _json_offsets(m_on)
            compacted = any(before_off[k][0] != after_off[k][0] for k in before_off if k in after_off and before_off[k][1] == after_off[k][1])
            assert not (mode & abi.PART_JSON) or compacted, (epoch, mode, tag)
            gone = before_keys - set(m_on.clusters)
            moved = {last} if gone and last not in gone else set()
            regrouped = {k for k in before_keys & set(m_on.clusters)
                         if len(m_on.clusters[k]["spec"].get("workerGroupSpecs") or []) != regrouped_before[k]}
            may_be_full = any(row_of[k] in big_rows for k in gone | moved | regrouped)
            inc = incremental(got, got.clusters.shape[0])
            assert inc or may_be_full, (epoch, tag, sorted(gone | moved | regrouped))
            if not inc:
                full[tag] += 1
        print("packer nine options", dict(kinds), "full passes", dict(full))
        assert min(kinds[k] for k in ("create", "delete", "regroup", "grow")) >= 5, kinds
    finally:
        on.close()
        off.close()


def test_group_packer_nine_options(oracle_mod):
    """Two shards on one device with every option: a RayCluster deleted, one given a worker group, one scaled up past its bucket, by
    turns.  Each shard's pass equals a from-scratch full pass of the same engine, and is incremental unless the epoch deleted or
    regrouped a RayCluster of a shard that holds one grown earlier (the row it vacates, or the last row a deletion moves, or the row a
    moved RayCluster took over, may hold a region)."""
    caps = dict(PACKER_CAPS, max_clusters=128, max_groups=1024, max_wtd=1024, max_pods=8192, max_jobs=256, max_creates=1 << 20)
    gp = GroupPacker([0, 0], **caps, **ALL)
    try:
        for sh in gp.shards:
            assert sh.engine.get_option(abi.OPT_LARGE_GROWTH) == 1 and sh.engine.get_option(abi.OPT_GROUP_EDITS) == 1
        clusters, pods, jobs = objects(9)
        for c in clusters:
            gp.upsert_cluster(c)
        for p in pods:
            gp.upsert_pod(p)
        gp.flush()
        flags = gp.flags(fetch_pod_lists=0)
        gp.reconcile(flags)
        rng = np.random.default_rng(4)
        live = list(clusters)
        grown = set()
        n_inc = 0
        for epoch in range(12):
            c = copy.deepcopy(live[int(rng.integers(len(live)))])
            ns = c.get("namespace", "default")
            sh_of = gp.shard_of(ns, c["name"])
            may_be_full = epoch % 3 != 2 and any(gp.shard_of(*k) == sh_of for k in grown)
            if epoch % 3 == 0:
                gp.delete_cluster(ns, c["name"])
                live = [x for x in live if (x.get("namespace", "default"), x["name"]) != (ns, c["name"])]
            elif epoch % 3 == 1:
                c["spec"].setdefault("workerGroupSpecs", []).append({"groupName": f"extra{epoch}", "replicas": 2, "minReplicas": 0,
                                                                      "maxReplicas": 4, "numOfHosts": 1})
                c["generation"] = c.get("generation", 1) + 1
                gp.upsert_cluster(c)
            else:
                src = [p for p in pods if p.get("namespace", "default") == ns and p["labels"].get("ray.io/cluster") == c["name"]]
                for k in range(300 if src else 0):
                    q = copy.deepcopy(src[k % len(src)])
                    q["name"] = f"{q['name']}-g{epoch}-{k}"
                    gp.upsert_pod(q)
                grown.add((ns, c["name"]))
            gp.flush()
            got = gp.reconcile(flags)
            for i, g in enumerate(got):
                inc = incremental(g, g.clusters.shape[0])
                assert inc or (i == sh_of and may_be_full), (epoch, i, sh_of)
                n_inc += inc
            for sh, g, fl in zip(gp.shards, got, flags):
                sh.engine.set_incremental(False)
                full = sh.engine.reconcile(fl)
                sh.engine.set_incremental(True)
                d = full.diff(g)
                assert not d, (epoch, d[:6])
            gp.reconcile(flags)  # (the first pass after incremental epochs come back is a full one)
        assert n_inc >= 2 * 12 - 4, n_inc
    finally:
        gp.close()

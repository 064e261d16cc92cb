"""KR_OPT_HUGE_GROWTH: a RayCluster that grows past KR_LARGE_MAX_PODS Pods in an incremental epoch (a large one scaling past it, an
ordinary one jumping past it, a huge one outgrowing its region) gets a region and tiles in that epoch (k_inc_grow<true>,
kuberay_b200/csrc/kr_large.cuh; the tile kernels of kr_huge.cuh over the reserve entries) instead of sending the pass to a full one.

Every epoch goes through harness.Driver: compared with the oracle, and every record the pass did not name equal to the previous
epoch's.  Where an epoch is expected to be incremental it is asserted to be, with the grown RayClusters among changed_clusters."""
import copy

import numpy as np
import pytest

from class_model import GROW_LIST_DIV, GROW_LIST_MIN, GROW_MAX, GROW_SPILL, Model, counts, large_region_cap, owners, region_arena
from test_gpu_cluster_deletes import _check as check_renumbered
from test_huge_growth_abi import resident_tiles
from harness import (PACKER_CAPS, Driver, Mirror, b32, device_incremental, events, head_row, huge_objects, incremental, most_workers,
                     move, packer_check, packer_stream, scale_to, set_phase, spec_bytes, workers)
from kuberay_b200 import abi, synthetic
from kuberay_b200.packer import GroupPacker, Packer

pytestmark = pytest.mark.gpu

HG = dict(large_clusters=True, huge_clusters=True, large_growth=True, huge_growth=True)
TILE = abi.LARGE_MAX_PODS  # arrival ranks per tile (kr_huge.cuh)
GROWN_NAMES = {"k_inc_grow", "k_huge_tiles", "k_huge_merge", "k_decide_large"}


def _fleet(seed, n_clusters=3000, groups=1, healthy=True, **kw):
    """RayClusters of 20 pods (the 64-pod stride), healthy, with room to scale: no group limits its replicas.  (A grown RayCluster's
    surplus Pods are scale-down actions, and every epoch that grows it reserves a new action run: a fleet of 3 000 RayClusters
    holds the runs of the growth steps below without a full pass to pack them again.)"""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=n_clusters, pods_per_cluster=20, groups=groups, seed=seed,
                                                           healthy=healthy, **kw))
    for c in range(n_clusters):
        snap.c_flags[c] &= ~np.uint32(abi.CF_SKIP | abi.CF_SUSPEND)
    return snap, flags


def _grown(got, clusters):
    assert got.changed_clusters is not None
    missing = set(int(c) for c in clusters) - set(got.changed_clusters.tolist())
    assert not missing, missing


def _flip(dr, c, step=97):
    """A churn epoch: PodReady flips on RayCluster c's workers."""
    rows = workers(dr.snap, c)[::step]
    dr.snap.p_packed[rows] ^= np.uint32(1 << abi.PP_READY_SHIFT)
    dr.commit_rows(rows)
    return dr.check(dr.oracle, expect_incremental=True)


def _grow(snap, sizes):
    """Worker Pods of the ordinary RayClusters (of at most 256 Pods, last rows first) move into worker group 0 of each RayCluster c
    of `sizes` until it lists sizes[c] Pods; no RayCluster with more Pods gives any.  -> the pod rows that moved."""
    moved = []
    for c, size in sizes.items():
        own = owners(snap)
        cnt = counts(snap, own)
        worker = ((snap.p_packed >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER
        donors = np.flatnonzero(worker & (own >= 0) & (own != c) & (cnt[np.maximum(own, 0)] <= 256))[::-1]
        need = size - int(cnt[c])
        assert 0 <= need <= donors.size, (c, size, donors.size)
        move(snap, donors[:need], c)
        moved.append(donors[:need])
    return np.concatenate(moved)


def _driver(snap, flags, oracle_mod, slack=1.25, **kw):
    dr = Driver(snap, flags, slack=slack, max_creates=1 << 18, **kw)
    dr.oracle = oracle_mod
    dr.check(oracle_mod, expect_incremental=False)
    return dr


def test_step_growth_past_the_largest_cluster(oracle_mod):
    """A large RayCluster scales 8 000 -> 8 193 -> 12 000 -> 20 000 Pods, one epoch per step: every epoch stays incremental, the
    fleet keeps its stride, and the tile kernels sort the grown RayCluster; a churn epoch afterwards is incremental too."""
    snap, flags = _fleet(1)
    c = 600
    synthetic.grow_clusters(snap, [c], 8000)
    dr = _driver(snap, flags, oracle_mod, **HG)
    try:
        stride = dr.eng.get_option(abi.OPT_BUCKET_STRIDE)
        assert stride == 64
        sizes = [8193, 12000, 20000]
        for size, rows in zip(sizes, synthetic.grow_epochs(snap, [c], sizes)):
            dr.commit_rows(rows)
            got, names = dr.check(oracle_mod, expect_incremental=True, profiled=True)
            _grown(got, [c])
            assert GROWN_NAMES <= set(names), names
            assert got.clusters["n_pods"][c] == size
            assert dr.eng.get_option(abi.OPT_BUCKET_STRIDE) == stride
        _flip(dr, c)
    finally:
        dr.close()


def test_huge_regrowth_with_pods_leaving(oracle_mod):
    """A huge RayCluster outgrows its region twice while some of its Pods leave in the same epochs: its old tiles are retired, its
    old region (more than 8 192 records) copied by the whole launch, and the stale records dropped by the tiles' compaction."""
    snap, flags = _fleet(2)
    c = 10
    synthetic.grow_clusters(snap, [c], 9000)
    dr = _driver(snap, flags, oracle_mod, **HG)
    try:
        rng = np.random.default_rng(5)
        for size in (11300, 15000):
            leave = rng.choice(workers(snap, c), 25, replace=False)
            rows = next(synthetic.grow_epochs(snap, [c], [size + 25]))
            move(snap, leave, 200)
            dr.commit_rows(np.concatenate([rows, leave]))
            got, names = dr.check(oracle_mod, expect_incremental=True, profiled=True)
            _grown(got, [c, 200])
            assert GROWN_NAMES <= set(names), names
            assert got.clusters["n_pods"][c] == size
        assert dr.eng.get_option(abi.OPT_BUCKET_STRIDE) == 64
        _flip(dr, c)
    finally:
        dr.close()


def test_ordinary_cluster_jumps_past_the_largest(oracle_mod):
    """An ordinary RayCluster (20 Pods, no region) takes 9 000 Pods in one epoch: it is listed, given a region and tiles, and decided
    by one of the CTAs past the per-cluster list."""
    snap, flags = _fleet(3)
    c = 700
    dr = _driver(snap, flags, oracle_mod, **HG)
    try:
        dr.commit_rows(next(synthetic.grow_epochs(snap, [c], [9000])))
        got, names = dr.check(oracle_mod, expect_incremental=True, profiled=True)
        _grown(got, [c])
        assert GROWN_NAMES <= set(names), names
        assert got.clusters["n_pods"][c] == 9000
        _flip(dr, c)
    finally:
        dr.close()


def test_mixed_epoch(oracle_mod):
    """A huge regrowth, a large crossing, an ordinary jump past 8 192 and an ordinary promotion in one epoch, beside Pod deletions,
    failures and PodReady flips."""
    snap, flags = _fleet(4, n_clusters=3500)
    _grow(snap, {10: 9000, 20: 8000})
    dr = _driver(snap, flags, oracle_mod, **HG)
    try:
        rows = [_grow(snap, {10: 11300, 20: 8300, 1500: 8500, 1600: 300})]
        gone = workers(snap, 1700)[:4]
        snap.p_packed[gone] |= np.uint32(abi.PP_TOMBSTONE)
        fail = workers(snap, 10)[:3]
        set_phase(snap, fail, abi.PHASE_FAILED)
        flip = np.concatenate([workers(snap, 20)[:5], workers(snap, 1701)[:5]])
        snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        dr.commit_rows(np.concatenate(rows + [gone, fail, flip]))
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        _grown(got, [10, 20, 1500, 1600, 1700, 1701])
        assert [got.clusters["n_pods"][c] for c in (10, 20, 1500, 1600)] == [11300, 8300, 8500, 300]
        _flip(dr, 1500)
    finally:
        dr.close()


@pytest.mark.parametrize("kind", ["recreate", "recreate_rehash", "multihost", "wtd", "wide"])
def test_features_of_a_grown_huge_cluster(kind, oracle_mod):
    """A large RayCluster with a RayCluster feature crosses 8 192 Pods, then regrows as a huge one: Recreate-gated (with its spec
    re-hashed in the regrowth epoch, or not), a multi-host group, workersToDelete names of Pods that just joined, more than 32
    worker groups."""
    extra = dict(autoscaling_frac=1.0, wtd_group_frac=1.0) if kind == "wtd" else dict(multihost_frac=0.25) if kind == "multihost" else {}
    snap, flags = _fleet(5, groups=2 if kind == "multihost" else 1, healthy=kind != "wtd", **extra)
    options = dict(HG)
    if kind == "multihost":
        c = next(c for c in range(100, 3000) if (snap.g_num_hosts[int(snap.c_group_off[c]):int(snap.c_group_off[c]) + 2] > 1).any())
    elif kind == "wtd":
        c = next(c for c in range(300, 3000) if snap.g_wtd_cnt[snap.c_group_off[c]] >= 1)
        snap.c_flags[c] &= ~np.uint32(abi.CF_SKIP | abi.CF_SUSPEND | abi.CF_UPGRADE_RECREATE)
        snap.c_flags[c] |= np.uint32(abi.CF_HEAD_EXPECT_OK | abi.CF_AUTOSCALING)
        options["wtd_edits"] = True
    else:
        c = 30
    if kind.startswith("recreate"):
        snap.c_flags[c] |= np.uint32(abi.CF_UPGRADE_RECREATE)
        h = head_row(snap, c)
        snap.h_version_state[h] = abi.VER_CURRENT
        snap.h_annot_state[h] = abi.ANNOT_HASH32
        snap.h_annot_hash.reshape(-1, 32)[h] = np.frombuffer(b32(spec_bytes(snap, c)), dtype=np.uint8)
    if kind == "wide":
        snap = synthetic.widen_clusters(snap, [c], 40)
        options["wide_clusters"] = True
    synthetic.grow_clusters(snap, [c], 8000)
    dr = _driver(snap, flags, oracle_mod, **options)
    try:
        for size in (8500, 11000):
            rows = next(synthetic.grow_epochs(snap, [c], [size]))
            if kind == "recreate_rehash" and size == 11000:
                snap.json[int(snap.c_json_off[c]) + 3] ^= 0x20  # its spec no longer matches the annotation
                np.copyto(dr.views["json"], snap.json)
                dr.eng.commit(abi.PART_JSON)
            if kind == "wtd":
                set_phase(snap, rows, abi.PHASE_RUNNING)
                snap.p_packed[rows] &= ~np.uint32(abi.PP_RAY_TERMINATED)
                g = int(snap.c_group_off[c])
                scale_to(snap, g, workers(snap, c).size - 2)
                snap.w_name_id[int(snap.g_wtd_off[g])] = snap.p_name_id[rows[-1]]  # a Pod that just joined
                dr.commit_objects()
            dr.commit_rows(rows)
            got, names = dr.check(oracle_mod, expect_incremental=True, profiled=True)
            _grown(got, [c])
            assert GROWN_NAMES <= set(names), names
        if kind == "recreate_rehash":
            assert got.clusters["path"][c] == abi.PATH_RECREATE_DELETE_ALL
        _flip(dr, c)
    finally:
        dr.close()


def _moves_driver(oracle_mod):
    snap, flags = synthetic.generate(synthetic.config("C2", n_clusters=3500, pods_per_cluster=16, groups=2, seed=41))
    _grow(snap, {3499: 9000})
    dr = Driver(snap, flags, slack=1.25, max_creates=1 << 18, cluster_deletes=True, group_edits=True, large_moves=True, **HG)
    dr.check(oracle_mod, expect_incremental=None)
    dr.check(oracle_mod, expect_incremental=None)
    dr.eng.commit(abi.PART_OBJECTS)  # (records the group names for the regroup)
    dr.check(oracle_mod, expect_incremental=None)
    return dr


def test_huge_moved_or_regrouped_and_grown(oracle_mod):
    """KR_OPT_LARGE_MOVES: a huge RayCluster moved by swap-remove (it carries its tiles) grows past its carried region in the same
    epoch; then, regrouped in place, it grows again.  Its carried tiles are retired and new ones appended each time."""
    dr = _moves_driver(oracle_mod)
    try:
        old = dr.snap
        dr.use(synthetic.delete_clusters(old, [12]))  # 3499 (huge) moves into row 12
        dr.commit_objects()
        dr.commit_rows(_grow(dr.snap, {12: 11500}))
        # (every other RayCluster keeps its row: its records must equal the previous epoch's, its groups at the shifted indices)
        got, names = check_renumbered(dr, oracle_mod, old, synthetic.swap_remove_order(old.dims["clusters"], [12]), True, profiled=True)
        assert "k_inc_large_release" in names and GROWN_NAMES <= set(names), names
        _grown(got, [12])
        assert got.clusters["n_pods"][12] == 11500
        g0 = int(dr.snap.c_group_off[12])
        groups = [(g, None) for g in range(g0, g0 + int(dr.snap.c_group_cnt[12]))]
        old = dr.snap
        dr.use(synthetic.regroup_clusters(old, {12: groups + [(g0, int(old.g_name_id.max()) + 1)]}))
        dr.commit_objects()
        dr.commit_rows(_grow(dr.snap, {12: 14500}))
        got, names = check_renumbered(dr, oracle_mod, old, np.arange(old.dims["clusters"]), True, profiled=True)
        assert GROWN_NAMES <= set(names), names
        _grown(got, [12])
        assert got.clusters["n_pods"][12] == 14500
        dr.oracle = oracle_mod
        _flip(dr, 12)
    finally:
        dr.close()


# ------------------------------------------------------------------------------------------------ limits
def test_more_tiles_than_the_reserve(oracle_mod):
    """A huge RayCluster of 170 000 Pods (26 tiles) regrown by one Pod needs 33 tiles, one more than KR_HUGE_GROW_TILES: that epoch
    is a full pass, and the next one is incremental again.  The capacities (slack 1.6) leave the region arena and the resident tiles
    room for the regrowth, and its group asks for the Pods that join (no action run to reserve), so the reserve is the only limit
    the epoch meets."""
    snap, flags = _fleet(6, n_clusters=12000)
    c, stride = 100, 64
    room = stride + large_region_cap(170000, stride)
    size = room + 1
    assert -(-room // TILE) == 26 and -(-(stride + large_region_cap(size, stride)) // TILE) == abi.HUGE_GROW_TILES + 1
    synthetic.grow_clusters(snap, [c], 170000)
    scale_to(snap, int(snap.c_group_off[c]), size - 1)
    dr = _driver(snap, flags, oracle_mod, slack=1.6, **HG)
    try:
        assert dr.eng.get_option(abi.OPT_BUCKET_STRIDE) == stride
        cfg, nc, groups = dr.eng.cfg, snap.dims["clusters"], snap.c_group_cnt.astype(np.int64)
        m = HugeGrowthModel(nc, snap.dims["pods"], True, False, arena=region_arena(cfg.max_pods), tile_cap=resident_tiles(cfg.max_pods))
        m.full_pass(counts(snap, owners(snap)), groups)
        assert m.stride == stride and m.caps[c] == room - stride
        rows = next(synthetic.grow_epochs(snap, [c], [size]))
        peak = counts(snap, owners(snap))
        assert m.cursor + large_region_cap(size, stride) <= m.arena  # (the arena holds the new region)
        assert abi.HUGE_GROW_TILES + 1 <= m.tile_cap  # (and the resident tiles the regrown RayCluster's)
        assert m.grow(peak, groups) == "tile reserve"
        dr.commit_rows(rows)
        dr.check(oracle_mod, expect_incremental=False)
        _flip(dr, c, step=997)
    finally:
        dr.close()


def test_a_huge_cluster_shrinks_and_another_grows(oracle_mod):
    """A huge RayCluster of 20 000 Pods (4 tiles) keeps its region and tiles while 15 000 of its Pods move to an ordinary RayCluster,
    which grows huge in the same epoch.  The resident tiles stay within the engine's tile capacity (test_huge_growth_abi.py shows the
    region arena always fills first); here the new region does not fit the arena, so the epoch is a full pass that lays the regions
    out again, and the next epoch is incremental."""
    snap, flags = _fleet(11, n_clusters=1300)
    a, b = 10, 1290  # (b keeps its Pods: grow_clusters drains the first rows)
    synthetic.grow_clusters(snap, [a], 20000)
    dr = _driver(snap, flags, oracle_mod, slack=1.0, **HG)
    try:
        cfg, nc, groups = dr.eng.cfg, snap.dims["clusters"], snap.c_group_cnt.astype(np.int64)
        m = HugeGrowthModel(nc, snap.dims["pods"], True, False, arena=region_arena(cfg.max_pods), tile_cap=resident_tiles(cfg.max_pods))
        own = owners(snap)
        m.full_pass(counts(snap, own), groups)
        rows = workers(snap, a)[:15000]
        move(snap, rows, b)
        peak = counts(snap, own) + np.bincount(owners(snap)[rows], minlength=nc)
        assert m.grow(peak, groups) == "arena"
        dr.commit_rows(rows)
        dr.check(oracle_mod, expect_incremental=False)
        assert dr.prev.clusters["n_pods"][b] == counts(snap, owners(snap))[b] > abi.LARGE_MAX_PODS
        _flip(dr, b)
    finally:
        dr.close()


def test_more_pods_than_the_spill(oracle_mod):
    """An ordinary RayCluster taking more than KR_GROW_SPILL Pods past its bucket in one epoch is a full pass."""
    snap, flags = _fleet(7, n_clusters=1300)
    dr = _driver(snap, flags, oracle_mod, **HG)
    try:
        stride = dr.eng.get_option(abi.OPT_BUCKET_STRIDE)
        dr.commit_rows(next(synthetic.grow_epochs(snap, [50], [stride + GROW_SPILL + 1])))
        dr.check(oracle_mod, expect_incremental=False)
        _flip(dr, 50)
    finally:
        dr.close()


def test_a_full_region_arena(oracle_mod):
    """A huge RayCluster regrown on small capacities abandons its regions until the arena has no room for the next one: that step
    is a full pass, which lays the regions out again from offset 0, and the next step fits again."""
    snap, flags = _fleet(8, n_clusters=1300)
    c = 10
    synthetic.grow_clusters(snap, [c], 9000)
    dr = _driver(snap, flags, oracle_mod, slack=1.0, **HG)
    try:
        stride = dr.eng.get_option(abi.OPT_BUCKET_STRIDE)
        arena = region_arena(dr.eng.cfg.max_pods)
        used, room, full_at, sizes = large_region_cap(9000, stride), stride + large_region_cap(9000, stride), None, []
        for k in range(3):
            size = room + 100
            sizes.append(size)
            cap = large_region_cap(size, stride)
            if used + cap > arena and full_at is None:
                full_at = k
            used, room = used + cap, stride + cap
        assert full_at == 1, (sizes, arena)  # (the fleet's shape puts the arena's end at the second step)
        for k, rows in enumerate(synthetic.grow_epochs(snap, [c], sizes[:2])):
            dr.commit_rows(rows)
            got, _ = dr.check(oracle_mod, expect_incremental=k != full_at)
            if k != full_at:
                _grown(got, [c])
        _flip(dr, c)
    finally:
        dr.close()


@pytest.mark.parametrize("off", ["large_clusters", "huge_clusters", "large_growth", "huge_growth"])
def test_without_a_prerequisite_the_crossing_is_a_full_pass(off, oracle_mod):
    """With one of the four options off, a large RayCluster crossing 8 192 Pods is a full pass.  The next epoch is incremental when
    the fleet stays on the bucket pipeline (KR_OPT_HUGE_CLUSTERS keeps the huge RayCluster there)."""
    snap, flags = _fleet(9, n_clusters=1300)
    c = 600
    synthetic.grow_clusters(snap, [c], 8000)
    options = dict(HG, **{off: False})
    dr = Driver(snap, flags, max_creates=1 << 18, **options)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        dr.commit_rows(next(synthetic.grow_epochs(snap, [c], [8193])))
        dr.check(oracle_mod, expect_incremental=False)
        rows = workers(snap, c)[::97]
        snap.p_packed[rows] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        dr.commit_rows(rows)
        dr.check(oracle_mod, expect_incremental=off in ("large_growth", "huge_growth"))
    finally:
        dr.close()


def test_option_on_without_growth_equals_option_off(oracle_mod):
    """A fleet with a huge and a large RayCluster, churned without any growth: with the option on every pass equals the option-off
    twin's, and both are incremental."""
    snap, flags = _fleet(10, n_clusters=1300)
    _grow(snap, {10: 9000, 20: 3000})
    base = dict(large_clusters=True, huge_clusters=True, large_growth=True)
    on = Driver(copy.deepcopy(snap), copy.deepcopy(flags), max_creates=1 << 18, huge_growth=True, **base)
    off = Driver(copy.deepcopy(snap), copy.deepcopy(flags), max_creates=1 << 18, **base)
    try:
        assert on.eng.get_option(abi.OPT_HUGE_GROWTH) == 1 and off.eng.get_option(abi.OPT_HUGE_GROWTH) == 0
        for e in range(6):
            outs = []
            for dr in (on, off):
                if e:
                    r = np.random.default_rng(100 + e)
                    rows = np.concatenate([r.choice(workers(dr.snap, 10), 40, replace=False), r.choice(workers(dr.snap, 20), 20, replace=False),
                                           r.choice(dr.snap.dims["pods"], 30, replace=False)])
                    dr.snap.p_packed[rows] ^= np.uint32(1 << abi.PP_READY_SHIFT)
                    set_phase(dr.snap, rows[::9], abi.PHASE_FAILED)
                    dr.commit_rows(rows)
                got, _ = dr.check(oracle_mod, expect_incremental=e > 0)
                outs.append(got)
            assert not outs[1].diff(outs[0]), e
    finally:
        on.close()
        off.close()


# ------------------------------------------------------------------------------------------------ seeded stream
class HugeGrowthModel(Model):
    """Model with KR_OPT_HUGE_GROWTH: a RayCluster may grow past 8 192 Pods in an incremental epoch; the epoch takes the full pass
    when the tiles it appends pass KR_HUGE_GROW_TILES, or the resident tiles would pass the engine's tile capacity."""

    def __init__(self, *a, tile_cap, **kw):
        super().__init__(*a, huge=True, **kw)
        self.tile_cap = tile_cap

    def tiles(self, cap):
        span = self.stride + cap
        return -(-span // TILE) if span > abi.LARGE_MAX_PODS else 0

    def grow(self, peak, groups):
        over = np.flatnonzero(peak > self.limits())
        if not over.size:
            return None
        if len(over) > GROW_MAX:
            return "grow list"
        if int((peak[over] - self.limits()[over]).sum()) > GROW_SPILL:
            return "spill"
        caps = {int(c): large_region_cap(int(peak[c]), self.stride) for c in over}
        added = sum(self.tiles(cap) for cap in caps.values())
        if added > abi.HUGE_GROW_TILES:
            return "tile reserve"
        resident = sum(self.tiles(cap) for c, cap in self.caps.items() if c not in caps)
        if resident + added > self.tile_cap:
            return "tile capacity"
        if self.arena is not None and self.cursor + sum(caps.values()) > self.arena:
            return "arena"
        wide = groups > 32 if self.wide else np.zeros(groups.size, dtype=bool)
        listed = sum(1 for c in caps if c not in self.caps and not wide[c])
        if listed and len(self.per_cluster_list(groups)) + listed > max(GROW_LIST_MIN, self.nc // GROW_LIST_DIV):
            return "list cap"
        for c in sorted(caps):
            self.caps[c], self.offs[c] = caps[c], self.cursor
            self.cursor += caps[c]
        return None


@pytest.mark.parametrize("seed", [1, 2])
def test_seeded_stream(seed, oracle_mod):
    """16 epochs on a fleet with large and huge RayClusters: each epoch some of a few RayClusters scale up by random steps (past
    8 192 Pods and past their regions), Pods leave them, and PodReady flips.  HugeGrowthModel predicts each epoch's pass; the
    stream must see incremental epochs that cross 8 192 Pods and regrow huge RayClusters."""
    snap, flags = _fleet(20 + seed)
    hot = [10, 20, 30, 40]
    _grow(snap, {10: 9000, 20: 6000})
    for c in hot:  # (the autoscaler asked for the Pods ahead: joining ones fill the creates, no surplus to scale down)
        scale_to(snap, int(snap.c_group_off[c]), 40000)
    dr = Driver(snap, flags, slack=1.25, max_creates=1 << 20, **HG)
    rng = np.random.default_rng(seed)
    try:
        cfg = dr.eng.cfg
        nc = snap.dims["clusters"]
        m = HugeGrowthModel(nc, snap.dims["pods"], True, False, arena=region_arena(cfg.max_pods), tile_cap=resident_tiles(cfg.max_pods))
        groups = snap.c_group_cnt.astype(np.int64)
        own = owners(snap)
        m.full_pass(counts(snap, own), groups)
        dr.check(oracle_mod, expect_incremental=False)
        assert dr.eng.get_option(abi.OPT_BUCKET_STRIDE) == m.stride
        res_act, res_cre = dr.prev.act_cnt.astype(np.int64), np.bincount(snap.g_cluster_idx, weights=dr.prev.groups["n_create"], minlength=nc).astype(np.int64)
        act_ext, cre_ext = dr.prev.act_pod_idx.size, dr.prev.create_idx.size
        seen = set()
        for e in range(16):
            before = counts(snap, own)
            rows = []
            rows.append(_grow(snap, {c: int(before[c]) + int(rng.integers(50, 2000)) for c in rng.choice(hot, int(rng.integers(1, 3)), replace=False).tolist()}))
            c = int(rng.choice(hot))
            if workers(snap, c).size > 40:
                leave = rng.choice(workers(snap, c), 20, replace=False)
                move(snap, leave, int(rng.integers(1000, nc)))
                rows.append(leave)
            flip = rng.choice(snap.dims["pods"], 40, replace=False)
            snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
            rows.append(flip)
            rows = np.unique(np.concatenate(rows))
            new_own = owners(snap)
            joined = np.bincount(new_own[rows][(new_own[rows] >= 0) & (new_own[rows] != own[rows])], minlength=nc)
            peak = before + joined
            saved = (dict(m.caps), dict(m.offs), m.cursor)  # (a full pass starts from the regions before the epoch)
            crossed = bool(((peak > abi.LARGE_MAX_PODS) & (peak > m.limits())).any())
            cause = "sort pipeline" if not m.valid else m.grow(peak, groups)
            now = counts(snap, new_own)
            dr.commit_rows(rows)
            got, _ = dr.check(oracle_mod)
            inc = incremental(got, nc)
            if cause is None:
                n_act = got.act_cnt.astype(np.int64)
                n_cre = np.bincount(snap.g_cluster_idx, weights=got.groups["n_create"], minlength=nc).astype(np.int64)
                if act_ext + int(n_act[n_act > res_act].sum()) > snap.dims["pods"] or cre_ext + int(n_cre[n_cre > res_cre].sum()) > cfg.max_creates:
                    cause = "arena (reserved runs)"
            if cause is None:
                assert inc, (e, "an epoch the resident state can absorb took the full pass", seen)
                if crossed:
                    seen.add("incremental past 8192")
            elif cause != "arena (reserved runs)":
                assert not inc, (e, "an epoch that must take the full pass was incremental", cause)
            seen.add(f"{'incremental' if inc else 'full'}: {cause}")
            n_act = got.act_cnt.astype(np.int64)
            n_cre = np.bincount(snap.g_cluster_idx, weights=got.groups["n_create"], minlength=nc).astype(np.int64)
            if inc:
                res_act, res_cre = np.maximum(res_act, n_act), np.maximum(res_cre, n_cre)
            else:
                m.caps, m.offs, m.cursor = saved
                m.full_pass(now, groups)
                res_act, res_cre = n_act, n_cre
            act_ext, cre_ext = got.act_pod_idx.size, got.create_idx.size
            assert dr.eng.get_option(abi.OPT_BUCKET_STRIDE) == m.stride
            own = new_own
        print("huge growth stream", seed, sorted(seen))
        assert "incremental past 8192" in seen, seen
    finally:
        dr.close()


# ------------------------------------------------------------------------------------------------ packers
def _scaling_pods(pods, owner, n):
    src = [p for p in pods if (p.get("namespace"), p["labels"].get("ray.io/cluster")) == owner and p["labels"].get("ray.io/node-type") == "worker"]
    out = []
    for i in range(n):
        q = copy.deepcopy(src[i % len(src)])
        q["name"] = f"{q['name']}-scale-{i}"
        out.append(q)
    return out


ALL = dict(large_clusters=True, wide_clusters=True, huge_clusters=True, wtd_edits=True, spec_rows=True, cluster_creates=True,
           cluster_deletes=True, group_edits=True, large_growth=True, large_moves=True, huge_growth=True)


def test_native_packer_stream(oracle_mod):
    """The native packer with every option on against a twin with all of them off: the largest RayCluster scales past 8 192 Pods,
    regrows and shrinks over the epochs, beside seeded informer events.  Every epoch equals the oracle and the twin, and the
    option keeps more epochs incremental."""
    clusters, pods, jobs = huge_objects(5, 7000)
    owner = most_workers(pods)
    n_now = sum((p.get("namespace"), p["labels"].get("ray.io/cluster")) == owner for p in pods)
    extra = _scaling_pods(pods, owner, 9000)
    caps = dict(PACKER_CAPS, max_clusters=256, max_groups=4096, max_wtd=4096, max_pods=32768, max_heads=1024, max_creates=1 << 20)
    results = []
    for on in (True, False):
        pk = Packer(**caps, **(ALL if on else {}))
        try:
            assert pk.engine.get_option(abi.OPT_HUGE_GROWTH) == int(on)
            m = Mirror(copy.deepcopy(clusters), copy.deepcopy(pods), jobs, pk)
            pk.flush()
            packer_check(m, oracle_mod, lean=True)
            counter, r = [0], np.random.default_rng(7)

            def step(epoch):
                k = (1300, 1500, 5000, 9000, 3000, 6000, 6000, 0)[epoch] if epoch < 8 else 0
                live = {q["name"] for q in m.live_pods()}
                for q in extra[:k]:
                    if q["name"] not in live:
                        m.upsert_pod(copy.deepcopy(q))
                for q in extra[k:]:
                    if q["name"] in live:
                        m.delete_pod(q.get("namespace", "default"), q["name"])
                events(r, m, counter, structural=False)

            gots, _ = packer_stream(m, oracle_mod, 8, step)
            assert n_now + 1300 > abi.LARGE_MAX_PODS
            results.append((gots, [device_incremental(g) for g in gots]))
        finally:
            pk.close()
    (on, inc_on), (off, inc_off) = results
    for a, b in zip(on, off):
        assert not a.diff(b)
    print("native packer huge growth: incremental", inc_on, "twin", inc_off)
    assert sum(inc_on) > sum(inc_off), (inc_on, inc_off)


def test_group_packer_stream(oracle_mod):
    """A GroupPacker of two shards with every option on: one RayCluster scales past 8 192 Pods and regrows; each shard's pass equals
    a full pass of the same engine, and the shards keep their epochs incremental."""
    caps = dict(PACKER_CAPS, max_clusters=256, max_groups=4096, max_wtd=4096, max_pods=32768, max_heads=1024, max_creates=1 << 20)
    gp = GroupPacker([0, 0], **caps, **ALL)
    try:
        assert all(sh.engine.get_option(abi.OPT_HUGE_GROWTH) == 1 for sh in gp.shards)
        clusters, pods, jobs = huge_objects(9, 7000)
        owner = most_workers(pods)
        extra = _scaling_pods(pods, owner, 8000)
        for c in clusters:
            gp.upsert_cluster(c)
        for p in pods:
            gp.upsert_pod(p)
        gp.flush()
        flags = gp.flags(fetch_pod_lists=0)
        gp.reconcile(flags)
        n_inc = 0
        for e, k in enumerate((1300, 4000, 8000, 2000)):
            for q in extra[:k]:
                gp.upsert_pod(copy.deepcopy(q))
            for q in extra[k:]:
                gp.delete_pod(q.get("namespace", "default"), q["name"])
            gp.flush()
            got = gp.reconcile(flags)
            n_inc += sum(incremental(g, g.clusters.shape[0]) for g in got)
            for sh, g, fl in zip(gp.shards, got, flags):
                sh.engine.set_incremental(False)
                full = sh.engine.reconcile(fl)
                sh.engine.set_incremental(True)
                assert not full.diff(g), e
            gp.reconcile(flags)
        print("group packer huge growth: incremental shard passes", n_inc)
        assert n_inc >= 2 * 4 - 1, n_inc
    finally:
        gp.close()

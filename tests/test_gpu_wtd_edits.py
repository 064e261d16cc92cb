"""KR_OPT_WTD_EDITS: scaleStrategy.workersToDelete edits (renames, lists that grow and shrink) keep the device-side incremental
epoch: the next pass rebuilds the name table (k_inc_wtd_release / _clear / _insert / _resolve in kuberay_b200/csrc/kr_incr.cuh)
and re-decides the RayClusters whose Pods were named before or are named now.

Every epoch is compared with the CPU oracle, records the pass did not name must be unchanged since the previous epoch, and with the
option on every epoch that changes only lists, pod rows and non-key object rows must be incremental."""
import copy

import numpy as np
import pytest

from harness import (PACKER_CAPS, POD_COLS, REBUILD, Driver, Mirror, arena_stream, autoscale_objects, device_incremental, events, flip_ready,
                     incremental, lists_of, objects, packer_check, packer_stream, with_wtd_lists, workers_of)
from kuberay_b200 import abi, synthetic
from kuberay_b200.live import LiveArena
from kuberay_b200.packer import Packer

pytestmark = pytest.mark.gpu

GHOST = 0x7FFE0000      # name ids no Pod carries


def _driver(snap, flags, wtd_edits=True, **opts):
    """Fixed layout with room for the lists to grow; KR_OPT_WTD_EDITS on unless told otherwise; `opts` turns on other options."""
    return Driver(snap, flags, wtd_room=512, **opts, wtd_edits=wtd_edits)


def _snap(seed, **kw):
    p = dict(n_clusters=300, pods_per_cluster=16, groups=3, autoscaling_frac=1.0, wtd_group_frac=0.3, seed=seed)
    p.update(kw)
    snap, flags = synthetic.generate(synthetic.config("C2", **p))
    return snap, flags


def _action_of(got, c, row):
    pods, codes = got.actions_of(c)
    hit = np.flatnonzero(pods == row)
    return int(codes[hit[0]]) if hit.size else abi.ACT_KEEP


@pytest.mark.parametrize("target", ["own", "other_group", "nowhere", "orphan"])
def test_rename_in_place(target, oracle_mod):
    snap, flags = _snap(3)
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        lists = lists_of(dr.snap)
        gs = [g for g in range(snap.dims["groups"]) if lists[g] and workers_of(snap, g).size >= 3 and
              (target != "other_group" or snap.c_group_cnt[snap.g_cluster_idx[g]] >= 2)][:6]
        assert len(gs) >= 3
        old = {g: lists[g][0] for g in gs}
        pick = {}
        for g in gs:
            own = [int(r) for r in workers_of(snap, g) if int(snap.p_name_id[r]) not in lists[g]]
            if target in ("own", "orphan"):
                pick[g] = own[0]
            elif target == "other_group":
                c = int(snap.g_cluster_idx[g])
                other = [h for h in range(int(snap.c_group_off[c]), int(snap.c_group_off[c] + snap.c_group_cnt[c])) if h != g and workers_of(snap, h).size]
                pick[g] = int(workers_of(snap, other[0])[0])
        if target == "orphan":  # one epoch earlier the picked Pods lose their RayCluster (ray.io/cluster names none)
            rows = list(pick.values())
            dr.snap.p_cluster_name_id[rows] = np.uint32(GHOST) + np.arange(len(rows), dtype=np.uint32)
            dr.commit_rows(rows)
            dr.check(oracle_mod, expect_incremental=True)
        for g in gs:
            lists[g][0] = GHOST + 100 + g if target == "nowhere" else int(dr.snap.p_name_id[pick[g]])
        dr.set_wtd_lists(lists)
        got, names = dr.check(oracle_mod, expect_incremental=True, profiled=True)
        assert set(REBUILD) <= set(names), names
        for g in gs:
            e = int(dr.snap.g_wtd_off[g])
            if target == "nowhere":
                assert got.wtd_pod_idx[e] == -1
            else:
                assert got.wtd_pod_idx[e] == pick[g]
            if target == "other_group":  # resolves, but is not one of its own group's names
                assert _action_of(got, int(snap.g_cluster_idx[g]), pick[g]) != abi.ACT_DELETE_WTD
        for g in gs:
            lists[g][0] = old[g]
        dr.set_wtd_lists(lists)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


def test_lists_grow_from_empty_and_shrink_to_empty(oracle_mod):
    """n_wtd crosses 0 both ways (the Bloom staging of k_match2 switches in the full pass), the first and the last name of the
    snapshot move, and an edit of the first group shifts every later offset."""
    snap, flags = _snap(4, wtd_group_frac=0.0)
    assert snap.dims["wtd"] == 0
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        G = snap.dims["groups"]
        with_workers = [g for g in range(G) if workers_of(snap, g).size >= 4]
        first, mid, last = with_workers[0], with_workers[len(with_workers) // 2], with_workers[-1]
        lists = [[] for _ in range(G)]
        lists[first] = [int(snap.p_name_id[r]) for r in workers_of(snap, first)[:2]]
        lists[last] = [int(snap.p_name_id[workers_of(snap, last)[-1]])]
        dr.set_wtd_lists(lists)
        _, names = dr.check(oracle_mod, expect_incremental=True, profiled=True)
        assert "k_inc_wtd_resolve" in names and "k_inc_wtd_release" not in names, names   # (no old names to release)
        lists[mid] = [int(snap.p_name_id[r]) for r in workers_of(snap, mid)[:3]] + [GHOST]
        lists[first] = lists[first][1:]                                       # every later offset moves
        dr.set_wtd_lists(lists)
        dr.check(oracle_mod, expect_incremental=True)
        lists[first] = [int(snap.p_name_id[r]) for r in workers_of(snap, first)[1:4]]
        lists[last] = []
        dr.set_wtd_lists(lists)
        dr.check(oracle_mod, expect_incremental=True)
        dr.set_wtd_lists([[] for _ in range(G)])
        _, names = dr.check(oracle_mod, expect_incremental=True, profiled=True)
        assert "k_inc_wtd_release" in names and "k_inc_wtd_resolve" not in names, names
        rows = np.arange(3, snap.dims["pods"], 97, dtype=np.uint32)
        flip_ready(dr.snap, rows)
        dr.commit_rows(rows)
        _, names = dr.check(oracle_mod, expect_incremental=True, profiled=True)
        assert not set(REBUILD) & set(names), names                           # an epoch without an edit rebuilds nothing
        dr.eng.set_incremental(False)
        dr.check(oracle_mod, expect_incremental=False)                        # a full pass over what the epochs left
    finally:
        dr.close()


def test_duplicate_names(oracle_mod):
    snap, flags = _snap(5)
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        lists = lists_of(dr.snap)
        multi = [c for c in range(snap.dims["clusters"]) if snap.c_group_cnt[c] >= 2][:4]
        for c in multi:
            a, b = int(snap.c_group_off[c]), int(snap.c_group_off[c]) + 1
            if not workers_of(snap, a).size:
                continue
            x = int(snap.p_name_id[workers_of(snap, a)[0]])
            lists[a] = [x, x] + lists[a]          # twice in its own group's list
            lists[b] = lists[b] + [x]             # and in another group's
        dr.set_wtd_lists(lists)
        dr.check(oracle_mod, expect_incremental=True)
        for c in multi:
            a = int(snap.c_group_off[c])
            lists[a] = lists[a][1:]
        dr.set_wtd_lists(lists)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


@pytest.mark.parametrize("pods_first", [False, True])
@pytest.mark.parametrize("what", ["deleted", "readded", "moved"])
def test_named_pod_changes_in_the_same_epoch(what, pods_first, oracle_mod):
    snap, flags = _snap(6)
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        s = dr.snap
        lists = lists_of(s)
        gs = [g for g in range(s.dims["groups"]) if lists[g] and workers_of(s, g).size >= 4][:5]
        # free rows one epoch earlier (Pods deleted)
        free = [int(workers_of(s, g)[-1]) for g in gs]
        for c in POD_COLS:
            s.cols[c][free] = 0
        s.p_packed[free] = np.uint32(abi.PP_TOMBSTONE)
        dr.commit_rows(free)
        dr.check(oracle_mod, expect_incremental=True)
        named = [int(workers_of(s, g)[0]) for g in gs]
        for g, r in zip(gs, named):
            lists[g][0] = int(s.p_name_id[r])
        new = with_wtd_lists(s, lists)
        rows = list(named)
        if what == "deleted":
            for c in POD_COLS:
                new.cols[c][named] = 0
            new.p_packed[named] = np.uint32(abi.PP_TOMBSTONE)
        elif what == "readded":       # the same Pod (same name) comes back in a free row
            for c in POD_COLS:
                new.cols[c][free] = new.cols[c][named]
                new.cols[c][named] = 0
            new.p_packed[named] = np.uint32(abi.PP_TOMBSTONE)
            rows += free
        else:                          # the same name under another RayCluster of the same namespace
            for r in named:
                ns = new.p_ns_id[r]
                others = np.flatnonzero((new.c_ns_id == ns) & (new.c_name_id != new.p_cluster_name_id[r]) & (new.c_group_cnt > 0))
                c2 = int(others[0])
                new.p_cluster_name_id[r] = new.c_name_id[c2]
                new.p_group_name_id[r] = new.g_name_id[int(new.c_group_off[c2])]
        dr.use(new)
        if pods_first:
            dr.commit_rows(rows)
            dr.commit_objects()
        else:
            dr.commit_objects()
            dr.commit_rows(rows)
        dr.check(oracle_mod, expect_incremental=True)
        dr.set_wtd_lists([[] for _ in range(s.dims["groups"])])
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


def test_multihost_lists(oracle_mod):
    """Whole-replica deletes through the list (KR_ERR_MH_WTD), and g_wtd_cnt moving with names that resolve to nothing (decide_multihost2
    reads the count itself)."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=300, pods_per_cluster=42, groups=2, multihost_frac=0.5, autoscaling_frac=1.0,
                                                           wtd_group_frac=0.3, seed=7))
    assert flags.gate_multihost_indexing == 1
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        lists = lists_of(snap)
        mh = [g for g in range(snap.dims["groups"]) if snap.g_num_hosts[g] > 1 and workers_of(snap, g).size >= 8]
        named, ghosts = mh[:6], [g for g in mh[6:] if not lists[g]][:6]
        assert named and ghosts
        for g in named:
            lists[g] = [int(snap.p_name_id[workers_of(snap, g)[4]])]
        dr.set_wtd_lists(lists)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        assert (got.clusters["err_kind"][snap.g_cluster_idx[named]] == abi.ERR_MH_WTD).any()
        for g in ghosts:
            lists[g] = [GHOST + g]
        dr.set_wtd_lists(lists)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        assert (got.groups["flags"][ghosts] & abi.GR_WTD_EXECUTED).any()
        for g in named + ghosts:
            lists[g] = []
        dr.set_wtd_lists(lists)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        assert not (got.groups["flags"][ghosts] & abi.GR_WTD_EXECUTED).any()
    finally:
        dr.close()


def test_edits_inside_large_huge_wide_and_recreate_clusters(oracle_mod):
    snap, flags = synthetic.generate(synthetic.config("C2", n_clusters=700, pods_per_cluster=16, groups=1, n_wide=2, wide_groups=40,
                                                      recreate_frac=0.05, autoscaling_frac=1.0, wtd_group_frac=0.2, seed=8))
    huge, large = 350, 0                                       # (cluster 0 is wide as well)
    synthetic.grow_clusters(snap, [huge], abi.LARGE_MAX_PODS + 1500)
    synthetic.grow_clusters(snap, [large], 600)
    g35 = int(snap.c_group_off[large]) + 35
    snap.p_group_name_id[workers_of(snap, int(snap.c_group_off[large]))[:6]] = snap.g_name_id[g35]
    dr = _driver(snap, flags, large_clusters=True, wide_clusters=True, huge_clusters=True)
    try:
        _, names = dr.check(oracle_mod, expect_incremental=False, profiled=True)
        assert dr.eng.get_option(abi.OPT_BUCKET_STRIDE) != 0 and "k_huge_merge" in names, names
        s = dr.snap
        lists = lists_of(s)
        assert s.c_group_cnt[large] > 32 and workers_of(s, int(s.c_group_off[large])).size > 256
        recreate = [c for c in np.flatnonzero(s.c_flags & abi.CF_UPGRADE_RECREATE) if s.c_group_cnt[c] and workers_of(s, int(s.c_group_off[c])).size >= 2][:3]
        edits = {}
        g = int(s.c_group_off[large]); w = workers_of(s, g); edits[g] = w[[0, w.size // 2, -1]]                  # large: region ranks
        g = int(s.c_group_off[huge]); w = workers_of(s, g); edits[g] = w[[0, 8190, 8191, 8192, w.size - 1]]    # huge: across tiles
        edits[g35] = workers_of(s, g35)[:2]                                                                      # wide: group slot > 31
        for c in recreate:
            g = int(s.c_group_off[c]); edits[g] = workers_of(s, g)[:2]
        for g, rows in edits.items():
            assert rows.size
            lists[g] = [int(s.p_name_id[r]) for r in rows]
        dr.set_wtd_lists(lists)
        _, names = dr.check(oracle_mod, expect_incremental=True, profiled=True)
        assert {"k_inc_wtd_resolve", "k_decide_large", "k_huge_merge"} <= set(names), names
        # the autoscaler's next step: the named Pods are gone and the lists are cleared
        new = with_wtd_lists(dr.snap, [[] if g in edits else lst for g, lst in enumerate(lists)])
        gone = np.concatenate(list(edits.values()))
        for c in POD_COLS:
            new.cols[c][gone] = 0
        new.p_packed[gone] = np.uint32(abi.PP_TOMBSTONE)
        dr.use(new)
        dr.commit_objects()
        dr.commit_rows(gone)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


def test_option_toggled_mid_stream(oracle_mod):
    snap, flags = _snap(9)
    dr = _driver(snap, flags, wtd_edits=False)
    try:
        assert dr.eng.get_option(abi.OPT_WTD_EDITS) == 0
        dr.check(oracle_mod, expect_incremental=False)
        lists = lists_of(snap)
        gs = [g for g in range(snap.dims["groups"]) if workers_of(snap, g).size >= 3][:8]

        def edit(k):
            for g in gs:
                lists[g] = [int(snap.p_name_id[r]) for r in workers_of(snap, g)[:k]]
            dr.set_wtd_lists(lists)

        for step, (on, k) in enumerate([(False, 1), (True, 2), (True, 2), (False, 2), (True, 1), (True, 0), (False, 1)]):
            dr.eng.set_wtd_edits(on)
            assert dr.eng.get_option(abi.OPT_WTD_EDITS) == int(on)
            if step == 2:                           # a rename: same lengths, other names
                for g in gs:
                    lists[g] = [int(snap.p_name_id[r]) for r in workers_of(snap, g)[1:3]]
                dr.set_wtd_lists(lists)
            else:
                edit(k)
            dr.check(oracle_mod, expect_incremental=on)   # with the option off the same edit takes the full pass, as before
            rows = np.arange(step, snap.dims["pods"], 131, dtype=np.uint32)
            flip_ready(dr.snap, rows)
            dr.commit_rows(rows)
            dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


# ---------------------------------------------------------------------------------------------------- seeded streams
def _autoscale_arrays(rng, dr, pending):
    """One epoch of autoscaler traffic on the snapshot: last epoch's named Pods are deleted and their lists cleared; 1 % of the
    groups (at least 2) get 1-3 names of their own running workers with replicas lowered.  Returns the rows it rewrote."""
    s = dr.snap
    lists = lists_of(s)
    rows = []
    for g, named in pending.items():
        lists[g] = []
        for c in POD_COLS:
            s.cols[c][named] = 0
        s.p_packed[named] = np.uint32(abi.PP_TOMBSTONE)
        rows += list(named)
    pending.clear()
    G = s.dims["groups"]
    for g in rng.choice(G, max(2, G // 100), replace=False):
        g = int(g)
        w = workers_of(s, g, running=True)
        if lists[g] or w.size < 2:
            continue
        k = int(rng.integers(1, min(3, w.size) + 1))
        named = rng.choice(w, k, replace=False)
        lists[g] = [int(s.p_name_id[r]) for r in named]
        s.g_replicas[g] = max(0, int(s.g_replicas[g]) - k)
        pending[g] = named
    return lists, rows


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_stream_through_the_engine(seed, oracle_mod):
    rng = np.random.default_rng(seed)
    snap, flags = _snap(20 + seed, n_clusters=400, groups=2, wtd_group_frac=0.1)
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        pending = {}
        n_inc = 0
        for epoch in range(40):
            lists, rows = _autoscale_arrays(rng, dr, pending)
            new = with_wtd_lists(dr.snap, lists)
            # informer churn: 1 % PodReady flips
            flip = rng.choice(np.flatnonzero((new.p_packed & abi.PP_TOMBSTONE) == 0), max(1, new.dims["pods"] // 100), replace=False)
            flip_ready(new, flip)
            dr.use(new)
            if epoch % 2:
                dr.commit_rows(rows + flip.tolist())
                dr.commit_objects()
            else:
                dr.commit_objects()
                dr.commit_rows(rows + flip.tolist())
            got, _ = dr.check(oracle_mod)
            n_inc += incremental(got, new.dims["clusters"])
        # (an epoch may still take the full pass for a reason of its own: the action list full of abandoned runs is packed again)
        assert n_inc >= 38, n_inc
    finally:
        dr.close()


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_stream_through_the_native_packer(seed, oracle_mod):
    rng = np.random.default_rng(seed)
    clusters, pods, jobs = objects(seed, big=True)
    pk = Packer(**PACKER_CAPS, wtd_edits=True)
    try:
        assert pk.engine.get_option(abi.OPT_WTD_EDITS) == 1
        m = Mirror(copy.deepcopy(clusters), copy.deepcopy(pods), jobs, pk)
        pk.flush()
        packer_check(m, oracle_mod, lean=True)
        pending, counter = {}, [0]

        def step(epoch):
            autoscale_objects(rng, m, pending)
            events(rng, m, counter, structural=False)
        gots, _ = packer_stream(m, oracle_mod, 40, step)
        inc = [device_incremental(g) for g in gots]
        assert sum(inc) >= 36, inc
    finally:
        pk.close()


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_stream_through_the_live_arena(seed, oracle_mod):
    rng = np.random.default_rng(seed)
    clusters, pods, jobs = objects(seed, big=True)
    arena = LiveArena(clusters, pods, jobs, spare_rows=64, wtd_edits=True)
    try:
        pending, counter = {}, [0]

        def step(epoch):
            autoscale_objects(rng, arena, pending)
            events(rng, arena, counter, structural=False)
        inc = [device_incremental(g) for g in arena_stream(arena, oracle_mod, 40, step)]
        assert arena.engine.get_option(abi.OPT_WTD_EDITS) == 1
        assert sum(inc) >= 34 and arena.stats["rebase"] <= 2, (inc, arena.stats)
    finally:
        arena.close()

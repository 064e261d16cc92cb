"""KR_OPT_HUGE_CLUSTERS: RayClusters of more than KR_LARGE_MAX_PODS pods decided on the bucket pipeline, their pods put in List
order tile by tile (kuberay_b200/csrc/kr_huge.cuh: k_huge_tiles, k_huge_merge) and decided by k_decide_large.

Every pass is compared with the oracle and with the same snapshot run with the option off and KR_OPT_LARGE_CLUSTERS on (the
sort pipeline then decides it): Results.diff covers every result array except the run order inside the two arenas and
pod_start, which only mean something when the full pod lists are fetched."""
import copy

import numpy as np
import pytest

from harness import (POD_COLS, SORT_KERNELS, Driver, Mirror, arena_stream, b32, compact, device_incremental, events, grown_fleet, head_row,
                     huge_objects, members, move, packer_check, packer_stream, parity_on_off, run, scale_to, set_phase, spec_bytes, workers)
from kuberay_b200 import abi, synthetic
from kuberay_b200.engine import Engine
from kuberay_b200.live import LiveArena
from kuberay_b200.packer import Packer

pytestmark = pytest.mark.gpu

HUGE_KERNELS = {"k_match2", "k_decide2", "k_huge_tiles", "k_huge_merge", "k_decide_large"}
MAX_CREATES = 1 << 18  # (drained donor clusters ask for many pods)


def _parity(snap, flags, oracle_mod, wide=False):
    return parity_on_off(snap, flags, oracle_mod, "huge_clusters", large_clusters=True, wide_clusters=wide, max_creates=MAX_CREATES)


def _on_the_tile_path(names, stride):
    assert HUGE_KERNELS <= set(names), names
    assert not SORT_KERNELS & set(names), names
    assert stride == 64  # the rest of the fleet keeps its stride


# 8 193 .. 100 000 pods; 16 447 / 16 449 and 24 575 / 24 577 put the region's last rank (stride 64) one short of and one past a
# tile edge
@pytest.mark.parametrize("size", [8193, 12000, 16383, 16384, 16385, 16447, 16449, 24575, 24577, 40000, 100000])
def test_one_huge_cluster_stays_on_the_bucket_pipeline(size, oracle_mod):
    snap, flags = grown_fleet(size)
    got, names, stride = _parity(snap, flags, oracle_mod)
    assert got.clusters["n_pods"][0] == size
    _on_the_tile_path(names, stride)


def _decision_fleet(seed, size=12000, n_huge=3, n_clusters=2400):
    """Several huge RayClusters with their own case each (see the callers), in a fleet of ordinary ones."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=n_clusters, pods_per_cluster=20, groups=1, seed=seed, healthy=True))
    big = [0, n_clusters // 3, 2 * n_clusters // 3][:n_huge]
    synthetic.grow_clusters(snap, big, size)
    for c in big:
        snap.c_flags[c] &= ~np.uint32(abi.CF_SKIP | abi.CF_SUSPEND | abi.CF_UPGRADE_RECREATE)
        snap.c_flags[c] |= np.uint32(abi.CF_HEAD_EXPECT_OK)
        scale_to(snap, int(snap.c_group_off[c]), workers(snap, c).size)
    return snap, compact(flags), big


@pytest.mark.parametrize("random_delete", [False, True])
def test_decisions_that_span_tiles(random_delete, oracle_mod):
    snap, flags, (a, b, c) = _decision_fleet(3)
    flags.env_random_pod_delete = int(random_delete)
    wa, wb, wc = workers(snap, a), workers(snap, b), workers(snap, c)
    # a: unhealthy pods early and late in List order -> the group aborts after them
    set_phase(snap, np.concatenate([wa[100:120], wa[9000:9020]]), abi.PHASE_FAILED)
    # b: scale down by 9 000 (a delete prefix across several tiles), autoscaling on so random delete matters
    snap.c_flags[b] |= np.uint32(abi.CF_AUTOSCALING)
    scale_to(snap, int(snap.c_group_off[b]), wb.size - 9000)
    # c: scale up across replica-index windows, labels on every pod
    snap.p_packed[wc] |= np.uint32(abi.PP_HAS_REPLICA_IDX)
    snap.p_replica_index[wc] = np.arange(wc.size, dtype=np.int32) * 2  # every even index in use
    scale_to(snap, int(snap.c_group_off[c]), wc.size + 3000)
    got, names, stride = _parity(snap, flags, oracle_mod)
    _on_the_tile_path(names, stride)
    assert got.groups["n_unhealthy"][snap.c_group_off[a]] == 40
    assert got.groups["n_create"][snap.c_group_off[c]] == 3000


@pytest.mark.parametrize("random_delete", [False, True])
def test_workers_to_delete_inside_a_huge_cluster(random_delete, oracle_mod):
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=1200, pods_per_cluster=20, groups=1, autoscaling_frac=1.0,
                                                           wtd_group_frac=1.0, seed=21))
    flags = compact(flags)
    flags.env_random_pod_delete = int(random_delete)
    c = next(c for c in range(600, 1200) if snap.g_wtd_cnt[snap.c_group_off[c]] >= 2)
    synthetic.grow_clusters(snap, [c], 10000)
    m = members(snap, c)
    set_phase(snap, m, abi.PHASE_RUNNING)
    snap.p_packed[m] &= ~np.uint32(abi.PP_RAY_TERMINATED)
    snap.c_flags[c] &= ~np.uint32(abi.CF_SKIP | abi.CF_SUSPEND | abi.CF_UPGRADE_RECREATE)
    snap.c_flags[c] |= np.uint32(abi.CF_HEAD_EXPECT_OK | abi.CF_AUTOSCALING)
    g = int(snap.c_group_off[c])
    w = workers(snap, c)
    scale_to(snap, g, w.size - 5)
    off, cnt = int(snap.g_wtd_off[g]), int(snap.g_wtd_cnt[g])
    other = snap.p_name_id[workers(snap, c + 1)[0]]
    snap.w_name_id[off:off + cnt] = [snap.p_name_id[w[-1]], np.uint32(0x7F000000 + c)] + [other] * (cnt - 2)
    got, names, stride = _parity(snap, flags, oracle_mod)
    _on_the_tile_path(names, stride)
    _, codes = got.actions_of(c)
    assert abi.ACT_DELETE_WTD in codes.tolist()
    assert (got.wtd_pod_idx[off:off + cnt] == -1).any()


def test_heads_and_suspend_inside_huge_clusters(oracle_mod):
    snap, flags, (a, b, c) = _decision_fleet(4)
    wb = workers(snap, b)  # b: a second head, late in List order
    snap.p_packed[wb[-7]] = (snap.p_packed[wb[-7]] & ~np.uint32(3 << abi.PP_NODE_TYPE_SHIFT)) | np.uint32(abi.NT_HEAD << abi.PP_NODE_TYPE_SHIFT)
    snap.g_flags[snap.c_group_off[c]] |= np.uint32(abi.GF_SUSPEND)  # c: suspended worker group
    snap.c_flags[a] |= np.uint32(abi.CF_SUSPEND)                     # a: the whole RayCluster suspended
    got, names, stride = _parity(snap, flags, oracle_mod)
    _on_the_tile_path(names, stride)
    assert got.clusters["n_heads"][b] == 2


@pytest.mark.parametrize("spin", [True, False])
def test_recreate_gate_inside_huge_clusters(spin, oracle_mod, monkeypatch):
    """Recreate-gated huge RayClusters: one whose annotation names another spec (every pod deleted), one whose annotation is the
    digest of its spec; then an incremental epoch recommits the spec JSON and the second gate flips."""
    if not spin:
        monkeypatch.setenv("KR_NO_HASH_SPIN", "1")
    snap, flags, (a, b, _c) = _decision_fleet(8)
    ah = snap.h_annot_hash.reshape(-1, 32)
    for cl, match in ((a, False), (b, True)):
        snap.c_flags[cl] |= np.uint32(abi.CF_UPGRADE_RECREATE)
        h = head_row(snap, cl)
        snap.h_version_state[h] = abi.VER_CURRENT
        snap.h_annot_state[h] = abi.ANNOT_HASH32
        digest = b32(spec_bytes(snap, cl))
        ah[h] = np.frombuffer(digest if match else digest[::-1], dtype=np.uint8)
    got, names, stride = _parity(snap, flags, oracle_mod)
    _on_the_tile_path(names, stride)
    assert got.clusters["path"][a] == abi.PATH_RECREATE_DELETE_ALL and got.clusters["path"][b] == abi.PATH_NORMAL
    dr = Driver(snap, flags, max_creates=MAX_CREATES, large_clusters=True, huge_clusters=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        snap.json[int(snap.c_json_off[b]) + 3] ^= 0x20  # b's spec no longer matches its annotation
        np.copyto(dr.views["json"], snap.json)
        dr.eng.commit(abi.PART_JSON)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        assert got.clusters["path"][b] == abi.PATH_RECREATE_DELETE_ALL
    finally:
        dr.close()


def test_multihost_group_inside_a_huge_cluster(oracle_mod):
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=800, pods_per_cluster=20, groups=2, multihost_frac=0.25, seed=9))
    synthetic.grow_clusters(snap, [0], 9000)
    for gate in (1, 0):
        flags.gate_multihost_indexing = gate
        _, names, stride = _parity(snap, compact(flags), oracle_mod)
        _on_the_tile_path(names, stride)


def test_a_huge_cluster_that_is_also_wide(oracle_mod):
    snap, flags = grown_fleet(10000, n_clusters=800)
    snap = synthetic.widen_clusters(snap, [0], 40)
    _, names, stride = _parity(snap, flags, oracle_mod, wide=True)
    _on_the_tile_path(names, stride)


def test_huge_large_wide_and_ordinary_clusters_together(oracle_mod):
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=1500, pods_per_cluster=20, groups=1, seed=17))
    synthetic.grow_clusters(snap, [0, 700], 9500)
    synthetic.grow_clusters(snap, [300, 1000, 0, 700], 2000)  # (0 and 700 listed so that they give no pods)
    snap = synthetic.widen_clusters(snap, [700, 1000, 1200, 1400], 36)  # a huge, a large and two ordinary wide ones
    got, names, stride = _parity(snap, compact(flags), oracle_mod, wide=True)
    _on_the_tile_path(names, stride)
    assert "k_large_sort" in names
    assert (got.clusters["n_pods"][[0, 700]] == 9500).all()


# ------------------------------------------------------------------------------------------------ the option


def test_option_defaults_off_and_round_trips():
    snap, _ = grown_fleet(300)
    eng = Engine.for_snapshot(snap)
    try:
        assert eng.get_option(abi.OPT_HUGE_CLUSTERS) == 0
        for v in (1, 1, 0, 1):
            eng.set_huge_clusters(bool(v))
            assert eng.get_option(abi.OPT_HUGE_CLUSTERS) == v
    finally:
        eng.close()


def test_no_effect_without_the_large_option(oracle_mod):
    snap, flags = grown_fleet(9000)
    got, names, stride = run(snap, flags, profiled=True, max_creates=MAX_CREATES, huge_clusters=True)
    assert not oracle_mod.run(snap, flags).diff(got)
    assert "k_match2" not in names and "k_huge_tiles" not in names and stride == 0


def test_turning_the_option_on_after_a_pass(oracle_mod):
    """With KR_OPT_LARGE_CLUSTERS on, a RayCluster of 9 000 pods sends the pass to the radix pipeline; turning the option on takes
    effect at the next pass (same snapshot, same sizes), and turning it off goes back."""
    snap, flags = grown_fleet(9000)
    want = oracle_mod.run(snap, flags)
    eng = Engine.for_snapshot(snap, large_clusters=True, max_creates=MAX_CREATES)
    try:
        eng.load(snap)
        for huge in (False, True, False):
            eng.set_huge_clusters(huge)
            names = {k for k, _ in eng.reconcile_profiled(flags)["kernels"]}
            assert not want.diff(eng.reconcile(flags))
            if huge:
                assert "k_huge_merge" in names and "k_scatter" not in names and eng.get_option(abi.OPT_BUCKET_STRIDE) == 64
            else:
                assert "k_scatter" in names and "k_match2" not in names and eng.get_option(abi.OPT_BUCKET_STRIDE) == 0
    finally:
        eng.close()


def test_a_fleet_without_huge_clusters_launches_nothing_new(oracle_mod):
    snap, flags = synthetic.generate(synthetic.config("C3L", n_clusters=1000))
    flags = compact(flags)
    off, names_off, _ = run(snap, flags, profiled=True, max_creates=MAX_CREATES, large_clusters=True, huge_clusters=False)
    on, names_on, _ = run(snap, flags, profiled=True, max_creates=MAX_CREATES, large_clusters=True, huge_clusters=True)
    assert names_on == names_off and "k_huge_tiles" not in names_on
    assert not off.diff(on) and not oracle_mod.run(snap, flags).diff(on)


# ------------------------------------------------------------------------------------------------ incremental epochs

@pytest.mark.parametrize("seed", [1, 2])
def test_incremental_epoch_streams(seed, oracle_mod):
    """Seeded epochs of status flips, deletions (free rows), additions and moves inside and outside two huge RayClusters; one epoch
    removes pods from every tile of one (its bucket and region are compacted), then growth past the region takes a full pass, and
    shrinking below KR_LARGE_MAX_PODS + 1 pods keeps the epochs incremental."""
    rng = np.random.default_rng(seed)
    snap, flags, big = _decision_fleet(30 + seed, size=10000, n_huge=2, n_clusters=2000)
    nc = snap.dims["clusters"]
    dr = Driver(snap, flags, max_creates=MAX_CREATES, large_clusters=True, huge_clusters=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        assert dr.eng.get_option(abi.OPT_BUCKET_STRIDE) == 64
        free, saved = np.zeros(0, dtype=np.int64), {}
        for epoch in range(8):
            rows = []
            wa, wb = workers(snap, big[0]), workers(snap, big[1])
            flip = rng.choice(wa, 40, replace=False)
            snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT); rows += flip.tolist()
            fail = rng.choice(wb, 8, replace=False)
            set_phase(snap, fail, abi.PHASE_FAILED if epoch % 2 == 0 else abi.PHASE_RUNNING); rows += fail.tolist()
            small = rng.choice(np.setdiff1d(np.arange(nc), big), 6, replace=False)
            ws = np.concatenate([workers(snap, s)[:1] for s in small])
            snap.p_packed[ws] ^= np.uint32(1 << abi.PP_READY_SHIFT); rows += ws.tolist()
            # the pods deleted one epoch earlier come back (the first two into a huge cluster)
            for r in free.tolist():
                for col in POD_COLS:
                    snap.cols[col][r] = saved[r][col]
            if free.size:
                move(snap, free[:2], big[epoch % 2])
            rows += free.tolist()
            # deletions -> free rows, from both huge clusters and an ordinary one
            gone = np.concatenate([rng.choice(np.setdiff1d(wa, flip), 6, replace=False), rng.choice(np.setdiff1d(wb, fail), 3, replace=False),
                                   workers(snap, int(small[0]))[1:2]])
            saved = {int(r): {col: snap.cols[col][r].copy() for col in POD_COLS} for r in gone}
            for col in POD_COLS:
                snap.cols[col][gone] = 0
            snap.p_packed[gone] = np.uint32(abi.PP_TOMBSTONE)
            free = gone
            rows += gone.tolist()
            # moves between a huge and an ordinary cluster, both ways
            out = rng.choice(np.setdiff1d(workers(snap, big[0]), np.concatenate([flip, gone])), 3, replace=False)
            move(snap, out, int(small[1]))
            into = workers(snap, int(small[2]))[:2]
            move(snap, into, big[1])
            rows += out.tolist() + into.tolist()
            dr.commit_rows(rows, journal=epoch % 2 == 0)
            dr.check(oracle_mod, expect_incremental=True)
        # pods leave every tile of big[0]: its bucket and region are compacted in arrival order
        wa = workers(snap, big[0])
        out = rng.choice(wa, 400, replace=False)
        dests = np.setdiff1d(np.arange(nc), big)[:400]
        for r, d in zip(out.tolist(), dests.tolist()):
            move(snap, np.array([r]), d)
        dr.commit_rows(out)
        dr.check(oracle_mod, expect_incremental=True)
        flip = workers(snap, big[0])[::97]
        snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        dr.commit_rows(flip)
        dr.check(oracle_mod, expect_incremental=True)
        # replicas of a huge cluster through the object commit
        snap.g_replicas[snap.c_group_off[big[1]]] -= 1000
        dr.commit_objects()
        dr.check(oracle_mod, expect_incremental=True)
        # shrinking below KR_LARGE_MAX_PODS + 1 pods: still on the tile path, still incremental
        wb = workers(snap, big[1])
        out = wb[:wb.size - 8000]
        dests = np.setdiff1d(np.arange(nc), big)
        for i in range(0, out.size, 30):  # (30 more pods per ordinary cluster keep it within the stride)
            move(snap, out[i:i + 30], int(dests[i // 30 + 500]))
        dr.commit_rows(out)
        dr.check(oracle_mod, expect_incremental=True)
        assert members(snap, big[1]).size <= abi.LARGE_MAX_PODS
        flip = workers(snap, big[1])[::50]
        snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        dr.commit_rows(flip)
        dr.check(oracle_mod, expect_incremental=True)
        # growth past big[0]'s region (about 1.25x its pods at the last full pass): one full pass, then incremental again
        donors = np.concatenate([workers(snap, c) for c in range(1000, 2000) if c not in big])[:4000]
        move(snap, donors, big[0])
        dr.commit_rows(donors)
        dr.check(oracle_mod, expect_incremental=False)
        assert dr.eng.get_option(abi.OPT_BUCKET_STRIDE) == 64
        flip = workers(snap, big[0])[::31]
        snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        dr.commit_rows(flip)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


# ------------------------------------------------------------------------------------------------ the ingestion side

def test_native_packer_keeps_incremental_epochs_with_a_huge_cluster(oracle_mod):
    rng = np.random.default_rng(41)
    clusters, pods, jobs = huge_objects(5, 9000)
    pk = Packer(max_clusters=256, max_groups=4096, max_wtd=4096, max_pods=32768, max_heads=1024, max_jobs=64, max_creates=1 << 16,
                max_json_bytes=4 << 20, large_clusters=True, huge_clusters=True)
    try:
        m = Mirror(copy.deepcopy(clusters), copy.deepcopy(pods), jobs, pk)
        pk.flush()
        _, first = packer_check(m, oracle_mod, lean=True)
        assert int(first.clusters["n_pods"].max()) >= 9000
        assert pk.engine.get_option(abi.OPT_HUGE_CLUSTERS) == 1 and pk.engine.get_option(abi.OPT_BUCKET_STRIDE) != 0
        counter = [0]
        gots, modes = packer_stream(m, oracle_mod, 10, lambda epoch: events(rng, m, counter, structural=False))
        incremental = [device_incremental(g) for g in gots]
        assert any(mo & abi.PACK_POD_ROWS for mo in modes)
        # (the cloned pods are surplus workers: the huge cluster's ~9 000 scale-down deletes take one action run, and an epoch that
        # adds to it needs a new run, which the action list may not hold beside the abandoned one; that epoch takes the full pass,
        # which packs the list again)
        assert sum(incremental) >= 5, incremental
    finally:
        pk.close()


def test_live_arena_keeps_incremental_epochs_with_a_huge_cluster(oracle_mod):
    rng = np.random.default_rng(43)
    clusters, pods, jobs = huge_objects(7, 9000)
    live = LiveArena(clusters, pods, jobs, spare_rows=64, large_clusters=True, huge_clusters=True)
    counter = [0]
    try:
        def step(epoch):
            if epoch == 1:  # (epoch 0's pass, the first one, took the bucket pipeline)
                assert live.engine.get_option(abi.OPT_BUCKET_STRIDE) != 0
            events(rng, live, counter, structural=False)
        gots = arena_stream(live, oracle_mod, 12, step)
        assert all(int(got.clusters["n_pods"].max()) >= 8193 for got in gots)
        n_inc = sum(device_incremental(got) for got in gots)
        assert n_inc >= 6, (n_inc, live.stats)
    finally:
        live.close()

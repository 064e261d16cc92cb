"""KR_OPT_LARGE_GROWTH: a RayCluster that outgrows its bucket or its region in an incremental epoch gets a region in that epoch
(k_inc_grow, kuberay_b200/csrc/kr_large.cuh) instead of sending the pass to a full one.

Every epoch goes through harness.Driver: compared with the oracle, and every record the pass did not name equal to the previous
epoch's.  Where an epoch is expected to be incremental it is asserted to be, with the grown RayClusters among changed_clusters."""
import copy

import numpy as np
import pytest

from harness import (PACKER_CAPS, POD_COLS, Driver, Mirror, b32, device_incremental, events, head_row, most_workers, move, objects,
                     packer_check, packer_stream, scale_to, set_phase, spec_bytes, workers)
from kuberay_b200 import abi, synthetic
from kuberay_b200.packer import Packer

pytestmark = pytest.mark.gpu

GROW = dict(large_clusters=True, large_growth=True)


def _fleet(seed, n_clusters=600, groups=1, **kw):
    """RayClusters of 20 pods (the 64-pod stride), healthy, with room to scale: no group limits its replicas."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=n_clusters, pods_per_cluster=20, groups=groups, seed=seed,
                                                           healthy=True, **kw))
    for c in range(n_clusters):
        snap.c_flags[c] &= ~np.uint32(abi.CF_SKIP | abi.CF_SUSPEND)
    return snap, flags


def _grown(got, clusters):
    assert got.changed_clusters is not None
    missing = set(int(c) for c in clusters) - set(got.changed_clusters.tolist())
    assert not missing, missing


def test_stride_crossings(oracle_mod):
    """One ordinary RayCluster scales 20 -> 64 -> 128 -> 256 -> 300 Pods, one epoch per step: every epoch stays incremental and the
    fleet keeps its 64-Pod stride."""
    snap, flags = _fleet(1)
    dr = Driver(snap, flags, max_creates=1 << 16, **GROW)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        assert dr.eng.get_option(abi.OPT_BUCKET_STRIDE) == 64
        for i, rows in enumerate(synthetic.grow_epochs(snap, [300], [64, 65, 128, 129, 256, 300])):
            dr.commit_rows(rows)
            got, names = dr.check(oracle_mod, expect_incremental=True, profiled=i == 1)
            _grown(got, [300])
            assert got.clusters["n_pods"][300] == [64, 65, 128, 129, 256, 300][i]
            if i == 1:
                assert {"k_inc_admit", "k_inc_grow", "k_large_sort", "k_decide_large"} <= set(names), names
            assert dr.eng.get_option(abi.OPT_BUCKET_STRIDE) == 64
        flip = workers(snap, 300)[::7].tolist() + workers(snap, 5)[:3].tolist()
        snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        dr.commit_rows(flip)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


@pytest.mark.parametrize("options", [dict(large_clusters=True), dict(large_growth=True)], ids=["growth_off", "large_off"])
def test_without_the_options_growth_is_a_full_pass(options, oracle_mod):
    """The twin of test_stride_crossings with KR_OPT_LARGE_GROWTH off, and with it on but KR_OPT_LARGE_CLUSTERS off: the stride
    crossing is a full pass, and the epoch after it incremental again."""
    snap, flags = _fleet(1)
    dr = Driver(snap, flags, max_creates=1 << 16, **options)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        for rows in synthetic.grow_epochs(snap, [300], [65]):
            dr.commit_rows(rows)
            dr.check(oracle_mod, expect_incremental=False)
        flip = workers(snap, 300)[::7]
        snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        dr.commit_rows(flip)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


def test_regrowth_with_pods_leaving(oracle_mod):
    """A large RayCluster outgrows its region twice while some of its Pods leave in the same epochs: the stale records of the old
    region are copied with the live ones and dropped by the compaction."""
    snap, flags = _fleet(2)
    synthetic.grow_clusters(snap, [10], 400)
    dr = Driver(snap, flags, max_creates=1 << 16, **GROW)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rng = np.random.default_rng(5)
        for size in (700, 1300):
            leave = rng.choice(workers(snap, 10), 25, replace=False)
            rows = next(synthetic.grow_epochs(snap, [10], [size + 25]))
            move(snap, leave, 200)
            dr.commit_rows(np.concatenate([rows, leave]))
            got, _ = dr.check(oracle_mod, expect_incremental=True)
            _grown(got, [10, 200])
            assert got.clusters["n_pods"][10] == size
        assert dr.eng.get_option(abi.OPT_BUCKET_STRIDE) == 64
    finally:
        dr.close()


def test_several_at_once_with_other_events(oracle_mod):
    snap, flags = _fleet(3)
    dr = Driver(snap, flags, max_creates=1 << 16, **GROW)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        grow = [20, 40, 60, 80, 100, 120]
        rows = next(synthetic.grow_epochs(snap, grow, [150]))
        gone = workers(snap, 250)[:4]
        snap.p_packed[gone] |= np.uint32(abi.PP_TOMBSTONE)
        fail = workers(snap, 251)[:3]
        set_phase(snap, fail, abi.PHASE_FAILED)
        flip = workers(snap, 252)[:5]
        snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        dr.commit_rows(np.concatenate([rows, gone, fail, flip]))
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        _grown(got, grow + [250, 251, 252])
        # and again past the regions the first epoch gave
        rows = next(synthetic.grow_epochs(snap, grow[:3], [400]))
        dr.commit_rows(rows)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        _grown(got, grow[:3])
    finally:
        dr.close()


def test_promoted_cluster_with_a_recreate_gate(oracle_mod):
    """A Recreate-gated RayCluster promoted in an epoch that also re-hashes its spec, and in one that does not."""
    snap, flags = _fleet(4)
    c = 30
    snap.c_flags[c] |= np.uint32(abi.CF_UPGRADE_RECREATE)
    h = head_row(snap, c)
    snap.h_version_state[h] = abi.VER_CURRENT
    snap.h_annot_state[h] = abi.ANNOT_HASH32
    snap.h_annot_hash.reshape(-1, 32)[h] = np.frombuffer(b32(spec_bytes(snap, c)), dtype=np.uint8)
    dr = Driver(snap, flags, max_creates=1 << 16, **GROW)
    try:
        got, _ = dr.check(oracle_mod, expect_incremental=False)
        assert got.clusters["path"][c] == abi.PATH_NORMAL
        steps = synthetic.grow_epochs(snap, [c], [100, 200])
        dr.commit_rows(next(steps))
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        _grown(got, [c])
        snap.json[int(snap.c_json_off[c]) + 3] ^= 0x20  # its spec no longer matches the annotation
        np.copyto(dr.views["json"], snap.json)
        dr.eng.commit(abi.PART_JSON)
        dr.commit_rows(next(steps))
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        _grown(got, [c])
        assert got.clusters["path"][c] == abi.PATH_RECREATE_DELETE_ALL
    finally:
        dr.close()


def test_promoted_cluster_with_a_multihost_group(oracle_mod):
    snap, flags = _fleet(5, n_clusters=400, groups=2, multihost_frac=0.25)
    c = next(c for c in range(100, 400) if (snap.g_num_hosts[int(snap.c_group_off[c]):int(snap.c_group_off[c]) + 2] > 1).any())
    dr = Driver(snap, flags, max_creates=1 << 16, **GROW)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        for rows in synthetic.grow_epochs(snap, [c], [90, 180]):
            dr.commit_rows(rows)
            got, _ = dr.check(oracle_mod, expect_incremental=True)
            _grown(got, [c])
    finally:
        dr.close()


def test_promoted_cluster_with_workers_to_delete(oracle_mod):
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=600, pods_per_cluster=20, groups=1, autoscaling_frac=1.0,
                                                           wtd_group_frac=1.0, seed=21))
    c = next(c for c in range(300, 600) if snap.g_wtd_cnt[snap.c_group_off[c]] >= 1)
    snap.c_flags[c] &= ~np.uint32(abi.CF_SKIP | abi.CF_SUSPEND | abi.CF_UPGRADE_RECREATE)
    snap.c_flags[c] |= np.uint32(abi.CF_HEAD_EXPECT_OK | abi.CF_AUTOSCALING)
    g = int(snap.c_group_off[c])
    dr = Driver(snap, flags, max_creates=1 << 16, wtd_edits=True, **GROW)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rows = next(synthetic.grow_epochs(snap, [c], [150]))
        set_phase(snap, rows, abi.PHASE_RUNNING)
        snap.p_packed[rows] &= ~np.uint32(abi.PP_RAY_TERMINATED)
        scale_to(snap, g, workers(snap, c).size - 2)
        off = int(snap.g_wtd_off[g])
        snap.w_name_id[off] = snap.p_name_id[workers(snap, c)[-1]]  # a Pod that just joined
        dr.commit_objects()
        dr.commit_rows(rows)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        _grown(got, [c])
        assert abi.ACT_DELETE_WTD in got.actions_of(c)[1].tolist()
    finally:
        dr.close()


def test_promoted_wide_cluster_is_decided_once(oracle_mod):
    """A RayCluster of more than 32 worker groups (KR_OPT_WIDE_CLUSTERS: on the per-cluster list already) outgrows its bucket: it
    gets a region and stays one entry of the list."""
    snap, flags = _fleet(7, n_clusters=300)
    snap = synthetic.widen_clusters(snap, [40], 40)
    dr = Driver(snap, flags, max_creates=1 << 16, wide_clusters=True, **GROW)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rows = next(synthetic.grow_epochs(snap, [40], [120]))
        dr.commit_rows(rows)
        got, names = dr.check(oracle_mod, expect_incremental=True, profiled=True)
        _grown(got, [40])
        assert "k_inc_grow" in names and "k_decide_large" in names
    finally:
        dr.close()


def test_created_cluster_adopts_more_than_its_bucket(oracle_mod):
    """KR_OPT_CLUSTER_CREATES: a RayCluster appended after the last row adopts more resident orphan Pods than its bucket holds."""
    full, flags = _fleet(8, n_clusters=401)
    synthetic.grow_clusters(full, [400], 100)
    before = synthetic.first_clusters(full, 400, free_pods=False)
    dr = Driver(full, flags, slack=1.25, max_creates=1 << 16, cluster_creates=True, **GROW)
    try:
        dr.use(before)
        dr.commit_objects(abi.PART_ALL)
        for c in POD_COLS:
            dr.views[c][:] = before.cols[c]
        dr.eng.commit(abi.PART_ALL)
        dr.check(oracle_mod, expect_incremental=False)
        dr.prev = None  # (the RayCluster count changes: Driver.check compares records of equal shapes only)
        dr.use(full)
        dr.commit_objects()
        np.copyto(dr.views["json"], full.json)
        dr.eng.commit_spec_rows(np.array([400], dtype=np.uint32))
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        _grown(got, [400])
        assert got.clusters["n_pods"][400] == 100
    finally:
        dr.close()


def test_past_the_largest_cluster_is_a_full_pass(oracle_mod):
    for huge in (False, True):
        snap, flags = _fleet(9, n_clusters=700)
        dr = Driver(snap, flags, max_creates=1 << 16, huge_clusters=huge, **GROW)
        try:
            dr.check(oracle_mod, expect_incremental=False)
            rows = next(synthetic.grow_epochs(snap, [600], [abi.LARGE_MAX_PODS + 1]))
            dr.commit_rows(rows)
            dr.check(oracle_mod, expect_incremental=False)
            flip = workers(snap, 600)[::97]
            snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
            dr.commit_rows(flip)
            dr.check(oracle_mod, expect_incremental=huge)
        finally:
            dr.close()


def test_more_promotions_than_the_grow_list_holds(oracle_mod):
    snap, flags = _fleet(10)
    dr = Driver(snap, flags, max_creates=1 << 16, **GROW)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rows = next(synthetic.grow_epochs(snap, list(range(65)), [70]))
        dr.commit_rows(rows)
        dr.check(oracle_mod, expect_incremental=False)
        flip = workers(snap, 3)[:5]
        snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        dr.commit_rows(flip)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


def test_the_list_cap(oracle_mod):
    """40 promotions fit the per-cluster list of a 600-RayCluster fleet (64 entries); 30 more in the next epoch would pass it."""
    snap, flags = _fleet(11)
    dr = Driver(snap, flags, max_creates=1 << 16, **GROW)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rows = next(synthetic.grow_epochs(snap, list(range(40)), [70]))
        dr.commit_rows(rows)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        _grown(got, range(40))
        rows = next(synthetic.grow_epochs(snap, list(range(40, 70)), [70]))
        dr.commit_rows(rows)
        dr.check(oracle_mod, expect_incremental=False)
        flip = workers(snap, 45)[:5]
        snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        dr.commit_rows(flip)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


def _region_cap(count, stride):
    """large_region_cap (kr_bucket2.cuh) for a RayCluster of at most LARGE_MAX_PODS Pods."""
    return min((count + count // 4 + 31) // 32 * 32, abi.LARGE_MAX_PODS) - stride


def test_a_full_region_arena(oracle_mod):
    """Repeated regrowth on small capacities: 24 RayClusters step up together, each step just past the room the last one gave, so
    every step abandons their regions and allocates larger ones past them.  The region arena (1.25 x max_pods + 32 per possible
    large RayCluster, kr_engine.cu) is sized so that the abandoned regions fill it at a known step, and at no other cap: that step
    is a full pass, which lays the regions out again from offset 0, and the next step fits again."""
    snap, flags = _fleet(12)
    grow = list(range(560, 584))
    sizes = [65, 97, 129, 193, 257, 353]
    dr = Driver(snap, flags, max_creates=1 << 16, **GROW)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        stride = dr.eng.get_option(abi.OPT_BUCKET_STRIDE)
        assert stride == 64
        np_ = dr.eng.cfg.max_pods
        arena = np_ * 5 // 4 + 32 * (np_ // 257 + 1)
        used, full_at = 0, None
        for k, size in enumerate(sizes[:-1]):
            used += len(grow) * _region_cap(size, stride)
            if used > arena:
                full_at = k
                break
        assert full_at == 4, (used, arena)  # (the fleet's shape puts the arena's end at the fifth step)
        for k, rows in enumerate(synthetic.grow_epochs(snap, grow, sizes)):
            dr.commit_rows(rows)
            got, _ = dr.check(oracle_mod, expect_incremental=k != full_at)
            if k != full_at:
                _grown(got, grow)
            assert dr.eng.get_option(abi.OPT_BUCKET_STRIDE) == 64
    finally:
        dr.close()


def test_a_later_full_pass(oracle_mod):
    """A full pass after promotions gives the same results and lays the regions out again; the epochs after it are incremental."""
    snap, flags = _fleet(13)
    dr = Driver(snap, flags, max_creates=1 << 16, **GROW)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        steps = synthetic.grow_epochs(snap, [7, 8], [100, 200, 350])
        dr.commit_rows(next(steps))
        inc, _ = dr.check(oracle_mod, expect_incremental=True)
        dr.eng.set_incremental(False)
        full, _ = dr.check(oracle_mod, expect_incremental=False)
        dr.eng.set_incremental(True)
        assert not inc.diff(full)
        flip = workers(snap, 7)[::9]  # (the pass after the option comes back is a full one: none left resident state)
        snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        dr.commit_rows(flip)
        dr.check(oracle_mod, expect_incremental=False)
        for rows in steps:
            dr.commit_rows(rows)
            got, _ = dr.check(oracle_mod, expect_incremental=True)
            _grown(got, [7, 8])
    finally:
        dr.close()


def _scaling_pods(pods, owner, n):
    src = [p for p in pods if (p.get("namespace"), p["labels"].get("ray.io/cluster")) == owner and p["labels"].get("ray.io/node-type") == "worker"]
    out = []
    for i in range(n):
        q = copy.deepcopy(src[i % len(src)])
        q["name"] = f"{q['name']}-scale-{i}"
        out.append(q)
    return out


def test_native_packer_stream(oracle_mod):
    """The native packer with the option on against a twin with it off: a RayCluster scales up past its bucket and down again over
    the epochs, beside seeded informer events.  Every epoch equals the oracle and the twin."""
    clusters, pods, jobs = objects(7, max_clusters=16)
    extra = _scaling_pods(pods, most_workers(pods), 150)
    results = []
    for growth in (True, False):
        pk = Packer(**PACKER_CAPS, large_clusters=True, large_growth=growth)
        try:
            assert pk.engine.get_option(abi.OPT_LARGE_GROWTH) == int(growth)
            m = Mirror(copy.deepcopy(clusters), copy.deepcopy(pods), jobs, pk)
            pk.flush()
            packer_check(m, oracle_mod, lean=True)
            counter, r = [0], np.random.default_rng(7)

            def step(epoch):
                k = (40, 80, 150, 60, 10, 150, 100, 0)[epoch]
                live = {q["name"] for q in m.live_pods()}
                for q in extra[:k]:
                    if q["name"] not in live:
                        m.upsert_pod(copy.deepcopy(q))
                for q in extra[k:]:
                    if q["name"] in live:
                        m.delete_pod(q.get("namespace", "default"), q["name"])
                events(r, m, counter, structural=False)

            gots, _ = packer_stream(m, oracle_mod, 8, step)
            results.append((gots, [device_incremental(g) for g in gots]))
        finally:
            pk.close()
    (on, inc_on), (off, inc_off) = results
    for a, b in zip(on, off):
        assert not a.diff(b)
    assert sum(inc_on) > sum(inc_off), (inc_on, inc_off)

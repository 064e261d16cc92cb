"""KR_OPT_WIDE_CLUSTERS: RayClusters of more than 32 worker groups decided on the bucket pipeline by the per-cluster kernels
(kuberay_b200/csrc/kr_large.cuh).

Every full pass is compared with the oracle and with the same snapshot run with the option off (the sort pipeline then decides it):
Results.diff covers every result array except the run order inside the two arenas and pod_start, which only mean something when
the full pod lists are fetched.  Incremental epochs are compared with a from-scratch oracle run after each epoch."""
import collections
import copy
import functools

import numpy as np
import pytest

from harness import (BUCKET_KERNELS, OBJ_COLS, PACKER_CAPS, POD_COLS, SORT_KERNELS, Driver, Mirror, b32, compact, device_incremental, events,
                     group_pods, head_row, lists_of, members, objects, packer_check, packer_stream, parity_on_off, run, scale_to, set_phase,
                     spec_bytes, with_wtd_lists, workers)
from kuberay_b200 import abi, synthetic
from kuberay_b200.engine import Engine
from kuberay_b200.packer import Packer

pytestmark = pytest.mark.gpu

_parity = functools.partial(parity_on_off, option="wide_clusters")


def _wide_fleet(n_groups=48, wide=(0,), n_clusters=300, pods=60, seed=12, **kw):
    """n_clusters RayClusters x 20 pods (the 64-pod stride); each of `wide` first grows to `pods` pods, then its worker group 0 is
    split into n_groups groups (its workers round-robin, so the groups past slot 32 hold pods too)."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=n_clusters, pods_per_cluster=20, groups=1, seed=seed, **kw))
    synthetic.grow_clusters(snap, list(wide), pods)
    snap = synthetic.widen_clusters(snap, list(wide), n_groups)
    return snap, compact(flags)


def _on_the_bucket_pipeline(names, stride, want_stride=64):
    assert BUCKET_KERNELS <= set(names), names
    assert not SORT_KERNELS & set(names), names
    assert stride == want_stride


# ------------------------------------------------------------------------------------------------ group-count edges

@pytest.mark.parametrize("n_groups", [33, 48, 64, 1000])
def test_one_wide_cluster_stays_on_the_bucket_pipeline(n_groups, oracle_mod):
    snap, flags = _wide_fleet(n_groups)
    got, names, stride = _parity(snap, flags, oracle_mod)
    assert snap.c_group_cnt[0] == n_groups and got.clusters["n_pods"][0] == 60
    _on_the_bucket_pipeline(names, stride)


def test_several_wide_clusters(oracle_mod):
    snap, flags = _wide_fleet(40, wide=(0, 50, 51, 150, 299))
    _, names, stride = _parity(snap, flags, oracle_mod)
    _on_the_bucket_pipeline(names, stride)


def test_every_cluster_wide(oracle_mod):
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=200, pods_per_cluster=40, groups=33, seed=5))
    _, names, stride = _parity(snap, compact(flags), oracle_mod)
    _on_the_bucket_pipeline(names, stride)


def test_a_cluster_at_the_worker_group_limit(oracle_mod):
    snap, flags = _wide_fleet(65534, wide=(7,), n_clusters=60)
    assert snap.c_group_cnt[7] == 65534
    _, names, stride = _parity(snap, flags, oracle_mod)
    _on_the_bucket_pipeline(names, stride)


def test_32_worker_groups_stay_on_the_warp_decide(oracle_mod):
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=200, pods_per_cluster=40, groups=32, seed=6))
    _, names, stride = _parity(snap, compact(flags), oracle_mod)
    assert {"k_match2", "k_decide2"} <= set(names) and not {"k_large_sort", "k_decide_large"} & set(names), names
    assert not SORT_KERNELS & set(names) and stride == 64


# ------------------------------------------------------------------------------------------------ decisions at slots >= 32

def _decision_fleet(seed, wide=(0, 100, 200), **kw):
    """Wide RayClusters of 48 groups x 60 pods, healthy, every group at its pod count (see the callers for each one's case)."""
    snap, flags = _wide_fleet(48, wide=wide, seed=seed, healthy=True, **kw)
    for c in wide:
        snap.c_flags[c] &= ~np.uint32(abi.CF_SKIP | abi.CF_SUSPEND | abi.CF_UPGRADE_RECREATE)
        snap.c_flags[c] |= np.uint32(abi.CF_HEAD_EXPECT_OK)
        for gi in range(48):
            scale_to(snap, int(snap.c_group_off[c]) + gi, group_pods(snap, c, gi).size)
    return snap, flags, list(wide)


@pytest.mark.parametrize("random_delete", [False, True])
def test_creates_scale_downs_and_unhealthy_pods_past_slot_32(random_delete, oracle_mod):
    snap, flags, (a, b, c) = _decision_fleet(3)
    flags.env_random_pod_delete = int(random_delete)
    ga, gb, gc = (int(snap.c_group_off[x]) for x in (a, b, c))
    # a: an unhealthy pod in group 40 -> the groups stop after it
    set_phase(snap, group_pods(snap, a, 40)[:1], abi.PHASE_FAILED)
    # b: autoscaling; group 33 scaled to 0 and group 47 up by 3
    snap.c_flags[b] |= np.uint32(abi.CF_AUTOSCALING)
    scale_to(snap, gb + 33, 0)
    scale_to(snap, gb + 47, group_pods(snap, b, 47).size + 3)
    # c: creates in groups 32..47 with replica-index labels on every pod
    wc = workers(snap, c)
    snap.p_packed[wc] |= np.uint32(abi.PP_HAS_REPLICA_IDX)
    snap.p_replica_index[wc] = np.arange(wc.size, dtype=np.int32) % 3
    for gi in range(32, 48):
        scale_to(snap, gc + gi, group_pods(snap, c, gi).size + gi - 30)
    got, names, stride = _parity(snap, flags, oracle_mod)
    _on_the_bucket_pipeline(names, stride)
    assert got.groups["n_unhealthy"][ga + 40] == 1 and got.clusters["stop_after_group"][a] == 40
    assert got.groups["n_create"][gb + 47] == 3
    assert (got.groups["n_create"][gc + 32:gc + 48] == np.arange(2, 18)).all()
    _, codes = got.actions_of(b)
    assert (abi.ACT_DELETE_RANDOM in codes.tolist()) == bool(random_delete)


@pytest.mark.parametrize("random_delete", [False, True])
def test_workers_to_delete_past_slot_32(random_delete, oracle_mod):
    snap, flags, (a, b, _c) = _decision_fleet(4)
    flags.env_random_pod_delete = int(random_delete)
    lists = {}
    for x in (a, b):
        snap.c_flags[x] |= np.uint32(abi.CF_AUTOSCALING)
        g0 = int(snap.c_group_off[x])
        own = group_pods(snap, x, 41)
        other = group_pods(snap, x, 3)[0]  # a pod of another group of the same cluster
        scale_to(snap, g0 + 41, own.size - 1)
        lists[g0 + 41] = [snap.p_name_id[own[-1]], snap.p_name_id[other], 0x7F000000 + x]
        lists[g0 + 35] = [snap.p_name_id[workers(snap, x + 1)[0]]]  # a pod of another RayCluster
    new = lists_of(snap)
    for g, names in lists.items():
        new[g] = names
    snap = with_wtd_lists(snap, new)
    got, names, stride = _parity(snap, flags, oracle_mod)
    _on_the_bucket_pipeline(names, stride)
    for x in (a, b):
        g = int(snap.c_group_off[x]) + 41
        _, codes = got.actions_of(x)
        assert abi.ACT_DELETE_WTD in codes.tolist()
        assert got.groups["flags"][g] & abi.GR_WTD_EXECUTED
        off = int(snap.g_wtd_off[g])
        assert got.wtd_pod_idx[off + 2] == -1  # the name no pod carries


def test_heads_and_suspend_inside_wide_clusters(oracle_mod):
    snap, flags, (a, b, c, _d) = _decision_fleet(5, wide=(0, 100, 200, 250))
    # a: a second head; b: an unhealthy head; c: worker group 44 suspended; 250: the whole RayCluster suspended
    wa = workers(snap, a)
    snap.p_packed[wa[7]] = (snap.p_packed[wa[7]] & ~np.uint32(3 << abi.PP_NODE_TYPE_SHIFT)) | np.uint32(abi.NT_HEAD << abi.PP_NODE_TYPE_SHIFT)
    head_b = members(snap, b)[((snap.p_packed[members(snap, b)] >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_HEAD]
    set_phase(snap, head_b, abi.PHASE_FAILED)
    snap.g_flags[int(snap.c_group_off[c]) + 44] |= np.uint32(abi.GF_SUSPEND)
    snap.c_flags[250] |= np.uint32(abi.CF_SUSPEND)
    got, names, stride = _parity(snap, flags, oracle_mod)
    _on_the_bucket_pipeline(names, stride)
    assert got.clusters["n_heads"][a] == 2 and got.clusters["head_action"][b] == abi.HEAD_DELETE
    _, codes = got.actions_of(c)
    assert abi.ACT_DELETE_GROUP_SUSPEND in codes.tolist()


@pytest.mark.parametrize("spin", [True, False])
def test_recreate_gates_inside_wide_clusters(spin, oracle_mod, monkeypatch):
    """Recreate-gated wide RayClusters: one whose annotation names another spec (every pod deleted), one whose annotation is the
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
    _on_the_bucket_pipeline(names, stride)
    assert got.clusters["path"][a] == abi.PATH_RECREATE_DELETE_ALL and got.clusters["path"][b] == abi.PATH_NORMAL
    dr = Driver(snap, flags, max_creates=1 << 16, wide_clusters=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        snap.json[int(snap.c_json_off[b]) + 3] ^= 0x20  # b's spec no longer matches its annotation
        np.copyto(dr.views["json"], snap.json)
        dr.eng.commit(abi.PART_JSON)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        assert got.clusters["path"][b] == abi.PATH_RECREATE_DELETE_ALL
    finally:
        dr.close()


def test_multihost_groups_inside_a_wide_cluster(oracle_mod):
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=300, pods_per_cluster=20, groups=2, multihost_frac=0.5, seed=9))
    c = next(c for c in range(300) if snap.g_num_hosts[snap.c_group_off[c]] == 4)
    synthetic.grow_clusters(snap, [c], 60)
    snap = synthetic.widen_clusters(snap, [c], 40)  # every one of its first 40 groups multi-host, replicas spread over them
    for gate in (1, 0):
        flags.gate_multihost_indexing = gate
        _, names, stride = _parity(snap, compact(flags), oracle_mod)
        _on_the_bucket_pipeline(names, stride)


def test_wide_and_large_together(oracle_mod):
    """A 40-group RayCluster of 3 000 pods: with both options a region and the per-cluster kernels; with the wide option alone the
    stride cannot hold it and the sort pipeline decides, as before."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=600, pods_per_cluster=20, groups=1, seed=11))
    synthetic.grow_clusters(snap, [10], 3000)
    snap = synthetic.widen_clusters(snap, [10], 40)
    flags = compact(flags)
    got, names, stride = _parity(snap, flags, oracle_mod, large_clusters=True)
    _on_the_bucket_pipeline(names, stride)
    assert got.clusters["n_pods"][10] == 3000
    only_wide, names, stride = run(snap, flags, profiled=True, wide_clusters=True)
    assert not oracle_mod.run(snap, flags).diff(only_wide)
    assert "k_match2" not in names and "k_decide_large" not in names and stride == 0


# ------------------------------------------------------------------------------------------------ incremental epochs

def test_incremental_epochs_in_wide_clusters(oracle_mod):
    snap, flags, big = _decision_fleet(6)
    rng = np.random.default_rng(3)
    dr = Driver(snap, flags, max_creates=1 << 16, wide_clusters=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        assert dr.eng.get_option(abi.OPT_BUCKET_STRIDE) == 64
        for epoch in range(6):
            rows = []
            # status flips and failures in groups >= 32
            hi = np.concatenate([group_pods(snap, big[0], gi) for gi in range(32, 48)])
            flip = rng.choice(hi, 6, replace=False)
            snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT); rows += flip.tolist()
            fail = np.concatenate([group_pods(snap, big[1], gi) for gi in (33, 40)])
            set_phase(snap, fail, abi.PHASE_FAILED if epoch % 2 == 0 else abi.PHASE_RUNNING); rows += fail.tolist()
            # a pod of group 45 deleted (a free row) and pods moving between a wide and an ordinary cluster, both ways (as many
            # leave big[2] as join it: its bucket holds 64 records and the stale ones leave only when the epoch compacts it)
            gone = group_pods(snap, big[2], 45)[:1]
            for col in POD_COLS:
                snap.cols[col][gone] = 0
            snap.p_packed[gone] = np.uint32(abi.PP_TOMBSTONE)
            rows += gone.tolist()
            small = int(rng.integers(1, 99))
            out = group_pods(snap, big[2], 33 + epoch)[:1]
            snap.p_ns_id[out], snap.p_cluster_name_id[out] = snap.c_ns_id[small], snap.c_name_id[small]
            snap.p_group_name_id[out] = snap.g_name_id[snap.c_group_off[small]]
            into = workers(snap, small)[:1]
            g = int(snap.c_group_off[big[2]]) + 40 + epoch
            snap.p_ns_id[into], snap.p_cluster_name_id[into] = snap.c_ns_id[big[2]], snap.c_name_id[big[2]]
            snap.p_group_name_id[into] = snap.g_name_id[g]
            rows += out.tolist() + into.tolist()
            dr.commit_rows(rows, journal=epoch % 2 == 0)
            got, _ = dr.check(oracle_mod, expect_incremental=True)
            assert set(big) <= set(got.changed_clusters.tolist())
        # replica edits of group 40 through the object commit, and through the row-granular one
        g40 = int(snap.c_group_off[big[0]]) + 40
        snap.g_replicas[g40] += 3
        dr.commit_objects()
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        assert got.groups["n_create"][g40] >= 3 and big[0] in got.changed_clusters.tolist()
        snap.g_replicas[g40] -= 3
        for col in OBJ_COLS:
            np.copyto(dr.views[col], snap.cols[col])
        dr.eng.commit_object_rows([big[0]], [])
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        assert big[0] in got.changed_clusters.tolist()
    finally:
        dr.close()


def test_dirty_wide_clusters_overflow_the_group_staging(oracle_mod):
    """200 RayClusters of 48 groups: the staging holds 64 clusters and 64 x 32 group records, so 60 dirty wide RayClusters
    (2 880 groups) come back as whole arrays; 10 of them come back packed."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=200, pods_per_cluster=40, groups=1, seed=13))
    snap = synthetic.widen_clusters(snap, np.arange(200), 48)
    flags = compact(flags)
    dr = Driver(snap, flags, max_creates=1 << 16, wide_clusters=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        for n_dirty in (60, 10):
            dirty = np.arange(0, 200, 200 // n_dirty)[:n_dirty]
            rows = np.concatenate([group_pods(snap, c, 35)[:1] for c in dirty])  # (39 workers: groups 0..38 hold one each)
            assert rows.size == n_dirty
            snap.p_packed[rows] ^= np.uint32(1 << abi.PP_READY_SHIFT)
            dr.commit_rows(rows)
            got, _ = dr.check(oracle_mod, expect_incremental=True)
            assert sorted(got.changed_clusters.tolist()) == dirty.tolist()
    finally:
        dr.close()


def _grouped(base, counts):
    """`base` (one group per RayCluster) with cluster c's group 0 split into counts[c] groups."""
    snap = base
    for n in sorted(set(counts.values())):
        snap = synthetic.widen_clusters(snap, [c for c, k in counts.items() if k == n], n)
    return snap


@pytest.mark.parametrize("first_wide", [True, False])
def test_a_cluster_crossing_32_groups(first_wide, oracle_mod):
    """Clusters 5 and 6 trade worker groups (same group table size): 30 + 36 -> 34 + 32.  The epoch is structural, the full pass
    after it reclassifies, and the epochs after that are incremental again."""
    base, flags = synthetic.generate(synthetic.SynthParams(n_clusters=300, pods_per_cluster=40, groups=1, seed=14))
    flags = compact(flags)
    a = _grouped(base, {5: 30, 6: 36})
    b = _grouped(base, {5: 34, 6: 32})
    start, end = (a, b) if first_wide else (b, a)
    dr = Driver(start, flags, max_creates=1 << 16, wide_clusters=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rows = dr.switch(end)
        dr.commit_rows(rows)
        dr.check(oracle_mod, expect_incremental=False)
        flip = np.concatenate([workers(end, 5)[::7], workers(end, 6)[::7]])
        end.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        dr.commit_rows(flip)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


@pytest.mark.parametrize("entry", ["parts", "rows"])
def test_the_first_wide_cluster_appears_and_the_last_leaves(entry, oracle_mod):
    """Clusters 5 and 6 go from 30 + 4 groups to 33 + 1 (the snapshot's first wide RayCluster) and back, through
    kr_snapshot_commit_parts(KR_PART_OBJECTS) or kr_snapshot_commit_object_rows."""
    base, flags = synthetic.generate(synthetic.SynthParams(n_clusters=300, pods_per_cluster=40, groups=1, seed=15))
    flags = compact(flags)
    narrow = _grouped(base, {5: 30, 6: 4})
    wide = _grouped(base, {5: 33})
    dr = Driver(narrow, flags, max_creates=1 << 16, wide_clusters=True)
    try:
        got, _ = dr.check(oracle_mod, expect_incremental=False)
        for nxt in (wide, narrow):
            rows = dr.switch(nxt, commit=entry == "parts")
            if entry == "rows":
                for col in OBJ_COLS:
                    np.copyto(dr.views[col], nxt.cols[col])
                dr.eng.commit_object_rows([5, 6], [])
            dr.commit_rows(rows)
            dr.check(oracle_mod, expect_incremental=False)
            names = {k for k, _ in dr.eng.reconcile_profiled(dr.flags)["kernels"]}  # (an epoch without changes)
            assert ("k_decide_large" in names) == (nxt is wide)
            dr.eng.fetch()  # (an unfetched epoch makes the next one return every record)
            flip = workers(nxt, 5)[::5]
            nxt.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
            dr.commit_rows(flip)
            dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


def test_turning_the_option_on_after_a_pass(oracle_mod):
    snap, flags = _wide_fleet(48, wide=(0, 99))
    want = oracle_mod.run(snap, flags)
    eng = Engine.for_snapshot(snap, max_creates=1 << 16)
    try:
        eng.load(snap)
        for wide in (False, True, False, True):
            eng.set_wide_clusters(wide)
            assert eng.get_option(abi.OPT_WIDE_CLUSTERS) == int(wide)
            names = {k for k, _ in eng.reconcile_profiled(flags)["kernels"]}
            got = eng.reconcile(flags)
            assert not want.diff(got)
            if wide:
                assert BUCKET_KERNELS <= names and not SORT_KERNELS & names
            else:
                assert "k_match2" not in names and "k_decide_large" not in names
    finally:
        eng.close()


def test_native_packer_keeps_incremental_epochs_with_a_wide_cluster(oracle_mod):
    """A fleet with a RayCluster of 40 worker groups behind the native packer, KR_OPT_WIDE_CLUSTERS set through kr_packer_engine:
    every epoch equals the oracle and the pod-row epochs stay incremental on the device."""
    rng = np.random.default_rng(37)
    clusters, pods, jobs = objects(5, max_clusters=16)
    spec_groups = {(c["namespace"], c["name"], g["groupName"]): (c, g) for c in clusters for g in c["spec"]["workerGroupSpecs"]}
    owner = next(k for k, _ in collections.Counter((p.get("namespace"), p["labels"].get("ray.io/cluster"), p["labels"].get("ray.io/group"))
                                                   for p in pods if p["labels"].get("ray.io/node-type") == "worker").most_common()
                 if k in spec_groups)
    cl, src_g = spec_groups[owner]
    groups = cl["spec"]["workerGroupSpecs"]
    for k in range(40 - len(groups)):
        g = copy.deepcopy(src_g)
        g["groupName"] = f"{src_g['groupName']}-w{k}"
        g["numOfHosts"] = 1
        groups.append(g)
        cl["expectations"][g["groupName"]] = True
    members = [p for p in pods if (p.get("namespace"), p["labels"].get("ray.io/cluster"), p["labels"].get("ray.io/group")) == owner]
    for i, p in enumerate(members):
        p["labels"]["ray.io/group"] = groups[i % len(groups)]["groupName"]
    pk = Packer(**PACKER_CAPS, wide_clusters=True)
    try:
        m = Mirror(copy.deepcopy(clusters), copy.deepcopy(pods), jobs, pk)
        pk.flush()
        _, first = packer_check(m, oracle_mod, lean=True)
        assert pk.engine.get_option(abi.OPT_WIDE_CLUSTERS) == 1 and pk.engine.get_option(abi.OPT_BUCKET_STRIDE) != 0
        counter = [0]
        gots, modes = packer_stream(m, oracle_mod, 10, lambda epoch: events(rng, m, counter, structural=False))
        incremental = [device_incremental(g) for g in gots]
        assert any(mo & abi.PACK_POD_ROWS for mo in modes)
        assert incremental[0] and sum(incremental) >= 5, incremental
    finally:
        pk.close()

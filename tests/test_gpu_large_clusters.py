"""KR_OPT_LARGE_CLUSTERS: RayClusters of 257..KR_LARGE_MAX_PODS pods decided on the bucket pipeline (kuberay_b200/csrc/kr_large.cuh).

Every pass is compared with the oracle and with the same snapshot run with the option off (the sort pipeline then decides it):
Results.diff covers every result array except the run order inside the two arenas and pod_start, which only mean something when
the full pod lists are fetched."""
import copy
import functools

import numpy as np
import pytest

from harness import (OBJ_COLS, PACKER_CAPS, SORT_KERNELS, Driver, Mirror, b32, compact, device_incremental, events, grown_fleet, head_row,
                     members, most_workers, objects, packer_check, packer_stream, parity_on_off, run, scale_to, set_phase, spec_bytes, workers)
from kuberay_b200 import abi, synthetic
from kuberay_b200.engine import Engine
from kuberay_b200.packer import Packer

pytestmark = pytest.mark.gpu

_parity = functools.partial(parity_on_off, option="large_clusters")


@pytest.mark.parametrize("size", [257, 1000, 1024, 1025, 4096, 8192])
def test_one_large_cluster_stays_on_the_bucket_pipeline(size, oracle_mod):
    snap, flags = grown_fleet(size)
    got, names, stride = _parity(snap, flags, oracle_mod)
    assert got.clusters["n_pods"][0] == size
    assert {"k_match2", "k_decide2", "k_large_sort", "k_decide_large"} <= set(names), names
    assert not SORT_KERNELS & set(names), names
    assert stride == 64  # the rest of the fleet keeps its stride


def test_past_the_largest_cluster_the_sort_pipeline_decides(oracle_mod):
    snap, flags = grown_fleet(abi.LARGE_MAX_PODS + 1)
    _, names, stride = _parity(snap, flags, oracle_mod)
    assert "k_match2" not in names and "k_decide_large" not in names and stride == 0


def test_option_off_keeps_the_sort_pipeline(oracle_mod):
    snap, flags = grown_fleet(257)
    got, names, stride = run(snap, flags, profiled=True, large_clusters=False)
    assert not oracle_mod.run(snap, flags).diff(got)
    assert "k_match2" not in names and "k_decide_large" not in names and stride == 0


def test_more_than_32_worker_groups_still_take_the_sort_pipeline(oracle_mod):
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=200, pods_per_cluster=40, groups=33, seed=5))
    _, names, _ = _parity(snap, compact(flags), oracle_mod)
    assert "k_match2" not in names and "k_decide_large" not in names


def _decision_fleet(seed, size=3000, n_large=3):
    """Several large RayClusters with their own case each (see the callers), in a fleet of ordinary ones."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=600, pods_per_cluster=20, groups=1, seed=seed, healthy=True))
    big = [0, 250, 500][:n_large]
    synthetic.grow_clusters(snap, big, size)
    for c in big:
        snap.c_flags[c] &= ~np.uint32(abi.CF_SKIP | abi.CF_SUSPEND | abi.CF_UPGRADE_RECREATE)
        snap.c_flags[c] |= np.uint32(abi.CF_HEAD_EXPECT_OK)
        scale_to(snap, int(snap.c_group_off[c]), workers(snap, c).size)
    return snap, compact(flags), big


@pytest.mark.parametrize("random_delete", [False, True])
def test_decisions_inside_large_clusters(random_delete, oracle_mod):
    snap, flags, (a, b, c) = _decision_fleet(3)
    flags.env_random_pod_delete = int(random_delete)
    wa, wb, wc = workers(snap, a), workers(snap, b), workers(snap, c)
    # a: unhealthy pods -> the group aborts after them
    set_phase(snap, wa[100:140], abi.PHASE_FAILED)
    # b: scale down by 300 (a long delete prefix), autoscaling on so random delete matters
    snap.c_flags[b] |= np.uint32(abi.CF_AUTOSCALING)
    scale_to(snap, int(snap.c_group_off[b]), wb.size - 300)
    # c: scale up across the replica-index windows at 1024 and 2048, labels on every pod
    snap.p_packed[wc] |= np.uint32(abi.PP_HAS_REPLICA_IDX)
    snap.p_replica_index[wc] = np.arange(wc.size, dtype=np.int32) * 2  # every even index in use
    scale_to(snap, int(snap.c_group_off[c]), wc.size + 1500)
    got, names, stride = _parity(snap, flags, oracle_mod, max_creates=1 << 16)
    assert "k_decide_large" in names and stride == 64
    assert got.groups["n_unhealthy"][snap.c_group_off[a]] == 40
    assert got.groups["n_create"][snap.c_group_off[c]] == 1500
    creates = got.creates_of(int(snap.c_group_off[c]))
    assert creates.max() > 2048


def test_heads_and_suspend_inside_large_clusters(oracle_mod):
    snap, flags, (a, b, c) = _decision_fleet(4)
    # b: a second head
    wb = workers(snap, b)
    snap.p_packed[wb[7]] = (snap.p_packed[wb[7]] & ~np.uint32(3 << abi.PP_NODE_TYPE_SHIFT)) | np.uint32(abi.NT_HEAD << abi.PP_NODE_TYPE_SHIFT)
    # c: suspended worker group
    snap.g_flags[snap.c_group_off[c]] |= np.uint32(abi.GF_SUSPEND)
    got, names, _ = _parity(snap, flags, oracle_mod)
    assert "k_decide_large" in names
    assert got.clusters["n_heads"][b] == 2
    # the whole of c suspended
    snap2, flags2, (a2, b2, c2) = _decision_fleet(5)
    snap2.c_flags[c2] |= np.uint32(abi.CF_SUSPEND)
    got, names, _ = _parity(snap2, flags2, oracle_mod)
    assert "k_decide_large" in names


def test_several_large_clusters_keep_the_fleet_stride(oracle_mod):
    """The C3L shape at a tenth of its size: 20 RayClusters of 2 000 pods among 1 000 ordinary ones."""
    snap, flags = synthetic.generate(synthetic.config("C3L", n_clusters=1000))
    _, names, stride = _parity(snap, compact(flags), oracle_mod)
    assert "k_decide_large" in names and stride == 128  # (the stride of the mean cluster size, as without large clusters)


def test_multihost_group_inside_a_large_cluster(oracle_mod):
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=400, pods_per_cluster=20, groups=2, multihost_frac=0.25, seed=9))
    synthetic.grow_clusters(snap, [0], 1200)
    for gate in (1, 0):
        flags.gate_multihost_indexing = gate
        _, names, _ = _parity(snap, compact(flags), oracle_mod)
        assert "k_decide_large" in names


# ------------------------------------------------------------------------------------------------ incremental epochs

def test_incremental_epochs_in_large_clusters(oracle_mod):
    snap, flags, big = _decision_fleet(6)
    rng = np.random.default_rng(3)
    dr = Driver(snap, flags, max_creates=1 << 16, large_clusters=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        assert dr.eng.get_option(abi.OPT_BUCKET_STRIDE) == 64
        for epoch in range(6):
            wa, wb = workers(snap, big[0]), workers(snap, big[1])
            rows = []
            # status flips in a large cluster
            flip = rng.choice(wa, 30, replace=False)
            snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT); rows += flip.tolist()
            fail = rng.choice(wb, 5, replace=False)
            set_phase(snap, fail, abi.PHASE_FAILED if epoch % 2 == 0 else abi.PHASE_RUNNING); rows += fail.tolist()
            # pods moving between a large and an ordinary cluster, both ways
            small = int(rng.integers(600 // 2 + 1, 599))
            out = rng.choice(wa, 4, replace=False)
            snap.p_ns_id[out], snap.p_cluster_name_id[out] = snap.c_ns_id[small], snap.c_name_id[small]
            snap.p_group_name_id[out] = snap.g_name_id[snap.c_group_off[small]]
            into = workers(snap, small)[:2]
            snap.p_ns_id[into], snap.p_cluster_name_id[into] = snap.c_ns_id[big[2]], snap.c_name_id[big[2]]
            snap.p_group_name_id[into] = snap.g_name_id[snap.c_group_off[big[2]]]
            rows += out.tolist() + into.tolist()
            dr.commit_rows(rows, journal=epoch % 2 == 0)
            dr.check(oracle_mod, expect_incremental=True)
        # replica edits of a large cluster through the object commit
        snap.g_replicas[snap.c_group_off[big[0]]] += 17
        dr.commit_objects()
        dr.check(oracle_mod, expect_incremental=True)
        # numOfHosts 1 -> 4 -> 1 of a large cluster's group, through both object-commit entry points
        g = int(snap.c_group_off[big[1]])
        for i, hosts in enumerate((4, 1, 4, 1)):
            snap.g_num_hosts[g] = hosts
            if i % 2:
                dr.commit_objects()
            else:
                for col in OBJ_COLS:
                    np.copyto(dr.views[col], snap.cols[col])
                dr.eng.commit_object_rows([big[1]], [])
            got, _ = dr.check(oracle_mod, expect_incremental=True)
            assert bool(got.groups["flags"][g] & abi.GR_MULTIHOST) == (hosts > 1)
    finally:
        dr.close()


def test_a_large_cluster_outgrowing_its_region(oracle_mod):
    snap, flags, big = _decision_fleet(7, size=1000, n_large=1)
    dr = Driver(snap, flags, max_creates=1 << 16, large_clusters=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        # its region holds about 1.25x: 400 more pods do not fit -> one full pass, then incremental again
        donors = np.concatenate([workers(snap, c) for c in range(300, 600)])[:400]
        snap.p_ns_id[donors], snap.p_cluster_name_id[donors] = snap.c_ns_id[big[0]], snap.c_name_id[big[0]]
        snap.p_group_name_id[donors] = snap.g_name_id[snap.c_group_off[big[0]]]
        dr.commit_rows(donors)
        dr.check(oracle_mod, expect_incremental=False)
        flip = workers(snap, big[0])[::50]
        snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        dr.commit_rows(flip)
        dr.check(oracle_mod, expect_incremental=True)
        # an ordinary cluster crossing 256 pods: a full pass classifies it, then incremental again
        donors = np.concatenate([workers(snap, c) for c in range(100, 200)])[:300]
        snap.p_ns_id[donors], snap.p_cluster_name_id[donors] = snap.c_ns_id[50], snap.c_name_id[50]
        snap.p_group_name_id[donors] = snap.g_name_id[snap.c_group_off[50]]
        dr.commit_rows(donors)
        dr.check(oracle_mod, expect_incremental=False)
        assert dr.eng.get_option(abi.OPT_BUCKET_STRIDE) == 64
        flip = workers(snap, 50)[::10]
        snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        dr.commit_rows(flip)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


def test_turning_the_option_on_after_a_pass(oracle_mod):
    """A pass with the option off sends a fleet with a RayCluster of more than 1024 pods to the radix pipeline; turning the option
    on afterwards takes effect at the next pass (same snapshot, same sizes), and turning it off goes back."""
    snap, flags = grown_fleet(2000)
    want = oracle_mod.run(snap, flags)
    eng = Engine.for_snapshot(snap, max_creates=1 << 16)
    try:
        eng.load(snap)
        for large in (False, True, False):
            eng.set_large_clusters(large)
            names = {k for k, _ in eng.reconcile_profiled(flags)["kernels"]}
            got = eng.reconcile(flags)
            assert not want.diff(got)
            if large:
                assert "k_decide_large" in names and "k_scatter" not in names and eng.get_option(abi.OPT_BUCKET_STRIDE) == 64
            else:
                assert "k_scatter" in names and "k_match2" not in names and eng.get_option(abi.OPT_BUCKET_STRIDE) == 0
    finally:
        eng.close()


@pytest.mark.parametrize("spin", [True, False])
def test_recreate_gate_inside_large_clusters(spin, oracle_mod, monkeypatch):
    """Recreate-gated large RayClusters: one whose annotation names another spec (every pod deleted), one whose annotation is the
    digest of its spec.  The gate reads the digest after the join with the hash stream: in the graph, where the bucket pipeline's
    gated warps wait for digests inside k_decide2 (spin), and on the two-phase schedule (KR_NO_HASH_SPIN=1).  Then an incremental
    epoch recommits the spec JSON: the digests are recomputed on the device and the gates flip."""
    if not spin:
        monkeypatch.setenv("KR_NO_HASH_SPIN", "1")
    snap, flags, (a, b, c) = _decision_fleet(8)
    ah = snap.h_annot_hash.reshape(-1, 32)
    for cl, match in ((a, False), (b, True)):
        assert snap.c_json_len[cl] > 8
        snap.c_flags[cl] |= np.uint32(abi.CF_UPGRADE_RECREATE)
        h = head_row(snap, cl)
        snap.h_version_state[h] = abi.VER_CURRENT
        snap.h_annot_state[h] = abi.ANNOT_HASH32
        digest = b32(spec_bytes(snap, cl))
        ah[h] = np.frombuffer(digest if match else digest[::-1], dtype=np.uint8)
    got, names, _ = _parity(snap, flags, oracle_mod)
    assert "k_decide_large" in names
    assert got.clusters["path"][a] == abi.PATH_RECREATE_DELETE_ALL and got.clusters["path"][b] == abi.PATH_NORMAL
    dr = Driver(snap, flags, max_creates=1 << 16, large_clusters=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        p = int(snap.c_json_off[b]) + 3
        snap.json[p] ^= 0x20                                   # b's spec no longer matches its annotation
        np.copyto(dr.views["json"], snap.json)
        dr.eng.commit(abi.PART_JSON)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        assert got.clusters["path"][b] == abi.PATH_RECREATE_DELETE_ALL
    finally:
        dr.close()


@pytest.mark.parametrize("random_delete", [False, True])
def test_workers_to_delete_inside_large_clusters(random_delete, oracle_mod):
    """scaleStrategy.workersToDelete of large RayClusters: names of pods the cluster lists (late in List order), names of pods of
    other RayClusters and names no pod carries."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=600, pods_per_cluster=20, groups=1, autoscaling_frac=1.0,
                                                           wtd_group_frac=1.0, seed=21))
    flags = compact(flags)
    flags.env_random_pod_delete = int(random_delete)
    cand = [c for c in range(300, 600) if snap.g_wtd_cnt[snap.c_group_off[c]] >= 2]
    big = cand[:2]
    synthetic.grow_clusters(snap, big, 1500)
    for c in big:
        m = members(snap, c)
        set_phase(snap, m, abi.PHASE_RUNNING)
        snap.p_packed[m] &= ~np.uint32(abi.PP_RAY_TERMINATED)
        snap.c_flags[c] &= ~np.uint32(abi.CF_SKIP | abi.CF_SUSPEND | abi.CF_UPGRADE_RECREATE)
        snap.c_flags[c] |= np.uint32(abi.CF_HEAD_EXPECT_OK | abi.CF_AUTOSCALING)
        g = int(snap.c_group_off[c])
        w = workers(snap, c)
        scale_to(snap, g, w.size - 5)
        off, cnt = int(snap.g_wtd_off[g]), int(snap.g_wtd_cnt[g])
        other = snap.p_name_id[workers(snap, c + 1)[0]]  # a pod of another RayCluster of the namespace
        snap.w_name_id[off:off + cnt] = [snap.p_name_id[w[-1]], np.uint32(0x7F000000 + c)] + [other] * (cnt - 2)
    got, names, _ = _parity(snap, flags, oracle_mod)
    assert "k_decide_large" in names
    for c in big:
        g = int(snap.c_group_off[c])
        _, codes = got.actions_of(c)
        assert abi.ACT_DELETE_WTD in codes.tolist()
        assert got.groups["flags"][g] & abi.GR_WTD_EXECUTED
        off, cnt = int(snap.g_wtd_off[g]), int(snap.g_wtd_cnt[g])
        assert (got.wtd_pod_idx[off:off + cnt] == -1).any()      # the missing name resolves to no pod


def test_native_packer_keeps_incremental_epochs_with_large_clusters(oracle_mod):
    """A fleet with a RayCluster of 600 pods behind the native packer, KR_OPT_LARGE_CLUSTERS set through kr_packer_engine: every
    epoch equals the oracle and the pod-row epochs (KR_PACK_POD_ROWS) stay incremental on the device."""
    rng = np.random.default_rng(31)
    clusters, pods, jobs = objects(5, max_clusters=16)
    owner = most_workers(pods)
    src = [p for p in pods if (p.get("namespace"), p["labels"].get("ray.io/cluster")) == owner and p["labels"].get("ray.io/node-type") == "worker"]
    for i in range(600 - len(src)):
        q = copy.deepcopy(src[i % len(src)])
        q["name"] = f"{q['name']}-big-{i}"
        pods.append(q)
    pk = Packer(**PACKER_CAPS, large_clusters=True)
    try:
        m = Mirror(copy.deepcopy(clusters), copy.deepcopy(pods), jobs, pk)
        pk.flush()
        _, first = packer_check(m, oracle_mod, lean=True)
        assert int(first.clusters["n_pods"].max()) >= 600
        assert pk.engine.get_option(abi.OPT_LARGE_CLUSTERS) == 1 and pk.engine.get_option(abi.OPT_BUCKET_STRIDE) != 0
        counter = [0]
        gots, modes = packer_stream(m, oracle_mod, 10, lambda epoch: events(rng, m, counter, structural=False))
        incremental = [device_incremental(g) for g in gots]
        assert any(mo & abi.PACK_POD_ROWS for mo in modes)
        assert incremental[0] and sum(incremental) >= 5, incremental
    finally:
        pk.close()

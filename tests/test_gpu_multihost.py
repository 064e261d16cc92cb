"""Multi-host worker groups (numOfHosts > 1 under the RayMultiHostIndexing gate) on the bucket pipeline: k_decide2's multi-host
branch (decide_multihost2, kuberay_b200/csrc/kr_bucket2.cuh) against the CPU oracle, in full passes, in device-side incremental
epochs and behind the native packer."""
import copy

import numpy as np
import pytest

from harness import (OBJ_COLS, PACKER_CAPS, POD_COLS, Driver, Mirror, compact, device_incremental, events, flip_ready, kernels, objects,
                     packer_check, packer_stream, parity, set_phase)
from kuberay_b200 import abi, synthetic
from kuberay_b200.packer import Packer

pytestmark = pytest.mark.gpu

MH_ACTS = {abi.ACT_DELETE_MH_INCOMPLETE, abi.ACT_DELETE_MH_UNHEALTHY, abi.ACT_DELETE_MH_WTD, abi.ACT_DELETE_MH_SCALE_DOWN}
SORT_PIPELINE = ("k_place", "k_decide_small", "k_decide", "k_creates")


def _bucket_only(names):
    return {"k_match2", "k_decide2"} <= set(names) and not any(k.startswith(SORT_PIPELINE) and not k.startswith("k_decide2") for k in names)


def _mh_snapshot(seed, **kw):
    """400 RayClusters x 42 pods, two worker groups, half of the groups numOfHosts=4.  The 21-worker groups' spare pod loses its
    replica-name label (an unlabelled member), some replicas are renamed "" (so unlabelled pods resolve to them), and some lose a
    pod to a fresh name (incomplete replicas)."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=400, pods_per_cluster=42, groups=2, multihost_frac=0.5, seed=seed, **kw))
    rng = np.random.default_rng(seed)
    rn = snap.cols["p_replica_name_id"]
    names, inv, cnt = np.unique(rn, return_inverse=True, return_counts=True)
    spare = np.flatnonzero((rn != 0) & (cnt[inv] < 4))
    rn[spare] = 0
    set_phase(snap, spare[rng.random(spare.size) < 0.3], abi.PHASE_FAILED)
    named = names[names != 0]
    rn[np.isin(rn, named[rng.random(named.size) < 0.2])] = abi.ID_EMPTY_STRING
    split = np.flatnonzero(rn > 1)
    split = split[rng.random(split.size) < 0.02]
    rn[split] = np.uint32(0x7F000000) + np.arange(split.size, dtype=np.uint32)
    return snap, flags


def test_multihost_snapshot_takes_the_bucket_pipeline(oracle_mod):
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=400, pods_per_cluster=41, groups=2, multihost_frac=0.5))
    assert flags.gate_multihost_indexing == 1 and (snap.g_num_hosts > 1).any()
    names = kernels(snap, compact(flags))
    assert _bucket_only(names), names
    got = parity(snap, flags, oracle_mod)
    assert (got.groups["flags"] & abi.GR_MULTIHOST).any()


def test_multihost_branch_matches_the_oracle_across_flags(oracle_mod):
    """The gate on and off, random pod deletion off and on, and autoscaling RayClusters with workersToDelete on most groups
    (whole-replica deletions): bit-exact every time, with every multi-host delete code produced somewhere."""
    seen = set()
    runs = [(_mh_snapshot(1), g, r) for g in (1, 0) for r in (0, 1)]
    runs += [(_mh_snapshot(2, autoscaling_frac=0.7, wtd_group_frac=0.9), 1, r) for r in (0, 1)]
    for (snap, flags), gate, rdel in runs:
        f = abi.kr_flags.from_buffer_copy(flags)
        f.gate_multihost_indexing, f.env_random_pod_delete = gate, rdel
        got = parity(snap, f, oracle_mod)
        acts = set(np.unique(got.sorted_action).tolist())
        if gate:
            assert _bucket_only(kernels(snap, compact(f)))
            seen |= acts & MH_ACTS
            assert (got.groups["flags"] & abi.GR_MULTIHOST).any()
        else:
            assert not acts & MH_ACTS and not (got.groups["flags"] & abi.GR_MULTIHOST).any()
    assert seen == MH_ACTS, seen


def _mh_members(snap):
    """Pod rows of multi-host groups, by group row (workers with a replica-name label)."""
    gkey = {}
    c_of = {(int(snap.c_ns_id[c]), int(snap.c_name_id[c])): c for c in range(snap.dims["clusters"])}
    out = {}
    for p in np.flatnonzero(snap.p_replica_name_id > 1):
        c = c_of.get((int(snap.p_ns_id[p]), int(snap.p_cluster_name_id[p])))
        if c is None:
            continue
        if c not in gkey:
            g0, gc = int(snap.c_group_off[c]), int(snap.c_group_cnt[c])
            gkey[c] = {int(snap.g_name_id[g]): g for g in range(g0, g0 + gc)}
        g = gkey[c].get(int(snap.p_group_name_id[p]))
        if g is not None and snap.g_num_hosts[g] > 1:
            out.setdefault(g, []).append(int(p))
    return out


def test_incremental_epochs_with_multihost_groups(oracle_mod):
    snap, flags = synthetic.generate(synthetic.config("C2", n_clusters=300, pods_per_cluster=41, groups=2, multihost_frac=0.5, wtd_group_frac=0.3, seed=5))
    rng = np.random.default_rng(5)
    dr = Driver(snap, flags, slack=1.2)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        cols = snap.cols
        members = _mh_members(snap)
        groups = sorted(members)
        assert len(groups) > 50
        pick = iter(rng.permutation(groups).tolist())

        def replica(g):
            rows = members[g]
            name = cols["p_replica_name_id"][rows[0]]
            return [p for p in rows if cols["p_replica_name_id"][p] == name]

        # 1. status flips inside replicas
        rows = [p for g in groups[:40] for p in replica(g)[:2]]
        flip_ready(snap, rows[::2]); set_phase(snap, rows[1::2], abi.PHASE_PENDING)
        dr.commit_rows(rows)
        dr.check(oracle_mod, expect_incremental=True)
        # 2. a replica loses a pod (deleted: a free row) -> incomplete
        free = [replica(next(pick))[1] for _ in range(4)]
        saved = {c: cols[c][free].copy() for c in POD_COLS}
        for c in POD_COLS:
            cols[c][free] = 0
        cols["p_packed"][free] = np.uint32(abi.PP_TOMBSTONE)
        dr.commit_rows(free)
        dr.check(oracle_mod, expect_incremental=True)
        # 3. an unhealthy pod deletes its whole replica
        bad = [replica(next(pick))[2] for _ in range(6)]
        set_phase(snap, bad, abi.PHASE_FAILED)
        dr.commit_rows(bad)
        dr.check(oracle_mod, expect_incremental=True)
        # 4. a pod's replica-name label rewritten (one replica short, another one pod over)
        moved = []
        for _ in range(6):
            g = next(pick)
            others = [p for p in members[g] if cols["p_replica_name_id"][p] != cols["p_replica_name_id"][members[g][0]]]
            if others:
                cols["p_replica_name_id"][members[g][0]] = cols["p_replica_name_id"][others[0]]
                moved.append(members[g][0])
        dr.commit_rows(moved)
        dr.check(oracle_mod, expect_incremental=True)
        # 5. pods added into a new replica (the four free rows, as a complete replica of another multi-host group)
        g = next(pick)
        src = replica(g)[0]
        for c in POD_COLS:
            cols[c][free] = cols[c][src]
        cols["p_name_id"][free] = np.uint32(0x7E000000) + np.arange(4, dtype=np.uint32)
        cols["p_replica_name_id"][free] = np.uint32(0x7E100000)
        cols["p_replica_index"][free] = 40
        dr.commit_rows(free)
        dr.check(oracle_mod, expect_incremental=True)
        del saved
        # 6. replicas raised and lowered: creates (lowest free replica indices) and scale-down of whole replicas
        dr.flags.env_random_pod_delete = 1
        dr.check(oracle_mod, expect_incremental=False)     # (other process flags: a full pass first)
        for i, g in enumerate(groups[:60]):
            cols["g_replicas"][g] = 9 if i % 2 else 1
            cols["g_min"][g] = 0
            cols["g_flags"][g] &= ~np.uint32(abi.GF_REPLICAS_NIL | abi.GF_MIN_NIL)
        dr.commit_objects()
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        mh = (got.groups["flags"] & abi.GR_MULTIHOST) != 0
        assert (got.groups["n_create"][mh] > 0).any() and abi.ACT_DELETE_MH_SCALE_DOWN in got.act_code[:got.n_actions]
        # 7. numOfHosts 1 -> 4 -> 1, on a group 0 (it travels in the cluster's input record) and on a group 1
        single = np.flatnonzero(snap.g_num_hosts == 1)
        offs = snap.c_group_off
        g0 = int(single[np.isin(single, offs)][0]); g1 = int(single[~np.isin(single, offs)][0])
        for hosts in (4, 1):
            cols["g_num_hosts"][[g0, g1]] = hosts
            dr.commit_objects()
            dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


@pytest.mark.parametrize("object_rows", [False, True])
def test_first_multihost_group_comes_and_the_last_one_leaves(object_rows, oracle_mod):
    """The snapshot gains its first multi-host group and loses its last through object commits: the incremental epoch runs the
    decide instantiation of the current state, and so does the next full pass (the captured graph is rebuilt)."""
    snap, flags = synthetic.generate(synthetic.config("C2", n_clusters=200, pods_per_cluster=41, groups=2, seed=17))
    assert not (snap.g_num_hosts > 1).any()
    dr = Driver(snap, flags)
    try:
        first, _ = dr.check(oracle_mod, expect_incremental=False)
        # a group 1 the pass reaches and decides (its cluster is reconciled, group 0 does not abort, it is neither suspended nor
        # waiting on expectations): as a multi-host group it is then decided by the multi-host branch
        gf = first.groups["flags"]
        ok = ((gf & abi.GR_PROCESSED) != 0) & ((gf & (abi.GR_SUSPENDED | abi.GR_EXPECT_PENDING)) == 0) & ~np.isin(np.arange(gf.size), snap.c_group_off)
        g = int(np.flatnonzero(ok)[0])
        c = int(snap.g_cluster_idx[g])
        snap.cols["g_replicas"][g] = 3
        snap.cols["g_flags"][g] &= ~np.uint32(abi.GF_REPLICAS_NIL)

        def commit(rows=(c,)):
            if object_rows:
                for col in OBJ_COLS:
                    np.copyto(dr.views[col], snap.cols[col])
                dr.eng.commit_object_rows(list(rows), [])
            else:
                dr.commit_objects()

        for hosts in (4, 1, 4):
            snap.cols["g_num_hosts"][g] = hosts
            commit()
            got, _ = dr.check(oracle_mod, expect_incremental=True)
            assert bool(got.groups["flags"][g] & abi.GR_MULTIHOST) == (hosts > 1)
        # a renamed worker group elsewhere is structural: a full pass, which must decide the multi-host group as well
        snap.cols["g_name_id"][0] = snap.cols["g_name_id"][0] + np.uint32(100000)
        commit((c, int(snap.g_cluster_idx[0])))
        got, _ = dr.check(oracle_mod, expect_incremental=False)
        assert got.groups["flags"][g] & abi.GR_MULTIHOST
        snap.cols["g_num_hosts"][g] = 1
        commit()
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        assert not (got.groups["flags"] & abi.GR_MULTIHOST).any()
    finally:
        dr.close()


@pytest.mark.parametrize("seed", [5, 6])
def test_native_packer_keeps_incremental_epochs_with_multihost_groups(seed, oracle_mod):
    """A fleet with multi-host worker groups behind the native packer: every epoch equals the oracle, and after the first one the
    passes are incremental on the device (the results name the RayClusters they recomputed)."""
    rng = np.random.default_rng(seed)
    clusters, pods, jobs = objects(seed, max_clusters=16)
    assert any(g["numOfHosts"] > 1 for c in clusters for g in c["spec"]["workerGroupSpecs"])
    pk = Packer(**PACKER_CAPS)
    try:
        m = Mirror(copy.deepcopy(clusters), copy.deepcopy(pods), jobs, pk)
        pk.flush()
        packer_check(m, oracle_mod, lean=True)
        counter = [0]
        gots, _ = packer_stream(m, oracle_mod, 10, lambda epoch: events(rng, m, counter, structural=False))
        incremental = [device_incremental(g) for g in gots]
        # (an epoch may still take the full pass for a reason of its own — e.g. a small fleet's action list filling up with the
        # abandoned runs of re-decided clusters is packed again by a full pass)
        assert incremental[0] and sum(incremental) >= 5, incremental
    finally:
        pk.close()

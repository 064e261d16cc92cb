"""Device-side incremental epochs (kuberay_b200/csrc/kr_incr.cuh) through the C ABI, on synthetic snapshots large enough to
have every kind of RayCluster (suspended, Recreate, autoscaling, workersToDelete, several groups, RayJobs).

Every epoch mutates the snapshot the way informer events do (pod status flips, deletions -> free rows, additions into free rows,
pods moving between RayClusters, head pods coming and going, replicas / flags / old-status edits of RayCluster rows), commits it
with the incremental entry points and compares the engine with a from-scratch oracle run over the mutated snapshot.  The pass
must name the records it recomputed; records it did not name must be the ones that did not change."""
import numpy as np
import pytest

from harness import OBJ_COLS, POD_COLS, Driver, flip_ready, incremental, set_phase
from kuberay_b200 import abi, synthetic
from kuberay_b200.snapshot import Snapshot

pytestmark = pytest.mark.gpu

def _node_type(snap):
    return (snap.cols["p_packed"] >> abi.PP_NODE_TYPE_SHIFT) & 3


@pytest.mark.parametrize("seed,groups,jobs", [(3, 1, False), (4, 3, True), (5, 2, False)])
def test_pod_and_object_epochs_match_a_full_pass(seed, groups, jobs, oracle_mod):
    rng = np.random.default_rng(seed)
    snap, flags = synthetic.generate(synthetic.config("C2", n_clusters=600, pods_per_cluster=24, groups=groups, jobs=jobs, recreate_frac=0.05, wtd_group_frac=0.3, seed=seed))
    dr = Driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        npods, nc = snap.dims["pods"], snap.dims["clusters"]
        free = np.zeros(0, dtype=np.uint32)
        saved = {}
        n_inc = 0
        for epoch in range(14):
            touched = []
            workers = np.nonzero((_node_type(snap) == abi.NT_WORKER) & ((snap.cols["p_packed"] & abi.PP_TOMBSTONE) == 0))[0].astype(np.uint32)
            # status updates
            upd = rng.choice(workers, 40, replace=False)
            flip_ready(snap, upd[:20]); set_phase(snap, upd[20:30], 4); set_phase(snap, upd[30:], 2)
            touched += upd.tolist()
            # additions into the rows freed one epoch earlier (the same pods come back, some under another RayCluster)
            for r in free.tolist():
                for c in POD_COLS:
                    snap.cols[c][r] = saved[r][c]
            if free.size > 2:
                mv = free[:2]
                donor = rng.choice(workers, 2, replace=False)
                for c in ("p_ns_id", "p_cluster_name_id", "p_group_name_id"):
                    snap.cols[c][mv] = snap.cols[c][donor]
            touched += free.tolist()
            # deletions -> free rows
            gone = np.setdiff1d(rng.choice(workers, 12, replace=False), np.concatenate([upd, free]))
            saved = {int(r): {c: snap.cols[c][r].copy() for c in POD_COLS} for r in gone}
            for c in POD_COLS:
                snap.cols[c][gone] = 0
            snap.cols["p_packed"][gone] = np.uint32(abi.PP_TOMBSTONE)
            touched += gone.tolist()
            free = gone.astype(np.uint32)
            # a head pod flips its phase (its cluster's head decisions change); head-aux rows keep their keys
            heads = np.nonzero(_node_type(snap) == abi.NT_HEAD)[0]
            h = rng.choice(heads, 3, replace=False)
            set_phase(snap, h[:1], 4); flip_ready(snap, h[1:])
            touched += h.tolist()
            if epoch % 2 == 0:  # object rows: replicas, expectation flags, old status, head-aux readiness
                cs = rng.choice(nc, 8, replace=False)
                for c in cs[:4]:
                    g = int(snap.cols["c_group_off"][c])
                    if snap.cols["c_group_cnt"][c]:
                        snap.cols["g_replicas"][g] = int(rng.integers(0, 40))
                snap.cols["c_flags"][cs[4:6]] ^= np.uint32(1 << 5)   # KR_CF_HEAD_EXPECT_OK
                snap.cols["c_old_state"][cs[6:]] = np.uint8(int(rng.integers(0, 4)))
                if snap.dims["heads"]:
                    hr = rng.choice(snap.dims["heads"], 3, replace=False)
                    snap.cols["h_ready_status"][hr] = np.uint8(int(rng.integers(0, 4)))
                dr.commit_objects()
            elif epoch % 4 == 1:
                dr.commit_objects()  # unchanged object rows: nothing may become dirty because of them
            dr.commit_rows(touched, journal=bool(epoch % 3))
            got, _ = dr.check(oracle_mod)
            inc = incremental(got, nc)
            n_inc += inc
            if inc:
                assert 0 < got.n_changed < nc
        assert n_inc >= 12, n_inc
    finally:
        dr.close()


def test_structural_changes_and_other_flags_take_the_full_pass(oracle_mod):
    snap, flags = synthetic.generate(synthetic.config("C2", n_clusters=200, pods_per_cluster=16, groups=2, wtd_group_frac=0.4, seed=9))
    dr = Driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rows = np.arange(5, dtype=np.uint32)
        flip_ready(snap, rows)
        dr.commit_rows(rows)
        dr.check(oracle_mod, expect_incremental=True)
        # a renamed worker group is a table key: the resident tables are stale
        snap.cols["g_name_id"][3] = snap.cols["g_name_id"][3] + np.uint32(100000)
        dr.commit_objects()
        dr.check(oracle_mod, expect_incremental=False)
        dr.check(oracle_mod, expect_incremental=True)   # nothing committed: an empty incremental epoch
        assert dr.prev.n_changed == 0
        # a workersToDelete name changed: structural as well (the name table is resident)
        if snap.dims["wtd"]:
            snap.cols["w_name_id"][0] = snap.cols["p_name_id"][int(np.nonzero(snap.cols["p_name_id"])[0][0])]
            dr.commit_objects()
            dr.check(oracle_mod, expect_incremental=False)
        # different process-level flags: full pass, then incremental again under the new flags
        dr.flags.env_random_pod_delete = 1
        dr.check(oracle_mod, expect_incremental=False)
        flip_ready(snap, rows)
        dr.commit_rows(rows, journal=False)
        dr.check(oracle_mod, expect_incremental=True)
        # asking for the full pod lists leaves the bucket pipeline (and the resident state) altogether
        dr.flags.fetch_pod_lists = 1
        got = dr.eng.reconcile(dr.flags)
        assert not oracle_mod.run(snap, dr.flags).diff(got) and got.changed_clusters is None
        dr.flags.fetch_pod_lists = 0
        dr.check(oracle_mod, expect_incremental=False)
        # pod columns uploaded wholesale
        flip_ready(snap, rows)
        for c in POD_COLS:
            np.copyto(dr.views[c], snap.cols[c])
        dr.eng.commit(abi.PART_COLUMNS)
        dr.check(oracle_mod, expect_incremental=False)
    finally:
        dr.close()


def test_unfetched_passes_and_repeated_rows(oracle_mod):
    snap, flags = synthetic.generate(synthetic.config("C2", n_clusters=300, pods_per_cluster=12, groups=1, seed=21))
    dr = Driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rng = np.random.default_rng(2)
        for it in range(3):  # passes whose results never reach the host, then one fetch: the host copy must still be complete
            rows = rng.choice(snap.dims["pods"], 30, replace=False).astype(np.uint32)
            flip_ready(snap, rows)
            dr.commit_rows(rows[:20])
            set_phase(snap, rows[10:], 3)
            dr.commit_rows(rows[10:])      # rows 10..19 are committed twice before the pass
            dr.eng.reconcile_device_only(dr.flags)
        got = dr.eng.fetch()
        assert not oracle_mod.run(snap, dr.flags).diff(got)
        rows = rng.choice(snap.dims["pods"], 10, replace=False).astype(np.uint32)
        flip_ready(snap, rows)
        dr.commit_rows(rows)
        dr.prev = None
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


def test_appended_rows_and_head_rows_come_and_go(oracle_mod):
    """Rows appended past the old end of the pod arena and head-aux rows added / removed (new live counts under the fixed layout)."""
    snap, flags = synthetic.generate(synthetic.config("C2", n_clusters=150, pods_per_cluster=10, groups=1, seed=33))
    dr = Driver(snap, flags, slack=1.5)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        cols = snap.cols
        heads = np.nonzero(_node_type(snap) == abi.NT_HEAD)[0]
        # 1. a head pod is deleted: its pod row becomes free and its head-aux row disappears (rows after it shift up)
        victim_row = 4
        p = int(cols["h_pod_idx"][victim_row])
        for c in POD_COLS:
            cols[c][p] = 0
        cols["p_packed"][p] = np.uint32(abi.PP_TOMBSTONE)
        nh, d = snap.dims["heads"], snap.dims
        workers = np.nonzero(_node_type(snap) == abi.NT_WORKER)[0][:3]
        # 2. three worker pods appended past the end, copies of existing workers
        snap2 = Snapshot(d["clusters"], d["groups"], d["wtd"], d["pods"] + 3, nh - 1, d["jobs"], d["json"])
        for name, _dt, m, dim in abi.COLUMNS:
            a = cols[name]
            if dim == "heads":
                a = np.delete(a.reshape(nh, m), victim_row, axis=0).reshape(-1)
            elif dim == "pods":
                a = np.concatenate([a, a[workers]])
            snap2.cols[name][:] = a
        snap2.cols["p_name_id"][-3:] = np.uint32(0x7FFF0000) + np.arange(3, dtype=np.uint32)
        assert snap2.dims["heads"] == nh - 1 and snap2.dims["pods"] == snap.dims["pods"] + 3
        dr.use(snap2)
        dr.commit_objects()
        dr.commit_rows([p] + list(range(snap.dims["pods"], snap2.dims["pods"])))
        got, _ = dr.check(oracle_mod)
        assert incremental(got, snap2.dims["clusters"]), "appended rows / a removed head row must not force a full pass"
        assert heads.size
    finally:
        dr.close()


def test_object_row_commits_equal_whole_object_commits(oracle_mod):
    """kr_snapshot_commit_object_rows: only the rewritten RayCluster (+ their groups') and head-aux rows travel.  Same results as the
    whole object part, incremental on the device; rows whose Recreate bit changes fall back to the whole part by themselves."""
    rng = np.random.default_rng(8)
    snap, flags = synthetic.generate(synthetic.config("C2", n_clusters=400, pods_per_cluster=12, groups=2, recreate_frac=0.1, seed=44))
    dr = Driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        nc, nh = snap.dims["clusters"], snap.dims["heads"]
        for epoch in range(6):
            cs = rng.choice(nc, 9, replace=False)
            for c in cs[:5]:
                g = int(snap.cols["c_group_off"][c]) + int(rng.integers(0, max(1, int(snap.cols["c_group_cnt"][c]))))
                if snap.cols["c_group_cnt"][c]:
                    snap.cols["g_replicas"][g] = int(rng.integers(0, 30))
                    snap.cols["g_flags"][g] ^= np.uint32(abi.GF_EXPECT_OK)
            snap.cols["c_flags"][cs[5:7]] ^= np.uint32(1 << 5)            # KR_CF_HEAD_EXPECT_OK
            snap.cols["c_old_counts"][5 * int(cs[7])] = int(rng.integers(0, 9))
            snap.cols["c_svc_count"][cs[8]] = np.uint8(int(rng.integers(0, 3)))
            hs = rng.choice(nh, 4, replace=False)
            snap.cols["h_ready_status"][hs] = np.uint8(int(rng.integers(0, 4)))
            snap.cols["h_pod_ip_id"][hs[:2]] = snap.cols["h_pod_ip_id"][hs[2:]]
            if epoch == 4:                                                  # a Recreate gate flips: the engine takes the whole object part itself
                snap.cols["c_flags"][cs[0]] ^= np.uint32(1 << 3)
            for c in OBJ_COLS:
                np.copyto(dr.views[c], snap.cols[c])
            dr.eng.commit_object_rows(cs, hs)
            rows = rng.choice(snap.dims["pods"], 15, replace=False).astype(np.uint32)
            flip_ready(snap, rows)
            dr.commit_rows(rows)
            got, _ = dr.check(oracle_mod, expect_incremental=True)
            assert got.n_changed <= 9 + 4 + 15 + 1
            if epoch != 4:
                assert dr.eng.last_profile()["h2d_bytes"] < 40000, dr.eng.last_profile()   # a few KB, not the 100+ KB object part
        # rows out of range are refused
        from kuberay_b200.engine import EngineError
        with pytest.raises(EngineError):
            dr.eng.commit_object_rows([nc], [])
        with pytest.raises(EngineError):
            dr.eng.commit_object_rows([], [nh])
    finally:
        dr.close()

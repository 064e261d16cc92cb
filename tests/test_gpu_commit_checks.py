"""The commits check their input before anything moves: a row commit refuses the rows the whole object commit would refuse, whichever
path it then takes, and a refused whole commit leaves the engine's record of the device as it was."""
import numpy as np
import pytest

from harness import POD_COLS, Driver, flip_ready, workers, workers_of
from kuberay_b200 import abi, synthetic
from kuberay_b200.engine import EngineError

pytestmark = pytest.mark.gpu


def _refused(call):
    with pytest.raises(EngineError) as ei:
        call()
    assert ei.value.code == abi.KR_E_INVALID, str(ei.value)


def test_row_commit_checks_its_rows_as_the_whole_commit_does(oracle_mod):
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=64, pods_per_cluster=16, groups=2, autoscaling_frac=0.5, seed=7))
    dr = Driver(snap, flags, slack=1.2)
    try:
        nc, nh = snap.dims["clusters"], snap.dims["heads"]
        # no state is resident yet: the row commit would take the whole object part, and still refuses a row out of range
        _refused(lambda: dr.eng.commit_object_rows([nc], []))
        _refused(lambda: dr.eng.commit_object_rows([], [nh]))
        dr.check(oracle_mod, expect_incremental=False)
        c = int(np.flatnonzero(snap.c_group_cnt >= 2)[0])
        g = int(snap.c_group_off[c]) + 1
        v = dr.views
        bad = [("g_cluster_idx", g, nc),                                                      # a group names no RayCluster
               ("g_wtd_off", g, snap.dims["wtd"] - int(snap.g_wtd_cnt[g]) + 1),              # its workersToDelete names run past n_wtd
               ("c_json_off", c, int(snap.c_json_off[c]) + 8)]                               # a misaligned spec offset
        for col, row, value in bad:
            old = v[col][row].copy()
            v[col][row] = value
            _refused(lambda: dr.eng.commit_object_rows([c], []))  # (nothing of it reached the device: no pass runs in between)
            v[col][row] = old
        # the views restored, the next epoch goes row by row again and equals the oracle
        rows = workers(snap, c)[:2]
        flip_ready(snap, rows)
        dr.eng.commit_object_rows([c], [])
        dr.commit_rows(rows)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


def _multihost(snap, c):
    off, cnt = int(snap.c_group_off[c]), int(snap.c_group_cnt[c])
    return bool((snap.g_num_hosts[off:off + cnt] > 1).any())


def test_refused_whole_commit_keeps_the_multihost_record(oracle_mod):
    """A whole object commit refused at row k, then a row commit that takes the multi-host group of the RayCluster a before k away:
    the multi-host RayCluster b after k must still be decided on the multi-host branch (RayMultiHostIndexing on)."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=120, pods_per_cluster=41, groups=1, multihost_frac=0.3, healthy=True, seed=11))
    assert flags.gate_multihost_indexing == 1
    cols = snap.cols
    nc = snap.dims["clusters"]
    a = next(c for c in range(nc) if _multihost(snap, c))
    k = a + 1
    cols["g_num_hosts"][int(snap.c_group_off[k]):int(snap.c_group_off[k] + snap.c_group_cnt[k])] = 1  # (a single-host row between them)
    b = next(c for c in range(k + 1, nc) if _multihost(snap, c))
    # one of b's replicas loses a Pod: with the gate it is incomplete, without it its Pods are ordinary workers
    gb = int(snap.c_group_off[b])
    members = workers_of(snap, gb)
    members = members[snap.p_replica_name_id[members] > 1]
    lost = int(members[snap.p_replica_name_id[members] == snap.p_replica_name_id[members[0]]][0])
    for col in POD_COLS:
        cols[col][lost] = 0
    cols["p_packed"][lost] = np.uint32(abi.PP_TOMBSTONE)
    off = abi.kr_flags.from_buffer_copy(flags)
    off.gate_multihost_indexing = 0
    (pods_on, acts_on), (pods_off, acts_off) = oracle_mod.run(snap, flags).actions_of(b), oracle_mod.run(snap, off).actions_of(b)
    assert abi.ACT_DELETE_MH_INCOMPLETE in acts_on and not (np.array_equal(pods_on, pods_off) and np.array_equal(acts_on, acts_off))

    dr = Driver(snap, flags, slack=1.2)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        # 1. the whole object part with row k's spec offset misaligned
        dr.views["c_json_off"][k] += 8
        _refused(lambda: dr.eng.commit(abi.PART_OBJECTS))
        # 2. row k restored; 3. a's group single-host, one of b's Pods flipped: a row commit of a and a pod commit
        dr.views["c_json_off"][k] -= 8
        cols["g_num_hosts"][int(snap.c_group_off[a]):int(snap.c_group_off[a] + snap.c_group_cnt[a])] = 1
        np.copyto(dr.views["g_num_hosts"], cols["g_num_hosts"])
        dr.eng.commit_object_rows([a], [])
        rows = workers(snap, b)[-1:]
        flip_ready(snap, rows)
        dr.commit_rows(rows)
        # 4. the pass, then a full one
        dr.check(oracle_mod)
        dr.commit_objects(abi.PART_ALL)
        dr.check(oracle_mod, expect_incremental=False)
    finally:
        dr.close()

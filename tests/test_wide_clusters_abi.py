"""The wide-RayCluster option without a device: its constant in the Python bindings matches include/kr_engine.h,
synthetic.widen_clusters builds consistent snapshots, and the oracle decides C3W-shaped fleets."""
import os
import re

import numpy as np

from kuberay_b200 import abi, synthetic

HEADER = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "kr_engine.h")).read()


def test_option_constant_matches_the_header():
    assert int(re.search(r"KR_OPT_WIDE_CLUSTERS\s*=\s*(\d+)", HEADER).group(1)) == abi.OPT_WIDE_CLUSTERS


def _workers_of(snap, c):
    m = (snap.p_ns_id == snap.c_ns_id[c]) & (snap.p_cluster_name_id == snap.c_name_id[c])
    return np.flatnonzero(m & (((snap.p_packed >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER))


def test_widen_clusters_splits_worker_group_0():
    snap, _ = synthetic.generate(synthetic.SynthParams(n_clusters=40, pods_per_cluster=60, groups=2, seed=3, autoscaling_frac=1.0, wtd_group_frac=1.0))
    wide = synthetic.widen_clusters(snap, [3, 17], 40)  # (validate()d inside)
    assert wide.dims["groups"] == snap.dims["groups"] + 2 * 39 and wide.dims["wtd"] == snap.dims["wtd"]
    assert wide.c_group_cnt[3] == 41 and wide.c_group_cnt[17] == 41 and wide.c_group_cnt[4] == 2
    assert (wide.w_name_id == snap.w_name_id).all()
    for c in (3, 17):
        g_old, g_new = int(snap.c_group_off[c]), int(wide.c_group_off[c])
        names = wide.g_name_id[g_new:g_new + 40]
        assert np.unique(names).size == 40 and names[0] == snap.g_name_id[g_old]
        assert wide.g_name_id[g_new + 40] == snap.g_name_id[g_old + 1]  # group 1 follows the split group
        assert wide.g_replicas[g_new:g_new + 40].sum() == snap.g_replicas[g_old]
        assert (wide.g_wtd_cnt[g_new + 1:g_new + 40] == 0).all() and wide.g_wtd_cnt[g_new] == snap.g_wtd_cnt[g_old]
        # group 0's workers, round-robin over the 40 groups in row order; group 1's keep their label
        w = _workers_of(snap, c)
        in0 = w[snap.p_group_name_id[w] == snap.g_name_id[g_old]]
        assert (wide.p_group_name_id[in0] == names[np.arange(in0.size) % 40]).all()
        in1 = w[snap.p_group_name_id[w] == snap.g_name_id[g_old + 1]]
        assert (wide.p_group_name_id[in1] == snap.p_group_name_id[in1]).all()
    # every other row keeps its values
    for name, _dt, _m, dim in abi.COLUMNS:
        if dim in ("clusters", "heads", "jobs", "json") and name not in ("c_group_off", "c_group_cnt"):
            assert (wide.cols[name] == snap.cols[name]).all(), name


def test_c3w_shape():
    snap, _ = synthetic.generate(synthetic.config("C3W", n_clusters=1000, n_wide=10))
    assert (snap.c_group_cnt > 32).sum() == 10 and snap.c_group_cnt.max() == 48


def test_oracle_decides_c3w_shaped_fleets(oracle_mod):
    snap, flags = synthetic.generate(synthetic.config("C3W", n_clusters=1000, n_wide=10))
    flags.fetch_pod_lists = 0
    got = oracle_mod.run(snap, flags)
    wide = np.flatnonzero(snap.c_group_cnt > 32)
    assert (got.clusters["n_pods"][wide] == 100).all()
    g = snap.c_group_off[wide].astype(np.int64)[:, None] + np.arange(48)[None, :]
    assert (got.groups["flags"][g.ravel()] != 0).any()
    assert not oracle_mod.run(snap, flags).diff(got)  # deterministic

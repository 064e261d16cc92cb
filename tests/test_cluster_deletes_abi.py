"""The RayCluster-deletion option without a device: its constant in the Python bindings matches include/kr_engine.h, the Go shim
declares it, the engine and packer entry points take it, off by default, and synthetic.delete_clusters swap-removes as the native
packer does."""
import inspect
import os
import re

import numpy as np

from harness import members
from kuberay_b200 import abi, synthetic
from kuberay_b200.engine import Engine
from kuberay_b200.packer import GroupPacker, Packer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "kr_engine.h")).read()


def test_option_constant_matches_the_header():
    assert int(re.search(r"KR_OPT_CLUSTER_DELETES\s*=\s*(\d+)", HEADER).group(1)) == abi.OPT_CLUSTER_DELETES == 10


def test_go_shim_declares_the_option():
    src = open(os.path.join(ROOT, "integration", "go", "krengine", "engine.go")).read()
    assert re.search(r"OptClusterDeletes\s*=\s*uint32\(C\.KR_OPT_CLUSTER_DELETES\)", src)
    assert "// OptClusterDeletes is KR_OPT_CLUSTER_DELETES (1:" in src


def test_engine_and_packers_take_the_keyword_off_by_default():
    assert inspect.signature(Engine.for_snapshot).parameters["cluster_deletes"].default is False
    assert inspect.signature(Packer.__init__).parameters["cluster_deletes"].default is False
    assert inspect.signature(Packer.set_options).parameters["cluster_deletes"].default is False
    assert inspect.signature(GroupPacker.__init__).parameters["cluster_deletes"].default is False
    assert callable(Engine.set_cluster_deletes)


def test_swap_remove_order():
    assert synthetic.swap_remove_order(6, [1]).tolist() == [0, 5, 2, 3, 4]
    assert synthetic.swap_remove_order(6, [5]).tolist() == [0, 1, 2, 3, 4]
    assert synthetic.swap_remove_order(6, [1, 5]).tolist() == [0, 4, 2, 3]  # (5 moved into row 1, then deleted from there)
    assert synthetic.swap_remove_order(6, [0, 4, 2]).tolist() == [5, 1, 3]


def test_delete_clusters_keeps_the_pods_as_orphans():
    snap, _ = synthetic.generate(synthetic.config("C2", n_clusters=40, pods_per_cluster=8, groups=3, seed=4, wtd_group_frac=0.5))
    rows = [3, 39, 17]
    order = synthetic.swap_remove_order(40, rows)
    out = synthetic.delete_clusters(snap, rows)
    assert out.dims["clusters"] == 37 and out.dims["pods"] == snap.dims["pods"]
    for new, old in enumerate(order):
        assert (out.c_ns_id[new], out.c_name_id[new], out.c_json_off[new]) == (snap.c_ns_id[old], snap.c_name_id[old], snap.c_json_off[old])
        g_new, g_old, G = int(out.c_group_off[new]), int(snap.c_group_off[old]), int(snap.c_group_cnt[old])
        assert out.c_group_cnt[new] == G and (out.g_cluster_idx[g_new:g_new + G] == new).all()
        assert np.array_equal(out.g_name_id[g_new:g_new + G], snap.g_name_id[g_old:g_old + G])
        for gi in range(G):
            a, b = int(out.g_wtd_off[g_new + gi]), int(snap.g_wtd_off[g_old + gi])
            n = int(snap.g_wtd_cnt[g_old + gi])
            assert np.array_equal(out.w_name_id[a:a + n], snap.w_name_id[b:b + n])
    assert out.dims["groups"] == int(out.c_group_cnt.sum()) and out.dims["wtd"] == int(out.g_wtd_cnt.sum())
    for c in (3, 17):  # the deleted RayClusters' Pods are still there, with no RayCluster of their key
        assert members(snap, c).size and np.array_equal(out.p_cluster_name_id, snap.p_cluster_name_id)
        assert not ((out.c_ns_id == snap.c_ns_id[c]) & (out.c_name_id == snap.c_name_id[c])).any()

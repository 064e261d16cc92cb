"""The worker-group-edit option without a device: its constant in the Python bindings matches include/kr_engine.h, the Go shim
declares it, the engine and packer entry points take it, off by default, and synthetic.regroup_clusters lays the groups out again."""
import inspect
import os
import re

import numpy as np

from kuberay_b200 import abi, synthetic
from kuberay_b200.engine import Engine
from kuberay_b200.packer import GroupPacker, Packer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "kr_engine.h")).read()


def test_option_constant_matches_the_header():
    assert int(re.search(r"KR_OPT_GROUP_EDITS\s*=\s*(\d+)", HEADER).group(1)) == abi.OPT_GROUP_EDITS == 11


def test_go_shim_declares_the_option():
    src = open(os.path.join(ROOT, "integration", "go", "krengine", "engine.go")).read()
    assert re.search(r"OptGroupEdits\s*=\s*uint32\(C\.KR_OPT_GROUP_EDITS\)", src)
    assert "// OptGroupEdits is KR_OPT_GROUP_EDITS (1:" in src
    assert "KR_OPT_GROUP_EDITS (1, with KR_OPT_FIXED_LAYOUT" in src  # (the option list of SetOption)


def test_engine_and_packers_take_the_keyword_off_by_default():
    assert inspect.signature(Engine.for_snapshot).parameters["group_edits"].default is False
    assert inspect.signature(Packer.__init__).parameters["group_edits"].default is False
    assert inspect.signature(Packer.set_options).parameters["group_edits"].default is False
    assert inspect.signature(GroupPacker.__init__).parameters["group_edits"].default is False
    assert callable(Engine.set_group_edits)


def test_regroup_clusters():
    snap, _ = synthetic.generate(synthetic.config("C2", n_clusters=30, pods_per_cluster=8, groups=3, seed=4, wtd_group_frac=0.5))
    g5, g9 = int(snap.c_group_off[5]), int(snap.c_group_off[9])
    new_id = int(snap.g_name_id.max()) + 100
    # RayCluster 5 gains a copy of its group 1 under a new name; RayCluster 9 loses its group 0 and has its groups reordered
    out = synthetic.regroup_clusters(snap, {5: [(g5, None), (g5 + 1, None), (g5 + 2, None), (g5 + 1, new_id)], 9: [(g9 + 2, None), (g9 + 1, None)]})
    assert out.dims["groups"] == snap.dims["groups"] and out.c_group_cnt[5] == 4 and out.c_group_cnt[9] == 2
    o5, o9 = int(out.c_group_off[5]), int(out.c_group_off[9])
    assert out.g_name_id[o5 + 3] == new_id and out.g_replicas[o5 + 3] == snap.g_replicas[g5 + 1]
    assert np.array_equal(out.g_name_id[o9:o9 + 2], snap.g_name_id[[g9 + 2, g9 + 1]])
    for g_new, g_old in ((o5 + 3, g5 + 1), (o9, g9 + 2)):
        a, b, n = int(out.g_wtd_off[g_new]), int(snap.g_wtd_off[g_old]), int(snap.g_wtd_cnt[g_old])
        assert out.g_wtd_cnt[g_new] == n and np.array_equal(out.w_name_id[a:a + n], snap.w_name_id[b:b + n])
    assert (out.g_cluster_idx[o5:o5 + 4] == 5).all() and out.dims["wtd"] == int(out.g_wtd_cnt.sum())
    for c in (0, 29):  # every other RayCluster keeps its groups, at shifted rows
        gn, go, G = int(out.c_group_off[c]), int(snap.c_group_off[c]), int(snap.c_group_cnt[c])
        assert np.array_equal(out.g_name_id[gn:gn + G], snap.g_name_id[go:go + G])
    assert np.array_equal(out.p_group_name_id, snap.p_group_name_id)

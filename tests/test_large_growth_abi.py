"""The large-growth option without a device: its constants in the Python bindings match include/kr_engine.h, the Go shim declares
it, the engine and packer entry points take it, off by default, the engine reads it back, and synthetic.grow_epochs scales
RayClusters up step by step."""
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
    assert int(re.search(r"KR_OPT_LARGE_GROWTH\s*=\s*(\d+)", HEADER).group(1)) == abi.OPT_LARGE_GROWTH == 12
    caps = dict(re.findall(r"(KR_GROW_\w+)\s*=\s*(\d+)", HEADER))
    assert caps == {"KR_GROW_MAX": "64", "KR_GROW_LIST_MIN": "64", "KR_GROW_LIST_DIV": "64", "KR_GROW_SPILL": "16384"}


def test_go_shim_declares_the_option():
    src = open(os.path.join(ROOT, "integration", "go", "krengine", "engine.go")).read()
    assert re.search(r"OptLargeGrowth\s*=\s*uint32\(C\.KR_OPT_LARGE_GROWTH\)", src)
    assert "// OptLargeGrowth is KR_OPT_LARGE_GROWTH (1:" in src
    assert "KR_OPT_LARGE_GROWTH (1, with KR_OPT_LARGE_CLUSTERS" in src  # (the option list of SetOption)


def test_engine_and_packers_take_the_keyword_off_by_default():
    assert inspect.signature(Engine.for_snapshot).parameters["large_growth"].default is False
    assert inspect.signature(Packer.__init__).parameters["large_growth"].default is False
    assert inspect.signature(Packer.set_options).parameters["large_growth"].default is False
    assert inspect.signature(GroupPacker.__init__).parameters["large_growth"].default is False
    assert callable(Engine.set_large_growth)


def test_set_large_growth_sends_the_option():
    calls = []

    class L:
        def kr_engine_set_option(self, h, option, value):
            calls.append((option, value))
            return 0

    eng = Engine.__new__(Engine)
    eng._L, eng._h = L(), None
    eng.set_large_growth(True)
    eng.set_large_growth(False)
    assert calls == [(abi.OPT_LARGE_GROWTH, 1), (abi.OPT_LARGE_GROWTH, 0)]


def test_packer_options_turn_it_on_only_when_asked():
    seen = []

    class E:
        def __getattr__(self, name):
            return lambda on=True: seen.append(name)

    pk = Packer.__new__(Packer)
    pk.engine = E()
    pk.set_options(large_clusters=True)
    assert seen == ["set_large_clusters"]
    pk.set_options(large_clusters=True, large_growth=True)
    assert seen[1:] == ["set_large_clusters", "set_large_growth"]


def test_grow_epochs():
    snap, _ = synthetic.generate(synthetic.SynthParams(n_clusters=60, pods_per_cluster=20, groups=1, seed=3))
    key = lambda c: (snap.p_ns_id == snap.c_ns_id[c]) & (snap.p_cluster_name_id == snap.c_name_id[c])  # noqa: E731
    before = int(key(7).sum())
    sizes = [64, 65, 130]
    for size, rows in zip(sizes, synthetic.grow_epochs(snap, [7], sizes)):
        assert int(key(7).sum()) == size
        assert rows.size == size - before and key(7)[rows].all()
        before = size

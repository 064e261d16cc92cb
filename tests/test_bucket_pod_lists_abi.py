"""The bucket-pipeline pod-lists option without a device: its value in the Python bindings matches include/kr_engine.h and the Go shim,
Engine.set_bucket_pod_lists sends it, the engine and packer entry points take it off by default, and the packers send it only when
asked for, in their order of options."""
import inspect
import os
import re

from kuberay_b200 import abi
from kuberay_b200.engine import Engine
from kuberay_b200.packer import GroupPacker, Packer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "kr_engine.h")).read()


def test_option_matches_the_header_and_the_go_shim():
    assert int(re.search(r"KR_OPT_BUCKET_POD_LISTS\s*=\s*(\d+)", HEADER).group(1)) == abi.OPT_BUCKET_POD_LISTS == 16
    src = open(os.path.join(ROOT, "integration", "go", "krengine", "engine.go")).read()
    assert re.search(r"OptBucketPodLists\s*=\s*uint32\(C\.KR_OPT_BUCKET_POD_LISTS\)", src)
    assert "// OptBucketPodLists is KR_OPT_BUCKET_POD_LISTS (1:" in src
    assert "KR_OPT_BUCKET_POD_LISTS (1:" in src.split("func (e *Engine) SetOption")[0].rsplit("// SetOption:", 1)[1]  # (the option list of SetOption)


def test_engine_and_packers_take_the_keyword_off_by_default():
    for fn in (Engine.for_snapshot, Packer.__init__, Packer.set_options, GroupPacker.__init__):
        assert inspect.signature(fn).parameters["bucket_pod_lists"].default is False
    assert callable(Engine.set_bucket_pod_lists)


def test_set_bucket_pod_lists_sends_the_option():
    calls = []

    class L:
        def kr_engine_set_option(self, h, option, value):
            calls.append((option, value))
            return 0

    eng = Engine.__new__(Engine)
    eng._L, eng._h = L(), None
    eng.set_bucket_pod_lists(True)
    eng.set_bucket_pod_lists(False)
    assert calls == [(abi.OPT_BUCKET_POD_LISTS, 1), (abi.OPT_BUCKET_POD_LISTS, 0)]


def test_packer_options_turn_it_on_only_when_asked_and_in_order():
    seen = []

    class E:
        def __getattr__(self, name):
            return lambda on=True: seen.append(name)

    pk = Packer.__new__(Packer)
    pk.engine = E()
    pk.set_options(large_clusters=True, huge_growth=True)
    assert "set_bucket_pod_lists" not in seen
    seen.clear()
    pk.set_options(large_clusters=True, large_moves=True, bucket_pod_lists=True, huge_growth=True)
    assert seen == ["set_large_clusters", "set_large_moves", "set_bucket_pod_lists", "set_huge_growth"]
    # every option of the packers' constructors reaches set_options in the same order
    names = list(inspect.signature(Packer.set_options).parameters)[1:]
    for ctor in (Packer.__init__, GroupPacker.__init__):
        params = list(inspect.signature(ctor).parameters)
        assert params[-len(names):] == names, ctor

"""The RayCluster-creation option without a device: its constant in the Python bindings matches include/kr_engine.h, the Go shim
declares it, and the engine and packer entry points take it, off by default."""
import inspect
import os
import re

from kuberay_b200 import abi
from kuberay_b200.engine import Engine
from kuberay_b200.packer import GroupPacker, Packer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "kr_engine.h")).read()


def test_option_constant_matches_the_header():
    assert int(re.search(r"KR_OPT_CLUSTER_CREATES\s*=\s*(\d+)", HEADER).group(1)) == abi.OPT_CLUSTER_CREATES == 9


def test_go_shim_declares_the_option():
    src = open(os.path.join(ROOT, "integration", "go", "krengine", "engine.go")).read()
    assert re.search(r"OptClusterCreates\s*=\s*uint32\(C\.KR_OPT_CLUSTER_CREATES\)", src)
    assert "// OptClusterCreates is KR_OPT_CLUSTER_CREATES (1:" in src


def test_engine_and_packers_take_the_keyword_off_by_default():
    assert inspect.signature(Engine.for_snapshot).parameters["cluster_creates"].default is False
    assert inspect.signature(Packer.__init__).parameters["cluster_creates"].default is False
    assert inspect.signature(Packer.set_options).parameters["cluster_creates"].default is False
    assert inspect.signature(GroupPacker.__init__).parameters["cluster_creates"].default is False
    assert callable(Engine.set_cluster_creates)

"""The workersToDelete-edit option without a device: its constant in the Python bindings matches include/kr_engine.h, the Go shim
declares it, and every entry point that creates an engine takes it."""
import inspect
import os
import re

from kuberay_b200 import abi
from kuberay_b200.engine import Engine
from kuberay_b200.live import LiveArena
from kuberay_b200.packer import Packer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "kr_engine.h")).read()


def test_option_constant_matches_the_header():
    assert int(re.search(r"KR_OPT_WTD_EDITS\s*=\s*(\d+)", HEADER).group(1)) == abi.OPT_WTD_EDITS == 7


def test_go_shim_declares_the_option():
    src = open(os.path.join(ROOT, "integration", "go", "krengine", "engine.go")).read()
    assert re.search(r"OptWtdEdits\s*=\s*uint32\(C\.KR_OPT_WTD_EDITS\)", src)
    assert "KR_OPT_WTD_EDITS (1:" in src


def test_every_engine_entry_point_takes_the_keyword():
    assert inspect.signature(Engine.for_snapshot).parameters["wtd_edits"].default is False
    assert inspect.signature(LiveArena.__init__).parameters["wtd_edits"].default is False
    assert inspect.signature(Packer.__init__).parameters["wtd_edits"].default is False
    assert callable(Engine.set_wtd_edits)

"""The row-granular spec commit without a device: its option and flush-mode constants in the Python bindings match
include/kr_engine.h, the entry point is in the symbol list, the Go shim declares all three, and every entry point that creates an
engine takes the keyword."""
import inspect
import os
import re

from kuberay_b200 import abi
from kuberay_b200.engine import Engine
from kuberay_b200.live import LiveArena
from kuberay_b200.packer import Packer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "kr_engine.h")).read()


def test_constants_match_the_header():
    assert int(re.search(r"KR_OPT_SPEC_ROWS\s*=\s*(\d+)", HEADER).group(1)) == abi.OPT_SPEC_ROWS == 8
    assert int(re.search(r"KR_PACK_SPEC_ROWS\s*=\s*(\d+)", HEADER).group(1)) == abi.PACK_SPEC_ROWS == 64
    assert re.search(r"int kr_snapshot_commit_spec_rows\(kr_engine \*e, const uint32_t \*cluster_rows, uint32_t n\);", HEADER)
    assert "kr_snapshot_commit_spec_rows" in abi.ENGINE_SYMBOLS
    # the mode bit is distinct from every other flush mode bit and commit part
    others = [abi.PACK_POD_ROWS, abi.PACK_FULL, abi.PACK_OBJECT_ROWS, abi.PART_COLUMNS, abi.PART_JSON, abi.PART_OBJECTS]
    assert all(abi.PACK_SPEC_ROWS & o == 0 for o in others)


def test_go_shim_declares_them():
    eng = open(os.path.join(ROOT, "integration", "go", "krengine", "engine.go")).read()
    pk = open(os.path.join(ROOT, "integration", "go", "krengine", "packer.go")).read()
    assert re.search(r"OptSpecRows\s*=\s*uint32\(C\.KR_OPT_SPEC_ROWS\)", eng)
    assert re.search(r"func \(e \*Engine\) CommitSpecRows\(clusterRows \[\]uint32\) error", eng)
    assert "C.kr_snapshot_commit_spec_rows(" in eng
    assert re.search(r"PackSpecRows\s*=\s*uint32\(C\.KR_PACK_SPEC_ROWS\)", pk)


def test_every_engine_entry_point_takes_the_keyword():
    assert inspect.signature(Engine.for_snapshot).parameters["spec_rows"].default is False
    assert inspect.signature(LiveArena.__init__).parameters["spec_rows"].default is False
    assert inspect.signature(Packer.__init__).parameters["spec_rows"].default is False
    assert callable(Engine.set_spec_rows) and callable(Engine.commit_spec_rows)

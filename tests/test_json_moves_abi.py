"""The device-side JSON move commit without a device: its option and flush-mode values in the Python bindings match
include/kr_engine.h and the Go shim, the entry point is declared and in the symbol list, Engine.set_json_moves sends the option, and
the engine and packer entry points take the keyword off by default, in their order of options."""
import inspect
import os
import re

from kuberay_b200 import abi
from kuberay_b200.engine import Engine, lib
from kuberay_b200.packer import GroupPacker, Packer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "kr_engine.h")).read()
GO = os.path.join(ROOT, "integration", "go", "krengine")


def test_values_match_the_header_and_the_go_shim():
    assert int(re.search(r"KR_OPT_JSON_MOVES\s*=\s*(\d+)", HEADER).group(1)) == abi.OPT_JSON_MOVES == 17
    assert int(re.search(r"KR_PACK_JSON_MOVES\s*=\s*(\d+)", HEADER).group(1)) == abi.PACK_JSON_MOVES == 128
    assert re.search(r"int kr_snapshot_commit_json_moves\(kr_engine \*e, const uint32_t \*cluster_rows, uint32_t n\);", HEADER)
    assert "kr_snapshot_commit_json_moves" in abi.ENGINE_SYMBOLS
    others = [abi.PACK_POD_ROWS, abi.PACK_FULL, abi.PACK_OBJECT_ROWS, abi.PACK_SPEC_ROWS, abi.PART_COLUMNS, abi.PART_JSON, abi.PART_OBJECTS]
    assert all(abi.PACK_JSON_MOVES & o == 0 for o in others)
    eng = open(os.path.join(GO, "engine.go")).read()
    pk = open(os.path.join(GO, "packer.go")).read()
    assert re.search(r"OptJsonMoves\s*=\s*uint32\(C\.KR_OPT_JSON_MOVES\)", eng)
    assert "// OptJsonMoves is KR_OPT_JSON_MOVES (1," in eng
    assert "KR_OPT_JSON_MOVES (1," in eng.split("func (e *Engine) SetOption")[0].rsplit("// SetOption:", 1)[1]  # (the option list of SetOption)
    assert re.search(r"func \(e \*Engine\) CommitJsonMoves\(clusterRows \[\]uint32\) error", eng)
    assert "C.kr_snapshot_commit_json_moves(" in eng
    assert re.search(r"PackJsonMoves\s*=\s*uint32\(C\.KR_PACK_JSON_MOVES\)", pk)


def test_the_library_exports_the_symbol():
    assert hasattr(lib(), "kr_snapshot_commit_json_moves")


def test_engine_and_packers_take_the_keyword_off_by_default():
    for fn in (Engine.for_snapshot, Packer.__init__, Packer.set_options, GroupPacker.__init__):
        params = list(inspect.signature(fn).parameters)
        assert inspect.signature(fn).parameters["json_moves"].default is False
        assert params.index("json_moves") == params.index("bucket_pod_lists") + 1, fn  # (in option order, before huge_growth)
    assert callable(Engine.set_json_moves) and callable(Engine.commit_json_moves)


def test_set_json_moves_sends_the_option():
    calls = []

    class L:
        def kr_engine_set_option(self, h, option, value):
            calls.append((option, value))
            return 0

    eng = Engine.__new__(Engine)
    eng._L, eng._h = L(), None
    eng.set_json_moves(True)
    eng.set_json_moves(False)
    assert calls == [(abi.OPT_JSON_MOVES, 1), (abi.OPT_JSON_MOVES, 0)]


def test_packer_options_turn_it_on_only_when_asked_and_in_order():
    seen = []

    class E:
        def __getattr__(self, name):
            return lambda on=True: seen.append(name)

    pk = Packer.__new__(Packer)
    pk.engine = E()
    pk.set_options(spec_rows=True, huge_growth=True)
    assert "set_json_moves" not in seen
    seen.clear()
    pk.set_options(spec_rows=True, bucket_pod_lists=True, json_moves=True, huge_growth=True)
    assert seen == ["set_spec_rows", "set_bucket_pod_lists", "set_json_moves", "set_huge_growth"]
    names = list(inspect.signature(Packer.set_options).parameters)[1:]
    for ctor in (Packer.__init__, GroupPacker.__init__):
        assert list(inspect.signature(ctor).parameters)[-len(names):] == names, ctor

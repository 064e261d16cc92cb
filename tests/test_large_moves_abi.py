"""The large-moves option without a device: its constant in the Python bindings matches include/kr_engine.h, the Go shim declares it,
the engine and packer entry points take it, off by default, set_large_moves sends it, and the region remap of the GPU test's model
(tests/test_gpu_large_moves.py) follows hand-written row maps."""
import inspect
import os
import re

from class_model import Model
from kuberay_b200 import abi
from kuberay_b200.engine import Engine
from kuberay_b200.packer import GroupPacker, Packer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "kr_engine.h")).read()


def test_option_constant_matches_the_header():
    assert int(re.search(r"KR_OPT_LARGE_MOVES\s*=\s*(\d+)", HEADER).group(1)) == abi.OPT_LARGE_MOVES == 13


def test_header_no_longer_lists_large_moves_as_open():
    assert "left open" not in HEADER
    assert HEADER.count("unless KR_OPT_LARGE_MOVES") == 2  # (KR_OPT_CLUSTER_DELETES and KR_OPT_GROUP_EDITS)


def test_go_shim_declares_the_option():
    src = open(os.path.join(ROOT, "integration", "go", "krengine", "engine.go")).read()
    assert re.search(r"OptLargeMoves\s*=\s*uint32\(C\.KR_OPT_LARGE_MOVES\)", src)
    assert "// OptLargeMoves is KR_OPT_LARGE_MOVES (1:" in src
    assert "KR_OPT_LARGE_MOVES (1, with" in src  # (the option list of SetOption)


def test_engine_and_packers_take_the_keyword_off_by_default():
    assert inspect.signature(Engine.for_snapshot).parameters["large_moves"].default is False
    assert inspect.signature(Packer.__init__).parameters["large_moves"].default is False
    assert inspect.signature(Packer.set_options).parameters["large_moves"].default is False
    assert inspect.signature(GroupPacker.__init__).parameters["large_moves"].default is False
    assert callable(Engine.set_large_moves)


def test_set_large_moves_sends_the_option():
    calls = []

    class L:
        def kr_engine_set_option(self, h, option, value):
            calls.append((option, value))
            return 0

    eng = Engine.__new__(Engine)
    eng._L, eng._h = L(), None
    eng.set_large_moves(True)
    eng.set_large_moves(False)
    assert calls == [(abi.OPT_LARGE_MOVES, 1), (abi.OPT_LARGE_MOVES, 0)]


def test_packer_options_turn_it_on_only_when_asked():
    seen = []

    class E:
        def __getattr__(self, name):
            return lambda on=True: seen.append(name)

    pk = Packer.__new__(Packer)
    pk.engine = E()
    pk.set_options(large_clusters=True, cluster_deletes=True)
    assert seen == ["set_large_clusters", "set_cluster_deletes"]
    pk.set_options(large_clusters=True, cluster_deletes=True, large_moves=True)
    assert seen[2:] == ["set_large_clusters", "set_cluster_deletes", "set_large_moves"]


def _model():
    """A model with the GPU test's option on (imported lazily: the GPU test module needs no device to import, only to run)."""
    from test_gpu_large_moves import MovesModel
    m = MovesModel.of(Model(10, 2000, True, True))
    m.caps, m.offs, m.cursor = {2: 200, 5: 300, 9: 500}, {2: 0, 5: 200, 9: 500}, 1000
    return m


def test_model_region_remap():
    # row 2 deleted, the last row (9) moves into it: the mover's region goes to row 2, row 9's entry goes
    m = _model()
    m.moves = {2: -1, 9: 2}
    assert m.row_map([2, 9], 3, 0, False) is None
    assert m.caps == {2: 500, 5: 300} and m.offs == {2: 500, 5: 200} and m.cursor == 1000
    # row 5 regrouped in place, row 9 deleted: the regrouped one keeps its region, the deleted one's is abandoned (cursor stays)
    m = _model()
    m.moves = {5: 5, 9: -1}
    assert m.row_map([5, 9], 3, 0, False) is None
    assert m.caps == {2: 200, 5: 300} and m.offs == {2: 0, 5: 200} and m.cursor == 1000
    # an ordinary row deleted and a large one (9) moving into it; a map over the cap takes the full pass and remaps nothing
    m = _model()
    m.moves = {3: -1, 9: 3}
    assert m.row_map([3, 9], 3, 0, False) is None and m.caps == {2: 200, 3: 500, 5: 300}
    m = _model()
    m.moves = {2: -1}
    assert m.row_map([2], 5000, 0, False) == "map cap" and m.caps == {2: 200, 5: 300, 9: 500}
    # without the option the same map is "large gone row"
    assert Model.row_map(m, [2], 2, 0, False) == "large gone row"

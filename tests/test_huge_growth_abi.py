"""The huge-growth option without a device: its value and the tile reserve in the Python bindings match include/kr_engine.h, the Go
shim declares it, the engine and packer entry points take it, off by default, and it is sent only when asked for; and the region
arena fills before the resident tiles can pass the engine's tile capacity."""
import inspect
import os
import re

import numpy as np

from class_model import region_arena
from kuberay_b200 import abi
from kuberay_b200.engine import Engine
from kuberay_b200.packer import GroupPacker, Packer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "kr_engine.h")).read()
ENGINE = open(os.path.join(ROOT, "kuberay_b200", "csrc", "kr_engine.cu")).read()


def resident_tiles(max_pods):
    """Resident tiles of the tile scratch an engine of kr_config.max_pods allocates (kr_engine.cu: resident_tiles)."""
    n_huge = max_pods // (abi.LARGE_MAX_PODS + 1)
    return (max_pods * 5 // 4 + 32 * (n_huge + 1)) // abi.LARGE_MAX_PODS + n_huge + 2


def test_option_and_reserve_match_the_header():
    assert int(re.search(r"KR_OPT_HUGE_GROWTH\s*=\s*(\d+)", HEADER).group(1)) == abi.OPT_HUGE_GROWTH == 14
    assert int(re.search(r"KR_HUGE_GROW_TILES\s*=\s*(\d+)", HEADER).group(1)) == abi.HUGE_GROW_TILES == 32


def test_go_shim_declares_the_option():
    src = open(os.path.join(ROOT, "integration", "go", "krengine", "engine.go")).read()
    assert re.search(r"OptHugeGrowth\s*=\s*uint32\(C\.KR_OPT_HUGE_GROWTH\)", src)
    assert "// OptHugeGrowth is KR_OPT_HUGE_GROWTH (1:" in src
    assert "KR_OPT_HUGE_GROWTH (1, with KR_OPT_LARGE_CLUSTERS" in src  # (the option list of SetOption)


def test_engine_and_packers_take_the_keyword_last_and_off_by_default():
    for fn in (Engine.for_snapshot, Packer.__init__, Packer.set_options, GroupPacker.__init__):
        params = inspect.signature(fn).parameters
        assert params["huge_growth"].default is False
        assert list(params)[-1] == "huge_growth"
    assert callable(Engine.set_huge_growth)


def test_set_huge_growth_sends_the_option():
    calls = []

    class L:
        def kr_engine_set_option(self, h, option, value):
            calls.append((option, value))
            return 0

    eng = Engine.__new__(Engine)
    eng._L, eng._h = L(), None
    eng.set_huge_growth(True)
    eng.set_huge_growth(False)
    assert calls == [(abi.OPT_HUGE_GROWTH, 1), (abi.OPT_HUGE_GROWTH, 0)]


def test_packer_options_turn_it_on_only_when_asked():
    seen = []

    class E:
        def __getattr__(self, name):
            return lambda on=True: seen.append(name)

    pk = Packer.__new__(Packer)
    pk.engine = E()
    pk.set_options(large_clusters=True, huge_clusters=True, large_growth=True)
    assert "set_huge_growth" not in seen
    seen.clear()
    pk.set_options(large_clusters=True, huge_clusters=True, large_growth=True, huge_growth=True)
    assert seen == ["set_large_clusters", "set_huge_clusters", "set_large_growth", "set_huge_growth"]


def test_resident_tiles_matches_the_engine():
    assert "const size_t Np = cfg.max_pods, n_huge = Np / (KR_LARGE_MAX_PODS + 1);" in ENGINE
    assert "return (Np * 5 / 4 + 32 * (n_huge + 1)) / kHugeTile + n_huge + 2;" in ENGINE
    assert "static constexpr int kHugeTile = KR_LARGE_MAX_PODS;" in open(os.path.join(ROOT, "kuberay_b200", "csrc", "kr_large.cuh")).read()


def test_the_arena_fills_before_the_tile_capacity():
    """The tile-capacity void of k_inc_grow<true> guards a state the arena rules out.  Every region in use lies in the arena, apart
    from the others.  A huge RayCluster lists more than 8 192 Pods, so its bucket and region span at least 10 272 ranks
    (large_region_cap) and its region holds at least 10 272 - stride records for its 2 tiles (k tiles need more than
    8 192 (k - 1) ranks: fewer tiles per record).  So the resident tiles are at most 2 x arena / (10 272 - stride), which is below
    resident_tiles for every max_pods up to 20 million and every stride."""
    np_ = np.arange(1, 20_000_001, dtype=np.int64)
    arena = region_arena(np_)
    cap = resident_tiles(np_)
    for stride in (64, 128, 256):
        most = 2 * arena // (10272 - stride)
        assert (most < cap).all(), np_[most >= cap][:5]

"""The host model of the engine's classification (tests/class_model.py) against the sources it restates: its constants by regex
against include/kr_engine.h and kuberay_b200/csrc, and large_region_cap against a transcription of the C expression with 32-bit
unsigned arithmetic at its edges.  The GPU streams trust the model's predictions only as far as these hold."""
import re
from pathlib import Path

import numpy as np

import class_model as cm
from kuberay_b200 import abi

ROOT = Path(__file__).resolve().parents[1]
CSRC = ROOT / "kuberay_b200" / "csrc"


def _source(path):
    return " ".join(path.read_text().split())


def test_constants_match_the_sources():
    h = _source(ROOT / "include" / "kr_engine.h")
    m = re.search(r"enum \{ KR_GROW_MAX = (\d+), KR_GROW_LIST_MIN = (\d+), KR_GROW_LIST_DIV = (\d+), KR_GROW_SPILL = (\d+) \};", h)
    assert m and tuple(map(int, m.groups())) == (cm.GROW_MAX, cm.GROW_LIST_MIN, cm.GROW_LIST_DIV, cm.GROW_SPILL)
    assert re.search(r"enum \{ KR_LARGE_MAX_PODS = (\d+) \};", h).group(1) == str(abi.LARGE_MAX_PODS)
    assert re.search(r"#define KR_SMEM_GROUPS (\d+)", _source(CSRC / "kr_decide.cuh")).group(1) == str(cm.SMEM_GROUPS)
    eng = _source(CSRC / "kr_engine.cu")
    assert re.search(r"constexpr uint32_t kMapMax = (\d+);", eng).group(1) == str(cm.MAP_MAX)
    assert re.search(r"constexpr uint32_t kAdoptMax = (\d+);", eng).group(1) == str(cm.ADOPT_MAX)
    # the region arena, the per-cluster list's cap and the first stride
    assert "const size_t entries = Np * 5 / 4 + 32 * (Np / 257 + 1);" in eng
    assert cm.region_arena(1000) == 1000 * 5 // 4 + 32 * (1000 // 257 + 1)
    assert "std::max<uint32_t>(KR_GROW_LIST_MIN, n.n_clusters / KR_GROW_LIST_DIV)" in eng
    assert "const uint64_t want = n.n_clusters ? ((uint64_t)n.n_pods * 5 / 4 + n.n_clusters - 1) / n.n_clusters : 0;" in eng
    assert "while (st < want && st < 512) st <<= 1; return st <= 256 ? st : 0;" in eng
    # the rules the model states: a gone row with a region voids the map; rows past a smaller count lose their regions before the
    # pass; a regrowth is not newly listed, nor a wide RayCluster
    assert "for (uint32_t o : m.gone) ok = ok && !std::binary_search(e->large_rows.begin(), e->large_rows.end(), o);" in eng
    assert "std::lower_bound(e->large_rows.begin(), e->large_rows.end(), e->sizes.n_clusters)" in eng
    large = _source(CSRC / "kr_large.cuh")
    assert "s_new[i] = e.z == 0 && !(wide && s.c_group_cnt[e.x] > KR_SMEM_GROUPS);" in large
    assert "s_ok = ok && off <= arena && (listed == 0 || n_list + listed <= list_cap);" in large


def _c_region_cap(count, stride):
    """The C expression of kr_bucket2.cuh's large_region_cap, evaluated in uint32 as the kernel does."""
    u = np.uint32
    with np.errstate(over="ignore"):
        want = ((u(count) + u(count) // u(4) + u(31)) // u(32)) * u(32)
        capped = want if count > abi.LARGE_MAX_PODS else (want if want < u(abi.LARGE_MAX_PODS) else u(abi.LARGE_MAX_PODS))
        return int(u(capped) - u(stride))


def test_region_cap_formula():
    src = _source(CSRC / "kr_bucket2.cuh")
    body = re.search(r"uint32_t large_region_cap\(uint32_t count, uint32_t stride\) \{ (.*?) \}", src).group(1)
    assert body == ("const uint32_t want = ((count + count / 4 + 31) / 32) * 32; return (count > KR_LARGE_MAX_PODS ? want : "
                    "(want < KR_LARGE_MAX_PODS ? want : (uint32_t)KR_LARGE_MAX_PODS)) - stride;"), body
    edges = [0, 1, 31, 32, 64, 65, 128, 129, 200, 255, 256, 257, 300, 1000, 6552, 6553, 6554, 6555, 8191, 8192, 8193, 9000, 65536]
    for count in edges:
        for stride in (0, 64, 128, 256):
            assert cm.large_region_cap(count, stride) == _c_region_cap(count, stride), (count, stride)
    # a RayCluster just past 256 Pods at the 64 stride holds 1.25 x rounded up to 32, and the cap binds from 6 554 Pods on
    assert cm.large_region_cap(257, 64) == 352 - 64
    assert cm.large_region_cap(6553, 64) == 8192 - 64 and cm.large_region_cap(6554, 64) == 8192 - 64
    assert cm.large_region_cap(8193, 64) == 10272 - 64


def _model(n=600, pods=12000):
    m = cm.Model(n, pods, large=True, wide=True, arena=cm.region_arena(20000))
    assert m.stride == 64
    m.valid = True
    return m


def test_growth_in_an_incremental_epoch():
    m = _model()
    groups = np.full(600, 2)
    peak = np.full(600, 20)
    peak[[5, 9]] = [65, 300]
    assert m.grow(peak, groups) is None
    assert m.caps == {5: cm.large_region_cap(65, 64), 9: cm.large_region_cap(300, 64)}
    assert m.offs == {5: 0, 9: m.caps[5]} and m.cursor == m.caps[5] + m.caps[9]
    # a regrowth: a new region at the cursor; the old one is abandoned
    cur = m.cursor
    peak[9] = 64 + m.caps[9] + 1
    assert m.grow(peak, groups) is None
    assert m.offs[9] == cur and m.caps[9] == cm.large_region_cap(int(peak[9]), 64)


def test_growth_limits():
    groups = np.full(600, 2)
    m = _model()
    peak = np.full(600, 20)
    peak[:65] = 70
    assert m.grow(peak, groups) == "grow list" and not m.caps
    m = _model(n=600)
    peak = np.full(600, 20)
    peak[:40] = 70
    assert m.grow(peak, groups) is None  # 40 listed of max(64, 600 / 64)
    peak[40:70] = 70
    assert m.grow(peak, groups) == "list cap"
    wide = groups.copy()
    wide[40:70] = 33  # wide ones are listed already: no cap binds
    assert m.grow(peak, wide) is None
    m = _model()
    peak = np.full(600, 20)
    peak[3] = abi.LARGE_MAX_PODS + 1
    assert m.grow(peak, groups) == "past 8192 pods"
    m = _model()
    m.cursor = m.arena - 100
    peak = np.full(600, 20)
    peak[3] = 300
    assert m.grow(peak, groups) == "arena"


def test_row_maps_and_shrinking():
    m = _model()
    groups = np.full(600, 2)
    counts = np.full(600, 20)
    counts[[10, 599]] = [400, 1200]
    m.full_pass(counts, groups)
    assert set(m.caps) == {10, 599} and m.stride == 64
    assert m.row_map([599], 1, 0, False) == "large gone row"
    assert m.row_map([4, 598], 3, 0, False) is None
    assert m.row_map([1], cm.MAP_MAX + 1, 0, False) == "map cap"
    assert m.row_map([], cm.MAP_MAX, cm.ADOPT_MAX, True) is None
    assert m.row_map([], cm.MAP_MAX, cm.ADOPT_MAX + 1, True) == "adoption cap"
    assert m.row_map([], cm.MAP_MAX, cm.ADOPT_MAX + 1, False) is None
    # the last row deleted: its region goes before the full pass, the other keeps its own
    m.full_pass(counts[:599], groups[:599])
    assert set(m.caps) == {10} and m.nc == 599

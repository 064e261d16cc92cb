"""No GPU: every launch in kuberay_b200/csrc/kr_engine.cu whose grid is sized by the SM count is covered by a multi-trip test in
tests/test_gpu_launch_shapes.py (its COVERAGE table), the grid rules its `Shapes` helper mirrors are the engine's, and the
read-only KR_OPT_SM_COUNT matches across the header, the Python bindings and the Go shim."""
import ast
import os
import re

from kuberay_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENGINE = open(os.path.join(ROOT, "kuberay_b200", "csrc", "kr_engine.cu")).read()
HEADER = open(os.path.join(ROOT, "include", "kr_engine.h")).read()
GPU_FILE = os.path.join(ROOT, "tests", "test_gpu_launch_shapes.py")
SM_SIZED = re.compile(r"\bsm_count\b|\bplace_ctas\b|\bhash_ctas_per_sm\b|\bctas_per_sm\b|^grid$|\(grid,")


def _top_level_args(text, start):
    """The comma-separated arguments from text[start] up to the closing parenthesis or `>>>` at depth 0."""
    args, depth, cur, i = [], 0, "", start
    while i < len(text):
        if depth == 0 and (text.startswith(">>>", i) or text[i] == ")"):
            break
        ch = text[i]
        depth += {"(": 1, ")": -1}.get(ch, 0)
        if ch == "," and depth == 0:
            args.append(cur.strip())
            cur = ""
        else:
            cur += ch
        i += 1
    return args + [cur.strip()]


def sm_sized_launches():
    """{kernel: [grid expressions]} of the launches whose grid reads the SM count (directly, through launch_hash's ctas_per_sm, or
    through launch_pass's incremental `grid`)."""
    out = {}
    for m in re.finditer(r"\b(k_\w+)(?:<[^<>;]*>)?<<<", ENGINE):
        grid = _top_level_args(ENGINE, m.end())[0]
        if SM_SIZED.search(grid):
            out.setdefault(m.group(1), []).append(grid)
    for m in re.finditer(r"\blaunch_pdl\((k_\w+)(?:<[^<>;]*>)?,\s*", ENGINE):
        grid = _top_level_args(ENGINE, m.end())[0]
        if SM_SIZED.search(grid):
            out.setdefault(m.group(1), []).append(grid)
    return out


def gpu_file():
    tree = ast.parse(open(GPU_FILE).read())
    coverage = tests = None
    for node in tree.body:
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "COVERAGE" for t in node.targets):
            coverage = ast.literal_eval(node.value)
    tests = {n.name for n in tree.body if isinstance(n, ast.FunctionDef) and n.name.startswith("test_")}
    return coverage, tests


def test_the_scan_finds_the_known_launches():
    found = sm_sized_launches()
    assert set(found) >= {"k_hash3", "k_hash2", "k_clear", "k_place_fused", "k_creates_fused", "k_inc_aux_clear", "k_inc_aux_insert",
                          "k_inc_wtd_clear", "k_inc_wtd_insert", "k_inc_wtd_resolve", "k_inc_orphan_adopt", "k_inc_grow", "k_inc_refresh",
                          "k_inc_admit", "k_inc_clusters_rekey", "k_inc_groups_gather"}, sorted(found)
    # launch_pass's incremental `grid` is the SM count's
    assert len(re.findall(r"const int grid = e->sm_count \* 2;", ENGINE)) == 1


def test_every_sm_sized_launch_has_a_multi_trip_test():
    coverage, tests = gpu_file()
    missing = sorted(set(sm_sized_launches()) - set(coverage))
    assert not missing, f"SM-sized launches without a test in test_gpu_launch_shapes.py's COVERAGE: {missing}"
    for kernel, names in coverage.items():
        assert names and set(names) <= tests, (kernel, set(names) - tests)


def test_shapes_mirror_the_grids():
    launches = sm_sized_launches()
    assert launches["k_hash3"] == ["std::min<uint32_t>(ngroups, (uint32_t)e->sm_count * 2)"]
    assert launches["k_hash2"] == ["std::min<uint32_t>((n + 127) / 128, (uint32_t)e->sm_count * ctas_per_sm)"]
    assert "if (ngroups <= (uint32_t)e->sm_count * 4)" in ENGINE and "const uint32_t ngroups = (n + 31) / 32;" in ENGINE
    assert re.search(r"k_hash3<1, 0><<<[^;]*, 64, sizeof\(H3Smem\)", ENGINE) and re.search(r"k_hash2<4, 1><<<[^;]*\), 128, 0,", ENGINE)
    assert "int hash_ctas_per_sm = 2;" in ENGINE and "int place_ctas = 1;" in ENGINE
    assert re.search(r"launch_hash\(e, e->sh, [^;]*, 4\);", ENGINE)  # kr_hash_batch: 4 CTAs per SM
    assert launches["k_place_fused"] == ["dim3(e->sm_count * e->place_ctas)"]
    assert launches["k_creates_fused"] == ["dim3(e->sm_count)"]
    assert re.search(r"launch_pdl\(k_place_fused, [^;]*, dim3\(1024\)", ENGINE) and re.search(r"launch_pdl\(k_creates_fused, [^;]*, dim3\(1024\)", ENGINE)
    emit = open(os.path.join(ROOT, "kuberay_b200", "csrc", "kr_emit.cuh")).read()
    assert "p0 < n; p0 += 4 * stride)" in emit  # four Pods per thread per trip
    assert "g < n.n_groups; g += gridDim.x * nw)" in emit  # one group per warp per trip
    for k in ("k_inc_aux_insert", "k_inc_wtd_insert", "k_inc_clusters_rekey"):
        assert re.fullmatch(r"std::min<uint32_t>\(grid, \(n\.n_\w+ \+ 255\) / 256 \+ 1\)", launches[k][0]), launches[k]
    assert launches["k_inc_refresh"] == ["std::min<uint32_t>((uint32_t)e->sm_count * 2, (e->sizes.n_clusters + 255) / 256 + 1)"]
    assert launches["k_inc_grow"] == ["e->sm_count", "e->sm_count"] and "k_inc_grow<true><<<e->sm_count, 256," in ENGINE
    large = open(os.path.join(ROOT, "kuberay_b200", "csrc", "kr_large.cuh")).read()
    assert "k < n_spill && k < KR_GROW_SPILL; k += gridDim.x * blockDim.x)" in large  # the spilled records, over the whole grid
    for k in ("k_inc_wtd_resolve", "k_inc_orphan_adopt"):
        assert all(g.startswith("std::min<uint32_t>((uint32_t)e->sm_count * 4, (") and g.endswith(" + 255) / 256 + 1)") for g in launches[k]), launches[k]


def test_sm_count_option_matches_everywhere():
    assert int(re.search(r"KR_OPT_SM_COUNT\s*=\s*(\d+)", HEADER).group(1)) == abi.OPT_SM_COUNT == 15
    assert "case KR_OPT_SM_COUNT: *value = (uint64_t)e->sm_count; return KR_OK;" in ENGINE
    assert 'if (option == KR_OPT_SM_COUNT) return fail(e, KR_E_INVALID, "KR_OPT_SM_COUNT can only be read");' in ENGINE
    # read once, at creation, after the device's count; at most that count, and only a positive number counts
    create = ENGINE[ENGINE.index("int kr_engine_create("):]
    dev = create.index("cudaDevAttrMultiProcessorCount")
    env = create.index('getenv("KR_SM_COUNT")')
    assert dev < env and ENGINE.count('getenv("KR_SM_COUNT")') == 1
    assert 'if (const char *g = getenv("KR_SM_COUNT")) if (atoi(g) > 0) e->sm_count = std::min(e->sm_count, atoi(g));' in create
    go = open(os.path.join(ROOT, "integration", "go", "krengine", "engine.go")).read()
    assert re.search(r"OptSMCount\s*=\s*uint32\(C\.KR_OPT_SM_COUNT\)", go)
    assert re.search(r"C\.kr_engine_get_option\(e\.h, C\.uint32_t\(option\), &v\)", go)

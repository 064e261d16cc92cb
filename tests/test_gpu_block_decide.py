"""The block decide of the per-cluster kernels (kuberay_b200/csrc/kr_decide.cuh: decide_cluster_block): a large RayCluster is decided
by the 4 warps of k_decide_large, a huge one by the 16 warps of k_decide_huge, each warp over its own contiguous range of List
positions.  Every case puts a decision on, or next to, the edge of a warp's range.

Every full pass is compared with the oracle and with the same snapshot with the option that takes the RayCluster off the bucket
pipeline (the sort pipeline then decides it); every incremental epoch with the oracle."""
import numpy as np
import pytest

from harness import (POD_COLS, Driver, b32, compact, grown_fleet, head_row, members, move, parity_on_off, scale_to, set_phase, spec_bytes,
                     with_wtd_lists, workers)
from kuberay_b200 import abi, synthetic

pytestmark = pytest.mark.gpu

MAX_CREATES = 1 << 18
WARPS = {"large": 4, "huge": 16}  # warps of k_decide_large / k_decide_huge (kr_large.cuh)
SIZE = {"large": 3000, "huge": 12000}


def edge(P, kind, k=1):
    """First List position of warp k's range for a RayCluster of P pods."""
    w = WARPS[kind]
    per = ((P + w - 1) // w + 31) // 32 * 32
    return min(k * per, P)


def _parity(snap, flags, oracle_mod, kind, wide=False):
    if kind == "large":
        return parity_on_off(snap, flags, oracle_mod, "large_clusters", wide_clusters=wide, max_creates=MAX_CREATES)
    return parity_on_off(snap, flags, oracle_mod, "huge_clusters", large_clusters=True, wide_clusters=wide, max_creates=MAX_CREATES)


def _launched(names, huge):
    assert "k_decide_large" in names, names
    assert ("k_decide_huge" in names) == huge, names


def _fleet(kind, n_big=3, seed=5, groups=1, n_clusters=None):
    """Ordinary RayClusters of 20 pods and n_big healthy ones of SIZE[kind] pods, their worker group asking for what it has."""
    n_clusters = n_clusters or max(600, n_big * SIZE[kind] // 10)
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=n_clusters, pods_per_cluster=20, groups=groups, seed=seed, healthy=True))
    big = [i * (n_clusters // n_big) for i in range(n_big)]
    synthetic.grow_clusters(snap, big, SIZE[kind])
    for c in big:
        snap.c_flags[c] &= ~np.uint32(abi.CF_SKIP | abi.CF_SUSPEND | abi.CF_UPGRADE_RECREATE | abi.CF_AUTOSCALING)
        snap.c_flags[c] |= np.uint32(abi.CF_HEAD_EXPECT_OK)
        snap.c_suspend_status[c] = abi.SUSPEND_NONE
        snap.c_ext_err_kind[c] = abi.EXT_ERR_NONE
        for gi in range(int(snap.c_group_cnt[c])):
            g = int(snap.c_group_off[c]) + gi
            scale_to(snap, g, int((snap.p_group_name_id[workers(snap, c)] == snap.g_name_id[g]).sum()))
    return snap, compact(flags), big


def _put_head_at(snap, c, p):
    """Swap RayCluster c's head with the pod at List position p (every pod column; the head-aux row follows)."""
    m = members(snap, c)
    h = head_row(snap, c)
    a, b = int(snap.h_pod_idx[h]), int(m[p])
    for col in POD_COLS:
        snap.cols[col][[a, b]] = snap.cols[col][[b, a]]
    snap.h_pod_idx[h] = b


def _make_head(snap, row):
    snap.p_packed[row] = (snap.p_packed[row] & ~np.uint32(3 << abi.PP_NODE_TYPE_SHIFT)) | np.uint32(abi.NT_HEAD << abi.PP_NODE_TYPE_SHIFT)


# ------------------------------------------------------------------------------------------------ sizes at awkward warp splits
@pytest.mark.parametrize("size", [257, 300, 2047, 2048, 2049, 8192, 8193, 16385, 20000, 100000])
def test_sizes_at_awkward_warp_splits(size, oracle_mod):
    snap, flags = grown_fleet(size)
    huge = size > abi.LARGE_MAX_PODS
    got, names, stride = _parity(snap, flags, oracle_mod, "huge" if huge else "large")
    assert got.clusters["n_pods"][0] == size and stride == 64
    _launched(names, huge)


# ------------------------------------------------------------------------------------------------ decisions across warp ranges
@pytest.mark.parametrize("kind", ["large", "huge"])
@pytest.mark.parametrize("where", ["first", "last", "edge", "before_edge"])
def test_head_position(kind, where, oracle_mod):
    snap, flags, (a, b, c) = _fleet(kind)
    P = members(snap, a).size
    p = {"first": 0, "last": P - 1, "edge": edge(P, kind), "before_edge": edge(P, kind, 2) - 1}[where]
    for cl in (a, b, c):
        _put_head_at(snap, cl, p)
    set_phase(snap, [int(snap.h_pod_idx[head_row(snap, b)])], abi.PHASE_FAILED)  # b: its head is deleted
    _make_head(snap, members(snap, c)[edge(P, kind, WARPS[kind] - 1)])              # c: a second head in the last range
    got, names, _ = _parity(snap, flags, oracle_mod, kind)
    _launched(names, kind == "huge")
    assert got.clusters["head_pod_idx"][a] == members(snap, a)[p]
    assert got.clusters["head_action"][b] == abi.HEAD_DELETE
    assert got.clusters["head_action"][c] == abi.HEAD_MULTIPLE and got.clusters["n_heads"][c] == 2


@pytest.mark.parametrize("kind", ["large", "huge"])
def test_unhealthy_pods_in_the_first_and_last_range(kind, oracle_mod):
    snap, flags, (a, b, _c) = _fleet(kind)
    for cl, ends in ((a, (True, True)), (b, (False, True))):
        m = members(snap, cl)
        rows = ([m[1], m[2]] if ends[0] else []) + ([m[-1], m[-2]] if ends[1] else [])
        set_phase(snap, rows, abi.PHASE_FAILED)
    got, names, _ = _parity(snap, flags, oracle_mod, kind)
    _launched(names, kind == "huge")
    assert got.groups["n_unhealthy"][snap.c_group_off[a]] == 4


@pytest.mark.parametrize("kind", ["large", "huge"])
@pytest.mark.parametrize("random_delete", [False, True])
def test_scale_down_prefix_around_a_range_edge(kind, random_delete, oracle_mod):
    """a / b / c: a delete prefix whose last pod is one before, at, and one past the first position of warp 1's range (the head is
    at position 0, so the k-th candidate sits at position k)."""
    snap, flags, big = _fleet(kind)
    flags.env_random_pod_delete = int(random_delete)
    for cl, d in zip(big, (-1, 0, 1)):
        m = members(snap, cl)
        _put_head_at(snap, cl, 0)
        snap.c_flags[cl] |= np.uint32(abi.CF_AUTOSCALING)
        last = edge(m.size, kind) + d  # position of the last deleted pod
        scale_to(snap, int(snap.c_group_off[cl]), workers(snap, cl).size - last)
    got, names, _ = _parity(snap, flags, oracle_mod, kind)
    _launched(names, kind == "huge")
    for cl, d in zip(big, (-1, 0, 1)):
        m = members(snap, cl)
        idx, codes = got.actions_of(cl)
        if random_delete:
            assert sorted(idx.tolist()) == m[1:edge(m.size, kind) + d + 1].tolist()
        else:
            assert idx.size == 0


@pytest.mark.parametrize("kind", ["large", "huge"])
@pytest.mark.parametrize("random_delete", [False, True])
def test_workers_to_delete_spread_over_ranges(kind, random_delete, oracle_mod):
    snap, flags, (a, b, _c) = _fleet(kind)
    flags.env_random_pod_delete = int(random_delete)
    lists = [[] for _ in range(snap.dims["groups"])]
    for cl, down in ((a, 0), (b, 300)):
        m = members(snap, cl)
        snap.c_flags[cl] |= np.uint32(abi.CF_AUTOSCALING)
        g = int(snap.c_group_off[cl])
        picks = [m[edge(m.size, kind, k) + o] for k in range(WARPS[kind]) for o in (1, 5)]
        lists[g] = [int(snap.p_name_id[r]) for r in picks] + [0x7F000000 + cl]
        scale_to(snap, g, workers(snap, cl).size - len(picks) - down)
    snap = with_wtd_lists(snap, lists)
    got, names, _ = _parity(snap, flags, oracle_mod, kind)
    _launched(names, kind == "huge")
    _, codes = got.actions_of(a)
    assert (codes == abi.ACT_DELETE_WTD).sum() == 2 * WARPS[kind]


@pytest.mark.parametrize("kind", ["large", "huge"])
def test_32_interleaved_worker_groups(kind, oracle_mod):
    """Every warp sees every worker group; one group scales down across ranges, one up, one has an unhealthy pod late in List order,
    and some pods name no group of theirs."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=SIZE[kind] // 8, pods_per_cluster=20, groups=32, seed=11, healthy=True))
    flags = compact(flags)
    a, b = 0, SIZE[kind] // 16
    synthetic.grow_clusters(snap, [a, b], SIZE[kind])
    for cl in (a, b):
        snap.c_flags[cl] &= ~np.uint32(abi.CF_SKIP | abi.CF_SUSPEND | abi.CF_UPGRADE_RECREATE | abi.CF_AUTOSCALING)
        snap.c_flags[cl] |= np.uint32(abi.CF_HEAD_EXPECT_OK)
        snap.c_suspend_status[cl] = abi.SUSPEND_NONE
        snap.c_ext_err_kind[cl] = abi.EXT_ERR_NONE
        w = workers(snap, cl)
        g0, G = int(snap.c_group_off[cl]), int(snap.c_group_cnt[cl])
        assert G == 32
        snap.p_group_name_id[w] = snap.g_name_id[g0 + np.arange(w.size) % G]
        snap.p_group_name_id[w[::97]] = np.uint32(0x7E000000)  # in no group
        for gi in range(G):
            scale_to(snap, g0 + gi, int((snap.p_group_name_id[w] == snap.g_name_id[g0 + gi]).sum()))
        scale_to(snap, g0 + 3, int(snap.g_replicas[g0 + 3]) - w.size // 64)
        scale_to(snap, g0 + 7, int(snap.g_replicas[g0 + 7]) + 40)
    wb = workers(snap, b)
    set_phase(snap, [wb[wb.size - 40 + 20]], abi.PHASE_FAILED)
    snap.g_flags[snap.c_group_off[a] + 5] |= np.uint32(abi.GF_SUSPEND)
    snap.g_flags[snap.c_group_off[a] + 9] &= ~np.uint32(abi.GF_EXPECT_OK)
    got, names, _ = _parity(snap, flags, oracle_mod, kind)
    _launched(names, kind == "huge")
    assert got.clusters["stop_after_group"][b] < 32  # a group aborts: the ones after it are never reached


@pytest.mark.parametrize("kind", ["large", "huge"])
@pytest.mark.parametrize("case", ["suspended_group", "suspend", "suspending", "skip", "status_only_error", "head_expectations",
                                  "group_expectations", "no_group"])
def test_cluster_and_group_states(kind, case, oracle_mod):
    snap, flags, (a, b, _c) = _fleet(kind)
    g = int(snap.c_group_off[a])
    if case == "suspended_group":
        snap.g_flags[g] |= np.uint32(abi.GF_SUSPEND)
    elif case == "suspend":
        snap.c_flags[a] |= np.uint32(abi.CF_SUSPEND)
    elif case == "suspending":
        snap.c_suspend_status[a] = abi.SUSPEND_SUSPENDING
    elif case == "skip":
        snap.c_flags[a] |= np.uint32(abi.CF_SKIP)
    elif case == "status_only_error":
        snap.c_ext_err_kind[a] = abi.EXT_ERR_STATUS_ONLY_NIL
    elif case == "head_expectations":
        snap.c_flags[a] &= ~np.uint32(abi.CF_HEAD_EXPECT_OK)
    elif case == "group_expectations":
        snap.g_flags[g] &= ~np.uint32(abi.GF_EXPECT_OK)
    else:
        m = members(snap, a)
        snap.p_group_name_id[m[[edge(m.size, kind) - 1, edge(m.size, kind), m.size - 1]]] = np.uint32(0x7E000000)
        scale_to(snap, g, workers(snap, a).size - 3 - 100)
    b_flip = members(snap, b)[[edge(members(snap, b).size, kind, k) for k in range(1, WARPS[kind])]]
    set_phase(snap, b_flip, abi.PHASE_PENDING)  # b: not all running, a pod at the head of every range but the first
    _, names, _ = _parity(snap, flags, oracle_mod, kind)
    _launched(names, kind == "huge")


@pytest.mark.parametrize("kind", ["large", "huge"])
def test_recreate_gate_equal_and_different(kind, oracle_mod):
    snap, flags, (a, b, _c) = _fleet(kind)
    ah = snap.h_annot_hash.reshape(-1, 32)
    for cl, match in ((a, False), (b, True)):
        snap.c_flags[cl] |= np.uint32(abi.CF_UPGRADE_RECREATE)
        h = head_row(snap, cl)
        snap.h_version_state[h] = abi.VER_CURRENT
        snap.h_annot_state[h] = abi.ANNOT_HASH32
        digest = b32(spec_bytes(snap, cl))
        ah[h] = np.frombuffer(digest if match else digest[::-1], dtype=np.uint8)
    got, names, _ = _parity(snap, flags, oracle_mod, kind)
    _launched(names, kind == "huge")
    assert got.clusters["path"][a] == abi.PATH_RECREATE_DELETE_ALL and got.clusters["path"][b] == abi.PATH_NORMAL


@pytest.mark.parametrize("kind", ["large", "huge"])
def test_multihost_groups(kind, oracle_mod):
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=SIZE[kind] // 10, pods_per_cluster=20, groups=2, multihost_frac=0.25, seed=9))
    synthetic.grow_clusters(snap, [0], SIZE[kind])
    for gate in (1, 0):
        flags.gate_multihost_indexing = gate
        _, names, _ = _parity(snap, compact(flags), oracle_mod, kind)
        _launched(names, kind == "huge")


def test_wide_and_non_wide_large_and_huge_clusters_in_one_fleet(oracle_mod):
    """A wide huge RayCluster stays with k_decide_large (warp 0), a non-wide one goes to k_decide_huge; likewise for large ones."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=2000, pods_per_cluster=20, groups=1, seed=17))
    synthetic.grow_clusters(snap, [0, 700], 9500)
    synthetic.grow_clusters(snap, [300, 1000, 0, 700], 2000)
    snap = synthetic.widen_clusters(snap, [700, 1000, 1400], 36)
    got, names, _ = _parity(snap, compact(flags), oracle_mod, "huge", wide=True)
    _launched(names, True)
    assert (got.clusters["n_pods"][[0, 700]] == 9500).all()


def test_a_wide_huge_cluster_alone(oracle_mod):
    """The huge part of the list holds only a wide RayCluster: k_decide_huge is launched over it and leaves it to k_decide_large."""
    snap, flags = grown_fleet(10000, n_clusters=800)
    snap = synthetic.widen_clusters(snap, [0], 40)
    got, names, _ = _parity(snap, flags, oracle_mod, "huge", wide=True)
    _launched(names, True)
    assert got.clusters["n_pods"][0] == 10000


# ------------------------------------------------------------------------------------------------ incremental epochs
def _names(dr):
    return {k for k, _ in dr.eng.reconcile_profiled(dr.flags)["kernels"]}


def test_churn_across_the_ranges_of_a_huge_cluster(oracle_mod):
    rng = np.random.default_rng(3)
    snap, flags, big = _fleet("huge", n_big=2, n_clusters=3000)
    dr = Driver(snap, flags, max_creates=MAX_CREATES, large_clusters=True, huge_clusters=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        for epoch in range(6):
            rows = []
            for cl in big:
                m = members(snap, cl)
                at = [edge(m.size, "huge", k) + o for k in range(WARPS["huge"]) for o in (-1, 0)] + rng.choice(m.size, 30).tolist()
                rows += m[np.clip(at, 1, m.size - 1)].tolist()
            snap.p_packed[rows] ^= np.uint32(1 << abi.PP_READY_SHIFT)
            if epoch == 3:
                set_phase(snap, rows[:5], abi.PHASE_FAILED)
            dr.commit_rows(rows, journal=epoch % 2 == 0)
            _, names = dr.check(oracle_mod, expect_incremental=True, profiled=True)
            assert {"k_decide_large", "k_decide_huge"} <= set(names), names
        snap.g_replicas[snap.c_group_off[big[0]]] -= 5000  # a scale-down across most ranges through the object commit
        dr.commit_objects()
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


@pytest.mark.parametrize("target", [100, 0])
def test_a_huge_cluster_shrinking_under_huge_growth(target, oracle_mod):
    """With KR_OPT_HUGE_GROWTH a huge RayCluster that shrinks keeps its place in the huge part of the list until the next full pass."""
    snap, flags, big = _fleet("huge", n_big=1, n_clusters=3000)
    dr = Driver(snap, flags, max_creates=MAX_CREATES, large_clusters=True, huge_clusters=True, large_growth=True, huge_growth=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        m = members(snap, big[0])
        keep = m[:target]
        out = np.setdiff1d(m, keep)
        snap.p_packed[out] = np.uint32(abi.PP_TOMBSTONE)
        for col in POD_COLS:
            if col != "p_packed":
                snap.cols[col][out] = 0
        dr.commit_rows(out)
        got, names = dr.check(oracle_mod, expect_incremental=True, profiled=True)
        assert got.clusters["n_pods"][big[0]] == target
        assert "k_decide_huge" in names
        flip = keep[1::7]
        snap.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        dr.commit_rows(flip)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


def test_growth_that_promotes_a_cluster_in_the_pass(oracle_mod):
    """k_inc_grow lists a RayCluster in the pass (a CTA of k_decide_large past the list) and makes another huge, while a huge one
    is decided by k_decide_huge."""
    snap, flags, big = _fleet("huge", n_big=1, n_clusters=4000)
    dr = Driver(snap, flags, slack=1.5, max_creates=MAX_CREATES, large_clusters=True, huge_clusters=True, large_growth=True, huge_growth=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        donors = np.concatenate([workers(snap, c)[:8] for c in range(2000, 4000) if c not in big])
        a, b = 1000, 1500
        move(snap, donors[:500], a)
        move(snap, donors[500:500 + 8400], b)
        dr.commit_rows(donors[:8900])
        got, names = dr.check(oracle_mod, expect_incremental=True, profiled=True)
        assert "k_inc_grow" in names and "k_decide_huge" in names
        assert got.clusters["n_pods"][b] > abi.LARGE_MAX_PODS
    finally:
        dr.close()


def test_a_move_with_large_moves(oracle_mod):
    """KR_OPT_LARGE_MOVES: deleting a row swap-removes the last RayCluster, a huge one, into it; the moved RayCluster keeps its
    region and tiles and is decided again in the incremental pass, by k_decide_huge."""
    snap, flags = synthetic.generate(synthetic.config("C2", n_clusters=1400, pods_per_cluster=16, groups=2, seed=41))
    synthetic.grow_clusters(snap, [1399, 1300], 9000)
    dr = Driver(snap, flags, slack=1.25, max_creates=MAX_CREATES, large_clusters=True, huge_clusters=True, cluster_deletes=True,
                large_moves=True)
    try:
        dr.check(oracle_mod, expect_incremental=None)
        dr.check(oracle_mod, expect_incremental=None)
        dr.use(synthetic.delete_clusters(dr.snap, [12]))
        dr.commit_objects()
        dr.prev = None
        got, names = dr.check(oracle_mod, expect_incremental=True, profiled=True)
        assert "k_decide_huge" in names, names
        assert got.clusters["n_pods"][12] == 9000
        rows = members(dr.snap, 12)[::37]
        dr.snap.p_packed[rows] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        dr.commit_rows(rows)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


def test_seeded_stream_with_every_option(oracle_mod):
    rng = np.random.default_rng(12)
    snap, flags, big = _fleet("huge", n_big=2, n_clusters=3000)
    synthetic.grow_clusters(snap, [1500], 2500)
    opts = dict(large_clusters=True, huge_clusters=True, wide_clusters=True, large_growth=True, huge_growth=True, large_moves=True)
    dr = Driver(snap, flags, slack=1.3, max_creates=MAX_CREATES, **opts)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        n_inc = 0
        for epoch in range(10):
            rows = []
            for cl in big + [1500]:
                m = members(snap, cl)
                rows += rng.choice(m[1:], 40, replace=False).tolist()
            snap.p_packed[rows] ^= np.uint32(1 << abi.PP_READY_SHIFT)
            fail = rng.choice(rows, 3, replace=False)
            set_phase(snap, fail, abi.PHASE_FAILED if epoch % 2 else abi.PHASE_RUNNING)
            if epoch % 3 == 2:
                donors = np.concatenate([workers(snap, c)[:2] for c in rng.choice(np.arange(2000, 3000), 60, replace=False)])
                move(snap, donors, big[epoch % 2])
                rows += donors.tolist()
            dr.commit_rows(rows)
            got, _ = dr.check(oracle_mod)
            n_inc += got.changed_clusters is not None
        assert n_inc >= 6, n_inc
    finally:
        dr.close()

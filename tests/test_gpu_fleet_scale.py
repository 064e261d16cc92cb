"""The engine at the fleet sizes where kernel paths switch on that smaller snapshots never reach, against the CPU oracle and
hashlib: the radix sort's pass count, the fused and the chained-scan bucket starts and create fills, the orphan-tile scan past its
first chunk, a saturated workersToDelete Bloom bitmap and incremental epochs whose changed records outgrow the staging — most of
them at C3x10 (100 000 RayClusters x 100 Pods).  Then one long-lived engine, graphs on and off, walked up and down across those
thresholds and through same-size commits that change only the launch shape, every pass equal to a fresh oracle run.

Every threshold is mirrored in `Scale` (test_scale_mirrors_the_engine_constants, which needs no GPU, keeps the mirror honest); a
test that claims to cross one asserts that its sizes fall on the side it names, and that the profiled pass took that path."""
import os
import re

import numpy as np
import pytest

from harness import Driver, b32, compact, flip_ready, kernels, move, parity, room_caps, set_phase, spec_bytes
from kuberay_b200 import abi, synthetic
from kuberay_b200.engine import Engine
from kuberay_b200.snapshot import Snapshot

gpu = pytest.mark.gpu
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "kuberay_b200", "csrc")


class Scale:
    """The engine's fleet-size thresholds, mirrored from kuberay_b200/csrc:

    * kFusedMaxCounters (kr_emit.cuh:122): k_place_fused while n_clusters + 2 + mtiles fits, k_scan_counts + k_place above
      (launch_pass, kr_engine.cu:1065); k_creates_fused while n_groups + n_clusters + 1 fits, k_scan_actions / k_scan_creates /
      k_create_fill above (kr_engine.cu:1128, 1142);
    * kScanChunk (kr_bucket.cuh:17): counters per block of a chained scan; the orphan-tile scan of k_scan_counts spans more than
      one chunk past kScanChunk match tiles (kr_bucket.cuh:74-80);
    * kMatchTile = kSortThreads * kMatchItems (kr_common.cuh:152-156): Pods per match tile (mtiles, kr_engine.cu:449);
    * kRadixBits (kr_common.cuh:157): the radix sort sorts keys in [0, n_clusters] in ceil(bits / kRadixBits) passes
      (kr_engine.cu:1080-1082); the bucket pipeline's list builder (launch_lists) sorts the same keys with its own loop,
      `shift += kRadixBits` while `shift < bits` (list_passes);
    * KR_FAST_MAX_BUCKET (kr_bucket.cuh:12): the largest RayCluster the fast pipeline's in-warp sort takes; more sends the pass to
      the radix pipeline (and sets force_radix for the layout);
    * the workersToDelete Bloom bitmap: 64 bits per name, a power of two from 1024 bits, capped at 2^17 (scratch_layout,
      kr_engine.cu:475-478);
    * the incremental staging: packed records for capc = max(64, n_clusters / 4) RayClusters (inc_stage_layout, kr_engine.cu:54)."""

    fused_max = 48 * 1024
    scan_chunk = 8192
    match_tile = 256 * 2
    radix_bits = 8
    fast_max_bucket = 1024
    bloom_per_name = 64
    bloom_min = 1024
    bloom_cap = 1 << 17
    stage_min, stage_div = 64, 4

    @classmethod
    def mtiles(cls, n_pods):
        return max(1, -(-n_pods // cls.match_tile))

    @classmethod
    def fused_place(cls, n_clusters, n_pods):
        return n_clusters + 2 + cls.mtiles(n_pods) <= cls.fused_max

    @classmethod
    def fused_creates(cls, n_groups, n_clusters):
        return n_groups + n_clusters + 1 <= cls.fused_max

    @classmethod
    def radix_passes(cls, n_clusters):
        bits = 1
        while (1 << bits) <= n_clusters:
            bits += 1
        return -(-bits // cls.radix_bits)

    @classmethod
    def list_passes(cls, n_clusters):
        bits = 1
        while (1 << bits) <= n_clusters:
            bits += 1
        passes, shift = 0, 0
        while shift < bits:
            passes, shift = passes + 1, shift + cls.radix_bits
        return passes

    @classmethod
    def bloom_bits(cls, n_wtd):
        bits = cls.bloom_min
        while bits < cls.bloom_per_name * n_wtd and bits < cls.bloom_cap:
            bits <<= 1
        return bits

    @classmethod
    def capc(cls, n_clusters):
        return max(cls.stage_min, n_clusters // cls.stage_div)


def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _one(pattern, text):
    m = re.findall(pattern, text)
    assert len(m) == 1, (pattern, m)
    return m[0]


def test_scale_mirrors_the_engine_constants():
    """No GPU: the constants and rules Scale mirrors, read out of the kernel sources."""
    emit, bucket, common, engine = (_source(n) for n in ("kr_emit.cuh", "kr_bucket.cuh", "kr_common.cuh", "kr_engine.cu"))
    a, b = _one(r"constexpr uint32_t kFusedMaxCounters = (\d+) \* (\d+);", emit)
    assert int(a) * int(b) == Scale.fused_max
    assert int(_one(r"constexpr uint32_t kScanChunk = (\d+);", bucket)) == Scale.scan_chunk
    assert int(_one(r"#define KR_FAST_MAX_BUCKET (\d+)u", bucket)) == Scale.fast_max_bucket
    threads, items = int(_one(r"constexpr int kSortThreads = (\d+);", common)), int(_one(r"constexpr int kMatchItems = (\d+);", common))
    _one(r"constexpr int kMatchTile = kSortThreads \* kMatchItems;", common)
    assert threads * items == Scale.match_tile
    assert int(_one(r"constexpr int kRadixBits = (\d+);", common)) == Scale.radix_bits
    # the rules that use them
    _one(r"mtiles = \(uint32_t\)\(\(n\.n_pods \+ kMatchTile - 1\) / kMatchTile\)", engine)
    _one(r"fuse_place = !e->no_fuse && \(uint64_t\)n\.n_clusters \+ 2 \+ mtiles <= kFusedMaxCounters", engine)
    assert len(re.findall(r"\(uint64_t\)n\.n_groups \+ n\.n_clusters \+ 1 (?:<=|>) kFusedMaxCounters", engine)) == 2
    _one(r"while \(\(1ull << bits\) <= n\.n_clusters\) bits\+\+;", engine)
    _one(r"passes = \(int\)\(\(bits \+ kRadixBits - 1\) / kRadixBits\)", engine)
    _one(r"while \(\(1ull << bits\) <= Nc\) bits\+\+;  // keys are in \[0, n_clusters\]", engine)   # launch_lists
    _one(r"for \(uint32_t shift = 0; shift < bits; shift \+= kRadixBits\)", engine)
    assert int(_one(r"atoi\(g\) : (\d+)ull;", engine)) == Scale.bloom_per_name
    lo, cap = _one(r"uint64_t bits = (\d+);\s*while \(bits < per_name \* n\.n_wtd && bits < \(1ull << (\d+)\)\) bits <<= 1;", engine)
    assert int(lo) == Scale.bloom_min and 1 << int(cap) == Scale.bloom_cap
    lo, div = _one(r"L\.capc = std::max<uint32_t>\((\d+), n_clusters / (\d+)\);", engine)
    assert (int(lo), int(div)) == (Scale.stage_min, Scale.stage_div)
    _one(r"inc_stage_layout\(n\.n_clusters, n\.n_groups\)", engine)     # (the live count, not the capacity)
    # the rules themselves, at the boundaries the tests below use
    assert [Scale.radix_passes(n) for n in (255, 256, 65535, 65536)] == [1, 2, 2, 3]
    assert [Scale.list_passes(n) for n in (255, 256, 65535, 65536)] == [1, 2, 2, 3]
    assert Scale.fused_place(Scale.fused_max - 3, 1) and not Scale.fused_place(Scale.fused_max - 2, 1)
    assert Scale.fused_creates(Scale.fused_max - 1, 0) and not Scale.fused_creates(Scale.fused_max, 0)
    assert Scale.bloom_bits(16384) == Scale.bloom_cap and Scale.bloom_bits(30000) == Scale.bloom_cap and Scale.bloom_bits(100) == 8192


# ------------------------------------------------------------------------------------------------ helpers

def _copy(snap):
    d = snap.dims
    out = Snapshot(d["clusters"], d["groups"], d["wtd"], d["pods"], d["heads"], d["jobs"], d["json"])
    for name in out.cols:
        out.cols[name][:] = snap.cols[name]
    return out


def _owners(snap):
    """The RayCluster row of every pod row, -1 for orphans (their RayCluster is not in the snapshot)."""
    ckey = (snap.c_ns_id.astype(np.uint64) << np.uint64(32)) | snap.c_name_id.astype(np.uint64)
    order = np.argsort(ckey)
    pkey = (snap.p_ns_id.astype(np.uint64) << np.uint64(32)) | snap.p_cluster_name_id.astype(np.uint64)
    pos = np.minimum(np.searchsorted(ckey[order], pkey), order.size - 1)
    return np.where(ckey[order][pos] == pkey, order[pos], -1)


def _orphan_tiles(snap):
    """The match tiles that hold orphan pods."""
    live = (snap.p_packed & abi.PP_TOMBSTONE) == 0
    return np.unique(np.flatnonzero((_owners(snap) < 0) & live) // Scale.match_tile)


def _check_digests(snap, res):
    want = np.frombuffer(b"".join(b32(spec_bytes(snap, c)) for c in range(snap.dims["clusters"])), dtype=np.uint8).reshape(-1, 32)
    bad = np.flatnonzero((res.hash != want).any(axis=1))
    assert not bad.size, (bad.size, bad[:10].tolist())


class _Threaded:
    """The oracle module with its runs on 8 threads (Driver.check calls oracle.run(snap, flags))."""

    def __init__(self, oracle):
        self.oracle = oracle

    def run(self, snap, flags):
        return self.oracle.run(snap, flags, threads=8)


def _profiled(snap, flags, reports=None, **kw):
    """A fresh engine: a profiled pass, then a pass (graph) -> (results of the second, kernel names of the first).  `reports`, a
    list, receives both passes' kr_last_pass reports."""
    eng = Engine.for_snapshot(snap, **kw)
    try:
        eng.load(snap)
        names = [k for k, _ in eng.reconcile_profiled(flags)["kernels"]]
        if reports is not None:
            reports.append(eng.last_pass())
        got = eng.reconcile(flags)
        if reports is not None:
            reports.append(eng.last_pass())
        return got, names
    finally:
        eng.close()


def _fleet(n_clusters, pods_per_cluster=4, groups=1, seed=21, **kw):
    return synthetic.generate(synthetic.SynthParams(n_clusters=n_clusters, pods_per_cluster=pods_per_cluster, groups=groups, seed=seed, **kw))


# ------------------------------------------------------------------------------------------------ boundary parity, fresh engine

def _bucket_lists(snap, flags, oracle, **opts):
    """A fresh engine with KR_OPT_BUCKET_POD_LISTS fetching the lists: a profiled full pass, then an incremental one with nothing
    committed in between, both on the bucket pipeline and equal to the oracle with the lists fetched on both sides.
    -> (results of the second pass, kernel names of the first)."""
    f = abi.kr_flags.from_buffer_copy(flags)
    f.fetch_pod_lists = 1
    want = oracle.run(snap, f, threads=8)
    assert want.sorted_pod_idx.size == snap.dims["pods"]
    eng = Engine.for_snapshot(snap, bucket_pod_lists=True, **opts)
    try:
        eng.load(snap)
        names = [k for k, _ in eng.reconcile_profiled(f)["kernels"]]
        for kind in ("full", "incremental"):
            got = eng.fetch() if kind == "full" else eng.reconcile(f)
            rep = eng.last_pass()
            assert rep["pipeline"] == "bucket" and rep["kind"] == kind, rep
            d = want.diff(got)
            assert not d, (kind, d[:20])
            assert got.sorted_pod_idx.size == snap.dims["pods"]
    finally:
        eng.close()
    assert {"k_match2", "k_lists_owner", "k_lists_gather"} <= set(names), names
    return got, names


@gpu
@pytest.mark.parametrize("n_clusters", [255, 256, 65535, 65536])
@pytest.mark.parametrize("how", ["forced", "large_cluster", "bucket_lists", "bucket_lists_large"])
def test_radix_pass_count_at_its_boundaries(n_clusters, how, oracle_mod, monkeypatch):
    """Keys run over [0, n_clusters] (the orphan bucket is n_clusters), so 256 and 65 536 RayClusters need one more 8-bit pass
    than 255 and 65 535.  The radix pipeline is reached with KR_FORCE_RADIX=1, and by itself through one RayCluster of more than
    KR_FAST_MAX_BUCKET pods on the full-list path.  The bucket pipeline's list builder (KR_OPT_BUCKET_POD_LISTS) sorts the same keys
    with its own loop, whose first digit no other path histograms with k_hist; with KR_OPT_LARGE_CLUSTERS that large RayCluster
    stays on the bucket pipeline, and its Pods come from its region."""
    snap, flags = _fleet(n_clusters, pods_per_cluster=8 if n_clusters < 1000 else 4, orphan_frac=0.01)
    size = Scale.fast_max_bucket + 76
    if how == "forced":
        monkeypatch.setenv("KR_FORCE_RADIX", "1")
    elif how != "bucket_lists":
        synthetic.grow_clusters(snap, [0], size)
    if how.startswith("bucket_lists"):
        got, names = _bucket_lists(snap, flags, oracle_mod, **({"large_clusters": True} if how == "bucket_lists_large" else {}))
    else:
        got = parity(snap, flags, oracle_mod)
        names = kernels(snap, flags)
    assert got.n_orphans > 0
    assert how in ("forced", "bucket_lists") or got.clusters["n_pods"][0] == size > Scale.fast_max_bucket
    passes = Scale.list_passes(n_clusters) if how.startswith("bucket_lists") else Scale.radix_passes(n_clusters)
    assert names.count("k_scatter") == passes == {255: 1, 256: 2, 65535: 2, 65536: 3}[n_clusters], names
    assert "k_place_fused" not in names and "k_place" not in names


def _fused_place_edge(fused):
    """The most RayClusters (4 Pods, 1 % orphans) whose bucket starts fit k_place_fused, or one more."""
    pods = lambda nc: nc * 4 + int(nc * 4 * 0.01)  # noqa: E731  (synthetic.generate's pod count)
    nc = Scale.fused_max - 2 - Scale.mtiles(pods(Scale.fused_max))
    while not Scale.fused_place(nc, pods(nc)):
        nc -= 1
    while Scale.fused_place(nc + 1, pods(nc + 1)):
        nc += 1
    return nc if fused else nc + 1


@gpu
@pytest.mark.parametrize("fused", [True, False])
def test_bucket_starts_on_either_side_of_the_fused_limit(fused, oracle_mod):
    nc = _fused_place_edge(fused)
    snap, flags = _fleet(nc, orphan_frac=0.01)
    d = snap.dims
    counters = d["clusters"] + 2 + Scale.mtiles(d["pods"])
    assert (counters <= Scale.fused_max) == fused and abs(counters - Scale.fused_max) <= 2, counters
    assert not Scale.fused_creates(d["groups"], d["clusters"])    # (one group each: the create fill is past its limit already)
    got = parity(snap, flags, oracle_mod)
    assert got.n_orphans > 0
    names = kernels(snap, flags)
    if fused:
        assert "k_place_fused" in names and "k_scan_counts" not in names and "k_place" not in names, names
    else:
        assert "k_place_fused" not in names and {"k_scan_counts", "k_place"} <= set(names), names
    assert "k_scatter" not in names and {"k_scan_creates", "k_scan_actions", "k_create_fill"} <= set(names), names


@gpu
@pytest.mark.parametrize("fused", [True, False])
def test_create_fill_on_either_side_of_the_fused_limit(fused, oracle_mod):
    """Three worker groups per RayCluster: the groups push n_groups + n_clusters + 1 over the limit while the bucket starts
    (n_clusters + 2 + mtiles) stay fused."""
    nc = (Scale.fused_max - 1) // 4 + (0 if fused else 1)
    snap, flags = _fleet(nc, pods_per_cluster=7, groups=3)
    d = snap.dims
    assert d["groups"] == 3 * nc and Scale.fused_creates(d["groups"], d["clusters"]) == fused
    assert d["groups"] + d["clusters"] + 1 - Scale.fused_max in ((-3, 0) if fused else (1, 4))
    assert Scale.fused_place(d["clusters"], d["pods"])
    got = parity(snap, flags, oracle_mod)
    assert got.n_create_total > 0 and got.n_actions > 0
    names = kernels(snap, flags)
    assert "k_place_fused" in names
    unfused = {"k_scan_creates", "k_scan_actions", "k_create_fill"}
    if fused:
        assert "k_creates_fused" in names and not unfused & set(names), names
    else:
        assert "k_creates_fused" not in names and unfused <= set(names), names


# ------------------------------------------------------------------------------------------------ C3x10 on every pipeline

@pytest.fixture(scope="module")
def c3x10(oracle_mod):
    """synthetic.config("C3x10") and its oracle results (shared: the tests below only read them)."""
    snap, flags = synthetic.generate(synthetic.config("C3x10"))
    return snap, flags, oracle_mod.run(snap, flags, threads=8)


@gpu
@pytest.mark.parametrize("pipeline", ["bucket", "bucket_lists", "fast", "radix", "no_fuse"])
def test_c3x10_parity_on_every_pipeline(pipeline, c3x10, monkeypatch):
    """bucket_lists: KR_OPT_BUCKET_POD_LISTS builds the lists of 10 M Pods on the bucket pipeline, in three sort passes; the module's
    oracle results fetched the lists, so they are compared byte for byte."""
    snap, flags, want = c3x10
    d = snap.dims
    nc, mt = d["clusters"], Scale.mtiles(d["pods"])
    assert not Scale.fused_place(nc, d["pods"]) and not Scale.fused_creates(d["groups"], nc)
    tiles = _orphan_tiles(snap)
    assert mt > 2 * Scale.scan_chunk and tiles.size > 1000 and (tiles >= Scale.scan_chunk).sum() > 100 and (tiles >= 2 * Scale.scan_chunk).any()
    env = {"radix": "KR_FORCE_RADIX", "no_fuse": "KR_NO_FUSE"}.get(pipeline)
    if env:
        monkeypatch.setenv(env, "1")
    f = compact(flags) if pipeline == "bucket" else flags
    reports = []
    got, names = _profiled(snap, f, reports, bucket_pod_lists=pipeline == "bucket_lists")
    diff = want.diff(got)
    assert not diff, "\n".join(diff[:20])
    assert got.n_orphans == want.n_orphans > 0
    _check_digests(snap, got)
    if pipeline.startswith("bucket"):
        assert [(r["pipeline"], r["kind"]) for r in reports] == [("bucket", "full"), ("bucket", "incremental")], reports
    if pipeline == "bucket_lists":
        assert want.sorted_pod_idx.size == got.sorted_pod_idx.size == d["pods"]
        assert {"k_match2", "k_decide2", "k_lists_owner", "k_lists_gather"} <= set(names), names
        assert names.count("k_scatter") == Scale.list_passes(nc) == 3, names
    elif pipeline == "bucket":
        assert got.sorted_pod_idx.size == 0 and {"k_match2", "k_decide2"} <= set(names), names
    elif pipeline == "radix":
        assert names.count("k_scatter") == Scale.radix_passes(nc) == 3, names
    else:
        assert {"k_match", "k_scan_counts", "k_place", "k_scan_creates", "k_create_fill"} <= set(names) and "k_scatter" not in names, names


@gpu
def test_c3x10_with_a_saturated_wtd_bitmap(oracle_mod):
    """Every eligible group names workers to delete: about 30 000 names share a bitmap capped at 2^17 bits, so most pods pass
    the Bloom test and fall through to the table probe; named deletions happen all over the fleet."""
    snap, flags = synthetic.generate(synthetic.config("C3x10", wtd_group_frac=1.0))
    n_wtd = snap.dims["wtd"]
    assert n_wtd > Scale.bloom_cap // 8 and Scale.bloom_bits(n_wtd) == Scale.bloom_cap and Scale.bloom_bits(n_wtd) / n_wtd < 8
    got, lean = parity(snap, flags, oracle_mod, both=True)
    for res in (got, lean):
        assert (res.wtd_pod_idx >= 0).sum() > 10000
        assert (res.sorted_action == abi.ACT_DELETE_WTD).sum() > 1000 if res.sorted_action.size else True
    _check_digests(snap, lean)


# ------------------------------------------------------------------------------------------------ incremental epochs at C3x10

@gpu
def test_c3x10_incremental_epochs_packed_and_whole(c3x10, oracle_mod):
    _c3x10_epochs(c3x10, oracle_mod, lists=False)


@gpu
def test_c3x10_incremental_epochs_packed_and_whole_with_lists(c3x10, oracle_mod):
    _c3x10_epochs(c3x10, oracle_mod, lists=True)


def _c3x10_epochs(c3x10, oracle_mod, lists):
    """Bucket pipeline, compact results: a 0.1 % Pod churn epoch (changed records come back packed), an epoch in which one Pod
    moves from a late RayCluster to an early one, an epoch that dirties more RayClusters than the staging holds (the fetch copies
    the whole record arrays), all through commit_pod_values, then an object commit.  `lists`: KR_OPT_BUCKET_POD_LISTS fetching the
    lists every epoch; the Pod's move shifts the start of every RayCluster between the two while the epoch names only those two,
    so the fetch must patch starts into records it did not bring back."""
    snap, flags = _copy(c3x10[0]), abi.kr_flags.from_buffer_copy(c3x10[1])
    nc, n_pods = snap.dims["clusters"], snap.dims["pods"]
    records = nc * abi.cluster_result_dtype.itemsize           # the whole cluster-record array (the fetch's small part holds more)
    lists_b = 5 * n_pods + 4 * nc if lists else 0              # sorted_pod_idx + sorted_action, and pod_start, in every fetch
    rng = np.random.default_rng(5)
    owner = _owners(snap)
    worker = ((snap.p_packed >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER
    oracle = _Threaded(oracle_mod)
    dr = Driver(snap, flags, bucket_pod_lists=lists)
    dr.flags.fetch_pod_lists = int(lists)

    def epoch(kind):
        got, _ = dr.check(oracle, expect_incremental=kind == "incremental")
        rep = dr.eng.last_pass()
        assert rep["pipeline"] == "bucket" and rep["kind"] == kind, rep
        assert got.sorted_pod_idx.size == (n_pods if lists else 0)
        d2h = dr.eng.last_profile()["d2h_bytes"]
        assert d2h >= lists_b, (d2h, lists_b)
        return got, d2h - lists_b

    try:
        _, full = epoch("full")
        rows = rng.choice(n_pods, n_pods // 1000, replace=False)
        flip_ready(snap, rows[::2]); set_phase(snap, rows[1::2], abi.PHASE_FAILED)
        dr.commit_rows(rows)
        got, d2h = epoch("incremental")
        assert got.changed_clusters is not None and 0 < got.n_changed <= Scale.capc(nc), got.n_changed
        assert d2h < full - records // 2                                                 # packed
        # a worker of RayCluster nc - 10 moves to RayCluster 10
        before = got.clusters["pod_start"].copy()
        late, early = nc - 10, 10
        moved = np.flatnonzero(worker & (owner == late))[:1]
        move(snap, moved, early)
        owner[moved] = early
        dr.commit_rows(moved)
        got, d2h = epoch("incremental")
        assert sorted(got.changed_clusters.tolist()) == [early, late], got.changed_clusters
        assert d2h < full - records // 2                                                 # packed
        if lists:
            after = got.clusters["pod_start"]
            assert np.array_equal(after[:early + 1], before[:early + 1]) and np.array_equal(after[late + 1:], before[late + 1:])
            assert np.array_equal(after[early + 1:late + 1], before[early + 1:late + 1] + 1)
        # one worker of 40 % of the RayClusters
        cl, first = np.unique(owner[worker & (owner >= 0)], return_index=True)
        rows = np.flatnonzero(worker & (owner >= 0))[first[cl % 5 < 2]]
        flip_ready(snap, rows)
        dr.commit_rows(rows)
        got, d2h = epoch("incremental")
        assert got.changed_clusters is not None and got.n_changed > Scale.capc(nc), (got.n_changed, Scale.capc(nc))
        assert d2h > full - records // 2                                                 # whole arrays
        g = rng.choice(snap.dims["groups"], 2000, replace=False)
        snap.g_replicas[g] += 2
        dr.commit_objects()
        got, _ = epoch("incremental")
        assert got.changed_clusters is not None and np.isin(snap.g_cluster_idx[g], got.changed_clusters).all()
    finally:
        dr.close()


# ------------------------------------------------------------------------------------------------ one long-lived engine

def _recreate(snap, frac):
    out = _copy(snap)
    on = np.random.default_rng(3).random(out.dims["clusters"]) < frac
    out.c_flags[:] = (out.c_flags & ~np.uint32(abi.CF_UPGRADE_RECREATE)) | np.where(on, np.uint32(abi.CF_UPGRADE_RECREATE), np.uint32(0))
    return out


def _multihost(snap, c):
    """RayCluster c's worker group 0 turns into a multi-host group (numOfHosts = 4, its workers one replica)."""
    out = _copy(snap)
    g = int(out.c_group_off[c])
    out.g_num_hosts[g] = 4
    rows = np.flatnonzero(_owners(out) == c)
    rows = rows[((out.p_packed[rows] >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER]
    out.p_replica_name_id[rows] = np.uint32(0x7D000000)
    return out


def _grown(snap, size):
    out = _copy(snap)
    synthetic.grow_clusters(out, [0], size)
    return out


@pytest.fixture(scope="module")
def walk():
    """(label, snapshot, flags) steps: 1 k -> 30 k -> 70 k -> 20 k -> 1 k RayClusters of 4 Pods (all with orphans), a 70 k step with
    a RayCluster past the fast pipeline's bucket, and at 20 k same-size commits that change only the launch shape."""
    s1, f = _fleet(1000, seed=31)
    s30, _ = _fleet(30000, seed=32)
    s70, _ = _fleet(70000, seed=33)
    s20, _ = _fleet(20000, seed=34)
    big = Scale.fast_max_bucket + 100
    base = _recreate(s20, 0.0)
    steps = [("1k", s1), ("30k", s30), ("70k", s70), ("70k large", _grown(s70, big)), ("20k", base),
             ("20k recreate", _recreate(base, 0.3)), ("20k no recreate", base), ("20k multihost", _multihost(base, 7)),
             ("20k no multihost", base), ("20k large", _grown(base, big)), ("20k large gone", base), ("1k again", s1)]
    return [(label, s, f) for label, s in steps]


@gpu
@pytest.mark.parametrize("fixed_layout, bucket_pod_lists", [pytest.param(False, False, id="False"), pytest.param(True, False, id="True"),
                                                            pytest.param(False, True, id="False-lists"), pytest.param(True, True, id="True-lists")])
def test_one_engine_across_every_launch_shape(fixed_layout, bucket_pod_lists, walk, oracle_mod, monkeypatch):
    """One engine with capacities for the largest step (CUDA graph on) and its twin created with KR_NO_GRAPH=1, both loaded with
    every step in turn; each step's passes (full lists and compact results) equal the oracle and each other.  The first pass of a
    step keeps the previous step's flags, so it replays the previous graph unless something invalidated it.  With
    KR_OPT_BUCKET_POD_LISTS the passes that fetch the lists stay on the bucket pipeline wherever a step qualifies for it, and the
    graph of the same flags gains or loses a sort pass of the list builder as the walk crosses 65 536 RayClusters."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sizes = [s.dims for _, s, _ in walk]
    hash_tp = [(d["clusters"] + 31) // 32 > 4 * sms for d in sizes]
    assert not hash_tp[0] and hash_tp[1]                                                    # hash regime: latency -> throughput
    assert Scale.fused_place(sizes[1]["clusters"], sizes[1]["pods"]) and not Scale.fused_place(sizes[2]["clusters"], sizes[2]["pods"])
    assert Scale.fused_creates(sizes[0]["groups"], sizes[0]["clusters"]) and not Scale.fused_creates(sizes[1]["groups"], sizes[1]["clusters"])
    assert Scale.fused_creates(sizes[4]["groups"], sizes[4]["clusters"])                   # ... and back below at 20 k
    assert Scale.radix_passes(sizes[3]["clusters"]) == 3 and Scale.radix_passes(sizes[9]["clusters"]) == 2
    assert sizes[3] == sizes[2] and all(sizes[i] == sizes[4] for i in range(5, 11))
    rec = [int(((s.c_flags & abi.CF_UPGRADE_RECREATE) != 0).sum()) for _, s, _ in walk]
    assert rec[4] == 0 and rec[5] > 1000 and rec[6] == 0
    assert (walk[7][1].g_num_hosts > 1).sum() == 1 and (walk[8][1].g_num_hosts > 1).sum() == 0
    caps = room_caps(max((s for _, s, _ in walk), key=lambda s: s.dims["pods"]))
    engines = []
    try:
        engines.append(Engine(0, **caps))
        monkeypatch.setenv("KR_NO_GRAPH", "1")
        engines.append(Engine(0, **caps))
        monkeypatch.delenv("KR_NO_GRAPH")
        for eng in engines:
            if fixed_layout:
                eng.set_fixed_layout(True)
            eng.set_bucket_pod_lists(bucket_pod_lists)
        assert Scale.list_passes(sizes[2]["clusters"]) == 3 and Scale.list_passes(sizes[4]["clusters"]) == 2
        for k, (label, snap, flags) in enumerate(walk):
            want = oracle_mod.run(snap, flags, threads=8)
            runs = [flags, compact(flags)] if k % 2 == 0 else [compact(flags), flags]
            for eng in engines:
                eng.load(snap)
            for f in runs:
                graph, plain = (eng.reconcile(f) for eng in engines)
                for eng, res in zip(engines, (graph, plain)):
                    d = want.diff(res)
                    assert not d, (label, f.fetch_pod_lists, d[:10])
                    assert f.fetch_pod_lists or res.sorted_pod_idx.size == 0
                    if bucket_pod_lists and f.fetch_pod_lists and "large" not in label:  # (a step past the bucket may stay off it)
                        assert eng.last_pass()["pipeline"] == "bucket", (label, eng.last_pass())
                        assert res.sorted_pod_idx.size == snap.dims["pods"]
                assert not graph.diff(plain), label
            if "large" in label and "gone" not in label:
                assert want.clusters["n_pods"][0] > Scale.fast_max_bucket
    finally:
        for eng in engines:
            eng.close()


# ------------------------------------------------------------------------------------------------ KR_NO_PDL rung

@gpu
def test_parity_without_programmatic_dependent_launch(oracle_mod, monkeypatch):
    """KR_NO_PDL=1, the last rung of the fallback ladder: every kernel waits for its predecessor the ordinary way."""
    monkeypatch.setenv("KR_NO_PDL", "1")
    snap, flags = synthetic.generate(synthetic.config("C3"))
    got, lean = parity(snap, flags, oracle_mod, both=True)
    assert got.n_actions > 0 and got.n_create_total > 0 and lean.n_actions == got.n_actions

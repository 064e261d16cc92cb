"""Every pass at the launch grids of parts with fewer SMs than an H100 SXM.

The engine sizes the grids of its grid-stride and persistent kernels by the SM count (kr_engine.cu: launch_hash, k_clear,
k_place_fused, k_creates_fused, the incremental kernels, kr_hash_batch).  At 132 SMs the suite's fleets give almost every CTA of
them one trip, so a kernel that forgets per-warp state between items, builds a shared table once per CTA wrongly, or covers only
its first grid's worth of rows passes unseen.  KR_SM_COUNT=<n> (DESIGN §4.5) lays those grids out for n SMs on the whole device:
here at {1, 2, 3, 7, 16, 114 (an H100 PCIe), the device's count}, with fleets sized by `Shapes` so that each SM-sized kernel
takes at least 3 trips per CTA at one SM.  Every pass is compared with the CPU oracle and hashlib; incremental epochs must be
incremental exactly where they are at the device's own count.  KR_HASH_CTAS and KR_PLACE_CTAS move the same grids the other way.

Each of these kernel faults makes a test here fail at one SM: k_creates_fused filling only its first group per warp,
k_inc_aux_insert, k_inc_refresh or k_inc_groups_gather without its grid-stride loop, k_hash2 skipping its second trip,
k_place_fused stopping after its first trip, k_inc_wtd_resolve covering only its first gridDim.x * 256 Pod rows, and k_inc_grow
placing only the first gridDim.x * 256 spilled records.

COVERAGE names, for each kernel whose grid reads the SM count, the tests here that drive it through many trips;
tests/test_launch_shapes_src.py fails on CPU when a new SM-sized launch is missing from it.  On an H100 80GB HBM3 (700 W power
limit) the file's 81 tests took 46 s."""
import copy
import os

import numpy as np
import pytest

from harness import (PACKER_CAPS, Mirror, SpecDriver, b32, events, head_row, incremental, lists_of, objects, packer_stream, parity,
                     scale_to, with_wtd_lists, workers_of)
from kuberay_b200 import abi, synthetic
from kuberay_b200.engine import Engine
from kuberay_b200.packer import GroupPacker, Packer

pytestmark = pytest.mark.gpu

SM_COUNTS = (1, 2, 3, 7, 16, 114, None)  # None: the device's own count (KR_SM_COUNT unset)
ALL = dict(large_clusters=True, wide_clusters=True, huge_clusters=True, wtd_edits=True, spec_rows=True, cluster_creates=True,
           cluster_deletes=True, group_edits=True, large_growth=True, large_moves=True, huge_growth=True)

COVERAGE = {
    "k_hash3": ("test_hash_batch", "test_pass_digests"),
    "k_hash2": ("test_hash_batch", "test_pass_digests", "test_full_pass", "test_epochs_every_option"),
    "k_clear": ("test_full_pass",),
    "k_place_fused": ("test_full_pass", "test_ctas_per_sm"),
    "k_creates_fused": ("test_full_pass", "test_ctas_per_sm"),
    "k_inc_aux_clear": ("test_epochs_every_option",),
    "k_inc_aux_insert": ("test_epochs_every_option",),
    "k_inc_wtd_clear": ("test_epochs_every_option",),
    "k_inc_wtd_insert": ("test_epochs_every_option",),
    "k_inc_wtd_resolve": ("test_epochs_every_option", "test_structural_epochs"),
    "k_inc_orphan_adopt": ("test_structural_epochs",),
    "k_inc_clusters_rekey": ("test_structural_epochs",),
    "k_inc_groups_gather": ("test_structural_epochs",),
    "k_inc_admit": ("test_epochs_every_option", "test_structural_epochs"),
    "k_inc_grow": ("test_structural_epochs",),
    "k_inc_refresh": ("test_epochs_every_option",),
}


class Shapes:
    """The SM-sized grids, mirrored from kuberay_b200/csrc/kr_engine.cu (tests/test_launch_shapes_src.py reads them out of it):

    * launch_hash: k_hash3 (CTAs of one producer / consumer pair, one group of 32 messages per pair per round) while
      ceil(n / 32) <= 4 sm, on min(groups, 2 sm) CTAs; else k_hash2<4, 1> (128 messages per CTA per trip) on
      min(ceil(n / 128), sm * ctas) CTAs, ctas = KR_HASH_CTAS (2) in a pass and 4 in kr_hash_batch;
    * k_place_fused: sm * KR_PLACE_CTAS CTAs of 1024 threads, four Pods per thread per trip;
    * k_creates_fused: sm CTAs of 32 warps, one worker group per warp per trip;
    * the incremental kernels: min(sm * 2 (or * 4 for the two that read every pod row), rows / 256 + 1) CTAs of 256 threads, and
      k_inc_grow on sm CTAs of 256 threads."""

    hash3_groups_per_sm, hash3_ctas_per_sm, hash2_msgs = 4, 2, 128
    pass_hash_ctas, batch_hash_ctas = 2, 4
    place_threads, place_items = 1024, 4
    creates_warps = 32
    inc_threads = 256

    @classmethod
    def hash3(cls, sm, n):
        return -(-n // 32) <= cls.hash3_groups_per_sm * sm

    @classmethod
    def hash_trips(cls, sm, n, ctas=pass_hash_ctas):
        """Rounds of k_hash3 / trips of k_hash2 per CTA."""
        if cls.hash3(sm, n):
            groups = -(-n // 32)
            return -(-groups // min(groups, cls.hash3_ctas_per_sm * sm))
        blocks = -(-n // cls.hash2_msgs)
        return -(-blocks // min(blocks, sm * ctas))

    @classmethod
    def place_trips(cls, sm, n_pods, place_ctas=1):
        return -(-n_pods // (sm * place_ctas * cls.place_threads * cls.place_items))

    @classmethod
    def creates_trips(cls, sm, n_groups):
        return -(-n_groups // (sm * cls.creates_warps))

    @classmethod
    def inc_trips(cls, sm, rows, per_sm=2, grid_rows=None):
        """grid_rows: the row count the grid is capped by, when it is not the one the loop walks (k_inc_refresh)."""
        grid_rows = rows if grid_rows is None else grid_rows
        return -(-rows // (min(sm * per_sm, -(-grid_rows // cls.inc_threads) + 1) * cls.inc_threads))

    @classmethod
    def grow_trips(cls, sm, spilled):
        """k_inc_grow: sm CTAs of 256 threads over the spilled records (and one CTA per grown RayCluster over its old region)."""
        return -(-spilled // (sm * cls.inc_threads))


@pytest.fixture(scope="module")
def device_sms():
    eng = Engine(0, max_clusters=1)
    try:
        return eng.get_option(abi.OPT_SM_COUNT)
    finally:
        eng.close()


@pytest.fixture(params=SM_COUNTS, ids=lambda n: f"sm{n or 'dev'}")
def sm(request, monkeypatch, device_sms):
    """KR_SM_COUNT for the engines the test creates (each reads it at kr_engine_create).  -> the effective SM count."""
    n = request.param
    if n is None:
        monkeypatch.delenv("KR_SM_COUNT", raising=False)
        want = device_sms
    else:
        monkeypatch.setenv("KR_SM_COUNT", str(n))
        want = min(n, device_sms)
    eng = Engine(0, max_clusters=1)
    try:
        assert eng.get_option(abi.OPT_SM_COUNT) == want
        with pytest.raises(Exception):
            eng._check(eng._L.kr_engine_set_option(eng._h, abi.OPT_SM_COUNT, 1))
    finally:
        eng.close()
    return want


def test_switch_is_clamped_to_the_device(device_sms, monkeypatch):
    """At most the device's count; a value that is not a positive number is ignored (the device's count, as when unset)."""
    for value, want in (("0", device_sms), ("-3", device_sms), ("junk", device_sms), ("", device_sms), (str(device_sms + 100), device_sms),
                        ("1", 1), ("5", min(5, device_sms))):
        monkeypatch.setenv("KR_SM_COUNT", value)
        eng = Engine(0, max_clusters=1)
        try:
            assert eng.get_option(abi.OPT_SM_COUNT) == want, value
        finally:
            eng.close()


# ------------------------------------------------------------------------------------------------ full passes
def _fleet(n_clusters=600, ppc=16, seed=5, **kw):
    """n_clusters RayClusters of 3 worker groups: every other group asks for 3-9 more replicas (many creates per group, so each
    k_creates_fused warp fills several groups in turn), every fifth for 3 fewer with random delete on, a third of the groups name
    workersToDelete, a tenth of the RayClusters are Recreate-gated."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=n_clusters, pods_per_cluster=ppc, groups=3, seed=seed, healthy=True,
                                                           wtd_group_frac=0.3, recreate_frac=0.1, autoscaling_frac=0.3, **kw))
    snap.c_flags[:] &= ~np.uint32(abi.CF_SKIP | abi.CF_SUSPEND)
    for g in range(snap.dims["groups"]):
        if g % 2 == 0:
            scale_to(snap, g, int(snap.g_replicas[g]) + 3 + g % 7)
        elif g % 5 == 0:
            scale_to(snap, g, max(0, int(snap.g_replicas[g]) - 3))
    lists = lists_of(snap)
    for g in range(0, snap.dims["groups"], 3):
        lists[g] += [int(snap.p_name_id[p]) for p in workers_of(snap, g)[:1 + g % 2]]
    flags.env_random_pod_delete = 1
    return with_wtd_lists(snap, lists), flags


FULL = {"plain": ({}, {}), "radix": ({"KR_FORCE_RADIX": "1"}, {}), "no fuse": ({"KR_NO_FUSE": "1"}, {}), "no graph": ({"KR_NO_GRAPH": "1"}, {}),
        "classes": ({}, dict(ppc=40, n_large=3, large_pods=1500, n_wide=3, wide_groups=40))}


@pytest.mark.parametrize("variant", list(FULL))
def test_full_pass(variant, sm, oracle_mod, monkeypatch):
    """Parity on the bucket pipeline (compact results) and the sort pipeline (full pod lists), and down the fallback ladder; the
    'classes' fleet adds large, wide and huge RayClusters with their options on."""
    env, extra = FULL[variant]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    snap, flags = _fleet(**extra)
    opts = {}
    if variant == "classes":
        synthetic.grow_clusters(snap, [7], 9000)  # a huge one (more than LARGE_MAX_PODS)
        opts = dict(large_clusters=True, wide_clusters=True, huge_clusters=True)
    d = snap.dims
    assert Shapes.place_trips(1, d["pods"]) >= 3 and Shapes.hash_trips(1, d["clusters"]) >= 3
    got, lean = parity(snap, flags, oracle_mod, both=True, max_creates=1 << 20, **opts)
    creating = np.flatnonzero(got.groups["n_create"] > 0)
    assert creating.size > 100 and got.n_actions > 50, (creating.size, got.n_actions)
    # creates in the third trip of every warp at one SM, and several groups per warp at the smallest counts
    assert creating.max() >= 2 * Shapes.creates_warps and Shapes.creates_trips(1, d["groups"]) >= 3
    assert (got.groups["n_create"] >= 3).sum() > 50


@pytest.mark.parametrize("knob,value", [("KR_HASH_CTAS", "1"), ("KR_HASH_CTAS", "8"), ("KR_PLACE_CTAS", "2"), ("KR_PLACE_CTAS", "4")])
@pytest.mark.parametrize("fleet", ["sort", "hash"])
def test_ctas_per_sm(knob, value, fleet, oracle_mod, monkeypatch):
    """More CTAs per SM than the defaults (and one hash CTA per SM): a sort-pipeline fleet and a fleet in the hash's throughput
    regime, at the device's SM count."""
    monkeypatch.delenv("KR_SM_COUNT", raising=False)
    monkeypatch.setenv(knob, value)
    if fleet == "sort":
        snap, flags = _fleet()
    else:
        from test_gpu_regimes import _check_digests, _throughput_snapshot
        eng = Engine(0, max_clusters=1)
        sms = eng.get_option(abi.OPT_SM_COUNT)
        eng.close()
        snap, flags = _throughput_snapshot(128 * 2 * sms + 1500)
    got, lean = parity(snap, flags, oracle_mod, both=True, max_creates=1 << 20)
    if fleet == "hash":
        _check_digests(snap, got)
        _check_digests(snap, lean)


# ------------------------------------------------------------------------------------------------ hash
def test_hash_batch(sm):
    """kr_hash_batch against hashlib: every length at the SHA-1 block edges and a few KB, at message counts just below and above
    the k_hash3 / k_hash2 boundary, and (at the small counts) many k_hash2 trips."""
    from test_gpu_regimes import _hash_messages
    rng = np.random.default_rng(sm)
    edge = 4 * sm * 32
    sizes = [edge - 5, edge + 33] + ([4 * Shapes.batch_hash_ctas * sm * Shapes.hash2_msgs + 77] if sm <= 16 else [])
    assert Shapes.hash3(sm, sizes[0]) and not Shapes.hash3(sm, sizes[1])
    assert Shapes.hash_trips(sm, sizes[0], Shapes.batch_hash_ctas) == 2 or sizes[0] <= 2 * sm * 32
    if sm <= 16:
        assert Shapes.hash_trips(sm, sizes[2], Shapes.batch_hash_ctas) >= 5
    eng = Engine(0, max_clusters=1)
    try:
        for n in sizes:
            msgs = _hash_messages(n, rng)
            for i, ln in enumerate((0, 55, 56, 63, 64, 119, 120, 127, 128, 4096 + 57)):
                msgs[(i * 7919) % n] = rng.integers(0, 256, ln, dtype=np.uint8).tobytes()
            got = eng.hash_batch(msgs)
            bad = [i for i, (m, h) in enumerate(zip(msgs, got)) if b32(m).decode() != h]
            assert not bad, (n, len(bad), [len(msgs[i]) for i in bad[:10]])
    finally:
        eng.close()


@pytest.mark.parametrize("side", ["k_hash3", "k_hash2"])
def test_pass_digests(side, sm, oracle_mod):
    """The pass's digests against hashlib at a RayCluster count just below / above the boundary, 30 % of them Recreate-gated (their
    decide waits for the digest on the bucket pipeline).  Either outcome of the wait is correct; which one it was is printed."""
    from test_gpu_regimes import _check_digests, _throughput_snapshot
    n = 4 * sm * 32 - 3 if side == "k_hash3" else 4 * sm * 32 + 40
    assert Shapes.hash3(sm, n) == (side == "k_hash3")
    snap, flags = _throughput_snapshot(n, seed=100 + sm)
    eng = Engine.for_snapshot(snap)
    try:
        eng.load(snap)
        want = oracle_mod.run(snap, flags, threads=8)
        for fetch in (1, 0):
            flags.fetch_pod_lists = fetch
            got = eng.reconcile(flags)
            rep = eng.last_pass()
            _check_digests(snap, got)
            d = want.diff(got)
            assert not d, (fetch, d[:6])
            print(f"sm {sm} {side} n {n} fetch {fetch}: pipeline {rep['pipeline']}, hash_wait gave up: {rep['hash_wait']}")
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ incremental epochs
def _node_type(s, p, to):
    s.p_packed[p] = (s.p_packed[p] & ~np.uint32(3 << abi.PP_NODE_TYPE_SHIFT)) | np.uint32(to << abi.PP_NODE_TYPE_SHIFT)


def _epochs(dr, rng):
    """The edits of test_epochs_every_option, committed on SpecDriver dr one epoch per step; yields each epoch's label."""
    from test_gpu_field_epochs import with_heads
    s = dr.snap
    nc = s.dims["clusters"]
    # Pod status churn over more rows than k_inc_admit's grid covers in two trips at one SM
    rows = rng.choice(s.dims["pods"], 1600, replace=False)
    s.p_packed[rows] ^= np.uint32(1 << abi.PP_READY_SHIFT)
    dr.commit_rows(rows)
    yield "pod churn"
    # object-row edits: replicas of the first group of all but the first 50 RayClusters (k_inc_refresh's dirty list: three trips at one SM)
    for c in range(50, nc):
        g = int(s.c_group_off[c])
        scale_to(s, g, int(s.g_replicas[g]) + 1 + c % 3)
    dr.commit_objects()
    yield "object rows"
    # a head Pod stops being one (its head-aux row goes), then comes back
    c = int(rng.integers(nc // 2, nc))
    hr = head_row(s, c)
    p = int(s.h_pod_idx[hr])
    _node_type(s, p, abi.NT_WORKER)
    dr.use(with_heads(s, drop=[hr]))
    dr.commit_objects()
    dr.commit_rows([p])
    yield "head removed"
    s = dr.snap
    _node_type(s, p, abi.NT_HEAD)
    dr.use(with_heads(s, add=[p]))
    dr.commit_objects()
    dr.commit_rows([p])
    yield "head added"
    # workersToDelete edits: names renamed to other Pods of their RayCluster, one list one name longer and another one shorter
    s = dr.snap
    lists = lists_of(s)
    named = [g for g, lst in enumerate(lists) if lst]
    for g in named[::3]:
        c = int(s.g_cluster_idx[g])
        own = np.flatnonzero((s.p_ns_id == s.c_ns_id[c]) & (s.p_cluster_name_id == s.c_name_id[c]))
        lists[g][0] = int(s.p_name_id[own[int(rng.integers(own.size))]])
    lists[named[-1]].append(lists[named[-2]].pop())
    dr.set_wtd_lists(lists)
    yield "workersToDelete"
    # spec-row edits of more RayClusters than k_hash3 takes at one SM, Recreate-gated ones among them; a fifth move to the arena's end
    for c in rng.choice(nc, 700, replace=False):
        body = dr.body(int(c))
        dr.edit(int(c), body[:-1] + b" " if int(c) % 2 else body + b"  ", move=int(c) % 5 == 0)
    dr.commit_specs()
    yield "spec rows"


def test_epochs_every_option(sm, oracle_mod, monkeypatch):
    """Pod churn, object-row edits, a head Pod removed and added (k_inc_aux_*), workersToDelete edits (k_inc_wtd_*) and spec-row
    edits (k_inc_refresh, the hash over a row list), with every option on, each epoch checked by the Driver's rule and the oracle,
    equal to a twin engine at the device's SM count and incremental exactly where the twin's epoch is."""
    snap, flags = _fleet(n_clusters=1100, ppc=8, seed=17)
    assert Shapes.inc_trips(1, snap.dims["heads"]) >= 3 and Shapes.inc_trips(1, snap.dims["pods"], per_sm=4) >= 3
    assert Shapes.inc_trips(1, snap.dims["groups"]) >= 3 and Shapes.inc_trips(1, 1600) >= 3 and Shapes.hash_trips(1, 700) >= 3
    assert Shapes.inc_trips(1, 1050, grid_rows=snap.dims["clusters"]) >= 3  # k_inc_refresh: its grid follows n_clusters, its loop the dirty list
    knob = os.environ.get("KR_SM_COUNT")
    monkeypatch.delenv("KR_SM_COUNT", raising=False)
    twin = SpecDriver(copy.deepcopy(snap), abi.kr_flags.from_buffer_copy(flags), **ALL)
    if knob is not None:
        monkeypatch.setenv("KR_SM_COUNT", knob)
    dr = SpecDriver(snap, flags, **ALL)
    try:
        assert dr.eng.get_option(abi.OPT_SM_COUNT) == sm
        for d in (dr, twin):
            d.check(oracle_mod, expect_incremental=False)
        kinds = {}
        for label, _ in zip(_epochs(dr, np.random.default_rng(3)), _epochs(twin, np.random.default_rng(3))):
            got, _ = dr.check(oracle_mod, expect_incremental=None)
            want, _ = twin.check(oracle_mod, expect_incremental=None)
            kind, twin_kind = dr.eng.last_pass()["kind"], twin.eng.last_pass()["kind"]
            assert kind == twin_kind, (label, kind, twin_kind, dr.eng.last_pass()["why"])
            d = want.diff(got)
            assert not d, (label, d[:6])
            kinds[label] = kind
        print(f"sm {sm}: {kinds}")
        assert set(kinds.values()) == {"incremental"}, kinds  # (as every one is at the device's count)
    finally:
        dr.close()
        twin.close()


def test_structural_epochs(sm, oracle_mod, monkeypatch):
    """RayClusters created among waiting orphans (k_inc_orphan_adopt), deleted by swap-remove (k_inc_clusters_rekey,
    k_inc_groups_gather), regrouped, and grown past their bucket and their region by more records than k_inc_grow's grid holds in
    two trips, with every option on, on test_gpu_structural_streams' Fleet (whose model predicts each epoch and checks that every
    RayCluster the pass did not name keeps its records).  A twin Fleet at the device's SM count takes the same edits: each epoch
    must be incremental on both (last_pass), with equal results, and the profiled pass must have run the kernel it is for."""
    from test_gpu_structural_streams import Fleet, _universe
    uni, flags = _universe(1300, 1150, pods_per_cluster=8, seed=40 + sm)
    assert Shapes.inc_trips(1, 1150) >= 3 and Shapes.inc_trips(1, uni.dims["pods"], per_sm=4) >= 3
    assert Shapes.inc_trips(1, 2 * (1150 - 100)) >= 3 and Shapes.grow_trips(1, 800) >= 3  # (groups shifted, records spilled below)
    knob = os.environ.get("KR_SM_COUNT")
    monkeypatch.delenv("KR_SM_COUNT", raising=False)
    tw = Fleet(copy.deepcopy(uni), abi.kr_flags.from_buffer_copy(flags), list(range(1150)), oracle_mod, seed=sm)
    if knob is not None:
        monkeypatch.setenv("KR_SM_COUNT", knob)
    f = Fleet(uni, flags, list(range(1150)), oracle_mod, seed=sm)
    ran = []
    run = f.run

    def profiled_run(profiled, device_only):
        got, names = run(True, False)
        ran.append(set(names))
        return got, names
    f.run = profiled_run
    fleets = (f, tw)
    try:
        assert f.eng.get_option(abi.OPT_SM_COUNT) == sm
        donors = np.arange(0, 600)

        def epoch(kernels, label):
            (got, inc, cause), (want, tinc, tcause) = f.epoch(), tw.epoch()
            kinds = f.eng.last_pass()["kind"], tw.eng.last_pass()["kind"]
            assert inc and tinc and kinds == ("incremental", "incremental"), (label, kinds, cause, tcause)
            d = want.diff(got)
            assert not d, (label, d[:6])
            assert set(kernels) <= ran[-1], (label, set(kernels) - ran[-1])

        for x in fleets:
            x.flip(1600)
            x.create(1150)                       # its Pods were orphans
            x.create(1151)
        epoch({"k_inc_orphan_adopt", "k_inc_admit"}, "create")
        for x in fleets:
            x.delete(100)                         # a low row: the last RayCluster moves into it, the groups after it shift
            x.regroup(800, x.groups(800) + [(int(x.uni.c_group_off[800]), x.fresh_id())])
        epoch({"k_inc_clusters_rekey", "k_inc_groups_gather"}, "delete and regroup")
        for x in fleets:
            x.set_count(900, x.model.stride + 900, donors)   # 900 records past its bucket: a region
            x.set_count(901, x.model.stride + 90, donors)
        epoch({"k_inc_grow"}, "grow past the bucket")
        assert f.order.index(900) in f.model.caps and f.model.caps[f.order.index(900)] >= 900
        for x in fleets:
            x.set_count(900, x.model.stride + x.model.caps[x.order.index(900)] + 800, donors)  # 800 past its region
            x.flip(300)
        epoch({"k_inc_grow"}, "grow past the region")
        for x in fleets:
            x.delete(x.order[-1])
            x.create(1152)
            x.flip(200)
        epoch({"k_inc_orphan_adopt"}, "delete and create")
    finally:
        for x in fleets:
            x.close()


# ------------------------------------------------------------------------------------------------ the native packers
def test_native_packer_stream(oracle_mod, monkeypatch):
    """The native packer with every option on at two SMs and its twin at the device's count, on one informer stream: every epoch
    both equal the oracle and each other."""
    monkeypatch.delenv("KR_SM_COUNT", raising=False)
    caps = dict(PACKER_CAPS, max_clusters=256, max_groups=2048, max_wtd=1024, max_pods=16384, max_heads=1024, max_jobs=256, max_creates=1 << 20)
    dev = Packer(**caps, **ALL)
    monkeypatch.setenv("KR_SM_COUNT", "2")
    two = Packer(**caps, **ALL)
    try:
        assert two.engine.get_option(abi.OPT_SM_COUNT) == 2 and dev.engine.get_option(abi.OPT_SM_COUNT) > 2
        clusters, pods, jobs = objects(11, max_clusters=120)
        ms = [Mirror(copy.deepcopy(clusters), copy.deepcopy(pods), copy.deepcopy(jobs), pk) for pk in (two, dev)]
        counters = [[0], [0]]
        runs = []
        for i, m in enumerate(ms):
            def step(epoch, m=m, i=i):
                events(np.random.default_rng(500 + epoch), m, counters[i], structural=epoch % 3 == 2)
            runs.append(packer_stream(m, oracle_mod, 12, step, lean=lambda e: e % 4 != 3))
        for e, (a, b) in enumerate(zip(runs[0][0], runs[1][0])):
            d = b.diff(a)
            assert not d, (e, d[:6])
        assert runs[0][1] == runs[1][1]
    finally:
        two.close()
        dev.close()


def test_group_packer_three_shards(oracle_mod, monkeypatch):
    """Three shards on device 0 at three SMs, every option on, against a twin group packer at the device's count: each shard's pass
    equals the twin shard's and a full pass of its own engine."""
    monkeypatch.delenv("KR_SM_COUNT", raising=False)
    caps = dict(PACKER_CAPS, max_clusters=128, max_groups=1024, max_wtd=1024, max_pods=8192, max_jobs=256, max_creates=1 << 20)
    dev = GroupPacker([0, 0, 0], **caps, **ALL)
    monkeypatch.setenv("KR_SM_COUNT", "3")
    three = GroupPacker([0, 0, 0], **caps, **ALL)
    try:
        assert all(sh.engine.get_option(abi.OPT_SM_COUNT) == 3 for sh in three.shards)
        clusters, pods, jobs = objects(9)
        gps = (three, dev)
        for gp in gps:
            for c in clusters:
                gp.upsert_cluster(c)
            for p in pods:
                gp.upsert_pod(p)
            gp.flush()
        flags = three.flags(fetch_pod_lists=0)
        n_inc = 0
        for epoch in range(8):
            outs = []
            for gp in gps:
                rng = np.random.default_rng(epoch)
                for k in rng.choice(len(pods), 40, replace=False):
                    p = copy.deepcopy(pods[int(k)])
                    p["phase"] = ["Running", "Pending", "Failed"][int(rng.integers(3))]
                    p["conditions"] = [{"type": "Ready", "status": ["True", "False"][int(rng.integers(2))]}]
                    gp.upsert_pod(p)
                gp.flush()
                outs.append(gp.reconcile(flags))
            for i, (a, b) in enumerate(zip(*outs)):
                d = b.diff(a)
                assert not d, (epoch, i, d[:6])
                n_inc += incremental(a, a.clusters.shape[0])
            for sh, g, fl in zip(three.shards, outs[0], flags):
                sh.engine.set_incremental(False)
                full = sh.engine.reconcile(fl)
                sh.engine.set_incremental(True)
                d = full.diff(g)
                assert not d, (epoch, d[:6])
            three.reconcile(flags)  # (the first pass after incremental epochs come back is a full one)
            dev.reconcile(flags)
        assert n_inc >= 3 * 8 - 6, n_inc
    finally:
        three.close()
        dev.close()

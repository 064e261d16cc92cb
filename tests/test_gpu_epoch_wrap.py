"""Incremental epochs across the wrap of the engine's epoch counters, every pass checked against the oracle.

The device tells current state from stale state by a 32-bit stamp: the running epoch's is the epoch counter + 1, and 0 means "not
this epoch".  Before the counter comes within kEpochMargin (8) of 2^32 - 1 the engine zeroes the stamps, dirty flags and counters
again, as on a new layout, and runs a full pass that reports KR_FULL_EPOCH_WRAP.  KR_EPOCH_BASE seeds the counter (and the host's
row, spec and pull stamp counters) near the wrap, so each stream here crosses it within a few epochs.  Without that rule the
incremental epoch whose stamp is 0 takes every untouched Pod as retired and every RayCluster as having lost a row: `trajectory`
checks from the seed and the reported passes that each stream holds such an epoch after the wrap, so each stream would catch it.

On an H100 80GB HBM3 (700 W power limit) the file's nine tests took 5.4 s (8.7 s of wall time with the interpreter's start)."""
import copy

import numpy as np
import pytest

from harness import (OBJ_COLS, PACKER_CAPS, POD_COLS, Driver, Mirror, SpecDriver, autoscale_objects, device_incremental, flip_ready,
                     grown_fleet, members, move, objects, packer_check, run, spec_edits, workers)
from test_gpu_field_epochs import BIG_ROLES, MAX_CREATES, SMALL_ROLES, Fleet, copy_snap, partner
from test_gpu_structural_streams import ALL as STRUCTURAL_ALL, _packer_events
from kuberay_b200 import abi, synthetic
from kuberay_b200.engine import EngineError
from kuberay_b200.packer import GroupPacker, Packer

pytestmark = pytest.mark.gpu

U32 = 1 << 32
LIMIT = U32 - 1 - 8        # a counter past this before a pass is zeroed again (kEpochMargin in kr_engine.cu)
BASE = U32 - 12            # the wrap lands a few epochs into a stream
BIG_OPTIONS = dict(large_clusters=True, huge_clusters=True, wide_clusters=True, wtd_edits=True)
EVERY_OPTION = dict(STRUCTURAL_ALL, large_moves=True, huge_growth=True)


@pytest.fixture
def seeded(monkeypatch):
    """seeded(base): engines created from now on start their epoch counters at `base`."""
    def seed(base=BASE):
        monkeypatch.setenv("KR_EPOCH_BASE", str(base))
    return seed


def trajectory(reps, base):
    """From the seed and the passes' reports: (index of the pass that must zero the counters again, index of the incremental pass that
    without that rule would have stamped with 0).  A full pass closes attempts + 1 epochs (one more for a digest-wait rerun), an
    incremental one 1; the pass after the wrap runs as an incremental epoch would without the rule, when nothing else made it full."""
    fixed = unfixed = base
    wrap_at = zero_at = None
    for i, rep in enumerate(reps):
        if wrap_at is None and fixed > LIMIT:
            wrap_at, fixed = i, 0
        as_inc = rep["kind"] == "incremental" or (i == wrap_at and rep["why"] == ["EPOCH_WRAP"] and rep["attempts"] == 0)
        if zero_at is None and as_inc and (unfixed + 1) % U32 == 0:
            zero_at = i
        n = 1 if rep["kind"] == "incremental" else rep["attempts"] + 1 + int(rep["hash_wait"])
        fixed, unfixed = fixed + n, (unfixed + n) % U32
    return wrap_at, zero_at


def check_wrap(reps, base, full_ok=()):
    """Exactly one pass reports EPOCH_WRAP, the predicted one, and it is full; the epoch that would stamp 0 without the rule is in the
    stream and incremental; every other pass is incremental, except the first and those of `full_ok`.  -> the wrap's index."""
    wrap_at, zero_at = trajectory(reps, base)
    wraps = [i for i, r in enumerate(reps) if "EPOCH_WRAP" in r["why"]]
    assert wraps == [wrap_at], (wraps, wrap_at, reps)
    assert reps[wrap_at]["kind"] == "full", reps[wrap_at]
    assert zero_at is not None and zero_at > wrap_at and reps[zero_at]["kind"] == "incremental", (zero_at, wrap_at)
    for i, r in enumerate(reps[1:], 1):
        assert r["kind"] == "incremental" or i == wrap_at or i in full_ok, (i, r)
    return wrap_at


# ------------------------------------------------------------------------------------------------ every class through the wrap
class WrapFleet(Driver):
    """The fleet of test_gpu_field_epochs (one RayCluster of every class, large, huge and wide among them, each with an ordinary
    partner) on one engine with those classes' options on.  Every epoch edits every role through each stamp path."""

    def __init__(self, fleet):
        self.fleet, self.roles = fleet, SMALL_ROLES + BIG_ROLES
        super().__init__(copy_snap(fleet.snap), fleet.flags, slack=1.1, max_creates=MAX_CREATES, **BIG_OPTIONS)
        s = self.snap
        self.dp = {r: int(workers(s, r)[-1]) for r in self.roles}       # a worker deleted and added back by turns
        self.dp_vals = {r: {c: s.cols[c][self.dp[r]].copy() for c in POD_COLS} for r in self.roles}
        self.reps, self.want = [], None

    def edit(self, e):
        """Epoch e's edits of every role: Pod tp's readiness (a status update rewritten in place), Pod wp into the partner or back,
        Pod dp deleted or added back, and group 0's replicas (an object row commit)."""
        f, s = self.fleet, copy_snap(self.snap)
        for r in self.roles:
            flip_ready(s, [f.tp[r]])
            home = r if e % 2 else partner(r)
            s.p_ns_id[f.wp[r]], s.p_cluster_name_id[f.wp[r]] = s.c_ns_id[home], s.c_name_id[home]
            d = self.dp[r]
            for c in POD_COLS:
                s.cols[c][d] = self.dp_vals[r][c] if e % 2 else 0
            if not e % 2:
                s.p_packed[d] = abi.PP_TOMBSTONE
            s.g_replicas[int(s.c_group_off[r])] += 1 if e % 2 == 0 else -1
        rows = np.flatnonzero(np.logical_or.reduce([s.cols[c] != self.snap.cols[c] for c in POD_COLS]))
        self.snap = s
        for c in OBJ_COLS:
            np.copyto(self.views[c], s.cols[c])
        self.eng.commit_object_rows(list(self.roles), [])
        self.commit_rows(rows, journal=e % 2 == 0)

    def step(self, oracle):
        got, _ = self.check(oracle)
        self.reps.append(self.eng.last_pass())
        want = oracle.run(self.snap, self.flags)
        if self.want is not None:  # every role's record moved: each epoch's edits reach the results
            for r in self.roles:
                assert self.want.clusters[r].tobytes() != want.clusters[r].tobytes(), (len(self.reps), r)
        self.want = want
        return got


def test_every_class_through_the_wrap(seeded, oracle_mod):
    seeded()
    fleet = Fleet(True, oracle_mod)
    dr = WrapFleet(fleet)
    try:
        dr.step(oracle_mod)
        for e in range(14):
            dr.edit(e)
            dr.step(oracle_mod)
        check_wrap(dr.reps, BASE)
        # one more incremental epoch re-matches every Pod of the roles and their partners; it must equal a fresh engine's full
        # pass, so the bucket positions and other resident state no record shows have to be right too
        s = copy_snap(dr.snap)
        for r in dr.roles:
            for c in (r, partner(r)):
                s.p_packed[members(s, c)] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        rows = np.flatnonzero(np.logical_or.reduce([s.cols[c] != dr.snap.cols[c] for c in POD_COLS]))
        dr.snap = s
        dr.commit_rows(rows)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        fresh, _, _ = run(s, dr.flags, max_creates=MAX_CREATES, **BIG_OPTIONS)
        d = fresh.diff(got)
        assert not d, d[:6]
    finally:
        dr.close()


# ------------------------------------------------------------------------------------------------ where the wrap lands
def small_fleet(seed):
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=300, pods_per_cluster=20, groups=2, recreate_frac=0.0, seed=seed))
    flags.fetch_pod_lists = 0
    return snap, flags


def churn(dr, e):
    n = dr.snap.dims["pods"]
    rows = np.arange(5 + e, n, n // 6, dtype=np.int64)[:6]
    flip_ready(dr.snap, rows)
    dr.commit_rows(rows, journal=e % 2 == 0)


@pytest.mark.parametrize("case", ["first incremental epoch", "void first attempt", "flags change"])
def test_where_the_wrap_lands(case, seeded, oracle_mod):
    """The wrap on the first incremental epoch after the full pass; on a full pass whose first attempt voids (a RayCluster outgrew
    its bucket: the stride widens); on a pass already full for a flags change, which then reports both causes."""
    before = 3                             # epochs between the first pass and the one that wraps
    base = LIMIT if case == "first incremental epoch" else LIMIT - before
    if case == "first incremental epoch":
        before = 0
    seeded(base)
    dr = Driver(*small_fleet(6))
    reps = []
    try:
        for e in range(before + 10):
            if e == before + 1 and case == "void first attempt":
                rows = np.concatenate([workers(dr.snap, c) for c in (1, 2, 3, 4)])
                move(dr.snap, rows, 0)     # 20 + ~76 Pods in a 64-record bucket
                dr.commit_rows(rows)
            elif e == before + 1 and case == "flags change":
                dr.flags.gate_status_conditions ^= 1
            elif e:
                churn(dr, e)
            dr.check(oracle_mod)
            reps.append(dr.eng.last_pass())
        at = check_wrap(reps, base)
        assert at == before + 1, (at, reps)
        want = {"first incremental epoch": ["EPOCH_WRAP"], "void first attempt": ["EPOCH_WRAP"], "flags change": ["FLAGS", "EPOCH_WRAP"]}[case]
        assert reps[at]["why"] == want, reps[at]
        if case == "void first attempt":
            assert reps[at]["attempts"] >= 1 and reps[at]["stride"] == 128, reps[at]
    finally:
        dr.close()


def test_a_wrap_inside_the_first_full_pass(seeded, oracle_mod):
    """A seed one short of 2^32 - 1 under a first pass whose first attempt voids: the counter would pass 2^32 - 1 on its second attempt.
    The first pass zeroes instead, and the epochs after it are incremental."""
    seeded(U32 - 2)
    dr = Driver(*grown_fleet(100))
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rep = dr.eng.last_pass()
        assert rep["why"] == ["FIRST", "EPOCH_WRAP"] and rep["attempts"] >= 1, rep
        for e in range(1, 6):
            churn(dr, e)
            dr.check(oracle_mod, expect_incremental=True)
            assert dr.eng.last_pass()["why"] == []
    finally:
        dr.close()


# ------------------------------------------------------------------------------------------------ native and group packers
def test_native_packer_every_option_through_the_wrap(seeded, oracle_mod):
    """RayClusters created, deleted, regrouped and grown past their bucket, workersToDelete edits and spec edits (row by row), with
    every option on: k_inc_clusters_insert, k_inc_grow and the name-table and spec-row paths run on both sides of the wrap."""
    seeded()
    caps = dict(PACKER_CAPS, max_clusters=256, max_groups=2048, max_wtd=1024, max_pods=16384, max_jobs=256, max_creates=1 << 20)
    pk = Packer(**caps, **EVERY_OPTION)
    try:
        m = Mirror(*objects(5), pk)
        reps, tags = [], set()
        counter, deleted, gen, pending = [0], {}, [2], {}
        rng = np.random.default_rng(77)
        for epoch in range(16):
            if epoch:
                tags.add(_packer_events(m, rng, counter, deleted))
                autoscale_objects(rng, m, pending)
                spec_edits(rng, m, gen, 2)
            pk.flush()
            _, got = packer_check(m, oracle_mod, lean=True)
            rep = pk.last_pass()
            assert (rep["kind"] == "incremental") == device_incremental(got), (epoch, rep)
            reps.append(rep)
        wraps = [i for i, r in enumerate(reps) if "EPOCH_WRAP" in r["why"]]
        assert len(wraps) == 1 and reps[wraps[0]]["kind"] == "full", reps
        assert sum(r["kind"] == "incremental" for r in reps[wraps[0] + 1:]) >= 3, reps
        assert {"create", "delete", "regroup", "grow"} & tags, tags
    finally:
        pk.close()


def test_group_packer_through_the_wrap(seeded):
    """Two shards, each engine seeded: each shard's kr_last_pass reports the wrap once, and every pass equals a full pass of the same
    engine."""
    seeded()
    gp = GroupPacker([0, 0], **PACKER_CAPS)
    try:
        clusters, pods, jobs = objects(7, big=True)
        for c in clusters:
            gp.upsert_cluster(c)
        for p in pods:
            gp.upsert_pod(p)
        for j in jobs:
            gp.upsert_job(j)
        flags = gp.flags(fetch_pod_lists=0)
        live = [p for p in pods if (p.get("labels") or {}).get("ray.io/node-type") == "worker"]
        rng = np.random.default_rng(8)
        reps = [[], []]
        for epoch in range(14):
            for _ in range(4 if epoch else 0):
                p = copy.deepcopy(live[int(rng.integers(len(live)))])
                p["phase"] = ["Running", "Pending", "Failed"][int(rng.integers(3))]
                gp.upsert_pod(p)
            gp.flush()
            got = gp.reconcile(flags)
            for i, rep in enumerate(gp.last_passes()):
                reps[i].append(rep)
            if epoch in (6, 13):  # a full pass of each shard's own engine over the same state (the next pass is full: DISABLED)
                for sh, g, fl in zip(gp.shards, got, flags):
                    sh.engine.set_incremental(False)
                    d = sh.engine.reconcile(fl).diff(g)
                    sh.engine.set_incremental(True)
                    assert not d, (epoch, d[:6])
        for i in (0, 1):
            wraps = [k for k, r in enumerate(reps[i]) if "EPOCH_WRAP" in r["why"]]
            assert len(wraps) == 1 and reps[i][wraps[0]]["kind"] == "full", (i, reps[i])
    finally:
        gp.close()


# ------------------------------------------------------------------------------------------------ the host's stamp counters
def test_pod_values_across_the_row_epoch_wrap(seeded, oracle_mod):
    """kr_snapshot_commit_pod_values stamps each call's rows to refuse a row listed twice: the call on which that counter wraps still
    refuses one, and accepts a row the call before it listed."""
    seeded(U32 - 2)                        # the first call stamps with 2^32 - 1, the second wraps
    for twice in (False, True):
        dr = Driver(*small_fleet(11))
        try:
            dr.check(oracle_mod, expect_incremental=False)
            rows = workers(dr.snap, 7)[:3]
            flip_ready(dr.snap, rows)
            dr.commit_rows(rows)
            flip_ready(dr.snap, rows[:1])
            vals = lambda rs: np.stack([dr.snap.cols[c][rs].view(np.uint32) for c in POD_COLS], axis=1)  # noqa: E731
            if twice:
                with pytest.raises(EngineError):
                    dr.eng.commit_pod_values(rows[[0, 0]], vals(rows[[0, 0]]))
                continue
            dr.eng.commit_pod_values(rows[:1], vals(rows[:1]))
            dr.check(oracle_mod, expect_incremental=True)
        finally:
            dr.close()


def _mutate(b: bytes, salt: int) -> bytes:
    x = bytearray(b)
    x[len(x) // 2] = ord("a") + salt % 26
    return bytes(x)


def test_spec_rows_across_the_spec_and_pull_epoch_wraps(seeded, oracle_mod):
    """Spec rows listed over two calls, one row in both, epoch after epoch while the spec and pull stamp counters wrap: each row is
    pulled and hashed once per epoch (the commits' and the hash order's counted bytes), a row listed again after a pass is pulled
    again, and the digests equal the oracle's and a twin's that takes the whole arena."""
    seeded(U32 - 3)
    snap, flags = synthetic.generate(synthetic.config("C2", n_clusters=300, pods_per_cluster=16, groups=3, recreate_frac=0.2, seed=3))
    dr = SpecDriver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        for e in range(6):
            a, b = 10 + e % 2, 40 + 3 * e     # row a is listed in every epoch: after each pass it must be pulled again
            for c in (a, b):
                dr.edit(c, _mutate(dr.body(c), e))
            dr.apply()
            dr.commit_specs(rows=[a, b, a], calls=2)
            counted = sum(16 + (int(dr.snap.c_json_len[c]) + 15) // 16 * 16 for c in (a, b))
            dr.check(oracle_mod, expect_incremental=None, h2d=counted)
            if dr.eng.last_pass()["kind"] == "incremental":  # (the hash order of the two rows)
                assert dr.eng.last_profile()["h2d_bytes"] == counted + 4 * 2
    finally:
        dr.close()

"""The spec hash runs on its own stream beside the pass, and the bucket pipeline's Recreate gates wait for their digest inside
k_decide2 (the spin schedule).  The wait is bounded: a warp that gives up flags the pass (KR_TOTALS_HASH_WAIT) and the engine runs
it again on the two-phase schedule (k_decide2_phase1 after the hash).  Short specs hash in microseconds, so neither that rerun
nor a missing join between the two streams would show in any result.

Here some RayClusters carry specs of GIANT bytes.  One lane hashes a message serially and its warp stores the digests only when
it has finished, so a giant message holds back its own digest and those of the gates hashed beside it for about 30 times the
wait's budget: every pass on the spin schedule falls back, deterministically.  Each pass is checked against the CPU oracle, each
digest against hashlib, and each incremental epoch by the Driver's rule (records the pass did not name stay as they were).

Whether a pass fell back is read from kr_profile.n_kernels of the unprofiled pass: it counts k_decide2_phase1, which the spin
schedule does not launch, so it is one more than on a fresh engine over the same fleet with short specs."""
import functools
import time

import numpy as np
import pytest

from harness import Driver, SpecDriver, b32, compact, flip_ready, grown_fleet, head_row, members, spec_bytes, with_json
from kuberay_b200 import abi, synthetic
from kuberay_b200.engine import Engine

pytestmark = pytest.mark.gpu

GIANT = 16 << 20                 # bytes of a giant spec
WAIT_S = 40_000 * 100e-9         # k_decide2's digest wait: 40 000 x __nanosleep(100), about 4 ms nominal
N_GATES = 40                     # Recreate gates of a slow fleet: the giant one and the 31 hashed in its warp, and more


@functools.lru_cache(maxsize=None)
def giant(seed):
    """GIANT bytes of text, a different body for each seed."""
    body = np.random.default_rng(seed).integers(ord("a"), ord("z") + 1, GIANT, dtype=np.uint8)
    body[0], body[-1] = ord("{"), ord("}")
    return body.tobytes()


def readable(snap):
    """RayClusters whose Recreate gate reads the digest once gated: not skipped, not suspended, no external error."""
    ok = ((snap.c_flags & np.uint32(abi.CF_SKIP | abi.CF_SUSPEND)) == 0) & (snap.c_suspend_status == 0) & (snap.c_ext_err_kind == 0)
    return np.flatnonzero(ok)


def place(snap, specs):
    """A copy of `snap` whose RayClusters in `specs` (row -> bytes) take new ranges at the arena's end, in that order."""
    end = (snap.dims["json"] + 15) // 16 * 16
    out = with_json(snap, end + sum((len(b) + 15) // 16 * 16 for b in specs.values()))
    for c, b in specs.items():
        out.json[end:end + len(b)] = np.frombuffer(b, dtype=np.uint8)
        out.c_json_off[c], out.c_json_len[c] = end, len(b)
        end += (len(b) + 15) // 16 * 16
    return out


def gate(snap, rows):
    """Recreate gates on `rows` (head VER_CURRENT, ANNOT_HASH32): every other head carries its spec's digest, the rest a wrong one."""
    ah = snap.h_annot_hash.reshape(-1, 32)
    for i, c in enumerate(rows):
        h = head_row(snap, c)
        snap.c_flags[c] |= np.uint32(abi.CF_UPGRADE_RECREATE)
        snap.h_version_state[h], snap.h_annot_state[h] = abi.VER_CURRENT, abi.ANNOT_HASH32
        annotate(snap, c, spec_bytes(snap, c), i % 2 == 0)


def annotate(snap, c, body, match):
    """RayCluster c's head annotation: the digest of `body`, or (not `match`) a wrong one."""
    d = b32(body)
    snap.h_annot_hash.reshape(-1, 32)[head_row(snap, c)] = np.frombuffer(d if match else d[::-1], dtype=np.uint8)


def slow_fleet(base=None, seed=21, keep=()):
    """A fleet on the bucket pipeline (600 RayClusters of 20 Pods, 2 worker groups, or `base`) with N_GATES Recreate gates, the
    first of them on a giant spec at the arena's end, and a giant spec on a RayCluster without a gate just before it.  Rows in
    `keep` get neither.  -> (snapshot, compact flags, gated rows, the ungated giant's row)."""
    if base is None:
        base = synthetic.generate(synthetic.SynthParams(n_clusters=600, pods_per_cluster=20, groups=2, recreate_frac=0.0, seed=seed))
    snap, flags = base
    rows = readable(snap)
    rows = rows[~np.isin(rows, keep)]
    gates, plain = [int(c) for c in rows[1:1 + 2 * N_GATES:2]], int(rows[0])
    snap = place(snap, {plain: giant(1), gates[0]: giant(2)})
    gate(snap, gates)
    return snap, compact(flags), gates, plain


@pytest.fixture(scope="module")
def fleet():
    return slow_fleet()


def check_digests(snap, res):
    want = np.frombuffer(b"".join(b32(spec_bytes(snap, c)) for c in range(snap.dims["clusters"])), dtype=np.uint8).reshape(-1, 32)
    bad = np.flatnonzero((res.hash != want).any(axis=1))
    assert not bad.size, (bad.size, bad[:10].tolist(), [int(snap.c_json_len[c]) for c in bad[:10]])


def check(snap, flags, got, oracle):
    d = oracle.run(snap, flags, threads=8).diff(got)
    assert not d, d[:6]
    check_digests(snap, got)


def short(snap):
    """A copy of `snap` with every spec cut to at most 64 KB: the same kernels, and a hash done long before a gate reads it."""
    out = with_json(snap, snap.dims["json"])
    out.c_json_len[:] = np.minimum(out.c_json_len, 1 << 16)
    return out


def n_kernels(snap, flags, **kw):
    """kr_profile.n_kernels of the first, unprofiled pass of a fresh engine (Engine.for_snapshot keywords `kw`) over `snap`."""
    eng = Engine.for_snapshot(snap, max_creates=1 << 16, **kw)
    try:
        eng.load(snap)
        eng.reconcile(flags)
        return eng.last_profile()["n_kernels"]
    finally:
        eng.close()


def phase1_extra(eng, snap, flags, **kw):
    """Kernels eng's last unprofiled full pass over `snap` ran beyond a fresh engine's over its short-spec copy: 1 after a
    fallback (k_decide2_phase1), 0 on the spin schedule."""
    return eng.last_profile()["n_kernels"] - n_kernels(short(snap), flags, **kw)


def off_spin(eng, **kw):
    """Whether eng left the spin schedule: over a new layout of short gated specs it launches k_decide2_phase1, a fresh engine not."""
    probe, pflags = synthetic.generate(synthetic.SynthParams(n_clusters=200, pods_per_cluster=20, groups=1, recreate_frac=0.0, seed=5))
    gate(probe, readable(probe)[:20].tolist())
    pflags = compact(pflags)
    eng.load(probe)
    eng.reconcile(pflags)
    return eng.last_profile()["n_kernels"] == n_kernels(probe, pflags, **kw) + 1


def driver_extra(dr, **opts):
    """phase1_extra for a Driver's engine: the fresh engine is a Driver on the same capacities and options."""
    ref = Driver(short(dr.snap), abi.kr_flags.from_buffer_copy(dr.flags), json_room=dr.eng.cfg.max_json_bytes - dr.snap.dims["json"], **opts)
    try:
        ref.eng.reconcile(ref.flags)
        return dr.eng.last_profile()["n_kernels"] - ref.eng.last_profile()["n_kernels"]
    finally:
        ref.close()


def rewrite_tail(snap, c, salt):
    """Rewrite the last 64 bytes of RayCluster c's spec in place (new bytes, same length) -> the new spec."""
    off, ln = int(snap.c_json_off[c]), int(snap.c_json_len[c])
    tail = snap.json[off + ln - 64:off + ln]
    tail[:] = ord("A") + (np.arange(64) + salt) % 26
    return spec_bytes(snap, c)


def commit_json(dr):
    """The whole JSON arena and the object part, on a Driver (and its twin)."""
    for d in (dr, getattr(dr, "twin", None)):
        if d is not None:
            np.copyto(d.views["json"], d.snap.json)
            Driver.commit_objects(d, abi.PART_OBJECTS | abi.PART_JSON)


# ------------------------------------------------------------------------------------------------ the wait runs out

def test_giant_spec_outlasts_the_digest_wait():
    """One lane's serial SHA-1 over a giant spec takes at least 10 x the wait's budget.  The same bytes split over 256 messages
    (the same copies, hashed in parallel) are timed too, and only the difference is counted."""
    body = giant(1)
    split = [body[i:i + GIANT // 256] for i in range(0, GIANT, GIANT // 256)]
    eng = Engine(0, max_clusters=1)
    try:
        assert eng.hash_batch([body]) == [b32(body).decode()]          # (also sizes the staging buffers)
        t0 = time.perf_counter()
        eng.hash_batch([body])
        t1 = time.perf_counter()
        got = eng.hash_batch(split)
        t2 = time.perf_counter()
    finally:
        eng.close()
    assert got == [b32(m).decode() for m in split]
    assert (t1 - t0) - (t2 - t1) >= 10 * WAIT_S, (t1 - t0, t2 - t1)


def test_fallback_then_the_same_engine_onward(oracle_mod, monkeypatch):
    """A fresh engine's first full pass falls back; then on the same engine: a graph replay, a whole JSON commit that rewrites the
    giant spec's last bytes and a full pass, and incremental epochs (Pod churn on gated RayClusters; spec rows that turn a short
    gated spec giant and the giant one short, checked against a twin that commits the whole arena)."""
    snap, flags, gates, plain = slow_fleet(seed=22)
    dr = SpecDriver(snap, flags, json_room=GIANT + (1 << 20))
    try:
        got, _ = dr.check(oracle_mod, expect_incremental=False)
        check_digests(dr.snap, got)
        assert driver_extra(dr) == 1
        monkeypatch.setenv("KR_NO_HASH_SPIN", "1")                    # a twin on the two-phase schedule from the start
        spinless = Driver(dr.snap, abi.kr_flags.from_buffer_copy(dr.flags), json_room=GIANT + (1 << 20))
        monkeypatch.delenv("KR_NO_HASH_SPIN")
        try:
            assert not spinless.eng.reconcile(spinless.flags).diff(got)
            assert spinless.eng.last_profile()["n_kernels"] == dr.eng.last_profile()["n_kernels"]
        finally:
            spinless.close()
        # full passes on the same engine: the graph captured on the two-phase schedule, replayed; then a JSON commit first
        dr.eng.set_incremental(False)
        dr.twin.eng.set_incremental(False)
        got, _ = dr.check(oracle_mod, expect_incremental=False)
        assert driver_extra(dr) == 1
        body = rewrite_tail(dr.snap, gates[0], 3)
        annotate(dr.snap, gates[0], body, True)                        # still the true digest, of the new bytes
        annotate(dr.snap, gates[2], spec_bytes(dr.snap, gates[2]), False)
        commit_json(dr)
        got, _ = dr.check(oracle_mod, expect_incremental=False)
        check_digests(dr.snap, got)
        assert got.clusters["path"][gates[0]] == abi.PATH_NORMAL and got.clusters["path"][gates[2]] == abi.PATH_RECREATE_DELETE_ALL
        dr.eng.set_incremental(True)
        dr.twin.eng.set_incremental(True)
        dr.prev = None
        dr.check(oracle_mod, expect_incremental=False)
        # incremental epochs: Pod churn on gated RayClusters, then the two spec rows
        rows = np.concatenate([members(dr.snap, c)[:3] for c in gates[::4]])
        flip_ready(dr.snap, rows)
        dr.commit_rows(rows)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        check_digests(dr.snap, got)
        grow, shrink = gates[5], gates[0]
        dr.edit(grow, giant(3))
        dr.edit(shrink, b'{"rayVersion":"2.9.0"}')
        dr.apply()
        annotate(dr.snap, grow, giant(3), True)
        annotate(dr.snap, shrink, spec_bytes(dr.snap, shrink), False)
        dr.commit_specs()
        dr.commit_objects(twin=False)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        check_digests(dr.snap, got)
        assert got.clusters["path"][grow] == abi.PATH_NORMAL and got.clusters["path"][shrink] == abi.PATH_RECREATE_DELETE_ALL
    finally:
        dr.close()


# ------------------------------------------------------------------------------------------------ the ladder

def _two_big(seed=24):
    """1 200 RayClusters of 20 Pods (1 worker group), row 400 grown to 9 000 Pods and row 0 to 1 100."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=1200, pods_per_cluster=20, groups=1, recreate_frac=0.0, seed=seed))
    synthetic.grow_clusters(snap, [400], 9000)
    synthetic.grow_clusters(snap, [400, 0], 1100)                     # (row 400 neither grows nor gives)
    return snap, flags


@pytest.mark.parametrize("variant", ["ladder", "large", "huge", "gated_large_huge"])
def test_first_pass_walks_the_ladder_after_the_wait_runs_out(variant, oracle_mod):
    """One RayCluster of more than 1 024 Pods on a fresh engine: the first attempt voids, as the cluster outgrows the 64-Pod stride.
    k_match2 flags the void before k_decide2 starts, and then no warp of k_decide2 decides, so none waits for a digest.  Without
    options the pass walks every step (strides 64, 128, 256, the sort pipeline, the radix pipeline) without ever waiting, and the
    engine stays on the spin schedule.  With KR_OPT_LARGE_CLUSTERS (and KR_OPT_HUGE_CLUSTERS for a RayCluster of more than 8 192
    Pods) the void gives the cluster its region, the next attempt waits and runs out, and the rerun on the two-phase schedule
    stands.  With Recreate gates on a large and on a huge RayCluster, k_decide_large and k_decide_huge read their digests (the
    huge one's spec giant) after the join."""
    opts = {} if variant == "ladder" else dict(large_clusters=True, huge_clusters=True)
    keep = ()
    if variant in ("ladder", "large", "huge"):
        base = grown_fleet({"ladder": 1100, "large": 1100, "huge": 9000}[variant])
    else:
        snap0, flags0 = _two_big()
        base = (place(snap0, {400: giant(4)}), flags0)
        keep = (0, 400)
    snap, flags, gates, _ = slow_fleet(base, keep=keep)
    if keep:
        gate(snap, list(keep))
    eng = Engine.for_snapshot(snap, max_creates=1 << 16, **opts)
    try:
        eng.load(snap)
        got = eng.reconcile(flags)
        check(snap, flags, got, oracle_mod)
        if variant == "ladder":
            assert eng.get_option(abi.OPT_BUCKET_STRIDE) == 0
            assert not off_spin(eng, **opts)
        else:
            assert eng.get_option(abi.OPT_BUCKET_STRIDE) == 64
            assert phase1_extra(eng, snap, flags, **opts) == 1
            assert off_spin(eng, **opts)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ every schedule and pipeline

ENVS = {"default": {}, "no_spin": {"KR_NO_HASH_SPIN": "1"}, "no_pdl": {"KR_NO_PDL": "1"}, "no_graph": {"KR_NO_GRAPH": "1"},
        "no_fuse": {"KR_NO_FUSE": "1"}, "radix": {"KR_FORCE_RADIX": "1"}}


@pytest.mark.parametrize("fetch", [0, 1, 2])
@pytest.mark.parametrize("env", list(ENVS))
def test_every_schedule_and_pipeline(env, fetch, fleet, oracle_mod, monkeypatch):
    """Compact results take the bucket pipeline (the radix one under KR_FORCE_RADIX) and the full pod lists the sort pipeline;
    only the bucket pipeline's spin schedule waits, and falls back.  fetch = 2: the full pod lists on an engine with
    KR_OPT_BUCKET_POD_LISTS, which keeps the bucket pipeline and its spin schedule, so the fallback reruns the list builder behind
    k_decide2_phase1.  A second pass follows on the same engine."""
    for k, v in ENVS[env].items():
        monkeypatch.setenv(k, v)                                       # (kr_engine_create reads them)
    snap, flags, _, _ = fleet
    flags = abi.kr_flags.from_buffer_copy(flags)
    flags.fetch_pod_lists = min(fetch, 1)
    opts = dict(bucket_pod_lists=True) if fetch == 2 else {}
    bucket = fetch != 1 and env != "radix"
    eng = Engine.for_snapshot(snap, max_creates=1 << 16, **opts)
    try:
        eng.load(snap)
        for first in (True, False):
            got = eng.reconcile(flags)
            check(snap, flags, got, oracle_mod)
            rep = eng.last_pass()
            assert (rep["pipeline"] == "bucket") == bucket, rep
            assert got.sorted_pod_idx.size == (snap.dims["pods"] if fetch else 0)
            if first:
                spin = bucket and env != "no_spin"
                assert rep["kind"] == "full" and rep["hash_wait"] == spin, rep
                assert phase1_extra(eng, snap, flags, **opts) == (1 if spin else 0)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ every entry point

@pytest.mark.parametrize("entry", ["reconcile", "profiled", "device_only"])
def test_every_entry_point(entry, fleet, oracle_mod):
    """kr_reconcile_batch; kr_reconcile_batch_profiled (it hashes on the main stream once the JSON landed, and never waits) and
    kr_results_fetch, then an unprofiled pass; kr_reconcile_device_only and kr_results_fetch."""
    snap, flags, _, _ = fleet
    eng = Engine.for_snapshot(snap, max_creates=1 << 16)
    try:
        eng.load(snap)
        if entry == "profiled":
            names = [k for k, _ in eng.reconcile_profiled(flags)["kernels"]]
            assert "k_decide2_phase1" in names, names
            check(snap, flags, eng.fetch(), oracle_mod)
            eng.set_incremental(False)
            check(snap, flags, eng.reconcile(flags), oracle_mod)
        elif entry == "device_only":
            eng.reconcile_device_only(flags)
            check(snap, flags, eng.fetch(), oracle_mod)
        else:
            check(snap, flags, eng.reconcile(flags), oracle_mod)
        assert phase1_extra(eng, snap, flags) == 1
    finally:
        eng.close()


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("regime", ["latency", "throughput"])
def test_hash_batch_with_a_giant_message(regime):
    """kr_hash_batch: the giant among messages at the SHA-1 block edges and of a few KB (k_hash3), and among more than
    4 x SMs x 32 messages, where k_hash2<4, 1> takes it."""
    rng = np.random.default_rng(9)
    lens = [0, 1, 55, 56, 63, 64, 119, 120, 127, 128, 4095, 4096, 9000]
    if regime == "throughput":
        lens = lens + [i % 201 for i in range(4 * _sms() * 32 + 700)]
    blob = rng.integers(0, 256, 10_000, dtype=np.uint8).tobytes()
    msgs = [blob[i % 97:i % 97 + n] for i, n in enumerate(lens)]
    at = int(rng.integers(len(msgs)))
    msgs[at:at] = [giant(5)]
    eng = Engine(0, max_clusters=1)
    try:
        got = eng.hash_batch(msgs)
    finally:
        eng.close()
    bad = [i for i, (m, h) in enumerate(zip(msgs, got)) if b32(m).decode() != h]
    assert not bad, (len(bad), [len(msgs[i]) for i in bad[:10]])


def test_full_pass_in_the_throughput_regime(oracle_mod):
    """More than 4 x SMs x 32 RayClusters: the pass hashes with k_hash2<4, 1>, the giant gate's lane among them."""
    n = 4 * _sms() * 32 + 2000
    base = synthetic.generate(synthetic.SynthParams(n_clusters=n, pods_per_cluster=4, groups=1, recreate_frac=0.0, seed=26))
    snap, flags, _, _ = slow_fleet(base)
    eng = Engine.for_snapshot(snap, max_creates=1 << 16)
    try:
        eng.load(snap)
        check(snap, flags, eng.reconcile(flags), oracle_mod)
        assert phase1_extra(eng, snap, flags) == 1
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ the upload window

def _window_fleet(seed):
    """A slow fleet padded to a JSON arena of 64 MB and more, the last range a gated RayCluster's spec of a few KB.
    -> (snapshot, flags, that RayCluster's row)."""
    snap, flags, gates, _ = slow_fleet(seed=seed)
    last = gates[7]
    body = spec_bytes(snap, last)
    snap = with_json(snap, 64 << 20)
    snap = place(snap, {last: body})
    assert snap.dims["json"] >= 64 << 20 and int(snap.c_json_off[last]) + (len(body) + 15) // 16 * 16 == snap.dims["json"]
    return snap, flags, last


@pytest.mark.parametrize("how", ["whole", "spec_rows", "profiled"])
def test_spec_rewritten_at_the_arena_end(how, oracle_mod):
    """The spec at the end of the arena is rewritten in place (same length, new bytes, the head annotated with the new digest)
    and committed right before the pass: a hash that started before that range landed gives the old digest.  Through a whole
    commit (a full pass, then an incremental one), through kr_snapshot_commit_spec_rows, and before a profiled pass."""
    snap, flags, last = _window_fleet(23)
    json_room = 1 << 20 if how == "spec_rows" else 0
    dr = SpecDriver(snap, flags, json_room=json_room) if how == "spec_rows" else Driver(snap, flags, json_room=json_room)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        salt = 0

        def rewrite(match):
            nonlocal salt
            salt += 1
            body = rewrite_tail(dr.snap, last, salt)
            annotate(dr.snap, last, body, match)
            return body

        if how == "whole":
            dr.eng.set_incremental(False)
            rewrite(True)
            commit_json(dr)
            got, _ = dr.check(oracle_mod, expect_incremental=False)
            assert got.clusters["path"][last] == abi.PATH_NORMAL and driver_extra(dr) == 1
            dr.eng.set_incremental(True)
            dr.prev = None
            dr.check(oracle_mod, expect_incremental=False)
            rewrite(False)
            commit_json(dr)
            got, _ = dr.check(oracle_mod, expect_incremental=True)
            assert got.clusters["path"][last] == abi.PATH_RECREATE_DELETE_ALL
        elif how == "spec_rows":
            body = rewrite(True)
            dr.edit(last, body)
            dr.commit_specs()
            dr.commit_objects(twin=False)
            got, _ = dr.check(oracle_mod, expect_incremental=True)
            assert got.clusters["path"][last] == abi.PATH_NORMAL
        else:
            rewrite(True)
            commit_json(dr)
            got, _ = dr.check(oracle_mod, expect_incremental=True, profiled=True)
            assert got.clusters["path"][last] == abi.PATH_NORMAL
            dr.eng.set_incremental(False)
            rewrite(False)
            commit_json(dr)
            got, _ = dr.check(oracle_mod, expect_incremental=False, profiled=True)
            assert got.clusters["path"][last] == abi.PATH_RECREATE_DELETE_ALL
        check_digests(dr.snap, got)
    finally:
        dr.close()


# ------------------------------------------------------------------------------------------------ the incremental joins

def test_giant_spec_rows_on_every_class(oracle_mod):
    """Incremental epochs with KR_OPT_LARGE_CLUSTERS, KR_OPT_HUGE_CLUSTERS and KR_OPT_WIDE_CLUSTERS: giant spec rows re-hashed on a
    gated small, large (1 100 Pods), huge (9 000 Pods) and wide (48 worker groups) RayCluster; a whole JSON commit (the full
    re-hash and k_inc_mark_recreate); then an epoch without a JSON change, which keeps every resident digest."""
    snap, flags = _two_big(seed=27)
    snap = synthetic.widen_clusters(snap, [780], 48)                  # (rows 1.. gave their workers to rows 0 and 400)
    big = [0, 400, 780]
    snap, flags, gates, _ = slow_fleet((snap, flags), keep=big)
    gate(snap, big)
    opts = dict(large_clusters=True, huge_clusters=True, wide_clusters=True)
    dr = SpecDriver(snap, flags, json_room=4 * GIANT + (1 << 20), **opts)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        assert driver_extra(dr, **opts) == 1
        rows = [gates[3]] + big
        for i, c in enumerate(rows):
            dr.edit(c, giant(10 + i))
        dr.apply()
        for i, c in enumerate(rows):
            annotate(dr.snap, c, giant(10 + i), i % 2 == 1)
        dr.commit_specs()
        dr.commit_objects(twin=False)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        check_digests(dr.snap, got)
        body = rewrite_tail(dr.snap, big[1], 5)                       # the whole arena, with the huge RayCluster's giant rewritten
        annotate(dr.snap, big[1], body, True)
        commit_json(dr)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        check_digests(dr.snap, got)
        assert got.clusters["path"][big[1]] == abi.PATH_NORMAL
        pods = np.concatenate([members(dr.snap, c)[:4] for c in rows])
        flip_ready(dr.snap, pods)
        dr.commit_rows(pods)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        check_digests(dr.snap, got)
    finally:
        dr.close()


def test_renumbering_epoch_moves_a_digest_beside_a_giant_re_hash(oracle_mod):
    """KR_OPT_CLUSTER_DELETES: a RayCluster is deleted and swap-remove moves the last row, a gated one, into its place
    (k_inc_digest_move carries its digest), while another row's spec turns giant (re-hashed on the hash stream in the same
    epoch); then an epoch of Pod churn without a JSON change."""
    snap, flags, gates, plain = slow_fleet(seed=28)
    n = snap.dims["clusters"]
    last = n - 1
    if last not in gates:
        gate(snap, [last])
    victim = next(c for c in range(n) if c not in gates and c != plain)
    dr = SpecDriver(snap, flags, json_room=GIANT + (1 << 20), cluster_deletes=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        new = synthetic.delete_clusters(dr.snap, [victim])
        assert new.c_name_id[victim] == dr.snap.c_name_id[last]
        dr.use(new)
        edited = gates[9]
        dr.edit(edited, giant(6))
        dr.apply()
        annotate(dr.snap, edited, giant(6), True)
        dr.commit_specs()
        dr.commit_objects(twin=False)
        prev, dr.prev = dr.prev, None                                   # (rows moved: the records are compared below)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        check_digests(dr.snap, got)
        assert got.clusters["path"][edited] == abi.PATH_NORMAL
        assert bytes(got.hash[victim]) == bytes(prev.hash[last])
        named = set(got.changed_clusters.tolist()) if got.changed_clusters is not None else set()
        kept = [c for c in range(n - 1) if c != victim and c not in named]
        assert np.array_equal(got.clusters[kept], prev.clusters[kept]) and np.array_equal(got.hash[kept], prev.hash[kept])
        pods = np.concatenate([members(dr.snap, c)[:3] for c in (victim, edited, gates[1])])
        flip_ready(dr.snap, pods)
        dr.commit_rows(pods)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        check_digests(dr.snap, got)
    finally:
        dr.close()

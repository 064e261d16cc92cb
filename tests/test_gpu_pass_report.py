"""kr_last_pass on the H100: every pass reports its kind, pipeline, attempts, stride and digest-wait fallback, and a full pass the
KR_FULL_* rules (DESIGN §4.3) that kept it from being an incremental epoch.  Each cause is driven alone and must be the only bit,
with the results equal to the oracle; the options' "keeps the epoch" cases report an incremental pass with no cause; the full-pass
ladder reports its attempts and pipeline; and over random native-packer streams (options all on and all off, each epoch's pass also
run profiled on a twin, which must report the same) and on every shard of a group packer the reported kind agrees with what the results
show.

KR_FULL_ARENA's per-cluster sort scratch overrun (k_large_sort, k_huge_merge) cannot happen while the regions hold distinct live rows,
and the action-list cursor would need abandoned runs of a whole arena's worth of Pods; the create-arena cursor is the one driven
here (test_arena_create_cursor)."""
import copy

import numpy as np
import pytest

import test_gpu_cluster_creates as cc
import test_gpu_cluster_deletes as cd
import test_gpu_group_edits as ge
from harness import (PACKER_CAPS, Driver, Mirror, events, flip_ready, grown_fleet, incremental, lists_of, move, device_incremental, objects,
                     packer_check, scale_to, spec_edits, workers)
from test_gpu_large_growth import GROW, _fleet as growth_fleet
from test_gpu_wide_clusters import _wide_fleet
from kuberay_b200 import abi, synthetic
from kuberay_b200.engine import EngineError
from kuberay_b200.packer import GroupPacker, Packer
from kuberay_b200.snapshot import Snapshot

pytestmark = pytest.mark.gpu


def fleet(seed=3):
    """300 RayClusters of 20 Pods, two worker groups: the 64-record stride of the bucket pipeline.  -> (snapshot, compact flags)."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=300, pods_per_cluster=20, groups=2, recreate_frac=0.0, seed=seed))
    flags.fetch_pod_lists = 0
    return snap, flags


def churn(dr, k=6):
    """A few Pod status updates (Ready flips) committed as journal rows."""
    n = dr.snap.dims["pods"]
    rows = np.arange(5, n, n // k, dtype=np.int64)[:k]
    flip_ready(dr.snap, rows)
    dr.commit_rows(rows)


def expect(dr, kind, why=(), **fields):
    rep = dr.eng.last_pass()
    assert rep["kind"] == kind and rep["why"] == list(why), rep
    for k, v in fields.items():
        assert rep[k] == v, (k, rep)
    return rep


def first(dr, oracle):
    dr.check(oracle, expect_incremental=False)
    return expect(dr, "full", ["FIRST"], pipeline="bucket", attempts=0, hash_wait=False, stride=dr.eng.get_option(abi.OPT_BUCKET_STRIDE))


def test_first_pass_then_incremental_epochs_plain_and_profiled(oracle_mod):
    dr = Driver(*fleet())
    try:
        rep = first(dr, oracle_mod)
        assert rep["stride"] == 64
        for profiled in (False, True, False):
            churn(dr)
            dr.check(oracle_mod, expect_incremental=True, profiled=profiled)
            expect(dr, "incremental", [], why_full=0, pipeline="bucket", attempts=0, stride=64)
    finally:
        dr.close()


def test_no_report_before_a_pass():
    dr = Driver(*fleet())
    try:
        with pytest.raises(Exception):
            dr.eng.last_pass()
    finally:
        dr.close()


def drop_last_pod(snap):
    """A copy of `snap` without its last Pod row (a worker)."""
    d = snap.dims
    assert d["pods"] - 1 not in set(snap.h_pod_idx.tolist())
    out = Snapshot(d["clusters"], d["groups"], d["wtd"], d["pods"] - 1, d["heads"], d["jobs"], d["json"])
    for name, _dt, _m, dim in abi.COLUMNS:
        out.cols[name][:] = snap.cols[name][:-1] if dim == "pods" else snap.cols[name]
    return out


@pytest.mark.parametrize("cause", ["COLUMNS", "FLAGS", "DISABLED", "OPTION", "STRUCTURAL", "SIZES"])
def test_each_commit_or_setting_cause_alone(cause, oracle_mod):
    dr = Driver(*fleet(seed=4))
    try:
        first(dr, oracle_mod)
        churn(dr)
        if cause == "COLUMNS":
            dr.eng.commit()                                            # kr_snapshot_commit: every column wholesale
        elif cause == "FLAGS":
            dr.flags.gate_status_conditions ^= 1
        elif cause == "DISABLED":
            dr.eng.set_incremental(False)
        elif cause == "OPTION":
            dr.eng.set_large_clusters(True)
        elif cause == "STRUCTURAL":
            dr.snap.cols["g_name_id"][3] += np.uint32(100000)           # a renamed worker group: a table key
            dr.commit_objects()
        elif cause == "SIZES":
            dr.use(drop_last_pod(dr.snap))                             # fewer Pod rows under the fixed layout
            dr.commit_objects()
        dr.check(oracle_mod, expect_incremental=False)
        expect(dr, "full", [cause], pipeline="bucket")
        churn(dr)
        if cause == "DISABLED":  # every pass stays full, for the same reason, until the option comes back
            dr.check(oracle_mod, expect_incremental=False)
            expect(dr, "full", [cause])
            dr.eng.set_incremental(True)
            dr.check(oracle_mod, expect_incremental=False)
            expect(dr, "full", [cause])
            churn(dr)
        dr.check(oracle_mod, expect_incremental=True)
        expect(dr, "incremental", [])
    finally:
        dr.close()


def test_pod_lists_then_flags_back(oracle_mod):
    """fetch_pod_lists = 1: first a flags change, then (sort pipeline, nothing resident) POD_LISTS, also on the way back."""
    dr = Driver(*fleet(seed=5))
    try:
        first(dr, oracle_mod)
        dr.flags.fetch_pod_lists = 1
        dr.check(oracle_mod, expect_incremental=False)
        expect(dr, "full", ["FLAGS"], pipeline="sort", stride=0)
        churn(dr)
        dr.check(oracle_mod, expect_incremental=False)
        expect(dr, "full", ["POD_LISTS"], pipeline="sort")
        dr.flags.fetch_pod_lists = 0
        churn(dr)
        dr.check(oracle_mod, expect_incremental=False)
        expect(dr, "full", ["POD_LISTS"], pipeline="bucket")
        churn(dr)
        dr.check(oracle_mod, expect_incremental=True)
        expect(dr, "incremental", [])
    finally:
        dr.close()


# ------------------------------------------------------------------------------------------------ the full pass's ladder

def test_a_large_cluster_leaves_the_bucket_pipeline_and_reports_large_next(oracle_mod):
    dr = Driver(*grown_fleet(300))
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rep = expect(dr, "full", ["FIRST"], pipeline="sort", stride=0)
        assert rep["attempts"] >= 1
        churn(dr)
        dr.check(oracle_mod, expect_incremental=False)
        expect(dr, "full", ["LARGE"], pipeline="sort", attempts=0)
    finally:
        dr.close()
    dr = Driver(*grown_fleet(300), large_clusters=True)                # the option keeps it on the bucket pipeline
    try:
        dr.check(oracle_mod, expect_incremental=False)
        expect(dr, "full", ["FIRST"], pipeline="bucket")
        churn(dr)
        dr.check(oracle_mod, expect_incremental=True)
        expect(dr, "incremental", [])
    finally:
        dr.close()


def test_a_widened_stride_counts_its_attempts(oracle_mod):
    dr = Driver(*grown_fleet(100))
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rep = expect(dr, "full", ["FIRST"], pipeline="bucket")
        assert rep["attempts"] >= 1 and rep["stride"] == dr.eng.get_option(abi.OPT_BUCKET_STRIDE) == 128, rep
        churn(dr)
        dr.check(oracle_mod, expect_incremental=True)
        expect(dr, "incremental", [], stride=128)
    finally:
        dr.close()


@pytest.mark.parametrize("growth", [False, True])
def test_a_cluster_outgrowing_its_bucket(growth, oracle_mod):
    """Without a growth option the incremental attempt voids on the device (OVERFLOW) and the full pass widens the stride; with
    KR_OPT_LARGE_GROWTH the epoch stays incremental."""
    opts = dict(large_clusters=True, large_growth=True) if growth else {}
    dr = Driver(*fleet(seed=6), **opts)
    try:
        first(dr, oracle_mod)
        rows = np.concatenate([workers(dr.snap, c) for c in (1, 2, 3, 4)])
        move(dr.snap, rows, 0)                                         # 20 + ~76 Pods in a 64-record bucket
        dr.commit_rows(rows)
        dr.check(oracle_mod, expect_incremental=growth)
        if growth:
            expect(dr, "incremental", [])
        else:
            rep = expect(dr, "full", ["OVERFLOW"], pipeline="bucket")
            assert rep["attempts"] >= 1 and rep["stride"] == 128, rep
    finally:
        dr.close()


def test_the_digest_wait_fallback_is_reported(oracle_mod):
    from test_gpu_hash_wait import GIANT, slow_fleet
    snap, flags, _gates, _plain = slow_fleet(seed=24)
    dr = Driver(snap, flags, json_room=GIANT + (1 << 20))
    try:
        dr.check(oracle_mod, expect_incremental=False)
        expect(dr, "full", ["FIRST"], pipeline="bucket", hash_wait=True)
    finally:
        dr.close()


# ------------------------------------------------------------------------------------------------ streams and shards

ALL = dict(large_clusters=True, wide_clusters=True, huge_clusters=True, wtd_edits=True, spec_rows=True, cluster_creates=True,
           cluster_deletes=True, group_edits=True, large_growth=True, large_moves=True, huge_growth=True)


@pytest.mark.parametrize("seed", [31, 32])
@pytest.mark.parametrize("all_options", [False, True])
def test_reports_agree_with_the_results_over_packer_streams(seed, all_options, oracle_mod):
    """Two packers take the same events; the twin runs every epoch's pass profiled and must report what the plain pass reports."""
    clusters, pods, jobs = objects(seed, big=True)
    opts = ALL if all_options else {}
    pk, twin = Packer(**dict(PACKER_CAPS, max_pods=8192), **opts), Packer(**dict(PACKER_CAPS, max_pods=8192), **opts)
    kinds = []
    try:
        sides = [(Mirror(copy.deepcopy(clusters), copy.deepcopy(pods), jobs, p), np.random.default_rng(seed), [0], [2]) for p in (pk, twin)]
        profiled = lambda f: (twin.engine.reconcile_profiled(f), twin.engine.fetch())[1]  # noqa: E731
        for epoch in range(15):
            reps = []
            for (m, rng, counter, gen), run in zip(sides, (None, profiled)):
                if epoch:
                    if all_options:
                        spec_edits(rng, m, gen, int(rng.integers(1, 3)))
                    events(rng, m, counter, structural=True)
                m.pk.flush()
                _, got = packer_check(m, oracle_mod, lean=True, run=run)
                rep = m.pk.last_pass()
                assert (rep["kind"] == "incremental") == device_incremental(got), (epoch, rep, got.n_changed)
                assert (rep["why_full"] != 0) == (rep["kind"] == "full"), (epoch, rep)
                reps.append(rep)
            plain, prof = reps
            assert (prof["kind"], prof["why"], prof["pipeline"], prof["stride"]) == (plain["kind"], plain["why"], plain["pipeline"], plain["stride"]), (epoch, plain, prof)
            if epoch == 0:
                assert plain["why"] == ["FIRST"]
            kinds.append(plain["kind"])
    finally:
        pk.close()
        twin.close()
    assert "incremental" in kinds, kinds


def test_every_shard_of_a_group_packer_reports_its_own():
    clusters, pods, jobs = objects(7, big=True)
    gp = GroupPacker([0, 0], **PACKER_CAPS)
    try:
        for c in clusters:
            gp.upsert_cluster(c)
        for p in pods:
            gp.upsert_pod(p)
        for j in jobs:
            gp.upsert_job(j)
        gp.flush()
        gp.reconcile(gp.flags(fetch_pod_lists=0))
        assert [r["why"] for r in gp.last_passes()] == [["FIRST"], ["FIRST"]]
        live = [p for p in pods if (p.get("labels") or {}).get("ray.io/node-type") == "worker"]
        rng = np.random.default_rng(7)
        for epoch in range(4):
            touched = []
            for _ in range(3):
                p = copy.deepcopy(live[int(rng.integers(len(live)))])
                p["phase"] = ["Running", "Pending", "Failed"][int(rng.integers(3))]
                gp.upsert_pod(p)
                touched.append(p)
            gp.flush()
            res = gp.reconcile(gp.flags(fetch_pod_lists=0))
            reps = gp.last_passes()
            for i, (rep, x) in enumerate(zip(reps, res)):
                assert (rep["kind"] == "incremental") == device_incremental(x), (epoch, i, rep)
                assert rep["kind"] == "incremental" and rep["why_full"] == 0, (epoch, i, rep)
        # a flags change on one shard only: that shard alone reports it
        flags = gp.flags(fetch_pod_lists=0)
        flags[1].gate_status_conditions ^= 1
        gp.reconcile(flags)
        assert [(r["kind"], r["why"]) for r in gp.last_passes()] == [("incremental", []), ("full", ["FLAGS"])]
    finally:
        gp.close()


# ------------------------------------------------------------------------------------------------ the rest of the causes alone

def test_capacity_overrun_then_the_next_pass(oracle_mod):
    """A full pass whose creates overrun max_creates fails (KR_E_CAPACITY); the pass after it (every RayCluster skipped now, so nothing
    to create) reports why nothing was resident."""
    snap, flags = fleet(seed=10)
    dr = Driver(snap, flags, max_creates=1)
    try:
        with pytest.raises(EngineError):
            dr.eng.reconcile(dr.flags)
        dr.snap.c_flags[:] |= np.uint32(abi.CF_SKIP)
        dr.commit_objects()
        dr.check(oracle_mod, expect_incremental=False)
        expect(dr, "full", ["CAPACITY"], pipeline="bucket")
        churn(dr)
        dr.check(oracle_mod, expect_incremental=True)
        expect(dr, "incremental", [])
    finally:
        dr.close()


def test_arena_create_cursor(oracle_mod):
    """The create arena is sized to the first pass's creates plus 8.  One group asks for 20 more Pods while others stop creating:
    the full pass would fit, but the incremental decide cannot reuse the abandoned places and its cursor runs past the end."""
    snap, flags = fleet(seed=11)
    probe = Driver(copy.deepcopy(snap), abi.kr_flags.from_buffer_copy(flags), max_creates=1 << 16)
    try:
        got, _ = probe.check(oracle_mod, expect_incremental=False)
        extent = int(got.create_idx.size)  # (the pass's create extent)
        g_create, g_running = got.groups["n_create"].astype(np.int64), got.groups["n_running"].astype(np.int64)
    finally:
        probe.close()
    creating = [g for g in np.flatnonzero(g_create > 0).tolist() if snap.g_num_hosts[g] <= 1]
    up = creating[0]
    down, freed = [], 0
    for g in creating[1:]:
        if snap.g_cluster_idx[g] != snap.g_cluster_idx[up] and freed < 40:
            down.append(g)
            freed += int(g_create[g])
    assert freed >= 40, freed
    dr = Driver(snap, flags, max_creates=extent + 8)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        scale_to(dr.snap, up, int(g_running[up] + g_create[up] + 20))
        for g in down:
            scale_to(dr.snap, g, int(g_running[g]))
        dr.commit_objects()
        dr.check(oracle_mod, expect_incremental=False)
        expect(dr, "full", ["ARENA"], pipeline="bucket")
    finally:
        dr.close()


@pytest.mark.parametrize("on", [False, True])
def test_wide_cluster(on, oracle_mod):
    dr = Driver(*_wide_fleet(48), wide_clusters=on)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        expect(dr, "full", ["FIRST"], pipeline="bucket" if on else "sort")
        churn(dr)
        dr.check(oracle_mod, expect_incremental=on)
        if on:
            expect(dr, "incremental", [])
        else:
            expect(dr, "full", ["WIDE"], pipeline="sort")
    finally:
        dr.close()


@pytest.mark.parametrize("huge", [False, True])
def test_growth_past_the_largest_cluster(huge, oracle_mod):
    """KR_OPT_LARGE_GROWTH without KR_OPT_HUGE_GROWTH refuses a RayCluster that grows past KR_LARGE_MAX_PODS (GROW_LIMIT, relabelled by
    the host from k_inc_admit's store or set by k_inc_grow); with the huge options the epoch stays incremental."""
    snap, flags = growth_fleet(9, n_clusters=700)
    extra = dict(huge_clusters=True, huge_growth=True) if huge else {}
    dr = Driver(snap, flags, max_creates=1 << 16, **GROW, **extra)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rows = next(synthetic.grow_epochs(snap, [600], [abi.LARGE_MAX_PODS + 1]))
        dr.commit_rows(rows)
        dr.check(oracle_mod, expect_incremental=huge)
        if huge:
            expect(dr, "incremental", [])
        else:
            expect(dr, "full", ["GROW_LIMIT"])
    finally:
        dr.close()


def _off_driver(snap, flags, room=None):
    """A Driver with no option on, on `snap` (capacities from `room`), before its first pass."""
    dr = Driver(room if room is not None else snap, flags, slack=1.25)
    if room is not None:
        dr.use(snap)
        dr.commit_objects(abi.PART_ALL)
        for c in ("p_ns_id", "p_cluster_name_id", "p_group_name_id", "p_name_id", "p_packed", "p_replica_index", "p_replica_name_id"):
            dr.views[c][:] = snap.cols[c]
        dr.eng.commit(abi.PART_ALL)
    return dr


@pytest.mark.parametrize("on", [False, True])
def test_creation(on, oracle_mod):
    full, flags = cc._fleet(204, seed=61)
    before = cc._prefix(full, 203)
    dr = cc._driver(before, flags, full) if on else _off_driver(before, flags, room=full)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        expect(dr, "full", ["FIRST"])
        cc._create(dr, full)
        cc._check(dr, oracle_mod, expect_incremental=on)
        expect(dr, *(("incremental", []) if on else ("full", ["SIZES"])))
    finally:
        dr.close()


@pytest.mark.parametrize("on", [False, True])
def test_deletion(on, oracle_mod):
    snap, flags = cd._fleet(300, seed=3, wtd_group_frac=0.0)
    dr = cd._driver(snap, flags) if on else _off_driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        cd._epoch(dr, synthetic.delete_clusters(snap, [137]))
        dr.prev = None
        dr.check(oracle_mod, expect_incremental=on)
        expect(dr, *(("incremental", []) if on else ("full", ["SIZES"])))
    finally:
        dr.close()


@pytest.mark.parametrize("case", ["map_cap", "arena"])
def test_mass_deletion(case, oracle_mod):
    """2 100 of 4 400 RayClusters deleted by swap-remove.  The first 2 100: 2 100 holes and the 2 100 rows that fill them, past the
    map's 4 096 rows (ROW_MAP).  Every other one: 1 150 holes below the new count and the 2 100 rows past it, inside the cap; the map is
    followed, and the re-decided moved RayClusters need new places past the end of an arena already full of the runs of the last
    pass (ARENA, from the device)."""
    snap, flags = cd._fleet(4400, seed=5, pods_per_cluster=2, groups=1)
    dr = cd._driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        gone = np.arange(2100) if case == "map_cap" else np.arange(0, 4400, 2)[:2100]
        cd._epoch(dr, synthetic.delete_clusters(snap, gone))
        dr.prev = None
        dr.check(oracle_mod, expect_incremental=False)
        expect(dr, "full", ["ROW_MAP" if case == "map_cap" else "ARENA"])
        dr.check(oracle_mod, expect_incremental=True)
        expect(dr, "incremental", [])
    finally:
        dr.close()


@pytest.mark.parametrize("on", [False, True])
def test_large_deletion(on, oracle_mod):
    """Deleting a large RayCluster (one with a region): ROW_MAP without KR_OPT_LARGE_MOVES, incremental with it."""
    snap, flags = grown_fleet(300)
    dr = cd._driver(snap, flags, large_clusters=True, large_moves=on)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        cd._epoch(dr, synthetic.delete_clusters(snap, [0]))
        dr.prev = None
        dr.check(oracle_mod, expect_incremental=on)
        expect(dr, *(("incremental", []) if on else ("full", ["ROW_MAP"])))
    finally:
        dr.close()


@pytest.mark.parametrize("on", [False, True])
def test_group_edit(on, oracle_mod):
    snap, flags = ge._fleet(300, seed=3, wtd_group_frac=0.0)
    dr = ge._driver(snap, flags) if on else Driver(snap, flags, slack=1.5)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        old, c = dr.snap, 137
        src = int(old.c_group_off[c])
        ge._epoch(dr, synthetic.regroup_clusters(old, {c: ge._groups(old, c) + [(src, ge._fresh_id(old))]}))
        dr.prev = None
        dr.check(oracle_mod, expect_incremental=on)
        expect(dr, *(("incremental", []) if on else ("full", ["SIZES"])))
    finally:
        dr.close()


@pytest.mark.parametrize("on", [False, True])
def test_workers_to_delete_rename(on, oracle_mod):
    snap, flags = synthetic.generate(synthetic.config("C2", n_clusters=300, pods_per_cluster=20, groups=2, wtd_group_frac=0.3, recreate_frac=0.0, seed=8))
    dr = Driver(snap, flags, wtd_edits=on)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        lists = lists_of(dr.snap)
        g = next(g for g, names in enumerate(lists) if names)
        lists[g][0] = int(dr.snap.p_name_id.max()) + 1                  # a rename (to a Pod that does not exist): the count stays
        dr.set_wtd_lists(lists)
        dr.check(oracle_mod, expect_incremental=on)
        expect(dr, *(("incremental", []) if on else ("full", ["STRUCTURAL"])))
    finally:
        dr.close()


def test_spec_edits_keep_the_epoch(oracle_mod):
    """A spec edited in place, committed as a spec row and as the whole JSON arena: both epochs stay incremental (no option decides
    this on the engine; KR_OPT_SPEC_ROWS only picks the native packer's commit)."""
    dr = Driver(*fleet(seed=12))
    try:
        first(dr, oracle_mod)
        for whole in (False, True):
            c = 17 + int(whole)
            off, ln = int(dr.snap.c_json_off[c]), int(dr.snap.c_json_len[c])
            dr.snap.json[off + ln // 2] = ord("x") if dr.snap.json[off + ln // 2] != ord("x") else ord("y")
            np.copyto(dr.views["json"][:dr.snap.dims["json"]], dr.snap.json)
            if whole:
                dr.eng.commit(abi.PART_JSON)
            else:
                dr.eng.commit_spec_rows([c])
            dr.check(oracle_mod, expect_incremental=True)
            expect(dr, "incremental", [])
    finally:
        dr.close()

"""KR_OPT_BUCKET_POD_LISTS on the H100: with the option on, kr_flags.fetch_pod_lists = 1 keeps the bucket pipeline and the incremental
epochs, and the lists the bucket pipeline builds from its resident state (kuberay_b200/csrc/kr_lists.cuh) are byte for byte the sort
pipeline's: sorted_pod_idx, sorted_action and every pod_start, after full passes and after incremental ones.

Every epoch is compared with the oracle and with a twin engine that has the option off (a fresh engine, the sort pipeline): the lists
byte for byte, the action runs owner by owner (their order is the bucket pipeline's, unspecified).  The fleet has every class the
bucket pipeline decides: orphans and free rows, multi-host groups, Recreate gates, suspended RayClusters, workersToDelete lists, and a
large, a huge and a wide RayCluster; the large and huge ones stay untouched across several fetching epochs, so their per-cluster
sort segments, which share sorted_pod_idx, are written by one pass and never read by a later one."""
import os
import subprocess
import sys

import numpy as np
import pytest

from harness import PACKER_CAPS, Driver, Mirror, events, flip_ready, members, move, objects, packer_check, workers
from kuberay_b200 import abi, synthetic
from kuberay_b200 import snapshot as snp
from kuberay_b200.engine import Engine
from kuberay_b200.packer import Packer

pytestmark = pytest.mark.gpu

CLASSES = dict(large_clusters=True, wide_clusters=True, huge_clusters=True)
HUGE, LARGE, WIDE = 5, 40, 70


def fleet(seed):
    """900 RayClusters of 24 Pods in two worker groups with every class of the bucket pipeline, a huge (9 000 Pods), a large (1 200) and
    a wide (40 groups) one, orphans and free rows.  -> (snapshot, flags fetching the lists)."""
    snap, flags = synthetic.generate(synthetic.SynthParams(
        n_clusters=900, pods_per_cluster=24, groups=2, recreate_frac=0.05, suspended_frac=0.03, wtd_group_frac=0.2, multihost_frac=0.08,
        orphan_frac=0.01, autoscaling_frac=0.3, jobs=True, seed=seed))
    synthetic.grow_clusters(snap, [HUGE], 9000)
    synthetic.grow_clusters(snap, [HUGE, LARGE], 1200)
    snap = synthetic.widen_clusters(snap, [WIDE], 40)
    tombstone(snap, np.arange(11, snap.dims["pods"], 701))
    flags.fetch_pod_lists = 1
    return snap, flags


def tombstone(snap, rows):
    """Pods deleted: their rows become free rows."""
    for col in ("p_ns_id", "p_cluster_name_id", "p_group_name_id", "p_name_id", "p_replica_index", "p_replica_name_id"):
        snap.cols[col][rows] = 0
    snap.p_packed[rows] = np.uint32(abi.PP_TOMBSTONE)


def twin(snap, flags):
    """The same snapshot on a fresh engine with the option off (fetch_pod_lists = 1: the sort pipeline)."""
    eng = Engine.for_snapshot(snap, max_creates=1 << 20, **CLASSES)
    try:
        eng.load(snap)
        res = eng.reconcile(flags)
        assert eng.last_pass()["pipeline"] != "bucket"
        return res
    finally:
        eng.close()


def check(dr, oracle, kind):
    """One pass of the driver's engine: the bucket pipeline, of `kind`, equal to the oracle and, lists byte for byte, to the twin."""
    got = dr.eng.reconcile(dr.flags)
    rep = dr.eng.last_pass()
    assert rep["pipeline"] == "bucket" and rep["kind"] == kind, rep
    d = oracle.run(dr.snap, dr.flags).diff(got)
    assert not d, d[:6]
    if dr.flags.fetch_pod_lists:
        ref = twin(dr.snap, dr.flags)
        d = ref.diff(got)
        assert not d, d[:6]
        assert np.array_equal(got.sorted_pod_idx, ref.sorted_pod_idx)
        assert np.array_equal(got.sorted_action, ref.sorted_action)
        assert np.array_equal(got.clusters["pod_start"], ref.clusters["pod_start"])
    else:
        assert got.sorted_pod_idx.size == 0 and not got.clusters["pod_start"].any()
    return got


def open_driver(snap, flags, **options):
    dr = Driver(snap, flags, max_creates=1 << 20, bucket_pod_lists=True, **options)
    dr.flags.fetch_pod_lists = 1  # (the Driver asks for the compact results)
    return dr


@pytest.mark.parametrize("seed", [1, 2])
def test_every_fleet_class_full_and_incremental(seed, oracle_mod):
    fleet_stream(seed, oracle_mod, lambda epoch: epoch % 3 == 2)


def fleet_stream(seed, oracle_mod, big):
    """The fleet, a full pass and six incremental epochs of Pod churn, a moved and a deleted Pod; the large, huge and wide
    RayClusters also churn in the epochs where big(epoch), and stay untouched in the others."""
    dr = open_driver(*fleet(seed), **CLASSES)
    rng = np.random.default_rng(seed)
    try:
        assert dr.eng.get_option(abi.OPT_BUCKET_POD_LISTS) == 1
        check(dr, oracle_mod, "full")
        ordinary = np.array([c for c in range(dr.snap.dims["clusters"]) if c not in (HUGE, LARGE, WIDE)])
        for epoch in range(6):
            rows = [workers(dr.snap, int(c))[:2] for c in rng.choice(ordinary, 30, replace=False)]
            if big(epoch):
                rows += [workers(dr.snap, c)[::97] for c in (HUGE, LARGE, WIDE)]
            rows = np.concatenate(rows)
            flip_ready(dr.snap, rows)
            a, b = (int(c) for c in rng.choice(ordinary, 2, replace=False))  # a Pod changes RayCluster
            moved = workers(dr.snap, a)[:1]
            move(dr.snap, moved, b)
            gone = workers(dr.snap, int(rng.choice(ordinary)))[:1]  # and one is deleted
            tombstone(dr.snap, gone)
            dr.commit_rows(np.concatenate([rows, moved, gone]))
            check(dr, oracle_mod, "incremental")
    finally:
        dr.close()


def small_fleet(seed=4):
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=300, pods_per_cluster=20, groups=2, orphan_frac=0.02, seed=seed))
    flags.fetch_pod_lists = 1
    return snap, flags


def test_pass_report_while_the_flag_toggles(oracle_mod):
    """fetch_pod_lists 0 -> 1 -> 1 -> 0 -> 1: every pass on the bucket pipeline, every one after the first incremental; a pass without
    the lists leaves every pod_start 0 again."""
    dr = open_driver(*small_fleet())
    try:
        for i, fetch in enumerate((0, 1, 1, 0, 1)):
            if i:
                rows = np.arange(3 + i, dr.snap.dims["pods"], 613)
                flip_ready(dr.snap, rows)
                dr.commit_rows(rows)
            dr.flags.fetch_pod_lists = fetch
            check(dr, oracle_mod, "incremental" if i else "full")
            rep = dr.eng.last_pass()
            assert rep["why"] == (["FIRST"] if i == 0 else []), rep
    finally:
        dr.close()


def test_an_early_cluster_grows_and_every_later_start_moves(oracle_mod):
    """Three Pods join RayCluster 2: the epoch re-decides only the RayClusters they touched, yet every later RayCluster's list starts
    three places further on, and the fetch brings back those starts."""
    dr = open_driver(*small_fleet(6))
    try:
        before = check(dr, oracle_mod, "full").clusters["pod_start"].copy()
        donor = workers(dr.snap, 200)[:3]
        move(dr.snap, donor, 2)
        dr.commit_rows(donor)
        got = check(dr, oracle_mod, "incremental")
        changed = set(got.changed_clusters.tolist())
        assert changed == {2, 200}, changed
        after = got.clusters["pod_start"]
        assert np.array_equal(after[:3], before[:3])
        assert np.array_equal(after[3:201], before[3:201] + 3)
        assert np.array_equal(after[201:], before[201:])
        assert members(dr.snap, 2).size == after[3] - after[2]
    finally:
        dr.close()


@pytest.mark.parametrize("seed", [3, 4])
def test_native_packer_stream_fetching_every_third_epoch(seed, oracle_mod):
    """A seeded native packer stream with every option and this one: each epoch against the oracle, the lists every third epoch
    compared Pod key by Pod key (the two sides intern and number differently)."""
    opts = dict(CLASSES, wtd_edits=True, spec_rows=True, cluster_creates=True, cluster_deletes=True, group_edits=True, large_growth=True,
                large_moves=True, huge_growth=True, bucket_pod_lists=True)
    pk = Packer(**PACKER_CAPS, **opts)
    try:
        m = Mirror(*objects(seed), pk)
        pk.flush()
        rng, counter = np.random.default_rng(seed), [0]
        for epoch in range(12):
            if epoch:
                events(rng, m, counter, structural=True)
                pk.flush()
            lean = epoch % 3 != 0
            want, got = packer_check(m, oracle_mod, lean=lean)
            rep = pk.last_pass()
            assert rep["kind"] == "full" or rep["why"] == [], rep
            if lean:
                continue
            assert rep["pipeline"] == "bucket", rep
            _, meta = snp.pack_objects([m.clusters[k] for k in sorted(m.clusters)], m.live_pods(), m.jobs)  # (packer_check's packing)
            for ci, key in enumerate(meta.cluster_keys):
                r = pk.cluster_row(*key)
                ws, gs, n = int(want.clusters["pod_start"][ci]), int(got.clusters["pod_start"][r]), int(got.clusters["n_pods"][r])
                assert [pk.pod_key(int(p)) for p in got.sorted_pod_idx[gs:gs + n]] == [meta.pod_keys[int(p)] for p in want.sorted_pod_idx[ws:ws + n]], (epoch, key)
                assert np.array_equal(got.sorted_action[gs:gs + n], want.sorted_action[ws:ws + n]), (epoch, key)
    finally:
        pk.close()


def test_launch_shapes_at_eight_sms():
    """The whole path under KR_SM_COUNT=8, where the SM-sized kernels of the passes around the builder take many grid-stride trips (a
    subprocess: the engine reads it at creation)."""
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "import test_gpu_bucket_pod_lists as t\n"
            "from oracle import oracle\n"
            "assert t.Engine(0, 1, 1, 1, 64, 1, 1, 1, 64).get_option(t.abi.OPT_SM_COUNT) == 8\n"
            "t.test_every_fleet_class_full_and_incremental(1, oracle)\n"
            "t.test_an_early_cluster_grows_and_every_later_start_moves(oracle)\n") % (os.path.dirname(os.path.abspath(__file__)),
                                                                                    os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    env = dict(os.environ, KR_SM_COUNT="8")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-4000:]


# ------------------------------------------------------------------------------------------------ list edges

def keep_pods(snap, rows):
    """A copy of `snap` with only the pod rows `rows` (in that order) and the head-aux rows of the heads among them; every
    RayCluster, group, name and the JSON arena stay."""
    d = snap.dims
    rows = np.asarray(rows, dtype=np.int64)
    new_p = np.full(d["pods"], -1, dtype=np.int64)
    new_p[rows] = np.arange(rows.size)
    heads = np.flatnonzero(new_p[snap.h_pod_idx] >= 0) if d["heads"] else np.zeros(0, np.int64)
    out = snap_like(snap, pods=rows.size, heads=heads.size)
    for name, _dt, mult, dim in abi.COLUMNS:
        src = snap.cols[name]
        if dim == "pods":
            out.cols[name][:] = src[rows]
        elif dim == "heads":
            out.cols[name][:] = src.reshape(-1, mult)[heads].reshape(-1)
        else:
            out.cols[name][:] = src
    out.h_pod_idx[:] = new_p[snap.h_pod_idx[heads]]
    return out.validate()


def snap_like(snap, **dims):
    d = dict(snap.dims, **dims)
    return snp.Snapshot(d["clusters"], d["groups"], d["wtd"], d["pods"], d["heads"], d["jobs"], d["json"])


def orphan(snap, rows):
    """Pods whose RayCluster is not in the snapshot."""
    snap.p_cluster_name_id[rows] = np.uint32(0x7E000000)


def tile_fleet(n_pods, tail):
    """RayClusters of 8 Pods in row order (no shuffle), cut to exactly `n_pods` rows, the first RayCluster's rows first.  tail:
    "orphans" — the last three rows are orphans; "flush" — the last RayCluster's Pods are the last rows; "empty" — so are those of
    the RayCluster before it, and the last two RayClusters have no Pods (their starts are n_pods)."""
    nc = n_pods // 8 + 4
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=nc, pods_per_cluster=8, groups=1, orphan_frac=0.0, shuffle=False, seed=n_pods))
    total = snap.dims["pods"]
    end = total - (16 if tail == "empty" else 0)
    snap = keep_pods(snap, np.arange(end - n_pods, end))
    if tail == "orphans":
        orphan(snap, np.arange(max(0, n_pods - 3), n_pods))
    flags.fetch_pod_lists = 1
    return snap, flags


@pytest.mark.parametrize("tail", ["orphans", "flush", "empty"])
@pytest.mark.parametrize("n_pods", [1, 255, 256, 257, 2047, 2048, 2049])
def test_pod_counts_around_the_tiles(n_pods, tail, oracle_mod):
    """Pod counts at the edges of k_lists_gather's 256-thread blocks (its thread one past the end writes the starts of the
    trailing RayClusters without Pods) and of the sort's tiles; a full pass, then an incremental epoch that flips one Pod."""
    snap, flags = tile_fleet(n_pods, tail)
    assert snap.dims["pods"] == n_pods
    dr = open_driver(snap, flags)
    try:
        got = check(dr, oracle_mod, "full")
        if tail == "orphans":
            assert got.n_orphans == min(3, n_pods)
        else:
            assert got.n_orphans == 0 and got.clusters["n_pods"][-1 - 2 * (tail == "empty")] > 0
        if tail == "empty":
            assert (got.clusters["n_pods"][-2:] == 0).all() and (got.clusters["pod_start"][-2:] == n_pods).all()
        rows = np.array([n_pods // 2])
        flip_ready(dr.snap, rows)
        dr.commit_rows(rows)
        check(dr, oracle_mod, "incremental")
    finally:
        dr.close()


@pytest.mark.parametrize("shape", ["all_orphans", "no_clusters", "no_pods"])
def test_fleets_without_lists_to_build(shape, oracle_mod):
    """Every Pod an orphan (every RayCluster's list empty, each starting at 0), no RayClusters at all (kr_snapshot_begin takes
    the layout: every Pod in the orphans' segment), and no Pods."""
    snap, flags = tile_fleet(300, "flush")
    if shape == "all_orphans":
        orphan(snap, np.arange(snap.dims["pods"]))
    elif shape == "no_clusters":
        snap = synthetic.first_clusters(snap, 0, free_pods=False)
    else:
        snap = keep_pods(snap, [])
    dr = open_driver(snap, flags)
    try:
        got = check(dr, oracle_mod, "full")
        assert not got.clusters["pod_start"].any()
        if shape != "no_pods":
            assert got.n_orphans == snap.dims["pods"]
    finally:
        dr.close()


def test_structural_void_then_full_then_incremental(oracle_mod):
    """A renamed worker group is a table key: the incremental attempt flags KR_INC_STRUCTURAL (k_lists_owner then leaves every
    owner unset) and the full pass that follows builds the lists; Pod churn after that is incremental again."""
    dr = open_driver(*small_fleet(8))
    try:
        check(dr, oracle_mod, "full")
        rows = np.arange(5, dr.snap.dims["pods"], 331)
        flip_ready(dr.snap, rows)
        dr.snap.g_name_id[7] += np.uint32(100000)
        dr.commit_objects()
        dr.commit_rows(rows)
        check(dr, oracle_mod, "full")
        assert dr.eng.last_pass()["why"] == ["STRUCTURAL"], dr.eng.last_pass()
        donor = workers(dr.snap, 250)[:2]
        move(dr.snap, donor, 1)
        dr.commit_rows(donor)
        check(dr, oracle_mod, "incremental")
    finally:
        dr.close()


@pytest.mark.parametrize("seed", [5])
def test_large_and_huge_redecided_in_consecutive_epochs(seed, oracle_mod):
    """The large, huge and wide RayClusters re-decided in every epoch: each pass's per-cluster kernels find their sort segments in
    sorted_pod_idx overwritten by the lists of the pass before, and must sort them again before the builder overwrites them."""
    fleet_stream(seed, oracle_mod, lambda epoch: True)

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
    dr = open_driver(*fleet(seed), **CLASSES)
    rng = np.random.default_rng(seed)
    try:
        assert dr.eng.get_option(abi.OPT_BUCKET_POD_LISTS) == 1
        check(dr, oracle_mod, "full")
        ordinary = np.array([c for c in range(dr.snap.dims["clusters"]) if c not in (HUGE, LARGE, WIDE)])
        for epoch in range(6):
            rows = [workers(dr.snap, int(c))[:2] for c in rng.choice(ordinary, 30, replace=False)]
            if epoch % 3 == 2:  # every third epoch also the large, huge and wide ones; the others leave them untouched
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

"""Incrementally maintained arena (kuberay_b200/live.py, SURVEY §8(f) rank 1): Pod add / update / delete events become
single-row uploads, free rows are KR_PP_TOMBSTONE rows.

CPU: an arena with free rows must decide exactly like the same objects packed from scratch (oracle on both).
GPU: after every epoch of random events the engine (kr_snapshot_commit_parts(KR_PART_OBJECTS) + kr_snapshot_commit_pod_rows)
must equal the oracle on the arena byte for byte, and most epochs must take the incremental path.
"""
import numpy as np
import pytest

import fuzz_objects
from harness import events
from kuberay_b200 import abi
from kuberay_b200.live import LiveArena


def _same_decisions(arena_snap, a: abi.Results, fresh_snap, b: abi.Results, rows):
    """a = pass over the arena (free rows present), b = pass over the same objects packed from scratch."""
    live_rows = np.array([i for i, p in enumerate(rows) if p is not None], dtype=np.int64)
    to_fresh = np.full(len(rows), -1, dtype=np.int64)
    to_fresh[live_rows] = np.arange(live_rows.size)
    for fld in a.clusters.dtype.names:
        if fld in ("pod_start", "head_pod_idx"):
            continue
        assert np.array_equal(a.clusters[fld], b.clusters[fld]), fld
    hp = a.clusters["head_pod_idx"]
    assert np.array_equal(np.where(hp >= 0, to_fresh[np.maximum(hp, 0)], hp), b.clusters["head_pod_idx"])
    assert np.array_equal(a.groups, b.groups) and np.array_equal(a.hash, b.hash) and np.array_equal(a.jobs, b.jobs)
    assert np.array_equal(a.create_idx[:a.n_create_total], b.create_idx[:b.n_create_total])
    w = a.wtd_pod_idx.astype(np.int64)
    assert np.array_equal(np.where(w >= 0, to_fresh[np.maximum(w, 0)], w), b.wtd_pod_idx.astype(np.int64))
    keep = a.sorted_action != abi.ACT_TOMBSTONE
    assert int((~keep).sum()) == sum(p is None for p in rows)
    assert np.array_equal(to_fresh[a.sorted_pod_idx[keep]], b.sorted_pod_idx.astype(np.int64))
    assert np.array_equal(a.sorted_action[keep], b.sorted_action)
    assert (a.n_orphans, a.n_actions, a.n_create_total) == (b.n_orphans, b.n_actions, b.n_create_total)
    assert np.array_equal(to_fresh[a.act_pod_idx[:a.n_actions]], b.act_pod_idx[:b.n_actions].astype(np.int64))
    assert np.array_equal(a.act_code[:a.n_actions], b.act_code[:b.n_actions]) and np.array_equal(a.act_start, b.act_start)


@pytest.mark.parametrize("seed", [1, 2, 3, 4, 5, 6])
def test_arena_with_free_rows_decides_like_a_fresh_pack(seed, oracle_mod):
    rng = np.random.default_rng(seed)
    clusters, pods, jobs = fuzz_objects.generate(seed, big=True)
    live = LiveArena(clusters, pods, jobs, spare_rows=6, engine=False)
    counter = [0]
    for epoch in range(12):
        events(rng, live, counter, structural=True)
        live.flush()
        a = oracle_mod.run(live.snap, live.meta.flags)
        fresh, fmeta = live.fresh_pack()
        b = oracle_mod.run(fresh, fmeta.flags)
        _same_decisions(live.snap, a, fresh, b, live.rows)


@pytest.mark.gpu
@pytest.mark.parametrize("lean", [False, True])
@pytest.mark.parametrize("seed", [11, 12, 13, 14])
def test_incremental_epochs_match_the_oracle(seed, lean, oracle_mod):
    """lean (kr_flags.fetch_pod_lists = 0) is the production configuration: the bucket pipeline, and after its first pass the
    device-side incremental epochs (kr_incr.cuh) — every epoch must still equal a from-scratch oracle run over the arena, and most
    epochs must really have been incremental on the device (the pass names the records it recomputed)."""
    rng = np.random.default_rng(seed)
    clusters, pods, jobs = fuzz_objects.generate(seed, big=True)
    live = LiveArena(clusters, pods, jobs, spare_rows=16)
    counter = [0]
    device_incremental = 0
    try:
        for epoch in range(25):
            events(rng, live, counter, structural=(epoch % 8 == 7))
            live.flush()
            flags = live.meta.flags
            flags.fetch_pod_lists = 0 if lean else 1
            got = live.reconcile(flags)
            want = oracle_mod.run(live.snap, flags)
            d = want.diff(got)
            assert not d, (epoch, d[:6], got.n_changed)
            if got.changed_clusters is not None or (got.n_changed == 0 and live.snap.dims["clusters"]):
                device_incremental += 1
                assert got.n_changed <= live.snap.dims["clusters"] and len(set(got.changed_clusters.tolist() if got.changed_clusters is not None else [])) == got.n_changed
        assert live.stats["incremental"] >= 12 and live.stats["rebase"] >= 1 and live.stats["rows"] > 0, live.stats
        # (a snapshot with a multi-host group is decided by the sort pipeline: no resident buckets, no device-side incremental epochs)
        eligible = lean and not (live.snap.g_num_hosts > 1).any() and int(live.snap.c_group_cnt.max(initial=0)) <= 32
        assert device_incremental >= (10 if eligible else 0) and (lean or device_incremental == 0), (device_incremental, live.stats)
    finally:
        live.close()

"""KR_OPT_CLUSTER_DELETES: RayClusters deleted by swap-remove (the last RayCluster moves into each hole, as the native packer does) keep
the device-side incremental epoch.  The next pass releases the deleted RayClusters' Pods (orphans from then on), brings every moved
RayCluster to its new row, shifts the per-group results and re-decides only the moved and created RayClusters.

Every epoch is compared with the CPU oracle.  The records of the RayClusters a pass did not name must equal the previous epoch's
after the move: kept rows compare at the same row, and their group records at the shifted group indices."""
import copy

import numpy as np
import pytest

from harness import (PACKER_CAPS, POD_COLS, REBUILD, Driver, Mirror, events, flip_ready, incremental, members, move, objects, packer_check,
                     with_wtd_lists)
from kuberay_b200 import abi, synthetic
from kuberay_b200.packer import GroupPacker, Packer

pytestmark = pytest.mark.gpu

NEW = "k_inc_clusters_release"  # the first kernel of a renumbering epoch


def _fleet(n, seed, **kw):
    p = dict(n_clusters=n, pods_per_cluster=16, groups=2, seed=seed)
    p.update(kw)
    return synthetic.generate(synthetic.config("C2", **p))


def _driver(snap, flags, room=None, creates=False, **opts):
    """A Driver on `snap` (capacities from `room`, default `snap`) with the option on, after its first (full) pass."""
    dr = Driver(room if room is not None else snap, flags, slack=1.25, cluster_deletes=True, cluster_creates=creates, **opts)
    if room is not None:
        dr.use(snap)
        dr.commit_objects(abi.PART_ALL)
        for c in POD_COLS:
            dr.views[c][:] = snap.cols[c]
        dr.eng.commit(abi.PART_ALL)
    return dr


def _epoch(dr, new, created=(), pods_before=False):
    """One renumbering epoch: begin with `new`'s counts, the object part, the created RayClusters' specs as spec rows, and the pod
    rows that differ (committed before the object part when `pods_before`, else after it)."""
    changed = np.flatnonzero(np.any([dr.snap.cols[c] != new.cols[c] for c in POD_COLS], axis=0))
    if pods_before:
        for c in POD_COLS:
            dr.snap.cols[c][changed] = new.cols[c][changed]
        dr.commit_rows(changed)
    dr.use(new)
    dr.commit_objects()
    created = np.asarray(created, dtype=np.uint32)
    if created.size:
        np.copyto(dr.views["json"][:new.dims["json"]], new.json)
        dr.eng.commit_spec_rows(created)
    if not pods_before and changed.size:
        dr.commit_rows(changed)


def _check(dr, oracle, old, order, expect_incremental, profiled=False):
    """A pass against the oracle; when incremental, the records of the kept RayClusters it did not name against the previous epoch's
    (order[new row] = old row, -1: created).  -> (results, kernel names of a profiled pass)."""
    prev = dr.prev
    dr.prev = None
    got, names = dr.check(oracle, expect_incremental=expect_incremental, profiled=profiled)
    if expect_incremental and prev is not None:
        order = np.asarray(order)
        ch = set(got.changed_clusters.tolist()) if got.changed_clusters is not None else set()
        new = dr.snap
        for c in range(new.dims["clusters"]):
            if order[c] != c or c in ch:
                continue
            assert got.clusters[c].tobytes() == prev.clusters[c].tobytes(), c
            assert got.act_cnt[c] == prev.act_cnt[c], c
            assert bytes(got.hash[c]) == bytes(prev.hash[c]), c
            g_new, g_old, G = int(new.c_group_off[c]), int(old.c_group_off[c]), int(new.c_group_cnt[c])
            assert got.groups[g_new:g_new + G].tobytes() == prev.groups[g_old:g_old + G].tobytes(), c
    return got, names


def _live(snap, c):
    m = members(snap, c)
    return int(np.count_nonzero((snap.p_packed[m] & abi.PP_TOMBSTONE) == 0))


@pytest.mark.parametrize("where", ["first", "middle", "before_last", "last"])
def test_single_deletion(where, oracle_mod):
    snap, flags = _fleet(300, seed=3, wtd_group_frac=0.0)  # (no workersToDelete names: a shifted name re-touches the Pods it names)
    d = {"first": 0, "middle": 137, "before_last": 298, "last": 299}[where]
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        for step in range(3):  # three deletions in a row, each incremental
            old = dr.snap
            order = synthetic.swap_remove_order(old.dims["clusters"], [min(d, old.dims["clusters"] - 1)])
            new = synthetic.delete_clusters(old, [min(d, old.dims["clusters"] - 1)])
            orphans = dr.prev.n_orphans
            lost = _live(old, min(d, old.dims["clusters"] - 1))
            _epoch(dr, new)
            got, names = _check(dr, oracle_mod, old, order, True, profiled=True)
            assert NEW in names and "k_hash" not in names and "k_hash_rows" not in names, names
            assert got.n_orphans == orphans + lost, (got.n_orphans, orphans, lost)
            moved = [c for c in range(new.dims["clusters"]) if order[c] != c]
            ch = got.changed_clusters.tolist() if got.changed_clusters is not None else []
            assert sorted(ch) == moved, (ch, moved)  # only the moved RayCluster is re-decided
        rows = np.arange(5, dr.snap.dims["pods"], 89, dtype=np.uint32)  # an ordinary epoch afterwards
        flip_ready(dr.snap, rows)
        dr.commit_rows(rows)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


@pytest.mark.parametrize("k", [7, 300])
def test_batch(k, oracle_mod):
    snap, flags = _fleet(800, seed=k, wtd_group_frac=0.3)
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rows = np.random.default_rng(k).choice(800, size=k, replace=False)
        order = synthetic.swap_remove_order(800, rows)
        new = synthetic.delete_clusters(snap, rows)
        _epoch(dr, new)
        _check(dr, oracle_mod, snap, order, True)
        flip_ready(dr.snap, np.arange(1, dr.snap.dims["pods"], 37))
        dr.commit_rows(np.arange(1, dr.snap.dims["pods"], 37))
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


def test_more_than_the_cap_takes_the_full_pass(oracle_mod):
    snap, flags = _fleet(4400, seed=5, pods_per_cluster=2, groups=1)
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rows = np.arange(0, 4400, 2)[:2100]  # 2 100 deleted and as many moved: more than 4 096 rows
        new = synthetic.delete_clusters(snap, rows)
        _epoch(dr, new)
        dr.check(oracle_mod, expect_incremental=False)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


def test_deletion_with_creation(oracle_mod):
    """Both options: a RayCluster created in the row a deleted one vacated, and a RayCluster deleted and created again under its name
    in the same epoch, which adopts its old Pods."""
    full, flags = _fleet(306, seed=11)
    before = synthetic.select_clusters(full, np.arange(300))
    dr = _driver(before, flags, room=full, creates=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        # (a) RayCluster 20 deleted (299 moves into its hole), RayCluster 300 created after the last row
        order = list(synthetic.swap_remove_order(300, [20])) + [300]
        new = synthetic.select_clusters(full, order)
        _epoch(dr, new, created=[299])
        got, names = _check(dr, oracle_mod, before, [o if o < 300 else -1 for o in order], True, profiled=True)
        assert NEW in names and "k_hash_rows" in names and "k_hash" not in names, names
        assert {20, 299} <= set(got.changed_clusters.tolist())
        # (b) the last row deleted and a new RayCluster created in its place: a vacated row below the old count
        old = dr.snap
        order2 = list(order[:-1]) + [301]
        new = synthetic.select_clusters(full, order2)
        _epoch(dr, new, created=[299])
        _check(dr, oracle_mod, old, list(range(299)) + [-1], True)
        # (c) RayCluster 5 deleted and created again under its name in the same epoch (the last row moves into its hole; the new one
        # is appended): its Pods are orphans for a moment and come back to it
        old = dr.snap
        o3 = list(order2)
        o3[5], o3[-1] = o3[-1], o3[5]
        new = synthetic.select_clusters(full, o3)
        orphans = dr.prev.n_orphans
        _epoch(dr, new, created=[5, 299])
        got, _ = _check(dr, oracle_mod, old, [c if c not in (5, 299) else -1 for c in range(300)], True)
        assert got.n_orphans == orphans
    finally:
        dr.close()


def test_recreate_gated_and_multihost(oracle_mod):
    snap, flags = _fleet(300, seed=31, recreate_frac=0.2, multihost_frac=0.1)
    rc = np.flatnonzero(snap.c_flags & abi.CF_UPGRADE_RECREATE)
    mh = [c for c in range(300) if (snap.g_num_hosts[int(snap.c_group_off[c]):int(snap.c_group_off[c] + snap.c_group_cnt[c])] > 1).any()]
    assert rc.size > 4 and len(mh) > 4
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        # a multi-host RayCluster and a Recreate-gated one deleted, and the last rows (of either class, or both) moved into their holes
        for d in (int(mh[0]), int(rc[0]), int(rc[-1]) - 5):
            old = dr.snap
            rows = [d]
            order = synthetic.swap_remove_order(old.dims["clusters"], rows)
            _epoch(dr, synthetic.delete_clusters(old, rows))
            got, names = _check(dr, oracle_mod, old, order, True, profiled=True)
            assert "k_hash" not in names and "k_hash_rows" not in names, names  # (the digest moved, nothing re-hashed)
    finally:
        dr.close()


def test_workers_to_delete(oracle_mod):
    """Names in deleted, moved and merely shifted RayClusters, and a deleted RayCluster's Pod named in another RayCluster's list."""
    snap, flags = _fleet(200, seed=41, wtd_group_frac=0.5)
    named = [c for c in range(200) if snap.g_wtd_cnt[int(snap.c_group_off[c]):int(snap.c_group_off[c] + snap.c_group_cnt[c])].sum()]
    assert len(named) > 20
    # RayCluster 199 (the one that moves) names a Pod of RayCluster named[1], which is deleted in the second epoch
    g = int(snap.c_group_off[199])
    lists = [list(snap.w_name_id[int(snap.g_wtd_off[x]):int(snap.g_wtd_off[x] + snap.g_wtd_cnt[x])]) for x in range(snap.dims["groups"])]
    victim = members(snap, named[1])[2]
    lists[g] = lists[g] + [int(snap.p_name_id[victim])]
    snap = with_wtd_lists(snap, lists)
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        for d in (named[0], named[1]):
            old = dr.snap
            order = synthetic.swap_remove_order(old.dims["clusters"], [d])
            _epoch(dr, synthetic.delete_clusters(old, [d]))
            got, names = _check(dr, oracle_mod, old, order, True, profiled=True)
            assert set(REBUILD) <= set(names), names
    finally:
        dr.close()


@pytest.mark.parametrize("when", ["before", "after"])
def test_same_epoch_pod_events(when, oracle_mod):
    """A status update on a Pod of the moved RayCluster, a Pod of the deleted RayCluster removed, and a Pod re-labelled into the moved
    RayCluster, committed before or after the object part."""
    snap, flags = _fleet(250, seed=51)
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        d = 40
        order = synthetic.swap_remove_order(250, [d])
        new = synthetic.delete_clusters(snap, [d])
        mv = members(snap, 249)
        flip_ready(new, mv[1:3])
        gone = members(snap, d)[3]
        for c in POD_COLS:
            new.cols[c][gone] = 0
        new.p_packed[gone] = np.uint32(abi.PP_TOMBSTONE)
        other = members(snap, 100)[4]
        move(new, [other], d)  # (row d now holds the moved RayCluster)
        _epoch(dr, new, pods_before=when == "before")
        got, _ = _check(dr, oracle_mod, snap, order, True)
        assert {d, 100} <= set(got.changed_clusters.tolist())
    finally:
        dr.close()


def test_wide_deleted_moved_and_created(oracle_mod):
    """With KR_OPT_WIDE_CLUSTERS, RayClusters of more than 32 worker groups deleted, moved and (with both options) created keep the
    incremental epoch: the per-cluster kernels take the new wide set."""
    snap, flags = _fleet(122, seed=61)
    full = synthetic.widen_clusters(snap, [60, 119, 121], 40)
    before = synthetic.select_clusters(full, np.arange(120))
    dr = _driver(before, flags, room=full, creates=True, wide_clusters=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        order = list(range(120))
        for rows, created in (([3], []), ([60], []), ([10], [121])):  # 119 (wide) moves into row 3; 60 (wide) deleted; 121 (wide) created
            old = dr.snap
            order = [order[i] for i in synthetic.swap_remove_order(len(order), rows)] + created
            new = synthetic.select_clusters(full, order)
            _epoch(dr, new, created=[len(order) - 1] if created else [])
            old_rows = [c if c < old.dims["clusters"] and int(old.c_name_id[c]) == int(new.c_name_id[c]) else -1 for c in range(len(order))]
            _check(dr, oracle_mod, old, old_rows, True)
    finally:
        dr.close()


def test_large_deleted_or_moved_takes_the_full_pass(oracle_mod):
    """A large RayCluster (KR_OPT_LARGE_CLUSTERS) deleted or moved takes the full pass: its region does not move with it.  The epoch
    after it is incremental again."""
    grown, flags = _fleet(200, seed=62)
    synthetic.grow_clusters(grown, [199, 50], 300)
    dr = _driver(grown, flags, large_clusters=True)
    try:
        dr.check(oracle_mod, expect_incremental=None)
        dr.check(oracle_mod, expect_incremental=None)
        for rows in ([7], [50]):  # a large one moved (199 into row 7), then a large one deleted
            _epoch(dr, synthetic.delete_clusters(dr.snap, rows))
            dr.check(oracle_mod, expect_incremental=False)
        flip_ready(dr.snap, np.arange(3, dr.snap.dims["pods"], 41))
        dr.commit_rows(np.arange(3, dr.snap.dims["pods"], 41))
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


@pytest.mark.parametrize("case", ["delete_then_append", "append_then_delete", "delete_then_delete", "delete_then_same_counts"])
def test_two_object_commits_in_one_epoch(case, oracle_mod):
    """Two begin / object-commit rounds before one pass.  A renumbering after an append of the same epoch (rows the device tables do
    not hold yet), a count change after a renumbering, and a second renumbering take the full pass; an object part of the same counts
    after a renumbering keeps the incremental epoch.  Every pass is compared with the oracle."""
    full, flags = _fleet(306, seed=91, wtd_group_frac=0.3)
    before = synthetic.select_clusters(full, np.arange(300))
    dr = _driver(before, flags, room=full, creates=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        one = list(synthetic.swap_remove_order(300, [20]))  # RayCluster 20 deleted, 299 moves into its hole
        if case == "append_then_delete":
            first = list(range(300)) + [300]
            second = [first[i] for i in synthetic.swap_remove_order(301, [20])]
            rounds = [(first, [300]), (second, [])]
        elif case == "delete_then_append":
            rounds = [(one, []), (one + [300], [299])]
        elif case == "delete_then_delete":
            rounds = [(one, []), ([one[i] for i in synthetic.swap_remove_order(299, [40])], [])]
        else:
            rounds = [(one, []), (one, [])]
        for order, created in rounds:
            _epoch(dr, synthetic.select_clusters(full, order), created=created)
        dr.prev = None
        dr.check(oracle_mod, expect_incremental=case == "delete_then_same_counts")
        flip_ready(dr.snap, np.arange(3, dr.snap.dims["pods"], 41))
        dr.commit_rows(np.arange(3, dr.snap.dims["pods"], 41))
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


@pytest.mark.parametrize("event", ["option_off", "non_swap", "duplicate_key", "group_count", "toggled"])
def test_still_full_passes(event, oracle_mod):
    snap, flags = _fleet(204, seed=71)
    if event == "duplicate_key":  # RayCluster 9 holds RayCluster 30's key (the lowest row keeps it)
        snap.c_ns_id[30], snap.c_name_id[30] = snap.c_ns_id[9], snap.c_name_id[9]
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        if event in ("option_off", "toggled"):
            dr.eng.set_cluster_deletes(False)
        if event == "non_swap":  # rows 3 and 4 swapped, the last one deleted
            order = list(range(203))
            order[3], order[4] = 4, 3
            new = synthetic.select_clusters(snap, order)
        elif event == "group_count":  # RayCluster 10 deleted and 203 (moving into its row) gains a worker group
            new = synthetic.delete_clusters(synthetic.widen_clusters(snap, [203], 3), [10])
        else:
            new = synthetic.delete_clusters(snap, [30 if event == "duplicate_key" else 12])
        _epoch(dr, new)
        if event == "toggled":
            dr.eng.set_cluster_deletes(True)  # (read at begin and at the object commit: both saw it off)
        dr.check(oracle_mod, expect_incremental=False)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


def test_option_off_twin(oracle_mod):
    """The same deletion epochs with the option off: full passes, and records identical to the option-on engine's."""
    snap, flags = _fleet(260, seed=72)
    on, off = _driver(snap, flags), _driver(snap, flags)
    off.eng.set_cluster_deletes(False)
    try:
        for dr in (on, off):
            dr.check(oracle_mod, expect_incremental=False)
        for rows in ([3], [17, 100, 250], [0]):
            old = on.snap
            new = synthetic.delete_clusters(old, [r for r in rows if r < old.dims["clusters"]])
            order = synthetic.swap_remove_order(old.dims["clusters"], [r for r in rows if r < old.dims["clusters"]])
            _epoch(on, new)
            _epoch(off, copy.deepcopy(new))
            got, _ = _check(on, oracle_mod, old, order, True)
            twin, _ = off.check(oracle_mod, expect_incremental=False)
            d = twin.diff(got)
            assert not d, d[:6]
    finally:
        on.close()
        off.close()


def test_transfer_size(oracle_mod):
    """A deletion epoch moves the object part plus the row map (the gone rows and their targets, the moved and created rows, the
    moved digests, 4 B per shifted group and per shifted name), no spec JSON, and hashes nothing."""
    snap, flags = _fleet(400, seed=81, wtd_group_frac=0.3)
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        dr.commit_objects()  # an object part that changed nothing: the baseline
        objects = dr.eng.last_profile()["h2d_bytes"]
        dr.check(oracle_mod, expect_incremental=True)
        rows = [5, 77, 310]
        new = synthetic.delete_clusters(snap, rows)
        dr.use(new)
        dr.commit_objects()
        h2d = dr.eng.last_profile()["h2d_bytes"]
        g0 = int(new.c_group_off[min(rows)])
        shifted = (new.dims["groups"] - g0) + (new.dims["wtd"] - int(new.g_wtd_off[g0]))
        gone, init = 2 * len(rows), len(rows)
        assert h2d <= objects + 4 * (2 * gone + init + 2 * init + shifted) + 6 * 16, (h2d, objects, shifted)
        _, names = _check(dr, oracle_mod, snap, synthetic.swap_remove_order(400, rows), True, profiled=True)
        assert "k_hash" not in names and "k_hash_rows" not in names, names
    finally:
        dr.close()


def _stream(m, rng, counter, deleted):
    """One epoch's informer events: Pod and RayCluster events, RayClusters deleted (their Pods stay: orphans), created, or created
    again under an old name."""
    u = rng.random()
    if u >= 0.5:
        events(rng, m, counter, structural=False)
    keys = sorted(m.clusters)
    if u < 0.3 and len(keys) > 8:
        for _ in range(int(rng.integers(1, 4))):
            key = keys.pop(int(rng.integers(len(keys))))
            deleted[key] = m.clusters[key]
            m.delete_cluster(*key)
    elif u < 0.4 and deleted:
        key = sorted(deleted)[int(rng.integers(len(deleted)))]
        counter[0] += 1
        m.upsert_cluster(dict(deleted.pop(key), resourceVersion=90_000 + counter[0]))
    elif u < 0.5:
        src = copy.deepcopy(m.clusters[keys[int(rng.integers(len(keys)))]])
        counter[0] += 1
        src["name"], src["generation"], src["resourceVersion"] = f"{src['name']}-c{counter[0]}", 1, 50_000 + counter[0]
        m.upsert_cluster(src)


def test_packer_stream_against_option_off(oracle_mod):
    caps = dict(PACKER_CAPS, max_clusters=200, max_groups=1024, max_wtd=1024, max_pods=8192, max_jobs=256, max_creates=1 << 20)
    on, off = Packer(**caps, cluster_creates=True, cluster_deletes=True), Packer(**caps)
    try:
        objs = objects(5)
        m_on, m_off = Mirror(*copy.deepcopy(objs), on), Mirror(*copy.deepcopy(objs), off)
        rng_on, rng_off = np.random.default_rng(13), np.random.default_rng(13)
        c_on, c_off, d_on, d_off = [0], [0], {}, {}
        n_del = n_inc = n_json = 0
        for epoch in range(300):
            before = len(m_on.clusters)
            if before < caps["max_clusters"] - 4:
                _stream(m_on, rng_on, c_on, d_on)
                _stream(m_off, rng_off, c_off, d_off)
            deleting = len(m_on.clusters) < before
            mode = on.flush()
            off.flush()
            _, got = packer_check(m_on, oracle_mod, lean=True)
            _, twin = packer_check(m_off, oracle_mod, lean=True)
            assert np.array_equal(got.clusters, twin.clusters)
            if deleting and epoch:
                n_del += 1
                n_inc += incremental(got, got.clusters.shape[0])
                n_json += bool(mode & abi.PART_JSON)  # (only a flush that compacts the JSON arena sends it)
        print(f"deletion epochs {n_del}, incremental {n_inc}, with KR_PART_JSON {n_json}")
        assert n_del > 40 and n_inc > n_del // 2 and n_json * 10 <= n_del, (n_del, n_inc, n_json)
    finally:
        on.close()
        off.close()


def test_group_packer_two_shards_one_device(oracle_mod):
    caps = dict(PACKER_CAPS, max_clusters=128, max_groups=1024, max_wtd=1024, max_pods=8192, max_jobs=256)
    gp = GroupPacker([0, 0], **caps, cluster_deletes=True)
    try:
        assert all(sh.engine.get_option(abi.OPT_CLUSTER_DELETES) == 1 for sh in gp.shards)
        clusters, pods, jobs = objects(7)
        for c in clusters:
            gp.upsert_cluster(c)
        for p in pods:
            gp.upsert_pod(p)
        gp.flush()
        flags = gp.flags(fetch_pod_lists=0)
        gp.reconcile(flags)
        rng = np.random.default_rng(3)
        live = list(clusters)
        n_inc, epochs = 0, min(12, len(live) - 2)
        for epoch in range(epochs):
            c = live.pop(int(rng.integers(len(live))))
            sh_del = gp.shard_of(c.get("namespace", "default"), c["name"])
            gp.delete_cluster(c.get("namespace", "default"), c["name"])
            gp.flush()
            got = gp.reconcile(flags)
            n_inc += incremental(got[sh_del], got[sh_del].clusters.shape[0])
            for sh, g, f in zip(gp.shards, got, flags):
                sh.engine.set_incremental(False)
                full = sh.engine.reconcile(f)
                sh.engine.set_incremental(True)
                d = full.diff(g)
                assert not d, (epoch, d[:6])
            gp.reconcile(flags)  # (the full pass above left the resident state: the next deletion is incremental again)
        assert epochs >= 4 and n_inc >= epochs - 1, (n_inc, epochs)
    finally:
        gp.close()

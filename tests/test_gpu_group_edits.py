"""KR_OPT_GROUP_EDITS: a RayCluster whose list of worker groups changed (groups appended, as a RayService in-place update does,
removed, renamed or reordered) keeps the device-side incremental epoch.  The next pass releases the RayCluster's Pods, initialises it
again in its own row, matches its Pods against the new groups, shifts the group records of the RayClusters after it and re-decides
only it, plus the RayClusters whose Pods a rebuilt workersToDelete name table touched.

Every epoch is compared with the CPU oracle.  The records of the RayClusters a pass did not name must equal the previous epoch's,
their group records at the shifted group indices."""
import copy

import numpy as np
import pytest

from harness import (PACKER_CAPS, POD_COLS, REBUILD, Driver, Mirror, events, flip_ready, incremental, members, objects, packer_check,
                     run, scale_to, spec_bytes, with_json, workers)
from kuberay_b200 import abi, synthetic
from kuberay_b200.packer import GroupPacker, Packer

pytestmark = pytest.mark.gpu

NEW = "k_inc_clusters_release"  # the first kernel of an epoch whose row map has gone rows


def _fleet(n, seed, **kw):
    p = dict(n_clusters=n, pods_per_cluster=16, groups=2, seed=seed)
    p.update(kw)
    return synthetic.generate(synthetic.config("C2", **p))


def _driver(snap, flags, slack=1.5, **opts):
    """A Driver on `snap` with the option on (room for half as many groups and names again), after nothing was run yet."""
    return Driver(snap, flags, slack=slack, group_edits=True, **opts)


def _fresh_id(snap, k=0):
    """A name id no row of `snap` uses."""
    cols = ("g_name_id", "p_group_name_id", "p_name_id", "w_name_id", "c_name_id", "p_cluster_name_id")
    return max(int(snap.cols[c].max()) for c in cols if snap.cols[c].size) + 1 + k


def _groups(snap, c):
    g0 = int(snap.c_group_off[c])
    return [(g, None) for g in range(g0, g0 + int(snap.c_group_cnt[c]))]


def _respec(snap, rows):
    """A copy of `snap` whose RayClusters `rows` have a new spec (one byte longer) at the end of a grown JSON arena."""
    end = (snap.dims["json"] + 15) // 16 * 16
    bodies = {int(c): spec_bytes(snap, c) + b" " for c in rows}
    out = with_json(snap, end + sum((len(b) + 15) // 16 * 16 for b in bodies.values()))
    for c, body in bodies.items():
        out.json[end:end + len(body)] = np.frombuffer(body, dtype=np.uint8)
        out.c_json_off[c], out.c_json_len[c] = end, len(body)
        end += (len(body) + 15) // 16 * 16
    return out


def _epoch(dr, new, specs=(), spec_first=False, pods_before=False):
    """One edit epoch: begin with `new`'s counts, the object part, the re-emitted specs `specs` as spec rows (before the object part
    with `spec_first`, else after it) and the pod rows that differ (before the object part with `pods_before`, else after it)."""
    changed = np.flatnonzero(np.any([dr.snap.cols[c] != new.cols[c] for c in POD_COLS], axis=0))
    if pods_before:
        for c in POD_COLS:
            dr.snap.cols[c][changed] = new.cols[c][changed]
        dr.commit_rows(changed)
    dr.use(new)
    specs = np.asarray(sorted(specs), dtype=np.uint32)

    def spec_rows():
        np.copyto(dr.views["json"][:new.dims["json"]], new.json)
        for name in ("c_json_off", "c_json_len"):
            dr.views[name][:] = new.cols[name]
        dr.eng.commit_spec_rows(specs)
    if specs.size and spec_first:
        spec_rows()
    dr.commit_objects()
    if specs.size and not spec_first:
        spec_rows()
    if not pods_before and changed.size:
        dr.commit_rows(changed)


def _named_clusters(*snaps):
    """RayClusters (of the last snapshot) with a Pod whose name some workersToDelete list of any of `snaps` holds."""
    new = snaps[-1]
    names = np.unique(np.concatenate([s.w_name_id for s in snaps]))
    rows = np.flatnonzero(np.isin(new.p_name_id, names))
    keys = {(int(new.p_ns_id[p]), int(new.p_cluster_name_id[p])) for p in rows}
    return {c for c in range(new.dims["clusters"]) if (int(new.c_ns_id[c]), int(new.c_name_id[c])) in keys}


def _check(dr, oracle, old, regrouped, expect_incremental=True, profiled=False, order=None, others=()):
    """A pass against the oracle.  When incremental: the regrouped rows are among changed_clusters, every other named row is one
    whose Pods a rebuilt name table touched (or one of `others`), and every RayCluster it did not name keeps the previous epoch's
    records, its group records at the shifted indices (order[new row] = old row, -1: created; default: every row stays).
    -> (results, kernel names of a profiled pass)."""
    prev = dr.prev
    dr.prev = None
    got, names = dr.check(oracle, expect_incremental=expect_incremental, profiled=profiled)
    new = dr.snap
    if expect_incremental and prev is not None:
        ch = set(got.changed_clusters.tolist()) if got.changed_clusters is not None else set()
        assert set(regrouped) <= ch, (sorted(regrouped), sorted(ch))
        extra = ch - set(regrouped) - set(others)
        assert not extra or extra <= _named_clusters(old, new), sorted(extra)
        order = np.arange(new.dims["clusters"]) if order is None else np.asarray(order)
        for c in range(new.dims["clusters"]):
            o = int(order[c])
            if o != c or c in ch:
                continue
            assert got.clusters[c].tobytes() == prev.clusters[o].tobytes(), c
            assert got.act_cnt[c] == prev.act_cnt[o], c
            assert bytes(got.hash[c]) == bytes(prev.hash[o]), c
            g_new, g_old, G = int(new.c_group_off[c]), int(old.c_group_off[o]), int(new.c_group_cnt[c])
            assert G == int(old.c_group_cnt[o]), c
            assert got.groups[g_new:g_new + G].tobytes() == prev.groups[g_old:g_old + G].tobytes(), c
    return got, names


def _label(snap, c, k, name_id):
    """k of RayCluster c's worker Pods relabelled for the group `name_id` (which it does not have yet)."""
    w = workers(snap, c)[:k]
    snap.p_group_name_id[w] = name_id
    return w


@pytest.mark.parametrize("labelled", [False, True])
@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_append(where, k, labelled, oracle_mod):
    """Groups appended to one RayCluster, twice in a row, with or without Pods already labelled for them."""
    snap, flags = _fleet(300, seed=3, wtd_group_frac=0.0)
    c = {"first": 0, "middle": 137, "last": 299}[where]
    ids = [_fresh_id(snap, j) for j in range(2 * k)]
    if labelled:  # (Pods of the first new group exist before it does: in no group until then)
        _label(snap, c, 3, ids[0])
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        for step in range(2):
            old = dr.snap
            src = int(old.c_group_off[c])
            new = synthetic.regroup_clusters(old, {c: _groups(old, c) + [(src, ids[step * k + j]) for j in range(k)]})
            _epoch(dr, new)
            got, names = _check(dr, oracle_mod, old, [c], profiled=True)
            assert NEW in names and "k_hash" not in names and "k_hash_rows" not in names, names
            assert sorted(got.changed_clusters.tolist()) == [c]
        rows = np.arange(5, dr.snap.dims["pods"], 89, dtype=np.uint32)  # an ordinary epoch afterwards
        flip_ready(dr.snap, rows)
        dr.commit_rows(rows)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


@pytest.mark.parametrize("which", ["first", "middle", "last"])
def test_remove(which, oracle_mod):
    """A group removed from a RayCluster of three while its Pods live on: they stay among the RayCluster's Pods, in no group."""
    snap, flags = _fleet(200, seed=5, groups=3, wtd_group_frac=0.0)
    c = 77
    gi = {"first": 0, "middle": 1, "last": 2}[which]
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        g0 = int(snap.c_group_off[c])
        gone = workers(snap, c)[snap.p_group_name_id[workers(snap, c)] == snap.g_name_id[g0 + gi]]
        assert gone.size
        new = synthetic.regroup_clusters(snap, {c: [p for j, p in enumerate(_groups(snap, c)) if j != gi]})
        _epoch(dr, new)
        got, _ = _check(dr, oracle_mod, snap, [c])
        assert sorted(got.changed_clusters.tolist()) == [c]
    finally:
        dr.close()


@pytest.mark.parametrize("case", ["rename_first", "rename_second", "reorder", "down_to_zero_and_back"])
def test_rename_reorder_and_counts(case, oracle_mod):
    """Renamed and reordered groups, and group counts 2 -> 1 -> 0 -> 1 (the table slot's group-0 name changes with each)."""
    snap, flags = _fleet(200, seed=7, wtd_group_frac=0.0)
    c = 42
    g0 = int(snap.c_group_off[c])
    fresh = _fresh_id(snap)
    _label(snap, c, 2, fresh)
    if case == "rename_first":
        steps = [[(g0, fresh), (g0 + 1, None)]]
    elif case == "rename_second":
        steps = [[(g0, None), (g0 + 1, fresh)]]
    elif case == "reorder":
        steps = [[(g0 + 1, None), (g0, None)]]
    else:
        steps = [[(g0 + 1, None)], [], [(g0, fresh)]]
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        for pairs in steps:
            old = dr.snap
            _epoch(dr, synthetic.regroup_clusters(old, {c: pairs}))
            got, _ = _check(dr, oracle_mod, old, [c])
            assert sorted(got.changed_clusters.tolist()) == [c]
    finally:
        dr.close()


@pytest.mark.parametrize("wtd_edits", [False, True])
def test_workers_to_delete(wtd_edits, oracle_mod):
    """A group with workersToDelete names appended (a copy of a named group) and a named group removed: the name table is rebuilt,
    with KR_OPT_WTD_EDITS off or on."""
    snap, flags = _fleet(200, seed=41, wtd_group_frac=0.5)
    named = [g for g in range(snap.dims["groups"]) if snap.g_wtd_cnt[g]]
    assert len(named) > 20
    dr = _driver(snap, flags, wtd_edits=wtd_edits)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        g = named[3]
        c = int(snap.g_cluster_idx[g])
        old = dr.snap
        new = synthetic.regroup_clusters(old, {c: _groups(old, c) + [(g, _fresh_id(old))]})
        _epoch(dr, new)
        _, names = _check(dr, oracle_mod, old, [c], profiled=True)
        assert set(REBUILD) <= set(names), names
        old = dr.snap
        g = [x for x in range(old.dims["groups"]) if old.g_wtd_cnt[x]][10]
        c = int(old.g_cluster_idx[g])
        _epoch(dr, synthetic.regroup_clusters(old, {c: [p for p in _groups(old, c) if p[0] != g]}))
        _check(dr, oracle_mod, old, [c])
    finally:
        dr.close()


def test_multihost_arrives_and_leaves(oracle_mod):
    """The fleet's first multi-host group arrives through an append, and the last one leaves through its removal."""
    snap, flags = _fleet(200, seed=13, multihost_frac=0.0, wtd_group_frac=0.0)
    assert (snap.g_num_hosts <= 1).all()
    c = 60
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        new = synthetic.regroup_clusters(snap, {c: _groups(snap, c) + [(int(snap.c_group_off[c]), _fresh_id(snap))]})
        new.g_num_hosts[int(new.c_group_off[c]) + 2] = 2
        _epoch(dr, new)
        _check(dr, oracle_mod, snap, [c])
        old = dr.snap
        _epoch(dr, synthetic.regroup_clusters(old, {c: _groups(old, c)[:2]}))
        _check(dr, oracle_mod, old, [c])
    finally:
        dr.close()


def test_recreate_gated_respec(oracle_mod):
    """A Recreate-gated RayCluster gains a group with a new spec: its digest changes and it deletes all its Pods.  The spec row is
    hashed once; a Recreate-gated RayCluster regrouped without a new spec keeps its digest."""
    snap, flags = _fleet(200, seed=31, recreate_frac=0.3, wtd_group_frac=0.0)
    rc = np.flatnonzero(snap.c_flags & abi.CF_UPGRADE_RECREATE)
    assert rc.size > 4
    c, c2 = int(rc[1]), int(rc[3])
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        new = _respec(synthetic.regroup_clusters(snap, {c: _groups(snap, c) + [(int(snap.c_group_off[c]), _fresh_id(snap))]}), [c])
        _epoch(dr, new, specs=[c])
        got, names = _check(dr, oracle_mod, snap, [c], profiled=True)
        assert "k_hash_rows" in names and "k_hash" not in names, names
        old = dr.snap
        _epoch(dr, synthetic.regroup_clusters(old, {c2: _groups(old, c2)[:1]}))
        got, names = _check(dr, oracle_mod, old, [c2], profiled=True)
        assert "k_hash_rows" not in names and "k_hash" not in names, names
    finally:
        dr.close()


def test_suspended_append(oracle_mod):
    snap, flags = _fleet(150, seed=17, wtd_group_frac=0.0)
    c = 20
    fresh = _fresh_id(snap)
    _label(snap, c, 4, fresh)
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        new = synthetic.regroup_clusters(snap, {c: _groups(snap, c) + [(int(snap.c_group_off[c]), fresh)]})
        g = int(new.c_group_off[c]) + 2
        new.g_flags[g] |= np.uint32(abi.GF_SUSPEND)
        _epoch(dr, new)
        _check(dr, oracle_mod, snap, [c])
    finally:
        dr.close()


@pytest.mark.parametrize("wide", [False, True])
def test_crossing_32_groups(wide, oracle_mod):
    """A RayCluster grows from 2 to 34 groups: incremental with KR_OPT_WIDE_CLUSTERS (the per-cluster kernels take it), a correct
    full pass without it."""
    snap, flags = _fleet(200, seed=19, wtd_group_frac=0.0)
    c = 90
    src = int(snap.c_group_off[c])
    dr = _driver(snap, flags, slack=1.5, wide_clusters=wide)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        new = synthetic.regroup_clusters(snap, {c: _groups(snap, c) + [(src, _fresh_id(snap, j)) for j in range(32)]})
        _epoch(dr, new)
        _check(dr, oracle_mod, snap, [c], expect_incremental=wide)
        if wide:  # and back under 32
            old = dr.snap
            _epoch(dr, synthetic.regroup_clusters(old, {c: _groups(old, c)[:2]}))
            _check(dr, oracle_mod, old, [c])
    finally:
        dr.close()


@pytest.mark.parametrize("when", ["before", "after"])
def test_with_creation_deletion_and_pod_events(when, oracle_mod):
    """One epoch: Pod events, a RayCluster created after the last row, RayCluster 20 deleted by swap-remove with the last one (299)
    moving into its row and gaining a group there, and RayCluster 50 regrouped; pod rows committed before or after the object part."""
    full, flags = _fleet(306, seed=11, wtd_group_frac=0.3)
    before = synthetic.select_clusters(full, np.arange(300))
    dr = _driver(before, flags, cluster_creates=True, cluster_deletes=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        order = list(synthetic.swap_remove_order(300, [20])) + [300]
        new = synthetic.select_clusters(full, order)
        new = synthetic.regroup_clusters(new, {20: _groups(new, 20) + [(int(new.c_group_off[20]), _fresh_id(new))],
                                               50: _groups(new, 50)[1:]})
        flip_ready(new, members(new, 20)[1:3])
        flip_ready(new, members(new, 120)[:2])
        _epoch(dr, new, specs=[299], pods_before=when == "before")
        got, names = _check(dr, oracle_mod, before, [20, 50, 299], profiled=True, others=[120], order=[o if o < 300 else -1 for o in order])
        assert NEW in names, names
    finally:
        dr.close()


@pytest.mark.parametrize("spec_first", [False, True])
def test_spec_row_order(spec_first, oracle_mod):
    """A RayService-style append with a re-emitted spec: the spec row committed before or after the object part, hashed once."""
    snap, flags = _fleet(200, seed=23, wtd_group_frac=0.0)
    c = 111
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        new = _respec(synthetic.regroup_clusters(snap, {c: _groups(snap, c) + [(int(snap.c_group_off[c]), _fresh_id(snap))]}), [c])
        _epoch(dr, new, specs=[c], spec_first=spec_first)
        got, names = _check(dr, oracle_mod, snap, [c], profiled=True)
        assert names.count("k_hash_rows") == 1 and "k_hash" not in names, names
    finally:
        dr.close()


def test_create_cursor_passes_the_arena_end(oracle_mod):
    """Appending a group of 8 replicas and removing it again, epoch after epoch, on an engine whose create arena holds the fleet's
    creates plus a little: each append reserves fresh places, so the cursor passes the arena's end, that epoch falls back to a full
    pass, and every record stays right."""
    snap, flags = _fleet(120, seed=29, wtd_group_frac=0.0)
    base, _, _ = run(snap, flags)
    dr = Driver(snap, flags, slack=1.5, max_creates=int(base.n_create_total) + 24, group_edits=True)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        fresh = _fresh_id(snap)
        n_inc = n_full = 0
        for step in range(12):
            old = dr.snap
            c = 10 + step
            new = synthetic.regroup_clusters(old, {c: _groups(old, c) + [(int(old.c_group_off[c]), fresh)]})
            scale_to(new, int(new.c_group_off[c]) + int(new.c_group_cnt[c]) - 1, 8)
            _epoch(dr, new)
            got, _ = _check(dr, oracle_mod, old, [c], expect_incremental=None)
            inc = incremental(got, new.dims["clusters"])
            n_inc += inc
            n_full += not inc
            old = dr.snap
            _epoch(dr, synthetic.regroup_clusters(old, {c: _groups(old, c)[:-1]}))
            _check(dr, oracle_mod, old, [c], expect_incremental=None)
        assert n_inc >= 4 and n_full >= 1, (n_inc, n_full)
    finally:
        dr.close()


@pytest.mark.parametrize("event", ["option_off", "large", "over_the_cap", "recounted_in_the_same_epoch"])
def test_still_full_passes(event, oracle_mod):
    """Each takes the full pass, with the right records, and the epoch after it is incremental again."""
    n = 4200 if event == "over_the_cap" else 200
    snap, flags = _fleet(n, seed=71, pods_per_cluster=2 if n > 1000 else 16, groups=1 if n > 1000 else 2, wtd_group_frac=0.0)
    if event == "large":
        synthetic.grow_clusters(snap, [50], 300)
    dr = _driver(snap, flags, large_clusters=event == "large", max_creates=1 << 16)  # (renamed groups leave their Pods in no group)
    try:
        dr.check(oracle_mod, expect_incremental=None)
        dr.check(oracle_mod, expect_incremental=None if event == "large" else True)
        if event == "option_off":
            dr.eng.set_group_edits(False)
        fresh = _fresh_id(snap)
        if event == "over_the_cap":  # 4 100 RayClusters renamed their group
            new = synthetic.regroup_clusters(snap, {c: [(int(snap.c_group_off[c]), fresh)] for c in range(4100)})
        else:
            new = synthetic.regroup_clusters(snap, {50: _groups(snap, 50) + [(int(snap.c_group_off[50]), fresh)]})
        _epoch(dr, new)
        if event == "recounted_in_the_same_epoch":  # a second object commit that regroups again: the maps are not composed
            _epoch(dr, synthetic.regroup_clusters(new, {60: _groups(new, 60)[:1]}))
        dr.prev = None
        dr.check(oracle_mod, expect_incremental=False)
        if event == "option_off":
            dr.eng.set_group_edits(True)
        rows = np.arange(3, dr.snap.dims["pods"], 41, dtype=np.uint32)
        flip_ready(dr.snap, rows)
        dr.commit_rows(rows)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


def test_option_off_twin(oracle_mod):
    """The same edit epochs with the option off: full passes, and records identical to the option-on engine's."""
    snap, flags = _fleet(260, seed=72, wtd_group_frac=0.3)
    on, off = _driver(snap, flags), _driver(snap, flags)
    off.eng.set_group_edits(False)
    try:
        for dr in (on, off):
            dr.check(oracle_mod, expect_incremental=False)
        for step, c in enumerate((3, 130, 259)):
            old = on.snap
            g0 = int(old.c_group_off[c])
            pairs = _groups(old, c) + [(g0, _fresh_id(old))] if step != 1 else _groups(old, c)[1:]
            new = synthetic.regroup_clusters(old, {c: pairs})
            _epoch(on, new)
            _epoch(off, copy.deepcopy(new))
            got, _ = _check(on, oracle_mod, old, [c])
            twin, _ = off.check(oracle_mod, expect_incremental=False)
            d = twin.diff(got)
            assert not d, d[:6]
    finally:
        on.close()
        off.close()


def test_transfer_size(oracle_mod):
    """An edit epoch moves the object part plus the row map (the regrouped rows twice, 4 B per shifted group and per shifted name),
    no spec JSON, and hashes nothing."""
    snap, flags = _fleet(400, seed=81, wtd_group_frac=0.3)
    dr = _driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        dr.commit_objects()  # an object part that changed nothing: the baseline
        objects_h2d = dr.eng.last_profile()["h2d_bytes"]
        dr.check(oracle_mod, expect_incremental=True)
        c = 150
        new = synthetic.regroup_clusters(snap, {c: _groups(snap, c) + [(int(snap.c_group_off[c]), _fresh_id(snap))]})
        dr.use(new)
        dr.commit_objects()
        h2d = dr.eng.last_profile()["h2d_bytes"]
        g0 = int(new.c_group_off[c])
        shifted = (new.dims["groups"] - g0) + (new.dims["wtd"] - int(new.g_wtd_off[g0]))
        assert h2d <= objects_h2d + 4 * (2 + shifted) + 5 * 16, (h2d, objects_h2d, shifted)
        assert h2d < objects_h2d + new.dims["json"] // 2
        _, names = _check(dr, oracle_mod, snap, [c], profiled=True)
        assert "k_hash" not in names and "k_hash_rows" not in names, names
    finally:
        dr.close()


def _rayservice_append(m, rng, counter):
    """A RayService in-place update: one RayCluster gets a worker group appended (a copy of its last, or a fresh one), a new
    generation and a re-emitted spec; sometimes one of its groups is removed instead."""
    keys = sorted(m.clusters)
    key = keys[int(rng.integers(len(keys)))]
    c = copy.deepcopy(m.clusters[key])
    groups = c["spec"].setdefault("workerGroupSpecs", [])
    counter[0] += 1
    if groups and rng.random() < 0.25:
        gone = groups.pop(int(rng.integers(len(groups))))
        (c.get("expectations") or {}).pop(gone["groupName"], None)
    else:
        g = copy.deepcopy(groups[-1]) if groups else {"groupName": "", "replicas": 1, "minReplicas": 0, "maxReplicas": 5, "numOfHosts": 1}
        g["groupName"] = f"added-{counter[0]}"
        g["workersToDelete"] = []
        groups.append(g)
        c.setdefault("expectations", {"head": True})[g["groupName"]] = True
    c["generation"] = c.get("generation", 1) + 1
    c["resourceVersion"] = 70_000 + counter[0]
    c["specJson"] = bytes(c.get("specJson") or b"") + f"/g{counter[0]}".encode()
    m.upsert_cluster(c)


def test_packer_stream_against_option_off(oracle_mod):
    """The native packer: RayService-style appends (and removals) mixed with ordinary informer events, against a twin packer with the
    option off.  Edit flushes stay incremental and send their specs as spec rows."""
    caps = dict(PACKER_CAPS, max_clusters=128, max_groups=2048, max_wtd=1024, max_pods=8192, max_jobs=256, max_creates=1 << 20)
    on, off = Packer(**caps, group_edits=True, wtd_edits=True), Packer(**caps, wtd_edits=True)
    try:
        objs = objects(5)
        m_on, m_off = Mirror(*copy.deepcopy(objs), on), Mirror(*copy.deepcopy(objs), off)
        rng_on, rng_off = np.random.default_rng(13), np.random.default_rng(13)
        c_on, c_off = [0], [0]
        n_edit = n_inc = n_json = 0
        for epoch in range(120):
            u = rng_on.random()
            rng_off.random()
            if u >= 0.4:
                events(rng_on, m_on, c_on, structural=False)
                events(rng_off, m_off, c_off, structural=False)
            editing = u < 0.6 and epoch > 0
            if editing:
                _rayservice_append(m_on, rng_on, c_on)
                _rayservice_append(m_off, rng_off, c_off)
            mode = on.flush()
            off.flush()
            _, got = packer_check(m_on, oracle_mod, lean=True)
            _, twin = packer_check(m_off, oracle_mod, lean=True)
            assert np.array_equal(got.clusters, twin.clusters)
            if editing:
                n_edit += 1
                n_inc += incremental(got, got.clusters.shape[0])
                n_json += bool(mode & abi.PART_JSON)  # (only a flush that compacts the JSON arena sends it)
        print(f"edit epochs {n_edit}, incremental {n_inc}, with KR_PART_JSON {n_json}")
        assert n_edit > 40 and n_inc > n_edit * 3 // 4 and n_json * 10 <= n_edit, (n_edit, n_inc, n_json)
    finally:
        on.close()
        off.close()


def test_group_packer_two_shards_one_device(oracle_mod):
    caps = dict(PACKER_CAPS, max_clusters=128, max_groups=2048, max_wtd=1024, max_pods=8192, max_jobs=256)
    gp = GroupPacker([0, 0], **caps, group_edits=True)
    try:
        assert all(sh.engine.get_option(abi.OPT_GROUP_EDITS) == 1 for sh in gp.shards)
        clusters, pods, jobs = objects(7)
        for c in clusters:
            gp.upsert_cluster(c)
        for p in pods:
            gp.upsert_pod(p)
        gp.flush()
        flags = gp.flags(fetch_pod_lists=0)
        gp.reconcile(flags)
        rng = np.random.default_rng(3)
        live = {(c.get("namespace", "default"), c["name"]): c for c in clusters}
        n_inc, epochs = 0, 12
        for epoch in range(epochs):
            key = sorted(live)[int(rng.integers(len(live)))]
            c = copy.deepcopy(live[key])
            groups = c["spec"].setdefault("workerGroupSpecs", [])
            g = copy.deepcopy(groups[-1]) if groups else {"groupName": "", "replicas": 1, "minReplicas": 0, "maxReplicas": 5, "numOfHosts": 1}
            g["groupName"], g["workersToDelete"] = f"added-{epoch}", []
            groups.append(g)
            c["generation"] = c.get("generation", 1) + 1
            c["specJson"] = bytes(c.get("specJson") or b"") + f"/g{epoch}".encode()
            live[key] = c
            sh_edit = gp.shard_of(*key)
            gp.upsert_cluster(c)
            gp.flush()
            got = gp.reconcile(flags)
            n_inc += incremental(got[sh_edit], got[sh_edit].clusters.shape[0])
            for sh, g_res, f in zip(gp.shards, got, flags):
                sh.engine.set_incremental(False)
                full = sh.engine.reconcile(f)
                sh.engine.set_incremental(True)
                d = full.diff(g_res)
                assert not d, (epoch, d[:6])
            gp.reconcile(flags)  # (the full pass above left the resident state: the next edit is incremental again)
        # (an edit re-reserves the RayCluster's action and create places: now and then a cursor passes its arena's end, and that
        # epoch takes the full pass)
        assert n_inc >= epochs * 2 // 3, (n_inc, epochs)
    finally:
        gp.close()

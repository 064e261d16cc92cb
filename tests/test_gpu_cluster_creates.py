"""KR_OPT_CLUSTER_CREATES: RayClusters appended after the last row, and RayJobs created or deleted, keep the device-side incremental
epoch.  The next pass hashes only the new specs, moves the resident Pods labelled for the new RayClusters out of the orphans
(k_inc_orphan_adopt), inserts the RayClusters into the resident tables (k_inc_clusters_insert) and returns them among the changed
records.

A fleet is generated whole; the snapshot before a creation epoch is its prefix of RayClusters (with their groups and names), so the
RayClusters past the prefix are the ones the epoch appends.  Their Pods are either free rows before the epoch or already resident
(then they are orphans until their RayCluster appears).  Every epoch is compared with the CPU oracle, and the records of the RayClusters
a pass did not name must equal the previous epoch's."""
import copy

import numpy as np
import pytest

from harness import PACKER_CAPS, POD_COLS, Driver, Mirror, device_incremental, events, flip_ready, members, objects, packer_check, with_wtd_lists
from kuberay_b200 import abi, synthetic
from kuberay_b200.packer import GroupPacker, Packer
from kuberay_b200.snapshot import Snapshot

pytestmark = pytest.mark.gpu


def _fleet(n, seed, **kw):
    p = dict(n_clusters=n, pods_per_cluster=16, groups=2, seed=seed)
    p.update(kw)
    return synthetic.generate(synthetic.config("C2", **p))


def _prefix(full, k, free_pods=True, jobs=None, free_from=None):
    return synthetic.first_clusters(full, k, free_from=free_from, jobs=jobs, free_pods=free_pods)


def _select(full, order):
    """The RayClusters `order` of `full` (rows of `full`, in the new row order) with their groups and workersToDelete names laid out in
    that order; the Pods of every other RayCluster become free rows."""
    order = np.asarray(order, dtype=np.int64)
    d = full.dims
    goff, gcnt = full.c_group_off.astype(np.int64), full.c_group_cnt.astype(np.int64)
    groups = np.concatenate([np.arange(goff[c], goff[c] + gcnt[c]) for c in order] + [np.zeros(0, np.int64)])
    names = np.concatenate([np.arange(int(full.g_wtd_off[g]), int(full.g_wtd_off[g] + full.g_wtd_cnt[g])) for g in groups] + [np.zeros(0, np.int64)])
    out = Snapshot(order.size, groups.size, names.size, d["pods"], d["heads"], d["jobs"], d["json"])
    rows = {"clusters": order, "groups": groups, "wtd": names}
    for name, _dt, mult, dim in abi.COLUMNS:
        src = full.cols[name]
        out.cols[name][:] = (src.reshape(-1, mult)[rows[dim]].reshape(-1) if mult > 1 else src[rows[dim]]) if dim in rows else src
    cnt = gcnt[order]
    out.c_group_off[:] = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.uint32)
    out.g_cluster_idx[:] = np.repeat(np.arange(order.size), cnt).astype(np.uint32)
    out.g_wtd_off[:] = np.concatenate([[0], np.cumsum(out.g_wtd_cnt)[:-1]]).astype(np.uint32) if groups.size else 0
    gone = np.concatenate([members(full, c) for c in sorted(set(range(d["clusters"])) - set(order.tolist()))] + [np.zeros(0, np.int64)])
    for c in POD_COLS:
        out.cols[c][gone.astype(np.int64)] = 0
    out.p_packed[gone.astype(np.int64)] = np.uint32(abi.PP_TOMBSTONE)
    return out.validate()


def _driver(before, flags, full, **opts):
    """A Driver on `before` with room for `full` (the capacities are taken from the larger of the two)."""
    dr = Driver(full, flags, slack=1.25, cluster_creates=True, **opts)
    dr.use(before)
    dr.commit_objects(abi.PART_ALL)
    for c in POD_COLS:
        dr.views[c][:] = before.cols[c]
    dr.eng.commit(abi.PART_ALL)
    return dr


def _create(dr, new, pods=True):
    """Commit the creation epoch of snapshot `new` (a superset of dr.snap): begin, the object part, the new specs as spec rows,
    and, with `pods`, the pod rows that differ.  -> the new RayCluster rows."""
    old_nc = dr.snap.dims["clusters"]
    changed = np.flatnonzero(np.any([dr.snap.cols[c] != new.cols[c] for c in POD_COLS], axis=0))
    dr.use(new)
    dr.commit_objects()
    np.copyto(dr.views["json"], new.json)
    added = np.arange(old_nc, new.dims["clusters"], dtype=np.uint32)
    if added.size:
        dr.eng.commit_spec_rows(added)
    if pods and changed.size:
        dr.commit_rows(changed)
    return added


def _check(dr, oracle, expect_incremental, profiled=False):
    """Driver.check across a change of the RayCluster count: the records of the RayClusters that stayed are compared with the
    previous epoch's here when the pass did not name them."""
    prev, old_nc = dr.prev, (dr.prev.clusters.shape[0] if dr.prev is not None else 0)
    dr.prev = None
    got, names = dr.check(oracle, expect_incremental=expect_incremental, profiled=profiled)
    if expect_incremental and prev is not None:
        n = min(old_nc, got.clusters.shape[0])
        same = np.ones(n, dtype=bool)
        ch = got.changed_clusters[got.changed_clusters < n] if got.changed_clusters is not None else []
        same[ch] = False
        assert np.array_equal(got.clusters[:n][same], prev.clusters[:n][same])
        assert np.array_equal(got.act_cnt[:n][same], prev.act_cnt[:n][same])
        ng = int(prev.groups.shape[0])
        gs = same[np.minimum(dr.snap.g_cluster_idx[:ng], n - 1)] & (dr.snap.g_cluster_idx[:ng] < n)  # old groups of the RayClusters not named
        assert np.array_equal(got.groups[:ng][gs], prev.groups[gs])
    return got, names


@pytest.mark.parametrize("k", [1, 7, 300])
@pytest.mark.parametrize("pods", ["none", "same_epoch", "later_epoch"])
def test_plain_appends(k, pods, oracle_mod):
    full, flags = _fleet(400 + k, seed=k)
    before = _prefix(full, 400)
    dr = _driver(before, flags, full)
    try:
        _check(dr, oracle_mod, expect_incremental=False)
        target = _prefix(full, 400 + k, free_from=400) if pods == "none" else full
        added = _create(dr, target, pods=pods == "same_epoch")
        if pods == "later_epoch":  # the creation epoch carries no Pod: the new RayClusters are decided with none
            dr.snap = _prefix(full, 400 + k, free_from=400)
        orphans = dr.prev.n_orphans
        got, names = _check(dr, oracle_mod, expect_incremental=True, profiled=True)
        assert set(added.tolist()) <= set(got.changed_clusters.tolist())
        assert "k_inc_clusters_insert" in names and "k_hash_rows" in names and "k_hash" not in names, names
        assert ("k_inc_orphan_adopt" in names) == (orphans > 0), (orphans, names)
        if pods == "later_epoch":
            dr.use(full)
            dr.commit_rows(np.flatnonzero(np.any([dr.views[c] != full.cols[c] for c in POD_COLS], axis=0)))
            got, _ = _check(dr, oracle_mod, expect_incremental=True)
            assert set(added.tolist()) <= set(got.changed_clusters.tolist())
        rows = np.arange(5, full.dims["pods"], 89, dtype=np.uint32)  # an ordinary epoch afterwards
        flip_ready(dr.snap, rows)
        dr.commit_rows(rows)
        _check(dr, oracle_mod, expect_incremental=True)
    finally:
        dr.close()


@pytest.mark.parametrize("case", ["resident_orphans", "orphaned_incrementally", "orphan_edited", "recreated"])
def test_orphan_adoption(case, oracle_mod):
    full, flags = _fleet(208, seed=21)
    before = _prefix(full, 200, free_pods=case != "orphaned_incrementally")
    if case in ("resident_orphans", "orphan_edited", "recreated"):
        before = _prefix(full, 200, free_pods=False)
    dr = _driver(before if case != "recreated" else full, flags, full)
    try:
        _check(dr, oracle_mod, expect_incremental=False)
        if case == "orphaned_incrementally":  # the Pods arrive one epoch before their RayClusters: orphans of an incremental epoch
            target = _prefix(full, 200, free_pods=False)
            dr.use(target)
            dr.commit_rows(np.flatnonzero(np.any([dr.views[c] != target.cols[c] for c in POD_COLS], axis=0)))
            got, _ = _check(dr, oracle_mod, expect_incremental=True)
            assert got.n_orphans > 0
        if case == "recreated":  # RayClusters deleted (a full pass) and created again under the same names meet their old Pods
            gone = _prefix(full, 200, free_pods=False)
            dr.use(gone)
            dr.commit_objects()
            got, _ = _check(dr, oracle_mod, expect_incremental=False)
            assert got.n_orphans > 0
        new = copy.deepcopy(full)
        if case == "orphan_edited":
            r = members(full, 203)[1:3]
            flip_ready(new, r)
        added = _create(dr, new)
        got, names = _check(dr, oracle_mod, expect_incremental=True, profiled=True)
        assert "k_inc_orphan_adopt" in names, names
        assert set(added.tolist()) <= set(got.changed_clusters.tolist())
    finally:
        dr.close()


def test_recreate_gated_and_first_multihost(oracle_mod):
    full, flags = _fleet(260, seed=31, recreate_frac=0.2, multihost_frac=0.05)
    mh = [c for c in range(260) if (full.g_num_hosts[int(full.c_group_off[c]):int(full.c_group_off[c] + full.c_group_cnt[c])] > 1).any()]
    rc = np.flatnonzero(full.c_flags & abi.CF_UPGRADE_RECREATE)
    assert mh and rc.size
    k = min(mh[0], int(rc.max()))
    assert k > 20
    dr = _driver(_prefix(full, k, free_pods=False), flags, full)
    try:
        _check(dr, oracle_mod, expect_incremental=False)
        _create(dr, full)
        got, names = _check(dr, oracle_mod, expect_incremental=True, profiled=True)
        assert "k_inc_mark_rows" in names and "k_hash_rows" in names, names
    finally:
        dr.close()


def test_wide_with_option_large_and_overflow(oracle_mod):
    full, flags = _fleet(120, seed=41)
    wide = synthetic.widen_clusters(full, [119], 40)
    dr = _driver(_prefix(wide, 119), flags, wide, wide_clusters=True)
    try:
        _check(dr, oracle_mod, expect_incremental=False)
        _create(dr, wide)
        _check(dr, oracle_mod, expect_incremental=True)
    finally:
        dr.close()
    grown, flags = _fleet(300, seed=42)
    synthetic.grow_clusters(grown, [299], 200)  # its orphans outgrow the 64-pod stride once adopted
    for opts, inc in (({}, False), ({"large_clusters": True}, None)):
        dr = _driver(_prefix(grown, 299, free_pods=False), flags, grown, **opts)
        try:
            _check(dr, oracle_mod, expect_incremental=False)
            _create(dr, grown)
            _check(dr, oracle_mod, expect_incremental=inc)
        finally:
            dr.close()


@pytest.mark.parametrize("other", ["pod_events", "spec_rows", "wtd_edits", "job_created", "job_deleted", "two_commits", "new_names"])
def test_creation_with_other_events(other, oracle_mod):
    full, flags = _fleet(205, seed=51, jobs=True, wtd_group_frac=0.3)
    if other == "new_names":  # two created RayClusters name resident Pods of theirs (orphans until now) in workersToDelete
        lists = [full.w_name_id[int(o):int(o + n)].tolist() for o, n in zip(full.g_wtd_off, full.g_wtd_cnt)]
        for c in (201, 203):
            lists[int(full.c_group_off[c])] += full.p_name_id[members(full, c)[1:3]].tolist()
        full = with_wtd_lists(full, lists)
    nj = full.dims["jobs"]
    assert nj >= 2
    jobs_before = np.arange(nj - 1) if other == "job_created" else None
    before = _prefix(full, 200, jobs=jobs_before, free_pods=other != "new_names")
    assert before.dims["wtd"] < full.dims["wtd"] or other != "new_names"
    dr = _driver(before, flags, full, wtd_edits=other == "wtd_edits")
    try:
        _check(dr, oracle_mod, expect_incremental=False)
        new = copy.deepcopy(full)
        if other == "job_deleted":
            new = _prefix(full, 205, free_pods=False, jobs=np.arange(1, nj))
        if other == "pod_events":
            flip_ready(new, np.arange(3, 200 * 16, 61))
        if other == "wtd_edits":
            g = next(g for g in range(int(new.c_group_off[200])) if new.g_wtd_cnt[g])
            new.w_name_id[int(new.g_wtd_off[g])] = 0x7FFE0001
        if other == "spec_rows":
            c = 17
            body = bytearray(new.json[int(new.c_json_off[c]):int(new.c_json_off[c] + new.c_json_len[c])].tobytes())
            body[-2:-1] = b" "
            new.json[int(new.c_json_off[c]):int(new.c_json_off[c] + new.c_json_len[c])] = np.frombuffer(bytes(body), np.uint8)
            np.copyto(dr.views["json"][:new.dims["json"]], new.json)
            dr.eng.commit_spec_rows(np.array([c], dtype=np.uint32))
        if other == "two_commits":  # two object commits of one epoch that both append RayClusters
            _create(dr, _prefix(full, 202))
        _create(dr, new)
        _, names = _check(dr, oracle_mod, expect_incremental=True, profiled=True)
        assert "k_inc_clusters_insert" in names, names
        if other == "new_names":  # the new names are inserted and resolved; the name table is not rebuilt
            assert "k_inc_wtd_resolve" in names and "k_inc_wtd_clear" not in names, names
    finally:
        dr.close()


@pytest.mark.parametrize("event", ["deletion_with_creation", "group_added", "shrink"])
def test_still_full_passes(event, oracle_mod):
    full, flags = _fleet(204, seed=61)
    before = _prefix(full, 203)
    dr = _driver(before, flags, full)
    try:
        _check(dr, oracle_mod, expect_incremental=False)
        if event == "deletion_with_creation":
            # RayCluster 5 deleted (the last row moves into its hole, as the native packer does) and RayCluster 203 created in the
            # same epoch: the count stays, and the keys of row 5 change below the resident rows
            order = list(range(203))
            order[5] = 202
            order[202] = 203
            _create(dr, _select(full, order))
        elif event == "shrink":
            _create(dr, _prefix(full, 201))
        else:  # a worker group added to RayCluster 3 (every later group row moves)
            wide = _prefix(synthetic.widen_clusters(full, [3], 2), 203)
            changed = np.flatnonzero(np.any([dr.snap.cols[c] != wide.cols[c] for c in POD_COLS], axis=0))
            dr.use(wide)
            dr.commit_objects()
            dr.commit_rows(changed)
        _check(dr, oracle_mod, expect_incremental=False)
        _check(dr, oracle_mod, expect_incremental=True)  # (the full pass left the resident state: the next epoch is incremental)
    finally:
        dr.close()


def test_option_off_twin(oracle_mod):
    """The same creation epochs with the option off: full passes, and records identical to the option-on engine's."""
    full, flags = _fleet(212, seed=62)
    before = _prefix(full, 200, free_pods=False)
    on, off = _driver(before, flags, full), _driver(before, flags, full)
    off.eng.set_cluster_creates(False)
    try:
        for dr in (on, off):
            _check(dr, oracle_mod, expect_incremental=False)
        for k, inc in ((206, True), (212, True)):
            target = _prefix(full, k, free_pods=False)
            a = _create(on, target)
            b = _create(off, target)
            assert np.array_equal(a, b)
            got, _ = _check(on, oracle_mod, expect_incremental=inc)
            twin, _ = _check(off, oracle_mod, expect_incremental=False)
            d = twin.diff(got)
            assert not d, d[:6]
    finally:
        on.close()
        off.close()


def test_transfer_size(oracle_mod):
    full, flags = _fleet(230, seed=71)
    before = _prefix(full, 200)
    dr = _driver(before, flags, full)
    try:
        _check(dr, oracle_mod, expect_incremental=False)
        full = _prefix(full, 230, free_from=200)  # (the new RayClusters' Pods come in a later epoch)
        dr.use(full)
        dr.commit_objects()
        objects = dr.eng.last_profile()["h2d_bytes"]
        np.copyto(dr.views["json"], full.json)
        added = np.arange(200, 230, dtype=np.uint32)
        dr.eng.commit_spec_rows(added)
        specs = sum((int(full.c_json_len[c]) + 15) // 16 * 16 for c in added)
        _, names = _check(dr, oracle_mod, expect_incremental=True, profiled=True)
        h2d = dr.eng.last_profile()["h2d_bytes"]
        assert h2d <= objects + specs + 16 * added.size + 4 * added.size, (h2d, objects, specs)
        assert h2d < objects + full.dims["json"]
        assert "k_hash_rows" in names and "k_hash" not in names, names
    finally:
        dr.close()


def _creating_stream(m, rng, counter, created, deleted):
    """One epoch's informer events: Pod and RayCluster events, or a RayCluster created (with its Pods and maybe a RayJob) and nothing
    else; a created RayCluster is now and then deleted (its Pods stay: orphans) and later created again under its old name, so the
    creation meets its old Pods."""
    mine = sorted(k for k in m.clusters if "-c" in k[1])
    u = rng.random()
    if u >= 0.55:
        events(rng, m, counter, structural=False)
    if u < 0.1 and mine:
        key = mine[int(rng.integers(len(mine)))]
        deleted[key] = m.clusters[key]
        m.delete_cluster(*key)
        created.append(None)
    elif u < 0.25 and deleted:
        key = sorted(deleted)[int(rng.integers(len(deleted)))]
        c = deleted.pop(key)
        counter[0] += 1
        c = dict(c, resourceVersion=90_000 + counter[0])
        m.upsert_cluster(c)
        created.append(key)
    elif u < 0.55:
        src = copy.deepcopy(m.clusters[sorted(m.clusters)[int(rng.integers(len(m.clusters)))]])
        counter[0] += 1
        name = f"{src['name']}-c{counter[0]}"
        src["name"], src["generation"], src["resourceVersion"] = name, 1, 50_000 + counter[0]
        m.upsert_cluster(src)
        ns = src.get("namespace", "default")
        for i in range(int(rng.integers(0, 4))):
            m.upsert_pod({"namespace": ns, "name": f"{name}-w{i}", "labels": {"ray.io/cluster": name, "ray.io/node-type": "worker",
                          "ray.io/group": (src["spec"].get("workerGroupSpecs") or [{"groupName": "g"}])[0]["groupName"]},
                          "phase": "Running", "conditions": [{"type": "Ready", "status": "True"}], "restartPolicy": "Always"})
        if rng.random() < 0.5:
            m.upsert_job({"namespace": ns, "name": f"job-{name}", "status": {"rayClusterName": name, "rayClusterStatus": src.get("status")}})
        created.append((ns, name))
    elif m.jobs and u < 0.6:
        j = m.jobs[int(rng.integers(len(m.jobs)))]
        m.delete_job(j.get("namespace", "default"), j["name"])


def test_packer_stream_against_option_off(oracle_mod):
    caps = dict(PACKER_CAPS, max_clusters=160, max_groups=1024, max_wtd=1024, max_pods=8192, max_jobs=256, max_creates=1 << 20)
    on, off = Packer(**caps, cluster_creates=True), Packer(**caps)
    try:
        objs = objects(5)
        m_on, m_off = Mirror(*copy.deepcopy(objs), on), Mirror(*copy.deepcopy(objs), off)
        rng_on, rng_off = np.random.default_rng(9), np.random.default_rng(9)
        c_on, c_off, d_on, d_off = [0], [0], {}, {}
        n_inc = n_create = n_adopt = 0
        for epoch in range(300):
            created = []
            if len(m_on.clusters) < caps["max_clusters"] - 4:
                _creating_stream(m_on, rng_on, c_on, created, d_on)
                _creating_stream(m_off, rng_off, c_off, [], d_off)
            orphans_before = on.engine.fetch().n_orphans if epoch else 0
            stride = on.engine.get_option(abi.OPT_BUCKET_STRIDE)
            mode = on.flush()
            off.flush()
            assert not (mode & abi.PART_JSON) or not created or None in created or epoch == 0, (epoch, mode)
            _, got = packer_check(m_on, oracle_mod, lean=True)
            _, twin = packer_check(m_off, oracle_mod, lean=True)
            assert np.array_equal(got.clusters, twin.clusters)
            if len(created) == 1 and created[0] and epoch:  # a creation-only epoch (no RayCluster deleted)
                n_create += 1
                key = created[0]
                n_pods = sum(1 for p in m_on.live_pods() if (p.get("namespace", "default"), (p.get("labels") or {}).get("ray.io/cluster")) == key)
                if n_pods <= stride:  # (a RayCluster of more Pods than the bucket holds takes the full pass, which reclassifies)
                    n_inc += 1
                    assert got.changed_clusters is not None, (epoch, key, n_pods, stride)
                n_adopt += orphans_before > got.n_orphans
        assert n_inc > 50 and n_adopt > 5, (n_inc, n_create, n_adopt)
    finally:
        on.close()
        off.close()


def test_group_packer_two_shards_one_device(oracle_mod):
    """The option set per shard (kr_packer_engine of kr_group_packer_shard): RayClusters created on both shards of one device; each
    shard's incremental pass equals a full pass of its engine over the same state."""
    caps = dict(PACKER_CAPS, max_clusters=128, max_groups=1024, max_wtd=1024, max_pods=8192, max_jobs=256)
    gp = GroupPacker([0, 0], **caps, cluster_creates=True)
    try:
        assert all(sh.engine.get_option(abi.OPT_CLUSTER_CREATES) == 1 for sh in gp.shards)
        clusters, pods, jobs = objects(7)
        for c in clusters:
            gp.upsert_cluster(c)
        for p in pods:
            gp.upsert_pod(p)
        gp.flush()
        flags = gp.flags(fetch_pod_lists=0)
        gp.reconcile(flags)
        rng = np.random.default_rng(3)
        grew = [0] * gp.n
        for epoch in range(16):
            src = copy.deepcopy(clusters[int(rng.integers(len(clusters)))])
            src["name"], src["generation"], src["resourceVersion"] = f"{src['name']}-g{epoch}", 1, 70_000 + epoch
            gp.upsert_cluster(src)
            gp.flush()
            got = gp.reconcile(flags)
            sh_new = gp.shard_of(src.get("namespace", "default"), src["name"])
            grew[sh_new] += 1
            row = gp.shards[sh_new].cluster_row(src.get("namespace", "default"), src["name"])
            assert got[sh_new].changed_clusters is not None and row in got[sh_new].changed_clusters.tolist(), (epoch, sh_new)
            for sh, g, f in zip(gp.shards, got, flags):
                sh.engine.set_incremental(False)
                full = sh.engine.reconcile(f)
                sh.engine.set_incremental(True)
                d = full.diff(g)
                assert not d, (epoch, d[:6])
            gp.reconcile(flags)  # (the full pass above left the resident state: the next creation is incremental again)
        assert min(grew) > 0, grew  # (both shards created RayClusters)
    finally:
        gp.close()

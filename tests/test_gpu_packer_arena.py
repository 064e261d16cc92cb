"""The native packer's muted-spec JSON arena through its whole lifecycle: compaction inside an upsert (a re-emitted spec no longer
fits), compaction at flush (more than 1 MiB and more than half of the arena dead), compaction in the same epoch as a table that
changes shape, RayCluster deletion (the last row moves into the hole) and an arena too small even after compaction.

A compaction re-places every RayCluster's blob, so every c_json_off moves, while the epoch's object rows may still go row by row
(kr_snapshot_commit_object_rows of the edited RayClusters only).  Every epoch is checked against the oracle on an independently
packed snapshot (packer_check, digests included) and directly: each RayCluster's digest must be the base32hex SHA-1 of its
current specJson (passed verbatim, so sizes are exact), and the Recreate-gated RayClusters, whose head Pods carry the digest of their
spec and which are never edited, must stay on PATH_NORMAL: a digest computed from a stale range would delete all their Pods."""
import copy

import numpy as np
import pytest

from harness import L_CLUSTER, L_GROUP, L_TYPE, Mirror, b32, packer_check, spec_bytes
from kuberay_b200 import abi, synthetic
from kuberay_b200 import snapshot as snp
from kuberay_b200.engine import Engine, EngineError
from kuberay_b200.packer import Packer

pytestmark = pytest.mark.gpu

NS = "arena"


def _pad(n: int) -> int:
    return (n + 15) // 16 * 16


def _body(rng, n: int) -> bytes:
    return bytes(rng.integers(32, 127, size=n, dtype=np.uint8))


def _head(name, body: bytes, head_no=0):
    return {"namespace": NS, "name": f"{name}-head{head_no or ''}", "labels": {L_CLUSTER: name, L_TYPE: "head", L_GROUP: "headgroup"},
            "annotations": {snp.RECREATE_HASH_ANNOT: b32(body).decode(), snp.KUBERAY_VERSION_ANNOT: snp.KUBERAY_VERSION},
            "phase": "Running", "conditions": [{"type": "Ready", "status": "True"}], "podIP": "10.1.0.1", "restartPolicy": "Always"}


def _worker(name, k):
    return {"namespace": NS, "name": f"{name}-w{k}", "labels": {L_CLUSTER: name, L_TYPE: "worker", L_GROUP: "g0"}, "phase": "Running",
            "conditions": [{"type": "Ready", "status": "True"}], "restartPolicy": "Always"}


def _cluster(i, body: bytes, gated: bool):
    name = f"rc{i}"
    spec = {"workerGroupSpecs": [{"groupName": "g0", "replicas": 2, "minReplicas": 0, "maxReplicas": 4, "numOfHosts": 1}]}
    if gated:
        spec["upgradeStrategy"] = {"type": "Recreate"}
    if i == 1:  # (a list to rename in place)
        spec["workerGroupSpecs"][0]["workersToDelete"] = [f"{name}-w0"]
    return {"namespace": NS, "name": name, "uid": f"uid-{name}", "generation": 1, "resourceVersion": 100 + i, "spec": spec,
            "specJson": body, "status": {}, "expectations": {"head": True, "g0": True}}


def _fleet(rng, n, size):
    """n healthy RayClusters (a head Pod and two workers each); every third one Recreate-gated, its head Pod annotated with the
    digest of its spec.  size(i) -> the length of RayCluster i's specJson."""
    clusters, pods = [], []
    for i in range(n):
        c = _cluster(i, _body(rng, size(i)), gated=i % 3 == 0)
        clusters.append(c)
        pods += [_head(c["name"], c["specJson"])] + [_worker(c["name"], k) for k in range(2)]
    return clusters, pods


def _gated(m):
    return [k for k, c in m.clusters.items() if (c["spec"].get("upgradeStrategy") or {}).get("type") == "Recreate"]


def _editable(m):
    return sorted(k for k in m.clusters if k not in set(_gated(m)))


def _respec(m, key, body: bytes):
    c = copy.deepcopy(m.clusters[key])
    c["specJson"] = body
    c["generation"] += 1
    c["resourceVersion"] += 1
    m.upsert_cluster(c)


def _pod_status(rng, m, k):
    """k status updates of worker Pods (Ready flips): pod rows only."""
    workers = [p for p in m.live_pods() if p["labels"].get(L_TYPE) == "worker"]
    for i in rng.choice(len(workers), min(k, len(workers)), replace=False):
        p = copy.deepcopy(workers[int(i)])
        p["conditions"] = [{"type": "Ready", "status": "False" if p["conditions"][0]["status"] == "True" else "True"}]
        m.upsert_pod(p)


def _offsets(m):
    col = m.pk.column("c_json_off")
    return {k: int(col[m.pk.cluster_row(*k)]) for k in m.clusters}


def _verify(m, oracle_mod):
    """Every digest against its specJson and every gated RayCluster on PATH_NORMAL, then packer_check (the same pass again:
    an epoch without commits)."""
    got = m.pk.engine.reconcile(m.pk.flags(fetch_pod_lists=0))
    for key, c in m.clusters.items():
        r = m.pk.cluster_row(*key)
        assert bytes(got.hash[r]) == b32(c["specJson"]), (key, r)
    for key in _gated(m):
        assert got.clusters["path"][m.pk.cluster_row(*key)] == abi.PATH_NORMAL, key
    _, got = packer_check(m, oracle_mod, lean=True)
    return got


def _epoch(m, oracle_mod, events):
    """Apply `events(m)` (-> the RayClusters it re-emitted), flush, verify; -> (mode, whether the arena was compacted)."""
    before = _offsets(m)
    edited = set(events(m))
    mode = m.pk.flush()
    after = _offsets(m)
    compacted = any(before[k] != after[k] for k in before if k in after and k not in edited)
    _verify(m, oracle_mod)
    return mode, compacted


def _packer(cap, spec_rows):
    return Packer(max_clusters=64, max_groups=256, max_wtd=256, max_pods=1024, max_heads=128, max_jobs=16, max_creates=1 << 12,
                  max_json_bytes=cap, spec_rows=spec_rows)


def _start(clusters, pods, cap, spec_rows, oracle_mod):
    pk = _packer(cap, spec_rows)
    m = Mirror(copy.deepcopy(clusters), copy.deepcopy(pods), [], pk)
    assert pk.flush() == abi.PACK_FULL
    _verify(m, oracle_mod)
    return m


def _compaction_mode(mode, spec_rows):
    assert mode & abi.PART_JSON, mode
    assert not mode & abi.PACK_SPEC_ROWS, mode


@pytest.mark.parametrize("spec_rows", [False, True])
def test_compaction_inside_an_upsert(spec_rows, oracle_mod):
    rng = np.random.default_rng(1)
    clusters, pods = _fleet(rng, 24, lambda i: int(rng.integers(1024, 2049)))
    live = sum(_pad(len(c["specJson"])) for c in clusters)
    m = _start(clusters, pods, 2 * live, spec_rows, oracle_mod)
    try:
        n_compacted = 0
        for epoch in range(30):
            def events(m):
                keys = _editable(m)
                edit = [keys[int(i)] for i in rng.choice(len(keys), int(rng.integers(2, 5)), replace=False)]
                for k in edit:
                    _respec(m, k, _body(rng, int(rng.integers(1024, 2049))))
                _pod_status(rng, m, 3)
                return edit
            mode, compacted = _epoch(m, oracle_mod, events)
            assert mode & abi.PACK_OBJECT_ROWS and mode & abi.PACK_POD_ROWS and not mode & abi.PART_OBJECTS, (epoch, mode)
            if compacted:
                n_compacted += 1
                _compaction_mode(mode, spec_rows)
            elif spec_rows:
                assert mode & abi.PACK_SPEC_ROWS and not mode & abi.PART_JSON, (epoch, mode)
        assert n_compacted >= 3, n_compacted
    finally:
        m.pk.close()


@pytest.mark.parametrize("spec_rows", [False, True])
def test_compaction_at_flush(spec_rows, oracle_mod):
    rng = np.random.default_rng(2)
    clusters, pods = _fleet(rng, 12, lambda i: 48 << 10)
    m = _start(clusters, pods, 8 << 20, spec_rows, oracle_mod)
    try:
        seen, epoch = None, 0
        while seen is None or epoch < seen + 3:
            def events(m):
                keys = _editable(m)
                edit = [keys[int(i)] for i in rng.choice(len(keys), int(rng.integers(1, 3)), replace=False)]
                for k in edit:
                    _respec(m, k, _body(rng, int(rng.integers(47 << 10, 49 << 10))))
                _pod_status(rng, m, 2)
                return edit
            mode, compacted = _epoch(m, oracle_mod, events)
            assert mode & abi.PACK_OBJECT_ROWS and not mode & abi.PART_OBJECTS, (epoch, mode)
            if compacted:
                assert seen is None, epoch  # (once the dead bytes are gone it takes another 1 MiB of edits)
                seen = epoch
                _compaction_mode(mode, spec_rows)
                assert m.pk.engine.sizes.json_bytes == sum(_pad(len(c["specJson"])) for c in m.clusters.values())
            epoch += 1
            assert epoch < 40, "no compaction at flush"
    finally:
        m.pk.close()


def _force_compaction(rng, m, cap):
    """Re-emit the largest ungated spec one 16-byte block longer than the room left at the arena's end: the upsert compacts.  Must be
    the epoch's first JSON event (the room is read from the last flush)."""
    key = max(_editable(m), key=lambda k: len(m.clusters[k]["specJson"]))
    n = cap - m.pk.engine.sizes.json_bytes + 16
    live = sum(_pad(len(c["specJson"])) for c in m.clusters.values())
    assert live - _pad(len(m.clusters[key]["specJson"])) + _pad(n) <= cap
    _respec(m, key, _body(rng, n))
    return key


@pytest.mark.parametrize("spec_rows", [False, True])
@pytest.mark.parametrize("what", ["wtd_rename", "head_added", "created", "deleted"])
def test_compaction_with_a_shape_change(what, spec_rows, oracle_mod):
    """The compaction epoch also changes a table (the whole object part travels); the epoch after it carries Pod rows only."""
    rng = np.random.default_rng(3)
    clusters, pods = _fleet(rng, 12, lambda i: int(rng.integers(1024, 2049)))
    cap = sum(_pad(len(c["specJson"])) for c in clusters) + (32 << 10)
    m = _start(clusters, pods, cap, spec_rows, oracle_mod)
    try:
        for rnd in range(2):
            def events(m):
                edited = [_force_compaction(rng, m, cap)]
                if what == "wtd_rename":
                    c = copy.deepcopy(m.clusters[(NS, "rc1")])
                    g = c["spec"]["workerGroupSpecs"][0]
                    g["workersToDelete"] = ["rc1-w1" if g["workersToDelete"] == ["rc1-w0"] else "rc1-w0"]
                    m.upsert_cluster(c)
                    edited.append((NS, "rc1"))
                elif what == "head_added":
                    key = _editable(m)[rnd]
                    m.upsert_pod(_head(key[1], m.clusters[key]["specJson"], head_no=2))
                elif what == "created":
                    c = _cluster(100 + rnd, _body(rng, 300), gated=False)
                    m.upsert_cluster(c)
                    edited.append((NS, c["name"]))
                else:
                    key = [k for k in _editable(m) if k not in edited][0]
                    m.delete_cluster(*key)
                _pod_status(rng, m, 2)
                return edited
            mode, compacted = _epoch(m, oracle_mod, events)
            assert compacted and mode & abi.PART_OBJECTS, (rnd, mode)
            _compaction_mode(mode, spec_rows)
            mode, compacted = _epoch(m, oracle_mod, lambda m: _pod_status(rng, m, 4) or [])
            assert mode == abi.PACK_POD_ROWS and not compacted, mode
    finally:
        m.pk.close()


@pytest.mark.parametrize("spec_rows", [False, True])
def test_cluster_deletion_without_compaction(spec_rows, oracle_mod):
    """kr_packer_cluster_delete moves the last row into the hole: delete the first, a middle and the last row, each with a spec edit
    of another RayCluster in the same epoch (which a moved row sends as KR_PART_JSON)."""
    rng = np.random.default_rng(4)
    clusters, pods = _fleet(rng, 12, lambda i: int(rng.integers(256, 1024)))
    m = _start(clusters, pods, 1 << 20, spec_rows, oracle_mod)
    try:
        prev = _verify(m, oracle_mod)
        for pick in ("first", "middle", "last"):
            rows = {m.pk.cluster_row(*k): k for k in m.clusters}
            n = len(rows)
            gone = rows[{"first": 0, "middle": n // 2, "last": n - 1}[pick]]
            if gone in _gated(m):  # (the gated ones must stay; another row of the same kind)
                gone = rows[{"first": 1, "middle": n // 2 + 1, "last": n - 2}[pick]]
            n_pods = sum(p["labels"][L_CLUSTER] == gone[1] for p in m.live_pods())
            edit = [k for k in _editable(m) if k != gone][-1]
            m.delete_cluster(*gone)
            _respec(m, edit, _body(rng, 700))
            mode = m.pk.flush()
            assert mode & abi.PART_OBJECTS and mode & abi.PART_JSON and not mode & abi.PACK_SPEC_ROWS, (pick, mode)
            assert m.pk.cluster_row(*gone) == -1
            got = _verify(m, oracle_mod)
            assert got.n_orphans == prev.n_orphans + n_pods, (pick, got.n_orphans, prev.n_orphans, n_pods)
            prev = got
    finally:
        m.pk.close()


def test_arena_too_small_even_after_compaction(oracle_mod):
    rng = np.random.default_rng(5)
    clusters, pods = _fleet(rng, 6, lambda i: 1024)
    cap = sum(_pad(len(c["specJson"])) for c in clusters) + 4096
    m = _start(clusters, pods, cap, False, oracle_mod)
    try:
        key = _editable(m)[0]
        c = copy.deepcopy(m.clusters[key])
        c["specJson"], c["generation"] = _body(rng, 1024 + 4096 + 16), c["generation"] + 1
        with pytest.raises(EngineError) as ei:
            m.pk.upsert_cluster(c)
        assert ei.value.code == abi.KR_E_CAPACITY and "exceeds kr_config.max_json_bytes" in str(ei.value), str(ei.value)
    finally:
        m.pk.close()


def test_json_only_commit_then_object_rows(oracle_mod):
    """At the ABI, without the packer: a KR_PART_JSON commit that moves every range, then kr_snapshot_commit_object_rows of ONE
    RayCluster, must still decide every RayCluster from its new range (the row commit takes the whole object part); a JSON commit
    that moves one range, then the row commit of that RayCluster, stays row-granular."""
    snap, flags = synthetic.generate(synthetic.config("C2", n_clusters=300, pods_per_cluster=16, groups=3, recreate_frac=0.2, seed=3))
    flags.fetch_pod_lists = 0
    eng = Engine.for_snapshot(snap, slack=1.25)
    try:
        eng.set_fixed_layout(True)
        v = eng.load(snap)
        first = eng.reconcile(flags)
        assert not oracle_mod.run(snap, flags).diff(first)
        s = snap
        nc = s.dims["clusters"]
        body = lambda c: spec_bytes(s, c)  # noqa: E731
        head_of = {(int(s.p_ns_id[p]), int(s.p_cluster_name_id[p])): h for h, p in enumerate(s.h_pod_idx.tolist())}
        ann = s.h_annot_hash.reshape(-1, 32)
        gated = [c for c in range(nc) if s.c_flags[c] & abi.CF_UPGRADE_RECREATE and first.clusters["path"][c] == abi.PATH_NORMAL and
                 (int(s.c_ns_id[c]), int(s.c_name_id[c])) in head_of and bytes(ann[head_of[(int(s.c_ns_id[c]), int(s.c_name_id[c]))]]) == b32(body(c))]
        assert gated
        plain = [c for c in range(nc) if not s.c_flags[c] & abi.CF_UPGRADE_RECREATE]
        # 1. every range moves: the blobs laid out again starting from RayCluster 1, RayCluster 0 last
        blobs = [body(c) for c in range(nc)]
        old = s.c_json_off.copy()
        s.json[:] = 0
        pos = 0
        for c in list(range(1, nc)) + [0]:
            s.json[pos:pos + len(blobs[c])] = np.frombuffer(blobs[c], dtype=np.uint8)
            s.c_json_off[c] = pos
            pos += _pad(len(blobs[c]))
        assert pos <= s.dims["json"] and (s.c_json_off != old).all()
        np.copyto(v["json"], s.json)
        v["c_json_off"][:] = s.c_json_off
        eng.commit(abi.PART_JSON)
        h_json = eng.last_profile()["h2d_bytes"]
        c = plain[0]
        s.c_old_counts[5 * c] += 1
        v["c_old_counts"][5 * c] = s.c_old_counts[5 * c]
        eng.commit_object_rows([c])
        whole = eng.last_profile()["h2d_bytes"] - h_json
        got = eng.reconcile(flags)
        d = oracle_mod.run(s, flags).diff(got)
        assert not d, d[:6]
        for r in range(nc):
            assert bytes(got.hash[r]) == b32(blobs[r]), r
        assert (got.clusters["path"][gated] == abi.PATH_NORMAL).all()
        # 2. the ordinary spec edit: one range moves (shorter, same offset), the row commit lists its RayCluster
        c = plain[1]
        n = int(s.c_json_len[c]) - 20
        s.json[int(s.c_json_off[c]) + n:int(s.c_json_off[c]) + n + 20] = 0
        s.c_json_len[c] = n
        v["c_json_len"][c] = n
        np.copyto(v["json"], s.json)
        eng.commit(abi.PART_JSON)
        h_json = eng.last_profile()["h2d_bytes"]
        s.c_old_counts[5 * c] += 1
        v["c_old_counts"][5 * c] = s.c_old_counts[5 * c]
        eng.commit_object_rows([c])
        rows = eng.last_profile()["h2d_bytes"] - h_json
        assert 0 < rows and whole > 10 * rows, (rows, whole)  # (8.5 KB against 106 KB on this fleet)
        got = eng.reconcile(flags)
        d = oracle_mod.run(s, flags).diff(got)
        assert not d, d[:6]
        assert bytes(got.hash[c]) == b32(body(c))
        assert (got.clusters["path"][gated] == abi.PATH_NORMAL).all()
    finally:
        eng.close()

"""The group packer (kr_group_packer_*, kuberay_b200/csrc/kr_group_packer.cpp; DESIGN §6): one native packer per shard behind one
handle, events routed by (namespace, RayCluster name), every shard flushed and reconciled on its own worker thread.

Every event goes to the group packer, to one harness.Mirror per shard (the objects routed by kr_shard_of_key, so the oracle
sees each shard's own snapshot) and to a single-device Packer twin.  Each epoch, every shard's view from ONE GroupPacker.reconcile
must equal the oracle on its shard's objects (harness.packer_check), and the shards together must decide every RayCluster exactly as
the twin does.  Each shard reuses its own lowest free Pod row, so List order differs from the twin's: order-dependent choices are
checked only against the shard's own oracle.  The shards share device 0; with several GPUs one more run puts each on its own."""
import copy

import numpy as np
import pytest

from harness import L_CLUSTER, L_GROUP, L_TYPE, PACKER_CAPS, Mirror, events, objects, packer_check
from kuberay_b200 import abi
from kuberay_b200 import snapshot as snp
from kuberay_b200.engine import EngineError, lib
from kuberay_b200.packer import GroupPacker, Packer, shard_of_key

pytestmark = pytest.mark.gpu

NS = "gp"


class _Sink:
    """A shard's Packer view whose event calls do nothing: the shard receives its events through the group packer's routing.
    Reads (flags, rows, strings, columns, the engine) go to the shard."""

    def __init__(self, pk: Packer):
        self._pk = pk

    def __getattr__(self, name):
        return getattr(self._pk, name)

    def upsert_pod(self, *_):
        pass

    delete_pod = upsert_cluster = delete_cluster = upsert_job = delete_job = upsert_pod


def _key(o):
    return (o.get("namespace", "default"), o["name"])


def _job_cluster(j):
    return (j.get("status") or {}).get("rayClusterName") or None


class Router:
    """The informer side: every event goes to the group packer, to the Mirror of the shard kr_shard_of_key names, and to the twin.
    Looks like a LiveArena to harness.events (rows, row_of, clusters, upsert / delete)."""

    def __init__(self, clusters, pods, jobs, gp: GroupPacker, twin: Packer | None):
        self.gp, self.n = gp, gp.n
        self.m = [Mirror([], [], [], _Sink(sh)) for sh in gp.shards]
        self.twin = Mirror([], [], [], twin) if twin is not None else None
        self.clusters = {}
        for c in clusters:
            self.upsert_cluster(c)
        for p in pods:
            self.upsert_pod(p)
        for j in jobs:
            self.upsert_job(j)

    @property
    def rows(self):
        return [p for m in self.m for p in m.rows]

    @property
    def row_of(self):
        return {k: 0 for m in self.m for k in m.row_of}

    def live_pods(self):
        return [p for m in self.m for p in m.live_pods()]

    def upsert_pod(self, pod):
        key = _key(pod)
        s = shard_of_key(key[0], (pod.get("labels") or {}).get(L_CLUSTER), self.n)
        self.gp.upsert_pod(pod)
        for i, m in enumerate(self.m):
            if i != s and key in m.row_of:  # relabelled: it leaves its old shard
                m.delete_pod(*key)
        self.m[s].upsert_pod(pod)  # (asserts the shard gave the Pod the row its Mirror expects)
        if self.twin:
            self.twin.upsert_pod(pod)

    def delete_pod(self, ns, name):
        self.gp.delete_pod(ns, name)
        for m in self.m:
            m.delete_pod(ns, name)
        if self.twin:
            self.twin.delete_pod(ns, name)

    def upsert_cluster(self, c):
        key = _key(c)
        self.clusters[key] = c
        self.gp.upsert_cluster(c)
        self.m[shard_of_key(*key, self.n)].upsert_cluster(c)
        if self.twin:
            self.twin.upsert_cluster(c)

    def delete_cluster(self, ns, name):
        self.clusters.pop((ns, name), None)
        self.gp.delete_cluster(ns, name)
        self.m[shard_of_key(ns, name, self.n)].delete_cluster(ns, name)
        if self.twin:
            self.twin.delete_cluster(ns, name)

    def upsert_job(self, j):
        s = shard_of_key(j.get("namespace", "default"), _job_cluster(j), self.n)
        self.gp.upsert_job(j)
        for i, m in enumerate(self.m):
            if i != s:
                m.delete_job(*_key(j))
        self.m[s].upsert_job(j)
        if self.twin:
            self.twin.upsert_job(j)

    def delete_job(self, ns, name):
        self.gp.delete_job(ns, name)
        for m in self.m:
            m.delete_job(ns, name)
        if self.twin:
            self.twin.delete_job(ns, name)

    # ------------------------------------------------------------------ one epoch, checked
    def epoch(self, oracle_mod, lean: bool, twin=True):
        """flush, ONE GroupPacker.reconcile, then every shard against its oracle, the jobs, the placement and the twin."""
        modes = self.gp.flush()
        res = self.gp.reconcile(self.gp.flags(fetch_pod_lists=0 if lean else 1))
        for i, m in enumerate(self.m):
            want, _ = packer_check(m, oracle_mod, lean, run=lambda _f, i=i: res[i])
            _check_jobs(m, want, res[i])
        self.check_placement()
        if twin and self.twin is not None:
            self.twin.pk.flush()
            tw = self.twin.pk.engine.reconcile(self.twin.pk.flags(fetch_pod_lists=0 if lean else 1))
            self.check_twin(res, tw)
            return modes, res, tw
        return modes, res, None

    def check_placement(self):
        """Every RayCluster on exactly one shard (its key's), every Pod on exactly one (its label's), every RayJob on one."""
        for key in self.clusters:
            rows = [sh.cluster_row(*key) for sh in self.gp.shards]
            assert [i for i, r in enumerate(rows) if r >= 0] == [shard_of_key(*key, self.n)], (key, rows)
        for p in self.live_pods():
            key = _key(p)
            rows = [sh.pod_row(*key) for sh in self.gp.shards]
            assert [i for i, r in enumerate(rows) if r >= 0] == [shard_of_key(key[0], (p.get("labels") or {}).get(L_CLUSTER), self.n)], (key, rows)
        assert [int(sh.engine.sizes.n_jobs) for sh in self.gp.shards] == [len(m.jobs) for m in self.m]

    def check_twin(self, res, tw):
        """The shards together decide every RayCluster as the single-device twin does (order-free fields)."""
        t = self.twin.pk
        assert sum(int(r.n_orphans) for r in res) == int(tw.n_orphans)
        assert sum(int(r.n_actions) for r in res) == int(tw.n_actions) and sum(int(r.n_create_total) for r in res) == int(tw.n_create_total)
        t_off = t.column("c_group_off")
        for key, c in self.clusters.items():
            s = shard_of_key(*key, self.n)
            sh = self.gp.shards[s]
            r, q = sh.cluster_row(*key), t.cluster_row(*key)
            a, b = res[s].clusters[r], tw.clusters[q]
            for f in ("path", "head_action", "err_kind", "status_err", "new_state", "counts", "cond_status", "cond_variant", "n_pods", "n_heads"):
                assert np.array_equal(a[f], b[f]), (key, f, a[f], b[f])
            assert bytes(res[s].hash[r]) == bytes(tw.hash[q]), key
            assert int(res[s].act_cnt[r]) == int(tw.act_cnt[q]), key
            g0, h0 = int(sh.column("c_group_off")[r]), int(t_off[q])
            for gi in range(int(sh.column("c_group_cnt")[r])):
                for f in ("expected", "n_list", "n_unhealthy", "n_running", "diff", "n_create", "flags"):
                    assert res[s].groups[g0 + gi][f] == tw.groups[h0 + gi][f], (key, gi, f)


def _check_jobs(m: Mirror, want, got):
    """RayJob roll-ups: the same records by RayCluster key (the two sides number jobs and clusters differently)."""
    pk = m.pk
    _snap, meta = snp.pack_objects([m.clusters[k] for k in sorted(m.clusters)], m.live_pods(), m.jobs)
    row_key = {pk.cluster_row(*k): k for k in m.clusters}

    def recs(res, key_of):
        return sorted((key_of(int(j["cluster_idx"])), int(j["cluster_state"]), int(j["not_ready"]), int(j["status_changed"])) for j in res.jobs)

    assert recs(want, lambda ci: tuple(meta.cluster_keys[ci]) if ci >= 0 else ("", "")) == recs(got, lambda r: tuple(row_key[r]) if r >= 0 else ("", ""))


def _fuzz(seed):
    clusters, pods, jobs = objects(seed, big=True)
    return copy.deepcopy(clusters), copy.deepcopy(pods), jobs


def _devices(n):
    return [0] * n


# ---------------------------------------------------------------------------------------------------------------- (1) + (2)
@pytest.mark.parametrize("n", [2, 3])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_every_shard_equals_its_oracle_and_the_twin_every_epoch(seed, n, oracle_mod):
    rng = np.random.default_rng(seed)
    clusters, pods, jobs = _fuzz(seed)
    gp, twin = GroupPacker(_devices(n), **PACKER_CAPS), Packer(**PACKER_CAPS)
    try:
        r = Router(clusters, pods, jobs, gp, twin)
        modes, _, _ = r.epoch(oracle_mod, lean=False)
        assert modes == [abi.PACK_FULL] * n
        r.epoch(oracle_mod, lean=True)
        counter = [0]
        for epoch in range(8):
            events(rng, r, counter, structural=True)
            modes, _, _ = r.epoch(oracle_mod, lean=bool(epoch % 2))
            assert not any(mo & abi.PACK_FULL for mo in modes)
    finally:
        gp.close()
        twin.close()


# ---------------------------------------------------------------------------------------------------------------- simple fleets
def _worker(cluster, k, group="g0", ready=True, ns=NS):
    return {"namespace": ns, "name": f"{cluster}-{group}-w{k}", "labels": {L_CLUSTER: cluster, L_TYPE: "worker", L_GROUP: group}, "phase": "Running",
            "conditions": [{"type": "Ready", "status": "True" if ready else "False"}], "restartPolicy": "Always"}


def _head(cluster, ns=NS):
    return {"namespace": ns, "name": f"{cluster}-head", "labels": {L_CLUSTER: cluster, L_TYPE: "head", L_GROUP: "headgroup"},
            "phase": "Running", "conditions": [{"type": "Ready", "status": "True"}], "podIP": "10.1.0.1", "restartPolicy": "Always"}


def _cluster(name, groups=(("g0", 2),), uid=True, ns=NS, rv=100):
    spec = {"workerGroupSpecs": [{"groupName": g, "replicas": k, "minReplicas": 0, "maxReplicas": max(k, 4), "numOfHosts": 1} for g, k in groups]}
    c = {"namespace": ns, "name": name, "generation": 1, "resourceVersion": rv, "spec": spec, "status": {},
         "expectations": {"head": True, **{g: True for g, _ in groups}}}
    if uid:
        c["uid"] = f"uid-{name}"
    return c


def _fleet(n_clusters, workers=2):
    """Healthy RayClusters (a head and `workers` workers each); every fourth one without a UID."""
    clusters, pods = [], []
    for i in range(n_clusters):
        name = f"rc{i}"
        clusters.append(_cluster(name, (("g0", workers),), uid=i % 4 != 0, rv=100 + i))
        pods += [_head(name)] + [_worker(name, k) for k in range(workers)]
    return clusters, pods


def _flip(r: Router, pod):
    p = copy.deepcopy(pod)
    p["conditions"] = [{"type": "Ready", "status": "False" if p["conditions"][0]["status"] == "True" else "True"}]
    r.upsert_pod(p)


def _one_cluster_per_shard(r: Router):
    """The first RayCluster (by key) of every shard."""
    return [sorted(m.clusters)[0] for m in r.m]


# ---------------------------------------------------------------------------------------------------------------- (3)
@pytest.mark.parametrize("n", [2, 3])
def test_churn_and_replica_edits_stay_incremental_on_every_shard(n, oracle_mod):
    clusters, pods = _fleet(8 * n)
    gp, twin = GroupPacker(_devices(n), **PACKER_CAPS), Packer(**PACKER_CAPS)
    try:
        r = Router(clusters, pods, [], gp, twin)
        assert all(len(m.clusters) >= 2 for m in r.m), [len(m.clusters) for m in r.m]
        r.epoch(oracle_mod, lean=True)
        for epoch in range(6):
            touched = _one_cluster_per_shard(r) if epoch % 2 == 0 else [sorted(m.clusters)[-1] for m in r.m]
            status_only = epoch < 4
            if status_only:  # Pod status churn: a Ready flip of one worker of one RayCluster per shard
                for key in touched:
                    _flip(r, next(p for p in r.live_pods() if p["labels"][L_CLUSTER] == key[1] and p["labels"][L_TYPE] == "worker"))
            else:  # replica edit of one RayCluster per shard (object rows)
                for key in touched:
                    c = copy.deepcopy(r.clusters[key])
                    c["spec"]["workerGroupSpecs"][0]["replicas"] = 3 + epoch
                    c["resourceVersion"] += 1
                    r.upsert_cluster(c)
            modes, res, tw = r.epoch(oracle_mod, lean=True)
            for i, x in enumerate(res):
                assert x.changed_clusters is not None and x.n_changed < gp.shards[i].engine.sizes.n_clusters, (epoch, i, x.n_changed)
                assert modes[i] == (abi.PACK_POD_ROWS if status_only else abi.PACK_OBJECT_ROWS), (epoch, i, modes[i])
            if status_only:
                # 32 B per touched Pod row on both sides (a journal entry: row id + 7 values); no head rows in these epochs
                shard_bytes = [sh.engine.last_profile()["h2d_bytes"] for sh in gp.shards]
                twin_bytes = twin.engine.last_profile()["h2d_bytes"]
                assert sum(shard_bytes) == twin_bytes == 32 * n, (shard_bytes, twin_bytes)
        # (6) the all-gather through the group packer's kr_group, after an incremental epoch
        gathered, slot, _used = gp.group.allgather_group_results()
        for i, x in enumerate(res):
            ng = int(gp.shards[i].engine.sizes.n_groups)
            assert slot >= 32 * ng
            for fld in ("expected", "n_list", "n_unhealthy", "n_running", "diff", "n_create", "flags"):
                assert np.array_equal(gathered[i][:ng][fld], x.groups[fld]), (i, fld)
            assert not gathered[i][ng:].view(np.uint8).any()
        # a RayCluster without a UID: c_uid_hash (FNV-1a of "ns/name") % n is its shard
        for key, c in r.clusters.items():
            if "uid" not in c:
                s = shard_of_key(*key, n)
                sh = gp.shards[s]
                assert int(sh.column("c_uid_hash")[sh.cluster_row(*key)]) % n == s, key
    finally:
        gp.close()
        twin.close()


# ---------------------------------------------------------------------------------------------------------------- (4)
@pytest.mark.parametrize("n", [2, 3])
def test_routing_edge_cases(n, oracle_mod):
    clusters, pods = _fleet(6)
    gp, twin = GroupPacker(_devices(n), **PACKER_CAPS), Packer(**PACKER_CAPS)
    try:
        r = Router(clusters, pods, [{"namespace": NS, "name": "job-a", "status": {}}], gp, twin)
        r.epoch(oracle_mod, lean=True)
        # a Pod before its RayCluster (an orphan on the shard of its label), then the RayCluster
        r.upsert_pod(_worker("late", 0))
        r.upsert_pod(_head("late"))
        _, res, _ = r.epoch(oracle_mod, lean=True)
        r.upsert_cluster(_cluster("late", (("g0", 1),)))
        _, res, _ = r.epoch(oracle_mod, lean=False)
        s = shard_of_key(NS, "late", n)
        assert int(res[s].clusters["n_pods"][gp.shards[s].cluster_row(NS, "late")]) == 2
        # a RayCluster deleted and re-created under its name with a new UID while its old Pods live: the new one counts them
        old = r.clusters[(NS, "rc1")]
        r.delete_cluster(NS, "rc1")
        r.epoch(oracle_mod, lean=True)
        new = copy.deepcopy(old)
        new["uid"], new["resourceVersion"] = "uid-rc1-recreated", 900
        r.upsert_cluster(new)
        _, res, _ = r.epoch(oracle_mod, lean=True)
        s = shard_of_key(NS, "rc1", n)
        assert int(res[s].clusters["n_pods"][gp.shards[s].cluster_row(NS, "rc1")]) == 3
        # a Pod relabelled to another RayCluster (pick one whose new label lives on another shard when there is one)
        src = next((p for p in r.live_pods() if p["labels"].get(L_TYPE) == "worker" and shard_of_key(NS, p["labels"][L_CLUSTER], n) != shard_of_key(NS, "rc2", n)),
                   next(p for p in r.live_pods() if p["labels"].get(L_TYPE) == "worker" and p["labels"][L_CLUSTER] != "rc2"))
        moved = copy.deepcopy(src)
        moved["labels"][L_CLUSTER] = "rc2"
        r.upsert_pod(moved)
        r.epoch(oracle_mod, lean=True)
        assert sum(sh.pod_row(NS, moved["name"]) >= 0 for sh in gp.shards) == 1
        assert gp.shards[shard_of_key(NS, "rc2", n)].pod_row(NS, moved["name"]) >= 0
        # a Pod without the label
        r.upsert_pod({"namespace": NS, "name": "stray", "labels": {}, "phase": "Running", "restartPolicy": "Always"})
        r.epoch(oracle_mod, lean=False)
        assert gp.shards[shard_of_key(NS, None, n)].pod_row(NS, "stray") >= 0
        # a RayJob whose cluster name is set later, then changed
        for target in ("rc3", "rc4", "rc5"):
            r.upsert_job({"namespace": NS, "name": "job-a", "status": {"rayClusterName": target, "rayClusterStatus": {"state": "ready"}}})
            _, res, _ = r.epoch(oracle_mod, lean=True)
            s = shard_of_key(NS, target, n)
            assert [int(sh.engine.sizes.n_jobs) for sh in gp.shards] == [int(i == s) for i in range(n)]
            assert int(res[s].jobs["cluster_idx"][0]) == gp.shards[s].cluster_row(NS, target)
        # deletes of unknown keys are no-ops
        for call in (gp.delete_pod, gp.delete_cluster, gp.delete_job):
            call(NS, "no-such-object")
            call("no-such-namespace", "rc0")
        r.delete_job(NS, "job-a")
        r.delete_pod(NS, "stray")
        r.epoch(oracle_mod, lean=True)
    finally:
        gp.close()
        twin.close()


# ---------------------------------------------------------------------------------------------------------------- (5)
def test_every_option_on_equals_the_all_off_twin(oracle_mod):
    n = 3
    rng = np.random.default_rng(7)
    clusters, pods = _fleet(9)
    clusters.append(_cluster("large", (("g0", 300),)))
    pods += [_head("large")] + [_worker("large", k) for k in range(300)]
    wide = [(f"g{k}", 1) for k in range(40)]
    clusters.append(_cluster("wide", wide))
    pods += [_head("wide")] + [_worker("wide", 0, group=g) for g, _ in wide]
    cap = dict(PACKER_CAPS, max_pods=8192)
    gp = GroupPacker(_devices(n), large_clusters=True, wide_clusters=True, huge_clusters=True, wtd_edits=True, spec_rows=True, **cap)
    twin = Packer(**cap)
    try:
        for sh in gp.shards:
            for opt in (abi.OPT_LARGE_CLUSTERS, abi.OPT_WIDE_CLUSTERS, abi.OPT_HUGE_CLUSTERS, abi.OPT_WTD_EDITS, abi.OPT_SPEC_ROWS):
                assert sh.engine.get_option(opt) == 1
        r = Router(clusters, pods, [], gp, twin)
        r.epoch(oracle_mod, lean=True)
        counter = [0]
        for epoch in range(8):
            events(rng, r, counter, structural=epoch % 3 == 2)
            if epoch % 2 == 0:  # a workersToDelete edit and a spec edit
                key = (NS, "large")
                c = copy.deepcopy(r.clusters[key])
                c["spec"]["workerGroupSpecs"][0]["workersToDelete"] = [f"large-g0-w{epoch}"]
                c["spec"]["rayVersion"] = f"2.{epoch}.0"
                c["generation"] += 1
                c["resourceVersion"] += 1
                r.upsert_cluster(c)
            r.epoch(oracle_mod, lean=epoch % 4 != 3)
    finally:
        gp.close()
        twin.close()


# ---------------------------------------------------------------------------------------------------------------- (7)
def test_a_shard_over_capacity_fails_the_flush_and_is_named(oracle_mod):
    n = 2
    gp = GroupPacker(_devices(n), **dict(PACKER_CAPS, max_groups=4))
    try:
        names = [f"rc{i}" for i in range(64)]
        full = next(s for s in range(n) if sum(shard_of_key(NS, x, n) == s for x in names) >= 3)
        mine = [x for x in names if shard_of_key(NS, x, n) == full][:3]
        for x in mine:  # 6 worker groups on one shard, 4 allowed
            gp.upsert_cluster(_cluster(x, (("g0", 1), ("g1", 1))))
        with pytest.raises(EngineError) as e:
            gp.flush()
        assert e.value.code == abi.KR_E_CAPACITY
        assert f"shard {full}:" in str(e.value) and "worker groups" in str(e.value), str(e.value)
    finally:
        gp.close()


# ---------------------------------------------------------------------------------------------------------------- one shard per GPU
def test_one_shard_per_device_when_the_box_has_several(oracle_mod):
    n = lib().kr_device_count()
    if n < 2:
        pytest.skip("one GPU: the shards share device 0 in the tests above")
    clusters, pods, jobs = _fuzz(5)
    gp, twin = GroupPacker(list(range(n)), **PACKER_CAPS), Packer(**PACKER_CAPS)
    try:
        r = Router(clusters, pods, jobs, gp, twin)
        r.epoch(oracle_mod, lean=True)
        rng, counter = np.random.default_rng(5), [0]
        for epoch in range(4):
            events(rng, r, counter, structural=True)
            r.epoch(oracle_mod, lean=bool(epoch % 2))
        assert [gp.group._L.kr_group_device(gp.group._h, i) for i in range(n)] == list(range(n))
    finally:
        gp.close()
        twin.close()

"""The native event-driven packer (kr_packer_*, kuberay_b200/csrc/kr_packer.cpp; SURVEY §8(f) rank 1).

Object-level differential test: the same RayClusters / Pods / RayJobs (tests/fuzz_objects.py, drawn from the whole input domain)
go (a) through the Python packer into the CPU oracle and (b) event by event through the native packer into the engine it owns.
Ids and row numbers differ between the two (different interning order, free rows), so the records are compared through the
strings and Pod keys they stand for.  Then random informer events are applied to both; most epochs must be incremental
(pod rows / small tables only) and every epoch must still agree."""
import copy

import numpy as np
import pytest

import fuzz_objects
from kuberay_b200 import abi
from kuberay_b200 import snapshot as snp
from kuberay_b200.packer import Packer
from test_live_arena import _events

pytestmark = pytest.mark.gpu

ID_FIELDS = ("head_ready_reason_id", "head_ready_msg_id")
PLAIN_FIELDS = ("path", "head_action", "err_kind", "status_err", "new_state", "state_changed", "needs_status_write", "head_update_annotations",
                "stop_after_group", "err_arg", "n_pods", "n_heads", "counts", "cond_status", "cond_variant", "status_flags")


class Mirror:
    """Holds the objects the way test_live_arena's LiveArena does (so its event generator can drive both sides)."""

    def __init__(self, clusters, pods, jobs, packer: Packer):
        self.clusters = {(c.get("namespace", "default"), c["name"]): c for c in clusters}
        self.rows = list(pods)
        self.row_of = {(p.get("namespace", "default"), p["name"]): i for i, p in enumerate(self.rows)}
        self.jobs = list(jobs)
        self.pk = packer
        for c in clusters:
            packer.upsert_cluster(c)
        for p in pods:
            packer.upsert_pod(p)
        for j in jobs:
            packer.upsert_job(j)

    def upsert_pod(self, pod):
        key = (pod.get("namespace", "default"), pod["name"])
        if key in self.row_of:
            self.rows[self.row_of[key]] = pod
        else:  # like the native packer: the lowest free row, else append — so both sides see the same List order
            free = [i for i, p in enumerate(self.rows) if p is None]
            if free:
                self.row_of[key] = free[0]; self.rows[free[0]] = pod
            else:
                self.row_of[key] = len(self.rows); self.rows.append(pod)
        self.pk.upsert_pod(pod)
        assert self.pk.pod_row(*key) == self.row_of[key]

    def delete_pod(self, ns, name):
        i = self.row_of.pop((ns, name), None)
        if i is not None:
            self.rows[i] = None
        self.pk.delete_pod(ns, name)

    def upsert_cluster(self, c):
        self.clusters[(c.get("namespace", "default"), c["name"])] = c
        self.pk.upsert_cluster(c)

    def delete_cluster(self, ns, name):
        self.clusters.pop((ns, name), None)
        self.pk.delete_cluster(ns, name)

    def upsert_job(self, j):
        key = (j.get("namespace", "default"), j["name"])
        keys = [(x.get("namespace", "default"), x["name"]) for x in self.jobs]
        self.jobs = [j if k == key else x for k, x in zip(keys, self.jobs)] + ([] if key in keys else [j])
        self.pk.upsert_job(j)

    def delete_job(self, ns, name):
        self.jobs = [x for x in self.jobs if (x.get("namespace", "default"), x["name"]) != (ns, name)]
        self.pk.delete_job(ns, name)

    def live_pods(self):
        return [p for p in self.rows if p is not None]


def check(m: Mirror, oracle_mod, lean: bool, run=None):
    """`run(flags) -> Results` takes the packer's pass another way than kr_reconcile_batch (default: pk.engine.reconcile)."""
    pk = m.pk
    clusters = [m.clusters[k] for k in sorted(m.clusters)]
    pods = m.live_pods()
    snap, meta = snp.pack_objects(clusters, pods, m.jobs)
    flags = meta.flags
    flags.fetch_pod_lists = 0 if lean else 1
    want = oracle_mod.run(snap, flags)
    f2 = pk.flags(fetch_pod_lists=flags.fetch_pod_lists)
    got = (run or pk.engine.reconcile)(f2)
    it = meta.interner
    assert got.n_orphans == want.n_orphans and got.n_actions == want.n_actions and got.n_create_total == want.n_create_total
    for ci, key in enumerate(meta.cluster_keys):
        r = pk.cluster_row(*key)
        assert r >= 0, key
        a, b = want.clusters[ci], got.clusters[r]
        for f in PLAIN_FIELDS:
            assert np.array_equal(a[f], b[f]), (key, f, a[f], b[f])
        for f in ID_FIELDS:
            assert (it.str(int(a[f])) or "") == (pk.string(int(b[f])) or ""), (key, f)
        assert [it.str(int(x)) or "" for x in a["head_ids"]] == [pk.string(int(x)) or "" for x in b["head_ids"]], key
        hp = int(a["head_pod_idx"])
        assert (meta.pod_keys[hp] if hp >= 0 else (None, None)) == (pk.pod_key(int(b["head_pod_idx"])) if int(b["head_pod_idx"]) >= 0 else (None, None))
        assert bytes(want.hash[ci]) == bytes(got.hash[r]), key
        # actions: (pod key, code) in List order (the mirror reuses the lowest free row exactly like the native packer)
        wa = [(meta.pod_keys[int(p)], int(c)) for p, c in zip(*want.actions_of(ci))]
        ga = [(pk.pod_key(int(p)), int(c)) for p, c in zip(*got.actions_of(r))]
        assert wa == ga, (key, wa, ga)
        # worker groups
        g0w = int(snap.c_group_off[ci])
        ng = int(snap.c_group_cnt[ci])
        for gi in range(ng):
            wg = want.groups[g0w + gi]
            # the native side's group rows follow ITS cluster order: find them through the record's group offset (arena column)
            gg = got.groups[_group_off(pk, r) + gi]
            for f in ("expected", "n_list", "n_unhealthy", "n_running", "diff", "n_create", "flags"):
                assert wg[f] == gg[f], (key, gi, f, wg[f], gg[f])
            assert sorted(want.creates_of(g0w + gi).tolist()) == sorted(got.creates_of(_group_off(pk, r) + gi).tolist())
    return want, got


def _group_off(pk: Packer, cluster_row: int) -> int:
    return int(pk.column("c_group_off")[cluster_row])


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_native_packer_agrees_with_python_packer_and_stays_incremental(seed, oracle_mod):
    rng = np.random.default_rng(seed)
    clusters, pods, jobs = fuzz_objects.generate(seed, big=True)
    for i, c in enumerate(clusters):
        c["generation"], c["resourceVersion"] = 1, 100 + i
    for i, j in enumerate(jobs):
        j.setdefault("name", f"rayjob-{i}")
    pk = Packer(max_clusters=64, max_groups=512, max_wtd=512, max_pods=4096, max_heads=256, max_jobs=64, max_creates=1 << 16, max_json_bytes=4 << 20)
    try:
        m = Mirror(copy.deepcopy(clusters), copy.deepcopy(pods), jobs, pk)
        assert pk.flush() == abi.PACK_FULL
        check(m, oracle_mod, lean=False)
        check(m, oracle_mod, lean=True)
        e0, v0 = pk.epoch()
        modes = []
        counter = [0]
        for epoch in range(10):
            _events(rng, m, counter, structural=True)
            mode = pk.flush()
            modes.append(mode)
            assert not mode & abi.PACK_FULL
            check(m, oracle_mod, lean=bool(epoch % 2))
        e1, v1 = pk.epoch()
        assert e1 == e0 + 10 and v1 > v0
        assert any(mo & abi.PACK_POD_ROWS for mo in modes) and not all(mo & abi.PART_JSON for mo in modes)
        # a spec change bumps the generation: the JSON is re-emitted and travels; an unchanged generation does not re-emit
        key = sorted(m.clusters)[0]
        c = copy.deepcopy(m.clusters[key])
        c.pop("specJson", None)  # (from here on this RayCluster's hash input comes from the emitter, on both sides)
        c["spec"]["rayVersion"] = "9.9.9"; c["generation"] = 2; c["resourceVersion"] = 999
        m.upsert_cluster(c)
        assert pk.flush() & abi.PART_JSON
        check(m, oracle_mod, lean=True)
        assert pk.cluster_epoch(pk.cluster_row(*key)) == (999, 2)
    finally:
        pk.close()

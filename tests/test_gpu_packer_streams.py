"""The native packer with five opt-in options on (KR_OPT_LARGE_CLUSTERS, _WIDE_CLUSTERS, _HUGE_CLUSTERS, _WTD_EDITS, _SPEC_ROWS),
against a twin packer with all of them off, on the same informer event stream.  (The structural options, KR_OPT_CLUSTER_CREATES,
_CLUSTER_DELETES, _GROUP_EDITS and _LARGE_GROWTH, run with these in tests/test_gpu_structural_streams.py.)

The fleet: about 150 RayClusters cloned from fuzz objects (multi-host groups, Recreate gates, RayJobs, every adversarial field),
plus healthy RayClusters of about 1 500 and 8 190 Pods, one of 9 000 Pods, three of 33-40 worker groups, one of 250 Pods and one of
32 worker groups.  Each epoch mixes Pod traffic and RayCluster status (harness.events), autoscaler workersToDelete edits
(harness.autoscale_objects) and spec edits with a bumped generation (harness.spec_edits); some epochs also
move a RayCluster across a class boundary (256 -> 257 Pods, 8 192 -> 8 193 Pods, 32 -> 33 worker groups, and back), create or delete
a RayCluster and a RayJob, and the JSON arena is small enough to be compacted a few times per stream.

Every epoch both packers equal the oracle (every 8th epoch with the full pod lists), equal each other, report the flush mode the
epoch calls for, and the all-on packer's pass rotates over kr_reconcile_batch, kr_reconcile_device_only + kr_results_fetch and
kr_reconcile_batch_profiled + kr_results_fetch.  Quiet epochs (no class move, no RayCluster created or deleted, no compaction, same
flags as the epoch before) must be incremental on the all-on packer: on an H100 80GB HBM3 (700 W power limit) 16 of 16 quiet epochs
were for seed 1 and 17 of 17 for seed 2, with 2 and 1 compactions; the file took 19 s of wall time there."""
import copy
import json

import numpy as np
import pytest

from harness import L_CLUSTER, L_GROUP, L_TYPE, Mirror, autoscale_objects, events, huge_objects, packer_check, spec_edits
from kuberay_b200 import abi
from kuberay_b200.engine import spec_json_emit
from kuberay_b200.packer import Packer

pytestmark = pytest.mark.gpu

NS = "fleet"
EPOCHS = 30
QUIET_MIN = 1.0   # share of quiet epochs that must be incremental (every one was, on the first H100 run)


def _healthy(name, groups, i):
    """A RayCluster whose worker groups [(name, workers)] each run exactly their replicas, with a head Pod; -> (cluster, pods)."""
    spec = {"workerGroupSpecs": [{"groupName": g, "replicas": n, "minReplicas": 0, "maxReplicas": n + 64, "numOfHosts": 1} for g, n in groups]}
    c = {"namespace": NS, "name": name, "uid": f"uid-{name}", "generation": 1, "resourceVersion": 50_000 + i, "spec": spec, "status": {},
         "expectations": {"head": True, **{g: True for g, _ in groups}}}
    pods = [{"namespace": NS, "name": f"{name}-head", "labels": {L_CLUSTER: name, L_TYPE: "head", L_GROUP: "headgroup"}, "phase": "Running",
             "conditions": [{"type": "Ready", "status": "True"}], "podIP": "10.2.0.1", "restartPolicy": "Always"}]
    pods += [_worker(name, g, k) for g, n in groups for k in range(n)]
    return c, pods


def _worker(name, group, k):
    return {"namespace": NS, "name": f"{name}-{group}-{k}", "labels": {L_CLUSTER: name, L_GROUP: group, L_TYPE: "worker"}, "phase": "Running",
            "conditions": [{"type": "Ready", "status": "True"}], "restartPolicy": "Always"}


BIG = {  # name -> worker groups
    "large": [("g0", 1499)],
    "edge8192": [("g0", 8189)],       # 8 190 Pods: 5 more cross 8 192 -> 8 193
    "huge": [("g0", 8999)],
    "wide33": [(f"g{k}", 2) for k in range(33)],
    "wide36": [(f"g{k}", 2) for k in range(36)],
    "wide40": [(f"g{k}", 1) for k in range(40)],
    "edge256": [("g0", 249)],         # 250 Pods: 10 more cross 256 -> 257
    "edge32": [(f"g{k}", 1) for k in range(32)],
}


def _fleet(seed):
    clusters, pods, jobs = huge_objects(seed, 0, n_clusters=150)
    for i, (name, groups) in enumerate(BIG.items()):
        c, p = _healthy(name, groups, i)
        clusters.append(c)
        pods += p
    return clusters, pods, jobs


def _json_bytes(clusters):
    """The live muted-spec JSON the packer lays out (16-byte aligned blobs)."""
    n = 0
    for c in clusters:
        b = c["specJson"] if "specJson" in c else spec_json_emit(json.dumps(c.get("spec") or {}).encode())
        n += (len(b) + 15) // 16 * 16
    return n


EDGE = ("edge256", "edge8192", "edge32")  # (their sizes move only in _class_moves' epochs)


class _Side:
    """The Mirror as the shared event generators see it, without the RayCluster objects `clusters_out` and the Pods of
    `pods_out`: harness.events would set a big RayCluster's replicas to 0-6 (thousands of deletes on one RayCluster are
    not the traffic this stream is about), and random Pod traffic would move the edge RayClusters across their boundaries."""

    def __init__(self, m, clusters_out, pods_out):
        self.m, self.row_of = m, m.row_of
        self.rows = [p for p in m.rows if p is not None and not (p.get("namespace") == NS and p["labels"].get(L_CLUSTER) in pods_out)]
        self.clusters = {k: c for k, c in m.clusters.items() if not (k[0] == NS and k[1] in clusters_out)}

    def upsert_pod(self, p):
        self.m.upsert_pod(p)

    def delete_pod(self, ns, name):
        self.m.delete_pod(ns, name)

    def upsert_cluster(self, c):
        self.m.upsert_cluster(c)


def _respec(m, name, edit):
    c = copy.deepcopy(m.clusters[(NS, name)])
    edit(c)
    c["generation"] += 1
    c["resourceVersion"] += 1
    m.upsert_cluster(c)


def _grow(m, name, n, tag):
    """n more workers in group g0, replicas raised to match."""
    def edit(c):
        c["spec"]["workerGroupSpecs"][0]["replicas"] += n
    _respec(m, name, edit)
    for k in range(n):
        m.upsert_pod(_worker(name, "g0", tag + k))


def _shrink(m, name, n, tag):
    def edit(c):
        c["spec"]["workerGroupSpecs"][0]["replicas"] -= n
    _respec(m, name, edit)
    for k in range(n):
        m.delete_pod(NS, f"{name}-g0-{tag + k}")


def _class_moves(m, epoch):
    """-> what the epoch does beyond the ordinary traffic ("" for nothing)."""
    if epoch == 3:
        _grow(m, "edge256", 10, 10_000)            # 250 -> 260 Pods
        return "257 pods"
    if epoch == 6:
        _grow(m, "edge8192", 5, 10_000)            # 8 190 -> 8 195 Pods
        return "8193 pods"
    if epoch == 9:
        def add(c):
            c["spec"]["workerGroupSpecs"].append({"groupName": "g32", "replicas": 1, "minReplicas": 0, "maxReplicas": 4, "numOfHosts": 1})
            c["expectations"]["g32"] = True
        _respec(m, "edge32", add)
        m.upsert_pod(_worker("edge32", "g32", 0))
        return "33 groups"
    if epoch == 12:
        _shrink(m, "edge256", 10, 10_000)
        return "256 pods"
    if epoch == 15:
        def drop(c):
            c["spec"]["workerGroupSpecs"].pop()
            c["expectations"].pop("g32")
        _respec(m, "edge32", drop)
        m.delete_pod(NS, "edge32-g32-0")
        return "32 groups"
    if epoch == 18:
        c, pods = _healthy("created", [("g0", 3), ("g1", 2)], 99)
        m.upsert_cluster(c)
        for p in pods:
            m.upsert_pod(p)
        m.upsert_job({"namespace": NS, "name": "job-created", "status": {"rayClusterName": "created", "rayClusterStatus": {"state": "ready"}}})
        return "created"
    if epoch == 21:
        _shrink(m, "edge8192", 5, 10_000)
        return "8192 pods"
    if epoch == 24:
        m.delete_cluster(NS, "created")
        m.delete_job(NS, "job-created")
        victim = sorted(k for k in m.clusters if k[0] != NS)[7]
        m.delete_cluster(*victim)
        return "deleted"
    return ""


def _offsets(m):
    col = m.pk.column("c_json_off")
    return {k: (int(col[m.pk.cluster_row(*k)]), m.clusters[k].get("generation")) for k in m.clusters}


def _runs(eng):
    """The all-on packer's pass, by epoch: the three callers of the engine's pass driver."""
    def device_only(f):
        eng.reconcile_device_only(f)
        return eng.fetch()

    def profiled(f):
        eng.reconcile_profiled(f)
        return eng.fetch()
    return [eng.reconcile, device_only, profiled]


@pytest.mark.parametrize("seed", [1, 2])
def test_all_options_on_against_all_off(seed, oracle_mod):
    clusters, pods, jobs = _fleet(seed)
    cap = _json_bytes(clusters) + (24 << 10)  # (room for a few epochs of spec edits: the arena is compacted a few times)
    opts = dict(large_clusters=True, wide_clusters=True, huge_clusters=True, wtd_edits=True, spec_rows=True)
    pks = [Packer(max_clusters=256, max_groups=2048, max_wtd=2048, max_pods=32768, max_heads=1024, max_jobs=256, max_creates=1 << 16,
                  max_json_bytes=cap, **(opts if on else {})) for on in (True, False)]
    try:
        for o in (abi.OPT_LARGE_CLUSTERS, abi.OPT_WIDE_CLUSTERS, abi.OPT_HUGE_CLUSTERS, abi.OPT_WTD_EDITS, abi.OPT_SPEC_ROWS):
            assert pks[0].engine.get_option(o) == 1 and pks[1].engine.get_option(o) == 0, o
        ms = [Mirror(copy.deepcopy(clusters), copy.deepcopy(pods), copy.deepcopy(jobs), pk) for pk in pks]
        for pk, m in zip(pks, ms):
            assert pk.flush() == abi.PACK_FULL
            packer_check(m, oracle_mod, lean=True)
        assert pks[0].engine.get_option(abi.OPT_BUCKET_STRIDE) != 0
        runs = _runs(pks[0].engine)
        gens, counters, pendings = [[2], [2]], [[0], [0]], [{}, {}]
        quiet, full_quiet, compactions, moves = [], [], 0, set()
        for epoch in range(EPOCHS):
            lean = epoch % 8 != 7
            outs = []
            for i, (pk, m) in enumerate(zip(pks, ms)):
                r = np.random.default_rng(1000 * seed + epoch)  # the same events on both sides
                before = _offsets(m)
                spec_edits(r, m, gens[i], int(r.integers(1, 4)))
                autoscale_objects(r, _Side(m, EDGE, EDGE), pendings[i])
                events(r, _Side(m, BIG, EDGE), counters[i], structural=False)
                move = _class_moves(m, epoch)
                mode = pk.flush()
                after = _offsets(m)
                compacted = any(before[k][0] != after[k][0] for k in before if k in after and before[k][1] == after[k][1])
                _, got = packer_check(m, oracle_mod, lean=lean, run=runs[epoch % 3] if i == 0 else None)
                outs.append((mode, got, compacted, move))
            (mode_on, got_on, compacted, move), (mode_off, got_off, compacted_off, _) = outs
            assert compacted == compacted_off, epoch
            d = got_off.diff(got_on)
            assert not d, (epoch, d[:6])
            # every epoch re-emits a spec: row by row unless a RayCluster row moved or the arena was compacted
            if compacted or move in ("created", "deleted"):
                assert mode_on & abi.PART_JSON and not mode_on & abi.PACK_SPEC_ROWS, (epoch, mode_on)
            else:
                assert mode_on & abi.PACK_SPEC_ROWS and not mode_on & abi.PART_JSON, (epoch, mode_on)
            assert mode_off & abi.PART_JSON and not mode_off & abi.PACK_SPEC_ROWS, (epoch, mode_off)
            compactions += compacted
            if move:
                moves.add(move)
            if lean and epoch % 8 != 0 and not move and not compacted:  # (the epoch after a pod-list epoch has other flags)
                inc = got_on.changed_clusters is not None or got_on.n_changed == 0
                quiet.append(inc)
                if not inc:
                    full_quiet.append((epoch, mode_on, got_on.n_changed))
        assert len(moves) == 8 and compactions >= 1, (moves, compactions)
        assert sum(quiet) >= QUIET_MIN * len(quiet), (sum(quiet), len(quiet), full_quiet)
        print(f"seed {seed}: {sum(quiet)} of {len(quiet)} quiet epochs incremental, {compactions} compactions")
    finally:
        for pk in pks:
            pk.close()

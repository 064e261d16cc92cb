"""The native packer's rewrite of every object field it packs, one field of a few objects per epoch.

The informer stream of the other packer tests (harness.events) changes Pod phases and readiness, replicas, readyWorkerReplicas,
expectations and head Pods.  Here each epoch rewrites one field of a few Pods, RayClusters and RayJobs of a fuzz_objects fleet to
another value from fuzz_objects' own domain: Pod phases (the empty, Unknown and unparsable ones included), Ready status, reason
and message, restartPolicy, rayContainerTerminated, deletionTimestamp, every label the packer reads (replica indices that do not
parse included), podIP and a head's recreate-hash and KubeRay-version annotations; a RayCluster's suspend, autoscaling, upgrade
strategy, a group's replicas / min / max / numOfHosts / suspend, the expectations, the skip-head-restart annotation, the head
Service, the external error, every old-status field and the deletionTimestamp; a RayJob's rayClusterName and rayClusterStatus.
So kr_packer.cpp's update path (interned strings against the ones the row held, a replica-index label parsed again, a head Pod's
annotation and version state) is checked on every field, not only on the first full pack.

The two annotation edits are written on head Pods (of a Recreate-gated RayCluster when there is one), the only Pods that read
them.  Every epoch equals the oracle: the RayCluster records (packer_check; every fourth epoch with the full pod lists) and the
RayJob roll-ups, compared by the RayCluster each RayJob found.  A flush after the first is never PACK_FULL,
and a lean epoch after a lean one is incremental on the device unless the epoch changed a table's shape (a Pod became or stopped
being a head)."""
import copy
import itertools

import numpy as np
import pytest

import fuzz_objects
from harness import L_CLUSTER, L_GROUP, L_TYPE, PACKER_CAPS, Mirror, device_incremental, objects, packer_check
from kuberay_b200 import abi
from kuberay_b200 import snapshot as snp
from kuberay_b200.packer import Packer

pytestmark = pytest.mark.gpu

EPOCHS = 30
L_RIDX, L_RNAME = fuzz_objects.L_RIDX, fuzz_objects.L_RNAME
pick = fuzz_objects._pick


def _label(key, values):
    def edit(rng, p, m):
        v = pick(rng, values(m) if callable(values) else values)
        if v is None:
            p["labels"].pop(key, None)
        else:
            p["labels"][key] = v
    return edit


def _field(key, values):
    def edit(rng, p, m):
        v = pick(rng, values)
        if v is None:
            p.pop(key, None)
        else:
            p[key] = v
    return edit


def _ready(rng, p, m):
    p["conditions"] = [{"type": "Ready", "status": pick(rng, ["True", "False", "Unknown", ""]), "reason": pick(rng, ["", "ContainersNotReady", "PodCompleted"]),
                        "message": pick(rng, ["", "m", "ray-head: boom"])}]


def _annotation(key, values):
    def edit(rng, p, m):
        ann = p.setdefault("annotations", {})
        v = pick(rng, values(m, p) if callable(values) else values)
        if v is None:
            ann.pop(key, None)
        else:
            ann[key] = v
    return edit


def _spec_hash(m, p):
    c = m.clusters.get((p.get("namespace", "default"), p["labels"].get(L_CLUSTER)))
    own = fuzz_objects._hash32(bytes(c["specJson"])) if c is not None else "short"
    return [own, fuzz_objects._hash32(b"other"), "short", "", None]


POD_EDITS = {
    "phase": _field("phase", fuzz_objects.PHASES),
    "ready": _ready,
    "restartPolicy": _field("restartPolicy", ["Always", "Never", "OnFailure", None]),
    "rayContainerTerminated": _field("rayContainerTerminated", [True, None]),
    "deletionTimestamp": _field("deletionTimestamp", ["2026-01-01T00:00:00Z", None]),
    "node type": _label(L_TYPE, ["worker", "head", "redis-cleanup", "bogus", None]),
    "group": _label(L_GROUP, [f"g{i}" for i in range(6)] + ["headgroup", None]),
    "cluster": _label(L_CLUSTER, lambda m: sorted({k[1] for k in m.clusters}) + ["nope", None]),
    "replica index": _label(L_RIDX, ["0", "1", "5", "-1", "abc", "007", "+3", "99999999999", "9223372036854775808", "", None]),
    "replica name": _label(L_RNAME, ["g0-r0", "g0-r1", "g1-r0", "g2-r3", None]),
    "podIP": _field("podIP", ["", "10.1.0.1", "10.1.0.2", None]),
    "recreate hash": _annotation(snp.RECREATE_HASH_ANNOT, _spec_hash),
    "kuberay version": _annotation(snp.KUBERAY_VERSION_ANNOT, [snp.KUBERAY_VERSION, "v0.0.1", "", None]),
}


def _spec(key, values):
    def edit(rng, c):
        v = pick(rng, values)
        if v is None:
            c["spec"].pop(key, None)
        else:
            c["spec"][key] = v
    return edit


def _group(key, values):
    def edit(rng, c):
        groups = c["spec"].get("workerGroupSpecs") or []
        if not groups:
            return False
        g = groups[int(rng.integers(len(groups)))]
        g[key] = values(rng) if callable(values) else pick(rng, values)
        if abs(fuzz_objects._expected(g)) > 300:  # (fuzz_objects keeps the create lists small the same way)
            g["replicas"], g["maxReplicas"], g["minReplicas"], g["numOfHosts"] = int(rng.integers(0, 7)), 5, None, 1
    return edit


def _status(key, values):
    def edit(rng, c):
        st = c.setdefault("status", {})
        v = values(rng, c) if callable(values) else pick(rng, values)
        if v is None:
            st.pop(key, None)
        else:
            st[key] = v
    return edit


def _annotation_c(rng, c):
    c["annotations"] = {snp.SKIP_HEAD_RESTART_ANNOT: pick(rng, ["true", "false"])} if rng.random() < 0.7 else {}


def _expectations(rng, c):
    c["expectations"] = {k: bool(rng.random() < 0.5) for k in ["head"] + [g["groupName"] for g in c["spec"].get("workerGroupSpecs") or []]}


def _head_service(rng, c):
    c["headService"] = {"count": pick(rng, [0, 1, 2]), "clusterIP": pick(rng, ["", "None", "10.0.0.1", "10.0.0.9"]), "name": f"{c['name']}-head-svc"}


def _ext_err(rng, c):
    if rng.random() < 0.3:
        c.pop("extErr", None)
    else:
        c["extErr"] = {"kind": int(rng.integers(0, 8)), "message": pick(rng, ["e1", "e2", "boom"])}


CLUSTER_EDITS = {
    "suspend": _spec("suspend", [True, False, None]),
    "enableInTreeAutoscaling": _spec("enableInTreeAutoscaling", [True, False, None]),
    "upgradeStrategy": _spec("upgradeStrategy", [{"type": "Recreate"}, {"type": "None"}, None]),
    "replicas": _group("replicas", fuzz_objects._replica_number),
    "minReplicas": _group("minReplicas", fuzz_objects._replica_number),
    "maxReplicas": _group("maxReplicas", fuzz_objects._replica_number),
    "numOfHosts": _group("numOfHosts", [1, 2, 4, 0, -1, 3, 65536]),
    "group suspend": _group("suspend", [True, False]),
    "expectations": _expectations,
    "skip-head-restart annotation": _annotation_c,
    "headService": _head_service,
    "extErr": _ext_err,
    "state": _status("state", ["", "ready", "suspended", "failed", "unhealthy", None]),
    "conditions": _status("conditions", lambda rng, c: fuzz_objects._conditions(rng)),
    "reason": _status("reason", ["old reason", "", None]),
    "readyWorkerReplicas": _status("readyWorkerReplicas", [0, 1, 3, 5, None]),
    "availableWorkerReplicas": _status("availableWorkerReplicas", [0, 1, 3, 5, None]),
    "desiredWorkerReplicas": _status("desiredWorkerReplicas", [0, 1, 3, 5, None]),
    "minWorkerReplicas": _status("minWorkerReplicas", [0, 1, 3, None]),
    "maxWorkerReplicas": _status("maxWorkerReplicas", [0, 1, 3, 5, None]),
    "head": _status("head", lambda rng, c: fuzz_objects._old_status(rng, c["name"]).get("head")),
    "endpoints": _status("endpoints", [{}, {"dashboard": "8265"}, {"client": "10001", "dashboard": "8265"}, None]),
    "deletionTimestamp": lambda rng, c: c.pop("deletionTimestamp", None) if "deletionTimestamp" in c else c.__setitem__("deletionTimestamp", "2026-01-01T00:00:00Z"),
}


HEAD_EDITS = ("recreate hash", "kuberay version")  # (read from head Pods only: they are written on a head, a Recreate-gated one first)


def _heads(m):
    return sum(1 for p in m.live_pods() if (p.get("labels") or {}).get(L_TYPE) == "head")


def _recreate(m, p):
    c = m.clusters.get((p.get("namespace", "default"), (p.get("labels") or {}).get(L_CLUSTER)))
    return c is not None and (c["spec"].get("upgradeStrategy") or {}).get("type") == "Recreate"


def _job_records(res, key_of):
    """The RayJob records as (RayCluster key, cluster_state, not_ready, status_changed), sorted: the packer numbers RayJobs and
    RayClusters its own way, so the two sides are compared by the RayCluster each RayJob found."""
    return sorted((key_of(int(j["cluster_idx"])), int(j["cluster_state"]), int(j["not_ready"]), int(j["status_changed"])) for j in res.jobs)


def _check_jobs(m, want, got):
    """packer_check compares the RayCluster records; this compares the RayJob roll-ups.  -> the oracle's records."""
    _snap, meta = snp.pack_objects([m.clusters[k] for k in sorted(m.clusters)], m.live_pods(), m.jobs)
    row_key = {m.pk.cluster_row(*k): k for k in m.clusters}
    w = _job_records(want, lambda ci: tuple(meta.cluster_keys[ci]) if ci >= 0 else ("", ""))
    assert len(want.jobs) == len(got.jobs) == len(m.jobs)
    assert w == _job_records(got, lambda r: tuple(row_key[r]) if r >= 0 else ("", ""))
    return w


def _epoch(rng, m, seen, turn):
    """2-4 objects, one field of each rewritten (the fields in turn, so that each comes up within a few epochs).  -> whether a Pod
    became or stopped being a head."""
    heads = _heads(m)
    for _ in range(int(rng.integers(2, 5))):
        kind = rng.random()
        if kind < 0.5:
            pods = m.live_pods()
            name = sorted(POD_EDITS)[next(turn["pod"]) % len(POD_EDITS)]
            if name in HEAD_EDITS:
                heads = [p for p in pods if (p.get("labels") or {}).get(L_TYPE) == "head"]
                pods = [p for p in heads if _recreate(m, p)] or heads
                if not pods:
                    continue
            p = copy.deepcopy(pods[int(rng.integers(len(pods)))])
            p.setdefault("labels", {})
            POD_EDITS[name](rng, p, m)
            m.upsert_pod(p)
            seen.add("pod " + name)
            if name in HEAD_EDITS and _recreate(m, p):
                seen.add(f"pod {name} (Recreate-gated head)")
        elif kind < 0.85 or not m.jobs:
            key = sorted(m.clusters)[int(rng.integers(len(m.clusters)))]
            c = copy.deepcopy(m.clusters[key])
            name = sorted(CLUSTER_EDITS)[next(turn["cluster"]) % len(CLUSTER_EDITS)]
            if CLUSTER_EDITS[name](rng, c) is False:
                continue
            m.upsert_cluster(c)
            seen.add("cluster " + name)
        else:
            j = copy.deepcopy(m.jobs[int(rng.integers(len(m.jobs)))])
            st = j.setdefault("status", {})
            if next(turn["job"]) % 2 == 0:
                st["rayClusterName"] = pick(rng, sorted({k[1] for k in m.clusters}) + ["missing", ""])
                seen.add("job rayClusterName")
            else:
                st["rayClusterStatus"] = fuzz_objects._old_status(rng, "x")
                seen.add("job rayClusterStatus")
            m.upsert_job(j)
    return _heads(m) != heads


@pytest.mark.parametrize("options", [{}, dict(large_clusters=True, wide_clusters=True, huge_clusters=True, wtd_edits=True, spec_rows=True)],
                         ids=["options-off", "options-on"])
def test_one_field_at_a_time_through_the_native_packer(options, oracle_mod):
    seen, n_inc, n_quiet, job_moves = set(), 0, 0, 0
    turn = {"pod": itertools.count(), "cluster": itertools.count(), "job": itertools.count()}
    for seed in (3, 11, 29):
        rng = np.random.default_rng(1000 + seed)
        clusters, pods, jobs = objects(seed, big=True)
        pk = Packer(**PACKER_CAPS, **options)
        try:
            m = Mirror(clusters, pods, jobs, pk)
            assert pk.flush() == abi.PACK_FULL
            want, got = packer_check(m, oracle_mod, lean=True)
            jobs_before = _check_jobs(m, want, got)
            prev_lean = True
            for epoch in range(EPOCHS):
                shape = _epoch(rng, m, seen, turn)
                mode = pk.flush()
                assert not mode & abi.PACK_FULL, (seed, epoch, mode)
                lean = epoch % 4 != 3
                want, got = packer_check(m, oracle_mod, lean=lean)
                jobs_now = _check_jobs(m, want, got)
                job_moves += jobs_now != jobs_before
                jobs_before = jobs_now
                if lean and prev_lean and not shape:
                    n_quiet += 1
                    assert device_incremental(got), (seed, epoch, mode, got.n_changed)
                    n_inc += 1
                prev_lean = lean
        finally:
            pk.close()
    print("packer fields", options, f"{n_inc} of {n_quiet} quiet epochs incremental, RayJob records moved in {job_moves} epochs", sorted(seen))
    want = {"pod " + k for k in POD_EDITS} | {"cluster " + k for k in CLUSTER_EDITS} | {"job rayClusterName", "job rayClusterStatus"}
    want |= {f"pod {k} (Recreate-gated head)" for k in HEAD_EDITS}
    assert want <= seen, sorted(want - seen)
    assert job_moves >= 2, job_moves  # (the RayJob comparison saw records change, not only the ones of the first pack)
    assert n_quiet >= 30

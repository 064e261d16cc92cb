"""The object-level Go model (tests/go_model.py) pinned to the reference's own tables, and then used as a second reference:
closed-loop reconcile rounds on twin fake clients, one side driven by RayClusterReconciler over a backend (here the CPU oracle;
tests/test_gpu_go_model.py runs every GPU pipeline), the other by the model, compared at what Go can observe.

One round: one snapshot of the client, every RayCluster decided from it, the side effects applied RayCluster by RayCluster in
key order, the status written.  After each round the Delete and Create calls, the events, the returned error, the new status,
whether it was written, the requeue and the RayJob results must agree; between rounds some created Pods turn Running and
Ready.  The model shares nothing with the engine or the oracle, so a misreading of raycluster_controller.go that both of those
share shows up here and nowhere else."""
import base64
import copy
import difflib
import hashlib
import json
import os
import pprint

import numpy as np
import pytest

import fuzz_objects
import go_model as gm
from kuberay_b200 import snapshot as snapmod
from kuberay_b200.reconciler import ApiError, Env, FakeClient, RayClusterReconciler

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
HOST_INDEX_LABEL = "ray.io/replica-host-index"


def load(name):
    with open(os.path.join(GOLD, name + ".json")) as f:
        return json.load(f)


# ------------------------------------------------------------------------------------------ the model against the Go tables
def test_model_should_delete_pod():
    """Test_ShouldDeletePod (raycluster_controller_unit_test.go:2380-2503)."""
    for case in load("should_delete_pod")["cases"]:
        pod = {"name": "p", "phase": case["phase"], "restartPolicy": case["restartPolicy"], "containers": [{"name": "ray"}],
               "containerStatuses": [{"name": "ray", "state": {"terminated": {"reason": "Error"}} if case["terminated"] else {}}]}
        for ntype in ("head", "worker"):
            got, reason = gm.should_delete_pod(pod, ntype)
            assert got == case["want"], case
            assert f"The {ntype} Pod p" in reason or f"the {ntype} Pod p" in reason


def test_model_head_pod_ready():
    """TestFindHeadPodReadyCondition / ...Message (utils/util_test.go:331-355, 934-1038)."""
    gold = load("head_pod_ready")
    for case in gold["status_cases"]:
        pod = {"phase": case["phase"], "conditions": [{"type": "Ready", "status": case["ready"]}]}
        assert gm.find_head_pod_ready_condition(pod)["status"] == case["want_status"]
    for case in gold["message_cases"]:
        pod = {"conditions": [{"type": "Ready", "status": "False", "reason": "ContainersNotReady", "message": case["message"]}],
               "containerStatuses": case["containerStatuses"]}
        got = gm.find_head_pod_ready_condition(pod)
        assert (got["reason"], got["message"]) == (case["want_reason"], case["want_message"]), case["name"]


def test_model_inconsistent_status():
    """TestInconsistentRayClusterStatus (utils/consistency_test.go:16-146)."""
    gold = load("inconsistent_status")
    for case in gold["cases"]:
        new = copy.deepcopy(gold["old"])
        new.update(case.get("set", {}))
        new.setdefault("endpoints", {}).update(case.get("set_endpoint", {}))
        new.setdefault("head", {}).update(case.get("set_head", {}))
        assert gm.inconsistent_status(gold["old"], new) == case["want"], case["name"]


def _groups(spec_groups):
    return {"spec": {"workerGroupSpecs": [{"groupName": f"g{i}", "replicas": g.get("replicas"), "minReplicas": g.get("min"),
                                           "maxReplicas": g.get("max"), "numOfHosts": g.get("hosts", 1), "suspend": g.get("suspend", False)}
                                          for i, g in enumerate(spec_groups)]}}


def test_model_replica_arithmetic():
    """utils/util_test.go:58-130, 408-475, 555-601, 603-710, 712-800, 802-894."""
    gold = load("replica_arithmetic")
    for c in gold["desired_replicas"]["cases"]:
        g = {"replicas": c["replicas"], "minReplicas": c["min"], "maxReplicas": c["max"], "numOfHosts": c["hosts"], "suspend": c["suspend"]}
        assert gm.desired_replicas(g) == c["want"], c
    for c in gold["min_max"]["cases"]:
        rc = _groups(c["groups"])
        assert (gm.calculate_min(rc), gm.calculate_max(rc)) == (c["want_min"], c["want_max"]), c["name"]
    for c in gold["desired_cluster"]["cases"]:
        assert gm.calculate_desired(_groups(c["groups"])) == c["want"], c["name"]
    for c in gold["max_overflow"]["cases"]:
        assert gm.calculate_max(_groups(c["groups"])) == c["want_max"], c["name"]
    ar = gold["available_ready"]
    pods = [{"name": p["name"], "labels": {gm.NODE_TYPE_LABEL: p["nodeType"]}, "phase": p["phase"],
             "conditions": [{"type": "Ready", "status": p["ready"]}] if "ready" in p else []} for p in ar["pods"]]
    assert (gm.calculate_available(pods), gm.calculate_ready(pods)) == (ar["want_available"], ar["want_ready"])
    for c in gold["check_all_pods_running"]["cases"]:
        pods = [{"phase": p["phase"], "conditions": [{"type": "Ready", "status": p["ready"]}] if "ready" in p else []} for p in c["pods"]]
        assert gm.check_all_pods_running(pods) == c["want"], c["name"]


class ModelApi:
    """go_model's API over a FakeClient: the same fake API server the reconciler mirror writes to, and the same Pod
    metadata builder for a Create (the manifests are pinned by the pod-builder tests)."""

    def __init__(self, client: FakeClient, env: Env):
        self.client, self.env = client, env
        self.builder = RayClusterReconciler(client, None, env)

    def delete(self, ns, name):
        try:
            return self.client.delete_pod(ns, name)
        except ApiError as e:
            raise gm.ApiError(str(e))

    def delete_collection(self, pods):
        for p in pods:
            self.delete(gm.ns_of(p), p["name"])

    def create(self, cluster, spec):
        if spec["nodeType"] == "head":
            pod = self.builder._build_pod(cluster, (-1, 0, 0, ""), cluster_hash=spec["hash"])
        else:
            idx = spec["replicaIndex"] if spec["replicaIndex"] is not None else 0
            pod = self.builder._build_pod(cluster, (spec["groupIndex"], idx, spec["hostIndex"], spec["replicaName"]))
        try:
            self.client.create_pod(pod)
        except ApiError as e:
            raise gm.ApiError(str(e))
        return pod["name"]

    def replica_group_name(self, group):
        return f"{group}-{self.client.gen_suffix()}"

    def update_head_annotations(self, pod, ann):
        cur = self.client.pods.get((gm.ns_of(pod), pod["name"]))
        if cur is not None:
            cur.setdefault("annotations", {}).update(ann)

    def event(self, kind, reason, msg):
        self.client.events.append((kind, reason, msg))


def cluster_hash(c) -> str:
    """GenerateHashWithoutReplicasAndWorkersToDelete's digest of the muted spec (the JSON itself is pinned by test_spec_json)."""
    raw = c["specJson"] if "specJson" in c else snapmod.spec_hash_input(c.get("spec") or {})
    raw = raw.encode() if isinstance(raw, str) else bytes(raw)
    return base64.b32hexencode(hashlib.sha1(raw).digest()).decode()


def model_pass(client: FakeClient, env: Env, key, now="now"):
    """One Reconcile of RayCluster `key` by the model, on the client as it stands."""
    m = gm.Model(ModelApi(client, env), copy.deepcopy(client.list_pods()), env.status_conditions_gate, env.multihost_indexing_gate,
                 env.enable_random_pod_delete)
    c = copy.deepcopy(client.clusters[key])
    out = m.reconcile(c, cluster_hash(c), fresh_pods=lambda: copy.deepcopy(client.list_pods()), now=now)
    if out["written"] is not None:
        client.clusters[key]["status"] = out["written"]
    return out


NS, CN = "default", "raycluster-sample"


def test_model_reconcile_scenarios():
    """The scenario tests on fixture F0 (raycluster_controller_unit_test.go:417-1010, 2093-2378), through the model."""
    from test_golden import SC, make_client
    for sc in SC["scenarios"]:
        client = make_client(sc)
        before = {p["name"] for p in client.pods_of(NS, CN, **{"ray.io/group": "small-group"})}
        m = gm.Model(ModelApi(client, Env(**sc.get("env", {}))), copy.deepcopy(client.list_pods()), **sc.get("env", {}))
        c = client.clusters[(NS, CN)]
        err = m.reconcile_pods(c, cluster_hash(c))
        assert (err is not None) == sc["want_err"], (sc["name"], err)
        after = {p["name"] for p in client.pods_of(NS, CN, **{"ray.io/group": "small-group"})}
        assert len(after) == sc["want_workers"], sc["name"]
        assert not set(sc.get("want_gone", [])) & after, sc["name"]
        if "want_heads" in sc:
            assert len(client.pods_of(NS, CN, **{"ray.io/node-type": "head"})) == sc["want_heads"], sc["name"]
        if "want_creates" in sc:
            assert (len(after - before), len(before - after)) == (sc["want_creates"], sc["want_deletes"]), sc["name"]


def test_model_recreate_upgrade():
    """TestShouldRecreatePodsForUpgrade (raycluster_controller_unit_test.go:3680-3814)."""
    from test_golden import SC
    for case in load("recreate_upgrade")["cases"]:
        cluster = copy.deepcopy(SC["base"]["cluster"])
        cluster["spec"]["upgradeStrategy"] = case["upgradeStrategy"]
        cur = cluster_hash(cluster)
        pods = []
        if case["head"] is not None:
            hp = copy.deepcopy(SC["base"]["pods"][0])
            hp["annotations"] = {gm.RECREATE_HASH_ANNOT: cur if case["head"]["hash"] == "<current>" else case["head"]["hash"],
                                 gm.KUBERAY_VERSION_ANNOT: gm.KUBERAY_VERSION if case["head"]["version"] == "<current>" else case["head"]["version"]}
            pods.append(hp)
        client = FakeClient([cluster], pods)
        m = gm.Model(ModelApi(client, Env()), copy.deepcopy(client.list_pods()))
        assert m.should_recreate_pods_for_upgrade(cluster, cur) == case["want"], case["name"]


def test_model_status_scenarios():
    """TestCalculateStatus and TestRayClusterProvisionedCondition (raycluster_controller_unit_test.go:1611-1723, 1946-2042)."""
    from test_golden import status_fixture
    gold = load("status_scenarios")
    cluster, pods = status_fixture()
    m = gm.Model(None, pods, status_conditions_gate=False)
    new, err = m.calculate_status(cluster, None)
    cs = gold["calculate_status"]
    assert err is None and new["state"] == "ready" and new["head"]["podIP"] == cs["headNodeIP"] and new["head"]["serviceIP"] == cs["headServiceIP"]
    cluster, pods = status_fixture(n_workers=0)
    new, _ = gm.Model(None, pods).calculate_status(cluster, None)
    assert (new.get("state", ""), new.get("reason", "")) == (gold["without_desired"]["want_state"], gold["without_desired"]["want_reason"])
    cluster, pods = status_fixture(n_workers=1, ready="False")
    cluster["spec"]["workerGroupSpecs"][0]["replicas"] = 1
    for st in gold["provisioned"]["steps"]:
        pods[0]["conditions"] = [{"type": "Ready", "status": st["head_ready"]}]
        pods[1]["conditions"] = [{"type": "Ready", "status": st["worker_ready"]}]
        new, err = gm.Model(None, pods).calculate_status(cluster, None)
        c = next(c for c in new["conditions"] if c["type"] == "RayClusterProvisioned")
        assert [c["status"], c["reason"]] == st["want"]
        cluster["status"] = new
    cluster, pods = status_fixture()
    new, _ = gm.Model(None, pods).calculate_status(cluster, gm.GoError("invalid", "FailedCreateHeadPod"))
    rf = next(c for c in new["conditions"] if c["type"] == "ReplicaFailure")
    assert (rf["status"], rf["reason"], rf["message"]) == ("True", "FailedCreateHeadPod", "FailedCreateHeadPod\ninvalid")


# ------------------------------------------------------------------------------------------ inputs
def inputs(seed, max_clusters=10):
    """fuzz_objects.generate(seed), plus what the fuzzer never produces: real containers and container states instead of the
    rayContainerTerminated shortcut (an empty terminated state among them), empty replica-name labels, head Service ports, deletionTimestamp together with suspend, and Recreate heads that
    carry the current digest and version.  Condition statuses are True, False or Unknown: metav1.Condition's enum and the
    kubelet's Pod conditions allow nothing else.  -> (clusters, pods, jobs, Env, rng)"""
    clusters, pods, jobs = fuzz_objects.generate(seed, max_clusters=max_clusters)
    return decorate(clusters, pods, jobs, seed)


def decorate(clusters, pods, jobs, seed):
    rng = np.random.default_rng(seed ^ 0x60DE1)
    for p in pods:
        term = p.pop("rayContainerTerminated", False)
        name = "ray-head" if gm.node_type(p) == "head" else "ray-worker"
        p["containers"] = [{"name": name}, {"name": "sidecar"}]
        sts = []
        if rng.random() < 0.3:
            sts.append({"name": "sidecar", "state": {"waiting": {"reason": "PodInitializing", "message": "init"}}})
        if term:
            sts.append({"name": name, "state": {"terminated": {"exitCode": int(rng.integers(0, 3)), "reason": "Error", "message": "ray exited"}}})
        elif rng.random() < 0.05:   # a terminated state with every field unset is still a non-nil pointer in Go
            sts.append({"name": name, "state": {"terminated": {}}})
        elif rng.random() < 0.4:
            sts.append({"name": name, "state": {"waiting": {"reason": "CrashLoopBackOff", "message": "back-off"}}})
        rng.shuffle(sts)
        p["containerStatuses"] = sts
        for c in p.get("conditions") or []:
            c["status"] = c.get("status") or "Unknown"
        if gm.node_type(p) == "worker" and gm.REPLICA_NAME_LABEL not in p["labels"] and rng.random() < 0.1:
            p["labels"][gm.REPLICA_NAME_LABEL] = ""   # present but empty: a replica group of its own, unlike an absent label
    for c in clusters:
        for cond in (c.get("status") or {}).get("conditions") or []:
            cond["status"] = cond.get("status") or "Unknown"
        svc = c.get("headService")
        if svc is not None and rng.random() < 0.6:
            svc["ports"] = [{"name": "dashboard", "targetPort": 8265}, {"name": "client", "nodePort": 30001}, {"name": "", "targetPort": 1},
                            {"name": "serve", "targetPort": "serve-port"}][: int(rng.integers(1, 5))]
        spec = c["spec"]
        if rng.random() < 0.06:
            c["deletionTimestamp"], spec["suspend"] = "2026-01-01T00:00:00Z", True
        if (spec.get("upgradeStrategy") or {}).get("type") == "Recreate" and rng.random() < 0.5:
            for p in pods:
                if gm.ns_of(p) == c["namespace"] and (p.get("labels") or {}).get(gm.CLUSTER_LABEL) == c["name"] and gm.node_type(p) == "head":
                    p["annotations"] = {gm.RECREATE_HASH_ANNOT: cluster_hash(c), gm.KUBERAY_VERSION_ANNOT: gm.KUBERAY_VERSION}
    env = Env(status_conditions_gate=bool(rng.random() < 0.75), multihost_indexing_gate=bool(rng.random() < 0.75),
              enable_random_pod_delete=bool(rng.random() < 0.4))
    return clusters, pods, jobs, env, rng


# ------------------------------------------------------------------------------------------ closed-loop rounds
def describe_create(pod):
    lb = pod.get("labels") or {}
    return (gm.ns_of(pod), lb.get(gm.NODE_TYPE_LABEL), lb.get(gm.GROUP_LABEL), lb.get(gm.REPLICA_INDEX_LABEL), lb.get(HOST_INDEX_LABEL),
            lb.get(gm.REPLICA_NAME_LABEL), pod["name"][:-5])


class RecordingClient(FakeClient):
    """FakeClient that logs every Delete that removed a Pod and every Create that stored one."""

    def __init__(self, *a):
        super().__init__(*a)
        self.log = []

    def delete_pod(self, ns, name):
        gone = super().delete_pod(ns, name)
        if gone:
            self.log.append(("delete", (ns, name)))
        return gone

    def create_pod(self, pod):
        super().create_pod(pod)
        self.log.append(("create", describe_create(pod)))


def _mark(client):
    return len(client.log), len(client.events)


def _observe(client, mark):
    log = client.log[mark[0]:]
    return {"deleted": sorted(k for op, k in log if op == "delete"), "created": [k for op, k in log if op == "create"],
            "events": client.events[mark[1]:]}


def engine_round(client, backend, env, now):
    """RayClusterReconciler over `backend`: one pass, then every RayCluster's side effects and status in key order."""
    r = RayClusterReconciler(client, backend, env)
    pr = r._pass()
    out = {}
    for ci, key in enumerate(pr.meta.cluster_keys):
        mark = _mark(client)
        old = client.clusters[key].get("status")
        requeue, err = r.reconcile_record(pr, ci, now)
        st = client.clusters[key].get("status")   # update_status stores a new object when it writes
        o = _observe(client, mark)
        o.update(error=err, requeue=requeue, written=copy.deepcopy(st) if st is not old else None)
        out[key] = o
    jobs = []
    for j in pr.res.jobs:
        ci = int(j["cluster_idx"])
        jobs.append({"cluster": None} if ci < 0 else {"cluster": pr.meta.cluster_keys[ci], "not_ready": bool(j["not_ready"]),
                                                       "status_changed": bool(j["status_changed"])})
    return out, jobs, pr


def model_round(client, env, now):
    """go_model: every RayCluster decided from the state at the start of the round, applied in key order."""
    cache = copy.deepcopy(client.list_pods())
    pre = copy.deepcopy(client.clusters)
    m = gm.Model(ModelApi(client, env), cache, env.status_conditions_gate, env.multihost_indexing_gate, env.enable_random_pod_delete)
    jobs = [gm.rayjob_rollup(j, pre) for j in client.jobs]
    out = {}
    for key in sorted(pre):
        mark = _mark(client)
        res = m.reconcile(pre[key], cluster_hash(pre[key]), fresh_pods=lambda: copy.deepcopy(client.list_pods()), now=now)
        if res["written"] is not None:
            client.clusters[key]["status"] = res["written"]
        o = _observe(client, mark)
        o.update(error=res["error"], requeue=res["requeue"], written=copy.deepcopy(res["written"]))
        out[key] = o
    return out, jobs


def _norm_status(st):
    if st is None:
        return None
    st = copy.deepcopy(st)
    for k in ("conditions", "state", "reason"):   # Go's zero values: a nil slice, an empty string
        if not st.get(k):
            st.pop(k, None)
    return st


def _client_text(client):
    return pprint.pformat({"pods": client.pods, "clusters": {k: _norm_status(c.get("status")) for k, c in client.clusters.items()}},
                          width=160).splitlines()


# record fields a decision maps to, named when a round differs (triage only)
FIELD_OF = {"deleted": "act_code / act_pod_idx (and wtd_pod_idx)", "created": "groups.n_create / create_idx, head_action",
            "events": "path, head_action, groups.flags", "error": "err_kind / err_arg, groups.flags (ABORTED)",
            "written": "needs_status_write, new_state, counts, cond_status / cond_variant, head_ids", "requeue": "needs_status_write, err_kind"}


def compare_round(seed, rnd, eng, mod, eng_client, mod_client):
    for key in sorted(set(eng) | set(mod)):
        e, m = eng.get(key), mod.get(key)
        assert e is not None and m is not None, (seed, rnd, key)
        for field in ("deleted", "created", "events", "error", "requeue"):
            if e[field] != m[field]:
                diff = "\n".join(difflib.unified_diff(_client_text(mod_client), _client_text(eng_client), "model", "engine", lineterm="", n=2))
                pytest.fail(f"seed {seed} round {rnd} cluster {key}: {field} ({FIELD_OF[field]})\n engine: {e[field]!r}\n  model: {m[field]!r}\n"
                            f"{diff[:6000]}")
        if (e["written"] is None) != (m["written"] is None) or _norm_status(e["written"]) != _norm_status(m["written"]):
            pytest.fail(f"seed {seed} round {rnd} cluster {key}: written status ({FIELD_OF['written']})\n engine: "
                        f"{pprint.pformat(_norm_status(e['written']), width=160)}\n  model: {pprint.pformat(_norm_status(m['written']), width=160)}")


def mark_running(client, rng):
    """As the envtest suites do (raycluster_controller_test.go:197-199): some Pods without a phase turn Running and Ready."""
    for k in sorted(client.pods):
        p = client.pods[k]
        if p.get("phase", "") == "" and rng.random() < 0.7:
            p["phase"] = "Running"
            p["conditions"] = [{"type": "Ready", "status": "True"}]
            p["podIP"] = "10.2.0.1"


def run_stream(seed, backend, clusters, pods, jobs, env, rng, rounds=3, failures=True, stats=None):
    """Twin clients through `rounds` rounds; the first difference fails with the seed, round, RayCluster and a diff."""
    base = RecordingClient(clusters, pods, jobs)
    if failures and rng.random() < 0.3:
        keys = sorted(base.pods)
        for i in rng.choice(len(keys), size=min(len(keys), 3), replace=False) if keys else []:
            base.fail_delete.add(keys[int(i)])
        if rng.random() < 0.5:
            base.fail_create.add(str(rng.choice(["head", "worker"])))
    eng_client, mod_client = copy.deepcopy(base), copy.deepcopy(base)
    stats = stats if stats is not None else {}
    for rnd in range(rounds):
        now = f"t{rnd}"
        eng, eng_jobs, pr = engine_round(eng_client, backend, env, now)
        mod, mod_jobs = model_round(mod_client, env, now)
        compare_round(seed, rnd, eng, mod, eng_client, mod_client)
        assert eng_jobs == mod_jobs, f"seed {seed} round {rnd}: RayJob results\n engine {eng_jobs}\n  model {mod_jobs}"
        assert eng_client.pods == mod_client.pods and eng_client.events == mod_client.events
        for o in mod.values():
            stats["deleted"] = stats.get("deleted", 0) + len(o["deleted"])
            stats["created"] = stats.get("created", 0) + len(o["created"])
            stats["written"] = stats.get("written", 0) + (o["written"] is not None)
            stats["warnings"] = stats.get("warnings", 0) + sum(1 for ev in o["events"] if ev[0] == "Warning")
            stats["errors"] = stats.get("errors", 0) + (o["error"] is not None)
        stats["clusters"] = max(stats.get("clusters", 0), len(pr.meta.cluster_keys))
        r2 = np.random.default_rng(seed * 31 + rnd)
        mark_running(eng_client, r2)
        mark_running(mod_client, np.random.default_rng(seed * 31 + rnd))
    return stats


class OracleBackend:
    def run(self, snap, flags):
        from oracle import oracle
        return oracle.run(snap, flags)


ORACLE_SEEDS = range(300)


def test_oracle_streams_against_the_model():
    """The CPU oracle through RayClusterReconciler == go_model, round after round, on decorated fuzz fleets."""
    stats = {}
    for seed in ORACLE_SEEDS:
        clusters, pods, jobs, env, rng = inputs(seed)
        run_stream(seed, OracleBackend(), clusters, pods, jobs, env, rng, stats=stats)
    for k in ("deleted", "created", "written", "warnings", "errors"):
        assert stats[k] > 0, stats


def wrapped_desired_stream(backend, autoscaling: bool, seed=0):
    """replicas 2^30 x numOfHosts 2 with the multi-host gate off: GetWorkerGroupDesiredReplicas wraps to -2^31 (an int32 multiply,
    utils/util.go:403), and reconcilePods takes diff = -2^31 - running in Go int (:757, :849): a scale-down past the running Pods
    without the autoscaler, nothing with it, and never 2^31 creates.  -> the stream's counters"""
    cluster = {"namespace": NS, "name": "wrap", "uid": "uid-wrap", "specJson": '{"wrap":1}', "status": {},
               "spec": {"enableInTreeAutoscaling": autoscaling,
                        "workerGroupSpecs": [{"groupName": "g", "replicas": 2 ** 30, "minReplicas": 0, "maxReplicas": 2 ** 31 - 1, "numOfHosts": 2}]}}
    ready = [{"type": "Ready", "status": "True"}]
    pods = [{"namespace": NS, "name": "wrap-head", "labels": {gm.CLUSTER_LABEL: "wrap", gm.NODE_TYPE_LABEL: "head"}, "phase": "Running",
             "conditions": ready, "podIP": "10.4.0.1"}]
    pods += [{"namespace": NS, "name": f"wrap-w{i}", "labels": {gm.CLUSTER_LABEL: "wrap", gm.NODE_TYPE_LABEL: "worker", gm.GROUP_LABEL: "g"},
              "phase": "Running", "conditions": ready} for i in range(3)]
    env = Env(multihost_indexing_gate=False)
    return run_stream(seed, backend, [cluster], pods, [], env, np.random.default_rng(seed), rounds=2, failures=False)


@pytest.mark.parametrize("autoscaling", [False, True])
def test_wrapped_desired_replicas_scale_down_not_up(autoscaling):
    stats = wrapped_desired_stream(OracleBackend(), autoscaling)
    assert stats["created"] == 0 and stats["deleted"] == (0 if autoscaling else 3), stats

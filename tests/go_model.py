"""A plain, object-level restatement of KubeRay's RayCluster controller (no test_ prefix: pytest does not collect it).

It reads the fixture object model of tests/golden/README.md (RayCluster, Pod and RayJob dicts, as FakeClient holds them) and
states what `raycluster_controller.go` does with them: which Pods it deletes and creates, which events it records, what error it
returns and what status it writes.  It shares nothing with the engine or the CPU oracle: no packer, no columns, no enums, no
imports from kuberay_b200 or oracle.  It is slow on purpose; every function cites the reference lines it restates (paths
relative to ray-operator/controllers/ray/).

Inputs that stand for calls outside reconcilePods, as kuberay_b200/snapshot.py documents them:
  * `expectations{head, <group>}`: rayClusterScaleExpectation.IsSatisfied per group (default satisfied);
  * `headService{count, clusterIP, name, ports}`: the head Services a List finds (default one, 10.0.0.1, <name>-head-svc);
  * `extErr{kind, message}`: an earlier sub-reconciler's error (:308-314), so reconcilePods is not reached.  kind 1 is a plain
    error, 2..6 carry one of the five ErrFailed* markers (utils/constant.go:322-328) in that order, 7 means "no error, status
    only".

Lists read the informer cache, which is the state at the start of the round (`pods`).  Create and Delete go to the API (`api`):
  api.delete(ns, name) -> bool           False on NotFound; raises ApiError on any other failure
  api.delete_collection(pods)            DeleteAllOf over the listed Pods; raises ApiError on a failure
  api.create(cluster, spec) -> str       the new Pod's name; spec = {nodeType, group, groupIndex, replicaIndex, hostIndex, replicaName}; raises ApiError
  api.replica_group_name(group) -> str   utils.GenerateRayWorkerReplicaGroupName (utils/util.go:377-379)
  api.event(type, reason, message)

Three places follow a convention the engine and its host mirror (kuberay_b200/reconciler.py) share instead of Go, marked
"(shared convention)" where they occur:
  * a random scale-down past the end of runningPods (:916-917, reachable only with a negative desired count) panics in Go, so
    calculateStatus never runs; here it ends reconcilePods with the error "negative desired replicas (N)" and the status is
    calculated and written as for any other error;
  * calculateStatus errors keep only their leading text: Go appends the List's filter labels (common/association.go:193,
    raycluster_controller.go:1727-1731);
  * calculateStatus lists the cache as it was at the start of the round, and the Pods as they stand only after a Create or
    Delete failed: the engine computes a RayCluster's status in the same pass as its decisions and recomputes it after a failure.
"""
from __future__ import annotations

import copy
import re

# utils/constant.go:19-48
CLUSTER_LABEL = "ray.io/cluster"
NODE_TYPE_LABEL = "ray.io/node-type"
GROUP_LABEL = "ray.io/group"
REPLICA_NAME_LABEL = "ray.io/worker-group-replica-name"
REPLICA_INDEX_LABEL = "ray.io/worker-group-replica-index"
RECREATE_HASH_ANNOT = "ray.io/upgrade-strategy-recreate-hash"   # utils/constant.go:27
KUBERAY_VERSION_ANNOT = "ray.io/kuberay-version"                 # utils/constant.go:29
SKIP_HEAD_RESTART_ANNOT = "ray.io/disable-provisioned-head-restart"  # utils/constant.go:34
KUBERAY_VERSION = "nightly"                                      # utils/constant.go:281
INT32_MAX, INT32_MIN = 2 ** 31 - 1, -2 ** 31
EXT_MARKERS = {2: "FailedDeleteAllPods", 3: "FailedDeleteHeadPod", 4: "FailedCreateHeadPod", 5: "FailedDeleteWorkerPod",
               6: "FailedCreateWorkerPod"}
ZERO_TIME = "{0001-01-01 00:00:00 +0000 UTC}"


class ApiError(Exception):
    """A Create or Delete the API server refused (anything but NotFound)."""


class GoError:
    """A Go error value: its Error() text, and the ErrFailed* marker errors.Join put in front of it, if any
    (utils/constant.go:313-336)."""

    def __init__(self, text: str, marker: str | None = None):
        self.marker = marker
        self.text = f"{marker}\n{text}" if marker else text

    def __repr__(self):
        return f"GoError({self.text!r})"


def ns_of(obj) -> str:
    return obj.get("namespace") or "default"   # utils.GetNamespace (utils/util.go:294-300)


def wrap32(x: int) -> int:
    return (x + 2 ** 31) % 2 ** 32 - 2 ** 31


def atoi(s) -> int | None:
    """strconv.Atoi: optional sign and ASCII digits, within Go's int (64 bits)."""
    if s is None or not re.fullmatch(r"[+-]?[0-9]+", s):
        return None
    v = int(s)
    return v if -2 ** 63 <= v < 2 ** 63 else None


# ------------------------------------------------------------------------------------------ replica arithmetic
def num_hosts(g) -> int:
    return wrap32(int(g.get("numOfHosts", 1)))   # a missing numOfHosts defaults to 1 in the CRD


def desired_replicas(g) -> int:
    """GetWorkerGroupDesiredReplicas (utils/util.go:386-404): the product is an int32 multiply."""
    mn = g.get("minReplicas")
    mn = 0 if mn is None else mn
    mx = g.get("maxReplicas")
    mx = INT32_MAX if mx is None else mx
    if g.get("suspend") is True:
        return 0
    r = g.get("replicas")
    w = mn if (r is None or r < mn) else (mx if r > mx else r)
    return wrap32(w * num_hosts(g))


def groups_of(cluster):
    return (cluster.get("spec") or {}).get("workerGroupSpecs") or []


def calculate_desired(cluster) -> int:
    """CalculateDesiredReplicas (utils/util.go:406-414), int32 sum."""
    return wrap32(sum(desired_replicas(g) for g in groups_of(cluster)))


def calculate_min(cluster) -> int:
    """CalculateMinReplicas (utils/util.go:416-428), int32 products and sum."""
    n = 0
    for g in groups_of(cluster):
        if g.get("suspend") is True:
            continue
        mn = g.get("minReplicas")
        n = wrap32(n + wrap32((0 if mn is None else mn) * num_hosts(g)))
    return n


def calculate_max(cluster) -> int:
    """CalculateMaxReplicas (utils/util.go:430-442): int64 sum, clamped to int32 (SafeInt64ToInt32 :284-292)."""
    n = 0
    for g in groups_of(cluster):
        if g.get("suspend") is True:
            continue
        mx = g.get("maxReplicas")
        n += (INT32_MAX if mx is None else mx) * num_hosts(g)
    return max(INT32_MIN, min(INT32_MAX, n))


def node_type(pod):
    return (pod.get("labels") or {}).get(NODE_TYPE_LABEL)


def is_running_and_ready(pod) -> bool:
    """IsRunningAndReady (utils/util.go:164-175)."""
    if pod.get("phase", "") != "Running":
        return False
    return any(c.get("type") == "Ready" and c.get("status") == "True" for c in pod.get("conditions") or [])


def calculate_ready(pods) -> int:
    """CalculateReadyReplicas (utils/util.go:444-458)."""
    return sum(1 for p in pods if node_type(p) == "worker" and is_running_and_ready(p))


def calculate_available(pods) -> int:
    """CalculateAvailableReplicas (utils/util.go:460-474)."""
    return sum(1 for p in pods if node_type(p) == "worker" and p.get("phase", "") == "Running")


def check_all_pods_running(pods) -> bool:
    """CheckAllPodsRunning (utils/util.go:583-603)."""
    if not pods:
        return False
    for p in pods:
        if p.get("phase", "") != "Running":
            return False
        if any(c.get("type") == "Ready" and c.get("status") != "True" for c in p.get("conditions") or []):
            return False
    return True


# ------------------------------------------------------------------------------------------ Pod predicates
def ray_container_terminated(pod) -> dict | None:
    """getRayContainerStateTerminated (raycluster_controller.go:1237-1248): the state of the status named like the first container."""
    containers = pod.get("containers") or []
    if not containers:
        return None
    for st in pod.get("containerStatuses") or []:
        if st.get("name") == containers[0].get("name"):
            return (st.get("state") or {}).get("terminated")
    return None


def fmt_terminated(t) -> str:
    """fmt's %v of a *corev1.ContainerStateTerminated: <nil>, or &{ExitCode Signal Reason Message StartedAt FinishedAt ContainerID}."""
    if t is None:
        return "<nil>"
    return (f"&{{{t.get('exitCode', 0)} {t.get('signal', 0)} {t.get('reason', '')} {t.get('message', '')} {ZERO_TIME} {ZERO_TIME} "
            f"{t.get('containerID', '')}}}")


def should_delete_pod(pod, ntype: str) -> tuple[bool, str]:
    """shouldDeletePod (raycluster_controller.go:1181-1231)."""
    ph, name, rp = pod.get("phase", ""), pod["name"], pod.get("restartPolicy", "")
    if ph in ("Failed", "Succeeded"):
        return True, (f"The {ntype} Pod {name} status is {ph} which is a terminal state. "
                      "KubeRay will delete the Pod and create new Pods in the next reconciliation if necessary.")
    term = ray_container_terminated(pod)
    if ph == "Running" and term is not None:
        if rp == "Never":
            return True, (f"The Pod status of the {ntype} Pod {name} is {ph}, and the Ray container terminated status is {fmt_terminated(term)}. "
                          f"The container is unable to restart due to its restart policy {rp}, so KubeRay will delete it.")
        return False, (f"The Pod status of the {ntype} Pod {name} is {ph}, and the Ray container terminated status is {fmt_terminated(term)}. "
                       f"However, KubeRay will not delete the Pod because its restartPolicy is set to {rp} and it should be able to restart automatically.")
    return False, (f"KubeRay does not need to delete the {ntype} Pod {name}. The Pod status is {ph}, and the Ray container terminated status is "
                   f"{fmt_terminated(term)}.")


def pod_status_text(pod) -> str:
    """The "Pod status / restart policy / terminated status" tail of the delete events (:703-710, 798-805, 947-948)."""
    return (f"Pod status: {pod.get('phase', '')}; Pod restart policy: {pod.get('restartPolicy', '')}; "
            f"Ray container terminated status: {fmt_terminated(ray_container_terminated(pod))}")


def find_head_pod_ready_condition(pod) -> dict:
    """FindHeadPodReadyCondition and firstNotReadyContainerStatus (utils/util.go:81-135)."""
    out = {"type": "HeadPodReady", "status": "False", "reason": "Unknown", "message": ""}
    for cond in pod.get("conditions") or []:
        if cond.get("type") != "Ready":
            continue
        out["status"] = cond.get("status", "")
        out["message"] = cond.get("message", "")
        reason = cond.get("reason", "")
        if cond.get("status") == "True" and reason == "":
            reason = "HeadPodRunningAndReady"
        if reason != "":
            out["reason"] = reason
        if reason == "ContainersNotReady":
            for st in pod.get("containerStatuses") or []:
                state = st.get("state") or {}
                sub = state.get("waiting") if state.get("waiting") is not None else state.get("terminated")
                if sub is not None:
                    if out["message"] != "":
                        out["message"] += "; "
                    out["message"] += f"{st.get('name', '')}: {sub.get('message', '')}"
                    out["reason"] = sub.get("reason", "")
                    break
        break
    return out


def find_suspend_status(status) -> str:
    """FindRayClusterSuspendStatus (utils/util.go:153-162)."""
    for c in (status or {}).get("conditions") or []:
        if c.get("type") in ("RayClusterSuspending", "RayClusterSuspended") and c.get("status") == "True":
            return c["type"]
    return ""


def set_condition(conds: list, new: dict):
    """meta.SetStatusCondition, without the wall-clock lastTransitionTime: update in place, or append."""
    for c in conds:
        if c.get("type") == new["type"]:
            c["status"], c["reason"], c["message"] = new["status"], new["reason"], new.get("message", "")
            return
    conds.append({"type": new["type"], "status": new["status"], "reason": new["reason"], "message": new.get("message", "")})


def _cond_key(c):
    return (c.get("type", ""), c.get("status", ""), c.get("reason", ""), c.get("message", ""), str(c.get("lastTransitionTime", "")),
            int(c.get("observedGeneration", 0)))


def _head_key(st):
    h = st.get("head") or {}
    return tuple(h.get(k, "") for k in ("podIP", "serviceIP", "podName", "serviceName"))


def inconsistent_status(old, new) -> bool:
    """InconsistentRayClusterStatus (utils/consistency.go:16-34): a nil endpoints map is not DeepEqual to an empty one."""
    old, new = old or {}, new or {}
    if old.get("state", "") != new.get("state", "") or old.get("reason", "") != new.get("reason", ""):
        return True
    for k in ("readyWorkerReplicas", "availableWorkerReplicas", "desiredWorkerReplicas", "minWorkerReplicas", "maxWorkerReplicas"):
        if int(old.get(k, 0)) != int(new.get(k, 0)):
            return True
    if old.get("endpoints") != new.get("endpoints") or (old.get("endpoints") is None) != (new.get("endpoints") is None):
        return True
    if _head_key(old) != _head_key(new):
        return True
    return [_cond_key(c) for c in old.get("conditions") or []] != [_cond_key(c) for c in new.get("conditions") or []]


def head_service(cluster) -> dict:
    return cluster.get("headService", {"count": 1, "clusterIP": "10.0.0.1", "name": f"{cluster['name']}-head-svc"})


# ------------------------------------------------------------------------------------------ the reconciler
class Model:
    """One RayClusterReconciler: the two feature gates and ENABLE_RANDOM_POD_DELETE, an API, and the informer cache's Pods."""

    def __init__(self, api, pods, status_conditions_gate=True, multihost_indexing_gate=True, enable_random_pod_delete=False):
        self.api = api
        self.pods = self.index(pods)
        self.gate_conditions = status_conditions_gate
        self.gate_multihost = multihost_indexing_gate
        self.random_delete = enable_random_pod_delete

    @staticmethod
    def index(pods) -> dict:
        """The cache's Pods by (namespace, ray.io/cluster label), each list name-ordered as fake-client Lists come back."""
        out: dict = {}
        for p in sorted(pods, key=lambda p: p["name"]):
            lb = p.get("labels") or {}
            if CLUSTER_LABEL in lb:
                out.setdefault((ns_of(p), lb[CLUSTER_LABEL]), []).append(p)
        return out

    # common/association.go: RayCluster{All,Head,Group}PodsAssociationOptions
    def list(self, cluster, pods=None, **labels):
        by_cluster = self.pods if pods is None else self.index(pods)
        return [p for p in by_cluster.get((ns_of(cluster), cluster["name"]), [])
                if all(k in (p.get("labels") or {}) and p["labels"][k] == v for k, v in labels.items())]

    def ev(self, kind, reason, msg):
        self.api.event(kind, reason, msg)

    def delete_all(self, pods):
        """deleteAllPods (raycluster_controller.go:130-146): one DeleteAllOf, only when a listed Pod is not terminating."""
        if any(not p.get("deletionTimestamp") for p in pods):
            self.api.delete_collection(pods)

    def random_delete_enabled(self, cluster) -> bool:
        """:898-912 and :1097-1104."""
        autoscaling = (cluster.get("spec") or {}).get("enableInTreeAutoscaling") is True
        return not autoscaling or self.random_delete

    # -------------------------------------------------------------------------------- reconcilePods (:619-935)
    def reconcile_pods(self, cluster, cluster_hash: str) -> GoError | None:
        spec = cluster.get("spec") or {}
        ns, name = ns_of(cluster), cluster["name"]
        exp = cluster.get("expectations") or {}
        suspend_status = find_suspend_status(cluster.get("status"))
        if suspend_status == "RayClusterSuspending" or (not self.gate_conditions and spec.get("suspend") is True):   # :628-644
            try:
                self.delete_all(self.list(cluster))
            except ApiError as e:
                self.ev("Warning", "FailedToDeletePodCollection", f"Failed deleting Pods due to suspension for RayCluster {ns}/{name}, {e}")
                return GoError(str(e), "FailedDeleteAllPods")
            self.ev("Normal", "DeletedPod", f"Deleted Pods for RayCluster {ns}/{name} due to suspension")
            return None
        if self.gate_conditions and (suspend_status == "RayClusterSuspended" or spec.get("suspend") is True):   # :646-654
            return None
        if self.should_recreate_pods_for_upgrade(cluster, cluster_hash):   # :656-670
            try:
                self.delete_all(self.list(cluster))
            except ApiError as e:
                self.ev("Warning", "FailedToDeletePodCollection",
                        f"Failed deleting Pods due to spec change with Recreate upgradeStrategy for RayCluster {ns}/{name}, {e}")
                return GoError(str(e), "FailedDeleteAllPods")
            self.ev("Normal", "DeletedPod", f"Deleted all Pods for RayCluster {ns}/{name} due to spec change with Recreate upgradeStrategy")
            return None

        heads = self.list(cluster, **{NODE_TYPE_LABEL: "head"})   # :672-676
        if not exp.get("head", True):   # :689-690
            pass
        elif len(heads) == 1:   # :691-712
            hp = heads[0]
            delete, reason = should_delete_pod(hp, "head")
            if delete:
                try:
                    if not self.api.delete(ns_of(hp), hp["name"]):
                        raise ApiError(f'pods "{hp["name"]}" not found')
                except ApiError as e:
                    self.ev("Warning", "FailedToDeleteHeadPod", f"Failed deleting head Pod {ns_of(hp)}/{hp['name']}; {pod_status_text(hp)}, {e}")
                    return GoError(str(e), "FailedDeleteHeadPod")
                self.ev("Normal", "DeletedHeadPod", f"Deleted head Pod {ns_of(hp)}/{hp['name']}; {pod_status_text(hp)}")
                return GoError(reason)
        elif len(heads) == 0:   # :713-737
            provisioned = any(c.get("type") == "RayClusterProvisioned" and c.get("status") == "True"
                              for c in (cluster.get("status") or {}).get("conditions") or [])
            if provisioned and (cluster.get("annotations") or {}).get(SKIP_HEAD_RESTART_ANNOT) == "true":   # :1127-1129
                return None
            try:   # createHeadPod (:1307-1337): the Pod has only a generateName when Create fails
                pod_name = self.api.create(cluster, {"nodeType": "head", "groupIndex": -1, "hash": cluster_hash})
            except ApiError as e:
                self.ev("Warning", "FailedToCreateHeadPod", f"Failed to create head Pod {ns}/, {e}")
                return GoError(str(e), "FailedCreateHeadPod")
            self.ev("Normal", "CreatedHeadPod", f"Created head Pod {ns}/{pod_name}")
        else:   # :738-748
            names = " ".join(p["name"] for p in heads)
            return GoError(f"{len(heads)} head pods found [{names}]. Please delete extra head pods")

        for gi, worker in enumerate(groups_of(cluster)):   # :750-933
            gname = worker["groupName"]
            if not exp.get(gname, True):   # :752-755
                continue
            expected = desired_replicas(worker)   # :757
            pods = self.list(cluster, **{GROUP_LABEL: gname})   # :760-763
            if worker.get("suspend") is True:   # :765-775
                try:
                    self.delete_all(pods)
                except ApiError as e:
                    self.ev("Warning", "FailedToDeleteWorkerPodCollection",
                            f"Failed deleting worker Pods for suspended group {gname} in RayCluster {ns}/{name}, {e}")
                    return GoError(str(e), "FailedDeleteWorkerPod")
                self.ev("Normal", "DeletedWorkerPod", f"Deleted all pods for suspended worker group {gname} in RayCluster {ns}/{name}")
                continue
            if num_hosts(worker) > 1 and self.gate_multihost:   # :777-784
                err = self.reconcile_multihost(cluster, gi, worker, pods)
                if err is not None:
                    return err
                continue
            deleted = set()   # :786-812
            n_unhealthy = 0
            for p in pods:
                delete, _reason = should_delete_pod(p, "worker")
                if delete:
                    n_unhealthy += 1
                    deleted.add(p["name"])
                    try:
                        if not self.api.delete(ns_of(p), p["name"]):
                            raise ApiError(f'pods "{p["name"]}" not found')
                    except ApiError as e:
                        self.ev("Warning", "FailedToDeleteWorkerPod", f"Failed deleting worker Pod {ns_of(p)}/{p['name']}; {pod_status_text(p)}, {e}")
                        return GoError(str(e), "FailedDeleteWorkerPod")
                    self.ev("Normal", "DeletedWorkerPod", f"Deleted worker Pod {ns_of(p)}/{p['name']}; {pod_status_text(p)}")
            if n_unhealthy > 0:
                return GoError(f"delete {n_unhealthy} unhealthy worker Pods")
            for victim in worker.get("workersToDelete") or []:   # :814-835
                try:
                    if self.api.delete(ns, victim):
                        deleted.add(victim)
                        self.ev("Normal", "DeletedWorkerPod", f"Deleted pod {ns}/{victim}")
                except ApiError as e:
                    self.ev("Warning", "FailedToDeleteWorkerPod", f"Failed deleting pod {ns}/{victim}, {e}")
                    return GoError(str(e), "FailedDeleteWorkerPod")
            running = [p for p in pods if p["name"] not in deleted]   # :837-842
            diff = expected - len(running)   # :849 (Go int: no wrap at these sizes)
            used = set()   # :853-864
            if self.gate_multihost:
                for p in running:
                    v = atoi((p.get("labels") or {}).get(REPLICA_INDEX_LABEL))
                    if v is not None:
                        used.add(v)
            if diff > 0:   # :865-890
                idx = 0
                for _ in range(diff):
                    if self.gate_multihost:
                        while idx in used:
                            idx += 1
                        used.add(idx)
                    err = self.create_worker(cluster, {"nodeType": "worker", "group": gname, "groupIndex": gi,
                                                       "replicaIndex": idx if self.gate_multihost else None, "hostIndex": 0, "replicaName": ""})
                    if err:
                        return err
            elif diff < 0 and self.random_delete_enabled(cluster):   # :894-928
                for i in range(-diff):
                    if i >= len(running):   # runningPods.Items[i] past the end: Go panics here (shared convention: an error)
                        return GoError(f"negative desired replicas ({expected})")
                    p = running[i]
                    try:
                        self.api.delete(ns_of(p), p["name"])
                    except ApiError as e:
                        self.ev("Warning", "FailedToDeleteWorkerPod", f"Failed deleting Pod {ns_of(p)}/{p['name']}, {e}")
                        return GoError(str(e), "FailedDeleteWorkerPod")
                    self.ev("Normal", "DeletedWorkerPod", f"Deleted Pod {ns_of(p)}/{p['name']}")
        return None

    def create_worker(self, cluster, spec) -> GoError | None:
        """createWorkerPod / createWorkerPodWithIndex (:1339-1385)."""
        ns = ns_of(cluster)
        try:
            pod_name = self.api.create(cluster, spec)
        except ApiError as e:
            self.ev("Warning", "FailedToCreateWorkerPod", f"Failed to create worker Pod for the cluster {ns}/{cluster['name']}, {e}")
            return GoError(str(e), "FailedCreateWorkerPod")
        self.ev("Normal", "CreatedWorkerPod", f"Created worker Pod {ns}/{pod_name}")
        return None

    def delete_pods(self, cluster, pods, gname, reason):
        """deletePods (raycluster_controller.go:937-956): NotFound is skipped without an event."""
        for p in pods:
            try:
                if not self.api.delete(ns_of(p), p["name"]):
                    continue
            except ApiError as e:
                self.ev("Warning", "FailedToDeleteWorkerPod", f"Failed deleting worker Pod {ns_of(p)}/{p['name']} for group {gname}; {pod_status_text(p)}, {e}")
                return GoError(str(e), "FailedDeleteWorkerPod")
            self.ev("Normal", "DeletedWorkerPod", f"Deleted worker Pod {ns_of(p)}/{p['name']} for group {gname}: {reason}")
        return None

    def reconcile_multihost(self, cluster, gi, worker, pods) -> GoError | None:
        """reconcileMultiHostWorkerGroup (:963-1125).  Where Go ranges over a map, replica groups are taken in order of their
        first Pod in the List (the engine's documented choice; Go's order is unspecified)."""
        gname, hosts = worker["groupName"], num_hosts(worker)
        replicas: dict[str, list] = {}   # :966-972
        for p in pods:
            lb = p.get("labels") or {}
            if REPLICA_NAME_LABEL in lb:
                replicas.setdefault(lb[REPLICA_NAME_LABEL], []).append(p)
        for rname, members in replicas.items():   # :974-984
            if len(members) < hosts:
                err = self.delete_pods(cluster, members, gname, "cleanup of incomplete multi-host group")
                return err or GoError(f"cleaned up incomplete replica group {rname}, requeueing")
        deleted = set()   # :986-1007
        for p in pods:
            if p["name"] in deleted:
                continue
            delete, reason = should_delete_pod(p, "worker")
            if delete:
                rname = (p.get("labels") or {}).get(REPLICA_NAME_LABEL, "")
                if rname not in replicas:
                    continue
                err = self.delete_pods(cluster, replicas[rname], gname, reason)
                if err:
                    return err
                deleted.update(m["name"] for m in replicas[rname])
        wtd = worker.get("workersToDelete") or []
        if wtd:   # :1009-1038
            victims: dict[str, dict] = {}
            for name in wtd:
                for p in pods:
                    if p["name"] == name:
                        for m in replicas.get((p.get("labels") or {}).get(REPLICA_NAME_LABEL, ""), []):
                            victims[m["name"]] = m
                        break
            if victims:
                # Go ranges over the map; the Pods are taken in List order
                order = [p for p in pods if p["name"] in victims]
                err = self.delete_pods(cluster, order, gname, "autoscaler scale-down request")
                return err or GoError(f"deleted {len(order)} worker Pods based on ScaleStrategy, requeueing")
        valid = [r for r, members in replicas.items() if not any(m["name"] in deleted for m in members)]   # :1040-1055
        expected = desired_replicas(worker)
        # :1058-1062: Go's % truncates toward zero
        if abs(expected) % hosts != 0:
            return GoError(f"desired worker pods ({expected}) is not a multiple of NumOfHosts ({hosts}) for group {gname}")
        to_create = int(expected / hosts) - len(valid)   # :1063-1064
        used = set()   # :1066-1077
        for r in valid:
            v = atoi((replicas[r][0].get("labels") or {}).get(REPLICA_INDEX_LABEL))
            if v is not None:
                used.add(v)
        if to_create > 0:   # :1079-1094
            idx = 0
            for _ in range(to_create):
                while idx in used:
                    idx += 1
                used.add(idx)
                rname = self.api.replica_group_name(gname)
                for j in range(hosts):
                    err = self.create_worker(cluster, {"nodeType": "worker", "group": gname, "groupIndex": gi, "replicaIndex": idx,
                                                       "hostIndex": j, "replicaName": rname})
                    if err:
                        return err
        elif to_create < 0 and self.random_delete_enabled(cluster):   # :1095-1118
            for r in valid[:-to_create]:
                err = self.delete_pods(cluster, replicas[r], gname, "scaling down")
                if err:
                    return err
        return None

    def should_recreate_pods_for_upgrade(self, cluster, cluster_hash: str) -> bool:
        """shouldRecreatePodsForUpgrade (:1131-1171).  A KubeRay version change rewrites the head's annotations through Update."""
        us = (cluster.get("spec") or {}).get("upgradeStrategy")
        if not isinstance(us, dict) or us.get("type") != "Recreate":
            return False
        heads = self.list(cluster, **{NODE_TYPE_LABEL: "head"})
        if heads:
            ann = heads[0].get("annotations") or {}
            version = ann.get(KUBERAY_VERSION_ANNOT, "")
            if version != "" and version != KUBERAY_VERSION:
                self.api.update_head_annotations(heads[0], {RECREATE_HASH_ANNOT: cluster_hash, KUBERAY_VERSION_ANNOT: KUBERAY_VERSION})
                return False
            actual = ann.get(RECREATE_HASH_ANNOT, "")
            if actual != "" and actual != cluster_hash:
                return True
        return False

    # -------------------------------------------------------------------------------- calculateStatus (:1552-1719)
    def calculate_status(self, cluster, reconcile_err: GoError | None, pods=None) -> tuple[dict | None, str | None]:
        """-> (new status without the wall-clock times, or None; the error calculateStatus returns)."""
        old = cluster.get("status") or {}
        new = copy.deepcopy(old)
        spec = cluster.get("spec") or {}
        conds = new.get("conditions") or []
        if self.gate_conditions:   # :1562-1577
            if reconcile_err is not None:
                if reconcile_err.marker:
                    set_condition(conds, {"type": "ReplicaFailure", "status": "True", "reason": reconcile_err.marker, "message": reconcile_err.text})
            else:
                conds[:] = [c for c in conds if c.get("type") != "ReplicaFailure"]
        runtime = self.list(cluster, pods)   # :1582-1585
        new["readyWorkerReplicas"] = calculate_ready(runtime)
        new["availableWorkerReplicas"] = calculate_available(runtime)
        new["desiredWorkerReplicas"] = calculate_desired(cluster)
        new["minWorkerReplicas"] = calculate_min(cluster)
        new["maxWorkerReplicas"] = calculate_max(cluster)
        if reconcile_err is None and len(runtime) == new["desiredWorkerReplicas"] + 1 and check_all_pods_running(runtime):   # :1599-1604
            new["state"] = "ready"
            new["reason"] = ""
        heads = [p for p in runtime if node_type(p) == "head"]   # common.GetRayClusterHeadPod (common/association.go)
        if len(heads) > 1:
            return None, "found multiple heads"   # (shared convention: without ". filter labels ...")
        head = heads[0] if heads else None
        if self.gate_conditions:   # :1606-1694
            if head is None:
                set_condition(conds, {"type": "HeadPodReady", "status": "False", "reason": "HeadPodNotFound", "message": "Head Pod not found"})
            else:
                set_condition(conds, find_head_pod_ready_condition(head))
            ss = find_suspend_status(new)
            provisioned = any(c["type"] == "RayClusterProvisioned" and c.get("status") == "True" for c in conds)
            if not provisioned and ss != "RayClusterSuspended":
                if check_all_pods_running(runtime):
                    set_condition(conds, {"type": "RayClusterProvisioned", "status": "True", "reason": "AllPodRunningAndReadyFirstTime",
                                          "message": "All Ray Pods are ready for the first time"})
                else:
                    set_condition(conds, {"type": "RayClusterProvisioned", "status": "False", "reason": "RayClusterPodsProvisioning",
                                          "message": "RayCluster Pods are being provisioned for first time"})
            if ss == "RayClusterSuspending":
                if not runtime:
                    set_condition(conds, {"type": "RayClusterProvisioned", "status": "False", "reason": "RayClusterPodsProvisioning",
                                          "message": "RayCluster has been suspended"})
                    set_condition(conds, {"type": "RayClusterSuspending", "status": "False", "reason": "RayClusterSuspending"})
                    set_condition(conds, {"type": "RayClusterSuspended", "status": "True", "reason": "RayClusterSuspended"})
            elif ss == "RayClusterSuspended":
                if spec.get("suspend") is False:
                    set_condition(conds, {"type": "RayClusterSuspended", "status": "False", "reason": "RayClusterSuspended"})
            else:
                set_condition(conds, {"type": "RayClusterSuspended", "status": "False", "reason": "RayClusterSuspended"})
                set_condition(conds, {"type": "RayClusterSuspending", "status": "True" if spec.get("suspend") is True else "False",
                                      "reason": "RayClusterSuspending"})
        if conds or "conditions" in old:
            new["conditions"] = conds
        if spec.get("suspend") is True and not runtime:   # :1696-1698
            new["state"] = "suspended"
        svc = head_service(cluster)   # updateEndpoints (:1747-1783)
        if svc.get("count", 1) != 0:
            eps = dict(new.get("endpoints") or {})
            for port in svc.get("ports") or []:
                if not port.get("name"):
                    continue
                if port.get("nodePort", 0):
                    eps[port["name"]] = str(port["nodePort"])
                elif isinstance(port.get("targetPort"), int) and port["targetPort"] != 0:
                    eps[port["name"]] = str(port["targetPort"])
                elif isinstance(port.get("targetPort"), str) and port["targetPort"] != "":
                    eps[port["name"]] = port["targetPort"]
            new["endpoints"] = eps
        pod_ip, pod_name = (head.get("podIP", ""), head["name"]) if head is not None else ("", "")   # updateHeadInfo (:1785-1806)
        cnt, ip = svc.get("count", 1), svc.get("clusterIP", "")   # getHeadServiceIPAndName (:1721-1745)
        if cnt < 1:   # (shared convention: these three without ". cluster name ..., filter labels ...")
            return None, "unable to find head service"
        if cnt > 1:
            return None, "found multiple head services"
        if ip == "":
            return None, "head service IP is empty"
        svc_ip = pod_ip if ip == "None" else ip
        new["head"] = {"podIP": pod_ip, "serviceIP": svc_ip, "podName": pod_name, "serviceName": svc.get("name", "")}
        return new, None

    # -------------------------------------------------------------------------------- Reconcile (:291-355)
    def reconcile(self, cluster, cluster_hash: str, fresh_pods=None, now: str = "now") -> dict:
        """One Reconcile of one RayCluster.  `fresh_pods()` is the cache after this reconcile's own writes: calculateStatus lists
        it only when a Create or Delete failed (shared convention; Go lists after every reconcilePods).
        -> {error, requeue, status (None: not written), decided status (None: calculateStatus failed)}."""
        if cluster.get("deletionTimestamp"):   # :291-294
            return {"error": None, "requeue": 0.0, "written": None, "status": None}
        ext = cluster.get("extErr") or {}
        kind = ext.get("kind", 0)
        if kind == 0:
            err = self.reconcile_pods(cluster, cluster_hash)
        elif kind == 7:
            err = None
        else:
            err = GoError(ext.get("message", ""), None)
            err.marker = EXT_MARKERS.get(kind)
        status_pods = fresh_pods() if (err is not None and err.marker and kind == 0) else None
        new, cerr = self.calculate_status(cluster, err, status_pods)
        written = None
        if cerr is None:
            new["lastUpdateTime"] = now
            if new.get("state", "") != (cluster.get("status") or {}).get("state", ""):   # :1711-1716
                new.setdefault("stateTransitionTimes", {})[new.get("state", "")] = now
            if inconsistent_status(cluster.get("status"), new):   # updateRayClusterStatus (:1951-1966)
                written = new
        final = err.text if err is not None else cerr
        requeue = 2.0 if (final is not None or written is not None) else 300.0   # :338-355
        return {"error": final, "requeue": requeue, "written": written, "status": new}


def rayjob_rollup(job, clusters: dict) -> dict:
    """What a RayJob reads of its RayCluster (rayjob_controller.go:203-216, 343) and whether its copy of the status changed
    (:880-905, InconsistentRayClusterStatus)."""
    name = (job.get("status") or {}).get("rayClusterName") or ""
    c = clusters.get((ns_of(job), name)) if name else None
    if c is None:
        return {"cluster": None}
    st = c.get("status") or {}
    return {"cluster": (ns_of(job), name), "not_ready": st.get("state", "") != "ready",
            "status_changed": inconsistent_status((job.get("status") or {}).get("rayClusterStatus"), st)}

"""Host-side mirror of the reference RayClusterReconciler for the hot path.

This is the Python statement of what the Go shim (INTEGRATION.md) does around the engine: it packs the watched objects,
asks a *backend* for one batched pass, and then performs the side effects the reference performs — Delete / Create /
Eventf / the returned error — in the reference's order, reading them off the DecisionRecord / StatusRecord instead of
recomputing them per object:

  reconcile_pods(instance)            ~ RayClusterReconciler.reconcilePods      (raycluster_controller.go:619-935)
  calculate_status(instance, err)     ~ RayClusterReconciler.calculateStatus     (raycluster_controller.go:1552-1719)
  update_status(instance, new)        ~ updateRayClusterStatus                   (raycluster_controller.go:1951-1966)

`backend` is anything with `run(snapshot, flags) -> abi.Results`: the CUDA engine (EngineBackend below) in production and
on the GPU tests; the tests inject the CPU oracle to pin the semantics against the reference's own test tables.
The FakeClient mirrors controller-runtime's fake client as the reference's unit tests use it: List returns objects ordered
by name, Delete removes immediately (raycluster_controller_unit_test.go:445-448,484).
"""
from __future__ import annotations

import copy
from dataclasses import dataclass, field

from . import abi
from . import podbuilder
from . import podmeta
from . import snapshot as snapmod

# event reasons (utils/constant.go:337-438)
EV_DELETED_POD = "DeletedPod"
EV_DELETED_HEAD_POD = "DeletedHeadPod"
EV_DELETED_WORKER_POD = "DeletedWorkerPod"
EV_CREATED_HEAD_POD = "CreatedHeadPod"
EV_CREATED_WORKER_POD = "CreatedWorkerPod"


@dataclass
class Env:
    """Process-level switches the reference reads at reconcile time."""
    status_conditions_gate: bool = True      # features.RayClusterStatusConditions
    multihost_indexing_gate: bool = True     # features.RayMultiHostIndexing
    enable_random_pod_delete: bool = False   # ENABLE_RANDOM_POD_DELETE == "true"


def _terminated_text(pod: dict) -> str:
    """fmt's %v of getRayContainerStateTerminated(pod) (raycluster_controller.go:1237-1248), a *ContainerStateTerminated:
    <nil>, or &{ExitCode Signal Reason Message StartedAt FinishedAt ContainerID} with zero times."""
    if not snapmod.ray_container_terminated(pod):
        return "<nil>"
    t = {}
    if "rayContainerTerminated" not in pod:
        ray_name = (pod.get("containers") or [{}])[0].get("name")
        t = next(((st.get("state") or {}).get("terminated") for st in pod.get("containerStatuses") or [] if st.get("name") == ray_name), {})
    zero = "{0001-01-01 00:00:00 +0000 UTC}"
    return f"&{{{t.get('exitCode', 0)} {t.get('signal', 0)} {t.get('reason', '')} {t.get('message', '')} {zero} {zero} {t.get('containerID', '')}}}"


def _should_delete(pod: dict) -> bool:
    """shouldDeletePod's verdict (raycluster_controller.go:1181-1231)."""
    ph = pod.get("phase", "")
    return ph in ("Failed", "Succeeded") or (ph == "Running" and snapmod.ray_container_terminated(pod) and pod.get("restartPolicy") == "Never")


def _pod_status_text(pod: dict) -> str:
    """The Pod part of the delete events (:703-710, 798-805, 947-948)."""
    return f"Pod status: {pod.get('phase', '')}; Pod restart policy: {pod.get('restartPolicy', '')}; Ray container terminated status: {_terminated_text(pod)}"


class ApiError(Exception):
    """A Create/Delete call that failed at the API server (anything but NotFound)."""


class FakeClient:
    """Minimal object store: RayClusters by (ns,name), Pods by (ns,name).  `fail_delete` / `fail_create` inject API-server
    failures (names / node types) the way the reference's tests do with interceptor funcs."""

    def __init__(self, clusters=(), pods=(), jobs=()):
        self.fail_delete: set[tuple[str, str]] = set()   # (ns, name) whose Delete returns an error
        self.fail_create: set[str] = set()               # node types ("head" / "worker") whose Create returns an error
        self.clusters = {(c.get("namespace", "default"), c["name"]): copy.deepcopy(c) for c in clusters}
        self.pods = {(p.get("namespace", "default"), p["name"]): copy.deepcopy(p) for p in pods}
        self.jobs = [copy.deepcopy(j) for j in jobs]
        self.events: list[tuple[str, str, str]] = []   # (type, reason, message)
        self._gen = 0

    def list_pods(self) -> list[dict]:
        return [self.pods[k] for k in sorted(self.pods)]  # fake client Lists come back name-ordered

    def delete_pod(self, ns: str, name: str) -> bool:
        """-> True if deleted, False if NotFound; raises ApiError on an injected failure."""
        if (ns, name) in self.fail_delete:
            raise ApiError(f"delete {ns}/{name}: injected failure")
        return self.pods.pop((ns, name), None) is not None

    def create_pod(self, pod: dict):
        if (pod.get("labels") or {}).get(snapmod.RAY_NODE_TYPE_LABEL) in self.fail_create:
            raise ApiError(f"create {pod.get('namespace', 'default')}/{pod['name']}: injected failure")
        self.pods[(pod.get("namespace", "default"), pod["name"])] = pod

    def gen_suffix(self) -> str:
        self._gen += 1
        return f"{self._gen:05d}"

    def pods_of(self, ns: str, cluster: str, **labels) -> list[dict]:
        out = []
        for p in self.list_pods():
            lb = p.get("labels") or {}
            if p.get("namespace", "default") == ns and lb.get(snapmod.RAY_CLUSTER_LABEL) == cluster and all(lb.get(k) == v for k, v in labels.items()):
                out.append(p)
        return out


class EngineBackend:
    """The product backend: the CUDA engine through the C ABI (raises if the library / a GPU is missing)."""

    def __init__(self, device: int = 0):
        self.device = device

    def run(self, snap, flags):
        from .engine import Engine
        eng = Engine.for_snapshot(snap, device=self.device)
        try:
            eng.load(snap)
            return eng.reconcile(flags)
        finally:
            eng.close()


@dataclass
class PassResult:
    snap: object
    meta: snapmod.PackMeta
    res: abi.Results
    pods: list = field(default_factory=list)


class RayClusterReconciler:
    def __init__(self, client: FakeClient, backend, env: Env | None = None):
        self.client = client
        self.backend = backend
        self.env = env or Env()

    # ------------------------------------------------------------------ one batched pass over everything in the client
    def _pass(self, overrides: dict | None = None) -> PassResult:
        clusters = []
        for key in sorted(self.client.clusters):
            c = copy.deepcopy(self.client.clusters[key])
            if overrides and key in overrides:
                c.update(overrides[key])
            clusters.append(c)
        pods = self.client.list_pods()
        snap, meta = snapmod.pack_objects(clusters, pods, self.client.jobs)
        f = meta.flags
        f.gate_status_conditions = 1 if self.env.status_conditions_gate else 0
        f.gate_multihost_indexing = 1 if self.env.multihost_indexing_gate else 0
        f.env_random_pod_delete = 1 if self.env.enable_random_pod_delete else 0
        f.fetch_pod_lists = 0  # the side effects below only need the compact action list
        res = self.backend.run(snap, f)
        return PassResult(snap, meta, res, pods)

    @staticmethod
    def _cluster_index(pr: PassResult, ns: str, name: str) -> int:
        return pr.meta.cluster_keys.index((ns, name))

    # ------------------------------------------------------------------ reconcilePods
    def reconcile_pods(self, ns: str, name: str) -> str | None:
        """Returns the error string reconcilePods would return, or None.  Side effects go to the FakeClient."""
        pr = self._pass()
        ci = self._cluster_index(pr, ns, name)
        return self._apply_decisions(pr, ci)

    def _apply_decisions(self, pr: PassResult, ci: int):
        """-> None, the plain error string reconcilePods returns, or ("Failed<Verb><Kind>Pod", message) when an API call
        failed: the reference records a Warning event, joins one of the five ErrFailed* markers (utils/constant.go:322-334)
        onto that error, and only those set the ReplicaFailure condition (raycluster_controller.go:1563-1571)."""
        self._stage = "FailedDeleteAllPods"
        self._warning = None   # (reason, message before the error) of the call in flight
        try:
            return self._apply_decisions_inner(pr, ci)
        except ApiError as ex:
            if self._warning:
                self.client.events.append(("Warning", self._warning[0], f"{self._warning[1]}, {ex}"))
            return (self._stage, str(ex))

    def _delete_listed(self, ns: str, name: str):
        """Delete of a Pod the List returned (:701, :796): NotFound is an error there, unlike at :823 and :920."""
        if not self.client.delete_pod(ns, name):
            raise ApiError(f'pods "{name}" not found')

    def _delete_collection(self, pods: list[tuple[str, str]], terminating: list[bool]):
        """deleteAllPods (:130-146): one DeleteAllOf, issued only when a listed Pod is not terminating yet."""
        if not all(terminating):
            for ns, name in pods:
                self.client.delete_pod(ns, name)

    def _apply_decisions_inner(self, pr: PassResult, ci: int) -> str | None:
        cl = self.client
        res, snap, meta = pr.res, pr.snap, pr.meta
        cr = res.clusters[ci]
        ns, cname = meta.cluster_keys[ci]
        cluster = cl.clusters[(ns, cname)]
        # the compact action list: only the pods this cluster must act on, in List order (what a shim running with
        # kr_flags.fetch_pod_lists = 0 downloads; the full sorted_pod_idx / sorted_action lists are not needed here)
        listed = [(int(res.act_pod_idx[i]), int(res.act_code[i])) for i in range(int(res.act_start[ci]), int(res.act_start[ci]) + int(res.act_cnt[ci]))]
        ev = cl.events.append
        path = int(cr["path"])
        if path == abi.PATH_SKIPPED:                # an earlier sub-reconciler's error is what Reconcile returns (:308-314)
            return (cluster.get("extErr") or {}).get("message", "") if cr["err_kind"] == abi.ERR_EXTERNAL else None
        if path == abi.PATH_SUSPENDING_DELETE_ALL:  # :633-643
            rows = [pi for pi, act in listed if act == abi.ACT_DELETE_ALL_SUSPEND]
            self._warning = ("FailedToDeletePodCollection", f"Failed deleting Pods due to suspension for RayCluster {ns}/{cname}")
            self._delete_collection([meta.pod_keys[pi] for pi in rows], [bool(pr.pods[pi].get("deletionTimestamp")) for pi in rows])
            ev(("Normal", EV_DELETED_POD, f"Deleted Pods for RayCluster {ns}/{cname} due to suspension"))
            return None
        if path == abi.PATH_SUSPENDED_NOOP:
            return None
        if path == abi.PATH_RECREATE_DELETE_ALL:    # :659-669
            rows = [pi for pi, act in listed if act == abi.ACT_DELETE_ALL_RECREATE]
            self._warning = ("FailedToDeletePodCollection", f"Failed deleting Pods due to spec change with Recreate upgradeStrategy for RayCluster {ns}/{cname}")
            self._delete_collection([meta.pod_keys[pi] for pi in rows], [bool(pr.pods[pi].get("deletionTimestamp")) for pi in rows])
            ev(("Normal", EV_DELETED_POD, f"Deleted all Pods for RayCluster {ns}/{cname} due to spec change with Recreate upgradeStrategy"))
            return None
        if cr["head_update_annotations"]:           # :1155-1162
            hp = cl.pods.get(meta.pod_keys[int(cr["head_pod_idx"])])
            if hp is not None:
                hp.setdefault("annotations", {})[snapmod.RECREATE_HASH_ANNOT] = bytes(res.hash[ci]).decode()
                hp["annotations"][snapmod.KUBERAY_VERSION_ANNOT] = snapmod.KUBERAY_VERSION
        ha = int(cr["head_action"])
        self._stage = "FailedDeleteHeadPod"         # :705
        if ha == abi.HEAD_DELETE:                   # :700-711
            pi = next(pi for pi, act in listed if act == abi.ACT_DELETE_HEAD)
            pod = pr.pods[pi]
            self._warning = ("FailedToDeleteHeadPod", f"Failed deleting head Pod {ns}/{pod['name']}; {_pod_status_text(pod)}")
            self._delete_listed(*meta.pod_keys[pi])
            ev(("Normal", EV_DELETED_HEAD_POD, f"Deleted head Pod {ns}/{pod['name']}; {_pod_status_text(pod)}"))
            return self._should_delete_reason(pod, "head")
        if ha == abi.HEAD_SKIP_RESTART:
            return None
        if ha == abi.HEAD_MULTIPLE:                 # :738-747
            names = [p["name"] for p in pr.pods if p.get("namespace", "default") == ns and (p.get("labels") or {}).get(snapmod.RAY_CLUSTER_LABEL) == cname
                     and p["labels"].get(snapmod.RAY_NODE_TYPE_LABEL) == "head"]  # the head List of :674, from the pass's cache
            return f"{int(cr['err_arg'])} head pods found [{' '.join(names)}]. Please delete extra head pods"   # %v of a []string
        self._stage = "FailedCreateHeadPod"         # :736
        if ha == abi.HEAD_CREATE:                   # :735, createHeadPod :1307-1337
            pod = self._build_pod(cluster, (-1, 0, 0, ""), cluster_hash=bytes(res.hash[ci]).decode())
            self._warning = ("FailedToCreateHeadPod", f"Failed to create head Pod {ns}/")   # :1330: the Pod has only a generateName
            cl.create_pod(pod)
            ev(("Normal", EV_CREATED_HEAD_POD, f"Created head Pod {ns}/{pod['name']}"))
        # worker groups in spec order (:751-933)
        groups = (cluster.get("spec") or {}).get("workerGroupSpecs") or []
        g0 = int(snap.c_group_off[ci])
        for gi, grp in enumerate(groups):
            gr = res.groups[g0 + gi]
            fl = int(gr["flags"])
            if not fl & abi.GR_PROCESSED:
                break
            gname = grp["groupName"]
            self._stage = "FailedDeleteWorkerPod"   # :770,800,826,922,949
            in_group = [(pi, act) for pi, act in listed if (pr.pods[pi].get("labels") or {}).get(snapmod.RAY_NODE_GROUP_LABEL) == gname]
            if fl & abi.GR_EXPECT_PENDING:
                continue
            if fl & abi.GR_SUSPENDED:               # :766-775
                rows = [pi for pi, act in in_group if act == abi.ACT_DELETE_GROUP_SUSPEND]
                self._warning = ("FailedToDeleteWorkerPodCollection", f"Failed deleting worker Pods for suspended group {gname} in RayCluster {ns}/{cname}")
                self._delete_collection([meta.pod_keys[pi] for pi in rows], [bool(pr.pods[pi].get("deletionTimestamp")) for pi in rows])
                ev(("Normal", EV_DELETED_WORKER_POD, f"Deleted all pods for suspended worker group {gname} in RayCluster {ns}/{cname}"))
                continue
            if fl & abi.GR_MULTIHOST:
                err = self._apply_multihost(pr, ci, gi, grp, in_group)
                if err:
                    return err
                continue
            unhealthy = [pi for pi, act in in_group if act == abi.ACT_DELETE_UNHEALTHY]
            for pi in unhealthy:                    # :790-806
                pod = pr.pods[pi]
                self._warning = ("FailedToDeleteWorkerPod", f"Failed deleting worker Pod {ns}/{pod['name']}; {_pod_status_text(pod)}")
                self._delete_listed(*meta.pod_keys[pi])
                ev(("Normal", EV_DELETED_WORKER_POD, f"Deleted worker Pod {ns}/{pod['name']}; {_pod_status_text(pod)}"))
            if unhealthy:
                return f"delete {len(unhealthy)} unhealthy worker Pods"  # :811
            if fl & abi.GR_WTD_EXECUTED:            # :817-835: one Delete per name, NotFound tolerated
                w0 = int(snap.g_wtd_off[g0 + gi])
                names = grp.get("workersToDelete") or (grp.get("scaleStrategy") or {}).get("workersToDelete") or []
                for k, nm in enumerate(names):
                    # Delete(ns, name) goes to the API server for EVERY name (:817-822): a Pod the informer snapshot does not
                    # hold yet (wtd_pod_idx == -1: not in the cache, or owned by another shard) is still deleted there;
                    # wtd_pod_idx only told the engine which listed pods leave runningPods (:837-842)
                    assert int(res.wtd_pod_idx[w0 + k]) < 0 or meta.pod_keys[int(res.wtd_pod_idx[w0 + k])] == (ns, nm)
                    self._warning = ("FailedToDeleteWorkerPod", f"Failed deleting pod {ns}/{nm}")
                    if cl.delete_pod(ns, nm):
                        ev(("Normal", EV_DELETED_WORKER_POD, f"Deleted pod {ns}/{nm}"))
                # (:835 clears worker.ScaleStrategy.WorkersToDelete on the loop's COPY of the group spec only — the CR keeps
                #  the names until the autoscaler removes them; later passes see NotFound and move on)
            self._stage = "FailedCreateWorkerPod"   # :879,887
            for k in range(int(gr["n_create"])):    # :865-890
                idx = int(res.create_idx[int(gr["create_off"]) + k])
                pod = self._build_pod(cluster, (gi, idx if self.env.multihost_indexing_gate else 0, 0, ""))   # :878 / :887
                self._warning = ("FailedToCreateWorkerPod", f"Failed to create worker Pod for the cluster {ns}/{cname}")
                cl.create_pod(pod)
                ev(("Normal", EV_CREATED_WORKER_POD, f"Created worker Pod {ns}/{pod['name']}"))
            self._stage = "FailedDeleteWorkerPod"   # :922
            for pi, act in in_group:                # :916-928
                if act == abi.ACT_DELETE_RANDOM:
                    self._warning = ("FailedToDeleteWorkerPod", f"Failed deleting Pod {ns}/{pr.pods[pi]['name']}")
                    cl.delete_pod(*meta.pod_keys[pi])
                    ev(("Normal", EV_DELETED_WORKER_POD, f"Deleted Pod {ns}/{pr.pods[pi]['name']}"))
            if fl & abi.GR_ABORTED:
                return f"negative desired replicas ({int(gr['expected'])})"
        return None

    def _apply_multihost(self, pr, ci, gi, grp, in_group) -> str | None:
        """reconcileMultiHostWorkerGroup side effects (:963-1125)."""
        cl, res, snap, meta = self.client, pr.res, pr.snap, pr.meta
        ns, cname = meta.cluster_keys[ci]
        cluster = cl.clusters[(ns, cname)]
        gr = res.groups[int(snap.c_group_off[ci]) + gi]
        cr = res.clusters[ci]
        gname = grp["groupName"]
        reasons = {abi.ACT_DELETE_MH_INCOMPLETE: "cleanup of incomplete multi-host group", abi.ACT_DELETE_MH_WTD: "autoscaler scale-down request",
                   abi.ACT_DELETE_MH_SCALE_DOWN: "scaling down"}
        # an unhealthy replica group is deleted with the reason of its first Pod (List order) that shouldDeletePod names (:992-999)
        trigger, rank = {}, {}
        for k, (pi, act) in enumerate(in_group):
            pod = pr.pods[pi]
            rname = (pod.get("labels") or {}).get(snapmod.REPLICA_NAME_LABEL)
            rank.setdefault(rname, k)
            if act == abi.ACT_DELETE_MH_UNHEALTHY and _should_delete(pod) and rname not in trigger:
                trigger[rname], rank[rname] = pod, k
        # deletePods runs one replica group at a time: unhealthy groups in the order of their trigger, then the others in the order
        # of their first Pod (:986-1007, 1108-1118)
        order = sorted(in_group, key=lambda e: (e[1] != abi.ACT_DELETE_MH_UNHEALTHY, rank[(pr.pods[e[0]].get("labels") or {}).get(snapmod.REPLICA_NAME_LABEL)]))
        for pi, act in order:
            if act in (abi.ACT_DELETE_MH_INCOMPLETE, abi.ACT_DELETE_MH_UNHEALTHY, abi.ACT_DELETE_MH_WTD, abi.ACT_DELETE_MH_SCALE_DOWN):
                pod = pr.pods[pi]
                self._warning = ("FailedToDeleteWorkerPod", f"Failed deleting worker Pod {ns}/{pod['name']} for group {gname}; {_pod_status_text(pod)}")
                if cl.delete_pod(*meta.pod_keys[pi]):
                    # (no trigger: the engine named a replica group shouldDeletePod does not; the event then shows it)
                    why = reasons.get(act) or self._should_delete_reason(trigger.get((pod.get("labels") or {}).get(snapmod.REPLICA_NAME_LABEL), pod), "worker")
                    cl.events.append(("Normal", EV_DELETED_WORKER_POD, f"Deleted worker Pod {ns}/{pod['name']} for group {gname}: {why}"))
        ek = int(cr["err_kind"])
        if int(gr["flags"]) & abi.GR_ABORTED:
            if ek == abi.ERR_MH_INCOMPLETE:         # :982 names the replica group whose Pods were deleted
                rname = next((pr.pods[pi].get("labels") or {}).get(snapmod.REPLICA_NAME_LABEL) for pi, act in in_group if act == abi.ACT_DELETE_MH_INCOMPLETE)
                return f"cleaned up incomplete replica group {rname}, requeueing"
            if ek == abi.ERR_MH_WTD:
                return f"deleted {int(cr['err_arg'])} worker Pods based on ScaleStrategy, requeueing"
            if ek == abi.ERR_MH_NOT_MULTIPLE:
                return f"desired worker pods ({int(gr['expected'])}) is not a multiple of NumOfHosts ({grp.get('numOfHosts', 1)}) for group {gname}"
        hosts = int(grp.get("numOfHosts", 1))
        self._stage = "FailedCreateWorkerPod"       # :1091
        for k in range(int(gr["n_create"])):        # one entry per replica group (:1082-1094)
            idx = int(res.create_idx[int(gr["create_off"]) + k])
            rname = f"{gname}-{cl.gen_suffix()}"
            for j in range(hosts):
                pod = self._build_pod(cluster, (gi, idx, j, rname))   # :1090
                self._warning = ("FailedToCreateWorkerPod", f"Failed to create worker Pod for the cluster {ns}/{cname}")
                cl.create_pod(pod)
                cl.events.append(("Normal", EV_CREATED_WORKER_POD, f"Created worker Pod {ns}/{pod['name']}"))
        return None

    def _build_pod(self, cluster: dict, create: tuple, cluster_hash: str | None = None) -> dict:
        """The new Pod's ObjectMeta from the native builder (kr_pod_meta_build: buildHeadPod / buildWorkerPod metadata,
        raycluster_controller.go:1387-1433); the fake API server then turns generateName into a name (5 generated characters)."""
        spec = cluster.get("spec") or {}
        grp = (spec.get("headGroupSpec") or {}) if create[0] < 0 else spec["workerGroupSpecs"][create[0]]
        pod_spec = None
        if ((grp.get("template") or {}).get("spec") or {}).get("containers"):
            # the RayCluster carries real Pod templates: the whole manifest, container half included (kr_pod_build: DefaultHead/WorkerPodTemplate + BuildPod)
            built = podbuilder.build_pods_native(cluster, [create], podbuilder.BuilderEnv(kuberay_version=snapmod.KUBERAY_VERSION,
                                                                                          multihost_indexing_gate=bool(self.env.multihost_indexing_gate)), cluster_hash=cluster_hash)[0]
            meta, pod_spec = built["metadata"], built["spec"]
        else:
            env = podmeta.PodMetaEnv(kuberay_version=snapmod.KUBERAY_VERSION, multihost_indexing_gate=bool(self.env.multihost_indexing_gate))
            meta = podmeta.build_pod_meta(cluster, [create], env, cluster_hash=cluster_hash)[0]
        name = meta.get("name") or meta["generateName"] + self.client.gen_suffix()
        pod = {"namespace": meta["namespace"], "name": name, "phase": "", "restartPolicy": (pod_spec or {}).get("restartPolicy") or "Always", "labels": meta["labels"],
               "annotations": meta["annotations"], "ownerReferences": meta["ownerReferences"]}
        if pod_spec is not None:
            pod["spec"] = pod_spec
        return pod

    @staticmethod
    def _should_delete_reason(pod: dict, node_type: str) -> str:
        """The reason string of shouldDeletePod (:1181-1231) — it is what reconcilePods returns as the error (:711)."""
        ph = pod.get("phase", "")
        if ph in ("Failed", "Succeeded"):
            return (f"The {node_type} Pod {pod['name']} status is {ph} which is a terminal state. "
                    "KubeRay will delete the Pod and create new Pods in the next reconciliation if necessary.")
        return (f"The Pod status of the {node_type} Pod {pod['name']} is {ph}, and the Ray container terminated status is "
                f"{_terminated_text(pod)}. The container is unable to restart due to its restart policy {pod.get('restartPolicy', '')}, so KubeRay will delete it.")

    # ------------------------------------------------------------------ calculateStatus
    def calculate_status(self, ns: str, name: str, reconcile_err=None) -> tuple[dict | None, str | None]:
        """-> (new status dict, calculate error).  reconcile_err: None, a plain string, or ("FailedCreateHeadPod", "message")."""
        if reconcile_err is None:
            ext = {"kind": abi.EXT_ERR_STATUS_ONLY_NIL}
        elif isinstance(reconcile_err, tuple):
            ext = {"kind": snapmod._REPLICA_FAILURE_KIND[reconcile_err[0]], "message": reconcile_err[1]}
        else:
            ext = {"kind": abi.EXT_ERR_PLAIN, "message": str(reconcile_err)}
        pr = self._pass({(ns, name): {"extErr": ext}})
        ci = self._cluster_index(pr, ns, name)
        return self.status_from_record(pr, ci)

    def status_from_record(self, pr: PassResult, ci: int) -> tuple[dict | None, str | None]:
        res, meta = pr.res, pr.meta
        it = meta.interner
        cr = res.clusters[ci]
        ns, cname = meta.cluster_keys[ci]
        old = copy.deepcopy(self.client.clusters[(ns, cname)].get("status") or {})
        serr = int(cr["status_err"])
        if serr:
            return None, {abi.SERR_MULTIPLE_HEADS: "found multiple heads", abi.SERR_NO_HEAD_SERVICE: "unable to find head service",
                          abi.SERR_MULTIPLE_HEAD_SERVICES: "found multiple head services", abi.SERR_EMPTY_SERVICE_IP: "head service IP is empty"}[serr]
        new = old
        st = int(cr["new_state"])
        if st != abi.STATE_OTHER:
            new["state"] = snapmod.STATE_NAMES[st]
        if int(cr["status_flags"]) & abi.SF_READY_BRANCH:
            new["reason"] = ""  # :1601-1602
        keys = ["readyWorkerReplicas", "availableWorkerReplicas", "desiredWorkerReplicas", "minWorkerReplicas", "maxWorkerReplicas"]
        for k, v in zip(keys, cr["counts"]):
            new[k] = int(v)
        conds_old = {c["type"]: c for c in old.get("conditions") or []}
        conds = []
        order = [c["type"] for c in old.get("conditions") or []]
        # a condition calculateStatus adds goes last, in the order of its SetStatusCondition calls (:1566, 1614-1622, 1630-1693)
        suspending = int(pr.snap.c_suspend_status[ci]) == abi.SUSPEND_SUSPENDING
        for slot in (abi.COND_REPLICA_FAILURE, abi.COND_HEAD_POD_READY, abi.COND_PROVISIONED,
                     *((abi.COND_SUSPENDING, abi.COND_SUSPENDED) if suspending else (abi.COND_SUSPENDED, abi.COND_SUSPENDING))):
            t = snapmod.COND_NAMES[slot]
            if t not in order and cr["cond_status"][slot] != abi.COND_ABSENT:
                order.append(t)
        for t in order:
            slot = snapmod._COND_SLOT.get(t)
            if slot is None:
                conds.append(conds_old[t]); continue
            stc = int(cr["cond_status"][slot])
            if stc == abi.COND_ABSENT:
                continue
            var = int(cr["cond_variant"][slot])
            cond = dict(conds_old.get(t) or {"type": t})
            cond["status"] = {abi.COND_TRUE: "True", abi.COND_FALSE: "False", abi.COND_UNKNOWN: "Unknown"}[stc]
            if slot == abi.COND_PROVISIONED and var in snapmod.PROV_VARIANT_STRINGS:
                cond["reason"], cond["message"] = snapmod.PROV_VARIANT_STRINGS[var]
            elif slot in (abi.COND_SUSPENDING, abi.COND_SUSPENDED) and var == abi.CV_CANONICAL:
                cond["reason"], cond["message"] = t, ""
            elif slot == abi.COND_HEAD_POD_READY and var in (abi.CV_HEAD_FROM_POD, abi.CV_HEAD_NOT_FOUND):
                cond["reason"] = it.str(int(cr["head_ready_reason_id"])) or ""
                cond["message"] = it.str(int(cr["head_ready_msg_id"])) or ""
            elif slot == abi.COND_REPLICA_FAILURE and var in snapmod.REPLICA_FAILURE_NAMES:
                cond["reason"] = snapmod.REPLICA_FAILURE_NAMES[var]
                mid = int(pr.snap.c_ext_err_msg_id[ci])
                if int(pr.snap.c_ext_err_kind[ci]) == var:
                    cond["message"] = it.str(mid) or ""
            conds.append(cond)
        if conds or "conditions" in old:
            new["conditions"] = conds
        hid = [int(x) for x in cr["head_ids"]]
        new["head"] = {"podIP": it.str(hid[0]) or "", "serviceIP": it.str(hid[1]) or "", "podName": it.str(hid[2]) or "", "serviceName": it.str(hid[3]) or ""}
        cluster = self.client.clusters[(ns, cname)]
        svc = cluster.get("headService", {"count": 1, "clusterIP": "10.0.0.1", "name": f"{cname}-head-svc"})
        new["endpoints"] = snapmod.compute_endpoints(old.get("endpoints"), svc)
        new["_needs_write"] = bool(cr["needs_status_write"])
        new["_state_changed"] = bool(cr["state_changed"])
        return new, None

    def update_status(self, ns: str, name: str, new_status: dict, now: str = "now") -> bool:
        """updateRayClusterStatus (:1951-1966): write iff InconsistentRayClusterStatus; returns `inconsistent`."""
        inconsistent = bool(new_status.pop("_needs_write", False))
        changed = bool(new_status.pop("_state_changed", False))
        new_status["lastUpdateTime"] = now
        if changed:
            new_status.setdefault("stateTransitionTimes", {})[new_status.get("state", "")] = now
        if inconsistent:
            self.client.clusters[(ns, name)]["status"] = new_status
        return inconsistent

    # ------------------------------------------------------------------ the full Reconcile body for one key (:296-355)
    def reconcile(self, ns: str, name: str, now: str = "now") -> tuple[float, str | None]:
        """-> (requeue seconds, error; 0 = no requeue).  One pass feeds both the decisions and the status, as the engine produces them —
        unless a side-effect call failed at the API server: the record's status was computed for reconcileErr == nil, so it
        is discarded and the status is re-evaluated (status-only pass, c_ext_err_kind = the ErrFailed* kind), which is what
        calculateStatus(ctx, instance, reconcileErr) sees in the reference (:308-316, 1563-1577, 1599)."""
        pr = self._pass()
        return self.reconcile_record(pr, self._cluster_index(pr, ns, name), now)

    def reconcile_record(self, pr: PassResult, ci: int, now: str = "now") -> tuple[float, str | None]:
        """The Reconcile body of RayCluster ci once the pass `pr` decided it."""
        ns, name = pr.meta.cluster_keys[ci]
        if int(pr.snap.c_flags[ci]) & abi.CF_SKIP:   # being deleted: no status, no requeue (:291-294)
            return 0.0, None
        err = self._apply_decisions(pr, ci)
        if isinstance(err, tuple):
            err = f"{err[0]}\n{err[1]}"   # errors.Join(ErrFailed..., err).Error(): also the ReplicaFailure message (:1570)
            new, cerr = self.calculate_status(ns, name, (err.split("\n", 1)[0], err))
        else:
            new, cerr = self.status_from_record(pr, ci)
        inconsistent = False
        if cerr is None:
            inconsistent = self.update_status(ns, name, new, now)
        final = err or cerr
        if final or inconsistent:
            return 2.0, final      # DefaultRequeueDuration (:51,338-340)
        return 300.0, None         # RAYCLUSTER_DEFAULT_REQUEUE_SECONDS (utils/constant.go:149-150)

"""Columnar snapshot container, string interner and the object -> column packer.

The packer is the Python statement of what the Go shim does before calling the engine
(INTEGRATION.md): it evaluates the host-only inputs the reference computes from strings —
FindRayClusterSuspendStatus (ray-operator/controllers/ray/utils/util.go:153-162),
FindHeadPodReadyCondition (utils/util.go:81-134), getRayContainerStateTerminated
(raycluster_controller.go:1237-1248), the head-Service lookup (raycluster_controller.go:1721-1745),
updateEndpoints (:1747-1783) — and interns every string to a u32 id.
"""
from __future__ import annotations

import ctypes as C
import re
from dataclasses import dataclass, field

import numpy as np

from . import abi

KUBERAY_VERSION = "nightly"  # utils/constant.go:281
RAY_CLUSTER_LABEL = "ray.io/cluster"  # utils/constant.go:19-21
RAY_NODE_TYPE_LABEL = "ray.io/node-type"
RAY_NODE_GROUP_LABEL = "ray.io/group"
REPLICA_NAME_LABEL = "ray.io/worker-group-replica-name"  # utils/constant.go:39-48
REPLICA_INDEX_LABEL = "ray.io/worker-group-replica-index"
RECREATE_HASH_ANNOT = "ray.io/upgrade-strategy-recreate-hash"  # utils/constant.go:27
KUBERAY_VERSION_ANNOT = "ray.io/kuberay-version"  # utils/constant.go:29
SKIP_HEAD_RESTART_ANNOT = "ray.io/disable-provisioned-head-restart"  # utils/constant.go:34
CONTAINERS_NOT_READY = "ContainersNotReady"
_ATOI_RE = re.compile(r"^[+-]?[0-9]+$")

_NODE_TYPE = {"head": abi.NT_HEAD, "worker": abi.NT_WORKER, "redis-cleanup": abi.NT_REDIS}
_PHASE = {"": abi.PHASE_EMPTY, "Pending": abi.PHASE_PENDING, "Running": abi.PHASE_RUNNING,
          "Succeeded": abi.PHASE_SUCCEEDED, "Failed": abi.PHASE_FAILED, "Unknown": abi.PHASE_UNKNOWN}
_COND = {"True": abi.COND_TRUE, "False": abi.COND_FALSE, "Unknown": abi.COND_UNKNOWN}
_STATE = {"": abi.STATE_EMPTY, "ready": abi.STATE_READY, "failed": abi.STATE_FAILED, "suspended": abi.STATE_SUSPENDED}
STATE_NAMES = {v: k for k, v in _STATE.items()}
_COND_SLOT = {"RayClusterProvisioned": abi.COND_PROVISIONED, "HeadPodReady": abi.COND_HEAD_POD_READY,
              "ReplicaFailure": abi.COND_REPLICA_FAILURE, "RayClusterSuspending": abi.COND_SUSPENDING,
              "RayClusterSuspended": abi.COND_SUSPENDED}
COND_NAMES = {v: k for k, v in _COND_SLOT.items()}
_REPLICA_FAILURE_KIND = {"FailedDeleteAllPods": abi.EXT_ERR_FAILED_DELETE_ALL_PODS, "FailedDeleteHeadPod": abi.EXT_ERR_FAILED_DELETE_HEAD_POD,
                         "FailedCreateHeadPod": abi.EXT_ERR_FAILED_CREATE_HEAD_POD, "FailedDeleteWorkerPod": abi.EXT_ERR_FAILED_DELETE_WORKER_POD,
                         "FailedCreateWorkerPod": abi.EXT_ERR_FAILED_CREATE_WORKER_POD}
REPLICA_FAILURE_NAMES = {v: k for k, v in _REPLICA_FAILURE_KIND.items()}
# (reason, message) pairs the controller writes itself (raycluster_controller.go:1630-1691)
_PROV_VARIANTS = {
    ("AllPodRunningAndReadyFirstTime", "All Ray Pods are ready for the first time"): abi.CV_PROV_ALL_READY,
    ("RayClusterPodsProvisioning", "RayCluster Pods are being provisioned for first time"): abi.CV_PROV_PROVISIONING,
    ("RayClusterPodsProvisioning", "RayCluster has been suspended"): abi.CV_PROV_SUSPENDED,
}
PROV_VARIANT_STRINGS = {v: k for k, v in _PROV_VARIANTS.items()}
HEAD_NOT_FOUND_REASON, HEAD_NOT_FOUND_MSG = "HeadPodNotFound", "Head Pod not found"


class Interner:
    """str -> u32. id 0 = absent (None), id 1 = "" (include/kr_engine.h KR_ID_*)."""

    def __init__(self):
        self._ids: dict[str, int] = {"": abi.ID_EMPTY_STRING}
        self._strs: list[str | None] = [None, ""]

    def id(self, s: str | None) -> int:
        if s is None:
            return abi.ID_ABSENT
        i = self._ids.get(s)
        if i is None:
            i = len(self._strs)
            self._ids[s] = i
            self._strs.append(s)
        return i

    def id0(self, s: str | None) -> int:
        """HeadInfo-style fields: the empty string is encoded as 0."""
        return abi.ID_ABSENT if not s else self.id(s)

    def str(self, i: int) -> str | None:
        return self._strs[i]

    def __len__(self):
        return len(self._strs)


def _align16(x: int) -> int:
    return (x + 15) & ~15


class Snapshot:
    """All columns of include/kr_engine.h kr_snapshot_bufs as host numpy arrays."""

    def __init__(self, n_clusters=0, n_groups=0, n_wtd=0, n_pods=0, n_heads=0, n_jobs=0, json_bytes=0):
        self.dims = {"clusters": n_clusters, "groups": n_groups, "wtd": n_wtd, "pods": n_pods, "heads": n_heads,
                     "jobs": n_jobs, "json": json_bytes}
        self.cols: dict[str, np.ndarray] = {}
        for name, dt, mult, dim in abi.COLUMNS:
            n = self.dims[dim] * mult
            self.cols[name] = np.zeros(max(n, 1), dtype=dt)[:n] if n == 0 else np.zeros(n, dtype=dt)

    def __getattr__(self, name):
        cols = self.__dict__.get("cols")
        if cols is not None and name in cols:
            return cols[name]
        raise AttributeError(name)

    def sizes(self) -> abi.kr_sizes:
        d = self.dims
        return abi.kr_sizes(d["clusters"], d["groups"], d["wtd"], d["pods"], d["heads"], d["jobs"], d["json"])

    def bufs(self) -> abi.kr_snapshot_bufs:
        """ctypes view over the numpy arrays (keep `self` alive while it is in use)."""
        b = abi.kr_snapshot_bufs()
        for name, dt, _m, _d in abi.COLUMNS:
            arr = self.cols[name]
            assert arr.flags["C_CONTIGUOUS"] and arr.dtype == dt, name
            ptr = arr.ctypes.data_as(C.POINTER(abi._CT[dt])) if arr.size else C.cast(None, C.POINTER(abi._CT[dt]))
            setattr(b, name, ptr)
        return b

    def nbytes(self) -> int:
        return sum(a.nbytes for a in self.cols.values())

    def validate(self):
        d = self.dims
        c = self.cols
        if d["clusters"]:
            off = c["c_group_off"].astype(np.int64)
            cnt = c["c_group_cnt"].astype(np.int64)
            exp = np.concatenate([[0], np.cumsum(cnt)[:-1]])
            assert (off == exp).all() and int(cnt.sum()) == d["groups"], "groups must be stored in cluster order (CSR)"
            assert (c["c_json_off"] % 16 == 0).all(), "json offsets must be 16-byte aligned"
            assert ((c["c_json_off"] + c["c_json_len"]) <= d["json"]).all()
        if d["groups"]:
            assert (c["g_cluster_idx"] < max(d["clusters"], 1)).all()
            assert int(c["g_wtd_cnt"].sum()) == d["wtd"]
        if d["heads"]:
            assert (c["h_pod_idx"] < max(d["pods"], 1)).all()
        return self


# ------------------------------------------------------------------------------------------- host-only evaluations

def find_suspend_status(conditions) -> int:
    """utils.FindRayClusterSuspendStatus (utils/util.go:153-162): first True among Suspending/Suspended, slice order."""
    for cond in conditions or []:
        if cond.get("type") in ("RayClusterSuspending", "RayClusterSuspended") and cond.get("status") == "True":
            return abi.SUSPEND_SUSPENDING if cond["type"] == "RayClusterSuspending" else abi.SUSPEND_SUSPENDED
    return abi.SUSPEND_NONE


def ray_container_terminated(pod: dict) -> bool:
    """getRayContainerStateTerminated(pod) != nil (raycluster_controller.go:1237-1248): a present `terminated` state counts even
    when it is empty."""
    if "rayContainerTerminated" in pod:
        return bool(pod["rayContainerTerminated"])
    containers = pod.get("containers") or []
    if not containers:
        return False
    ray_name = containers[0].get("name")
    for st in pod.get("containerStatuses") or []:
        if st.get("name") == ray_name:
            return (st.get("state") or {}).get("terminated") is not None
    return False


def head_pod_ready_condition(pod: dict) -> tuple[str, str, str]:
    """utils.FindHeadPodReadyCondition (utils/util.go:81-134) -> (status, reason, message)."""
    status, reason_out, message = "False", "Unknown", ""
    for cond in pod.get("conditions") or []:
        if cond.get("type") != "Ready":
            continue
        status = cond.get("status", "")
        message = cond.get("message", "") or ""
        reason = cond.get("reason", "") or ""
        if status == "True" and reason == "":
            reason = "HeadPodRunningAndReady"
        if reason != "":
            reason_out = reason
        if reason == CONTAINERS_NOT_READY:
            for st in pod.get("containerStatuses") or []:
                state = st.get("state") or {}
                sub = state.get("waiting") or state.get("terminated")
                if state.get("waiting") is not None or state.get("terminated") is not None:
                    if message != "":
                        message += "; "
                    message += f"{st.get('name', '')}: {(sub or {}).get('message', '')}"
                    reason_out = (sub or {}).get("reason", "")
                    break
        break
    return status, reason_out, message


def pod_ready_code(pod: dict) -> int:
    for cond in pod.get("conditions") or []:
        if cond.get("type") == "Ready":
            return _COND.get(cond.get("status", ""), abi.COND_UNKNOWN)
    return abi.COND_ABSENT


def pack_pod_word(pod: dict) -> tuple[int, int]:
    """-> (packed word, replica_index)."""
    labels = pod.get("labels") or {}
    pk = _NODE_TYPE.get(labels.get(RAY_NODE_TYPE_LABEL, ""), abi.NT_NONE) << abi.PP_NODE_TYPE_SHIFT
    pk |= _PHASE.get(pod.get("phase", ""), abi.PHASE_UNKNOWN) << abi.PP_PHASE_SHIFT
    pk |= pod_ready_code(pod) << abi.PP_READY_SHIFT
    if pod.get("restartPolicy") == "Never":
        pk |= abi.PP_RESTART_NEVER
    if ray_container_terminated(pod):
        pk |= abi.PP_RAY_TERMINATED
    if pod.get("deletionTimestamp"):
        pk |= abi.PP_HAS_DELETION_TS
    ridx = 0
    raw = labels.get(REPLICA_INDEX_LABEL)
    if raw is not None and _ATOI_RE.match(raw):  # strconv.Atoi: optional sign + ASCII decimal digits (:857-860)
        v = int(raw)
        if -(2 ** 63) <= v < 2 ** 63:  # fits Go int; the column is int32 — clamp (such an index can never be allocated)
            ridx = max(-(2 ** 31), min(2 ** 31 - 1, v))
            pk |= abi.PP_HAS_REPLICA_IDX
    return pk, ridx


def status_summary_key(status: dict | None) -> str:
    """Canonical encoding of exactly the fields InconsistentRayClusterStatus compares (utils/consistency.go:16-34)."""
    st = status or {}
    conds = [(c.get("type", ""), c.get("status", ""), c.get("reason", ""), c.get("message", ""),
              str(c.get("lastTransitionTime", "")), int(c.get("observedGeneration", 0))) for c in st.get("conditions") or []]
    head = st.get("head") or {}
    return repr((st.get("state", ""), st.get("reason", ""), int(st.get("readyWorkerReplicas", 0)), int(st.get("availableWorkerReplicas", 0)),
                 int(st.get("desiredWorkerReplicas", 0)), int(st.get("minWorkerReplicas", 0)), int(st.get("maxWorkerReplicas", 0)),
                 sorted((st.get("endpoints") or {}).items()) if st.get("endpoints") is not None else None,
                 (head.get("podIP", ""), head.get("serviceIP", ""), head.get("podName", ""), head.get("serviceName", "")), conds))


def compute_endpoints(old: dict | None, svc: dict | None) -> dict | None:
    """updateEndpoints (raycluster_controller.go:1747-1783): merge the head Service's ports into status.endpoints."""
    if not svc or svc.get("count", 1) == 0:
        return old
    out = dict(old) if old is not None else {}
    for port in svc.get("ports") or []:
        name = port.get("name", "")
        if not name:
            continue
        if port.get("nodePort", 0):
            out[name] = str(port["nodePort"])
        elif isinstance(port.get("targetPort"), int) and port["targetPort"] != 0:
            out[name] = str(port["targetPort"])
        elif isinstance(port.get("targetPort"), str) and port["targetPort"] != "":
            out[name] = port["targetPort"]
    return out


TOMBSTONE = {"tombstone": True}  # the pod "object" of a free arena row


@dataclass
class PackMeta:
    interner: Interner
    cluster_keys: list[tuple[str, str]] = field(default_factory=list)
    group_names: list[str] = field(default_factory=list)
    pod_keys: list[tuple[str, str]] = field(default_factory=list)
    flags: abi.kr_flags | None = None


def spec_hash_input(spec: dict) -> bytes:
    """The bytes GenerateHashWithoutReplicasAndWorkersToDelete hashes (utils/util.go:642-665): json.Marshal(mute(spec)), from
    the native emitter behind the C ABI (kr_spec_json_emit; host code of libkrengine.so, no device needed)."""
    import json

    from . import engine
    return engine.spec_json_emit(json.dumps(spec or {}).encode("utf-8"))


def pack_objects(clusters: list[dict], pods: list[dict], jobs: list[dict] | None = None, interner: Interner | None = None,
                 kuberay_version: str = KUBERAY_VERSION, spec_json=None) -> tuple[Snapshot, PackMeta]:
    """Pack object-level RayClusters / Pods / RayJobs (plain dicts, see tests/golden/README.md) into a Snapshot.

    `spec_json(cluster) -> bytes` supplies the muted-spec JSON. Default: cluster["specJson"] if present (bytes marshalled by
    the Go side), else the native emitter (spec_hash_input: kr_spec_json_emit over cluster["spec"]).
    """
    it = interner or Interner()
    jobs = jobs or []
    n_groups = sum(len((c.get("spec") or {}).get("workerGroupSpecs") or []) for c in clusters)
    n_wtd = sum(len(g.get("workersToDelete") or (g.get("scaleStrategy") or {}).get("workersToDelete") or [])
                for c in clusters for g in (c.get("spec") or {}).get("workerGroupSpecs") or [])
    head_rows = [i for i, p in enumerate(pods) if (p.get("labels") or {}).get(RAY_NODE_TYPE_LABEL) == "head"]
    blobs = []
    for c in clusters:
        if spec_json is not None:
            b = spec_json(c)
        elif "specJson" in c:
            b = c["specJson"].encode() if isinstance(c["specJson"], str) else bytes(c["specJson"])
        else:
            b = spec_hash_input(c.get("spec") or {})
        blobs.append(b)
    json_bytes = sum(_align16(len(b)) for b in blobs)
    s = Snapshot(len(clusters), n_groups, n_wtd, len(pods), len(head_rows), len(jobs), json_bytes)
    meta = PackMeta(it)
    g = w = 0
    joff = 0
    for ci, c in enumerate(clusters):
        spec = c.get("spec") or {}
        status = c.get("status") or {}
        ns, name = c.get("namespace", "default"), c["name"]
        meta.cluster_keys.append((ns, name))
        s.c_ns_id[ci] = it.id(ns)
        s.c_name_id[ci] = it.id(name)
        s.c_uid_hash[ci] = np.uint64(uid_hash64(c.get("uid") or f"{ns}/{name}"))
        fl = 0
        if spec.get("suspend") is True:
            fl |= abi.CF_SUSPEND
        if spec.get("suspend") is False:
            fl |= abi.CF_SUSPEND_SET_FALSE
        if spec.get("enableInTreeAutoscaling") is True:
            fl |= abi.CF_AUTOSCALING
        us = spec.get("upgradeStrategy")
        if (us.get("type") if isinstance(us, dict) else us) == "Recreate":
            fl |= abi.CF_UPGRADE_RECREATE
        if (c.get("annotations") or {}).get(SKIP_HEAD_RESTART_ANNOT) == "true":
            fl |= abi.CF_SKIP_HEAD_RESTART
        exp = c.get("expectations") or {}
        if exp.get("head", True):
            fl |= abi.CF_HEAD_EXPECT_OK
        if c.get("deletionTimestamp") or c.get("skip"):
            fl |= abi.CF_SKIP
        if status.get("reason", "") != "":
            fl |= abi.CF_OLD_REASON_NONEMPTY
        svc = c.get("headService", {"count": 1, "clusterIP": "10.0.0.1", "name": f"{name}-head-svc"})
        new_eps = compute_endpoints(status.get("endpoints"), svc)
        if new_eps != status.get("endpoints"):
            fl |= abi.CF_ENDPOINTS_CHANGED
        s.c_flags[ci] = fl
        s.c_suspend_status[ci] = find_suspend_status(status.get("conditions"))
        ext = c.get("extErr") or {}
        s.c_ext_err_kind[ci] = ext.get("kind", 0)
        s.c_ext_err_msg_id[ci] = it.id(ext["message"]) if "message" in ext else 0
        s.c_json_off[ci] = joff
        s.c_json_len[ci] = len(blobs[ci])
        s.json[joff:joff + len(blobs[ci])] = np.frombuffer(blobs[ci], dtype=np.uint8)
        joff += _align16(len(blobs[ci]))
        # old status
        st = status.get("state", "")
        s.c_old_state[ci] = _STATE.get(st, abi.STATE_OTHER)
        s.c_old_counts[5 * ci:5 * ci + 5] = [status.get("readyWorkerReplicas", 0), status.get("availableWorkerReplicas", 0),
                                            status.get("desiredWorkerReplicas", 0), status.get("minWorkerReplicas", 0),
                                            status.get("maxWorkerReplicas", 0)]
        for cond in status.get("conditions") or []:
            slot = _COND_SLOT.get(cond.get("type"))
            if slot is None:
                continue
            s.c_old_cond_status[5 * ci + slot] = _COND.get(cond.get("status", ""), abi.COND_UNKNOWN)
            reason, msg = cond.get("reason", ""), cond.get("message", "")
            if slot == abi.COND_PROVISIONED:
                var = _PROV_VARIANTS.get((reason, msg), abi.CV_OTHER)
            elif slot in (abi.COND_SUSPENDING, abi.COND_SUSPENDED):
                var = abi.CV_CANONICAL if (reason == cond["type"] and msg == "") else abi.CV_OTHER
            elif slot == abi.COND_HEAD_POD_READY:
                var = abi.CV_HEAD_NOT_FOUND if (reason, msg) == (HEAD_NOT_FOUND_REASON, HEAD_NOT_FOUND_MSG) else abi.CV_HEAD_FROM_POD
                s.c_old_cond_reason_id[ci] = it.id(reason)
                s.c_old_cond_msg_id[2 * ci] = it.id(msg)
            else:
                var = _REPLICA_FAILURE_KIND.get(reason, abi.CV_OTHER)
                s.c_old_cond_msg_id[2 * ci + 1] = it.id(msg)
            s.c_old_cond_variant[5 * ci + slot] = var
        head = status.get("head") or {}
        s.c_old_head_ids[4 * ci:4 * ci + 4] = [it.id0(head.get("podIP")), it.id0(head.get("serviceIP")),
                                              it.id0(head.get("podName")), it.id0(head.get("serviceName"))]
        cnt = svc.get("count", 1)
        s.c_svc_count[ci] = min(cnt, 2)
        ip = svc.get("clusterIP", "")
        s.c_svc_ip_kind[ci] = abi.SVCIP_EMPTY if ip == "" else (abi.SVCIP_NONE if ip == "None" else abi.SVCIP_NORMAL)
        s.c_svc_ip_id[ci] = it.id0(ip) if ip not in ("", "None") else 0
        s.c_svc_name_id[ci] = it.id0(svc.get("name", ""))
        s.c_summary_id[ci] = it.id(status_summary_key(status))
        # groups
        groups = spec.get("workerGroupSpecs") or []
        s.c_group_off[ci] = g
        s.c_group_cnt[ci] = len(groups)
        for grp in groups:
            meta.group_names.append(grp["groupName"])
            s.g_cluster_idx[g] = ci
            s.g_name_id[g] = it.id(grp["groupName"])
            gf = 0
            for key, col, nil in (("replicas", s.g_replicas, abi.GF_REPLICAS_NIL), ("minReplicas", s.g_min, abi.GF_MIN_NIL),
                                  ("maxReplicas", s.g_max, abi.GF_MAX_NIL)):
                v = grp.get(key)
                if v is None:
                    gf |= nil
                else:
                    col[g] = v
            s.g_num_hosts[g] = grp.get("numOfHosts", 1)
            if grp.get("suspend") is True:
                gf |= abi.GF_SUSPEND
            if exp.get(grp["groupName"], True):
                gf |= abi.GF_EXPECT_OK
            s.g_flags[g] = gf
            names = grp.get("workersToDelete") or (grp.get("scaleStrategy") or {}).get("workersToDelete") or []
            s.g_wtd_off[g] = w
            s.g_wtd_cnt[g] = len(names)
            for nm in names:
                s.w_name_id[w] = it.id(nm)
                w += 1
            g += 1
    for pi, p in enumerate(pods):
        if p.get("tombstone"):  # free row of an incrementally maintained arena (KR_PP_TOMBSTONE): all ids 0, matches nothing
            meta.pod_keys.append((None, None))
            s.p_packed[pi] = abi.PP_TOMBSTONE
            continue
        labels = p.get("labels") or {}
        ns = p.get("namespace", "default")
        meta.pod_keys.append((ns, p["name"]))
        s.p_ns_id[pi] = it.id(ns)
        s.p_cluster_name_id[pi] = it.id(labels.get(RAY_CLUSTER_LABEL))
        s.p_group_name_id[pi] = it.id(labels.get(RAY_NODE_GROUP_LABEL))
        s.p_name_id[pi] = it.id(p["name"])
        s.p_packed[pi], s.p_replica_index[pi] = pack_pod_word(p)
        s.p_replica_name_id[pi] = it.id(labels.get(REPLICA_NAME_LABEL))
    for hi, pi in enumerate(head_rows):
        p = pods[pi]
        ann = p.get("annotations") or {}
        st, reason, msg = head_pod_ready_condition(p)
        s.h_pod_idx[hi] = pi
        s.h_ready_status[hi] = _COND.get(st, abi.COND_UNKNOWN) if st != "" else abi.COND_UNKNOWN
        s.h_ready_reason_id[hi] = it.id(reason)
        s.h_ready_msg_id[hi] = it.id(msg)
        s.h_pod_ip_id[hi] = it.id0(p.get("podIP"))
        h = ann.get(RECREATE_HASH_ANNOT, "")
        if h == "":
            s.h_annot_state[hi] = abi.ANNOT_EMPTY
        elif len(h.encode()) == 32:
            s.h_annot_state[hi] = abi.ANNOT_HASH32
            s.h_annot_hash[32 * hi:32 * hi + 32] = np.frombuffer(h.encode(), dtype=np.uint8)
        else:
            s.h_annot_state[hi] = abi.ANNOT_OTHER
        v = ann.get(KUBERAY_VERSION_ANNOT, "")
        s.h_version_state[hi] = abi.VER_EMPTY if v == "" else (abi.VER_CURRENT if v == kuberay_version else abi.VER_DIFFERENT)
    for ji, j in enumerate(jobs):
        s.j_ns_id[ji] = it.id(j.get("namespace", "default"))
        s.j_cluster_name_id[ji] = it.id((j.get("status") or {}).get("rayClusterName") or None)
        s.j_summary_id[ji] = it.id(status_summary_key((j.get("status") or {}).get("rayClusterStatus")))
    meta.flags = abi.default_flags(id_head_not_found_reason=it.id(HEAD_NOT_FOUND_REASON), id_head_not_found_msg=it.id(HEAD_NOT_FOUND_MSG))
    return s.validate(), meta


def uid_hash64(uid: str) -> int:
    """FNV-1a 64 over the UID string: the sharding key (SURVEY §8(e))."""
    h = 0xCBF29CE484222325
    for b in uid.encode():
        h = ((h ^ b) * 0x100000001B3) & 0xFFFFFFFFFFFFFFFF
    return h

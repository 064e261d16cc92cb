"""ctypes binding of the native event-driven packer (kr_packer_*, kuberay_b200/csrc/kr_packer.cpp) + the adapter that turns the
dict objects of the test fixtures into the plain C structs a Go informer handler would fill from *corev1.Pod / *rayv1.RayCluster.

The adapter only extracts fields (the same cheap per-object derivations pack_objects does: flag bits, condition codes); interning,
row management, the CSR tables, the spec JSON and the incremental commits are the native packer's."""
from __future__ import annotations

import ctypes as C
import json

from . import abi
from . import snapshot as snp
from .engine import Engine, EngineError, Group, lib


def _s(v) -> abi.kr_str:
    if v is None:
        return abi.kr_str(None, 0)
    b = v if isinstance(v, bytes) else str(v).encode("utf-8")
    return abi.kr_str(b, len(b))


def pod_obj(pod: dict) -> abi.kr_pod_obj:
    """The kr_pod_obj an informer handler would fill from the Pod (its kr_str fields point into bytes the struct keeps alive)."""
    labels, ann = pod.get("labels") or {}, pod.get("annotations") or {}
    o = abi.kr_pod_obj()
    o.ns, o.name = _s(pod.get("namespace", "default")), _s(pod["name"])
    o.cluster, o.group = _s(labels.get(snp.RAY_CLUSTER_LABEL)), _s(labels.get(snp.RAY_NODE_GROUP_LABEL))
    o.replica_name, o.replica_index = _s(labels.get(snp.REPLICA_NAME_LABEL)), _s(labels.get(snp.REPLICA_INDEX_LABEL))
    o.node_type = snp._NODE_TYPE.get(labels.get(snp.RAY_NODE_TYPE_LABEL, ""), abi.NT_NONE)
    o.phase = snp._PHASE.get(pod.get("phase", ""), abi.PHASE_UNKNOWN)
    o.ready_cond = snp.pod_ready_code(pod)
    o.restart_never = 1 if pod.get("restartPolicy") == "Never" else 0
    o.ray_terminated = 1 if snp.ray_container_terminated(pod) else 0
    o.has_deletion_ts = 1 if pod.get("deletionTimestamp") else 0
    if o.node_type == abi.NT_HEAD:
        st, reason, msg = snp.head_pod_ready_condition(pod)
        o.head_ready_status = snp._COND.get(st, abi.COND_UNKNOWN) if st != "" else abi.COND_UNKNOWN
        o.head_ready_reason, o.head_ready_msg = _s(reason), _s(msg)
        o.pod_ip = _s(pod.get("podIP"))
        o.recreate_hash, o.kuberay_version = _s(ann.get(snp.RECREATE_HASH_ANNOT, "")), _s(ann.get(snp.KUBERAY_VERSION_ANNOT, ""))
    return o


def cluster_obj(c: dict):
    """-> (kr_cluster_obj, what must stay alive while the native call reads it)."""
    spec, status = c.get("spec") or {}, c.get("status") or {}
    ns, name = c.get("namespace", "default"), c["name"]
    o = abi.kr_cluster_obj()
    o.ns, o.name, o.uid = _s(ns), _s(name), _s(c.get("uid"))
    o.resource_version, o.generation = int(c.get("resourceVersion", 0)), int(c.get("generation", 0))
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
    if (c.get("annotations") or {}).get(snp.SKIP_HEAD_RESTART_ANNOT) == "true":
        fl |= abi.CF_SKIP_HEAD_RESTART
    exp = c.get("expectations") or {}
    if exp.get("head", True):
        fl |= abi.CF_HEAD_EXPECT_OK
    if c.get("deletionTimestamp") or c.get("skip"):
        fl |= abi.CF_SKIP
    if status.get("reason", "") != "":
        fl |= abi.CF_OLD_REASON_NONEMPTY
    svc = c.get("headService", {"count": 1, "clusterIP": "10.0.0.1", "name": f"{name}-head-svc"})
    if snp.compute_endpoints(status.get("endpoints"), svc) != status.get("endpoints"):
        fl |= abi.CF_ENDPOINTS_CHANGED
    o.flags = fl
    o.suspend_status = snp.find_suspend_status(status.get("conditions"))
    ext = c.get("extErr") or {}
    o.ext_err_kind = ext.get("kind", 0)
    o.ext_err_msg = _s(ext["message"]) if "message" in ext else _s(None)
    o.old_state = snp._STATE.get(status.get("state", ""), abi.STATE_OTHER)
    for k, key in enumerate(("readyWorkerReplicas", "availableWorkerReplicas", "desiredWorkerReplicas", "minWorkerReplicas", "maxWorkerReplicas")):
        o.old_counts[k] = status.get(key, 0)
    hr_reason = hr_msg = rf_msg = None
    for cond in status.get("conditions") or []:
        slot = snp._COND_SLOT.get(cond.get("type"))
        if slot is None:
            continue
        o.old_cond_status[slot] = snp._COND.get(cond.get("status", ""), abi.COND_UNKNOWN)
        reason, msg = cond.get("reason", ""), cond.get("message", "")
        if slot == abi.COND_PROVISIONED:
            var = snp._PROV_VARIANTS.get((reason, msg), abi.CV_OTHER)
        elif slot in (abi.COND_SUSPENDING, abi.COND_SUSPENDED):
            var = abi.CV_CANONICAL if (reason == cond["type"] and msg == "") else abi.CV_OTHER
        elif slot == abi.COND_HEAD_POD_READY:
            var = abi.CV_HEAD_NOT_FOUND if (reason, msg) == (snp.HEAD_NOT_FOUND_REASON, snp.HEAD_NOT_FOUND_MSG) else abi.CV_HEAD_FROM_POD
            hr_reason, hr_msg = reason, msg
        else:
            var = snp._REPLICA_FAILURE_KIND.get(reason, abi.CV_OTHER)
            rf_msg = msg
        o.old_cond_variant[slot] = var
    o.old_head_ready_reason, o.old_head_ready_msg, o.old_replica_failure_msg = _s(hr_reason), _s(hr_msg), _s(rf_msg)
    head = status.get("head") or {}
    for k, key in enumerate(("podIP", "serviceIP", "podName", "serviceName")):
        o.old_head[k] = _s(head.get(key))
    o.svc_count = min(svc.get("count", 1), 2)
    ip = svc.get("clusterIP", "")
    o.svc_ip_kind = abi.SVCIP_EMPTY if ip == "" else (abi.SVCIP_NONE if ip == "None" else abi.SVCIP_NORMAL)
    o.svc_ip = _s(ip) if ip not in ("", "None") else _s(None)
    o.svc_name = _s(svc.get("name", ""))
    o.status_summary = _s(snp.status_summary_key(status))
    groups = spec.get("workerGroupSpecs") or []
    garr = (abi.kr_group_obj * max(len(groups), 1))()
    keep = []
    for gi, grp in enumerate(groups):
        g = garr[gi]
        g.name = _s(grp["groupName"])
        gf = 0
        for key, fld, nil in (("replicas", "replicas", abi.GF_REPLICAS_NIL), ("minReplicas", "min_replicas", abi.GF_MIN_NIL), ("maxReplicas", "max_replicas", abi.GF_MAX_NIL)):
            v = grp.get(key)
            if v is None:
                gf |= nil
            else:
                setattr(g, fld, v)
        g.num_hosts = grp.get("numOfHosts", 1)
        if grp.get("suspend") is True:
            gf |= abi.GF_SUSPEND
        if exp.get(grp["groupName"], True):
            gf |= abi.GF_EXPECT_OK
        g.flags = gf
        names = grp.get("workersToDelete") or (grp.get("scaleStrategy") or {}).get("workersToDelete") or []
        warr = (abi.kr_str * max(len(names), 1))(*[_s(n) for n in names])
        keep.append(warr)
        g.workers_to_delete, g.n_workers_to_delete = warr, len(names)
    o.groups, o.n_groups = garr, len(groups)
    if "specJson" in c:  # bytes marshalled by the Go side: taken verbatim
        sj = c["specJson"].encode() if isinstance(c["specJson"], str) else bytes(c["specJson"])
        o.spec_json_verbatim = 1
    else:
        sj = json.dumps(spec).encode("utf-8")
    o.spec_json, o.spec_json_len = sj, len(sj)
    return o, (keep, garr, sj)


def job_obj(j: dict) -> abi.kr_job_obj:
    return abi.kr_job_obj(_s(j.get("namespace", "default")), _s(j["name"]), _s((j.get("status") or {}).get("rayClusterName") or None),
                          _s(snp.status_summary_key((j.get("status") or {}).get("rayClusterStatus"))))


def _bind(L):
    P = C.POINTER
    L.kr_packer_create.argtypes = [P(abi.kr_config), P(C.c_void_p)]
    L.kr_packer_destroy.argtypes = [C.c_void_p]; L.kr_packer_destroy.restype = None
    L.kr_packer_engine.argtypes = [C.c_void_p]; L.kr_packer_engine.restype = C.c_void_p
    L.kr_packer_pod_upsert.argtypes = [C.c_void_p, P(abi.kr_pod_obj)]
    L.kr_packer_pod_delete.argtypes = [C.c_void_p, abi.kr_str, abi.kr_str]
    L.kr_packer_cluster_upsert.argtypes = [C.c_void_p, P(abi.kr_cluster_obj)]
    L.kr_packer_cluster_delete.argtypes = [C.c_void_p, abi.kr_str, abi.kr_str]
    L.kr_packer_job_upsert.argtypes = [C.c_void_p, P(abi.kr_job_obj)]
    L.kr_packer_job_delete.argtypes = [C.c_void_p, abi.kr_str, abi.kr_str]
    L.kr_packer_flush.argtypes = [C.c_void_p, P(C.c_uint32)]
    L.kr_packer_sizes.argtypes = [C.c_void_p, P(abi.kr_sizes)]
    L.kr_packer_bufs.argtypes = [C.c_void_p, P(abi.kr_snapshot_bufs)]
    L.kr_packer_intern.argtypes = [C.c_void_p, abi.kr_str]; L.kr_packer_intern.restype = C.c_uint32
    L.kr_packer_string.argtypes = [C.c_void_p, C.c_uint32, P(abi.kr_str)]
    L.kr_packer_cluster_row.argtypes = [C.c_void_p, abi.kr_str, abi.kr_str]; L.kr_packer_cluster_row.restype = C.c_int64
    L.kr_packer_pod_row.argtypes = [C.c_void_p, abi.kr_str, abi.kr_str]; L.kr_packer_pod_row.restype = C.c_int64
    L.kr_packer_pod_key.argtypes = [C.c_void_p, C.c_uint32, P(abi.kr_str), P(abi.kr_str)]
    L.kr_packer_epoch.argtypes = [C.c_void_p, P(C.c_uint64), P(C.c_uint64)]
    L.kr_packer_cluster_epoch.argtypes = [C.c_void_p, C.c_uint32, P(C.c_uint64), P(C.c_uint64)]
    L.kr_packer_last_error.argtypes = [C.c_void_p]; L.kr_packer_last_error.restype = C.c_char_p


class Packer:
    def __init__(self, device=0, max_clusters=1024, max_groups=4096, max_wtd=4096, max_pods=65536, max_heads=2048, max_jobs=1024,
                 max_creates=65536, max_json_bytes=64 << 20, large_clusters=False, wide_clusters=False,
                 huge_clusters=False, wtd_edits=False, spec_rows=False, cluster_creates=False,
                 cluster_deletes=False, group_edits=False, large_growth=False, large_moves=False, bucket_pod_lists=False, json_moves=False,
                 huge_growth=False):
        L = self._L = lib()
        _bind(L)
        if L.kr_device_count() <= 0:
            raise EngineError(abi.KR_E_NO_DEVICE, "no CUDA device visible (this engine has no CPU fallback)")
        cfg = abi.kr_config(device, max_clusters, max_groups, max_wtd, max_pods, max_heads, max_jobs, max_creates, max_json_bytes)
        self._h = C.c_void_p()
        rc = L.kr_packer_create(C.byref(cfg), C.byref(self._h))
        if rc != 0:
            raise EngineError(rc, "kr_packer_create failed")
        self._owned = True
        self._attach_engine(cfg)
        self.set_options(large_clusters, wide_clusters, huge_clusters, wtd_edits, spec_rows, cluster_creates, cluster_deletes, group_edits,
                         large_growth, large_moves, bucket_pod_lists, json_moves, huge_growth)

    @classmethod
    def view(cls, handle: int, cfg: abi.kr_config) -> "Packer":
        """A Packer over a kr_packer it does not own (a group packer's shard: kr_group_packer_shard): every call works on it, close()
        only drops the view."""
        self = cls.__new__(cls)
        self._L = lib()
        _bind(self._L)
        self._h, self._owned = C.c_void_p(handle), False
        self._attach_engine(cfg)
        return self

    def _attach_engine(self, cfg: abi.kr_config):
        self.engine = Engine.__new__(Engine)  # a view over the packer's engine (not owned)
        self.engine._L, self.engine._h, self.engine.sizes, self.engine.cfg = self._L, C.c_void_p(self._L.kr_packer_engine(self._h)), abi.kr_sizes(), cfg

    def set_options(self, large_clusters=False, wide_clusters=False, huge_clusters=False, wtd_edits=False, spec_rows=False, cluster_creates=False,
                    cluster_deletes=False, group_edits=False, large_growth=False, large_moves=False, bucket_pod_lists=False, json_moves=False,
                    huge_growth=False):
        """Switch on the opt-in engine options of this packer's engine (kr_packer_engine)."""
        if large_clusters:  # KR_OPT_LARGE_CLUSTERS, set through kr_packer_engine()
            self.engine.set_large_clusters(True)
        if wide_clusters:  # KR_OPT_WIDE_CLUSTERS, likewise
            self.engine.set_wide_clusters(True)
        if huge_clusters:  # KR_OPT_HUGE_CLUSTERS, likewise
            self.engine.set_huge_clusters(True)
        if wtd_edits:  # KR_OPT_WTD_EDITS, likewise
            self.engine.set_wtd_edits(True)
        if spec_rows:  # KR_OPT_SPEC_ROWS, likewise: flush commits re-emitted specs row by row (PACK_SPEC_ROWS)
            self.engine.set_spec_rows(True)
        if cluster_creates:  # KR_OPT_CLUSTER_CREATES, likewise: a flush that only appends RayClusters / creates and deletes RayJobs stays incremental
            self.engine.set_cluster_creates(True)
        if cluster_deletes:  # KR_OPT_CLUSTER_DELETES, likewise: a flush that deletes RayClusters (swap-remove) stays incremental
            self.engine.set_cluster_deletes(True)
        if group_edits:  # KR_OPT_GROUP_EDITS, likewise: a flush that changes a RayCluster's worker groups stays incremental
            self.engine.set_group_edits(True)
        if large_growth:  # KR_OPT_LARGE_GROWTH, likewise: a RayCluster that scales past its bucket or region stays incremental
            self.engine.set_large_growth(True)
        if large_moves:  # KR_OPT_LARGE_MOVES, likewise: deleting, moving or regrouping a large RayCluster stays incremental
            self.engine.set_large_moves(True)
        if bucket_pod_lists:  # KR_OPT_BUCKET_POD_LISTS, likewise: fetching the pod lists keeps the pipeline and the incremental epoch
            self.engine.set_bucket_pod_lists(True)
        if json_moves:  # KR_OPT_JSON_MOVES, likewise: with spec_rows, a compaction of the JSON arena moves the specs on the device (PACK_JSON_MOVES)
            self.engine.set_json_moves(True)
        if huge_growth:  # KR_OPT_HUGE_GROWTH, likewise: a RayCluster that scales past LARGE_MAX_PODS Pods stays incremental
            self.engine.set_huge_growth(True)

    def _check(self, rc):
        if rc != 0:
            raise EngineError(rc, self._L.kr_packer_last_error(self._h).decode())

    def close(self):
        if self._h:
            self.engine._h = C.c_void_p()
            if self._owned:
                self._L.kr_packer_destroy(self._h)
            self._h = C.c_void_p()

    # ------------------------------------------------------------------ events (dict objects: tests/golden/README.md)
    def upsert_pod(self, pod: dict):
        self._check(self._L.kr_packer_pod_upsert(self._h, C.byref(pod_obj(pod))))

    def delete_pod(self, ns: str, name: str):
        self._check(self._L.kr_packer_pod_delete(self._h, _s(ns), _s(name)))

    def upsert_cluster(self, c: dict):
        o, _keep = cluster_obj(c)
        self._check(self._L.kr_packer_cluster_upsert(self._h, C.byref(o)))

    def delete_cluster(self, ns: str, name: str):
        self._check(self._L.kr_packer_cluster_delete(self._h, _s(ns), _s(name)))

    def upsert_job(self, j: dict):
        self._check(self._L.kr_packer_job_upsert(self._h, C.byref(job_obj(j))))

    def delete_job(self, ns: str, name: str):
        self._check(self._L.kr_packer_job_delete(self._h, _s(ns), _s(name)))

    # ------------------------------------------------------------------ epoch
    def flush(self) -> int:
        mode = C.c_uint32()
        self._check(self._L.kr_packer_flush(self._h, C.byref(mode)))
        self._check(self._L.kr_packer_sizes(self._h, C.byref(self.engine.sizes)))
        return mode.value

    def last_pass(self) -> dict:
        """Engine.last_pass of the packer's engine: the kind of the last pass and why it was not incremental."""
        return self.engine.last_pass()

    def flags(self, **kw) -> abi.kr_flags:
        return abi.default_flags(id_head_not_found_reason=self._L.kr_packer_intern(self._h, _s(snp.HEAD_NOT_FOUND_REASON)),
                                 id_head_not_found_msg=self._L.kr_packer_intern(self._h, _s(snp.HEAD_NOT_FOUND_MSG)), **kw)

    def column(self, name: str):
        """Read-only numpy view of one arena column the packer maintains (live rows only)."""
        import numpy as np
        bufs = abi.kr_snapshot_bufs()
        self._check(self._L.kr_packer_bufs(self._h, C.byref(bufs)))
        dt, mult, dim = next((d, m, dm) for n, d, m, dm in abi.COLUMNS if n == name)
        s = self.engine.sizes
        count = {"clusters": s.n_clusters, "groups": s.n_groups, "wtd": s.n_wtd, "pods": s.n_pods, "heads": s.n_heads, "jobs": s.n_jobs, "json": s.json_bytes}[dim] * mult
        ptr = C.cast(getattr(bufs, name), C.c_void_p).value
        if not count:
            return np.zeros(0, dtype=dt)
        return np.frombuffer((C.c_uint8 * (np.dtype(dt).itemsize * count)).from_address(ptr), dtype=dt, count=count)

    def string(self, i: int):
        out = abi.kr_str()
        self._check(self._L.kr_packer_string(self._h, int(i), C.byref(out)))
        return None if not out.p and out.n == 0 and i == 0 else C.string_at(out.p, out.n).decode()

    def cluster_row(self, ns, name) -> int:
        return int(self._L.kr_packer_cluster_row(self._h, _s(ns), _s(name)))

    def pod_row(self, ns, name) -> int:
        return int(self._L.kr_packer_pod_row(self._h, _s(ns), _s(name)))

    def pod_key(self, row: int):
        a, b = abi.kr_str(), abi.kr_str()
        self._check(self._L.kr_packer_pod_key(self._h, row, C.byref(a), C.byref(b)))
        return (None, None) if not a.p else (C.string_at(a.p, a.n).decode(), C.string_at(b.p, b.n).decode())

    def epoch(self) -> tuple[int, int]:
        e, v = C.c_uint64(), C.c_uint64()
        self._check(self._L.kr_packer_epoch(self._h, C.byref(e), C.byref(v)))
        return e.value, v.value

    def cluster_epoch(self, row: int) -> tuple[int, int]:
        rv, gen = C.c_uint64(), C.c_uint64()
        self._check(self._L.kr_packer_cluster_epoch(self._h, row, C.byref(rv), C.byref(gen)))
        return rv.value, gen.value


def shard_of_key(ns: str, cluster_name, n: int) -> int:
    """kr_shard_of_key: the shard of the routing key (namespace, RayCluster name); cluster_name None is an absent label."""
    return int(lib().kr_shard_of_key(_s(ns), _s(cluster_name), n))


class GroupPacker:
    """kr_group_packer: one native packer per shard behind one handle.  Events go to the shard of their (namespace, RayCluster
    name) key; flush() / reconcile() run every shard on its own worker thread.  `.shards` are non-owning Packer views
    (kr_group_packer_shard) for the per-shard reads; `.group` is the kr_group over the shards' engines (all-gather)."""

    def __init__(self, devices: list[int], max_clusters=1024, max_groups=4096, max_wtd=4096, max_pods=65536, max_heads=2048, max_jobs=1024,
                 max_creates=65536, max_json_bytes=64 << 20, large_clusters=False, wide_clusters=False, huge_clusters=False,
                 wtd_edits=False, spec_rows=False, cluster_creates=False, cluster_deletes=False, group_edits=False, large_growth=False,
                 large_moves=False, bucket_pod_lists=False, json_moves=False, huge_growth=False):
        L = self._L = lib()
        _bind(L)
        if L.kr_device_count() <= 0:
            raise EngineError(abi.KR_E_NO_DEVICE, "no CUDA device visible (this engine has no CPU fallback)")
        self.n = len(devices)
        cfg = abi.kr_config(0, max_clusters, max_groups, max_wtd, max_pods, max_heads, max_jobs, max_creates, max_json_bytes)
        dv = (C.c_int32 * max(self.n, 1))(*devices)
        self._h = C.c_void_p()
        rc = L.kr_group_packer_create(C.byref(cfg), dv, self.n, C.byref(self._h))
        if rc != 0:
            raise EngineError(rc, "kr_group_packer_create failed")
        self.shards = [Packer.view(L.kr_group_packer_shard(self._h, i), cfg) for i in range(self.n)]
        for sh in self.shards:  # options are per shard (the native group packer does not forward them)
            sh.set_options(large_clusters, wide_clusters, huge_clusters, wtd_edits, spec_rows, cluster_creates, cluster_deletes, group_edits,
                           large_growth, large_moves, bucket_pod_lists, json_moves, huge_growth)
        self.group = Group.__new__(Group)  # a view over the group packer's kr_group (not owned: close() is the group packer's)
        self.group._L, self.group._h, self.group.n, self.group.engines = L, C.c_void_p(L.kr_group_packer_group(self._h)), self.n, [sh.engine for sh in self.shards]

    def _check(self, rc):
        if rc != 0:
            raise EngineError(rc, self._L.kr_group_packer_last_error(self._h).decode())

    def close(self):
        if self._h:
            for sh in self.shards:
                sh.close()
            self.group._h = C.c_void_p()
            self._L.kr_group_packer_destroy(self._h)
            self._h = C.c_void_p()

    def shard_of(self, ns: str, cluster_name) -> int:
        return shard_of_key(ns, cluster_name, self.n)

    # ------------------------------------------------------------------ events
    def upsert_pod(self, pod: dict):
        self._check(self._L.kr_group_packer_pod_upsert(self._h, C.byref(pod_obj(pod))))

    def delete_pod(self, ns: str, name: str):
        self._check(self._L.kr_group_packer_pod_delete(self._h, _s(ns), _s(name)))

    def upsert_cluster(self, c: dict):
        o, _keep = cluster_obj(c)
        self._check(self._L.kr_group_packer_cluster_upsert(self._h, C.byref(o)))

    def delete_cluster(self, ns: str, name: str):
        self._check(self._L.kr_group_packer_cluster_delete(self._h, _s(ns), _s(name)))

    def upsert_job(self, j: dict):
        self._check(self._L.kr_group_packer_job_upsert(self._h, C.byref(job_obj(j))))

    def delete_job(self, ns: str, name: str):
        self._check(self._L.kr_group_packer_job_delete(self._h, _s(ns), _s(name)))

    # ------------------------------------------------------------------ epoch
    def flush(self) -> list[int]:
        """Every shard's kr_packer_flush, in parallel -> each shard's mode."""
        modes = (C.c_uint32 * self.n)()
        self._check(self._L.kr_group_packer_flush(self._h, modes))
        for sh in self.shards:
            sh._check(self._L.kr_packer_sizes(sh._h, C.byref(sh.engine.sizes)))
        return list(modes)

    def flags(self, **kw) -> list[abi.kr_flags]:
        """One kr_flags per shard (the HeadPodReady string ids are each shard's own)."""
        return [sh.flags(**kw) for sh in self.shards]

    def reconcile(self, flags: list[abi.kr_flags], copy: bool = True) -> list[abi.Results]:
        fl = (abi.kr_flags * self.n)(*flags)
        views = (abi.kr_results_view * self.n)()
        self._check(self._L.kr_group_packer_reconcile(self._h, fl, views))
        return [sh.engine._results(views[i], copy) for i, sh in enumerate(self.shards)]

    def last_passes(self) -> list[dict]:
        """Every shard's Engine.last_pass: each shard's engine reports its own pass."""
        return [sh.last_pass() for sh in self.shards]

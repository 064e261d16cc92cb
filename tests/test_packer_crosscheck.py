"""Cross-check of the packer's host-side evaluations against a second, independent reading of the Go source.

The engine decides from packed bits (p_packed, the head-aux rows); a packer bug would be invisible to the oracle-vs-engine parity
tests because both read the same packed snapshot.  Here the raw objects are evaluated again, by functions written directly from
the reference text (NOT sharing code with kuberay_b200/snapshot.py), and compared with what pack_objects encoded:
  shouldDeletePod + getRayContainerStateTerminated   raycluster_controller.go:1181-1248
  FindHeadPodReadyCondition + firstNotReadyContainerStatus   utils/util.go:81-134
  the replica-index label through strconv.Atoi        raycluster_controller.go:857-860
  node type / phase / PodReady / deletionTimestamp as the selectors and calculateStatus read them (:1583-1603, util.go:584-603)
  FindRayClusterSuspendStatus                          utils/util.go:153-162
plus the containerStatuses forms the fuzz generator does not produce (ray container found by NAME, not by position)."""
import copy
import re

import numpy as np
import pytest

import fuzz_objects
from kuberay_b200 import abi
from kuberay_b200 import snapshot as snp

L_TYPE, L_RIDX = "ray.io/node-type", "ray.io/worker-group-replica-index"


# ---- independent restatements (plain Python over the raw dicts) ----------------------------------------------------------------
def go_ray_container_terminated(pod):
    """getRayContainerStateTerminated: the status whose NAME equals spec.containers[0].name; nil when not found."""
    if "rayContainerTerminated" in pod:  # the fixtures' shorthand for "the ray container's state.terminated is set"
        return bool(pod["rayContainerTerminated"])
    containers = pod.get("containers") or []
    if not containers:
        return False
    want = containers[0].get("name")
    for cs in pod.get("containerStatuses") or []:
        if cs.get("name") == want:
            return (cs.get("state") or {}).get("terminated") is not None  # a non-nil pointer, even to an empty state
    return False


def go_should_delete_pod(pod):
    phase = pod.get("phase", "")
    if phase in ("Failed", "Succeeded"):
        return True
    if phase == "Running" and go_ray_container_terminated(pod):
        return pod.get("restartPolicy") == "Never"
    return False


def go_atoi(text):
    """strconv.Atoi: optional single sign, one or more ASCII digits, nothing else; must fit a 64-bit int."""
    if text is None:
        return None
    body = text[1:] if text[:1] in "+-" else text
    if body == "" or any(ch not in "0123456789" for ch in body):
        return None
    v = int(body)
    if text[:1] == "-":
        v = -v
    return v if -(1 << 63) <= v <= (1 << 63) - 1 else None


def go_find_head_pod_ready_condition(pod):
    status, reason, message = "False", "Unknown", ""
    for cond in pod.get("conditions") or []:
        if cond.get("type") != "Ready":
            continue
        status = cond.get("status", "")
        message = cond.get("message") or ""
        r = cond.get("reason") or ""
        if cond.get("status") == "True" and r == "":
            r = "HeadPodRunningAndReady"
        if r != "":
            reason = r
        if r == "ContainersNotReady":
            for cs in pod.get("containerStatuses") or []:
                st = cs.get("state") or {}
                pick = None
                if st.get("waiting") is not None:
                    pick = st["waiting"]
                elif st.get("terminated") is not None:
                    pick = st["terminated"]
                if pick is not None:
                    if message != "":
                        message += "; "
                    message += f"{cs.get('name', '')}: {pick.get('message', '')}"
                    reason = pick.get("reason", "")
                    break
        break
    return status, reason, message


def go_suspend_status(conditions):
    for c in conditions or []:
        if c.get("type") == "RayClusterSuspending" and c.get("status") == "True":
            return abi.SUSPEND_SUSPENDING
        if c.get("type") == "RayClusterSuspended" and c.get("status") == "True":
            return abi.SUSPEND_SUSPENDED
    return abi.SUSPEND_NONE


# ---- what the kernels do with the packed word (kr_common.cuh should_delete) -----------------------------------------------------
def packed_should_delete(pk):
    ph = (pk >> abi.PP_PHASE_SHIFT) & 7
    return ph in (abi.PHASE_FAILED, abi.PHASE_SUCCEEDED) or (ph == abi.PHASE_RUNNING and bool(pk & abi.PP_RAY_TERMINATED) and bool(pk & abi.PP_RESTART_NEVER))


PHASES = {"": abi.PHASE_EMPTY, "Pending": abi.PHASE_PENDING, "Running": abi.PHASE_RUNNING, "Succeeded": abi.PHASE_SUCCEEDED, "Failed": abi.PHASE_FAILED, "Unknown": abi.PHASE_UNKNOWN}
NODE_TYPES = {"head": abi.NT_HEAD, "worker": abi.NT_WORKER, "redis-cleanup": abi.NT_REDIS}
CONDS = {"True": abi.COND_TRUE, "False": abi.COND_FALSE, "Unknown": abi.COND_UNKNOWN}


def _check_snapshot(clusters, pods, jobs):
    snap, meta = snp.pack_objects(clusters, pods, jobs)
    it = meta.interner
    assert snap.dims["pods"] == len(pods)
    for i, pod in enumerate(pods):
        pk = int(snap.p_packed[i])
        labels = pod.get("labels") or {}
        assert packed_should_delete(pk) == go_should_delete_pod(pod), (i, pod)
        assert (pk >> abi.PP_NODE_TYPE_SHIFT) & 3 == NODE_TYPES.get(labels.get(L_TYPE, ""), abi.NT_NONE), pod
        assert (pk >> abi.PP_PHASE_SHIFT) & 7 == PHASES.get(pod.get("phase", ""), abi.PHASE_UNKNOWN), pod
        ready = next((c for c in pod.get("conditions") or [] if c.get("type") == "Ready"), None)
        want_ready = abi.COND_ABSENT if ready is None else CONDS.get(ready.get("status", ""), abi.COND_UNKNOWN)
        assert (pk >> abi.PP_READY_SHIFT) & 3 == want_ready, pod
        assert bool(pk & abi.PP_HAS_DELETION_TS) == bool(pod.get("deletionTimestamp")), pod
        v = go_atoi(labels.get(L_RIDX))
        assert bool(pk & abi.PP_HAS_REPLICA_IDX) == (v is not None), (labels.get(L_RIDX), pk)
        if v is not None and -(1 << 31) <= v < (1 << 31):
            assert int(snap.p_replica_index[i]) == v
        assert it.str(int(snap.p_name_id[i])) == pod["name"] and it.str(int(snap.p_ns_id[i])) == pod.get("namespace", "default")
    # head-aux rows: one per pod whose node-type label is head, in pod order
    heads = [i for i, p in enumerate(pods) if (p.get("labels") or {}).get(L_TYPE) == "head"]
    assert snap.dims["heads"] == len(heads) and snap.h_pod_idx.tolist() == heads
    for h, i in enumerate(heads):
        status, reason, message = go_find_head_pod_ready_condition(pods[i])
        assert int(snap.h_ready_status[h]) == CONDS.get(status, abi.COND_UNKNOWN), (pods[i], status)
        assert (it.str(int(snap.h_ready_reason_id[h])) or "") == reason and (it.str(int(snap.h_ready_msg_id[h])) or "") == message, (pods[i], reason, message)
    for ci, key in enumerate(meta.cluster_keys):
        c = next(c for c in clusters if (c.get("namespace", "default"), c["name"]) == key)
        assert int(snap.c_suspend_status[ci]) == go_suspend_status((c.get("status") or {}).get("conditions")), c.get("status")


@pytest.mark.parametrize("seed", range(40))
def test_packed_bits_agree_with_an_independent_reading_of_the_go_source(seed):
    clusters, pods, jobs = fuzz_objects.generate(seed, big=seed % 3 == 0)
    _check_snapshot(clusters, pods, jobs)


def test_container_status_forms_the_fuzzer_does_not_generate():
    """The Ray container is found BY NAME (containerStatuses has no guaranteed order, :1233-1236); a missing status means "not
    terminated"; ContainersNotReady takes the first waiting / terminated status, whatever container it belongs to."""
    clusters, pods, jobs = fuzz_objects.generate(7)
    base = {"namespace": clusters[0].get("namespace", "default"), "labels": {"ray.io/cluster": clusters[0]["name"], "ray.io/group": "headgroup", L_TYPE: "head"},
            "phase": "Running", "restartPolicy": "Never", "containers": [{"name": "ray-head"}, {"name": "sidecar"}]}
    variants = [
        ("t-sidecar-first", [{"name": "sidecar", "state": {"terminated": {"reason": "Error", "message": "boom"}}}, {"name": "ray-head", "state": {"running": {}}}]),
        ("t-ray-second", [{"name": "sidecar", "state": {"running": {}}}, {"name": "ray-head", "state": {"terminated": {"reason": "OOMKilled", "message": "oom"}}}]),
        ("t-no-status", []),
        ("t-other-name", [{"name": "not-ray", "state": {"terminated": {"reason": "Completed"}}}]),
        ("t-empty-terminated", [{"name": "ray-head", "state": {"terminated": {}}}]),
    ]
    extra = []
    for name, statuses in variants:
        p = copy.deepcopy(base)
        p["name"] = name
        p["containerStatuses"] = statuses
        p["conditions"] = [{"type": "Ready", "status": "False", "reason": "ContainersNotReady", "message": "containers with unready status: [ray-head]"}]
        extra.append(p)
    w = copy.deepcopy(base)
    w.update(name="t-waiting", containerStatuses=[{"name": "ray-head", "state": {"waiting": {"reason": "ImagePullBackOff", "message": "Back-off pulling image"}}}],
             conditions=[{"type": "Ready", "status": "False", "reason": "ContainersNotReady", "message": ""}])
    extra.append(w)
    allpods = pods + extra
    _check_snapshot(clusters, allpods, jobs)
    got = {p["name"]: (go_should_delete_pod(p), go_find_head_pod_ready_condition(p)) for p in extra}
    assert got["t-sidecar-first"][0] is False and got["t-ray-second"][0] is True and got["t-no-status"][0] is False and got["t-other-name"][0] is False
    assert got["t-empty-terminated"][0] is True
    assert got["t-sidecar-first"][1] == ("False", "Error", "containers with unready status: [ray-head]; sidecar: boom")
    assert got["t-waiting"][1] == ("False", "ImagePullBackOff", "ray-head: Back-off pulling image")


@pytest.mark.parametrize("text,want", [("0", 0), ("-1", -1), ("+3", 3), ("007", 7), ("", None), ("abc", None), ("1_000", None), (" 1", None), ("1 ", None), ("٣", None),
                                       ("9223372036854775807", 9223372036854775807), ("9223372036854775808", None), ("-9223372036854775808", -(1 << 63)), ("+", None), ("--1", None)])
def test_replica_index_label_parses_like_strconv_atoi(text, want):
    assert go_atoi(text) == want
    pk, ridx = snp.pack_pod_word({"labels": {L_RIDX: text}, "phase": "Running"})
    assert bool(pk & abi.PP_HAS_REPLICA_IDX) == (want is not None)
    assert re.fullmatch(r"[+-]?[0-9]+", text) is not None or want is None

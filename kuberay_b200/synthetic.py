"""Deterministic synthetic snapshots (SURVEY.md §8(d), BASELINE.json configs).

Everything is generated directly as columns (ids, not strings) with numpy, seed 20260921, so that 10^6..10^8 pods are
cheap to produce.  Distributions follow SURVEY §8(d): phase Running 96 % / Pending 2 % / Failed 1 % / Succeeded 1 %;
PodReady=True for 95 % of Running; ray-container-terminated 0.5 % (restartPolicy Never 50/50); replicas uniform in
[actual-3, actual+3] clamped by min=1, max in {2^31-1, 200}; workersToDelete 0-2 names on 10 % of autoscaling groups
(20 % of those names non-existent); 1 % clusters suspended; 1 % Recreate-upgrade with a head hash annotation (half of them
mismatching); 2 % expectation-unsatisfied groups; spec JSON from 4 templates (~1.5/2.5/4/6 KB) with cluster-specific fields;
pods emitted in a seeded shuffled order.
"""
from __future__ import annotations

import base64
import hashlib
from dataclasses import dataclass

import numpy as np

from . import abi
from .snapshot import Snapshot

SEED = 20260921

CONFIGS = {
    # name: (clusters, pods per cluster, groups per cluster)
    "C1": dict(n_clusters=10, pods_per_cluster=4, groups=1),
    "C2": dict(n_clusters=1000, pods_per_cluster=32, groups=1),
    "C3": dict(n_clusters=10000, pods_per_cluster=100, groups=1),
    "C3G3": dict(n_clusters=10000, pods_per_cluster=100, groups=3),
    "C3x10": dict(n_clusters=100000, pods_per_cluster=100, groups=1),
    "C4": dict(n_clusters=10000, pods_per_cluster=100, groups=1, jobs=True),
    "C5": dict(n_clusters=1000, pods_per_cluster=100, groups=1, autoscaling_frac=1.0),
    # C3 with TPU-slice style worker groups: a quarter of the groups have numOfHosts=4 (about 44 % of the RayClusters hold one)
    "C3MH": dict(n_clusters=10000, pods_per_cluster=100, groups=2, multihost_frac=0.25),
    # C3 with 20 large RayClusters of 2 000 pods each (worker pods of the other RayClusters move into them; the total stays 1 M):
    # the fleet KR_OPT_LARGE_CLUSTERS keeps on the bucket pipeline
    "C3L": dict(n_clusters=10000, pods_per_cluster=100, groups=1, n_large=20, large_pods=2000),
    # C3 with 100 wide RayClusters (1 %) of 48 worker groups each (one per accelerator type / node pool): the fleet
    # KR_OPT_WIDE_CLUSTERS keeps on the bucket pipeline
    "C3W": dict(n_clusters=10000, pods_per_cluster=100, groups=1, n_wide=100, wide_groups=48),
    # C3 with 2 huge RayClusters of 20 000 pods each (a batch-inference or data-processing job of CPU workers): the fleet
    # KR_OPT_HUGE_CLUSTERS (with KR_OPT_LARGE_CLUSTERS) keeps on the bucket pipeline
    "C3H": dict(n_clusters=10000, pods_per_cluster=100, groups=1, n_large=2, large_pods=20000),
}


@dataclass
class SynthParams:
    n_clusters: int = 10000
    pods_per_cluster: int = 100       # 1 head + (P-1) workers
    groups: int = 1
    clusters_per_namespace: int = 100  # benchmark/perf-tests/10000-raycluster/config.yaml:2-3,36-39
    autoscaling_frac: float = 0.3
    suspended_frac: float = 0.01
    recreate_frac: float = 0.01
    expect_pending_frac: float = 0.02
    wtd_group_frac: float = 0.10
    orphan_frac: float = 0.001
    multihost_frac: float = 0.0       # fraction of groups with numOfHosts=4 and replica-name labels
    steady_frac: float = 0.95         # clusters whose old status already equals the recomputed one are not forced
    jobs: bool = False
    shuffle: bool = True
    healthy: bool = False             # True: every pod Running+Ready (steady-state sweep, no unhealthy aborts)
    seed: int = SEED
    rank: int = 0                     # UID-hash shard (SURVEY §8(e)): keep clusters with uid_hash % world == rank
    world: int = 1
    cluster_id_base: int = 0          # global index of the first generated cluster (weak-scaling shards)
    n_large: int = 0                  # RayClusters (spread over the fleet) grown to large_pods pods with worker pods of the others
    large_pods: int = 2000
    n_wide: int = 0                   # RayClusters (spread over the fleet) whose worker group 0 is split into wide_groups groups
    wide_groups: int = 48


def _splitmix64(x: np.ndarray) -> np.ndarray:
    x = (x + np.uint64(0x9E3779B97F4A7C15)).astype(np.uint64)
    z = x
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


_TEMPLATE_SIZES = (1536, 2560, 4096, 6144)


def _json_templates() -> list[bytes]:
    """Four muted-spec JSON bodies of ~1.5/2.5/4/6 KB, shaped like json.Marshal(RayClusterSpec) output."""
    out = []
    for size in _TEMPLATE_SIZES:
        head = ('{"headGroupSpec":{"template":{"metadata":{},"spec":{"containers":[{"name":"ray-head","image":"rayproject/ray:2.46.0-XXXXXXXX",'
                '"ports":[{"name":"gcs-server","containerPort":6379},{"name":"dashboard","containerPort":8265},{"name":"client","containerPort":10001}],'
                '"env":[{"name":"CLUSTER_ID","value":"XXXXXXXX"}')
        tail = ('],"resources":{"limits":{"cpu":"2","memory":"4Gi"},"requests":{"cpu":"2","memory":"4Gi"}}}]}},"rayStartParams":{"dashboard-host":"0.0.0.0"}},'
                '"rayVersion":"2.46.0","workerGroupSpecs":[{"groupName":"group-0","minReplicas":null,"maxReplicas":null,"rayStartParams":{},'
                '"template":{"metadata":{},"spec":{"containers":[{"name":"ray-worker","image":"rayproject/ray:2.46.0-XXXXXXXX",'
                '"resources":{"limits":{"cpu":"1","memory":"2Gi"},"requests":{"cpu":"1","memory":"2Gi"}}}]}},"scaleStrategy":{}}]}')
        env = []
        i = 0
        while len(head) + len(tail) + sum(len(e) for e in env) < size - 48:
            env.append(',{"name":"RAY_ENV_%04d","value":"v%04d-XXXXXXXX"}' % (i, i))
            i += 1
        body = head + "".join(env) + tail
        out.append(body.encode())
    return out


def _patch_digits(arr2d: np.ndarray, template: bytes, values: np.ndarray):
    """Overwrite every 'XXXXXXXX' in each row with the 8-digit decimal of that row's value."""
    pos = []
    start = 0
    while True:
        k = template.find(b"XXXXXXXX", start)
        if k < 0:
            break
        pos.append(k)
        start = k + 8
    digits = np.zeros((values.size, 8), dtype=np.uint8)
    v = values.astype(np.int64).copy()
    for d in range(7, -1, -1):
        digits[:, d] = 48 + (v % 10)
        v //= 10
    for k in pos:
        arr2d[:, k:k + 8] = digits


def generate(params: SynthParams | None = None, **kw) -> tuple[Snapshot, abi.kr_flags]:
    p = params or SynthParams(**kw)
    rng = np.random.default_rng(p.seed + 7919 * p.rank)
    Nc, P, G = p.n_clusters, p.pods_per_cluster, p.groups
    W = P - 1  # workers per cluster
    assert W >= G >= 1 or (G >= 1 and W >= 0)

    # ---- id space (interner convention: 0 absent, 1 "")
    nns = max(1, (Nc + p.clusters_per_namespace - 1) // p.clusters_per_namespace)
    nid = 2
    ID_HEAD_NOT_FOUND_REASON, ID_HEAD_NOT_FOUND_MSG, ID_HEADGROUP, ID_READY_REASON, ID_NOTREADY_REASON, ID_NOTREADY_MSG = range(nid, nid + 6)
    nid += 6
    ns_ids = np.arange(nid, nid + nns, dtype=np.uint32); nid += nns
    group_ids = np.arange(nid, nid + G, dtype=np.uint32); nid += G
    cname_ids = np.arange(nid, nid + Nc, dtype=np.uint32); nid += Nc
    svc_name_ids = np.arange(nid, nid + Nc, dtype=np.uint32); nid += Nc
    svc_ip_ids = np.arange(nid, nid + Nc, dtype=np.uint32); nid += Nc
    Np_cluster = Nc * P
    n_orphans = int(Np_cluster * p.orphan_frac)
    Np = Np_cluster + n_orphans
    pod_name_ids = np.arange(nid, nid + Np, dtype=np.uint32); nid += Np
    pod_ip_base = nid; nid += Nc
    replica_name_base = nid; nid += Np
    ghost_cluster_id = nid; nid += 1
    ghost_name_base = nid; nid += 4 * Nc * G + 16
    summary_base = nid; nid += 2 * Nc + 2

    cidx = np.arange(Nc, dtype=np.int64)
    gcid = cidx + p.cluster_id_base  # global cluster number (unique across shards)
    c_ns = ns_ids[(cidx // p.clusters_per_namespace) % nns]

    # ---- cluster-level draws
    u = rng.random((Nc, 8))
    autoscaling = u[:, 0] < p.autoscaling_frac
    suspended_spec = u[:, 1] < p.suspended_frac
    recreate = (u[:, 2] < p.recreate_frac) & ~suspended_spec
    head_expect_pending = u[:, 3] < 0.005
    skip = u[:, 4] < 0.002

    # ---- groups
    Ng = Nc * G
    g_cluster = np.repeat(cidx, G)
    g_local = np.tile(np.arange(G), Nc)
    # workers of a cluster are split evenly over its groups
    base, extra = divmod(W, G)
    g_actual = (base + (g_local < extra)).astype(np.int64)
    gu = rng.random((Ng, 6))
    g_mh = gu[:, 5] < p.multihost_frac
    hosts = np.where(g_mh, 4, 1).astype(np.int32)
    actual_replicas = np.where(g_mh, g_actual // 4, g_actual)
    g_replicas = (actual_replicas + rng.integers(-3, 4, Ng)).astype(np.int64)
    if p.healthy:
        g_replicas = actual_replicas.copy()
    g_min = np.ones(Ng, dtype=np.int32)
    g_max = np.where(gu[:, 0] < 0.5, np.int64(2 ** 31 - 1), np.int64(200)).astype(np.int64)
    g_max = np.where(g_mh, 200, g_max)
    g_flags = np.full(Ng, abi.GF_EXPECT_OK, dtype=np.uint32)
    g_flags[gu[:, 1] < p.expect_pending_frac] &= ~np.uint32(abi.GF_EXPECT_OK)
    g_flags[gu[:, 2] < 0.005] |= abi.GF_SUSPEND
    g_flags[gu[:, 3] < 0.01] |= abi.GF_REPLICAS_NIL
    if p.healthy:
        g_flags[:] = abi.GF_EXPECT_OK

    # ---- pods (cluster-major order first, shuffled at the end)
    pc = np.repeat(cidx, P)                       # owning cluster
    slot = np.tile(np.arange(P), Nc)              # 0 = head, 1.. = workers
    is_head = slot == 0
    wslot = np.maximum(slot - 1, 0)
    # worker -> group: first (base+1)*extra workers in the fat groups
    cut = (base + 1) * extra
    pg_local = np.where(wslot < cut, wslot // max(base + 1, 1), extra + (wslot - cut) // max(base, 1)).astype(np.int64)
    pg_local = np.minimum(pg_local, G - 1)
    pu = rng.random((Nc * P, 4))
    phase = np.full(Nc * P, abi.PHASE_RUNNING, dtype=np.uint32)
    if not p.healthy:
        phase[pu[:, 0] < 0.04] = abi.PHASE_PENDING
        phase[pu[:, 0] < 0.02] = abi.PHASE_FAILED
        phase[pu[:, 0] < 0.01] = abi.PHASE_SUCCEEDED
        # heads are healthier: keep 99.8 % of heads Running
        phase[is_head & (pu[:, 3] > 0.002)] = abi.PHASE_RUNNING
    ready = np.where(phase == abi.PHASE_RUNNING, np.where(pu[:, 1] < 0.95, abi.COND_TRUE, abi.COND_FALSE), abi.COND_ABSENT).astype(np.uint32)
    if p.healthy:
        ready[:] = abi.COND_TRUE
    terminated = (pu[:, 2] < 0.005) & ~np.bool_(p.healthy)
    never = rng.random(Nc * P) < 0.5
    packed = (np.where(is_head, abi.NT_HEAD, abi.NT_WORKER).astype(np.uint32) << abi.PP_NODE_TYPE_SHIFT) \
        | (phase << abi.PP_PHASE_SHIFT) | (ready << abi.PP_READY_SHIFT)
    packed = packed | np.where(terminated, np.uint32(abi.PP_RAY_TERMINATED), np.uint32(0)) | np.where(never, np.uint32(abi.PP_RESTART_NEVER), np.uint32(0))
    # replica index labels: workers carry their position within the group for 90 % of clusters
    pos_in_group = np.where(wslot < cut, wslot % max(base + 1, 1), (wslot - cut) % max(base, 1)).astype(np.int64)
    pg_global = pc * G + pg_local
    mh_pod = g_mh[pg_global] & ~is_head
    rep_idx = np.where(mh_pod, pos_in_group // 4, pos_in_group).astype(np.int32)
    has_idx = (~is_head) & (rng.random(Nc * P) < 0.9)
    packed = packed | np.where(has_idx, np.uint32(abi.PP_HAS_REPLICA_IDX), np.uint32(0))
    rep_idx = np.where(has_idx, rep_idx, 0).astype(np.int32)
    rep_name = np.where(mh_pod, replica_name_base + (pg_global * 4096 + pos_in_group // 4), 0).astype(np.uint32)

    p_ns = c_ns[pc]
    p_cname = cname_ids[pc]
    p_gname = np.where(is_head, np.uint32(ID_HEADGROUP), group_ids[pg_local]).astype(np.uint32)
    p_name = pod_name_ids[:Nc * P]

    # ---- workersToDelete
    wtd_groups = np.flatnonzero(autoscaling[g_cluster] & (gu[:, 4] < p.wtd_group_frac) & ~np.bool_(p.healthy))
    wtd_cnt = np.zeros(Ng, dtype=np.uint32)
    wtd_cnt[wtd_groups] = rng.integers(0, 3, wtd_groups.size)
    g_wtd_off = np.concatenate([[0], np.cumsum(wtd_cnt)[:-1]]).astype(np.uint32) if Ng else np.zeros(0, np.uint32)
    Nw = int(wtd_cnt.sum())
    w_name = np.zeros(Nw, dtype=np.uint32)
    if Nw:
        w_group = np.repeat(np.arange(Ng), wtd_cnt)
        ghost = rng.random(Nw) < 0.2
        # pick an existing worker of that group: cluster-major pod index = c*P + 1 + first worker slot of group + k
        gl = g_local[w_group]
        first_slot = np.where(gl < extra, gl * (base + 1), cut + (gl - extra) * base)
        k = (rng.random(Nw) * np.maximum(g_actual[w_group], 1)).astype(np.int64)
        tgt = g_cluster[w_group] * P + 1 + first_slot + np.minimum(k, np.maximum(g_actual[w_group] - 1, 0))
        w_name = np.where(ghost | (g_actual[w_group] == 0), ghost_name_base + np.arange(Nw), p_name[np.minimum(tgt, Nc * P - 1)]).astype(np.uint32)

    # ---- JSON arena
    templates = _json_templates()
    tsel = (gcid % 4).astype(np.int64)
    lens = np.array([len(t) for t in templates], dtype=np.int64)
    padded = (lens + 15) & ~15
    c_json_len = lens[tsel].astype(np.uint32)
    c_json_off = np.concatenate([[0], np.cumsum(padded[tsel])[:-1]]).astype(np.uint64)
    json_bytes = int(padded[tsel].sum())
    json = np.zeros(json_bytes, dtype=np.uint8)
    for t in range(4):
        rows = np.flatnonzero(tsel == t)
        if rows.size == 0:
            continue
        block = np.tile(np.frombuffer(templates[t].ljust(int(padded[t]), b"\0"), dtype=np.uint8), (rows.size, 1))
        _patch_digits(block, templates[t], gcid[rows] % 100000000)
        idx = (c_json_off[rows].astype(np.int64)[:, None] + np.arange(int(padded[t]))[None, :])
        json[idx.ravel()] = block.ravel()

    # ---- head-aux rows
    head_pods_cm = np.flatnonzero(is_head)  # cluster-major pod index of every head
    Nh = head_pods_cm.size
    h_ready_status = np.where(ready[head_pods_cm] == abi.COND_TRUE, abi.COND_TRUE, abi.COND_FALSE).astype(np.uint8)
    h_reason = np.where(h_ready_status == abi.COND_TRUE, ID_READY_REASON, ID_NOTREADY_REASON).astype(np.uint32)
    h_msg = np.where(h_ready_status == abi.COND_TRUE, 1, ID_NOTREADY_MSG).astype(np.uint32)
    h_ip = (pod_ip_base + cidx).astype(np.uint32)
    h_annot_state = np.zeros(Nh, dtype=np.uint8)
    h_version_state = np.full(Nh, abi.VER_CURRENT, dtype=np.uint8)
    h_annot_hash = np.zeros((Nh, 32), dtype=np.uint8)
    for c in np.flatnonzero(recreate):
        off, ln = int(c_json_off[c]), int(c_json_len[c])
        true_hash = base64.b32hexencode(hashlib.sha1(json[off:off + ln].tobytes()).digest())
        r = rng.random()
        h_annot_state[c] = abi.ANNOT_HASH32
        if r < 0.5:
            h_annot_hash[c] = np.frombuffer(true_hash, dtype=np.uint8)
        elif r < 0.9:
            h_annot_hash[c] = np.frombuffer(true_hash[::-1], dtype=np.uint8)
        else:
            h_annot_hash[c] = np.frombuffer(true_hash[::-1], dtype=np.uint8)
            h_version_state[c] = abi.VER_DIFFERENT

    # ---- shuffle pods (informer List order is arbitrary)
    # orphans: pods labelled with a cluster name that is not in the snapshot
    o_ns = ns_ids[rng.integers(0, nns, n_orphans)] if n_orphans else np.zeros(0, np.uint32)
    all_ns = np.concatenate([p_ns, o_ns]).astype(np.uint32)
    all_cname = np.concatenate([p_cname, np.full(n_orphans, ghost_cluster_id, dtype=np.uint32)]).astype(np.uint32)
    all_gname = np.concatenate([p_gname, np.full(n_orphans, group_ids[0], dtype=np.uint32)]).astype(np.uint32)
    all_name = np.concatenate([p_name, pod_name_ids[Nc * P:]]).astype(np.uint32)
    all_packed = np.concatenate([packed, np.full(n_orphans, (abi.NT_WORKER << abi.PP_NODE_TYPE_SHIFT) | (abi.PHASE_RUNNING << abi.PP_PHASE_SHIFT) | (abi.COND_TRUE << abi.PP_READY_SHIFT), dtype=np.uint32)]).astype(np.uint32)
    all_ridx = np.concatenate([rep_idx, np.zeros(n_orphans, np.int32)]).astype(np.int32)
    all_rname = np.concatenate([rep_name, np.zeros(n_orphans, np.uint32)]).astype(np.uint32)
    perm = rng.permutation(Np) if p.shuffle else np.arange(Np)
    inv = np.empty(Np, dtype=np.int64)
    inv[perm] = np.arange(Np)

    s = Snapshot(Nc, Ng, Nw, Np, Nh, Nc if p.jobs else 0, json_bytes)
    s.p_ns_id[:] = all_ns[perm]; s.p_cluster_name_id[:] = all_cname[perm]; s.p_group_name_id[:] = all_gname[perm]
    s.p_name_id[:] = all_name[perm]; s.p_packed[:] = all_packed[perm]; s.p_replica_index[:] = all_ridx[perm]
    s.p_replica_name_id[:] = all_rname[perm]
    s.h_pod_idx[:] = inv[head_pods_cm].astype(np.uint32)
    s.h_ready_status[:] = h_ready_status; s.h_ready_reason_id[:] = h_reason; s.h_ready_msg_id[:] = h_msg; s.h_pod_ip_id[:] = h_ip
    s.h_annot_state[:] = h_annot_state; s.h_version_state[:] = h_version_state; s.h_annot_hash[:] = h_annot_hash.ravel()

    # ---- clusters
    s.c_ns_id[:] = c_ns; s.c_name_id[:] = cname_ids
    s.c_uid_hash[:] = _splitmix64(gcid.astype(np.uint64))
    fl = np.full(Nc, abi.CF_HEAD_EXPECT_OK, dtype=np.uint32)
    fl[autoscaling] |= abi.CF_AUTOSCALING
    fl[recreate] |= abi.CF_UPGRADE_RECREATE
    if not p.healthy:
        fl[suspended_spec] |= abi.CF_SUSPEND
        fl[head_expect_pending] &= ~np.uint32(abi.CF_HEAD_EXPECT_OK)
        fl[skip] |= abi.CF_SKIP
        fl[u[:, 5] < 0.01] |= abi.CF_SKIP_HEAD_RESTART
        fl[u[:, 6] < 0.005] |= abi.CF_ENDPOINTS_CHANGED
    s.c_flags[:] = fl
    # suspended-spec clusters: one third still "none", one third Suspending, one third Suspended
    ss = np.zeros(Nc, dtype=np.uint8)
    if not p.healthy:
        third = rng.integers(0, 3, Nc)
        ss[suspended_spec & (third == 1)] = abi.SUSPEND_SUSPENDING
        ss[suspended_spec & (third == 2)] = abi.SUSPEND_SUSPENDED
    s.c_suspend_status[:] = ss
    s.c_group_off[:] = (cidx * G).astype(np.uint32); s.c_group_cnt[:] = G
    s.c_json_off[:] = c_json_off; s.c_json_len[:] = c_json_len; s.json[:] = json
    s.c_svc_count[:] = 1; s.c_svc_ip_kind[:] = abi.SVCIP_NORMAL; s.c_svc_ip_id[:] = svc_ip_ids; s.c_svc_name_id[:] = svc_name_ids
    if not p.healthy:
        s.c_svc_count[u[:, 7] < 0.002] = 0
        s.c_svc_ip_kind[(u[:, 7] > 0.002) & (u[:, 7] < 0.006)] = abi.SVCIP_NONE
    # old status: mostly what a converged cluster would already hold
    s.c_old_state[:] = abi.STATE_READY
    exp_desired = np.zeros(Nc, dtype=np.int64)
    np.add.at(exp_desired, g_cluster, np.clip(np.where((g_flags & abi.GF_REPLICAS_NIL) != 0, 1, g_replicas), 1, g_max) * hosts * ((g_flags & abi.GF_SUSPEND) == 0))
    avail = np.zeros(Nc, dtype=np.int64); rdy = np.zeros(Nc, dtype=np.int64)
    np.add.at(avail, pc, (~is_head) & (phase == abi.PHASE_RUNNING))
    np.add.at(rdy, pc, (~is_head) & (phase == abi.PHASE_RUNNING) & (ready == abi.COND_TRUE))
    oc = s.c_old_counts.reshape(Nc, 5)
    live = (g_flags & abi.GF_SUSPEND) == 0
    exp_min = np.zeros(Nc, dtype=np.int64); exp_max = np.zeros(Nc, dtype=np.int64)
    np.add.at(exp_min, g_cluster, g_min.astype(np.int64) * hosts * live)
    np.add.at(exp_max, g_cluster, g_max.astype(np.int64) * hosts * live)
    oc[:, 0] = rdy; oc[:, 1] = avail; oc[:, 2] = exp_desired; oc[:, 3] = exp_min
    oc[:, 4] = np.clip(exp_max, -(2 ** 31), 2 ** 31 - 1)
    stale = rng.random(Nc) > p.steady_frac
    oc[stale, 1] += 1
    ocs = s.c_old_cond_status.reshape(Nc, 5); ocv = s.c_old_cond_variant.reshape(Nc, 5)
    ocs[:, abi.COND_PROVISIONED] = abi.COND_TRUE; ocv[:, abi.COND_PROVISIONED] = abi.CV_PROV_ALL_READY
    fresh = rng.random(Nc) < 0.05
    ocs[fresh, abi.COND_PROVISIONED] = abi.COND_FALSE; ocv[fresh, abi.COND_PROVISIONED] = abi.CV_PROV_PROVISIONING
    ocs[:, abi.COND_HEAD_POD_READY] = h_ready_status; ocv[:, abi.COND_HEAD_POD_READY] = abi.CV_HEAD_FROM_POD
    s.c_old_cond_reason_id[:] = h_reason
    s.c_old_cond_msg_id.reshape(Nc, 2)[:, 0] = h_msg
    ocs[:, abi.COND_SUSPENDING] = np.where(ss == abi.SUSPEND_SUSPENDING, abi.COND_TRUE, abi.COND_FALSE); ocv[:, abi.COND_SUSPENDING] = abi.CV_CANONICAL
    ocs[:, abi.COND_SUSPENDED] = np.where(ss == abi.SUSPEND_SUSPENDED, abi.COND_TRUE, abi.COND_FALSE); ocv[:, abi.COND_SUSPENDED] = abi.CV_CANONICAL
    oh = s.c_old_head_ids.reshape(Nc, 4)
    oh[:, 0] = h_ip; oh[:, 1] = svc_ip_ids; oh[:, 2] = p_name[head_pods_cm]; oh[:, 3] = svc_name_ids
    s.c_summary_id[:] = (summary_base + cidx).astype(np.uint32)

    # ---- groups
    s.g_cluster_idx[:] = g_cluster.astype(np.uint32); s.g_name_id[:] = group_ids[g_local]
    s.g_replicas[:] = g_replicas.astype(np.int32); s.g_min[:] = g_min; s.g_max[:] = g_max.astype(np.int32); s.g_num_hosts[:] = hosts
    s.g_flags[:] = g_flags; s.g_wtd_off[:] = g_wtd_off; s.g_wtd_cnt[:] = wtd_cnt
    s.w_name_id[:] = w_name

    # ---- RayJobs (config C4): 1:1 with clusters, 5 % with a changed roll-up
    if p.jobs:
        s.j_ns_id[:] = c_ns; s.j_cluster_name_id[:] = cname_ids
        jid = (summary_base + cidx).astype(np.uint32)
        changed = rng.random(Nc) < 0.05
        jid[changed] = (summary_base + Nc + cidx[changed]).astype(np.uint32)
        s.j_summary_id[:] = jid
        missing = rng.random(Nc) < 0.002
        s.j_cluster_name_id[missing] = ghost_cluster_id

    flags = abi.default_flags(id_head_not_found_reason=ID_HEAD_NOT_FOUND_REASON, id_head_not_found_msg=ID_HEAD_NOT_FOUND_MSG)
    if p.n_large:
        grow_clusters(s, np.linspace(0, Nc - 1, p.n_large).astype(np.int64), p.large_pods)
    if p.n_wide:
        s = widen_clusters(s, np.linspace(0, Nc - 1, p.n_wide).astype(np.int64), p.wide_groups)
    return s.validate(), flags


def grow_clusters(snap: Snapshot, clusters, size: int) -> None:
    """Move worker pods of the other RayClusters (first rows first) into worker group 0 of each of `clusters` until it lists
    `size` pods; the pod rows and every other table keep their shape."""
    taken = np.zeros(snap.dims["clusters"], dtype=bool)
    taken[np.asarray(clusters)] = True
    ckey = (snap.c_ns_id.astype(np.uint64) << np.uint64(32)) | snap.c_name_id.astype(np.uint64)
    order = np.argsort(ckey)
    pkey = (snap.p_ns_id.astype(np.uint64) << np.uint64(32)) | snap.p_cluster_name_id.astype(np.uint64)
    pos = np.minimum(np.searchsorted(ckey[order], pkey), order.size - 1)
    owner = np.where(ckey[order][pos] == pkey, order[pos], -1)
    worker = ((snap.p_packed >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER
    donors = np.flatnonzero(worker & (owner >= 0) & ~taken[np.maximum(owner, 0)])
    at = 0
    for c in clusters:
        need = size - int((owner == c).sum())
        if need <= 0:
            continue
        if at + need > donors.size:
            raise ValueError("not enough worker pods to grow the RayClusters")
        move = donors[at:at + need]
        at += need
        g0 = int(snap.c_group_off[c])
        snap.p_ns_id[move], snap.p_cluster_name_id[move], snap.p_group_name_id[move] = snap.c_ns_id[c], snap.c_name_id[c], snap.g_name_id[g0]


def grow_epochs(snap: Snapshot, clusters, sizes):
    """Scale `clusters` up over several epochs, as an autoscaler does: for each size in `sizes`, grow_clusters(snap, clusters, size)
    and yield the pod rows that changed (the Pods that joined)."""
    for size in sizes:
        before = (snap.p_ns_id.copy(), snap.p_cluster_name_id.copy())
        grow_clusters(snap, clusters, size)
        yield np.flatnonzero((snap.p_ns_id != before[0]) | (snap.p_cluster_name_id != before[1]))


_ID_COLUMNS = ("c_ns_id", "c_name_id", "c_ext_err_msg_id", "c_old_cond_reason_id", "c_old_cond_msg_id", "c_old_head_ids", "c_svc_ip_id",
               "c_svc_name_id", "c_summary_id", "g_name_id", "w_name_id", "p_ns_id", "p_cluster_name_id", "p_group_name_id", "p_name_id",
               "p_replica_name_id", "h_ready_reason_id", "h_ready_msg_id", "h_pod_ip_id", "j_ns_id", "j_cluster_name_id", "j_summary_id")


def widen_clusters(snap: Snapshot, clusters, n_groups: int) -> Snapshot:
    """A copy of `snap` in which worker group 0 of each of `clusters` is split into `n_groups` worker groups: the group row is copied
    under new names (its workersToDelete names stay with group 0), its worker pods are relabelled round-robin in row order and its
    replicas and minReplicas are split.  Every other row keeps its values; the group table (offsets, workersToDelete offsets) is
    rebuilt around the new rows."""
    d = snap.dims
    Nc = d["clusters"]
    clusters = np.unique(np.asarray(clusters, dtype=np.int64))
    assert n_groups >= 1 and (snap.c_group_cnt[clusters] >= 1).all()
    gcnt = snap.c_group_cnt.astype(np.int64)
    gcnt[clusters] += n_groups - 1
    # source row of every new group: group 0 of a widened cluster n_groups times, every other group once
    reps = np.ones(d["groups"], dtype=np.int64)
    reps[snap.c_group_off[clusters].astype(np.int64)] += n_groups - 1
    src = np.repeat(np.arange(d["groups"]), reps)
    out = Snapshot(Nc, int(gcnt.sum()), d["wtd"], d["pods"], d["heads"], d["jobs"], d["json"])
    for name, _dt, mult, dim in abi.COLUMNS:
        if dim == "groups":
            out.cols[name][:] = snap.cols[name][src]
        else:
            out.cols[name][:] = snap.cols[name]
    new_off = np.concatenate([[0], np.cumsum(gcnt)[:-1]]).astype(np.int64)
    out.c_group_off[:] = new_off.astype(np.uint32)
    out.c_group_cnt[:] = gcnt.astype(np.uint32)
    out.g_cluster_idx[:] = np.repeat(np.arange(Nc), gcnt).astype(np.uint32)
    next_id = max(int(snap.cols[c].max()) for c in _ID_COLUMNS if snap.cols[c].size) + 1
    worker = ((snap.p_packed >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER
    for c in clusters:
        g_old, g_new = int(snap.c_group_off[c]), int(new_off[c])
        rows = np.arange(g_new, g_new + n_groups)
        out.g_name_id[rows[1:]] = np.arange(next_id, next_id + n_groups - 1, dtype=np.uint32)
        next_id += n_groups - 1
        out.g_wtd_cnt[rows[1:]] = 0
        for col in ("g_replicas", "g_min"):
            v = int(snap.cols[col][g_old])
            out.cols[col][rows] = [v // n_groups + (k < v % n_groups) for k in range(n_groups)]
        members = np.flatnonzero(worker & (snap.p_ns_id == snap.c_ns_id[c]) & (snap.p_cluster_name_id == snap.c_name_id[c])
                                 & (snap.p_group_name_id == snap.g_name_id[g_old]))
        out.p_group_name_id[members] = out.g_name_id[rows[np.arange(members.size) % n_groups]]
    out.g_wtd_off[:] = np.concatenate([[0], np.cumsum(out.g_wtd_cnt)[:-1]]).astype(np.uint32) if out.dims["groups"] else 0
    return out.validate()


def first_clusters(snap: Snapshot, k: int, free_from: int | None = None, jobs=None, free_pods: bool = True) -> Snapshot:
    """The snapshot before RayClusters k.. of `snap` were created: its first k RayClusters with their groups and workersToDelete names
    (the rows a creation appends come after all of these), every pod row, head-aux row and the JSON arena.  With `free_pods` the Pods
    labelled for the RayClusters from row `free_from` (default k) on are free rows (KR_PP_TOMBSTONE, every id 0); without it they
    stay, as orphans.  `jobs`: the RayJob rows kept (default all)."""
    d = snap.dims
    g = int(snap.c_group_off[k]) if k < d["clusters"] else d["groups"]
    w = int(snap.g_wtd_off[g]) if g < d["groups"] else d["wtd"]
    jobs = np.arange(d["jobs"]) if jobs is None else np.asarray(jobs, dtype=np.int64)
    out = Snapshot(k, g, w, d["pods"], d["heads"], jobs.size, d["json"])
    rows = {"clusters": np.arange(k), "groups": np.arange(g), "wtd": np.arange(w), "jobs": jobs}
    for name, _dt, mult, dim in abi.COLUMNS:
        src = snap.cols[name]
        out.cols[name][:] = (src.reshape(-1, mult)[rows[dim]].reshape(-1) if mult > 1 else src[rows[dim]]) if dim in rows else src
    if free_pods:
        f0 = k if free_from is None else free_from
        ckey = (snap.c_ns_id[f0:].astype(np.uint64) << np.uint64(32)) | snap.c_name_id[f0:].astype(np.uint64)
        pkey = (snap.p_ns_id.astype(np.uint64) << np.uint64(32)) | snap.p_cluster_name_id.astype(np.uint64)
        gone = np.flatnonzero(np.isin(pkey, ckey) & (snap.p_cluster_name_id != 0))
        for name, _dt, _m, dim in abi.COLUMNS:
            if dim == "pods":
                out.cols[name][gone] = 0
        out.p_packed[gone] = np.uint32(abi.PP_TOMBSTONE)
    return out.validate()


def swap_remove_order(n: int, rows) -> np.ndarray:
    """The old row of each new row after deleting the RayClusters at (old) rows `rows` one by one by swap-remove, as the native
    packer does: the last RayCluster moves into each hole."""
    order = list(range(n))
    where = {c: c for c in order}
    for r in rows:
        pos = where.pop(int(r))
        last = order.pop()
        if last != int(r):
            order[pos] = last
            where[last] = pos
    return np.asarray(order, dtype=np.int64)


def select_clusters(snap: Snapshot, order) -> Snapshot:
    """The RayClusters at old rows `order`, in that row order, with their groups and workersToDelete names laid out again in row
    order; every pod row, head-aux row, RayJob row and the JSON arena stay as they are."""
    order = np.asarray(order, dtype=np.int64)
    d = snap.dims
    goff, gcnt = snap.c_group_off.astype(np.int64), snap.c_group_cnt.astype(np.int64)
    groups = np.concatenate([np.arange(goff[c], goff[c] + gcnt[c]) for c in order] + [np.zeros(0, np.int64)])
    names = np.concatenate([np.arange(int(snap.g_wtd_off[g]), int(snap.g_wtd_off[g] + snap.g_wtd_cnt[g])) for g in groups] + [np.zeros(0, np.int64)])
    out = Snapshot(order.size, groups.size, names.size, d["pods"], d["heads"], d["jobs"], d["json"])
    rows = {"clusters": order, "groups": groups, "wtd": names}
    for name, _dt, mult, dim in abi.COLUMNS:
        src = snap.cols[name]
        out.cols[name][:] = (src.reshape(-1, mult)[rows[dim]].reshape(-1) if mult > 1 else src[rows[dim]]) if dim in rows else src
    cnt = gcnt[order]
    out.c_group_off[:] = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.uint32) if order.size else 0
    out.g_cluster_idx[:] = np.repeat(np.arange(order.size), cnt).astype(np.uint32)
    out.g_wtd_off[:] = np.concatenate([[0], np.cumsum(out.g_wtd_cnt)[:-1]]).astype(np.uint32) if groups.size else 0
    return out.validate()


def delete_clusters(snap: Snapshot, rows) -> Snapshot:
    """The snapshot after the RayClusters at rows `rows` were deleted by swap-remove (swap_remove_order), with groups and names laid
    out again in row order.  Their Pods stay, as orphans (until garbage collection removes them)."""
    return select_clusters(snap, swap_remove_order(snap.dims["clusters"], rows))


def regroup_clusters(snap: Snapshot, edits) -> Snapshot:
    """A copy of `snap` in which each RayCluster c of `edits` has the worker groups edits[c]: a list of (source group row, name id)
    pairs, each group a copy of its source row (its workersToDelete names included) under that name (None: the source's own).
    Pod rows, head-aux rows, RayJob rows and the JSON arena stay; groups and names are laid out again in row order."""
    d = snap.dims
    goff, gcnt = snap.c_group_off.astype(np.int64), snap.c_group_cnt.astype(np.int64)
    src, names, owner = [], [], []
    for c in range(d["clusters"]):
        pairs = edits.get(c, [(g, None) for g in range(goff[c], goff[c] + gcnt[c])])
        for g, nm in pairs:
            src.append(int(g)); names.append(int(snap.g_name_id[g]) if nm is None else int(nm)); owner.append(c)
    src = np.asarray(src, dtype=np.int64)
    wsrc = np.concatenate([np.arange(int(snap.g_wtd_off[g]), int(snap.g_wtd_off[g] + snap.g_wtd_cnt[g])) for g in src] + [np.zeros(0, np.int64)])
    out = Snapshot(d["clusters"], src.size, wsrc.size, d["pods"], d["heads"], d["jobs"], d["json"])
    rows = {"groups": src, "wtd": wsrc}
    for name, _dt, _m, dim in abi.COLUMNS:
        out.cols[name][:] = snap.cols[name][rows[dim]] if dim in rows else snap.cols[name]
    out.g_name_id[:] = np.asarray(names, dtype=np.uint32)
    out.g_cluster_idx[:] = np.asarray(owner, dtype=np.uint32)
    cnt = np.bincount(np.asarray(owner, dtype=np.int64), minlength=d["clusters"])
    out.c_group_cnt[:] = cnt.astype(np.uint32)
    out.c_group_off[:] = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.uint32) if d["clusters"] else 0
    out.g_wtd_off[:] = np.concatenate([[0], np.cumsum(out.g_wtd_cnt)[:-1]]).astype(np.uint32) if src.size else 0
    return out.validate()


def config(name: str, **overrides) -> SynthParams:
    d = dict(CONFIGS[name])
    d.update(overrides)
    return SynthParams(**d)


def shard_by_uid(snap: Snapshot, rank: int, world: int) -> Snapshot:
    """UID-hash sharding (SURVEY §8(e)): keep clusters with uid_hash64 % world == rank, route every pod to its cluster's
    shard through the (ns_id, cluster_name_id) -> cluster table; orphans go to hash(ns, name) % world."""
    if world == 1:
        return snap
    d = snap.dims
    keep_c = (snap.c_uid_hash % np.uint64(world)) == np.uint64(rank)
    new_c = np.cumsum(keep_c) - 1
    ckey = (snap.c_ns_id.astype(np.uint64) << np.uint64(32)) | snap.c_name_id.astype(np.uint64)
    order = np.argsort(ckey)
    pkey = (snap.p_ns_id.astype(np.uint64) << np.uint64(32)) | snap.p_cluster_name_id.astype(np.uint64)
    pos = np.searchsorted(ckey[order], pkey)
    pos_c = np.minimum(pos, max(d["clusters"] - 1, 0))
    found = (d["clusters"] > 0) & (ckey[order][pos_c] == pkey)
    owner = np.where(found, snap.c_uid_hash[order][pos_c] % np.uint64(world), _splitmix64(pkey) % np.uint64(world))
    keep_p = owner == np.uint64(rank)
    new_p = np.cumsum(keep_p) - 1
    keep_g = keep_c[snap.g_cluster_idx] if d["groups"] else np.zeros(0, bool)
    keep_w = np.repeat(keep_g, snap.g_wtd_cnt) if d["groups"] else np.zeros(0, bool)
    keep_h = keep_p[snap.h_pod_idx] if d["heads"] else np.zeros(0, bool)
    keep_j = np.ones(d["jobs"], bool)
    if d["jobs"]:
        jkey = (snap.j_ns_id.astype(np.uint64) << np.uint64(32)) | snap.j_cluster_name_id.astype(np.uint64)
        jpos = np.minimum(np.searchsorted(ckey[order], jkey), max(d["clusters"] - 1, 0))
        jfound = ckey[order][jpos] == jkey
        jowner = np.where(jfound, snap.c_uid_hash[order][jpos] % np.uint64(world), _splitmix64(jkey) % np.uint64(world))
        keep_j = jowner == np.uint64(rank)
    # json arena is re-packed
    lens = snap.c_json_len[keep_c].astype(np.int64)
    padded = (lens + 15) & ~15
    out = Snapshot(int(keep_c.sum()), int(keep_g.sum()), int(keep_w.sum()), int(keep_p.sum()), int(keep_h.sum()), int(keep_j.sum()), int(padded.sum()))
    masks = {"clusters": keep_c, "groups": keep_g, "wtd": keep_w, "pods": keep_p, "heads": keep_h, "jobs": keep_j}
    for name, _dt, mult, dim in abi.COLUMNS:
        if dim == "json":
            continue
        src = snap.cols[name].reshape(d[dim], mult) if d[dim] else snap.cols[name].reshape(0, mult)
        out.cols[name][:] = src[masks[dim]].ravel()
    out.g_cluster_idx[:] = new_c[snap.g_cluster_idx[keep_g]].astype(np.uint32) if d["groups"] else 0
    gcnt = snap.c_group_cnt[keep_c]
    out.c_group_off[:] = np.concatenate([[0], np.cumsum(gcnt)[:-1]]).astype(np.uint32) if gcnt.size else 0
    out.g_wtd_off[:] = np.concatenate([[0], np.cumsum(out.g_wtd_cnt)[:-1]]).astype(np.uint32) if out.dims["groups"] else 0
    out.h_pod_idx[:] = new_p[snap.h_pod_idx[keep_h]].astype(np.uint32) if d["heads"] else 0
    off = np.concatenate([[0], np.cumsum(padded)[:-1]]).astype(np.int64) if padded.size else np.zeros(0, np.int64)
    out.c_json_off[:] = off.astype(np.uint64)
    src_off = snap.c_json_off[keep_c].astype(np.int64)
    for i in range(lens.size):
        out.json[off[i]:off[i] + lens[i]] = snap.json[src_off[i]:src_off[i] + lens[i]]
    return out.validate()

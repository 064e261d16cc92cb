"""Every GPU pipeline against the object-level Go model (tests/go_model.py): the closed-loop rounds of test_go_model.py with
RayClusterReconciler over the CUDA engine.  One Engine per arm lives across all rounds and seeds: each pass begins, fills and
commits a snapshot of whatever shape the client has grown or shrunk to."""
import numpy as np
import pytest

import fuzz_objects
import go_model as gm
from kuberay_b200 import abi
from kuberay_b200.engine import Engine
from test_go_model import decorate, inputs, run_stream, wrapped_desired_stream

pytestmark = pytest.mark.gpu

SEEDS = range(60)


class EngineArm:
    """A backend for RayClusterReconciler: one engine, sized once with room to grow, one full pass per call."""

    def __init__(self, fetch_pod_lists=0, profile=False, **options):
        self.fetch, self.profile, self.options = fetch_pod_lists, profile, options
        self.eng = None
        self.kernels, self.passes, self.saw_sorted, self.strides = set(), 0, False, set()

    def run(self, snap, flags):
        d = snap.dims
        if self.eng is None:
            self.eng = Engine(0, max_clusters=4 * d["clusters"] + 64, max_groups=4 * d["groups"] + 256, max_wtd=4 * d["wtd"] + 256,
                              max_pods=4 * d["pods"] + 8192, max_heads=4 * d["heads"] + 256, max_jobs=4 * d["jobs"] + 64,
                              max_creates=8 * d["pods"] + 65536, max_json_bytes=4 * d["json"] + 65536)
            for k, v in self.options.items():
                getattr(self.eng, f"set_{k}")(v)
        views = self.eng.begin(snap.sizes())
        self.eng.fill(views, snap)
        self.eng.commit()
        f = abi.kr_flags.from_buffer_copy(flags)
        f.fetch_pod_lists = self.fetch
        if self.profile:
            self.kernels |= {k for k, _ in self.eng.reconcile_profiled(f)["kernels"]}
        res = self.eng.reconcile(f)
        self.passes += 1
        self.saw_sorted |= res.sorted_pod_idx.size > 0
        self.strides.add(self.eng.get_option(abi.OPT_BUCKET_STRIDE))
        return res

    def close(self):
        if self.eng is not None:
            self.eng.close()


def _streams(arm, seeds=SEEDS, **kw):
    stats = {}
    try:
        for seed in seeds:
            clusters, pods, jobs, env, rng = inputs(seed)
            run_stream(seed, arm, clusters, pods, jobs, env, rng, stats=stats, **kw)
    finally:
        arm.close()
    for k in ("deleted", "created", "written", "errors"):
        assert stats[k] > 0, stats
    return stats


def test_bucket_pipeline_against_the_model():
    arm = EngineArm(fetch_pod_lists=0)
    stats = _streams(arm)
    assert stats["warnings"] > 0 and any(s > 0 for s in arm.strides), (stats, arm.strides)


def test_sort_pipeline_against_the_model():
    arm = EngineArm(fetch_pod_lists=1)
    _streams(arm)
    assert arm.saw_sorted


def test_radix_unfused_pipeline_against_the_model(monkeypatch):
    monkeypatch.setenv("KR_FORCE_RADIX", "1")
    monkeypatch.setenv("KR_NO_FUSE", "1")
    arm = EngineArm(fetch_pod_lists=1, profile=True)
    _streams(arm, seeds=range(30))
    assert "k_scatter" in arm.kernels and "k_place_fused" not in arm.kernels, sorted(arm.kernels)


def big_clusters(seed, n_large, n_huge, n_wide_groups=40):
    """Three RayClusters beside a fuzz fleet: one of n_large Pods, one of n_wide_groups worker groups and one of n_huge Pods.
    Each mixes a head (two for some seeds), unhealthy Pods, workersToDelete names, unparsable replica indices and replicas a
    little above or below what is there, spread so the unhealthy Pods and victims fall at the warp-range edges of the block
    decide (multiples of 32 and their neighbours)."""
    rng = np.random.default_rng(seed)
    clusters, pods = [], []
    for cname, n_pods, n_groups in (("large", n_large, 2), ("wide", 4 * n_wide_groups, n_wide_groups), ("huge", n_huge, 3)):
        groups = [{"groupName": f"g{gi}", "replicas": None, "minReplicas": 0, "maxReplicas": 2 ** 31 - 1, "numOfHosts": 1}
                  for gi in range(n_groups)]
        c = {"namespace": "big", "name": cname, "uid": f"uid-big-{cname}", "specJson": f'{{"big":"{cname}"}}',
             "spec": {"enableInTreeAutoscaling": bool(rng.random() < 0.3), "workerGroupSpecs": groups}, "status": {},
             "headService": {"count": 1, "clusterIP": "10.0.0.3", "name": f"{cname}-head-svc"}}
        n_heads = 2 if rng.random() < 0.2 else 1
        for h in range(n_heads):
            pods.append({"namespace": "big", "name": f"{cname}-head-{h}", "labels": {gm.CLUSTER_LABEL: cname, gm.NODE_TYPE_LABEL: "head"},
                         "phase": "Running", "restartPolicy": "Always", "conditions": [{"type": "Ready", "status": "True"}], "podIP": "10.3.0.1"})
        per = [0] * n_groups
        for i in range(n_pods - n_heads):
            gi = i % n_groups
            edge = i % 32 in (0, 31) or i % 256 in (255, 0)
            phase = "Failed" if edge and rng.random() < 0.05 else ("Running" if rng.random() < 0.9 else "Pending")
            p = {"namespace": "big", "name": f"{cname}-w{i:05d}", "labels": {gm.CLUSTER_LABEL: cname, gm.NODE_TYPE_LABEL: "worker",
                                                                             gm.GROUP_LABEL: f"g{gi}"},
                 "phase": phase, "restartPolicy": "Always", "conditions": [{"type": "Ready", "status": "True"}]}
            if rng.random() < 0.9:
                p["labels"][gm.REPLICA_INDEX_LABEL] = str(per[gi]) if rng.random() < 0.95 else "x"
            per[gi] += 1
            pods.append(p)
        for gi, g in enumerate(groups):
            g["replicas"] = max(0, per[gi] + int(rng.integers(-3, 4)))
            if rng.random() < 0.6:
                g["workersToDelete"] = [f"{cname}-w{int(rng.integers(0, n_pods)):05d}" for _ in range(int(rng.integers(1, 5)))]
        clusters.append(c)
    return clusters, pods


def fleet(seeds, max_clusters):
    """Decorated fuzz fleets of `seeds` in disjoint namespaces.  -> (clusters, pods, jobs, Env of the last seed)"""
    clusters, pods, jobs = [], [], []
    for seed in seeds:
        c, p, j = fuzz_objects.generate(seed, max_clusters=max_clusters)
        c, p, j, env, _rng = decorate(c, p, j, seed)
        for obj in c + p + j:
            obj["namespace"] = f"s{seed}-{obj.get('namespace', 'default')}"
        for obj in c:
            obj["uid"] = f"{obj['namespace']}/{obj['name']}"
        clusters += c
        pods += p
        jobs += j
    return clusters, pods, jobs, env


@pytest.mark.parametrize("seed", [0, 1])
def test_large_wide_huge_clusters_against_the_model(seed):
    """The three big RayClusters in a fleet of a couple of hundred fuzz ones (so the mean size fits a bucket stride)."""
    clusters, pods, jobs, env = fleet(range(100 + 20 * seed, 112 + 20 * seed), max_clusters=20)
    clusters += (big := big_clusters(seed, n_large=int(np.random.default_rng(seed).integers(300, 1201)), n_huge=9000))[0]
    pods += big[1]
    rng = np.random.default_rng(100 + seed)
    arm = EngineArm(fetch_pod_lists=0, profile=True, large_clusters=True, wide_clusters=True, huge_clusters=True)
    stats = {}
    try:
        run_stream(100 + seed, arm, clusters, pods, jobs, env, rng, rounds=3, stats=stats)
    finally:
        arm.close()
    assert {"k_match2", "k_decide_large", "k_decide_huge", "k_huge_merge"} <= arm.kernels, sorted(arm.kernels)
    # every pass stayed on the bucket pipeline: without wide_clusters the 40-group RayCluster sends the pass to the sort one (stride 0)
    assert 0 not in arm.strides, arm.strides
    for k in ("deleted", "created", "written"):
        assert stats[k] > 0, stats


def test_merged_fleet_against_the_model():
    """A few hundred fuzz seeds in disjoint namespaces: one pass decides thousands of RayClusters on a multi-CTA grid."""
    clusters, pods, jobs, env = fleet(range(300), max_clusters=20)
    arm = EngineArm(fetch_pod_lists=0)
    stats = {}
    try:
        run_stream(7, arm, clusters, pods, jobs, env, np.random.default_rng(7), rounds=3, failures=False, stats=stats)
    finally:
        arm.close()
    assert stats["clusters"] >= 2000, stats
    for k in ("deleted", "created", "written"):
        assert stats[k] > 0, stats


@pytest.mark.parametrize("fetch", [0, 1], ids=["bucket", "sort"])
@pytest.mark.parametrize("autoscaling", [False, True])
def test_wrapped_desired_replicas_scale_down_not_up(autoscaling, fetch):
    """The decide takes diff in Go int: a desired count that wrapped to -2^31 is a scale-down, never 2^31 creates."""
    arm = EngineArm(fetch_pod_lists=fetch)
    try:
        stats = wrapped_desired_stream(arm, autoscaling)
    finally:
        arm.close()
    assert stats["created"] == 0 and stats["deleted"] == (0 if autoscaling else 3), stats

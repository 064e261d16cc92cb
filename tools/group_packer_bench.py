"""The group packer (kr_group_packer_*) against the global-snapshot coordinator (kr_group_route + commit + reconcile) on the same
fleets: C5 (1 000 autoscaling RayClusters x 100 Pods) and C3 (10 000 RayClusters x 100 Pods), split into n = 1, 2 and 4 shards on
the visible devices (device 0 repeated when there is only one: the shards then share one GPU, so the figures measure coordination
overhead, not scaling — each line says which).

Every epoch flips the status of 1 % of the Pods (events handled before the timed window, as the shim's informer handlers do), then
times kr_group_packer_flush + kr_group_packer_reconcile (host clock; every shard's pass ends in its synchronising results fetch).
Reported per (fleet, n): median / min / max epoch ms, the sum and the maximum over the shards of kr_profile.h2d_bytes (median over
epochs), the share of shard passes that were incremental, and beside them one epoch (after a warm-up) of kr_group_route +
kr_group_commit + kr_group_reconcile over a global snapshot of the same objects.  The card name and power limit are read in the
same run.
Usage: python tools/group_packer_bench.py [--fleets C5,C3] [--shards 1,2,4] [--epochs 10] [--out DIR]"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from benchlib import Recorder  # noqa: E402
from kuberay_b200 import abi, snapshot as snp  # noqa: E402
from kuberay_b200.engine import Group, lib  # noqa: E402
from kuberay_b200.packer import GroupPacker  # noqa: E402

FLEETS = {"C5": dict(clusters=1000, pods=100, autoscaling=True), "C3": dict(clusters=10_000, pods=100, autoscaling=False)}


def cluster(c: int, autoscaling: bool, pods: int) -> dict:
    spec = {"workerGroupSpecs": [{"groupName": "workers", "replicas": pods - 1, "minReplicas": 0, "maxReplicas": 2 * pods}]}
    if autoscaling:
        spec["enableInTreeAutoscaling"] = True
    return {"namespace": f"ns{c % 50}", "name": f"rc-{c}", "uid": f"uid-{c}", "generation": 1, "resourceVersion": 1, "spec": spec,
            "status": {}, "expectations": {"head": True, "workers": True}}


def pod(c: int, i: int, running: bool) -> dict:
    head = i == 0
    labels = {snp.RAY_CLUSTER_LABEL: f"rc-{c}", snp.RAY_NODE_TYPE_LABEL: "head" if head else "worker"}
    labels[snp.RAY_NODE_GROUP_LABEL] = "headgroup" if head else "workers"
    return {"namespace": f"ns{c % 50}", "name": f"rc-{c}-{i}", "labels": labels, "phase": "Running" if running else "Pending",
            "conditions": [{"type": "Ready", "status": "True" if running else "False"}], "podIP": f"10.{c // 250}.{c % 250}.{i}" if head else None,
            "restartPolicy": "Always"}


def caps(nc: int, p: int, n: int) -> dict:
    """Per-shard capacities with room for an uneven split."""
    per = nc // n + nc // (4 * n) + 64
    return dict(max_clusters=per, max_groups=per, max_wtd=64, max_pods=per * p, max_heads=per, max_jobs=16,
                max_creates=max(1 << 16, per * p // 4), max_json_bytes=per * 1024)


def run(name: str, fleet: dict, n: int, devices: list[int], epochs: int, rng) -> dict:
    nc, p = fleet["clusters"], fleet["pods"]
    gp = GroupPacker(devices, **caps(nc, p, n))
    try:
        t = time.perf_counter()
        for c in range(nc):
            gp.upsert_cluster(cluster(c, fleet["autoscaling"], p))
        for c in range(nc):
            for i in range(p):
                gp.upsert_pod(pod(c, i, True))
        running = np.ones((nc, p), dtype=bool)
        gp.flush()
        flags = gp.flags(fetch_pod_lists=0)
        gp.reconcile(flags, copy=False)
        load_s = time.perf_counter() - t
        touch = max(1, nc * p // 100)

        def epoch():
            cs, ps = rng.integers(0, nc, touch), rng.integers(1, p, touch)
            for c, i in zip(cs.tolist(), ps.tolist()):
                running[c, i] = not running[c, i]
                gp.upsert_pod(pod(c, i, bool(running[c, i])))
            t0 = time.perf_counter()
            gp.flush()
            t1 = time.perf_counter()
            res = gp.reconcile(flags, copy=False)
            t2 = time.perf_counter()
            h2d = [sh.engine.last_profile()["h2d_bytes"] for sh in gp.shards]
            return (t2 - t0) * 1e3, (t1 - t0) * 1e3, (t2 - t1) * 1e3, sum(h2d), max(h2d), sum(r.changed_clusters is not None for r in res)

        epoch()  # warm-up
        rec = np.array([epoch() for _ in range(epochs)], dtype=np.float64)
        sizes = [int(sh.engine.sizes.n_clusters) for sh in gp.shards]
        objects = ([cluster(c, fleet["autoscaling"], p) for c in range(nc)], [pod(c, i, bool(running[c, i])) for c in range(nc) for i in range(p)])
    finally:
        gp.close()
    out = {"fleet": name, "clusters": nc, "pods": nc * p, "shards": n, "devices": devices,
           "note": "shards share one GPU: coordination overhead, not scaling" if len(set(devices)) < n else "one shard per GPU",
           "clusters_per_shard": sizes, "pod_events_per_epoch": touch, "epochs": epochs, "load_s": round(load_s, 1),
           "epoch_ms_median": round(float(np.median(rec[:, 0])), 4), "epoch_ms_min": round(float(rec[:, 0].min()), 4),
           "epoch_ms_max": round(float(rec[:, 0].max()), 4), "flush_ms_median": round(float(np.median(rec[:, 1])), 4),
           "reconcile_ms_median": round(float(np.median(rec[:, 2])), 4), "h2d_bytes_sum_median": int(np.median(rec[:, 3])),
           "h2d_bytes_max_shard_median": int(np.median(rec[:, 4])), "incremental_share": round(float(rec[:, 5].sum()) / (epochs * n), 4)}
    out.update(global_epoch(objects, n, devices))
    return out


def global_epoch(objects, n: int, devices: list[int]) -> dict:
    """kr_group_route + kr_group_commit + kr_group_reconcile of a global snapshot of the same objects (a warm-up, then one timed)."""
    snap, meta = snp.pack_objects(objects[0], objects[1], [])
    flags = meta.flags
    flags.fetch_pod_lists = 0
    d = snap.dims
    cap = abi.kr_config(0, d["clusters"] + 1, d["groups"] + 1, d["wtd"] + 1, d["pods"] + 1, d["heads"] + 1, d["jobs"] + 1, max(1 << 16, d["pods"] // 4), d["json"] + 64)
    grp = Group(cap, devices)
    try:
        for _ in range(2):
            t0 = time.perf_counter()
            grp.route(snap)
            t1 = time.perf_counter()
            grp.commit()
            res = grp.reconcile(flags, copy=False)
            t2 = time.perf_counter()
        h2d = [e.last_profile()["h2d_bytes"] for e in grp.engines]
    finally:
        grp.close()
    return {"global_route_commit_reconcile_ms": round((t2 - t0) * 1e3, 4), "global_route_ms": round((t1 - t0) * 1e3, 4),
            "global_h2d_bytes_sum": int(sum(h2d)), "global_incremental_share": round(sum(r.changed_clusters is not None for r in res) / n, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fleets", default="C5,C3")
    ap.add_argument("--shards", default="1,2,4")
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ndev = lib().kr_device_count()
    out = Recorder("group_packer_bench", a.out, visible_devices=ndev)
    rng = np.random.default_rng(1)
    for name in a.fleets.split(","):
        for n in [int(x) for x in a.shards.split(",")]:
            out.record(run(name, FLEETS[name], n, [i % ndev for i in range(n)], a.epochs, rng))
    out.finish()


if __name__ == "__main__":
    main()

"""KR_OPT_HUGE_GROWTH on one GPU: epochs that grow RayClusters past 8 192 Pods, with the option off and on, alternated (one JSON line
per run).

Workload: C3H (10 000 RayClusters x 100 Pods, 2 of them grown to 20 000 Pods) with one more RayCluster grown to 8 000 Pods, on an
engine with KR_OPT_LARGE_CLUSTERS, _HUGE_CLUSTERS and _LARGE_GROWTH (slack 1.25).  Each run is a fresh engine: two full passes,
then one epoch of one variant, committed as Pod values:
  * "crossing": the 8 000-Pod RayCluster scales to 8 300 Pods (past KR_LARGE_MAX_PODS: it becomes huge);
  * "huge regrowth": a 20 000-Pod RayCluster scales past its region (25 024 ranks) to 25 100 Pods;
  * "churn": PodReady flips on 1 000 Pods, nothing grows (with the option the incremental pass also launches k_huge_tiles and
    k_huge_merge over the empty reserve entries).
Reported per run: whether the epoch was incremental, its kernel ms (device events), its wall ms through the C ABI (host clock around
the commit and kr_reconcile_batch, results copy included), H2D and D2H bytes (kr_profile).  Then, option on, the "huge regrowth" epoch
once more, profiled, for the k_inc_grow time.  The card's name, power limit and clocks are read in the same run.
Usage: python tools/huge_growth_bench.py [--runs 3] [--out DIR]"""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kuberay_b200 import abi, synthetic  # noqa: E402
from kuberay_b200.engine import Engine  # noqa: E402

POD_COLS = [name for name, _dt, _m, dim in abi.COLUMNS if dim == "pods"]
CROSS = 5000  # the RayCluster grown to 8 000 Pods


def huge_rows(snap):
    cnt = np.bincount(owner(snap), minlength=snap.dims["clusters"] + 1)[:-1]
    return [int(c) for c in np.flatnonzero(cnt > 10000)]


def owner(snap):
    ckey = (snap.c_ns_id.astype(np.uint64) << np.uint64(32)) | snap.c_name_id.astype(np.uint64)
    pkey = (snap.p_ns_id.astype(np.uint64) << np.uint64(32)) | snap.p_cluster_name_id.astype(np.uint64)
    order = np.argsort(ckey)
    pos = np.minimum(np.searchsorted(ckey[order], pkey), order.size - 1)
    return np.where(ckey[order][pos] == pkey, order[pos], snap.dims["clusters"])


def grow(snap, c, size):
    """Worker Pods of the ordinary RayClusters (last rows first) move into RayCluster c's worker group 0 until it lists `size`
    Pods.  -> the pod rows that moved."""
    own = owner(snap)
    cnt = np.bincount(own, minlength=snap.dims["clusters"] + 1)
    worker = ((snap.p_packed >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER
    donors = np.flatnonzero(worker & (own < snap.dims["clusters"]) & (cnt[own] <= 256))[::-1]
    rows = donors[:size - int(cnt[c])]
    g0 = int(snap.c_group_off[c])
    snap.p_ns_id[rows], snap.p_cluster_name_id[rows], snap.p_group_name_id[rows] = snap.c_ns_id[c], snap.c_name_id[c], snap.g_name_id[g0]
    return rows


def plan(base, variant):
    """(the epoch's snapshot, its changed pod rows), prepared outside the timed window."""
    snap = copy.deepcopy(base)
    if variant == "crossing":
        rows = grow(snap, CROSS, 8300)
    elif variant == "huge regrowth":
        rows = grow(snap, huge_rows(snap)[0], 25100)
    else:
        rows = np.random.default_rng(3).choice(snap.dims["pods"], 1000, replace=False)
        snap.p_packed[rows] ^= np.uint32(1 << abi.PP_READY_SHIFT)
    return snap, np.unique(rows).astype(np.uint32)


def run(base, flags, snap, rows, on, profiled=False):
    eng = Engine.for_snapshot(base, slack=1.25, max_creates=1 << 20, large_clusters=True, huge_clusters=True, large_growth=True,
                              huge_growth=on)
    try:
        eng.load(base)
        eng.reconcile(flags)
        eng.reconcile(flags)
        t = time.perf_counter()
        eng.commit_pod_values(rows, np.stack([snap.cols[c][rows].view(np.uint32) for c in POD_COLS], axis=1))
        if profiled:
            kernels = [[k, round(ms, 4)] for k, ms in eng.reconcile_profiled(flags)["kernels"]]
            got = eng.fetch()
            return {"huge_growth": on, "incremental": got.changed_clusters is not None, "kernels": kernels}
        got = eng.reconcile(flags)
        wall = (time.perf_counter() - t) * 1e3
        p = eng.last_profile()
        return {"huge_growth": on, "incremental": got.changed_clusters is not None, "kernel_ms": round(p["kernels_ms"], 4),
                "wall_ms": round(wall, 4), "h2d_bytes": int(p["h2d_bytes"]), "d2h_bytes": int(p["d2h_bytes"])}
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    gpu = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    lines = [{"gpu": gpu, "fields": q}]
    print(json.dumps(lines[0]), flush=True)
    base, flags = synthetic.generate(synthetic.config("C3H"))
    grow(base, CROSS, 8000)
    flags.fetch_pod_lists = 0
    for variant in ("crossing", "huge regrowth", "churn"):
        snap, rows = plan(base, variant)
        for r in range(a.runs):
            for on in (False, True):
                rec = run(base, flags, snap, rows, on)
                rec.update({"workload": "C3H+8000", "variant": variant, "run": r, "rows": int(rows.size)})
                lines.append(rec)
                print(json.dumps(rec), flush=True)
    snap, rows = plan(base, "huge regrowth")
    rec = run(base, flags, snap, rows, True, profiled=True)
    rec.update({"workload": "C3H+8000", "variant": "huge regrowth, profiled"})
    lines.append(rec)
    print(json.dumps(rec), flush=True)
    gpu = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    lines.append({"gpu_after": gpu})
    print(json.dumps(lines[-1]), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "huge_growth_bench.jsonl"), "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()

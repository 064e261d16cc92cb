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
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from benchlib import Recorder, alternate, owners, timed_epoch  # noqa: E402
from kuberay_b200 import abi, synthetic  # noqa: E402
from kuberay_b200.engine import Engine  # noqa: E402

CROSS = 5000  # the RayCluster grown to 8 000 Pods


def huge_rows(snap):
    return [int(c) for c in np.flatnonzero(owners(snap)[1] > 10000)]


def grow(snap, c, size):
    """Worker Pods of the ordinary RayClusters (last rows first) move into RayCluster c's worker group 0 until it lists `size`
    Pods.  -> the pod rows that moved."""
    own, cnt = owners(snap)
    worker = ((snap.p_packed >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER
    donors = np.flatnonzero(worker & (own >= 0) & (cnt[own] <= 256))[::-1]
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
        if profiled:
            inc, kern = timed_epoch(eng, snap, rows, flags, profiled=True)
            return {"huge_growth": on, "incremental": inc, "kernels": [[k, round(ms, 4)] for k, ms in kern]}
        e = timed_epoch(eng, snap, rows, flags)
        p = eng.last_profile()
        return {"huge_growth": on, "incremental": e["incremental"], "kernel_ms": e["kernel_ms"], "wall_ms": e["wall_ms"],
                "h2d_bytes": int(p["h2d_bytes"]), "d2h_bytes": int(p["d2h_bytes"])}
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = Recorder("huge_growth_bench", a.out)
    base, flags = synthetic.generate(synthetic.config("C3H"))
    grow(base, CROSS, 8000)
    flags.fetch_pod_lists = 0
    for variant in ("crossing", "huge regrowth", "churn"):
        snap, rows = plan(base, variant)
        alternate(a.runs, lambda r, on: out.record(dict(run(base, flags, snap, rows, on), workload="C3H+8000", variant=variant, run=r,
                                                        rows=int(rows.size))))
    snap, rows = plan(base, "huge regrowth")
    out.record(dict(run(base, flags, snap, rows, True, profiled=True), workload="C3H+8000", variant="huge regrowth, profiled"))
    out.finish()


if __name__ == "__main__":
    main()

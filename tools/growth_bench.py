"""KR_OPT_LARGE_GROWTH on one GPU: RayClusters scaling past their bucket or region, with the option off and on, alternated (one JSON
line per run).

Workloads: C3 (10 000 RayClusters x 100 Pods) and C3L (C3 with 20 RayClusters of 2 000 Pods), KR_OPT_LARGE_CLUSTERS on, fixed layout.
Each run is one full pass, then, each epoch timed on its own (host clock around the Pod commit and kr_reconcile_batch, results copy
included; kernel ms from the device events of kr_profile):
  * churn:   5 epochs of 1 % Pod status flips (the steady epoch: its cost with the option on is the extra launches), then one more,
             profiled, for the per-kernel times;
  * cross1:  one ordinary RayCluster gains Pods until it lists stride + 16 (Pods move in from RayClusters at the end of the fleet);
  * cross10: ten more do the same in one epoch;
  * region1: a RayCluster given a region (the first of cross1) gains Pods past it (to 2.5 x its count);
  * churn again, once (the epoch after the growth).
Option on, one more profiled epoch promotes 48 RayClusters to stride + 8 .. 250 Pods and reports k_inc_grow, k_large_sort and k_decide_large
(the per-cluster kernels over mid-size promoted RayClusters, which size KR_GROW_MAX and the list cap).  The card's name and power
limit are read in the same run.
Usage: python tools/growth_bench.py [--runs 3] [--out DIR]"""
import argparse
import copy
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from benchlib import Recorder, alternate, churn_rows, owners, timed_epoch  # noqa: E402
from kuberay_b200 import abi, synthetic  # noqa: E402
from kuberay_b200.engine import Engine  # noqa: E402


class Fleet:
    """One engine on a snapshot; Pods move from donor RayClusters (the last rows) into chosen ones, one commit per epoch."""

    def __init__(self, snap, flags, on):
        self.snap, self.flags = snap, flags
        self.eng = Engine.for_snapshot(snap, max_creates=4 * snap.dims["pods"], large_clusters=True, large_growth=on)
        self.eng.set_fixed_layout(True)
        self.eng.load(snap)
        self.eng.reconcile(flags)
        self.stride = self.eng.get_option(abi.OPT_BUCKET_STRIDE)
        own, self.count = owners(snap)
        worker = ((snap.p_packed >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER
        n = snap.dims["clusters"]
        self.donors = list(np.flatnonzero(worker & (own >= n - n // 4))[::-1])  # the last quarter of the fleet gives Pods
        self.rng = np.random.default_rng(5)

    def grow(self, c, to):
        need = max(0, int(to) - int(self.count[c]))
        rows = np.array([self.donors.pop() for _ in range(need)], dtype=np.int64)
        s = self.snap
        s.p_ns_id[rows], s.p_cluster_name_id[rows] = s.c_ns_id[c], s.c_name_id[c]
        s.p_group_name_id[rows] = s.g_name_id[s.c_group_off[c]]
        self.count[c] += need
        return rows

    def churn(self):
        return churn_rows(self.snap, self.rng)

    def epoch(self, rows, profiled=False):
        return timed_epoch(self.eng, self.snap, rows, self.flags, profiled)


def run(base, flags, workload, on, r):
    f = Fleet(copy.deepcopy(base), flags, on)
    try:
        n = base.dims["clusters"]
        small = [int(c) for c in np.flatnonzero(f.count[:n - n // 4] <= f.stride)[:64]]  # (not donors)
        rec = {"workload": workload, "large_growth": on, "run": r, "stride": f.stride}
        churn = [f.epoch(f.churn()) for _ in range(5)]
        rec["churn_kernel_ms"] = [e["kernel_ms"] for e in churn]
        rec["churn_wall_ms"] = [e["wall_ms"] for e in churn]
        _, kern = f.epoch(f.churn(), profiled=True)  # (serialised, each kernel between events: where the option's extra time goes)
        rec["churn_profiled"] = [[k, round(ms, 4)] for k, ms in kern]
        rec["cross1"] = f.epoch(f.grow(small[0], f.stride + 16))
        rec["cross10"] = f.epoch(np.concatenate([f.grow(c, f.stride + 16) for c in small[1:11]]))
        rec["region1"] = f.epoch(f.grow(small[0], int(f.count[small[0]] * 5 // 2)))
        rec["churn_after"] = f.epoch(f.churn())
        rec["stride_after"] = f.eng.get_option(abi.OPT_BUCKET_STRIDE)
        if on:
            mid, lo = small[16:64], f.stride + 8
            rows = np.concatenate([f.grow(c, lo + (250 - lo) * i // len(mid)) for i, c in enumerate(mid)])
            inc, kern = f.epoch(rows, profiled=True)
            keep = ("k_inc_admit", "k_inc_grow", "k_decide2_dirty", "k_large_sort", "k_decide_large")
            rec["promote48_profiled"] = {"incremental": inc, "kernels": [[k, round(ms, 4)] for k, ms in kern if k in keep]}
        return rec
    finally:
        f.eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = Recorder("growth_bench", a.out)
    for workload in ("C3", "C3L"):
        base, flags = synthetic.generate(synthetic.config(workload))
        flags.fetch_pod_lists = 0
        alternate(a.runs, lambda r, on: out.record(run(base, flags, workload, on, r)))
    out.finish()


if __name__ == "__main__":
    main()

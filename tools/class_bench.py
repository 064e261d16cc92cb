"""The RayCluster-class options on one GPU: KR_OPT_LARGE_CLUSTERS, _WIDE_CLUSTERS or _HUGE_CLUSTERS (--option), off and on,
alternated, three runs each (one JSON line per measurement).

Per workload and setting: the full-pass ms (incremental epochs off; host clock around kr_reconcile_batch, so the results copy is
included), the stride, and the option's kernels alone in a profiled pass; then, on every workload but C3, 20 epochs of 1 % pod churn
(PodReady flips) with incremental epochs on: how many ran incrementally on the device and their median kernel ms.
  large  C3L (C3 with 20 RayClusters of 2 000 Pods): k_large_sort, k_decide_large and k_decide_huge;
         C3 (no large RayCluster: k_match2 only gains a branch).
  wide   C3W (C3 with 100 RayClusters of 48 worker groups) and ALLW (2 000 RayClusters x 100 pods x 40 worker groups, every one
         wide): k_large_sort and k_decide_large; C3 (no wide RayCluster: the option changes nothing the pass launches).
  huge   KR_OPT_LARGE_CLUSTERS on throughout; the pipeline too.  C3H (C3 with 2 RayClusters of 20 000 Pods): k_huge_tiles,
         k_huge_merge, k_decide_large and k_decide_huge; C3 (no huge RayCluster): the kernels launched, which must be the same.
Usage: python tools/class_bench.py --option large|wide|huge [--steps 30] [--runs 3] [--workloads W,...] [--out DIR]
(writes <option>_bench.jsonl under DIR)"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from benchlib import POD_COLS, Recorder, alternate, churn_rows, pod_values  # noqa: E402
from kuberay_b200 import abi, synthetic  # noqa: E402
from kuberay_b200.engine import Engine  # noqa: E402

WORKLOADS = {
    "C3": lambda: synthetic.config("C3"),
    "C3L": lambda: synthetic.config("C3L"),
    "C3W": lambda: synthetic.config("C3W"),
    "ALLW": lambda: synthetic.SynthParams(n_clusters=2000, pods_per_cluster=100, groups=40),
    "C3H": lambda: synthetic.config("C3H"),
}
OPTIONS = {  # the Engine.for_snapshot keywords with the option off / on, the workloads, and the kernels recorded
    "large": (lambda on: {"large_clusters": on}, ("C3L", "C3"), ("k_large_sort", "k_decide_large", "k_decide_huge")),
    "wide": (lambda on: {"wide_clusters": on}, ("C3W", "ALLW", "C3"), ("k_large_sort", "k_decide_large")),
    "huge": (lambda on: {"large_clusters": True, "huge_clusters": on}, ("C3H", "C3"),
             ("k_huge_tiles", "k_huge_merge", "k_decide_large", "k_decide_huge")),
}


def full_pass(snap, flags, opts, steps):
    """-> ms per full pass, the kernels of one profiled pass, the stride."""
    eng = Engine.for_snapshot(snap, **opts)
    try:
        eng.set_incremental(False)
        eng.load(snap)
        for _ in range(3):
            eng.reconcile(flags)
        t = time.perf_counter()
        for _ in range(steps):
            eng.reconcile(flags)
        ms = (time.perf_counter() - t) * 1e3 / steps
        return ms, eng.reconcile_profiled(flags)["kernels"], eng.get_option(abi.OPT_BUCKET_STRIDE)
    finally:
        eng.close()


def churn(snap, flags, opts, epochs=20, seed=1):
    """-> how many of the churn epochs ran incrementally, and their median kernel ms."""
    eng = Engine.for_snapshot(snap, **opts)
    rng = np.random.default_rng(seed)
    try:
        eng.set_fixed_layout(True)
        views = eng.load(snap)
        eng.reconcile(flags)
        n_inc, kms = 0, []
        for _ in range(epochs):
            rows = churn_rows(snap, rng)
            for c in POD_COLS:
                views[c][rows] = snap.cols[c][rows]
            eng.commit_pod_values(rows, pod_values(snap, rows))
            n_inc += eng.reconcile(flags).changed_clusters is not None
            kms.append(eng.last_profile()["kernels_ms"])
        return n_inc, float(np.median(kms))
    finally:
        eng.close()


def measure(option, name, snap, flags, run, on, steps):
    opts, _, kernels = OPTIONS[option]
    ms, kern, stride = full_pass(snap, flags, opts(on), steps)
    kd = dict(kern)
    rec = {"workload": name, "run": run, f"{option}_clusters": on}
    if option == "huge":
        rec.update(pipeline="bucket" if "k_match2" in kd else "sort", stride=stride, full_pass_ms=round(ms, 4))
    else:
        rec.update(full_pass_ms=round(ms, 4), stride=stride)
    if option == "huge" and name == "C3":
        rec["kernels"] = [k for k, _ in kern]
    else:
        rec.update({k + "_ms": kd.get(k) for k in kernels})
    if name != "C3":
        s2, _ = synthetic.generate(WORKLOADS[name]())
        rec["incremental_epochs_of_20"], rec["epoch_kernel_ms_median"] = churn(s2, flags, opts(on))
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--option", required=True, choices=sorted(OPTIONS))
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--workloads", default=None, help="comma-separated, of the option's own (default: all of them)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = Recorder(f"{a.option}_bench", a.out)
    for name in a.workloads.split(",") if a.workloads else OPTIONS[a.option][1]:
        snap, flags = synthetic.generate(WORKLOADS[name]())
        flags.fetch_pod_lists = 0
        alternate(a.runs, lambda run, on: out.record(measure(a.option, name, snap, flags, run, on, a.steps)))
    out.finish()


if __name__ == "__main__":
    main()

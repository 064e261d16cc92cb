"""KR_OPT_CLUSTER_CREATES on one GPU: RayCluster creation epochs with the option off and on, alternated (one JSON line per run).

Workload: C3 (10 000 RayClusters x 100 Pods) plus the RayClusters the epochs create.  Each run is a fixed-layout engine for the whole
fleet, one full pass over its first 10 000 RayClusters, then N epochs that each append `--new` RayClusters:
  * pods="with": the new RayClusters' Pods arrive in the same epoch (kr_snapshot_commit_pod_values), no resident orphan;
  * pods="orphans": their Pods are resident from the start (orphans until their RayCluster appears), so k_inc_orphan_adopt runs.
An epoch commits the object part, then the new specs as spec rows (option on) or the whole JSON arena (option off, as the native
packer does without the option).  Reported: incremental epochs out of N, median epoch kernel ms (device events), median epoch wall
ms through the C ABI (host clock around the commits and kr_reconcile_batch, results copy included), and, option on, the creation
kernels alone in one profiled epoch.
Usage: python tools/creates_bench.py [--epochs 10] [--runs 3] [--new 4] [--out DIR]"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from benchlib import OBJ_COLS, POD_COLS, Recorder, alternate, pod_values  # noqa: E402
from kuberay_b200 import abi, synthetic  # noqa: E402
from kuberay_b200.engine import Engine  # noqa: E402
KERNELS = ("k_inc_orphan_adopt", "k_inc_clusters_insert", "k_hash_rows", "k_inc_admit", "k_decide2_dirty")


def run(full, flags, base, on, pods, epochs, new):
    d = full.dims
    eng = Engine(0, d["clusters"], d["groups"], d["wtd"], d["pods"], d["heads"], d["jobs"], max(1024, d["pods"]), d["json"])
    try:
        eng.set_cluster_creates(on)
        eng.set_fixed_layout(True)
        cur = synthetic.first_clusters(full, base, free_pods=pods == "with")
        eng.load(cur)
        eng.reconcile(flags)
        n_inc, kms, wall, prof = 0, [], [], None
        for i in range(epochs):
            k = base + (i + 1) * new
            s = synthetic.first_clusters(full, k, free_pods=pods == "with")   # (prepared outside the timed window)
            rows = np.flatnonzero(np.any([cur.cols[c] != s.cols[c] for c in POD_COLS], axis=0)).astype(np.uint32)
            vals = pod_values(s, rows) if rows.size else None
            t = time.perf_counter()
            views = eng.begin(s.sizes())
            for c in OBJ_COLS:
                np.copyto(views[c], s.cols[c])
            if on:
                eng.commit(abi.PART_OBJECTS)
                eng.commit_spec_rows(np.arange(k - new, k, dtype=np.uint32))
            else:
                eng.commit(abi.PART_OBJECTS | abi.PART_JSON)
            if rows.size:
                eng.commit_pod_values(rows, vals)
            if on and i == epochs - 1:   # the last epoch profiled: the creation kernels alone
                prof = dict(eng.reconcile_profiled(flags)["kernels"])
                got = eng.fetch()
            else:
                got = eng.reconcile(flags)
                wall.append((time.perf_counter() - t) * 1e3)
                kms.append(eng.last_profile()["kernels_ms"])
            n_inc += got.changed_clusters is not None
            cur = s
        rec = {"workload": "C3", "cluster_creates": on, "pods": pods, "new_per_epoch": new, "incremental_epochs": n_inc, "epochs": epochs,
               "epoch_kernel_ms_median": round(float(np.median(kms)), 4), "epoch_wall_ms_median": round(float(np.median(wall)), 4)}
        if prof:
            rec.update({kn + "_ms": prof.get(kn) for kn in KERNELS})
        return rec
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--new", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = Recorder("creates_bench", a.out)
    base = synthetic.config("C3").n_clusters
    full, flags = synthetic.generate(synthetic.config("C3", n_clusters=base + a.epochs * a.new))
    flags.fetch_pod_lists = 0
    for pods in ("with", "orphans"):
        alternate(a.runs, lambda r, on: out.record(dict(run(full, flags, base, on, pods, a.epochs, a.new), run=r)))
    out.finish()


if __name__ == "__main__":
    main()

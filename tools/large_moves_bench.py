"""KR_OPT_LARGE_MOVES on one GPU: epochs that delete, move or regroup large RayClusters, with the option off and on, alternated (one
JSON line per run).

Workload: C3L (10 000 RayClusters x 100 Pods, 20 of them grown to 2 000 Pods) on a fixed-layout engine with KR_OPT_LARGE_CLUSTERS,
_CLUSTER_DELETES, _CLUSTER_CREATES and _GROUP_EDITS, and C3H (2 of 20 000 Pods) with _HUGE_CLUSTERS as well.  Each run is one full
pass (two: the first one classifies the large RayClusters), then N epochs of one variant, each committing the object part:
  * "delete large": a large RayCluster deleted from a middle row, its hole filled by the last row (an ordinary one);
  * "move large": an ordinary RayCluster deleted, its hole filled by the last row, which is large (the large RayClusters are laid
    out last for this variant);
  * "append group": a worker group appended to a large RayCluster (a copy of its first group under a new name);
  * "delete huge" / "move huge" (C3H, two epochs): a huge RayCluster moved into a deleted row's hole, then deleted.
Reported per run: incremental epochs, median epoch kernel ms (device events), median epoch wall ms through the C ABI (host clock
around the commits and kr_reconcile_batch, results copy included), median H2D and D2H bytes (kr_profile), and, option on, the kernel
list of the last epoch, profiled.  The card's name, power limit and clocks are read in the same run.
Usage: python tools/large_moves_bench.py [--epochs 10] [--runs 3] [--out DIR]"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from benchlib import OBJ_COLS, Recorder, alternate, owners  # noqa: E402
from kuberay_b200 import abi, synthetic  # noqa: E402
from kuberay_b200.engine import Engine  # noqa: E402


def large_rows(snap):
    """Rows of the RayClusters that list more than 256 Pods."""
    return [int(c) for c in np.flatnonzero(owners(snap)[1] > 256)]


def plan(base, variant, epochs, seed):
    """(the first snapshot, every epoch's snapshot), prepared outside the timed window."""
    rng = np.random.default_rng(seed)
    big = large_rows(base)
    if variant in ("move large", "huge"):  # the large RayClusters last: each deletion of an ordinary one moves one of them
        small = [c for c in range(base.dims["clusters"]) if c not in big]
        base = synthetic.select_clusters(base, small + big)
        big = large_rows(base)
    cur, out = base, []
    fresh = int(max(base.g_name_id.max(), base.p_group_name_id.max(), base.p_name_id.max(), base.c_name_id.max())) + 1
    for e in range(epochs if variant != "huge" else 2):
        n = cur.dims["clusters"]
        big = large_rows(cur)
        if variant == "delete large":
            cur = synthetic.delete_clusters(cur, [[c for c in big if c < n - 1][int(rng.integers(len(big) - 1))]])
        elif variant in ("move large", "huge"):
            if variant == "huge" and e == 1:
                cur = synthetic.delete_clusters(cur, [row])  # the huge RayCluster moved in the first epoch
            else:
                row = int(rng.integers(100, n - 100))
                cur = synthetic.delete_clusters(cur, [row])
        else:
            c = big[int(rng.integers(len(big)))]
            g0, G = int(cur.c_group_off[c]), int(cur.c_group_cnt[c])
            cur = synthetic.regroup_clusters(cur, {c: [(g, None) for g in range(g0, g0 + G)] + [(g0, fresh)]})
            fresh += 1
        out.append(cur)
    return base, out


def run(base, flags, steps, on, huge):
    d = base.dims
    eng = Engine(0, d["clusters"], d["groups"] + 64, d["wtd"] + 64 * int(base.g_wtd_cnt.max(initial=0)), d["pods"], d["heads"], d["jobs"],
                 max(1024, d["pods"]), d["json"])
    try:
        eng.set_large_clusters(True)
        eng.set_huge_clusters(huge)
        for opt in ("cluster_deletes", "cluster_creates", "group_edits"):
            getattr(eng, f"set_{opt}")(True)
        eng.set_large_moves(on)
        eng.set_fixed_layout(True)
        eng.load(base)
        eng.reconcile(flags)
        eng.reconcile(flags)
        n_inc, kms, wall, h2d, d2h, prof = 0, [], [], [], [], None
        for i, s in enumerate(steps):
            t = time.perf_counter()
            views = eng.begin(s.sizes())
            for c in OBJ_COLS:
                np.copyto(views[c], s.cols[c])
            eng.commit(abi.PART_OBJECTS)
            if on and i == len(steps) - 1 and len(steps) > 2:  # the last epoch profiled (serialised)
                prof = [[kn, round(ms, 4)] for kn, ms in eng.reconcile_profiled(flags)["kernels"]]
                got = eng.fetch()
            else:
                got = eng.reconcile(flags)
                wall.append((time.perf_counter() - t) * 1e3)
                p = eng.last_profile()
                kms.append(p["kernels_ms"]); h2d.append(p["h2d_bytes"]); d2h.append(p["d2h_bytes"])
            n_inc += got.changed_clusters is not None
        rec = {"large_moves": on, "incremental_epochs": n_inc, "epochs": len(steps),
               "epoch_kernel_ms_median": round(float(np.median(kms)), 4), "epoch_wall_ms_median": round(float(np.median(wall)), 4),
               "h2d_bytes_median": int(np.median(h2d)), "d2h_bytes_median": int(np.median(d2h)), "kernel_ms": [round(x, 4) for x in kms]}
        if prof:
            rec["kernels_last_epoch"] = prof
        return rec
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = Recorder("large_moves_bench", a.out)
    for workload, variants in (("C3L", ("delete large", "move large", "append group")), ("C3H", ("huge",))):
        snap, flags = synthetic.generate(synthetic.config(workload))
        flags.fetch_pod_lists = 0
        for variant in variants:
            base, steps = plan(snap, variant, a.epochs, seed=7)
            alternate(a.runs, lambda r, on: out.record(dict(run(base, flags, steps, on, workload == "C3H"), workload=workload, variant=variant,
                                                            run=r)))
    out.finish()


if __name__ == "__main__":
    main()

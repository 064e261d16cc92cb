"""KR_OPT_CLUSTER_DELETES on one GPU: RayCluster deletion epochs with the option off and on, alternated (one JSON line per run).

Workload: C3 (10 000 RayClusters x 100 Pods).  Each run is a fixed-layout engine, one full pass, then N epochs that each delete
`--k` random RayClusters by swap-remove (the last RayCluster moves into each hole, as the native packer does); their Pods stay, as
orphans until garbage collection would remove them:
  * variant "delete": nothing else happens in the epoch; it commits the object part;
  * variant "delete+create": the epoch also creates `--k` RayClusters after the last row (their Pods are resident from the start,
    orphans until then).  Option on (with KR_OPT_CLUSTER_CREATES): the object part, then the new specs as spec rows; option off: the
    object part and the whole JSON arena, as the native packer sends them without the options.
Reported: incremental epochs out of N, median epoch kernel ms (device events), median epoch wall ms through the C ABI (host clock
around the commits and kr_reconcile_batch, results copy included), and, option on, the renumbering kernels in one profiled epoch.
The card's name and power limit are read in the same run.
Usage: python tools/deletes_bench.py [--epochs 10] [--runs 3] [--k 4] [--out DIR]"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from benchlib import OBJ_COLS, Recorder, alternate  # noqa: E402
from kuberay_b200 import abi, synthetic  # noqa: E402
from kuberay_b200.engine import Engine  # noqa: E402
KERNELS = ("k_inc_digest_move", "k_inc_clusters_release", "k_inc_orphan_adopt", "k_inc_clusters_translate", "k_inc_clusters_rekey",
           "k_inc_groups_gather", "k_inc_clusters_insert", "k_hash_rows", "k_inc_admit", "k_decide2_dirty")


def plan(full, base, epochs, k, create, seed):
    """Per epoch: the old row of every new row (new RayClusters: rows of `full` past `base`) and the created rows."""
    rng = np.random.default_rng(seed)
    cur = list(range(base))
    nxt = base
    out = []
    for _ in range(epochs):
        rows = rng.choice(len(cur), size=k, replace=False)
        order = [cur[i] for i in synthetic.swap_remove_order(len(cur), rows)]
        created = []
        if create:
            created = list(range(len(order), len(order) + k))
            order += list(range(nxt, nxt + k))
            nxt += k
        out.append((order, created))
        cur = order
    return out


def run(full, flags, base, on, create, steps):
    d = full.dims
    eng = Engine(0, d["clusters"], d["groups"], d["wtd"], d["pods"], d["heads"], d["jobs"], max(1024, d["pods"]), d["json"])
    try:
        eng.set_cluster_deletes(on)
        eng.set_cluster_creates(on)
        eng.set_fixed_layout(True)
        cur = synthetic.select_clusters(full, np.arange(base))
        eng.load(cur)
        eng.reconcile(flags)
        n_inc, kms, wall, prof = 0, [], [], None
        for i, (order, created) in enumerate(steps):
            s = synthetic.select_clusters(full, order)   # (prepared outside the timed window)
            t = time.perf_counter()
            views = eng.begin(s.sizes())
            for c in OBJ_COLS:
                np.copyto(views[c], s.cols[c])
            if on or not created:
                eng.commit(abi.PART_OBJECTS)
                if created:
                    eng.commit_spec_rows(np.asarray(created, dtype=np.uint32))
            else:
                eng.commit(abi.PART_OBJECTS | abi.PART_JSON)
            if on and i == len(steps) - 1:   # the last epoch profiled: the renumbering kernels alone
                prof = dict(eng.reconcile_profiled(flags)["kernels"])
                got = eng.fetch()
            else:
                got = eng.reconcile(flags)
                wall.append((time.perf_counter() - t) * 1e3)
                kms.append(eng.last_profile()["kernels_ms"])
            n_inc += got.changed_clusters is not None or got.n_changed < s.dims["clusters"]
        rec = {"workload": "C3", "cluster_deletes": on, "variant": "delete+create" if create else "delete",
               "incremental_epochs": n_inc, "epochs": len(steps),
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
    ap.add_argument("--k", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = Recorder("deletes_bench", a.out)
    base = synthetic.config("C3").n_clusters
    full, flags = synthetic.generate(synthetic.config("C3", n_clusters=base + a.epochs * a.k))
    flags.fetch_pod_lists = 0
    for create in (False, True):
        steps = plan(full, base, a.epochs, a.k, create, seed=7)
        alternate(a.runs, lambda r, on: out.record(dict(run(full, flags, base, on, create, steps), k_per_epoch=a.k, run=r)))
    out.finish()


if __name__ == "__main__":
    main()

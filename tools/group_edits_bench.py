"""KR_OPT_GROUP_EDITS on one GPU: worker-group edit epochs with the option off and on, alternated (one JSON line per run).

Workload: C3 (10 000 RayClusters x 100 Pods) on a fixed-layout engine with room for the groups to come.  Each run is one full pass,
then N epochs that each edit `--k` random RayClusters:
  * variant "append": RayService-style, a worker group appended (a copy of the RayCluster's first group under a new name) with a
    re-emitted spec (one byte longer, at the end of the JSON arena).  Option on: the object part, then the specs as spec rows; option
    off: the object part and the whole JSON arena, as the native packer sends them without the option;
  * variant "remove": the RayCluster's last worker group removed (its Pods live on, in no group); the object part.
Reported: incremental epochs out of N, median epoch kernel ms (device events), median epoch wall ms through the C ABI (host clock
around the commits and kr_reconcile_batch, results copy included), median H2D and D2H bytes per epoch, and, option on, the kernel
list of the last epoch, profiled.  The card's name and power limit are read in the same run.
Usage: python tools/group_edits_bench.py [--epochs 10] [--runs 3] [--k 4] [--out DIR]"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from benchlib import OBJ_COLS, Recorder, alternate  # noqa: E402
from kuberay_b200 import abi, synthetic  # noqa: E402
from kuberay_b200.engine import Engine  # noqa: E402
from kuberay_b200.snapshot import Snapshot  # noqa: E402


def respec(snap, rows):
    """A copy of `snap` whose RayClusters `rows` have a spec one byte longer at the end of a grown JSON arena."""
    d = snap.dims
    end = (d["json"] + 15) // 16 * 16
    lens = {int(c): int(snap.c_json_len[c]) + 1 for c in rows}
    out = Snapshot(d["clusters"], d["groups"], d["wtd"], d["pods"], d["heads"], d["jobs"], end + sum((n + 15) // 16 * 16 for n in lens.values()))
    for name, _dt, _m, dim in abi.COLUMNS:
        if dim != "json":
            out.cols[name][:] = snap.cols[name]
    out.json[:d["json"]] = snap.json
    for c, n in lens.items():
        o = int(snap.c_json_off[c])
        out.json[end:end + n - 1] = snap.json[o:o + n - 1]
        out.json[end + n - 1] = 32
        out.c_json_off[c], out.c_json_len[c] = end, n
        end += (n + 15) // 16 * 16
    return out


def plan(base, epochs, k, variant, seed):
    """Every epoch's snapshot (prepared outside the timed window) and its re-emitted spec rows."""
    rng = np.random.default_rng(seed)
    cur, out = base, []
    fresh = int(max(base.g_name_id.max(), base.p_group_name_id.max(), base.p_name_id.max(), base.c_name_id.max())) + 1
    for _ in range(epochs):
        rows = sorted(int(c) for c in rng.choice(cur.dims["clusters"], size=k, replace=False))
        edits = {}
        for c in rows:
            g0, G = int(cur.c_group_off[c]), int(cur.c_group_cnt[c])
            groups = [(g, None) for g in range(g0, g0 + G)]
            if variant == "append":
                edits[c] = groups + [(g0, fresh)]
                fresh += 1
            else:
                edits[c] = groups[:-1]
        cur = synthetic.regroup_clusters(cur, edits)
        specs = []
        if variant == "append":
            cur, specs = respec(cur, rows), rows
        out.append((cur, specs))
    return out


def run(base, flags, room, on, steps):
    d = base.dims
    eng = Engine(0, d["clusters"], room["groups"], room["wtd"], d["pods"], d["heads"], d["jobs"], max(1024, d["pods"]), room["json"])
    try:
        eng.set_group_edits(on)
        eng.set_fixed_layout(True)
        eng.load(base)
        eng.reconcile(flags)
        n_inc, kms, wall, h2d, d2h, prof = 0, [], [], [], [], None
        for i, (s, specs) in enumerate(steps):
            t = time.perf_counter()
            views = eng.begin(s.sizes())
            for c in OBJ_COLS:
                np.copyto(views[c], s.cols[c])
            if specs:
                np.copyto(views["json"][:s.dims["json"]], s.json)
            if on or not specs:
                eng.commit(abi.PART_OBJECTS)
                if specs:
                    eng.commit_spec_rows(np.asarray(specs, dtype=np.uint32))
            else:
                eng.commit(abi.PART_OBJECTS | abi.PART_JSON)
            if on and i == len(steps) - 1:   # the last epoch profiled (serialised)
                prof = [[kn, round(ms, 4)] for kn, ms in eng.reconcile_profiled(flags)["kernels"]]
                got = eng.fetch()
            else:
                got = eng.reconcile(flags)
                wall.append((time.perf_counter() - t) * 1e3)
                p = eng.last_profile()
                kms.append(p["kernels_ms"]); h2d.append(p["h2d_bytes"]); d2h.append(p["d2h_bytes"])
            n_inc += got.changed_clusters is not None or got.n_changed < s.dims["clusters"]
        rec = {"workload": "C3", "group_edits": on, "incremental_epochs": n_inc, "epochs": len(steps),
               "epoch_kernel_ms_median": round(float(np.median(kms)), 4), "epoch_wall_ms_median": round(float(np.median(wall)), 4),
               "h2d_bytes_median": int(np.median(h2d)), "d2h_bytes_median": int(np.median(d2h))}
        if prof:
            rec["kernels_last_epoch"] = prof
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
    out = Recorder("group_edits_bench", a.out)
    base, flags = synthetic.generate(synthetic.config("C3"))
    flags.fetch_pod_lists = 0
    extra = a.epochs * a.k
    room = {"groups": base.dims["groups"] + extra, "wtd": base.dims["wtd"] + extra * int(base.g_wtd_cnt.max(initial=0)),
            "json": base.dims["json"] + 16 * extra + int(base.c_json_len.max()) * extra + 4096}
    for variant in ("append", "remove"):
        steps = plan(base, a.epochs, a.k, variant, seed=7)
        alternate(a.runs, lambda r, on: out.record(dict(run(base, flags, room, on, steps), variant=variant, k_per_epoch=a.k, run=r)))
    out.finish()


if __name__ == "__main__":
    main()

"""KR_OPT_HUGE_CLUSTERS on one GPU, KR_OPT_LARGE_CLUSTERS on throughout: the option off and on, alternated, three runs each (one
JSON line per measurement).

  C3H  the pipeline and stride, full-pass ms (incremental epochs off; host clock around kr_reconcile_batch, so the results copy is
       included), then 20 epochs of 1 % pod churn (PodReady flips) with incremental epochs on: how many ran incrementally on the
       device and their median kernel ms; k_huge_tiles, k_huge_merge, k_decide_large and k_decide_huge alone in a
       profiled pass;
  C3   the same full pass with the option off and on (no huge RayCluster): the kernels launched, which must be the same.
Usage: python tools/huge_bench.py [--steps 30] [--out DIR]"""
import argparse
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


def full_pass(snap, flags, huge, steps):
    eng = Engine.for_snapshot(snap, large_clusters=True, huge_clusters=huge)
    try:
        eng.set_incremental(False)
        eng.load(snap)
        for _ in range(3):
            eng.reconcile(flags)
        t = time.perf_counter()
        for _ in range(steps):
            eng.reconcile(flags)
        ms = (time.perf_counter() - t) * 1e3 / steps
        kern = eng.reconcile_profiled(flags)["kernels"]
        stride = eng.get_option(abi.OPT_BUCKET_STRIDE)
        return ms, kern, stride
    finally:
        eng.close()


def churn(snap, flags, huge, epochs=20, frac=0.01, seed=1):
    eng = Engine.for_snapshot(snap, large_clusters=True, huge_clusters=huge)
    rng = np.random.default_rng(seed)
    try:
        eng.set_fixed_layout(True)
        views = eng.begin(snap.sizes())
        eng.fill(views, snap)
        eng.commit()
        eng.reconcile(flags)
        n_inc, kms = 0, []
        for _ in range(epochs):
            rows = np.unique(rng.choice(snap.dims["pods"], int(snap.dims["pods"] * frac), replace=False)).astype(np.uint32)
            snap.cols["p_packed"][rows] ^= np.uint32(1 << abi.PP_READY_SHIFT)
            for c in POD_COLS:
                views[c][rows] = snap.cols[c][rows]
            eng.commit_pod_values(rows, np.stack([snap.cols[c][rows].view(np.uint32) for c in POD_COLS], axis=1))
            got = eng.reconcile(flags)
            n_inc += got.changed_clusters is not None
            kms.append(eng.last_profile()["kernels_ms"])
        return n_inc, float(np.median(kms))
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    gpu = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    lines = [{"gpu": gpu, "fields": q}]
    print(json.dumps(lines[0]), flush=True)
    for name in ("C3H", "C3"):
        snap, flags = synthetic.generate(synthetic.config(name))
        flags.fetch_pod_lists = 0
        for run in range(a.runs):
            for huge in (False, True):
                ms, kern, stride = full_pass(snap, flags, huge, a.steps)
                names = [k for k, _ in kern]
                kd = dict(kern)
                rec = {"workload": name, "run": run, "huge_clusters": huge, "pipeline": "bucket" if "k_match2" in names else "sort",
                       "stride": stride, "full_pass_ms": round(ms, 4)}
                if name == "C3H":
                    rec.update({k + "_ms": kd.get(k) for k in ("k_huge_tiles", "k_huge_merge", "k_decide_large", "k_decide_huge")})
                    s2, _ = synthetic.generate(synthetic.config(name))
                    rec["incremental_epochs_of_20"], rec["epoch_kernel_ms_median"] = churn(s2, flags, huge)
                else:
                    rec["kernels"] = names
                lines.append(rec)
                print(json.dumps(rec), flush=True)
    gpu = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    lines.append({"gpu_after": gpu})
    print(json.dumps(lines[-1]), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "huge_bench.jsonl"), "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()

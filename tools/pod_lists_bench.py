"""KR_OPT_BUCKET_POD_LISTS on one GPU: incremental epochs of C3 with 1 % Pod churn, fetching the full pod lists every epoch and every
third epoch, with the option off and on, alternated in one session (one JSON line per run).

Each run is a fresh engine on a fixed layout: one full pass, then EPOCHS epochs of PodReady flips on 1 % of the Pods, committed as
Pod values.  Per run: the mean wall ms per epoch through the C ABI (host clock around the commit and kr_reconcile_batch, results copy
included), the mean D2H bytes per epoch (kr_profile), and how many epochs were incremental.  With the option on, one more fetching
epoch is profiled for the builder's kernels (k_lists_init .. k_lists_gather, device events).  The card's name and power limit are read
in the same run.
Usage: python tools/pod_lists_bench.py [--runs 2] [--epochs 30] [--out DIR]"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from benchlib import Recorder, churn_rows, pod_values  # noqa: E402
from kuberay_b200 import abi, synthetic  # noqa: E402
from kuberay_b200.engine import Engine  # noqa: E402


def run(snap, flags, on, every, epochs, seed):
    eng = Engine.for_snapshot(snap, max_creates=1 << 21, bucket_pod_lists=on)
    try:
        eng.set_fixed_layout(True)
        eng.load(snap)
        flags.fetch_pod_lists = 0
        eng.reconcile(flags)
        rng = np.random.default_rng(seed)
        n = snap.dims["pods"]
        ms, d2h, inc = [], [], 0
        for e in range(epochs + 1):
            rows = churn_rows(snap, rng)
            vals = pod_values(snap, rows)
            flags.fetch_pod_lists = 1 if e % every == 0 else 0
            t0 = time.perf_counter()
            eng.commit_pod_values(rows, vals)
            got = eng.reconcile(flags)
            t1 = time.perf_counter()
            if e == 0:
                continue  # (warm-up: the first epoch captures and instantiates the pass's graph for these flags)
            ms.append((t1 - t0) * 1e3)
            d2h.append(eng.last_profile()["d2h_bytes"])
            inc += got.changed_clusters is not None
        out = {"option": on, "fetch_every": every, "epochs": epochs, "incremental": inc, "ms_per_epoch": round(float(np.mean(ms)), 4),
               "ms_p50": round(float(np.median(ms)), 4), "d2h_bytes_per_epoch": int(np.mean(d2h))}
        if on:
            rows = np.arange(0, n, 100, dtype=np.uint32)
            snap.cols["p_packed"][rows] ^= np.uint32(1 << abi.PP_READY_SHIFT)
            eng.commit_pod_values(rows, pod_values(snap, rows))
            flags.fetch_pod_lists = 1
            prof = eng.reconcile_profiled(flags)
            names = [k for k, _ in prof["kernels"]]
            lo, hi = names.index("k_lists_init"), len(names) - 1 - names[::-1].index("k_lists_gather")
            out["builder_us"] = round(1e3 * sum(t for _, t in prof["kernels"][lo:hi + 1]), 2)
            out["builder_kernels"] = [f"{k}:{round(1e3 * t, 2)}" for k, t in prof["kernels"][lo:hi + 1]]
        return out
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--epochs", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = Recorder("pod_lists_bench", a.out)
    for r in range(a.runs):
        for every in (1, 3):
            for on in (False, True):
                snap, flags = synthetic.generate(synthetic.config("C3"))
                out.record(dict(run(snap, flags, on, every, a.epochs, 100 + r), run=r))
    out.finish()


if __name__ == "__main__":
    main()

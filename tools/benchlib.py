"""What the engine-option benchmarks under tools/ share: the card read, the JSON-lines record writer, the off/on alternation, and the
Pod-side steps of their epochs (PodReady churn, Pod owners, one timed Pod-value epoch).

The scripts put the repository root on sys.path before they import this module, so they run against a development build too
(KR_ENGINE_LIB)."""
import json
import os
import subprocess
import time

import numpy as np

from kuberay_b200 import abi

CARD_FIELDS = "name,power.limit,clocks.sm,clocks.max.sm"
POD_COLS = [name for name, _dt, _m, dim in abi.COLUMNS if dim == "pods"]
OBJ_COLS = [name for name, _dt, _m, dim in abi.COLUMNS if dim not in ("pods", "json")]


def card() -> str:
    """The card's CARD_FIELDS, as nvidia-smi prints them."""
    return subprocess.run(["nvidia-smi", f"--query-gpu={CARD_FIELDS}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


class Recorder:
    """Prints each record as a JSON line and keeps it.  The first line is the card read before the run, with `head`'s fields;
    finish() adds the card read after the run and, given out_dir, writes every line to <out_dir>/<name>.jsonl."""

    def __init__(self, name: str, out_dir: str | None = None, **head):
        self.name, self.out_dir, self.lines = name, out_dir, []
        self.record({"gpu": card(), "fields": CARD_FIELDS, **head})

    def record(self, rec: dict):
        self.lines.append(rec)
        print(json.dumps(rec), flush=True)

    def finish(self):
        self.record({"gpu_after": card()})
        if self.out_dir:
            os.makedirs(self.out_dir, exist_ok=True)
            with open(os.path.join(self.out_dir, f"{self.name}.jsonl"), "w") as f:
                f.writelines(json.dumps(x) + "\n" for x in self.lines)


def alternate(runs: int, fn):
    """fn(run, on) for every run, the option off and then on."""
    for run in range(runs):
        for on in (False, True):
            fn(run, on)


def pod_values(snap, rows) -> np.ndarray:
    """The Pod columns of `rows`, one row each, as commit_pod_values takes them."""
    return np.stack([snap.cols[c][rows].view(np.uint32) for c in POD_COLS], axis=1)


def churn_rows(snap, rng, frac: float = 0.01) -> np.ndarray:
    """Flips PodReady on `frac` of the Pods, drawn without replacement.  -> their rows, sorted."""
    n = snap.dims["pods"]
    rows = np.unique(rng.choice(n, int(n * frac), replace=False)).astype(np.uint32)
    snap.cols["p_packed"][rows] ^= np.uint32(1 << abi.PP_READY_SHIFT)
    return rows


def owners(snap) -> tuple[np.ndarray, np.ndarray]:
    """Pod row -> RayCluster row (-1: none), and each RayCluster's Pod count."""
    ckey = (snap.c_ns_id.astype(np.uint64) << np.uint64(32)) | snap.c_name_id.astype(np.uint64)
    order = np.argsort(ckey)
    pkey = (snap.p_ns_id.astype(np.uint64) << np.uint64(32)) | snap.p_cluster_name_id.astype(np.uint64)
    pos = np.minimum(np.searchsorted(ckey[order], pkey), order.size - 1)
    own = np.where(ckey[order][pos] == pkey, order[pos], -1)
    return own, np.bincount(own[own >= 0], minlength=snap.dims["clusters"])


def timed_epoch(eng, snap, rows, flags, profiled: bool = False):
    """One epoch: commit `snap`'s Pod values at `rows`, then reconcile, with a host clock around both (results copy included).
    -> {incremental, wall_ms, kernel_ms (device events)}; profiled: (incremental, the pass's [(kernel, ms)], each kernel timed alone)."""
    rows = np.unique(rows).astype(np.uint32)
    t = time.perf_counter()
    eng.commit_pod_values(rows, pod_values(snap, rows))
    if profiled:
        kern = eng.reconcile_profiled(flags)["kernels"]
        return eng.fetch().changed_clusters is not None, kern
    got = eng.reconcile(flags)
    wall = (time.perf_counter() - t) * 1e3
    return {"incremental": got.changed_clusters is not None, "wall_ms": round(wall, 4), "kernel_ms": round(eng.last_profile()["kernels_ms"], 4)}

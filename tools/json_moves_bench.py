"""KR_OPT_JSON_MOVES through the native packer: C3-sized fleet (10 000 RayClusters x 100 Pods, muted specs of about 3.6 KB), fixed
layout, KR_OPT_SPEC_ROWS on, one JSON line per measurement.

Each measured epoch is one in which the packer compacts its JSON arena at flush.  Before it, untimed epochs re-emit the specs of a
few hundred "hot" RayClusters (rows 0..511, a 4 KB note each time) until one more such edit takes the dead bytes past half the arena's
cursor; the measured epoch then applies 10 000 Pod status updates, --k ordinary spec edits and that last hot edit, and times
kr_packer_flush + kr_reconcile_batch (host clock; the pass ends in the synchronising results fetch).  The hot blobs sit at the
arena's start, so the compaction moves almost every RayCluster's blob.  The option is off and on in alternating compaction epochs
of the same session (the packer reads it at each flush).  Reported per option: median / min / max epoch ms, median flush and
reconcile ms, the pass's kernel time, the engine's counted H2D / D2H bytes, the flush mode, whether the pass was incremental and
how many records it re-decided; then, from one separate profiled compaction epoch per option, the move kernels' device time
(torch.profiler) and the pass's kernel list.  The card name and power limit are read in the same run.
Usage: python tools/json_moves_bench.py [--clusters 10000] [--pods 100] [--epochs 5] [--k 10] [--out DIR]"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from benchlib import Recorder  # noqa: E402
from kuberay_b200 import abi  # noqa: E402
from kuberay_b200.packer import Packer  # noqa: E402
from spec_rows_bench import cluster, pod  # noqa: E402

HOT = 512
HOT_NOTE = 4 << 10


def pad(n):
    return (int(n) + 15) // 16 * 16


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clusters", type=int, default=10_000)
    ap.add_argument("--pods", type=int, default=100)
    ap.add_argument("--epochs", type=int, default=5, help="measured compaction epochs per option")
    ap.add_argument("--k", type=int, default=10, help="ordinary spec edits in a measured epoch")
    ap.add_argument("--events", type=int, default=10_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = Recorder("json_moves_bench", a.out, workload=f"{a.clusters} RayClusters x {a.pods} pods through the native packer, compaction epochs")
    Nc, P = a.clusters, a.pods
    pk = Packer(max_clusters=Nc + 16, max_groups=Nc + 16, max_wtd=64, max_pods=Nc * P + 1024, max_heads=Nc + 16, max_jobs=16,
                max_creates=max(1 << 16, Nc * P // 4), max_json_bytes=Nc * 4096 * 4 + 2 * HOT * HOT_NOTE, spec_rows=True)
    rng = np.random.default_rng(1)
    try:
        gen = np.ones(Nc, dtype=np.int64)
        t = time.perf_counter()
        for c in range(Nc):
            pk.upsert_cluster(cluster(c, 1))
        for c in range(Nc):
            for i in range(P):
                pk.upsert_pod(pod(c, i, True))
        running = np.ones((Nc, P), dtype=bool)
        pk.flush()
        flags = pk.flags(fetch_pod_lists=0)
        pk.engine.reconcile(flags)
        lens = pk.column("c_json_len")
        live = lambda: int(((lens[:Nc].astype(np.int64) + 15) // 16 * 16).sum())  # noqa: E731
        cursor = [live()]  # the packer's arena cursor: every blob it places goes there
        out.record({"load_s": round(time.perf_counter() - t, 1), "arena_bytes": cursor[0]})

        def edit(c, extra):
            gen[c] += 1
            pk.upsert_cluster(cluster(c, int(gen[c]), extra))
            cursor[0] += pad(lens[c])

        def compacts_after(extra):
            """Whether one more hot edit of this size makes the next flush compact (dead > cursor / 2 and > 1 MiB)."""
            cur = cursor[0] + pad(len(cluster(0, int(gen[0]) + 1, extra)["specJson"]))
            dead = cur - (live() - pad(lens[0]) + pad(len(cluster(0, int(gen[0]) + 1, extra)["specJson"])))
            return dead * 2 > cur and dead > (1 << 20)

        def flushed(mode):
            if mode & (abi.PACK_JSON_MOVES | abi.PART_JSON):  # compacted: the cursor is the live bytes
                cursor[0] = live()
            return mode

        def prepare():
            """Untimed epochs of hot edits, stopping one edit short of a compaction."""
            h = 0
            while True:
                extra = HOT_NOTE + int(rng.integers(0, 64))
                if compacts_after(extra):
                    break
                edit(h % HOT, extra)
                h += 1
                if h % HOT == 0:
                    flushed(pk.flush())
                    pk.engine.reconcile(flags)
            flushed(pk.flush())
            pk.engine.reconcile(flags)

        def events(k):
            cs, ps = rng.integers(HOT, Nc, a.events), rng.integers(1, P, a.events)
            for c, i in zip(cs.tolist(), ps.tolist()):
                running[c, i] = not running[c, i]
                pk.upsert_pod(pod(c, i, bool(running[c, i])))
            for c in rng.choice(np.arange(HOT, Nc), k, replace=False).tolist() if k else []:
                edit(c, int(rng.integers(0, 2)) * int(rng.integers(1, 64)))
            edit(0, HOT_NOTE)  # (past the threshold: this flush compacts)

        def epoch(on, profile=False):
            prepare()
            pk.engine.set_json_moves(on)
            events(a.k)
            if profile:
                import torch
                from torch.profiler import ProfilerActivity, profile as tprofile
                torch.cuda.synchronize()
                with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
                    mode = flushed(pk.flush())
                    torch.cuda.synchronize()
                moves = [(e.key, e.device_time_total / 1e3) for e in prof.key_averages() if "k_json_move" in e.key]
                kern = pk.engine.reconcile_profiled(flags)["kernels"]
                pk.engine.fetch()
                return mode, moves, kern
            t0 = time.perf_counter()
            mode = flushed(pk.flush())
            t1 = time.perf_counter()
            got = pk.engine.reconcile(flags)
            t2 = time.perf_counter()
            prof = pk.engine.last_profile()
            return mode, ((t2 - t0) * 1e3, (t1 - t0) * 1e3, (t2 - t1) * 1e3, prof["kernels_ms"], prof["h2d_bytes"], prof["d2h_bytes"],
                          int(got.n_changed), got.changed_clusters is not None)

        # alternating compaction epochs (a flush the model above expected to compact but did not is reported and skipped)
        rec, modes, misses, on = {False: [], True: []}, {}, [], False
        warm = {False: 1, True: 1}
        while min(len(rec[False]), len(rec[True])) < a.epochs and len(misses) < 8:
            mode, r = epoch(on)
            if not mode & (abi.PACK_JSON_MOVES | abi.PART_JSON):
                misses.append({"json_moves": on, "flush_mode": mode, "model_cursor": cursor[0], "model_dead": cursor[0] - live()})
                print(json.dumps(misses[-1]), flush=True)
                continue
            if warm[on]:
                warm[on] -= 1
            else:
                modes[on] = mode
                rec[on].append(r)
            on = not on
        assert min(len(rec[False]), len(rec[True])) == a.epochs, misses
        for on in (False, True):
            mode, moves, kern = epoch(on, profile=True)
            r = np.array([x[:6] for x in rec[on]], dtype=np.float64)
            out.record({"json_moves": on, "epochs": a.epochs, "pod_events": a.events, "spec_edits": a.k + 1,
                        "epoch_ms_median": round(float(np.median(r[:, 0])), 4), "epoch_ms_min": round(float(r[:, 0].min()), 4),
                        "epoch_ms_max": round(float(r[:, 0].max()), 4), "flush_ms_median": round(float(np.median(r[:, 1])), 4),
                        "reconcile_ms_median": round(float(np.median(r[:, 2])), 4), "pass_kernels_ms_median": round(float(np.median(r[:, 3])), 4),
                        "h2d_bytes_median": int(np.median(r[:, 4])), "d2h_bytes_median": int(np.median(r[:, 5])),
                        "incremental": int(sum(x[7] for x in rec[on])), "n_changed_median": int(np.median([x[6] for x in rec[on]])),
                        "flush_mode": modes[on], "profiled_flush_mode": mode, "move_kernels_ms": [(n, round(ms, 4)) for n, ms in moves],
                        "profiled_kernels_ms": [(n, round(ms, 4)) for n, ms in kern]})
    finally:
        pk.close()
    out.finish()


if __name__ == "__main__":
    main()

"""KR_OPT_SPEC_ROWS through the native packer: C3-sized fleet (10 000 RayClusters x 100 Pods, muted specs of about 3.6 KB), fixed
layout, one JSON line per measurement.

Every epoch applies 10 000 Pod status updates plus k spec edits (a new generation with a re-emitted spec of the same length or up to
64 bytes longer, as an image or env edit makes it), then times kr_packer_flush + kr_reconcile_batch (host clock; the pass ends in
the synchronising results fetch).  For each k in --ks the option is turned off and on on the same packer in alternating epochs
(the engine reads it at each flush).  Reported per (k, option): median / min / max epoch ms, median flush and reconcile ms, the
engine's counted H2D / D2H bytes of the epoch, the flush mode, and the kernel list with times of one separate profiled epoch.  The
card name and power limit are read in the same run.
Usage: python tools/spec_rows_bench.py [--clusters 10000] [--pods 100] [--epochs 10] [--ks 0,1,10,100,1000] [--out DIR]"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from benchlib import Recorder  # noqa: E402
from kuberay_b200 import snapshot as snp  # noqa: E402
from kuberay_b200.packer import Packer  # noqa: E402


def spec_json(c: int, gen: int, extra: int = 0) -> bytes:
    """About 3.6 KB of muted-spec JSON (the shape json.Marshal gives a RayClusterSpec); gen / extra vary the image and an env value."""
    env = ",".join('{"name":"ENV_%d","value":"value-%06d-%d"}' % (i, c, i) for i in range(60))
    body = ('{"headGroupSpec":{"rayStartParams":{"dashboard-host":"0.0.0.0"},"template":{"spec":{"containers":[{"env":[%s],'
            '"image":"rayproject/ray:2.46.0-%d-g%06d","name":"ray-head","resources":{}}]}}},"rayVersion":"2.46.0","workerGroupSpecs":'
            '[{"groupName":"workers","maxReplicas":200,"minReplicas":0,"rayStartParams":{},"template":{"spec":{"containers":'
            '[{"image":"rayproject/ray:2.46.0","name":"ray-worker","resources":{}}]}},"note":"%s"}]}') % (env, c, gen, "x" * extra)
    return body.encode()


def cluster(c: int, gen: int, extra: int = 0) -> dict:
    return {"namespace": f"ns{c % 50}", "name": f"rc-{c}", "uid": f"uid-{c}", "generation": gen, "resourceVersion": gen,
            "spec": {"workerGroupSpecs": [{"groupName": "workers", "replicas": 99, "minReplicas": 0, "maxReplicas": 200}]},
            "specJson": spec_json(c, gen, extra)}


def pod(c: int, i: int, running: bool) -> dict:
    head = i == 0
    labels = {snp.RAY_CLUSTER_LABEL: f"rc-{c}", snp.RAY_NODE_TYPE_LABEL: "head" if head else "worker"}
    if not head:
        labels[snp.RAY_NODE_GROUP_LABEL] = "workers"
    return {"namespace": f"ns{c % 50}", "name": f"rc-{c}-{i}", "labels": labels, "phase": "Running" if running else "Pending",
            "podIP": f"10.{c // 250}.{c % 250}.{i}" if head else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clusters", type=int, default=10_000)
    ap.add_argument("--pods", type=int, default=100)
    ap.add_argument("--epochs", type=int, default=10, help="timed epochs per (k, option)")
    ap.add_argument("--ks", default="0,1,10,100,1000")
    ap.add_argument("--events", type=int, default=10_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = Recorder("spec_rows_bench", a.out, workload=f"{a.clusters} RayClusters x {a.pods} pods through the native packer")
    Nc, P = a.clusters, a.pods
    pk = Packer(max_clusters=Nc + 16, max_groups=Nc + 16, max_wtd=64, max_pods=Nc * P + 1024, max_heads=Nc + 16, max_jobs=16,
                max_creates=max(1 << 16, Nc * P // 4), max_json_bytes=Nc * 4096 * 3)
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
        out.record({"load_s": round(time.perf_counter() - t, 1)})

        def prepare(k):
            """The epoch's events, handled before the timed window (as the shim's informer handlers do)."""
            cs, ps = rng.integers(0, Nc, a.events), rng.integers(1, P, a.events)
            for c, i in zip(cs.tolist(), ps.tolist()):
                running[c, i] = not running[c, i]
                pk.upsert_pod(pod(c, i, bool(running[c, i])))
            for c in rng.choice(Nc, k, replace=False).tolist() if k else []:
                gen[c] += 1
                pk.upsert_cluster(cluster(c, int(gen[c]), int(rng.integers(0, 2)) * int(rng.integers(1, 64))))

        def epoch(on, k, profiled=False):
            pk.engine.set_spec_rows(on)
            prepare(k)
            t0 = time.perf_counter()
            mode = pk.flush()
            t1 = time.perf_counter()
            if profiled:
                kern = pk.engine.reconcile_profiled(flags)["kernels"]
                pk.engine.fetch()
                return mode, kern
            got = pk.engine.reconcile(flags)
            t2 = time.perf_counter()
            prof = pk.engine.last_profile()
            return mode, ((t2 - t0) * 1e3, (t1 - t0) * 1e3, (t2 - t1) * 1e3, prof["h2d_bytes"], prof["d2h_bytes"],
                          got.changed_clusters is not None)

        for k in [int(x) for x in a.ks.split(",")]:
            for on in (False, True):
                epoch(on, k)  # warm-up of this shape
            rec = {False: [], True: []}
            modes = {}
            for _ in range(a.epochs):
                for on in (False, True):
                    modes[on], r = epoch(on, k)
                    rec[on].append(r)
            for on in (False, True):
                _, kern = epoch(on, k, profiled=True)
                r = np.array([x[:5] for x in rec[on]], dtype=np.float64)
                out.record({"k": k, "spec_rows": on, "epochs": a.epochs, "pod_events": a.events,
                            "epoch_ms_median": round(float(np.median(r[:, 0])), 4), "epoch_ms_min": round(float(r[:, 0].min()), 4),
                            "epoch_ms_max": round(float(r[:, 0].max()), 4), "flush_ms_median": round(float(np.median(r[:, 1])), 4),
                            "reconcile_ms_median": round(float(np.median(r[:, 2])), 4), "h2d_bytes_median": int(np.median(r[:, 3])),
                            "d2h_bytes_median": int(np.median(r[:, 4])), "incremental": int(sum(x[5] for x in rec[on])),
                            "flush_mode": modes[on], "profiled_kernels_ms": [(n, round(ms, 4)) for n, ms in kern]})
    finally:
        pk.close()
    out.finish()


if __name__ == "__main__":
    main()

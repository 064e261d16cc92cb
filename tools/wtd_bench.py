"""KR_OPT_WTD_EDITS on one GPU: the option off and on, alternated, three runs each (one JSON line per measurement).

Workloads: C5 (1 000 autoscaling RayClusters) and C3 with every RayCluster autoscaling.  Each run is a fixed-layout engine, one full
pass, then N epochs of autoscaler-like traffic: 1 % of the groups get 1-3 names of their own running workers with replicas
lowered, the next epoch deletes those Pods and clears the lists, plus 1 % PodReady churn every epoch.  Reported: incremental
epochs out of N, median epoch kernel ms (device events), median epoch wall ms through the C ABI (host clock around the object
commit, the pod commit and kr_reconcile_batch, results copy included), and, option on, the new kernels alone in one profiled
edit epoch.
Usage: python tools/wtd_bench.py [--epochs 20] [--runs 3] [--out DIR]"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from benchlib import OBJ_COLS, POD_COLS, Recorder, alternate, pod_values  # noqa: E402
from kuberay_b200 import abi, synthetic  # noqa: E402
from kuberay_b200.engine import Engine  # noqa: E402
from kuberay_b200.snapshot import Snapshot  # noqa: E402

NEW_KERNELS = ("k_inc_wtd_release", "k_inc_wtd_clear", "k_inc_wtd_insert", "k_inc_wtd_resolve")


def with_lists(snap, cnt, names):
    d = snap.dims
    out = Snapshot(d["clusters"], d["groups"], int(cnt.sum()), d["pods"], d["heads"], d["jobs"], d["json"])
    for name, _dt, _m, dim in abi.COLUMNS:
        if dim != "wtd":
            out.cols[name][:] = snap.cols[name]
    out.g_wtd_cnt[:] = cnt
    out.g_wtd_off[:] = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.uint32)
    out.w_name_id[:] = names
    return out


class Traffic:
    """Autoscaler-like epochs over a snapshot (numpy only, precomputed outside the timed window)."""

    def __init__(self, snap, seed):
        self.rng = np.random.default_rng(seed)
        s = snap
        c_of = {(int(a), int(b)): c for c, (a, b) in enumerate(zip(s.c_ns_id, s.c_name_id))}
        pk = s.p_packed
        worker = (((pk >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER) & (((pk >> abi.PP_PHASE_SHIFT) & 7) == abi.PHASE_RUNNING)
        self.members = {}
        for p in np.flatnonzero(worker):
            c = c_of.get((int(s.p_ns_id[p]), int(s.p_cluster_name_id[p])))
            if c is None:
                continue
            g0, gc = int(s.c_group_off[c]), int(s.c_group_cnt[c])
            for g in range(g0, g0 + gc):
                if s.g_name_id[g] == s.p_group_name_id[p]:
                    self.members.setdefault(g, []).append(int(p))
        self.lists = [s.w_name_id[int(s.g_wtd_off[g]):int(s.g_wtd_off[g] + s.g_wtd_cnt[g])].tolist() for g in range(s.dims["groups"])]
        self.pending = {}

    def epoch(self, s):
        """-> (snapshot of the epoch, pod rows rewritten)."""
        rows = []
        for g, named in self.pending.items():
            self.lists[g] = []
            for c in POD_COLS:
                s.cols[c][named] = 0
            s.p_packed[named] = np.uint32(abi.PP_TOMBSTONE)
            rows += named
            self.members[g] = [p for p in self.members[g] if p not in named]
        self.pending = {}
        G = s.dims["groups"]
        for g in self.rng.choice(G, max(1, G // 100), replace=False):
            g = int(g)
            m = self.members.get(g, [])
            if self.lists[g] or len(m) < 2:
                continue
            named = [int(x) for x in self.rng.choice(m, int(self.rng.integers(1, min(3, len(m)) + 1)), replace=False)]
            self.lists[g] = [int(s.p_name_id[r]) for r in named]
            s.g_replicas[g] = max(0, int(s.g_replicas[g]) - len(named))
            self.pending[g] = named
        live = np.flatnonzero((s.p_packed & abi.PP_TOMBSTONE) == 0)
        flip = self.rng.choice(live, max(1, s.dims["pods"] // 100), replace=False)
        s.p_packed[flip] ^= np.uint32(1 << abi.PP_READY_SHIFT)
        cnt = np.array([len(x) for x in self.lists], dtype=np.uint32)
        names = np.array([x for lst in self.lists for x in lst], dtype=np.uint32)
        return with_lists(s, cnt, names), np.unique(np.array(rows + flip.tolist(), dtype=np.uint32))


def run(name, wtd, epochs, seed):
    snap, flags = synthetic.generate(synthetic.config(name, **({"autoscaling_frac": 1.0} if name == "C3" else {})))
    flags.fetch_pod_lists = 0
    tr = Traffic(snap, seed)
    d = snap.dims
    wtd_cap = d["wtd"] + 3 * max(1, d["groups"] // 100) + 64
    eng = Engine(0, d["clusters"], d["groups"], wtd_cap, d["pods"], d["heads"], d["jobs"], max(1024, d["pods"]), d["json"])
    try:
        eng.set_wtd_edits(wtd)
        eng.set_fixed_layout(True)
        views = eng.load(snap)
        eng.reconcile(flags)
        n_inc, kms, wall, prof, n_wtd = 0, [], [], None, []
        cur = snap
        for i in range(epochs):
            s, rows = tr.epoch(cur)   # (prepared outside the timed window)
            n_wtd.append(s.dims["wtd"])
            t = time.perf_counter()
            if s.dims["wtd"] != cur.dims["wtd"]:
                views = eng.begin(s.sizes())
            for c in OBJ_COLS:
                np.copyto(views[c], s.cols[c])
            eng.commit(abi.PART_OBJECTS)
            eng.commit_pod_values(rows, pod_values(s, rows))
            if wtd and i == epochs - 1:   # the last epoch profiled: the new kernels alone
                prof = dict(eng.reconcile_profiled(flags)["kernels"])
                got = eng.fetch()
            else:
                got = eng.reconcile(flags)
                wall.append((time.perf_counter() - t) * 1e3)
                kms.append(eng.last_profile()["kernels_ms"])
            n_inc += got.changed_clusters is not None
            cur = s
        rec = {"workload": name if name == "C5" else "C3-autoscaling", "wtd_edits": wtd, "incremental_epochs": n_inc, "epochs": epochs,
               "epoch_kernel_ms_median": round(float(np.median(kms)), 4), "epoch_wall_ms_median": round(float(np.median(wall)), 4),
               "n_wtd_range": [min(n_wtd), max(n_wtd)]}
        if prof:
            rec.update({k + "_ms": prof.get(k) for k in NEW_KERNELS})
        return rec
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--workloads", default="C5,C3")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = Recorder("wtd_bench", a.out)
    for name in a.workloads.split(","):
        alternate(a.runs, lambda r, wtd: out.record(dict(run(name, wtd, a.epochs, seed=r + 1), run=r)))
    out.finish()


if __name__ == "__main__":
    main()

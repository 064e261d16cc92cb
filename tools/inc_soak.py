#!/usr/bin/env python
"""Randomised soak of the device-side incremental epochs (development aid; run on the GPU box): many epochs of mixed informer traffic —
status flips, deletions, additions into free rows and past the end of the arena, pods moving between RayClusters and namespaces, head
pods coming and going, RayCluster / group / head-aux row edits through BOTH object-commit entry points, JSON re-commits — each epoch
compared with a from-scratch oracle run; at the end, how many passes were incremental and full and how often each KR_FULL_* cause
sent a pass to the full pass (kr_last_pass).  usage: python tools/inc_soak.py [seeds] [epochs] [--bucket-pod-lists]
--bucket-pod-lists turns on KR_OPT_BUCKET_POD_LISTS and fetches the full pod lists every third epoch, compared with the oracle too."""
import collections
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from kuberay_b200 import abi, synthetic  # noqa: E402
from kuberay_b200.engine import Engine  # noqa: E402
from kuberay_b200.snapshot import Snapshot  # noqa: E402
from oracle import oracle  # noqa: E402

POD_COLS = [name for name, _dt, _m, dim in abi.COLUMNS if dim == "pods"]
OBJ_COLS = [name for name, _dt, _m, dim in abi.COLUMNS if dim not in ("pods", "json")]
HEAD_COLS = [(name, m) for name, _dt, m, dim in abi.COLUMNS if dim == "heads"]


def grow(snap, extra_pods, drop_head=None, add_head_for=None):
    """A new Snapshot with pod rows appended (copies of existing workers) and / or one head-aux row removed / added."""
    d = snap.dims
    nh = d["heads"] - (1 if drop_head is not None else 0) + (1 if add_head_for is not None else 0)
    out = Snapshot(d["clusters"], d["groups"], d["wtd"], d["pods"] + len(extra_pods), nh, d["jobs"], d["json"])
    for name, _dt, m, dim in abi.COLUMNS:
        a = snap.cols[name]
        if dim == "pods" and len(extra_pods):
            a = np.concatenate([a, a[extra_pods]])
        elif dim == "heads":
            a = a.reshape(d["heads"], m) if d["heads"] else a.reshape(0, m)
            if drop_head is not None:
                a = np.delete(a, drop_head, axis=0)
            if add_head_for is not None:
                row = a[0:1].copy() if len(a) else np.zeros((1, m), dtype=a.dtype)
                if name == "h_pod_idx":
                    row[:] = add_head_for
                a = np.concatenate([a, row])
            a = a.reshape(-1)
        out.cols[name][:] = a
    return out


KINDS, CAUSES = collections.Counter(), collections.Counter()


def run(seed, epochs, lists=False):
    rng = np.random.default_rng(seed)
    groups = int(rng.integers(1, 4))
    snap, flags = synthetic.generate(synthetic.config("C2", n_clusters=int(rng.integers(150, 500)), pods_per_cluster=int(rng.integers(8, 40)), groups=groups,
                                                      jobs=bool(rng.integers(2)), recreate_frac=0.08, wtd_group_frac=0.3, seed=1000 + seed))
    flags.fetch_pod_lists = 0
    eng = Engine.for_snapshot(snap, slack=1.6, max_creates=snap.dims["groups"] * 64 + 4096, bucket_pod_lists=lists)
    eng.set_fixed_layout(True)
    views = eng.begin(snap.sizes())
    eng.fill(views, snap)
    eng.commit()
    n_inc = n_full = 0
    free = []
    saved = {}
    for epoch in range(epochs):
        cols = snap.cols
        pk = cols["p_packed"]
        nt = (pk >> abi.PP_NODE_TYPE_SHIFT) & 3
        live = (pk & abi.PP_TOMBSTONE) == 0
        workers = np.nonzero((nt == abi.NT_WORKER) & live)[0]
        touched = []
        cluster_rows, head_rows = set(), set()
        whole_objects = False
        # pod traffic
        for _ in range(int(rng.integers(0, 60))):
            kind = rng.random()
            if kind < 0.55 and len(workers):       # status update
                r = int(rng.choice(workers))
                pk[r] ^= np.uint32(1 << abi.PP_READY_SHIFT) if rng.random() < 0.6 else np.uint32(0)
                if rng.random() < 0.3:
                    pk[r] = (pk[r] & ~np.uint32(7 << abi.PP_PHASE_SHIFT)) | np.uint32(int(rng.integers(1, 6)) << abi.PP_PHASE_SHIFT)
                touched.append(r)
            elif kind < 0.7 and len(workers):      # delete -> free row
                r = int(rng.choice(workers))
                if r in touched or r in free:
                    continue
                saved[r] = {c: cols[c][r].copy() for c in POD_COLS}
                for c in POD_COLS:
                    cols[c][r] = 0
                pk[r] = np.uint32(abi.PP_TOMBSTONE)
                free.append(r); touched.append(r)
            elif kind < 0.85 and free:             # add into a free row (the same pod again, or under another cluster / namespace)
                r = free.pop(int(rng.integers(len(free))))
                for c in POD_COLS:
                    cols[c][r] = saved[r][c]
                if rng.random() < 0.4 and len(workers):
                    donor = int(rng.choice(workers))
                    for c in ("p_ns_id", "p_cluster_name_id", "p_group_name_id"):
                        cols[c][r] = cols[c][donor]
                touched.append(r)
            elif len(workers):                     # a live pod moves to another cluster (labels rewritten)
                r, donor = int(rng.choice(workers)), int(rng.choice(workers))
                for c in ("p_ns_id", "p_cluster_name_id", "p_group_name_id"):
                    cols[c][r] = cols[c][donor]
                touched.append(r)
        # a head pod flips (its aux row keeps its key)
        if snap.dims["heads"] and rng.random() < 0.5:
            h = int(rng.integers(snap.dims["heads"]))
            cols["h_ready_status"][h] = np.uint8(int(rng.integers(0, 4)))
            cols["h_pod_ip_id"][h] = cols["h_pod_ip_id"][int(rng.integers(snap.dims["heads"]))]
            head_rows.add(h)
        # object rows
        for _ in range(int(rng.integers(0, 6))):
            c = int(rng.integers(snap.dims["clusters"]))
            if cols["c_group_cnt"][c]:
                g = int(cols["c_group_off"][c]) + int(rng.integers(int(cols["c_group_cnt"][c])))
                cols["g_replicas"][g] = int(rng.integers(0, 50))
                if rng.random() < 0.3:
                    cols["g_flags"][g] ^= np.uint32(abi.GF_EXPECT_OK)
            if rng.random() < 0.3:
                cols["c_flags"][c] ^= np.uint32(1 << int(rng.choice([0, 2, 3, 5])))   # suspend / autoscaling / Recreate / head expectation
            if rng.random() < 0.3:
                cols["c_old_state"][c] = np.uint8(int(rng.integers(0, 4)))
            cluster_rows.add(c)
        # structural now and then: arena growth, a head row removed / added, a renamed group
        new_snap = None
        if rng.random() < 0.12 and len(workers) > 3:
            extra = rng.choice(workers, 3, replace=False)
            new_snap = grow(snap, extra)
            new_snap.cols["p_name_id"][-3:] = np.uint32(0x70000000 + epoch * 8) + np.arange(3, dtype=np.uint32)
            touched += list(range(snap.dims["pods"], snap.dims["pods"] + 3))
            whole_objects = True
        elif rng.random() < 0.08 and snap.dims["heads"] > 2:
            h = int(rng.integers(snap.dims["heads"]))
            p = int(cols["h_pod_idx"][h])
            if p not in touched:
                for c in POD_COLS:
                    cols[c][p] = 0
                cols["p_packed"][p] = np.uint32(abi.PP_TOMBSTONE)
                touched.append(p)
                new_snap = grow(snap, [], drop_head=h)
                whole_objects = True
        elif rng.random() < 0.05 and snap.dims["groups"]:
            cols["g_name_id"][int(rng.integers(snap.dims["groups"]))] += np.uint32(1 << 20)
            whole_objects = True
        if new_snap is not None:
            snap = new_snap
            views = eng.begin(snap.sizes())
        for c in OBJ_COLS:
            np.copyto(views[c], snap.cols[c])
        if whole_objects or rng.random() < 0.3:
            eng.commit(abi.PART_OBJECTS | (abi.PART_JSON if rng.random() < 0.1 else 0))
        elif cluster_rows or head_rows:
            eng.commit_object_rows(sorted(cluster_rows), sorted(head_rows))
        rows = np.unique(np.asarray(touched, dtype=np.uint32))
        if rows.size:
            for c in POD_COLS:
                views[c][rows] = snap.cols[c][rows]
            if rng.random() < 0.5:
                eng.commit_pod_values(rows, np.stack([snap.cols[c][rows].view(np.uint32) for c in POD_COLS], axis=1))
            else:
                half = rows.size // 2
                eng.commit_pod_rows(rows[:half]) if half else None
                eng.commit_pod_rows(rows[half:])
        flags.fetch_pod_lists = int(lists and epoch % 3 == 0)
        if rng.random() < 0.15:
            eng.reconcile_device_only(flags)
            got = eng.fetch()
        else:
            got = eng.reconcile(flags)
        rep = eng.last_pass()
        KINDS[rep["kind"]] += 1
        CAUSES.update(rep["why"])
        assert (rep["kind"] == "incremental") == (got.changed_clusters is not None or got.n_changed < snap.dims["clusters"]), (seed, epoch, rep)
        want = oracle.run(snap, flags, threads=8)
        d = want.diff(got)
        assert not d, (seed, epoch, d[:5], got.n_changed)
        if got.changed_clusters is not None or got.n_changed < snap.dims["clusters"]:
            n_inc += 1
        else:
            n_full += 1
    eng.close()
    return n_inc, n_full


if __name__ == "__main__":
    lists = "--bucket-pod-lists" in sys.argv
    args = [x for x in sys.argv[1:] if x != "--bucket-pod-lists"]
    seeds = int(args[0]) if len(args) > 0 else 6
    epochs = int(args[1]) if len(args) > 1 else 60
    tot = [0, 0]
    for s in range(seeds):
        a, b = run(s, epochs, lists)
        tot[0] += a; tot[1] += b
        print(f"seed {s}: {a} incremental + {b} full epochs, all equal to the oracle", flush=True)
    print(f"soak ok: {tot[0]} incremental epochs, {tot[1]} full passes", flush=True)
    print(f"passes: {dict(KINDS)}; full-pass causes (KR_FULL_*, a pass may have several): {dict(CAUSES.most_common())}", flush=True)

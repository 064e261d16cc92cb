#!/usr/bin/env python
"""A few small passes over every kernel family, for `compute-sanitizer --tool {memcheck,racecheck,synccheck,initcheck}`
(development aid).  Usage on the GPU box:  compute-sanitizer --tool racecheck python tools/sanitize_run.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from kuberay_b200 import abi, synthetic  # noqa: E402
from kuberay_b200.engine import Engine  # noqa: E402


def one(snap, flags, label):
    eng = Engine.for_snapshot(snap)
    try:
        views = eng.load(snap)
        res = eng.reconcile(flags)
        rows = np.arange(0, snap.dims["pods"], 7, dtype=np.uint32)
        views["p_packed"][rows] ^= np.uint32(1 << 5)
        eng.commit_pod_rows(rows)
        eng.reconcile(flags)
        vals = np.stack([views[c][rows].view(np.uint32) for c, _d, _m, dim in abi.COLUMNS if dim == "pods"], axis=1)
        eng.commit(abi.PART_OBJECTS)
        eng.commit_pod_values(rows, vals)
        res = eng.reconcile(flags)
        print(label, "ok:", res.n_actions, "actions", res.n_create_total, "creates", flush=True)
    finally:
        eng.close()


def pod_lists(snap, flags, label):
    """KR_OPT_BUCKET_POD_LISTS (kr_lists.cuh): one fetching full pass and one fetching incremental pass on the bucket pipeline."""
    flags.fetch_pod_lists = 1
    eng = Engine.for_snapshot(snap, slack=1.2, bucket_pod_lists=True)
    eng.set_fixed_layout(True)
    try:
        views = eng.load(snap)
        eng.reconcile(flags)
        rows = np.arange(0, snap.dims["pods"], 7, dtype=np.uint32)
        views["p_packed"][rows] ^= np.uint32(1 << 5)
        eng.commit_pod_values(rows, np.stack([views[c][rows].view(np.uint32) for c, _d, _m, dim in abi.COLUMNS if dim == "pods"], axis=1))
        res = eng.reconcile(flags)
        print(label, "ok:", eng.last_pass()["kind"], "pass,", res.sorted_pod_idx.size, "Pods listed", flush=True)
    finally:
        eng.close()


def incremental(snap, flags, label, large=False, wide=False, huge=False):
    """Bucket pipeline + device-side incremental epochs (kr_incr.cuh): pod rows, object rows, a structural change, unfetched passes."""
    flags.fetch_pod_lists = 0
    eng = Engine.for_snapshot(snap, slack=1.2, large_clusters=large, wide_clusters=wide, huge_clusters=huge,
                              **({"max_creates": 1 << 16} if large else {}))
    eng.set_fixed_layout(True)
    try:
        views = eng.begin(snap.sizes())
        eng.fill(views, snap)
        eng.commit()
        eng.reconcile(flags)
        pod_cols = [c for c, _d, _m, dim in abi.COLUMNS if dim == "pods"]
        rng = np.random.default_rng(1)
        changed = 0
        for epoch in range(4):
            rows = np.unique(rng.integers(0, snap.dims["pods"], 60)).astype(np.uint32)
            views["p_packed"][rows] ^= np.uint32(1 << 5)
            gone = rows[:5]
            for c in pod_cols:
                views[c][gone] = 0
            views["p_packed"][gone] = np.uint32(abi.PP_TOMBSTONE)
            if snap.dims["groups"]:
                views["g_replicas"][epoch % snap.dims["groups"]] += 1
            eng.commit(abi.PART_OBJECTS)
            if epoch % 2:
                eng.commit_pod_rows(rows)
            else:
                eng.commit_pod_values(rows, np.stack([views[c][rows].view(np.uint32) for c in pod_cols], axis=1))
            if epoch == 2:
                eng.reconcile_device_only(flags)
                res = eng.fetch()
            else:
                res = eng.reconcile(flags)
            changed += int(res.n_changed) if res.changed_clusters is not None else 0
        if snap.dims["groups"]:
            views["g_name_id"][0] += 12345   # a table key: the next pass is a full one
            eng.commit(abi.PART_OBJECTS)
            res = eng.reconcile(flags)
        print(label, "ok:", res.n_actions, "actions;", changed, "records recomputed incrementally", flush=True)
    finally:
        eng.close()


def creations(snap, flags, label):
    """KR_OPT_CLUSTER_CREATES (kr_incr.cuh): the last 20 RayClusters appended under a fixed layout, each time after a full pass over
    the first ones — once with no resident orphan (k_inc_clusters_insert, and k_inc_wtd_resolve for their workersToDelete names), once
    with their Pods resident as orphans (k_inc_orphan_adopt as well)."""
    flags.fetch_pod_lists = 0
    nc, k = snap.dims["clusters"], snap.dims["clusters"] - 20
    # no Pod of the fleet is an orphan to begin with: the Pods no RayCluster of the fleet owns become free rows
    ckey = (snap.c_ns_id.astype(np.uint64) << np.uint64(32)) | snap.c_name_id.astype(np.uint64)
    pkey = (snap.p_ns_id.astype(np.uint64) << np.uint64(32)) | snap.p_cluster_name_id.astype(np.uint64)
    lost = np.flatnonzero(~np.isin(pkey, ckey))
    for c, _d, _m, dim in abi.COLUMNS:
        if dim == "pods":
            snap.cols[c][lost] = 0
    snap.p_packed[lost] = np.uint32(abi.PP_TOMBSTONE)
    inc = 0
    for orphans in (False, True):
        before = synthetic.first_clusters(snap, k, free_pods=not orphans)
        eng = Engine.for_snapshot(snap, slack=1.2, cluster_creates=True)
        eng.set_fixed_layout(True)
        try:
            views = eng.begin(before.sizes())
            eng.fill(views, before)
            eng.commit()
            eng.reconcile(flags)
            views = eng.begin(snap.sizes())
            eng.fill(views, snap)
            eng.commit(abi.PART_OBJECTS)
            eng.commit_spec_rows(np.arange(k, nc, dtype=np.uint32))
            moved = np.flatnonzero(np.any([before.cols[c] != snap.cols[c] for c, _d, _m, dim in abi.COLUMNS if dim == "pods"], axis=0))
            if moved.size:
                eng.commit_pod_rows(moved.astype(np.uint32))
            prof = eng.reconcile_profiled(flags)
            names = [n for n, _ in prof["kernels"]]
            assert ("k_inc_orphan_adopt" in names) == orphans and "k_inc_clusters_insert" in names, names
            inc += eng.fetch().changed_clusters is not None
        finally:
            eng.close()
    print(label, "ok:", inc, "of 2 creation epochs incremental", flush=True)


def deletions(snap, flags, label):
    """KR_OPT_CLUSTER_DELETES (kr_incr.cuh): 12 RayClusters deleted by swap-remove under a fixed layout after a full pass — once with
    no resident orphan before the epoch (k_inc_clusters_release, _translate, _rekey, k_inc_groups_gather, the name table rebuilt,
    k_inc_clusters_insert for the moved ones), once with orphans resident and RayClusters created in the same epoch (with
    KR_OPT_CLUSTER_CREATES: k_inc_orphan_adopt as well)."""
    flags.fetch_pod_lists = 0
    nc = snap.dims["clusters"]
    inc = 0
    for orphans in (False, True):
        k = nc - 8 if orphans else nc
        before = synthetic.select_clusters(snap, np.arange(k))
        if not orphans:  # no Pod of the fleet is an orphan to begin with: the Pods no RayCluster owns become free rows
            ckey = (snap.c_ns_id.astype(np.uint64) << np.uint64(32)) | snap.c_name_id.astype(np.uint64)
            pkey = (snap.p_ns_id.astype(np.uint64) << np.uint64(32)) | snap.p_cluster_name_id.astype(np.uint64)
            lost = np.flatnonzero(~np.isin(pkey, ckey))
            for c, _d, _m, dim in abi.COLUMNS:
                if dim == "pods":
                    before.cols[c][lost] = 0
            before.p_packed[lost] = np.uint32(abi.PP_TOMBSTONE)
        order = synthetic.swap_remove_order(k, np.arange(3, 3 + 12 * 7, 7))
        after = synthetic.select_clusters(before, order)
        if orphans:  # ... and the 8 RayClusters past the first k created after the last row
            after = synthetic.select_clusters(snap, np.concatenate([order, np.arange(k, nc)]))
        eng = Engine.for_snapshot(snap, slack=1.2, cluster_deletes=True, cluster_creates=orphans)
        eng.set_fixed_layout(True)
        try:
            views = eng.begin(before.sizes())
            eng.fill(views, before)
            eng.commit()
            eng.reconcile(flags)
            views = eng.begin(after.sizes())
            for c, _d, _m, dim in abi.COLUMNS:
                if dim not in ("pods", "json"):
                    np.copyto(views[c], after.cols[c])
            eng.commit(abi.PART_OBJECTS)
            if orphans:
                eng.commit_spec_rows(np.arange(order.size, after.dims["clusters"], dtype=np.uint32))
            prof = eng.reconcile_profiled(flags)
            names = [n for n, _ in prof["kernels"]]
            assert "k_inc_clusters_release" in names and ("k_inc_orphan_adopt" in names) == orphans, names
            got = eng.fetch()
            inc += got.changed_clusters is not None or got.n_changed < after.dims["clusters"]
        finally:
            eng.close()
    print(label, "ok:", inc, "of 2 deletion epochs incremental", flush=True)


def group_edits(snap, flags, label):
    """KR_OPT_GROUP_EDITS (kr_incr.cuh): a worker group appended to RayCluster 40 whose resident Pods are already labelled for it,
    then its first group removed while its Pods live on — each epoch releases the RayCluster, rekeys the table, gathers the shifted
    group records and initialises it again in its row."""
    flags.fetch_pod_lists = 0
    c = 40
    w = np.flatnonzero((snap.p_ns_id == snap.c_ns_id[c]) & (snap.p_cluster_name_id == snap.c_name_id[c]) &
                       (((snap.p_packed >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER))[:4]
    fresh = int(max(snap.g_name_id.max(), snap.p_group_name_id.max(), snap.p_name_id.max(), snap.c_name_id.max())) + 1
    snap.p_group_name_id[w] = fresh
    eng = Engine.for_snapshot(snap, slack=1.5, group_edits=True)
    eng.set_fixed_layout(True)
    inc = 0
    try:
        views = eng.load(snap)
        eng.reconcile(flags)
        g0, cur = int(snap.c_group_off[c]), snap
        for pairs in ([(g, None) for g in range(g0, g0 + int(snap.c_group_cnt[c]))] + [(g0, fresh)], None):
            if pairs is None:  # the first group removed
                g0 = int(cur.c_group_off[c])
                pairs = [(g, None) for g in range(g0 + 1, g0 + int(cur.c_group_cnt[c]))]
            cur = synthetic.regroup_clusters(cur, {c: pairs})
            views = eng.begin(cur.sizes())
            for col, _d, _m, dim in abi.COLUMNS:
                if dim not in ("pods", "json"):
                    np.copyto(views[col], cur.cols[col])
            eng.commit(abi.PART_OBJECTS)
            names = [n for n, _ in eng.reconcile_profiled(flags)["kernels"]]
            assert "k_inc_clusters_release" in names and "k_inc_clusters_insert" in names, names
            got = eng.fetch()
            inc += got.changed_clusters is not None
    finally:
        eng.close()
    print(label, "ok:", inc, "of 2 group-edit epochs incremental", flush=True)


def large_growth(snap, flags, label):
    """KR_OPT_LARGE_GROWTH (kr_incr.cuh, kr_large.cuh): RayCluster 40 outgrows its bucket (a promotion: k_inc_admit spills the
    records past the stride, k_inc_grow gives it a region and places them, the per-cluster kernels take it past their list), then its
    region (a regrowth: the old region copied into a new one)."""
    flags.fetch_pod_lists = 0
    eng = Engine.for_snapshot(snap, large_clusters=True, large_growth=True)
    eng.set_fixed_layout(True)
    inc = 0
    try:
        eng.load(snap)
        eng.reconcile(flags)
        for rows in synthetic.grow_epochs(snap, [40], [eng.get_option(abi.OPT_BUCKET_STRIDE) + 8, 300]):
            rows = rows.astype(np.uint32)
            cols = [c for c, _d, _m, dim in abi.COLUMNS if dim == "pods"]
            eng.commit_pod_values(rows, np.stack([snap.cols[c][rows].view(np.uint32) for c in cols], axis=1))
            names = [n for n, _ in eng.reconcile_profiled(flags)["kernels"]]
            assert "k_inc_grow" in names and "k_decide_large" in names, names
            inc += eng.fetch().changed_clusters is not None
    finally:
        eng.close()
    print(label, "ok:", inc, "of 2 growth epochs incremental", flush=True)


def block_decides(snap, flags, label):
    """The block decide (kr_decide.cuh: decide_cluster_block) in both of its launches: k_decide_large for a large RayCluster and
    k_decide_huge for a huge one, in a full pass, then in an incremental epoch that flips Pods of both."""
    flags.fetch_pod_lists = 0
    synthetic.grow_clusters(snap, [0], 9000)
    synthetic.grow_clusters(snap, [400], 1500)
    eng = Engine.for_snapshot(snap, slack=1.2, max_creates=1 << 18, large_clusters=True, huge_clusters=True)
    eng.set_fixed_layout(True)
    inc = 0
    try:
        eng.load(snap)
        for epoch in range(2):
            if epoch:
                key = lambda c: (snap.p_ns_id == snap.c_ns_id[c]) & (snap.p_cluster_name_id == snap.c_name_id[c])  # noqa: E731
                rows = np.concatenate([np.flatnonzero(key(0))[::53], np.flatnonzero(key(400))[::29]]).astype(np.uint32)
                snap.p_packed[rows] ^= np.uint32(1 << abi.PP_READY_SHIFT)
                cols = [c for c, _d, _m, dim in abi.COLUMNS if dim == "pods"]
                eng.commit_pod_values(rows, np.stack([snap.cols[c][rows].view(np.uint32) for c in cols], axis=1))
            names = [n for n, _ in eng.reconcile_profiled(flags)["kernels"]]
            assert "k_decide_large" in names and "k_decide_huge" in names, names
            inc += eng.fetch().changed_clusters is not None
    finally:
        eng.close()
    print(label, "ok:", inc, "of 1 epoch incremental", flush=True)


def large_moves(snap, flags, label, grown, edits, huge=False):
    """KR_OPT_LARGE_MOVES (kr_incr.cuh): the RayClusters `grown` made large, then each edit of `edits` in an epoch of its own: ("delete",
    rows) by swap-remove, or ("regroup", row) a worker group appended.  A large gone row is released by k_inc_large_release from its
    old region while the table is in the new numbering, and a moved or regrouped one's region goes back into the table behind
    k_inc_clusters_insert (k_inc_large_carry)."""
    flags.fetch_pod_lists = 0
    synthetic.grow_clusters(snap, grown, 9000 if huge else 600)
    eng = Engine.for_snapshot(snap, slack=1.25, large_clusters=True, huge_clusters=huge, cluster_deletes=True, group_edits=True, large_moves=True)
    eng.set_fixed_layout(True)
    inc = 0
    try:
        views = eng.load(snap)
        eng.reconcile(flags)
        eng.reconcile(flags)
        eng.commit(abi.PART_OBJECTS)  # (records the group names for the regroup)
        eng.reconcile(flags)
        for kind, arg in edits:
            if kind == "delete":
                snap = synthetic.delete_clusters(snap, arg)
            else:
                g0 = int(snap.c_group_off[arg])
                groups = [(g, None) for g in range(g0, g0 + int(snap.c_group_cnt[arg]))]
                snap = synthetic.regroup_clusters(snap, {arg: groups + [(g0, int(snap.g_name_id.max()) + 1)]})
            views = eng.begin(snap.sizes())
            for c, _dt, _m, dim in abi.COLUMNS:
                if dim not in ("pods", "json"):
                    np.copyto(views[c], snap.cols[c])
            eng.commit(abi.PART_OBJECTS)
            names = [n for n, _ in eng.reconcile_profiled(flags)["kernels"]]
            assert "k_inc_large_release" in names, names
            inc += eng.fetch().changed_clusters is not None
    finally:
        eng.close()
    print(label, "ok:", inc, f"of {len(edits)} epochs incremental", flush=True)


def huge_growth(snap, flags, label, grown, size, steps, move=False):
    """KR_OPT_HUGE_GROWTH (kr_large.cuh, kr_huge.cuh): RayCluster `grown` (made `size` Pods) scales to each of `steps` in an epoch of
    its own: past KR_LARGE_MAX_PODS (k_inc_grow<true> appends its tiles to the reserve entries, k_large_sort passes it over), or past
    a huge one's region (its resident tiles retired, its old region copied by the whole launch).  move: first an ordinary RayCluster
    deleted by swap-remove, so that the huge last row moves into its hole, carrying its tiles, and grows in the same epoch."""
    flags.fetch_pod_lists = 0
    synthetic.grow_clusters(snap, [grown], size)
    eng = Engine.for_snapshot(snap, slack=1.25, max_creates=1 << 18, large_clusters=True, huge_clusters=True, large_growth=True,
                              huge_growth=True, cluster_deletes=move, large_moves=move)
    eng.set_fixed_layout(True)
    cols = [c for c, _d, _m, dim in abi.COLUMNS if dim == "pods"]
    inc = 0
    try:
        views = eng.load(snap)
        eng.reconcile(flags)
        eng.reconcile(flags)
        if move:
            snap = synthetic.delete_clusters(snap, [12])
            views = eng.begin(snap.sizes())
            for c, _dt, _m, dim in abi.COLUMNS:
                if dim not in ("pods", "json"):
                    np.copyto(views[c], snap.cols[c])
            eng.commit(abi.PART_OBJECTS)
            grown = 12
        for rows in synthetic.grow_epochs(snap, [grown], steps):
            rows = rows.astype(np.uint32)
            eng.commit_pod_values(rows, np.stack([snap.cols[c][rows].view(np.uint32) for c in cols], axis=1))
            names = [n for n, _ in eng.reconcile_profiled(flags)["kernels"]]
            assert "k_inc_grow" in names and "k_huge_tiles" in names, names
            inc += eng.fetch().changed_clusters is not None
    finally:
        eng.close()
    print(label, "ok:", inc, f"of {len(steps)} growth epochs incremental", flush=True)


def wtd_edits(snap, flags, label):
    """KR_OPT_WTD_EDITS (kr_incr.cuh): workersToDelete renames, a list grown past the old n_wtd, then every list cleared — each epoch
    rebuilds the name table on the device (k_inc_wtd_release / _clear / _insert / _resolve)."""
    flags.fetch_pod_lists = 0
    d = snap.dims
    eng = Engine(0, d["clusters"], d["groups"], d["wtd"] + 64, d["pods"], d["heads"], d["jobs"], max(1024, d["pods"]), d["json"])
    eng.set_wtd_edits(True)
    eng.set_fixed_layout(True)
    try:
        views = eng.load(snap)
        eng.reconcile(flags)
        inc = 0
        names = views["p_name_id"][::97][:8].copy()
        for step in range(3):
            w = d["wtd"] + (4 if step == 1 else 0) if step < 2 else 0
            cnt = np.zeros(d["groups"], dtype=np.uint32)
            if w:
                cnt[:] = snap.g_wtd_cnt
                cnt[0] += w - d["wtd"]
            s2 = synthetic.Snapshot(d["clusters"], d["groups"], w, d["pods"], d["heads"], d["jobs"], d["json"])
            for c, _dt, _m, dim in abi.COLUMNS:
                if dim not in ("wtd", "json"):
                    s2.cols[c][:] = views[c]
            s2.g_wtd_cnt[:] = cnt
            s2.g_wtd_off[:] = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.uint32)
            s2.w_name_id[:] = np.resize(names, w) if w else 0
            views = eng.begin(s2.sizes())
            for c, _dt, _m, dim in abi.COLUMNS:
                if dim not in ("pods", "json"):
                    np.copyto(views[c], s2.cols[c])
            eng.commit(abi.PART_OBJECTS)
            inc += eng.reconcile(flags).changed_clusters is not None
        print(label, "ok:", inc, "of 3 epochs incremental", flush=True)
    finally:
        eng.close()


def spec_rows(snap, flags, label):
    """kr_snapshot_commit_spec_rows (kr_incr.cuh): specs rewritten in place and moved to the arena's end, pulled by k_spec_pull, then
    re-hashed over the row list, the listed Recreate gates marked (k_inc_mark_rows) and the digests gathered (k_inc_digest_gather)."""
    flags.fetch_pod_lists = 0
    d = snap.dims
    eng = Engine(0, d["clusters"], d["groups"], d["wtd"], d["pods"], d["heads"], d["jobs"], max(1024, d["pods"]), d["json"] + (1 << 20))
    eng.set_fixed_layout(True)
    try:
        views = eng.load(snap)
        eng.reconcile(flags)
        inc, end = 0, d["json"]
        for step in range(3):
            rows = np.arange(step, d["clusters"], 7, dtype=np.uint32)
            if step == 1:  # moved: every listed spec one byte longer at the arena's end
                s2 = synthetic.Snapshot(d["clusters"], d["groups"], d["wtd"], d["pods"], d["heads"], d["jobs"], end + 16 * (rows.size + 1) + int(views["c_json_len"][rows].sum()))
                views = eng.begin(s2.sizes())
                for c in rows.tolist():
                    o, n = int(views["c_json_off"][c]), int(views["c_json_len"][c])
                    views["json"][end:end + n] = views["json"][o:o + n]
                    views["json"][end + n:end + (n + 16) // 16 * 16] = 32
                    views["c_json_off"][c], views["c_json_len"][c] = end, n + 1
                    end += (n + 16) // 16 * 16
            else:  # in place: one byte rewritten
                for c in rows.tolist():
                    views["json"][int(views["c_json_off"][c])] ^= 1
            eng.commit_spec_rows(rows)
            inc += eng.reconcile(flags).changed_clusters is not None
        print(label, "ok:", inc, "of 3 epochs incremental", flush=True)
    finally:
        eng.close()


def main():
    deletions(*synthetic.generate(synthetic.config("C2", n_clusters=300, pods_per_cluster=20, groups=2, wtd_group_frac=0.3, recreate_frac=0.3)),
              "RayCluster deletions")
    creations(*synthetic.generate(synthetic.config("C2", n_clusters=300, pods_per_cluster=20, groups=2, wtd_group_frac=0.3, recreate_frac=0.3)),
              "RayCluster creations")
    group_edits(*synthetic.generate(synthetic.config("C2", n_clusters=300, pods_per_cluster=20, groups=2, wtd_group_frac=0.3, recreate_frac=0.3)),
                "worker-group edits")
    large_growth(*synthetic.generate(synthetic.config("C2", n_clusters=300, pods_per_cluster=20, groups=2, wtd_group_frac=0.3, recreate_frac=0.3)),
                 "RayClusters outgrowing their bucket and region")
    large_moves(*synthetic.generate(synthetic.config("C2", n_clusters=300, pods_per_cluster=20, groups=2, wtd_group_frac=0.3, recreate_frac=0.3)),
                "large RayCluster deleted in a middle row, a large one moving into it", [120, 299], [("delete", [120])])
    large_moves(*synthetic.generate(synthetic.config("C2", n_clusters=300, pods_per_cluster=20, groups=2, wtd_group_frac=0.3, recreate_frac=0.3)),
                "large RayCluster regrouped", [150], [("regroup", 150)])
    large_moves(*synthetic.generate(synthetic.config("C2", n_clusters=800, pods_per_cluster=20, groups=2)),
                "huge RayCluster moved, then deleted", [799], [("delete", [10]), ("delete", [10])], huge=True)
    huge_growth(*synthetic.generate(synthetic.config("C2", n_clusters=1300, pods_per_cluster=20, groups=2)),
                "large RayCluster crossing 8 192 Pods", 600, 8000, [8300])
    huge_growth(*synthetic.generate(synthetic.config("C2", n_clusters=1300, pods_per_cluster=20, groups=2)),
                "huge RayCluster outgrowing its region", 600, 9000, [11400])
    huge_growth(*synthetic.generate(synthetic.config("C2", n_clusters=1400, pods_per_cluster=16, groups=2)),
                "huge RayCluster moved by swap-remove and grown", 1399, 9000, [11400], move=True)
    spec_rows(*synthetic.generate(synthetic.config("C2", n_clusters=300, pods_per_cluster=20, groups=2, recreate_frac=0.3)), "spec rows")
    wtd_edits(*synthetic.generate(synthetic.config("C2", n_clusters=300, pods_per_cluster=20, groups=2, autoscaling_frac=1.0, wtd_group_frac=0.3)),
              "workersToDelete edits")
    incremental(*synthetic.generate(synthetic.config("C2", n_clusters=300, pods_per_cluster=20, groups=2, jobs=True, wtd_group_frac=0.3)), "incremental epochs")
    pod_lists(*synthetic.generate(synthetic.config("C2", n_clusters=300, pods_per_cluster=20, groups=2, wtd_group_frac=0.3, orphan_frac=0.02)),
              "pod lists on the bucket pipeline")
    incremental(*synthetic.generate(synthetic.config("C2", n_clusters=300, pods_per_cluster=41, groups=2, wtd_group_frac=0.3, multihost_frac=0.5)),
                "incremental epochs, multi-host groups")
    # large RayClusters in their own regions (KR_OPT_LARGE_CLUSTERS, kr_large.cuh): a full pass, then incremental epochs
    incremental(*synthetic.generate(synthetic.config("C3L", n_clusters=300, pods_per_cluster=20, large_pods=1200, n_large=3)),
                "incremental epochs, large RayClusters", large=True)
    # RayClusters of 48 worker groups decided one CTA each (KR_OPT_WIDE_CLUSTERS, kr_large.cuh): a full pass, then incremental epochs
    incremental(*synthetic.generate(synthetic.config("C3W", n_clusters=300, pods_per_cluster=60, n_wide=6)),
                "incremental epochs, wide RayClusters", wide=True)
    # a RayCluster of more than KR_LARGE_MAX_PODS pods sorted tile by tile (KR_OPT_HUGE_CLUSTERS, kr_huge.cuh): a full pass, then
    # incremental epochs (the deletions compact its bucket and region across tiles)
    incremental(*synthetic.generate(synthetic.config("C3H", n_clusters=700, pods_per_cluster=20, large_pods=9000, n_large=1)),
                "incremental epochs, huge RayCluster", large=True, huge=True)
    # a large and a huge RayCluster decided by every warp of their CTA (kr_decide.cuh: decide_cluster_block), full pass and epoch
    block_decides(*synthetic.generate(synthetic.config("C2", n_clusters=1200, pods_per_cluster=20, groups=2)), "block decides, large and huge")
    # keys built to collide (tests/table_keys.py): probe chains that start in the last slot of the cluster, workersToDelete and
    # head-aux tables and wrap, in a full pass and in incremental epochs
    from table_keys import k1, k2, k3
    for name, k in (("K1", k1()), ("K2", k2()), ("K3", k3())):
        incremental(k.snap, k.kflags, f"incremental epochs, colliding keys {name}", large=True, wide=True, huge=True)
    one(*synthetic.generate(synthetic.config("C2", n_clusters=200, jobs=True)), "fast pipeline")
    one(*synthetic.generate(synthetic.SynthParams(n_clusters=60, pods_per_cluster=41, groups=2, multihost_frac=0.5)), "multi-host")
    one(*synthetic.generate(synthetic.SynthParams(n_clusters=20, pods_per_cluster=200, groups=40)), "many groups")
    one(*synthetic.generate(synthetic.SynthParams(n_clusters=3, pods_per_cluster=1500, groups=2)), "big bucket -> radix")
    os.environ["KR_NO_FUSE"] = "1"
    one(*synthetic.generate(synthetic.config("C2", n_clusters=200)), "unfused scans")
    import fuzz_objects
    for seed in range(6):
        snap, flags = fuzz_objects.snapshot(seed, big=True)
        one(snap, flags, f"fuzz {seed}")
    eng = Engine(0, 1, 1, 1, 1, 1, 1, 16, 4096)
    msgs = [bytes([65 + i % 26]) * n for i, n in enumerate((0, 1, 55, 56, 63, 64, 65, 119, 120, 128, 1000, 4097))]
    print("hash_batch", len(eng.hash_batch(msgs)), flush=True)
    # above the throughput threshold ((n + 31) / 32 > 4 x SMs, kr_engine.cu) the engine hashes with k_hash2<4, 1>
    import torch
    n = 128 * torch.cuda.get_device_properties(0).multi_processor_count + 500
    msgs = [bytes([65 + i % 26]) * (i % 300) for i in range(n)]
    print("hash_batch, throughput regime", len(eng.hash_batch(msgs)), flush=True)
    eng.close()
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=n, pods_per_cluster=2, groups=1, recreate_frac=0.3))
    flags.fetch_pod_lists = 0   # bucket pipeline: the Recreate-gate warps wait for k_hash2's digests inside k_decide2
    one(snap, flags, "throughput-regime hash with Recreate gates")


if __name__ == "__main__":
    main()

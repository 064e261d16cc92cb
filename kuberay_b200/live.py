"""Incrementally maintained arena: the host-side mirror of what the shim's informer handlers do between epochs.

SURVEY §8(f) rank 1.  The device keeps the last snapshot; an epoch uploads only what changed:
  * Pod Add / Update / Delete events rewrite single rows of the seven per-pod columns (a deleted Pod's row becomes a
    KR_PP_TOMBSTONE row, an added Pod takes the lowest free row) -> kr_snapshot_commit_pod_rows(rows);
  * RayCluster / worker-group / workersToDelete / head-aux / RayJob rows are small -> kr_snapshot_commit_parts(KR_PART_OBJECTS);
  * spec changes -> KR_PART_JSON as well.
The engine runs with KR_OPT_FIXED_LAYOUT (arenas laid out for the capacities), so a change that moves a table's row count —
a RayCluster or a head Pod appears / disappears, the workersToDelete lists change length, a Pod is appended after the last
row — is still incremental: kr_snapshot_begin(new live counts) keeps every column where it is.  Only outgrowing a capacity
takes the full path ("rebase": a larger engine, everything uploaded).

This class re-packs the objects on the host with the ordinary packer and diffs the columns: it is the executable
statement of the protocol for the tests, not a fast packer (that is the Go shim's job).
"""
from __future__ import annotations

import heapq

import numpy as np

from . import abi
from . import snapshot as snp
from .engine import Engine

_POD_COLS = [name for name, _dt, _m, dim in abi.COLUMNS if dim == "pods"]
_OBJ_COLS = [name for name, _dt, _m, dim in abi.COLUMNS if dim not in ("pods", "json")]


def _is_head(pod: dict) -> bool:
    return (pod.get("labels") or {}).get(snp.RAY_NODE_TYPE_LABEL) == "head"


class LiveArena:
    def __init__(self, clusters: list[dict], pods: list[dict], jobs: list[dict] | None = None, spare_rows: int = 64, device: int = 0,
                 engine: bool = True, large_clusters: bool = False, wide_clusters: bool = False, huge_clusters: bool = False,
                 wtd_edits: bool = False, spec_rows: bool = False):
        self.clusters = {(c.get("namespace", "default"), c["name"]): c for c in clusters}
        self.jobs = list(jobs or [])
        self.rows: list[dict | None] = list(pods) + [None] * spare_rows
        self.interner = snp.Interner()
        self.device = device
        self.use_engine = engine
        self.large_clusters = large_clusters  # KR_OPT_LARGE_CLUSTERS on every engine this arena creates
        self.wide_clusters = wide_clusters    # ... and KR_OPT_WIDE_CLUSTERS
        self.huge_clusters = huge_clusters    # ... and KR_OPT_HUGE_CLUSTERS
        self.wtd_edits = wtd_edits            # ... and KR_OPT_WTD_EDITS
        self.spec_rows = spec_rows            # ... and KR_OPT_SPEC_ROWS: changed specs travel as kr_snapshot_commit_spec_rows
        self.engine: Engine | None = None
        self.stats = {"rebase": 0, "incremental": 0, "rows": 0}
        self._need_rebase = True
        self._dirty: set[int] = set()
        self._index()

    # ------------------------------------------------------------------ events
    def _index(self):
        self.row_of = {(p.get("namespace", "default"), p["name"]): i for i, p in enumerate(self.rows) if p is not None}
        self.free = [i for i, p in enumerate(self.rows) if p is None]
        heapq.heapify(self.free)

    def upsert_pod(self, pod: dict):
        key = (pod.get("namespace", "default"), pod["name"])
        row = self.row_of.get(key)
        if row is None:
            if not self.free:  # no free row: append after the last one (a new live count, still no layout change)
                self.rows.append(None)
                heapq.heappush(self.free, len(self.rows) - 1)
            row = heapq.heappop(self.free)
            self.row_of[key] = row
        self.rows[row] = pod
        self._dirty.add(row)

    def delete_pod(self, namespace: str, name: str) -> bool:
        row = self.row_of.pop((namespace, name), None)
        if row is None:
            return False
        self.rows[row] = None
        heapq.heappush(self.free, row)
        self._dirty.add(row)
        return True

    def upsert_cluster(self, cluster: dict):
        key = (cluster.get("namespace", "default"), cluster["name"])
        self.clusters[key] = cluster

    def delete_cluster(self, namespace: str, name: str):
        self.clusters.pop((namespace, name), None)

    # ------------------------------------------------------------------ epoch
    def pack(self) -> tuple[snp.Snapshot, snp.PackMeta]:
        pods = [p if p is not None else snp.TOMBSTONE for p in self.rows]
        return snp.pack_objects([self.clusters[k] for k in sorted(self.clusters)], pods, self.jobs, interner=self.interner)

    def fresh_pack(self) -> tuple[snp.Snapshot, snp.PackMeta]:
        """The same objects packed from scratch without free rows (same relative List order): the semantic reference."""
        pods = [p for p in self.rows if p is not None]
        return snp.pack_objects([self.clusters[k] for k in sorted(self.clusters)], pods, self.jobs, interner=self.interner)  # same ids

    def flush(self) -> str:
        """Bring the device copy up to date; returns "rebase" or "incremental"."""
        snap, meta = self.pack()
        if not self.use_engine:
            mode = "incremental" if (not self._need_rebase and getattr(self, "snap", None) is not None) else "rebase"
        elif self._need_rebase or self.engine is None or not self._fits(snap):
            # first epoch, or a table outgrew the capacities: new engine sized with slack, fixed layout, full upload
            if self.engine is not None:
                self.engine.close()
            self.engine = Engine.for_snapshot(snap, device=self.device, slack=1.5, large_clusters=self.large_clusters,
                                              wide_clusters=self.wide_clusters, huge_clusters=self.huge_clusters,
                                              wtd_edits=self.wtd_edits, spec_rows=self.spec_rows)
            self.engine.set_fixed_layout(True)
            self.views = self.engine.begin(snap.sizes())
            self.engine.fill(self.views, snap)
            self.engine.commit()
            mode = "rebase"
        else:
            # Under the fixed layout every column keeps its address, so any event is incremental: new live counts, the small
            # object columns, the spec JSON if it moved, and the pod rows the events touched (appended rows included).
            old_pods = self.snap.dims["pods"]
            if bytes(snap.sizes()) != bytes(self.snap.sizes()):
                self.views = self.engine.begin(snap.sizes())
            parts = 0
            if not np.array_equal(self.views["json"], snap.cols["json"]):
                if self.spec_rows and snap.dims["clusters"] == self.snap.dims["clusters"]:
                    # every RayCluster whose range or bytes differ (a repack moves every range after a length change), committed
                    # before the object part so that it finds the ranges where the digests say they are
                    rows = self._spec_rows_changed(snap)
                    np.copyto(self.views["json"], snap.cols["json"])
                    self.views["c_json_off"][rows] = snap.cols["c_json_off"][rows]
                    self.views["c_json_len"][rows] = snap.cols["c_json_len"][rows]
                    self.engine.commit_spec_rows(rows)
                else:
                    np.copyto(self.views["json"], snap.cols["json"])
                    parts |= abi.PART_JSON
            if any(not np.array_equal(self.views[c], snap.cols[c]) for c in _OBJ_COLS):
                for c in _OBJ_COLS:
                    np.copyto(self.views[c], snap.cols[c])
                parts |= abi.PART_OBJECTS
            if parts:
                self.engine.commit(parts)
            self._dirty.update(range(old_pods, snap.dims["pods"]))  # rows appended past the old end of the arena
            rows = np.array(sorted(r for r in self._dirty if r < snap.dims["pods"]), dtype=np.uint32)
            for c in _POD_COLS:
                self.views[c][rows] = snap.cols[c][rows]
            for c in _POD_COLS:  # every row that was not reported dirty must already be identical
                assert np.array_equal(self.views[c], snap.cols[c]), c
            self._epoch = getattr(self, "_epoch", 0) + 1
            if rows.size and self._epoch % 2:  # journal style: hand the rows over
                self.engine.commit_pod_values(rows, np.stack([snap.cols[c][rows].view(np.uint32) for c in _POD_COLS], axis=1))
            elif rows.size:                     # or let the device pull them from the arenas
                self.engine.commit_pod_rows(rows)
            self.stats["rows"] += int(rows.size)
            mode = "incremental"
        self.snap, self.meta = snap, meta
        self._need_rebase = False
        self._dirty.clear()
        self.stats[mode] += 1
        return mode

    def _spec_rows_changed(self, snap) -> np.ndarray:
        old, new = self.snap.cols, snap.cols
        moved = (old["c_json_off"] != new["c_json_off"]) | (old["c_json_len"] != new["c_json_len"])
        for c in np.flatnonzero(~moved):
            o, n = int(new["c_json_off"][c]), int(new["c_json_len"][c])
            moved[c] = not np.array_equal(old["json"][o:o + n], new["json"][o:o + n])
        return np.flatnonzero(moved).astype(np.uint32)

    def _fits(self, snap) -> bool:
        d, c = snap.dims, self.engine.cfg
        return (d["clusters"] <= c.max_clusters and d["groups"] <= c.max_groups and d["wtd"] <= c.max_wtd and d["pods"] <= c.max_pods and
                d["heads"] <= c.max_heads and d["jobs"] <= c.max_jobs and d["json"] <= c.max_json_bytes)

    def reconcile(self, flags: abi.kr_flags | None = None) -> abi.Results:
        return self.engine.reconcile(flags or self.meta.flags)

    def close(self):
        if self.engine is not None:
            self.engine.close()
            self.engine = None

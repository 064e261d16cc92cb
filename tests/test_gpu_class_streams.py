"""Randomised epoch streams that move RayClusters across every class boundary of the bucket pipeline, with KR_OPT_LARGE_CLUSTERS
and KR_OPT_WIDE_CLUSTERS on (kuberay_b200/csrc/kr_large.cuh, kr_incr.cuh).

A fleet of several hundred ordinary RayClusters carries large ones (a few hundred, a few thousand and close to 8 192 pods), wide
ones (33 to 100 worker groups, some 70 of them), one that is both, multi-host groups, Recreate gates and workersToDelete lists.
Every epoch mixes informer traffic with moves that push clusters across the strides, 256 / 257 pods, their region's capacity,
8 192 / 8 193 pods and 32 / 33 worker groups, and back; every epoch is compared with a from-scratch oracle run and the records the
pass did not name must be unchanged.

A host model of the engine's classification (Model) predicts the stride, the regions and the list of the per-cluster kernels, and
which epochs must be incremental: the ones that change no structural input and in which no cluster's records outgrow what its
bucket and region hold, nor the action list / create arena what their reservations hold."""
import collections
import json

import numpy as np
import pytest

from class_model import Model
from class_model import counts as _counts
from class_model import owners as _owners
from harness import OBJ_COLS, SORT_KERNELS, Driver, b32, head_row, incremental, scale_to, set_phase, spec_bytes, workers
from kuberay_b200 import abi, synthetic

pytestmark = pytest.mark.gpu


class Stream(Driver):
    """One seeded stream: the fleet, the epoch generators and the per-epoch checks."""

    def __init__(self, seed, oracle_mod):
        self.rng = rng = np.random.default_rng(seed)
        self.oracle = oracle_mod
        snap, flags = synthetic.generate(synthetic.SynthParams(
            n_clusters=800, pods_per_cluster=40, groups=1, shuffle=False, recreate_frac=0.05, wtd_group_frac=0.2, multihost_frac=0.08,
            autoscaling_frac=0.3, seed=7000 + seed))
        nc = snap.dims["clusters"]
        # roles (the fleet's first rows donate the pods the large ones grow with)
        self.A, self.B, self.C, self.D, self.F, self.G, self.X = 799, 798, 797, 796, 795, 794, 640
        self.E = 700  # 33 worker groups; E + 1 (one group) is its neighbour in the group table
        self.W = list(range(720, 790))  # 70 wide clusters of 33..40 groups
        sizes = {self.A: int(rng.integers(7700, 8000)), self.B: int(rng.integers(2000, 3500)), self.C: int(rng.integers(300, 480)),
                 self.D: int(rng.integers(1000, 1600)), self.F: int(rng.integers(45, 64)), self.G: 64}
        grown = []
        for c in sorted(sizes, key=sizes.get, reverse=True):  # (the ones grown already are listed too: they donate nothing)
            grown.append(c)
            synthetic.grow_clusters(snap, grown, sizes[c])
        snap = synthetic.widen_clusters(snap, [self.D], 40)
        snap = synthetic.widen_clusters(snap, [self.F], int(rng.integers(45, 52)))
        snap = synthetic.widen_clusters(snap, [self.G], 100)
        snap = synthetic.widen_clusters(snap, [self.E], 33)
        for n in (33, 36, 40):
            snap = synthetic.widen_clusters(snap, [c for c in self.W if c % 3 == n % 3], n)
        self.special = {self.A, self.B, self.C, self.D, self.F, self.G, self.X, self.E, self.E + 1, *self.W}
        self.ordinary = np.array([c for c in range(nc) if c not in self.special])
        for c in (self.A, self.B, self.D, self.F, self.G):  # healthy, not autoscaling, every group at its pod count
            self._healthy(snap, c)
        flags.env_random_pod_delete = int(seed % 2)
        flags.fetch_pod_lists = 0
        # B behind a Recreate gate whose annotation is the digest of its spec (a JSON re-commit flips it)
        snap.c_flags[self.B] |= np.uint32(abi.CF_UPGRADE_RECREATE)
        h = head_row(snap, self.B)
        snap.h_version_state[h], snap.h_annot_state[h] = abi.VER_CURRENT, abi.ANNOT_HASH32
        snap.h_annot_hash.reshape(-1, 32)[h] = np.frombuffer(b32(spec_bytes(snap, self.B)), dtype=np.uint8)
        super().__init__(snap, flags, max_creates=1 << 21, large_clusters=True, wide_clusters=True)
        self.model = Model(nc, snap.dims["pods"], True, True)
        self.own = _owners(snap)
        self.free, self.saved, self.next_name = [], {}, 0x7E000000
        self.json_flips = 0
        self.stats = collections.Counter()
        self.seen = set()
        self.res_act = self.res_cre = None
        self.begin_epoch()
        self.forced = "first pass"
        self.pass_(expect_full=True)
        assert self.eng.get_option(abi.OPT_BUCKET_STRIDE) == 64 and set(self.model.caps) == {self.A, self.B, self.C, self.D}

    # ------------------------------------------------------------------------------------------------ snapshot edits
    def _healthy(self, snap, c):
        m = np.flatnonzero(_owners(snap) == c)
        set_phase(snap, m, abi.PHASE_RUNNING)
        snap.p_packed[m] = (snap.p_packed[m] & ~np.uint32((3 << abi.PP_READY_SHIFT) | abi.PP_RAY_TERMINATED)) | np.uint32(abi.COND_TRUE << abi.PP_READY_SHIFT)
        snap.c_flags[c] &= ~np.uint32(abi.CF_SKIP | abi.CF_SUSPEND | abi.CF_UPGRADE_RECREATE | abi.CF_AUTOSCALING)
        snap.c_flags[c] |= np.uint32(abi.CF_HEAD_EXPECT_OK)
        g0 = int(snap.c_group_off[c])
        for gi in range(int(snap.c_group_cnt[c])):
            g = g0 + gi
            snap.g_num_hosts[g] = 1
            scale_to(snap, g, int((snap.p_group_name_id[workers(snap, c)] == snap.g_name_id[g]).sum()))
        return m

    def _relabel(self, rows, c):
        """Pods move into RayCluster c (a random worker group of it)."""
        s = self.snap
        rows = np.asarray(rows, dtype=np.int64)
        s.p_ns_id[rows], s.p_cluster_name_id[rows] = s.c_ns_id[c], s.c_name_id[c]
        g = int(s.c_group_off[c]) + self.rng.integers(0, max(1, int(s.c_group_cnt[c])), rows.size)
        s.p_group_name_id[rows] = s.g_name_id[g] if s.c_group_cnt[c] else 0
        self.touched.update(rows.tolist())

    def _live_workers(self, own, clusters):
        s = self.snap
        w = ((s.p_packed >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER
        rows = np.flatnonzero(w & np.isin(own, clusters) & ((s.p_packed & abi.PP_TOMBSTONE) == 0))
        return rows[~np.isin(rows, list(self.touched))]

    def set_count(self, c, target):
        """Bulk move: RayCluster c gains pods of ordinary clusters or gives some of its workers to the emptiest ordinary ones."""
        own = _owners(self.snap)
        cur = int((own == c).sum())
        if target > cur:
            src = self._live_workers(own, self.ordinary)
            self._relabel(self.rng.choice(src, target - cur, replace=False), c)
        elif target < cur:
            out = self.rng.choice(self._live_workers(own, [c]), cur - target, replace=False)
            counts = _counts(self.snap, own)[self.ordinary]
            sinks = self.ordinary[np.argsort(counts, kind="stable")][:max(1, out.size // 8 + 1)]
            for i, sink in enumerate(sinks):
                part = out[i::sinks.size]
                if part.size:
                    self._relabel(part, sink)
        assert int((_owners(self.snap) == c).sum()) == target

    def traffic(self):
        """inc_soak's informer mix: status flips, deletions into free rows, re-additions (some under another cluster), pods moving
        between clusters, head-aux edits and object-row edits.  Only readiness flips reach the per-cluster RayClusters: their pod
        counts move by the scheduled steps alone."""
        s, rng = self.snap, self.rng
        own = _owners(s)
        workers = self._live_workers(own, np.arange(s.dims["clusters"]))
        large = np.isin(own, list(self.special))
        for r in rng.choice(workers, int(rng.integers(10, 40)), replace=False).tolist():
            s.p_packed[r] ^= np.uint32(1 << abi.PP_READY_SHIFT)
            if not large[r] and rng.random() < 0.3:
                set_phase(s, [r], int(rng.integers(1, 6)))
            self.touched.add(r)
        workers = workers[~large[workers]]
        for r in rng.choice(workers, int(rng.integers(0, 10)), replace=False).tolist():  # deletions -> free rows
            if r in self.touched:
                continue
            self.saved[r] = {c: s.cols[c][r].copy() for c in ("p_ns_id", "p_cluster_name_id", "p_group_name_id", "p_name_id", "p_packed",
                                                                 "p_replica_index", "p_replica_name_id")}
            self._tombstone([r])
            self.free.append(r)
        for _ in range(int(rng.integers(0, 8))):  # re-additions: the same pod again, or under another cluster / namespace
            if not self.free:
                break
            r = self.free.pop(int(rng.integers(len(self.free))))
            if r in self.touched:
                self.free.append(r)
                continue
            for col, v in self.saved.pop(r).items():
                s.cols[col][r] = v
            if rng.random() < 0.4:
                self._relabel([r], int(rng.choice(self.ordinary)))
            self.touched.add(r)
        for r in rng.choice(workers, int(rng.integers(0, 8)), replace=False).tolist():  # moves between clusters
            if r not in self.touched:
                self._relabel([r], int(own[int(rng.choice(workers))]))
        if s.dims["heads"] and rng.random() < 0.5:
            h = int(rng.integers(s.dims["heads"]))
            s.h_ready_status[h] = np.uint8(int(rng.integers(0, 4)))
            s.h_pod_ip_id[h] = s.h_pod_ip_id[int(rng.integers(s.dims["heads"]))]
            self.head_rows.add(h)
        for c in rng.choice(self.ordinary, int(rng.integers(0, 6)), replace=False).tolist():
            if s.c_group_cnt[c]:
                g = int(s.c_group_off[c]) + int(rng.integers(int(s.c_group_cnt[c])))
                s.g_replicas[g] = int(rng.integers(0, 50))
                if rng.random() < 0.3:
                    s.g_flags[g] ^= np.uint32(abi.GF_EXPECT_OK)
            if rng.random() < 0.3:
                s.c_flags[c] ^= np.uint32(1 << int(rng.choice([0, 2, 3, 5])))
            if rng.random() < 0.3:
                s.c_old_state[c] = np.uint8(int(rng.integers(0, 4)))
            self.cluster_rows.add(c)

    def _tombstone(self, rows):
        for col in ("p_ns_id", "p_cluster_name_id", "p_group_name_id", "p_name_id", "p_replica_index", "p_replica_name_id"):
            self.snap.cols[col][rows] = 0
        self.snap.p_packed[rows] = np.uint32(abi.PP_TOMBSTONE)
        self.touched.update(int(r) for r in rows)

    def churn(self, c, other):
        """Case 2, one epoch: pods of large RayCluster c deleted, rows freed earlier reused by new pods of c, a row deleted and reused
        by another pod of c, pods moving between c and `other` both ways, and pods of D moving between its groups."""
        s, rng = self.snap, self.rng
        own = _owners(s)
        mine = self._live_workers(own, [c])
        gone = rng.choice(mine, int(rng.integers(3, 20)), replace=False)
        self._tombstone(gone)
        reuse = [r for r in self.free if r not in self.touched][:int(rng.integers(2, 12))]
        for r in gone[:2].tolist() + reuse:  # new pods (fresh names) of c in rows that were free
            if r in self.free:
                self.free.remove(r)
                self.saved.pop(r, None)
            s.p_packed[r] = (np.uint32(abi.NT_WORKER << abi.PP_NODE_TYPE_SHIFT) | np.uint32(abi.PHASE_RUNNING << abi.PP_PHASE_SHIFT)
                             | np.uint32(abi.COND_TRUE << abi.PP_READY_SHIFT))
            s.p_name_id[r] = self.next_name
            self.next_name += 1
            self._relabel([r], c)
        a_to_b = rng.choice(self._live_workers(own, [other]), int(rng.integers(1, 15)), replace=False)
        b_to_a = rng.choice(self._live_workers(own, [c]), int(rng.integers(1, 15)), replace=False)
        self._relabel(a_to_b, c)
        self._relabel(b_to_a, other)
        d = self._live_workers(own, [self.D])[:int(rng.integers(1, 20))]
        s.p_group_name_id[d] = s.g_name_id[int(s.c_group_off[self.D]) + rng.integers(0, int(s.c_group_cnt[self.D]), d.size)]
        self.touched.update(d.tolist())
        self.stats["churn"] += 1

    def hand_group(self, c, to_next):
        """The boundary between RayCluster c and c + 1 in the group table moves by one group (c's last, or c + 1's first, changes
        owner), and that group's pods are relabelled: c crosses 32 / 33 groups while every table keeps its size."""
        s = self.snap
        own = _owners(s)
        if to_next:
            g, new = int(s.c_group_off[c] + s.c_group_cnt[c] - 1), c + 1
            s.c_group_cnt[c] -= 1; s.c_group_cnt[c + 1] += 1; s.c_group_off[c + 1] -= 1
        else:
            g, new = int(s.c_group_off[c + 1]), c
            s.c_group_cnt[c] += 1; s.c_group_cnt[c + 1] -= 1; s.c_group_off[c + 1] += 1
        s.g_cluster_idx[g] = new
        old = c + 1 if new == c else c
        rows = np.flatnonzero((own == old) & (s.p_group_name_id == s.g_name_id[g]))
        s.p_ns_id[rows], s.p_cluster_name_id[rows] = s.c_ns_id[new], s.c_name_id[new]
        self.touched.update(rows.tolist())
        self.structural = True
        self.seen.add(f"{int(s.c_group_cnt[c])} groups")

    def scale_down(self, c):
        """List order: every pod of c healthy, its group 0 scaled down by a few pods (which ones go depends on List order).  A Recreate
        gate stays as it was."""
        gate = self.snap.c_flags[c] & np.uint32(abi.CF_UPGRADE_RECREATE)
        m = self._healthy(self.snap, c)
        self.snap.c_flags[c] |= gate
        self.touched.update(m.tolist())
        g = int(self.snap.c_group_off[c])
        self.snap.g_replicas[g] = max(0, int(self.snap.g_replicas[g]) - int(self.rng.integers(3, 40)))
        self.whole_objects = True
        self.stats["scale-downs"] += 1

    # ------------------------------------------------------------------------------------------------ one epoch
    def begin_epoch(self):
        self.touched, self.cluster_rows, self.head_rows = set(), set(), set()
        self.whole_objects = self.structural = self.json = self.device_only = False
        self.forced = None  # why the epoch must be a full pass (an option, the flags or a group count changed)

    def toggle(self, option):
        set_ = self.eng.set_large_clusters if option == "large" else self.eng.set_wide_clusters
        on = not getattr(self.model, option)
        set_(on)
        setattr(self.model, option, on)
        self.model.reset()
        self.forced = f"option {option} {'on' if on else 'off'}"

    def end_epoch(self):
        s = self.snap
        if self.json:
            np.copyto(self.views["json"], s.json)
            self.eng.commit(abi.PART_JSON)
        if self.whole_objects or self.structural:
            self.commit_objects()
        elif self.cluster_rows or self.head_rows:
            for col in OBJ_COLS:
                np.copyto(self.views[col], s.cols[col])
            self.eng.commit_object_rows(sorted(self.cluster_rows), sorted(self.head_rows))
        self.commit_rows(sorted(self.touched), journal=bool(self.rng.integers(2)))
        self.pass_(expect_full=self.structural or self.forced is not None)

    def pass_(self, expect_full=False):
        s, m = self.snap, self.model
        own = _owners(s)
        counts, groups = _counts(s, own), s.c_group_cnt.astype(np.int64)
        lim = m.limits()
        prev_own = self.own
        t = np.asarray(sorted(self.touched), dtype=np.int64)
        arrive = t[(own[t] >= 0) & (own[t] != prev_own[t])]
        before = _counts(s, prev_own) if self.res_act is not None else counts
        peak = before + np.bincount(own[arrive], minlength=s.dims["clusters"])
        over = np.flatnonzero(peak > lim) if m.stride else np.zeros(0, dtype=np.int64)
        # why this epoch may not be incremental, most certain first; None: it must be
        cause = None
        if expect_full:
            cause = self.forced or "group count"
        elif not m.valid:
            cause = "sort pipeline"
        elif over.size:  # a record past its bucket and region: k_inc_admit voids the epoch
            cause = ("past 8192 pods" if (counts[over] > abi.LARGE_MAX_PODS).any() else
                     "region" if any(int(c) in m.caps for c in over) else "stride")
            if any(int(c) in m.caps for c in over):
                self.seen.add("past the region edge")
        elif any(counts[c] == lim[c] for c in m.caps):
            self.seen.add("region edge")
        self.predicted = cause
        got, _ = self.check(self.oracle, device_only=self.device_only)
        inc = incremental(got, s.dims["clusters"])
        decided = got.clusters["path"] != abi.PATH_SKIPPED
        if self.json:  # B's Recreate gate flipped: every pod deleted after an odd number of re-commits, none after an even one
            assert (got.clusters["path"][self.B] == abi.PATH_RECREATE_DELETE_ALL) == bool(self.json_flips % 2), (self.json_flips, got.clusters[self.B])
        assert np.array_equal(got.clusters["n_pods"][decided], counts[decided])  # (the model counts what k_match2 counts)
        if cause is None and self.res_act is not None:
            n_act = got.act_cnt.astype(np.int64)
            n_cre = np.bincount(s.g_cluster_idx, weights=got.groups["n_create"], minlength=s.dims["clusters"]).astype(np.int64)
            acts = self.act_ext + int(n_act[n_act > self.res_act].sum())
            cres = self.cre_ext + int(n_cre[n_cre > self.res_cre].sum())
            if acts > s.dims["pods"] or cres > self.eng.cfg.max_creates:
                cause = "arena (reserved runs)"
        if cause is None or cause == "arena (reserved runs)":
            if cause is None:
                assert inc, ("an epoch the resident state can absorb took the full pass", self.stats)
        else:
            assert not inc, ("an epoch that must take the full pass was incremental", cause)
        self.stats["epochs"] += 1
        self.stats["incremental" if inc else f"full: {cause}"] += 1
        n_act = got.act_cnt.astype(np.int64)
        n_cre = np.bincount(s.g_cluster_idx, weights=got.groups["n_create"], minlength=s.dims["clusters"]).astype(np.int64)
        if inc:
            self.res_act, self.res_cre = np.maximum(self.res_act, n_act), np.maximum(self.res_cre, n_cre)
        else:
            m.full_pass(counts, groups)
            self.res_act, self.res_cre = n_act, n_cre
        self.act_ext, self.cre_ext = got.act_pod_idx.size, got.create_idx.size
        assert self.cre_ext < self.eng.cfg.max_creates
        assert self.eng.get_option(abi.OPT_BUCKET_STRIDE) == m.stride, (self.eng.get_option(abi.OPT_BUCKET_STRIDE), m.stride, cause)
        for n in (256, 257, abi.LARGE_MAX_PODS, abi.LARGE_MAX_PODS + 1):
            if (counts == n).any():
                self.seen.add(f"{n} pods")
        self.own = own
        return got, inc

    def kernels(self):
        """reconcile_profiled (an epoch without changes): which pipeline ran (incremental bucket-pipeline kernels, k_large_sort among them
        because the fleet always has wide clusters, or the sort pipeline) and the stride, against the model; then a fetch, so that the
        next epoch's results come back packed."""
        names = {k for k, _ in self.eng.reconcile_profiled(self.flags)["kernels"]}
        self.eng.fetch()
        m, groups = self.model, self.snap.c_group_cnt.astype(np.int64)
        if m.valid:
            assert not SORT_KERNELS & names, names
            assert ("k_large_sort" in names) == bool(m.per_cluster_list(groups)), (names, m.per_cluster_list(groups))
        else:
            assert "k_match2" not in names and "k_large_sort" not in names, names
        assert self.eng.get_option(abi.OPT_BUCKET_STRIDE) == m.stride
        self.stats["kernel checks"] += 1


def _episodes(st):
    """The class-crossing steps, grouped into episodes whose steps run in consecutive epochs.  A step is (ready, action): an
    episode waits (ordinary epochs) while its next step is not ready."""
    m, rng, s = st.model, st.rng, st.snap
    always = lambda: True  # noqa: E731
    on_bucket = lambda: m.valid  # noqa: E731
    has_region = lambda c: (lambda: m.valid and c in m.caps)  # noqa: E731

    def count(c, n):
        return lambda: st.set_count(c, n() if callable(n) else n)

    def json_flip():  # B's spec no longer matches (or again matches) the digest its Recreate gate compares
        assert s.c_flags[st.B] & abi.CF_UPGRADE_RECREATE
        s.json[int(s.c_json_off[st.B]) + 3] ^= 0x20
        st.json = True
        st.json_flips += 1

    def many_dirty():  # case 6: every per-cluster RayCluster and 150 ordinary ones dirty at once (past the staging buffer)
        own = _owners(s)
        for c in list(st.W) + [st.A, st.B, st.C, st.D, st.F, st.G] + rng.choice(st.ordinary, 150, replace=False).tolist():
            w = st._live_workers(own, [c])
            if w.size:
                r = int(rng.choice(w))
                s.p_packed[r] ^= np.uint32(1 << abi.PP_READY_SHIFT)
                st.touched.add(r)
        st.stats["many dirty"] += 1

    def flip_flags():
        st.flags.env_random_pod_delete ^= 1
        st.forced = "process flags"

    def device_only():
        st.device_only = True

    stride = lambda: m.stride  # noqa: E731
    return [
        # an ordinary cluster to the stride and one past it (the stride widens), twice
        [(on_bucket, count(st.X, stride)), (on_bucket, count(st.X, lambda: m.stride + 1)),
         (on_bucket, count(st.X, stride)), (on_bucket, count(st.X, lambda: m.stride + 1))],
        # 256 / 257: X becomes large, then keeps its region while it is small again
        [(on_bucket, count(st.X, 256)), (on_bucket, count(st.X, 257)), (on_bucket, count(st.X, lambda: int(rng.integers(20, 60))))],
        # exactly the region's edge, then one past it; then the cluster shrinks below 257 and loses its region at a later void
        # (which may widen the fleet stride)
        [(has_region(st.C), count(st.C, lambda: m.stride + m.caps[st.C])), (has_region(st.C), count(st.C, lambda: m.stride + m.caps[st.C] + 1)),
         (has_region(st.C), count(st.C, lambda: int(rng.integers(100, 200)))),
         (on_bucket, lambda: st.set_count(st.G, 300) if st.X in m.caps else st.set_count(st.X, m.stride + 1))],
        # a wide cluster past 256 pods gets a region, and keeps it when it shrinks
        [(on_bucket, count(st.F, 300)), (on_bucket, count(st.F, lambda: int(rng.integers(40, 64))))],
        # case 1: a large cluster at the stride or below, churned there, then regrown inside its region
        [(has_region(st.B), count(st.B, lambda: m.stride - int(rng.integers(0, 3)))), (always, lambda: st.churn(st.B, st.A)),
         (on_bucket, count(st.B, lambda: m.stride + m.caps.get(st.B, 0) - int(rng.integers(0, 40))))],
        # 8 192 / 8 193: the sort pipeline until an option change brings the layout back
        [(lambda: has_region(st.A)() and m.stride + m.caps[st.A] == abi.LARGE_MAX_PODS, count(st.A, abi.LARGE_MAX_PODS)),
         (always, count(st.A, abi.LARGE_MAX_PODS + 1)), (always, count(st.A, lambda: int(rng.integers(7000, 8100)))),
         (always, lambda: st.toggle("large")), (always, lambda: st.toggle("large"))],
        [(always, lambda: st.hand_group(st.E, True)), (always, lambda: st.hand_group(st.E, False))],  # 33 -> 32 -> 33 groups
        [(always, lambda: st.toggle("wide")), (always, lambda: st.toggle("wide"))],
        [(always, json_flip)], [(always, json_flip)],
        # case 2 and list order: leave / join / reuse in one epoch, then a scale-down that deletes by List order
        [(always, lambda: st.churn(st.A, st.B)), (always, lambda: st.scale_down(st.A))],
        [(always, lambda: st.churn(st.D, st.C)), (always, lambda: st.scale_down(st.D))],
        [(always, lambda: st.churn(st.C, st.D)), (always, lambda: st.scale_down(st.B))],
        [(always, many_dirty)], [(always, device_only)], [(always, flip_flags)],
    ]


def _run_stream(seed, oracle_mod):
    st = Stream(seed, oracle_mod)
    try:
        episodes = _episodes(st)
        order = st.rng.permutation(len(episodes))
        for i in order.tolist():
            for ready, action in episodes[i]:
                for _ in range(4):  # (a step that is not ready waits a few ordinary epochs, then is dropped: the checks below notice)
                    st.begin_epoch()
                    st.traffic()
                    go = ready()
                    if go:
                        action()
                    st.end_epoch()
                    if st.stats["epochs"] % 4 == 0:
                        st.kernels()
                    if go:
                        break
                else:
                    st.stats[f"dropped: episode {i}"] += 1
            for _ in range(int(st.rng.integers(0, 2))):  # an ordinary epoch between episodes now and then
                st.begin_epoch()
                st.traffic()
                st.end_epoch()
        report = dict(seed=seed, **st.stats, boundaries=sorted(st.seen))
        print("class stream", json.dumps(report))
        assert st.stats["incremental"] >= 0.4 * st.stats["epochs"], report
        # the stream reached every boundary it claims (a silent generator bug must not turn the test into a no-op)
        need = {"256 pods", "257 pods", "8192 pods", "8193 pods", "region edge", "past the region edge", "32 groups", "33 groups"}
        assert need <= st.seen, (need - st.seen, report)
        for cause in ("stride", "region", "past 8192 pods", "option large on", "option wide off", "group count", "process flags"):
            assert st.stats[f"full: {cause}"] >= 1, (cause, report)
        assert st.stats["churn"] >= 4 and st.stats["many dirty"] and st.stats["scale-downs"] >= 3 and not any(k.startswith("dropped") for k in st.stats), report
    finally:
        st.close()


@pytest.mark.parametrize("seed", range(6))
def test_class_crossing_streams(seed, oracle_mod):
    _run_stream(seed, oracle_mod)

"""KR_OPT_LARGE_MOVES: a large RayCluster (one with a region of the large-cluster arena) deleted, moved by swap-remove or regrouped
keeps the device-side incremental epoch.  A deleted one's Pods become orphans and its region is abandoned; a moved one carries its
region (offset and capacity, and a huge one its tiles) to its new row and is admitted there again; a regrouped one is initialised
again in its own row, keeping its region.

Every epoch is compared with the CPU oracle.  The streams run on the Fleet of test_gpu_structural_streams.py (every other option
on, tests/class_model.py predicting which epochs are incremental and where the regions are) with this option on as well, and the
model follows the regions to their new rows.  When a pass is incremental, every RayCluster it did not name keeps its records at its
new row, its group records at the shifted indices.  An option-off twin sees the same epochs: it takes the full pass at the large
events, with identical results."""
import collections
import copy
import json

import numpy as np
import pytest

import test_gpu_structural_streams as ss
from class_model import ADOPT_MAX, MAP_MAX, Model
from harness import PACKER_CAPS, POD_COLS, Driver, Mirror, flip_ready, incremental, members, objects, packer_check
from kuberay_b200 import abi, synthetic
from kuberay_b200.packer import GroupPacker, Packer

pytestmark = pytest.mark.gpu

RELEASE = "k_inc_large_release"


class MovesModel(Model):
    """Model with KR_OPT_LARGE_MOVES: a gone row with a region no longer voids the map; when the map is followed the regions go
    with their RayClusters (`moves`: old row -> new row, -1: deleted; a regrouped row maps to itself)."""
    moves = {}

    @classmethod
    def of(cls, m):
        out = cls.__new__(cls)
        out.__dict__.update(m.__dict__)
        return out

    def row_map(self, gone, n_rows, n_created, adopt):
        if n_rows > MAP_MAX:
            return "map cap"
        if adopt and n_created > ADOPT_MAX:
            return "adoption cap"
        self.remap(self.moves)
        return None

    def remap(self, moves):
        caps, offs = {}, {}
        for c in self.caps:
            to = moves.get(c, c)
            if to >= 0:
                caps[to], offs[to] = self.caps[c], self.offs[c]
        self.caps, self.offs = caps, offs


class MovesFleet(ss.Fleet):
    """The structural-streams Fleet with KR_OPT_LARGE_MOVES on (or, `on=False`, the same fleet without it: the twin)."""

    def __init__(self, universe, flags, live, oracle, seed, on=True):
        super().__init__(universe, flags, live, oracle, seed)
        if on:
            self.eng.set_large_moves(True)
            self.model = MovesModel.of(self.model)

    def moves(self):
        """Old row -> new row of every gone row whose RayCluster stays (itself when regrouped), -1 for a deleted one; tags the large ones."""
        pos = {u: i for i, u in enumerate(self.order)}
        out = {}
        for o, u in enumerate(self.old_order):
            to = pos.get(u, -1)
            if to == o and u not in self.regrouped:
                continue
            out[o] = to
            if o in self.model.caps:
                huge = self.model.stride + self.model.caps[o] > abi.LARGE_MAX_PODS
                kind = "delete" if to < 0 else "regroup" if to == o else "move"
                self.tags.add(f"{kind} {'huge' if huge else 'large'}")
        return out

    def finish(self, expect=None, profiled=False, device_only=False):
        self.model.moves = self.moves()
        return super().finish(expect=expect, profiled=profiled, device_only=device_only)

    def mirror(self, src):
        """This epoch's edits of fleet `src` (the same universe, order, touched rows, created and regrouped RayClusters)."""
        self.uni, self.order = copy.deepcopy(src.uni), list(src.order)
        self.touched, self.created, self.regrouped = set(src.touched), list(src.created), set(src.regrouped)
        self.twice, self.reset_layout = src.twice, src.reset_layout


@pytest.fixture
def twins(oracle_mod):
    """make(seed, **universe) -> (fleet with the option, twin without it) over the same universe."""
    made = []

    def make(seed, w32=(), **kw):
        snap, flags, live = ss._fleet(seed, **kw)
        if w32:  # (RayClusters of 32 worker groups: group 0 of 2 split into 31)
            snap = synthetic.widen_clusters(snap, list(w32), 31)
        pair = (MovesFleet(snap, flags, live, oracle_mod, seed), MovesFleet(copy.deepcopy(snap), copy.deepcopy(flags), live, oracle_mod, seed, on=False))
        made.extend(pair)
        return pair
    yield make
    for f in made:
        f.close()


def live_pods(f, u):
    return int(((f.uown() == u) & ((f.uni.p_packed & abi.PP_TOMBSTONE) == 0)).sum())


def epoch(on, off, large=True, **kw):
    """One epoch on both fleets: -> the option-on fleet's (results, incremental).  `large`: the epoch has a large event, which the twin
    takes as a full pass ("large gone row"); the results are identical either way."""
    off.mirror(on)
    got, inc, _ = on.finish(**kw)
    twin, twin_inc, cause = off.finish(**kw)
    assert not twin.diff(got)
    if large:
        assert not twin_inc and cause == "large gone row", (twin_inc, cause)
    on.begin()
    off.begin()
    return got, inc


def test_rayjob_deleted_in_the_last_row(twins):
    """A RayJob's RayCluster grows to 1 200 Pods and is deleted in the last row; its row is then re-created by another RayCluster,
    which starts without a region."""
    f, t = twins(1)
    donors = np.arange(0, 200)
    job = 360
    f.create(job)
    epoch(f, t, large=False)
    f.set_count(job, 1200, donors)
    _, inc = epoch(f, t, large=False)
    assert inc and len(f.order) - 1 in f.model.caps
    orphans, lost = f.prev.n_orphans, live_pods(f, job)
    f.delete(job)
    got, inc = epoch(f, t)
    assert inc and got.n_orphans == orphans + lost and "delete large" in f.seen
    f.create(361)  # into the row the RayJob held
    f.flip(20)
    got, inc = epoch(f, t, large=False)
    assert inc and len(f.order) - 1 not in f.model.caps


@pytest.mark.parametrize("mover", ["ordinary", "large", "none"])
def test_large_deleted_in_a_middle_row(mover, twins):
    """A large RayCluster in a middle row deleted.  Its mover (the last row) is ordinary, large with another region (the two
    numberings of the region table in one pass: every one of the deleted one's Pods must become an orphan and every one of the
    mover's stay in its new row), or, `none`, ordinary while the deleted one is the only large RayCluster of the fleet."""
    f, t = twins(2)
    donors = np.arange(0, 200)
    x, last = 250, f.order[-1]
    f.set_count(x, 400, donors)
    if mover == "large":
        f.set_count(last, 330, donors)
    elif mover == "ordinary":
        f.set_count(300, 500, donors)  # another large RayCluster elsewhere
    _, inc = epoch(f, t, large=False)
    assert inc and (f.order.index(x) in f.model.caps)
    assert len(f.model.caps) == (1 if mover == "none" else 2)
    orphans, lost = f.prev.n_orphans, live_pods(f, x)
    f.delete(x)
    got, inc = epoch(f, t, profiled=True)
    assert inc and got.n_orphans == orphans + lost, (got.n_orphans, orphans, lost)
    row = f.order.index(last)
    assert got.clusters["n_pods"][row] == (330 if mover == "large" else int((f.uown() == last).sum()))
    assert (row in f.model.caps) == (mover == "large") and len(f.model.caps) == (0 if mover == "none" else 1)
    f.flip(30)
    _, inc = epoch(f, t, large=False)
    assert inc


def test_moved_large_keeps_its_region(twins):
    """A large RayCluster moved by the deletion of an ordinary one carries its region: a later growth of another RayCluster is placed
    past the region cursor, not over the carried region, and the moved one scales up past its carried region in a later epoch."""
    f, t = twins(3)
    donors = np.arange(0, 200)
    last = f.order[-1]
    f.set_count(last, 600, donors)
    epoch(f, t, large=False)
    off, cap = f.model.offs[len(f.order) - 1], f.model.caps[len(f.order) - 1]
    f.delete(f.order[220])
    got, inc = epoch(f, t)
    assert inc and f.model.offs[220] == off and f.model.caps[220] == cap and "move large" in f.seen
    assert got.changed_clusters is not None and 220 in got.changed_clusters.tolist()
    f.set_count(f.order[100], 500, donors)
    _, inc = epoch(f, t, large=False)
    assert inc and f.model.offs[100] >= off + cap
    f.set_count(last, f.model.stride + cap + 40, donors)
    _, inc = epoch(f, t, large=False)
    assert inc and f.model.offs[220] > off


@pytest.mark.parametrize("growth", [True, False])
def test_moved_large_scales_past_its_carried_region(growth, twins):
    """Moved and scaled up past its carried region in the same epoch: with KR_OPT_LARGE_GROWTH it grows a region in that pass, without
    it the epoch takes the full pass."""
    f, t = twins(4)
    donors = np.arange(0, 200)
    last = f.order[-1]
    f.set_count(last, 400, donors)
    epoch(f, t, large=False)
    if not growth:
        for fl in (f, t):
            fl.eng.set_large_growth(False)
    cap = f.model.caps[len(f.order) - 1]
    f.delete(f.order[10])
    f.set_count(last, f.model.stride + cap + 30, donors)
    if growth:
        _, inc = epoch(f, t)
        assert inc and f.model.caps[10] > cap
    else:
        epoch_full_both(f, t)
    f.flip(20)
    _, inc = epoch(f, t, large=False)
    assert inc


def epoch_full_both(on, off):
    """An epoch the model has no rule for (growth off: the carried region overflows, k_inc_admit voids): both fleets take the full
    pass with identical results."""
    off.mirror(on)
    got, inc, _ = on.finish(expect="carried region overflows")
    twin, twin_inc, _ = off.finish(expect="carried region overflows")
    assert not inc and not twin_inc and not twin.diff(got)
    on.begin()
    off.begin()
    return got


@pytest.mark.parametrize("how", ["append", "prepend", "remove", "rename", "reorder"])
def test_regrouped_large(how, twins):
    """A large RayCluster regrouped (a RayService in-place update appends a worker group; or one removed, renamed, reordered) is
    initialised again in its row and keeps its region."""
    f, t = twins(5)
    donors = np.arange(0, 200)
    u = 120
    f.set_count(u, 450, donors)
    epoch(f, t, large=False)
    row = f.order.index(u)
    off, cap = f.model.offs[row], f.model.caps[row]
    gs = f.groups(u)
    new = {"append": gs + [(gs[0][0], f.fresh_id())], "prepend": [(gs[0][0], f.fresh_id())] + gs, "remove": gs[:-1],
           "rename": [(gs[0][0], f.fresh_id())] + gs[1:], "reorder": gs[::-1]}[how]
    f.regroup(u, new)
    f.flip(10)
    got, inc = epoch(f, t, profiled=True)
    assert inc and f.model.offs[row] == off and f.model.caps[row] == cap and "regroup large" in f.seen
    assert row in got.changed_clusters.tolist()
    f.flip(20)
    _, inc = epoch(f, t, large=False)
    assert inc


def test_large_and_wide(twins):
    """A RayCluster both large and wide (40 groups), moved, then deleted; and a 32-group large RayCluster regrouped to 33."""
    f, t = twins(6, wide=(359, 358))
    donors = np.arange(0, 200)
    f.set_count(359, 600, donors)
    f.set_count(358, 500, donors)
    epoch(f, t, large=False)
    f.delete(f.order[40])  # 359 (large and wide) moves into row 40
    _, inc = epoch(f, t)
    assert inc and 40 in f.model.caps
    f.delete(359)
    _, inc = epoch(f, t)
    assert inc
    f.flip(20)
    _, inc = epoch(f, t, large=False)
    assert inc


def test_regroup_32_to_33(twins):
    f, t = twins(7, w32=(150,))
    donors = np.arange(0, 200)
    u = 150
    assert f.uni.c_group_cnt[u] == 32
    f.set_count(u, 500, donors)
    epoch(f, t, large=False)
    gs = f.groups(u)
    f.regroup(u, gs + [(gs[0][0], f.fresh_id())])
    _, inc = epoch(f, t)
    assert inc and f.uni.c_group_cnt[u] == 33


@pytest.mark.parametrize("when", ["pods_in_epoch", "create_into_hole", "recreated_next_epoch"])
def test_same_epoch_events(when, twins):
    """Pod events on the deleted and the moved large RayClusters' Pods in the epoch that renumbers them; a RayCluster created into the
    vacated row; the deleted key created again in the next epoch, adopting its orphans."""
    f, t = twins(8)
    donors = np.arange(0, 200)
    x, last = 200, f.order[-1]
    f.set_count(x, 350, donors)
    f.set_count(last, 300, donors)
    epoch(f, t, large=False)
    f.delete(x)
    if when == "pods_in_epoch":  # (the deleted one's Pods and the moved one's)
        for u in (x, last):
            rows = f.workers(u)[:25]
            f.uni.p_packed[rows] ^= np.uint32(1 << abi.PP_READY_SHIFT)
            f.touched.update(rows.tolist())
    if when == "create_into_hole":  # RayCluster 365 created into the row x vacated, and the large mover stays where it was
        f.order = list(f.old_order)
        f.order[f.order.index(x)] = 365
        f.created.append(365)
    _, inc = epoch(f, t)
    assert inc
    if when == "recreated_next_epoch":
        f.create(x)
        _, inc = epoch(f, t, large=False)
        assert inc


def test_stream(oracle_mod):
    """A seeded stream of every structural event over all the options plus this one, twinned by an engine without it."""
    snap, flags = ss._universe(640, 480, 32, seed=9100, wide=(401, 501, 550, 600))
    snap = synthetic.widen_clusters(snap, [ss.WIDE32], 32)
    f = MovesFleet(snap, flags, list(range(480)), oracle_mod, 11)
    t = MovesFleet(copy.deepcopy(snap), copy.deepcopy(flags), list(range(480)), oracle_mod, 11, on=False)
    try:
        rng, donors, pool, deleted = f.rng, np.arange(0, 320), list(range(480, 640)), []
        big = [u for u in f.order if u >= 320][:6]
        for e in range(36):
            if e < 2:  # a few large RayClusters to delete, move and regroup
                for u in big[3 * e:3 * e + 3]:
                    f.set_count(u, 300 + 40 * (u % 5), donors)
            else:
                ss._stream_epoch(f, rng, donors, deleted, pool, ss.WIDE32)
                ss._scheduled(f, e, donors, deleted)
                large = [u for u in f.order if f.order.index(u) in f.model.caps and u not in f.regrouped and u not in f.created]
                if e % 6 == 2 and large and f.order[-1] not in large and f.order[-1] not in f.regrouped:
                    f.delete(large[0])  # (deleted from a middle row)
                    deleted.append(large[0])
                elif e % 6 == 4 and large and large[-1] in f.order[-3:]:
                    f.delete(f.order[int(rng.integers(10, 200))])  # (a large one may be the mover)
                elif e % 6 == 0 and large:
                    gs = f.groups(large[0])
                    f.regroup(large[0], gs + [(gs[0][0], f.fresh_id())])
                f.twice = e % 5 == 4
            t.mirror(f)
            got, inc, cause = f.finish(profiled=e % 7 == 3, device_only=e % 7 == 5)
            twin, twin_inc, twin_cause = t.finish()
            assert not twin.diff(got), e
            if inc and not twin_inc:
                f.stats[f"twin full: {twin_cause}"] += 1
            f.begin()
            t.begin()
        report = dict(**f.stats, events=sorted(f.seen))
        print("large moves stream", json.dumps(report))
        missing = {"delete large", "move large", "regroup large"} - f.seen
        assert not missing, (missing, report)
        assert f.stats["full: large gone row"] == 0 and f.stats["twin full: large gone row"] >= 3, report
    finally:
        f.close()
        t.close()


# ------------------------------------------------------------------------------------------------ huge RayClusters
def _huge_driver(on, oracle_mod):
    snap, flags = synthetic.generate(synthetic.config("C2", n_clusters=1400, pods_per_cluster=16, groups=2, seed=41))
    synthetic.grow_clusters(snap, [1399, 1300], 9000)
    dr = Driver(snap, flags, slack=1.25, max_creates=1 << 16, large_clusters=True, huge_clusters=True, cluster_deletes=True, large_moves=on)
    dr.check(oracle_mod, expect_incremental=None)
    dr.check(oracle_mod, expect_incremental=None)
    return dr


def test_huge_moved_and_deleted(oracle_mod):
    """A huge RayCluster (KR_OPT_HUGE_CLUSTERS, 9 000 Pods) moved by a deletion (it keeps its tiles), then deleted; against a twin
    without the option, which takes the full pass at both."""
    on, off = _huge_driver(True, oracle_mod), _huge_driver(False, oracle_mod)
    try:
        for rows in ([12], [1300]):  # 1399 (huge) moves into row 12; then huge 1300 is deleted
            old = on.snap
            new = synthetic.delete_clusters(old, rows)
            outs = []
            for dr, expect in ((on, True), (off, False)):
                dr.use(copy.deepcopy(new))
                dr.commit_objects()
                dr.prev = None
                got, names = dr.check(oracle_mod, expect_incremental=expect, profiled=expect)
                outs.append(got)
                if expect:
                    assert RELEASE in names and "k_huge_tiles" in names, names
            assert not outs[1].diff(outs[0])
        rows = np.arange(3, on.snap.dims["pods"], 41)
        for dr in (on, off):
            flip_ready(dr.snap, rows)
            dr.commit_rows(rows)
            dr.check(oracle_mod, expect_incremental=True)
    finally:
        on.close()
        off.close()


def test_transfer_size(oracle_mod):
    """A large deletion epoch fetches the changed records only: far fewer bytes than the full pass that the option-off twin takes."""
    grown, flags = synthetic.generate(synthetic.config("C2", n_clusters=400, pods_per_cluster=16, groups=2, seed=63))
    synthetic.grow_clusters(grown, [399, 50], 500)
    d2h = []
    for on in (True, False):
        dr = Driver(grown, flags, slack=1.25, large_clusters=True, cluster_deletes=True, large_moves=on)
        try:
            dr.check(oracle_mod, expect_incremental=None)
            dr.check(oracle_mod, expect_incremental=None)
            dr.use(synthetic.delete_clusters(dr.snap, [50]))
            dr.commit_objects()
            dr.prev = None
            dr.check(oracle_mod, expect_incremental=on)
            d2h.append(dr.eng.last_profile()["d2h_bytes"])
        finally:
            dr.close()
    assert d2h[0] * 4 < d2h[1], d2h


# ------------------------------------------------------------------------------------------------ the native packers
def test_native_packer_against_option_off(oracle_mod):
    """The native packer needs no change: with every option plus this one against a twin without this one, on one informer stream of
    creates, deletes, group edits and growth.  Both equal the oracle and each other every epoch, the option keeps at least as many
    epochs incremental, and some epoch that deletes, moves or regroups a large RayCluster is incremental only with it."""
    caps = dict(PACKER_CAPS, max_clusters=256, max_groups=2048, max_wtd=1024, max_pods=16384, max_jobs=256, max_creates=1 << 20)
    on, off = Packer(**caps, **ss.ALL, large_moves=True), Packer(**caps, **ss.ALL)
    try:
        assert on.engine.get_option(abi.OPT_LARGE_MOVES) == 1 and off.engine.get_option(abi.OPT_LARGE_MOVES) == 0
        objs = objects(5)
        ms = [Mirror(*copy.deepcopy(objs), pk) for pk in (on, off)]
        for pk, m in zip((on, off), ms):
            pk.flush()
            packer_check(m, oracle_mod, lean=True)
        state = [([0], {}), ([0], {})]
        tally = collections.Counter()
        for e in range(120):
            outs = []
            for (counter, deleted), m, pk in zip(state, ms, (on, off)):
                rng = np.random.default_rng(7000 + e)
                tag = ss._packer_events(m, rng, counter, deleted) if len(m.clusters) < caps["max_clusters"] - 8 else ""
                pk.flush()
                _, got = packer_check(m, oracle_mod, lean=True)
                outs.append((tag, got))
            (tag, got), (_, twin) = outs
            assert not twin.diff(got), e
            inc, twin_inc = incremental(got, got.clusters.shape[0]), incremental(twin, twin.clusters.shape[0])
            tally[f"{tag}: {'inc' if inc else 'full'} / twin {'inc' if twin_inc else 'full'}"] += 1
            tally["incremental"] += inc
            tally["twin incremental"] += twin_inc
        print("packer large moves", dict(tally))
        gained = sum(n for k, n in tally.items() if k.endswith("inc / twin full"))
        assert tally["incremental"] >= tally["twin incremental"] and gained >= 1, dict(tally)
    finally:
        on.close()
        off.close()


def test_group_packer_against_option_off(oracle_mod):
    caps = dict(PACKER_CAPS, max_clusters=128, max_groups=1024, max_wtd=1024, max_pods=8192, max_jobs=256, max_creates=1 << 20)
    gp = GroupPacker([0, 0], **caps, **ss.ALL, large_moves=True)
    try:
        assert all(sh.engine.get_option(abi.OPT_LARGE_MOVES) == 1 for sh in gp.shards)
        clusters, pods, jobs = objects(9)
        for c in clusters:
            gp.upsert_cluster(c)
        for p in pods:
            gp.upsert_pod(p)
        gp.flush()
        flags = gp.flags(fetch_pod_lists=0)
        gp.reconcile(flags)
        rng = np.random.default_rng(4)
        live = list(clusters)
        n_inc = 0
        for e in range(12):
            c = copy.deepcopy(live[int(rng.integers(len(live)))])
            ns = c.get("namespace", "default")
            if e % 3 == 0:
                gp.delete_cluster(ns, c["name"])
                live = [x for x in live if (x.get("namespace", "default"), x["name"]) != (ns, c["name"])]
            elif e % 3 == 1:
                c["spec"].setdefault("workerGroupSpecs", []).append({"groupName": f"extra{e}", "replicas": 2, "minReplicas": 0,
                                                                      "maxReplicas": 4, "numOfHosts": 1})
                c["generation"] = c.get("generation", 1) + 1
                gp.upsert_cluster(c)
            else:
                src = [p for p in pods if p.get("namespace", "default") == ns and p["labels"].get("ray.io/cluster") == c["name"]]
                for k in range(300 if src else 0):
                    q = copy.deepcopy(src[k % len(src)])
                    q["name"] = f"{q['name']}-g{e}-{k}"
                    gp.upsert_pod(q)
            gp.flush()
            got = gp.reconcile(flags)
            n_inc += sum(incremental(g, g.clusters.shape[0]) for g in got)
            for sh, g, fl in zip(gp.shards, got, flags):
                sh.engine.set_incremental(False)
                full = sh.engine.reconcile(fl)
                sh.engine.set_incremental(True)
                assert not full.diff(g), e
            gp.reconcile(flags)
        print("group packer large moves: incremental shard passes", n_inc)
        assert n_inc >= 2 * 12 - 2, n_inc  # (without the option, test_gpu_structural_streams.py allows four full passes here)
    finally:
        gp.close()

"""kr_snapshot_commit_json_moves and KR_OPT_JSON_MOVES: a compaction of the JSON arena moves the unchanged specs inside the device
arena (k_json_move_gather / k_json_move_scatter) instead of re-sending the arena, and no digest is recomputed.

Engine level, every epoch equals the CPU oracle and a twin engine fed the same layout through KR_PART_JSON: permuted re-layouts
(blobs moving up and down, onto other listed blobs' sources and onto their own), invalid move lists, a row whose bytes a move
overwrote, and moves beside spec rows, object rows, a whole JSON part and a skip_hash pass.  Native and group packers with
KR_OPT_SPEC_ROWS, every structural option and a small JSON arena run against a twin without KR_OPT_JSON_MOVES, through both
compaction triggers."""
import copy

import numpy as np
import pytest

from harness import OBJ_COLS, Mirror, SpecDriver, b32, events, flip_ready, incremental, members, objects, packer_check, with_json
from kuberay_b200 import abi, synthetic
from kuberay_b200.engine import Engine, EngineError
from kuberay_b200.packer import GroupPacker, Packer

pytestmark = pytest.mark.gpu

STRUCTURAL = dict(large_clusters=True, wide_clusters=True, huge_clusters=True, wtd_edits=True, spec_rows=True, cluster_creates=True,
                  cluster_deletes=True, group_edits=True, large_growth=True, large_moves=True)


def pad(n):
    return (int(n) + 15) // 16 * 16


def _snap(seed, **kw):
    p = dict(n_clusters=300, pods_per_cluster=16, groups=3, recreate_frac=0.2, seed=seed)
    p.update(kw)
    return synthetic.generate(synthetic.config("C2", **p))


class MoveDriver(SpecDriver):
    """A SpecDriver whose arena can be laid out again: relayout() places every blob anew, move() commits the moves on the first
    engine (the twin takes the whole JSON part and the object part)."""

    def relayout(self, order, start=0, bodies=None):
        """Every RayCluster's blob in `order` from byte `start` on (16-byte aligned, zero padded), `bodies` replacing some.
        -> the rows whose range changed and whose bytes stayed."""
        s = self.snap
        body = {c: self.body(c) for c in range(s.dims["clusters"])}
        body.update(bodies or {})
        need = start + sum(pad(len(b)) for b in body.values())
        new = with_json(s, max(need, s.dims["json"]))
        new.json[:] = 0
        moved, off = [], start
        for c in order:
            c = int(c)
            b = body[c]
            new.json[off:off + len(b)] = np.frombuffer(b, dtype=np.uint8)
            if off != int(s.c_json_off[c]) and c not in (bodies or {}):
                moved.append(c)
            new.c_json_off[c], new.c_json_len[c] = off, len(b)
            off += pad(len(b))
        self.use(new)
        return moved

    def stage(self):
        np.copyto(self.views["json"], self.snap.json)
        for name in ("c_json_off", "c_json_len"):
            self.views[name][:] = self.snap.cols[name]

    def move(self, rows, twin=True):
        self.stage()
        self.eng.commit_json_moves(rows)
        if twin:
            np.copyto(self.twin.views["json"], self.snap.json)
            self.twin.commit_objects(abi.PART_OBJECTS | abi.PART_JSON)


def _by_offset(snap):
    return np.argsort(snap.c_json_off[:snap.dims["clusters"]], kind="stable")


def _hash_kernels(names):
    return [k for k in names if k.startswith("k_hash")]


@pytest.mark.parametrize("layout", ["shuffle", "shift", "reverse"])
def test_permuted_relayout(layout, oracle_mod):
    snap, flags = _snap(21)
    dr = MoveDriver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        order = _by_offset(dr.snap)
        if layout == "shuffle":
            rows = dr.relayout(np.random.default_rng(3).permutation(order))
        elif layout == "shift":  # every blob 16 bytes up: each destination overlaps its own source
            rows = dr.relayout(order, start=16)
        else:
            rows = dr.relayout(order[::-1])
        assert len(rows) > 100
        dr.move(rows)
        got, names = dr.check(oracle_mod, profiled=True, h2d=24 * len(rows), h2d_after=24 * len(rows))
        assert got.n_changed == 0, got.n_changed  # no Recreate-gated RayCluster re-decided either
        assert not _hash_kernels(names), names
        # a full pass re-hashes every spec from the moved device bytes
        dr.eng.set_incremental(False)
        got, _ = dr.check(oracle_mod, expect_incremental=False)
        for c in range(0, dr.snap.dims["clusters"], 7):
            assert bytes(got.hash[c]) == b32(dr.body(c))
        dr.eng.set_incremental(True)
        rows = dr.relayout(np.random.default_rng(4).permutation(order))  # and again from there
        dr.move(rows)
        dr.check(oracle_mod, expect_incremental=None)  # (the full passes need not have left the resident state)
    finally:
        dr.close()


def test_invalid_lists_commit_nothing(oracle_mod):
    snap, flags = _snap(22)
    dr = MoveDriver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        nc = dr.snap.dims["clusters"]
        rows = dr.relayout(np.random.default_rng(5).permutation(nc))
        dr.stage()
        v = dr.views
        a, b = [c for c in rows if dr.snap.c_json_len[c] > 0][:2]

        def bad(lst, col=None, row=None, value=None):
            if col is not None:
                keep = v[col][row].copy()
                v[col][row] = value
            try:
                with pytest.raises(EngineError) as ei:
                    dr.eng.commit_json_moves(lst)
                assert ei.value.code == abi.KR_E_INVALID, ei.value
            finally:
                if col is not None:
                    v[col][row] = keep

        bad(rows + [nc])                                             # past n_clusters
        bad(rows + [rows[3]])                                        # repeated
        bad(rows, "c_json_len", a, int(v["c_json_len"][a]) + 1)      # another length
        bad(rows, "c_json_off", a, int(v["c_json_off"][a]) + 8)      # not 16-byte aligned
        bad(rows, "c_json_off", a, pad(dr.snap.dims["json"]) + 16)   # past json_bytes
        bad(rows, "c_json_off", a, int(v["c_json_off"][b]))          # two destinations overlap
        dr.move(rows)
        got, _ = dr.check(oracle_mod, h2d=24 * len(rows))
        assert got.n_changed == 0
    finally:
        dr.close()


def test_before_a_full_commit_is_a_state_error():
    snap, _ = _snap(23, n_clusters=20)
    eng = Engine.for_snapshot(snap)
    try:
        eng.begin(snap.sizes())
        with pytest.raises(EngineError) as ei:
            eng.commit_json_moves([0])
        assert ei.value.code == abi.KR_E_STATE
    finally:
        eng.close()


def test_overwritten_row_blocks_the_pass_until_its_spec_comes(oracle_mod):
    snap, flags = _snap(24)
    dr = MoveDriver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        s = dr.snap
        plain = [c for c in range(s.dims["clusters"]) if s.c_json_len[c] > 0]
        a, b = next((a, b) for a in plain for b in plain if a != b and pad(s.c_json_len[a]) <= pad(s.c_json_len[b]))
        end = pad(s.dims["json"])
        new = with_json(s, end + pad(s.c_json_len[b]))
        body_a, body_b = dr.body(a), dr.body(b)
        ob = int(s.c_json_off[b])
        new.json[ob:ob + pad(len(body_b))] = 0
        new.json[ob:ob + len(body_a)] = np.frombuffer(body_a, dtype=np.uint8)      # a moves onto b's range ...
        new.json[end:end + len(body_b)] = np.frombuffer(body_b, dtype=np.uint8)    # ... and b to the end (not listed)
        new.c_json_off[a], new.c_json_off[b] = ob, end
        dr.use(new)
        dr.move([a])
        with pytest.raises(EngineError) as ei:
            dr.eng.reconcile(dr.flags)
        assert ei.value.code == abi.KR_E_STATE and f"cluster {b}" in str(ei.value), ei.value
        dr.eng.commit_spec_rows([b])
        got, _ = dr.check(oracle_mod)
        assert bytes(got.hash[a]) == b32(body_a) and bytes(got.hash[b]) == b32(body_b)
    finally:
        dr.close()


@pytest.mark.parametrize("other", ["spec_rows", "object_rows", "part_json", "skip_hash"])
def test_moves_with_other_commits(other, oracle_mod):
    snap, flags = _snap(25)
    if other == "skip_hash":
        flags.skip_hash = 1
    dr = MoveDriver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        nc = dr.snap.dims["clusters"]
        rng = np.random.default_rng(6)
        edited = {}
        if other == "skip_hash":  # a spec row left pending by a skip_hash pass moves before it is hashed
            c = 5
            dr.edit(c, dr.body(c) + b"   ", move=True)
            dr.commit_specs()
            dr.check(oracle_mod)
            edited_pending = c
        if other == "spec_rows":
            recreate = [c for c in range(nc) if dr.snap.c_flags[c] & abi.CF_UPGRADE_RECREATE]
            for c in recreate[:2] + [int(x) for x in rng.choice(nc, 4, replace=False)]:
                edited[c] = dr.body(c)[:-3] + b"xyz" + b" " * int(rng.integers(0, 40))
        rows = dr.relayout(rng.permutation(nc), bodies=edited)
        dr.move(rows)
        if other == "spec_rows":
            dr.stage()
            dr.eng.commit_spec_rows(sorted(edited))
            dr.check(oracle_mod)
        elif other == "object_rows":
            s = dr.snap
            r = int(rng.integers(nc))
            pods = members(s, r)[:3]
            flip_ready(s, pods)
            s.c_old_counts[5 * r] += 1
            for col in OBJ_COLS:
                np.copyto(dr.views[col], s.cols[col])
            dr.eng.commit_object_rows([r], [])
            dr.twin.commit_objects()
            dr.commit_rows(pods)
            got, _ = dr.check(oracle_mod)
            assert got.n_changed <= 2
        elif other == "part_json":  # the whole part wins
            dr.eng.commit(abi.PART_JSON)
            dr.check(oracle_mod, expect_incremental=None)
        else:
            dr.flags.skip_hash = 0
            got, _ = dr.check(oracle_mod, expect_incremental=None)
            assert bytes(got.hash[edited_pending]) == b32(dr.body(edited_pending))
    finally:
        dr.close()


# ------------------------------------------------------------------------------------------------ packers
TRIGGERS = {
    # a full arena inside cluster_upsert: 64 KB hold at most 64 KB of dead bytes, so the flush's rule (more than 1 MiB) never fires
    "full": dict(max_json_bytes=64 << 10, burst=3),
    # dead bytes past half the cursor and 1 MiB at flush (every fifth epoch rewrites the hot specs 800 times), long before 4 MiB
    # fill up
    "flush": dict(max_json_bytes=4 << 20, burst=800),
}
CAPS = dict(max_clusters=128, max_groups=1024, max_wtd=1024, max_pods=8192, max_heads=256, max_jobs=128, max_creates=1 << 20)


def _epoch(m, rng, counter, gen, hot, reps):
    """Informer events, then the hot RayClusters' specs rewritten `reps` times each (dead bytes), then maybe a RayCluster deleted,
    created or given a worker group."""
    events(rng, m, counter, structural=False)
    for _ in range(reps):
        for key in hot:
            if key in m.clusters and rng.random() < 0.7:
                c = dict(m.clusters[key])
                c.pop("specJson", None)
                c["spec"] = dict(c["spec"], rayVersion="v" + "9" * int(rng.integers(500, 2000)))
                gen[0] += 1
                c["generation"], c["resourceVersion"] = gen[0], 10_000 + gen[0]
                m.upsert_cluster(c)
    keys = [k for k in sorted(m.clusters) if k not in hot]
    u = rng.random()
    counter[0] += 1
    if not keys:
        return
    if u < 0.15 and len(keys) > 6:
        m.delete_cluster(*keys[int(rng.integers(len(keys)))])
    elif u < 0.3:
        src = copy.deepcopy(m.clusters[keys[int(rng.integers(len(keys)))]])
        src["name"], src["generation"], src["resourceVersion"] = f"{src['name']}-c{counter[0]}", 1, 50_000 + counter[0]
        m.upsert_cluster(src)
    elif u < 0.45:
        c = copy.deepcopy(m.clusters[keys[int(rng.integers(len(keys)))]])
        c["spec"].setdefault("workerGroupSpecs", []).append({"groupName": f"added-{counter[0]}", "replicas": 1, "minReplicas": 0,
                                                              "maxReplicas": 4, "numOfHosts": 1})
        c["generation"] = c.get("generation", 1) + 1
        c["resourceVersion"] = 70_000 + counter[0]
        m.upsert_cluster(c)


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("trigger", ["full", "flush"])
def test_native_packer_streams(trigger, seed, oracle_mod):
    t = TRIGGERS[trigger]
    caps = dict(CAPS, max_json_bytes=t["max_json_bytes"])
    on, off = Packer(**caps, **STRUCTURAL, json_moves=True), Packer(**caps, **STRUCTURAL)
    try:
        assert on.engine.get_option(abi.OPT_JSON_MOVES) == 1 and off.engine.get_option(abi.OPT_JSON_MOVES) == 0
        objs = objects(seed, max_clusters=40)
        ms = [Mirror(*copy.deepcopy(objs), pk) for pk in (on, off)]
        for pk, m in zip((on, off), ms):
            assert pk.flush() == abi.PACK_FULL
            packer_check(m, oracle_mod, lean=True)
        hot = sorted(ms[0].clusters)[:4]
        state = [([0], [1]), ([0], [1])]  # (counter, last generation: the fuzz objects are at generation 1)
        compactions = inc_compactions = 0
        for epoch in range(40):
            outs = []
            for (counter, gen), m, pk in zip(state, ms, (on, off)):
                reps = t["burst"] if trigger == "full" or epoch % 5 == 4 else 1
                _epoch(m, np.random.default_rng(1000 * seed + epoch), counter, gen, hot, reps)
                mode = pk.flush()
                _, got = packer_check(m, oracle_mod, lean=True)
                outs.append((mode, got))
            (mode, got), (tmode, twin) = outs
            d = twin.diff(got)
            assert not d, (epoch, d[:6])
            inc, tinc = incremental(got, got.clusters.shape[0]), incremental(twin, twin.clusters.shape[0])
            assert inc or not tinc, (epoch, mode, tmode)
            if tmode & abi.PART_JSON:  # the twin compacted (with every structural option, nothing else sends the arena)
                compactions += 1
                inc_compactions += inc
                assert mode & abi.PACK_JSON_MOVES and not mode & abi.PART_JSON, (epoch, mode, tmode)
                assert mode & ~abi.PACK_JSON_MOVES & ~abi.PACK_SPEC_ROWS == tmode & ~abi.PART_JSON & ~abi.PACK_SPEC_ROWS, (epoch, mode, tmode)
                if inc and tinc:
                    assert got.n_changed <= twin.n_changed, (epoch, got.n_changed, twin.n_changed)
            else:
                assert mode == tmode, (epoch, mode, tmode)
        print(trigger, seed, "compactions", compactions, "incremental", inc_compactions)
        assert compactions >= 2 and inc_compactions >= 1, (compactions, inc_compactions)
    finally:
        on.close()
        off.close()


def test_group_packer_two_shards(oracle_mod):
    caps = dict(CAPS, max_json_bytes=TRIGGERS["full"]["max_json_bytes"])
    gps = [GroupPacker([0, 0], **caps, **STRUCTURAL, json_moves=True), GroupPacker([0, 0], **caps, **STRUCTURAL)]
    try:
        clusters, pods, jobs = objects(7, max_clusters=40)
        for gp in gps:
            for c in clusters:
                gp.upsert_cluster(copy.deepcopy(c))
            for p in pods:
                gp.upsert_pod(copy.deepcopy(p))
            gp.flush()
            gp.reconcile(gp.flags(fetch_pod_lists=0))
        keys = sorted((c.get("namespace", "default"), c["name"]) for c in clusters)
        live = {(c.get("namespace", "default"), c["name"]): c for c in clusters}
        rng = np.random.default_rng(8)
        moved = 0
        for epoch in range(30):
            edits = []
            for key in keys[:8] * 3:
                c = dict(live[key])
                c.pop("specJson", None)
                c["spec"] = dict(c["spec"], rayVersion="v" + "9" * int(rng.integers(500, 2000)))
                c["generation"], c["resourceVersion"] = 100 + len(edits) + 100 * epoch, 20_000 + 100 * epoch + len(edits)
                live[key] = c
                edits.append(c)
            outs = []
            for gp in gps:
                for c in edits:
                    gp.upsert_cluster(copy.deepcopy(c))
                modes = gp.flush()
                outs.append((modes, gp.reconcile(gp.flags(fetch_pod_lists=0))))
            (modes, got), (tmodes, twin) = outs
            for s in range(2):
                d = twin[s].diff(got[s])
                assert not d, (epoch, s, d[:6])
                if tmodes[s] & abi.PART_JSON:
                    moved += 1
                    assert modes[s] & abi.PACK_JSON_MOVES and not modes[s] & abi.PART_JSON, (epoch, s, modes[s])
                    assert incremental(got[s], got[s].clusters.shape[0]), (epoch, s)
                else:
                    assert modes[s] == tmodes[s], (epoch, s, modes[s], tmodes[s])
        assert moved >= 2, moved
    finally:
        for gp in gps:
            gp.close()


@pytest.mark.parametrize("side", ["without_spec_rows", "off"])
def test_option_settings(side, oracle_mod):
    """With KR_OPT_SPEC_ROWS off the option changes nothing; with the option off no move kernel runs."""
    torch = pytest.importorskip("torch")
    from torch.profiler import ProfilerActivity, profile
    caps = dict(CAPS, max_json_bytes=TRIGGERS["full"]["max_json_bytes"])
    opts = dict(STRUCTURAL, spec_rows=False) if side == "without_spec_rows" else STRUCTURAL
    on = Packer(**caps, **opts, json_moves=side != "off")
    off = Packer(**caps, **dict(opts))
    try:
        objs = objects(3, max_clusters=40)
        ms = [Mirror(*copy.deepcopy(objs), pk) for pk in (on, off)]
        for pk in (on, off):
            pk.flush()
        hot = sorted(ms[0].clusters)[:4]
        state = [([0], [1]), ([0], [1])]  # (counter, last generation: the fuzz objects are at generation 1)
        compacted, launched = 0, []
        for epoch in range(16):
            outs = []
            for (counter, gen), m, pk in zip(state, ms, (on, off)):
                _epoch(m, np.random.default_rng(77 + epoch), counter, gen, hot, TRIGGERS["full"]["burst"])
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    mode = pk.flush()
                    torch.cuda.synchronize()
                launched += [e.name for e in prof.events() if "k_json_move" in e.name]
                _, got = packer_check(m, oracle_mod, lean=True)
                outs.append((mode, got))
            (mode, got), (tmode, twin) = outs
            assert mode == tmode, (epoch, mode, tmode)
            assert not twin.diff(got)
            compacted += bool(tmode & abi.PART_JSON)
        assert compacted >= 1, compacted
        assert not launched, launched[:4]
    finally:
        on.close()
        off.close()

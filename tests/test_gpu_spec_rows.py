"""kr_snapshot_commit_spec_rows: an edit of a RayCluster's muted spec travels as its own JSON range plus two column entries; the
next pass re-hashes only the listed messages (k_hash3 / k_hash2 over the row list), re-decides only the listed Recreate-gated
RayClusters (k_inc_mark_rows) and fetches only their digests (k_inc_digest_gather).

Every epoch is compared with the CPU oracle (digests included), with a second engine fed the same stream through KR_PART_JSON,
records the pass did not name must be unchanged, and the epoch must stay incremental."""
import copy

import numpy as np
import pytest

from harness import (PACKER_CAPS, Mirror, SpecDriver, arena_stream, b32, device_incremental, events, flip_ready, incremental, objects,
                     packer_check, packer_stream, spec_edits)
from kuberay_b200 import abi, synthetic
from kuberay_b200.engine import Engine, EngineError
from kuberay_b200.live import LiveArena
from kuberay_b200.packer import Packer

pytestmark = pytest.mark.gpu


def _snap(seed, **kw):
    p = dict(n_clusters=300, pods_per_cluster=16, groups=3, recreate_frac=0.2, seed=seed)
    p.update(kw)
    return synthetic.generate(synthetic.config("C2", **p))


def counted(dr, rows):
    return sum(16 + (int(dr.snap.c_json_len[c]) + 15) // 16 * 16 for c in set(int(r) for r in rows))


def _plain_rows(snap, k, start=0):
    return [c for c in range(start, snap.dims["clusters"]) if not snap.c_flags[c] & abi.CF_UPGRADE_RECREATE][:k]


def _recreate_rows(snap):
    return [c for c in range(snap.dims["clusters"]) if snap.c_flags[c] & abi.CF_UPGRADE_RECREATE]


def _mutate(b: bytes, salt: int) -> bytes:
    x = bytearray(b)
    x[len(x) // 2] = ord("a") + salt % 26
    return bytes(x)


def test_edit_in_place_and_moved(oracle_mod):
    snap, flags = _snap(1)
    dr = SpecDriver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rows = _plain_rows(snap, 4)
        dr.edit(rows[0], _mutate(dr.body(rows[0]), 1))                     # same length, same range
        dr.edit(rows[1], dr.body(rows[1]) + b' ', move=True)               # one byte longer, at the arena's end
        dr.edit(rows[2], dr.body(rows[2])[:-40])                           # shorter: new range
        dr.commit_specs()
        got, names = dr.check(oracle_mod, profiled=True, h2d=counted(dr, rows[:3]), h2d_after=counted(dr, rows[:3]) + 4 * 3)
        assert "k_hash_rows" in names and "k_hash" not in names and "k_inc_mark_recreate" not in names, names
        for c in rows[:3]:
            assert bytes(got.hash[c]) == b32(dr.body(c))
    finally:
        dr.close()


@pytest.mark.parametrize("length", [55, 56, 63, 64, 119, 120, 1, 0])
def test_sha1_padding_edges(length, oracle_mod):
    snap, flags = _snap(2)
    dr = SpecDriver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rows = _plain_rows(snap, 3)
        for i, c in enumerate(rows):
            dr.edit(c, bytes((ord("{") + i + k) % 256 for k in range(length)), move=(i == 1))
        dr.commit_specs()
        got, _ = dr.check(oracle_mod, h2d=counted(dr, rows))
        for c in rows:
            assert bytes(got.hash[c]) == b32(dr.body(c))
    finally:
        dr.close()


def test_recreate_gate_switches_and_unedited_gates_stay(oracle_mod):
    snap, flags = _snap(3)
    dr = SpecDriver(snap, flags)
    try:
        first, _ = dr.check(oracle_mod, expect_incremental=False)
        rec = _recreate_rows(snap)
        # a Recreate RayCluster whose head annotation matches today's digest (no delete-all yet)
        s = dr.snap
        head_of = {(int(s.p_ns_id[p]), int(s.p_cluster_name_id[p])): h for h, p in enumerate(s.h_pod_idx.tolist())}
        def annotated(c):
            h = head_of.get((int(s.c_ns_id[c]), int(s.c_name_id[c])))
            return h is not None and s.h_annot_state[h] == abi.ANNOT_HASH32 and s.h_version_state[h] == abi.VER_CURRENT and \
                bytes(s.h_annot_hash.reshape(-1, 32)[h]) == b32(dr.body(c))
        on = [c for c in rec if first.clusters["path"][c] == abi.PATH_NORMAL and annotated(c)]
        assert len(on) >= 1 and len(rec) >= 6, (len(on), len(rec))
        c = on[0]
        old = dr.body(c)
        dr.edit(c, _mutate(old, 7))
        dr.commit_specs()
        got, names = dr.check(oracle_mod, profiled=True)
        assert "k_inc_mark_rows" in names and "k_inc_mark_recreate" not in names, names
        assert got.clusters["path"][c] == abi.PATH_RECREATE_DELETE_ALL != first.clusters["path"][c]
        assert set(got.changed_clusters.tolist()) == {c}  # no other Recreate RayCluster was re-decided
        dr.edit(c, old)  # back to the annotated spec: delete-all switches off
        dr.commit_specs()
        got, _ = dr.check(oracle_mod)
        assert got.clusters["path"][c] == first.clusters["path"][c]
        assert set(got.changed_clusters.tolist()) == {c}
    finally:
        dr.close()


@pytest.mark.parametrize("specs_first", [True, False])
def test_edit_with_pod_churn_and_object_rows(specs_first, oracle_mod):
    snap, flags = _snap(4)
    dr = SpecDriver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rec = _recreate_rows(snap)
        rows = rec[:2] + _plain_rows(snap, 2)
        for c in rows:
            dr.edit(c, dr.body(c) + b"  ", move=True)
        dr.apply()
        pods =np.flatnonzero((dr.snap.p_cluster_name_id == dr.snap.c_name_id[rows[0]]) & (dr.snap.p_ns_id == dr.snap.c_ns_id[rows[0]]))[:3]
        flip_ready(dr.snap, pods)
        dr.snap.c_old_counts[5 * rows[1]] += 1
        if specs_first:
            dr.commit_specs()
            dr.commit_objects(twin=False)
            dr.commit_rows(pods)
        else:  # the object commit finds moved ranges: the whole re-hash, still incremental
            dr.commit_objects(twin=False)
            dr.commit_rows(pods)
            dr.commit_specs()
        dr.check(oracle_mod)
    finally:
        dr.close()


def test_repeated_rows_and_two_calls(oracle_mod):
    snap, flags = _snap(5)
    dr = SpecDriver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rows = _plain_rows(snap, 6)
        for c in rows:
            dr.edit(c, _mutate(dr.body(c), c))
        dr.commit_specs(rows=rows + rows[:3] + rows[::2], calls=3)
        got, _ = dr.check(oracle_mod, h2d=counted(dr, rows), h2d_after=counted(dr, rows) + 4 * len(rows))
        for c in rows:
            assert bytes(got.hash[c]) == b32(dr.body(c))
    finally:
        dr.close()


def test_spec_rows_with_whole_arena_commit(oracle_mod):
    snap, flags = _snap(6)
    dr = SpecDriver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        a, b = _plain_rows(snap, 2)
        dr.edit(a, _mutate(dr.body(a), 3))
        dr.commit_specs()
        dr.edit(b, _mutate(dr.body(b), 4))
        dr.apply()
        np.copyto(dr.views["json"], dr.snap.json)
        dr.eng.commit(abi.PART_JSON)  # (the whole arena wins)
        dr.commit_specs(rows=[b])
        _, names = dr.check(oracle_mod, profiled=True)
        assert "k_hash" in names and "k_hash_rows" not in names, names
    finally:
        dr.close()


def test_state_errors_and_full_pass_without_resident_state(oracle_mod):
    snap, flags = _snap(7)
    d = snap.dims
    e = Engine.for_snapshot(snap, slack=1.5)
    try:
        e.begin(snap.sizes())
        with pytest.raises(EngineError) as ei:
            e.commit_spec_rows([0])
        assert ei.value.code == abi.KR_E_STATE
    finally:
        e.close()
    dr = SpecDriver(snap, flags)
    try:
        # committed but never reconciled: no resident state, the bytes land and the full pass hashes everything
        c = _plain_rows(snap, 1)[0]
        dr.edit(c, _mutate(dr.body(c), 9), move=True)
        dr.commit_specs()
        got, _ = dr.check(oracle_mod, expect_incremental=False)
        assert bytes(got.hash[c]) == b32(dr.body(c))
        # an option toggle drops the resident state as well
        dr.edit(c, _mutate(dr.body(c), 10))
        dr.commit_specs()
        dr.eng.set_incremental(False)
        dr.check(oracle_mod, expect_incremental=False)
        dr.eng.set_incremental(True)
        dr.check(oracle_mod, expect_incremental=False)
        assert d["clusters"] == dr.snap.dims["clusters"]
    finally:
        dr.close()


def test_skip_hash_leaves_rows_pending(oracle_mod):
    snap, flags = _snap(8)
    flags.skip_hash = 1
    dr = SpecDriver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        c = _plain_rows(snap, 1)[0]
        dr.edit(c, _mutate(dr.body(c), 11))
        dr.commit_specs()
        dr.check(oracle_mod)
        dr.flags.skip_hash = 0  # other flags: the full pass hashes the listed message with the others
        got, _ = dr.check(oracle_mod, expect_incremental=False)
        assert bytes(got.hash[c]) == b32(dr.body(c))
        dr.edit(c, _mutate(dr.body(c), 12))
        dr.commit_specs()
        got, _ = dr.check(oracle_mod)
        assert bytes(got.hash[c]) == b32(dr.body(c))
    finally:
        dr.close()


@pytest.mark.parametrize("moved", [False, True])
def test_row_edited_again_after_skip_hash_passes(moved, oracle_mod):
    """A skip_hash pass leaves the rows pending; once it has returned the caller may rewrite them, and a second commit of the same
    row must pull the new bytes (it is hashed once, by the next pass that hashes)."""
    snap, flags = _snap(12)
    flags.skip_hash = 1
    dr = SpecDriver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        c, other = _recreate_rows(snap)[0], _plain_rows(snap, 1)[0]
        dr.edit(c, _mutate(dr.body(c), 1))
        dr.edit(other, _mutate(dr.body(other), 2))
        dr.commit_specs()
        dr.check(oracle_mod)
        dr.edit(c, _mutate(dr.body(c), 3))                            # in place, same row, still pending
        dr.commit_specs()
        dr.check(oracle_mod)
        dr.edit(c, dr.body(c) + b"   ", move=moved)                  # then longer: a new range (moved) or the padded one
        dr.commit_specs()
        if moved:
            dr.commit_objects(twin=False)
        dr.check(oracle_mod)
        dr.flags.skip_hash = 0  # the next pass hashes: the full pass over the arena as it now is on the device
        got, _ = dr.check(oracle_mod, expect_incremental=False)
        assert bytes(got.hash[c]) == b32(dr.body(c)) and bytes(got.hash[other]) == b32(dr.body(other))
        dr.edit(c, _mutate(dr.body(c), 4))
        dr.commit_specs()
        got, _ = dr.check(oracle_mod)
        assert bytes(got.hash[c]) == b32(dr.body(c))
    finally:
        dr.close()


FLEETS = {  # smaller forms of C3L / C3H / C3W / C3MH
    "large": ("C3L", dict(n_clusters=300, pods_per_cluster=20, large_pods=1200, n_large=3)),
    "huge": ("C3H", dict(n_clusters=700, pods_per_cluster=20, large_pods=9000, n_large=1)),
    "wide": ("C3W", dict(n_clusters=300, pods_per_cluster=60, n_wide=6)),
    "multihost": ("C3MH", dict(n_clusters=300, pods_per_cluster=41, groups=2, multihost_frac=0.5)),
}


def _special_rows(snap, kind):
    d = snap.dims
    if kind == "wide":
        return [c for c in range(d["clusters"]) if snap.c_group_cnt[c] > 32]
    if kind == "multihost":
        return sorted({int(snap.g_cluster_idx[g]) for g in np.flatnonzero(snap.g_num_hosts > 1)})[:12]
    key = {(int(a), int(b)): c for c, (a, b) in enumerate(zip(snap.c_ns_id, snap.c_name_id))}
    cnt = np.zeros(d["clusters"], dtype=np.int64)
    for a, b in zip(snap.p_ns_id.tolist(), snap.p_cluster_name_id.tolist()):
        c = key.get((a, b))
        if c is not None:
            cnt[c] += 1
    return np.flatnonzero(cnt > (abi.LARGE_MAX_PODS if kind == "huge" else 256)).tolist()


@pytest.mark.parametrize("kind", sorted(FLEETS))
def test_edits_inside_large_huge_wide_and_multihost_clusters(kind, oracle_mod):
    """Spec edits of exactly the RayClusters the per-cluster kernels (k_large_sort / k_huge_* / k_decide_large) or the multi-host
    decide take, half of them Recreate-gated: one of those with a head annotation equal to its digest, so delete-all switches on and
    back off."""
    name, kw = FLEETS[kind]
    snap, flags = synthetic.generate(synthetic.config(name, recreate_frac=0.0, **kw))
    special = _special_rows(snap, kind)
    assert special, kind
    s = snap
    head_of = {(int(s.p_ns_id[p]), int(s.p_cluster_name_id[p])): h for h, p in enumerate(s.h_pod_idx.tolist())}
    gated = [c for c in special[::2] if (int(s.c_ns_id[c]), int(s.c_name_id[c])) in head_of]
    assert gated, kind
    ann = s.h_annot_hash.reshape(-1, 32)
    for i, c in enumerate(gated):
        s.c_flags[c] |= abi.CF_UPGRADE_RECREATE
        h = head_of[(int(s.c_ns_id[c]), int(s.c_name_id[c]))]
        s.h_annot_state[h], s.h_version_state[h] = abi.ANNOT_HASH32, abi.VER_CURRENT
        o, n = int(s.c_json_off[c]), int(s.c_json_len[c])
        ann[h] = np.frombuffer(b32(s.json[o:o + n].tobytes() if i == 0 else b"another spec"), dtype=np.uint8)
    opts = dict(large_clusters=True, wide_clusters=True, huge_clusters=True, wtd_edits=True)
    dr = SpecDriver(snap, flags, json_room=4 << 20, **opts)
    try:
        first, _ = dr.check(oracle_mod, expect_incremental=False)
        assert first.clusters["path"][gated[0]] == abi.PATH_NORMAL
        original = dr.body(gated[0])
        for rnd in range(4):
            rows = special if rnd != 2 else [gated[0]]
            for c in rows:
                dr.edit(c, original if (rnd == 2) else _mutate(dr.body(c), rnd) + b" " * (rnd % 2) * 20, move=bool((c + rnd) % 2))
            dr.commit_specs()
            # (switching delete-all of a large RayCluster on or off may outgrow the places its decide kept: that epoch may take the
            # full pass; the others must stay incremental)
            got, names = dr.check(oracle_mod, expect_incremental=None if rnd in (0, 2) else True, profiled=True)
            if incremental(got, dr.snap.dims["clusters"]):
                assert "k_hash_rows" in names and "k_inc_mark_rows" in names and "k_hash" not in names, names
            if got.changed_clusters is not None:
                assert set(got.changed_clusters.tolist()) <= set(gated), (kind, rnd)
            want = abi.PATH_NORMAL if rnd == 2 else abi.PATH_RECREATE_DELETE_ALL
            assert got.clusters["path"][gated[0]] == want, (kind, rnd)
    finally:
        dr.close()


def test_throughput_regime_every_row_edited(oracle_mod):
    """More than 4 x SMs x 32 listed rows: the pass takes k_hash2 over the row list."""
    snap, flags = _snap(10, n_clusters=17000, pods_per_cluster=2, groups=1, recreate_frac=0.01)
    dr = SpecDriver(snap, flags, json_room=64 << 20)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rows = list(range(snap.dims["clusters"]))
        for c in rows:
            dr.edit(c, _mutate(dr.body(c), c), move=(c % 3 == 0))
        dr.commit_specs()
        got, _ = dr.check(oracle_mod, h2d=counted(dr, rows))
    finally:
        dr.close()


def test_invalid_rows_offsets_and_ranges(oracle_mod):
    snap, flags = _snap(11)
    dr = SpecDriver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        nc = snap.dims["clusters"]
        with pytest.raises(EngineError) as ei:
            dr.eng.commit_spec_rows([0, nc])
        assert ei.value.code == abi.KR_E_INVALID
        v = dr.views
        off, ln = int(v["c_json_off"][1]), int(v["c_json_len"][1])
        v["c_json_off"][1] = off + 8
        with pytest.raises(EngineError) as ei:
            dr.eng.commit_spec_rows([1])
        assert ei.value.code == abi.KR_E_INVALID
        v["c_json_off"][1] = (snap.dims["json"] - 16) // 16 * 16
        v["c_json_len"][1] = 64
        with pytest.raises(EngineError) as ei:
            dr.eng.commit_spec_rows([1])
        assert ei.value.code == abi.KR_E_INVALID
        v["c_json_off"][1], v["c_json_len"][1] = off, ln
        dr.check(oracle_mod)  # nothing was committed
    finally:
        dr.close()


@pytest.mark.parametrize("seed", [1, 2])
def test_stream_through_the_engine(seed, oracle_mod):
    rng = np.random.default_rng(seed)
    snap, flags = _snap(30 + seed, n_clusters=400, groups=2)
    dr = SpecDriver(snap, flags, json_room=8 << 20)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        n_inc = 0
        nc = snap.dims["clusters"]
        for epoch in range(40):
            for c in rng.choice(nc, int(rng.integers(1, 12)), replace=False):
                b = dr.body(c)
                k = int(rng.integers(0, 3))
                dr.edit(c, _mutate(b, epoch) if k == 0 else (b + b" " * int(rng.integers(1, 70)) if k == 1 else b[:-int(rng.integers(1, 70))]),
                        move=bool(k and rng.integers(2)))
            live = np.flatnonzero((dr.snap.p_packed & abi.PP_TOMBSTONE) == 0)
            flip = rng.choice(live, max(1, live.size // 100), replace=False)
            flip_ready(dr.snap, flip)
            dr.commit_specs()
            if epoch % 2:
                dr.commit_rows(flip)
            else:
                dr.commit_objects(twin=False)
                dr.commit_rows(flip)
            got, _ = dr.check(oracle_mod, expect_incremental=None)
            n_inc += incremental(got, nc)
        assert n_inc >= 38, n_inc
    finally:
        dr.close()


def _twin_streams(seed, sides, oracle_mod, stream):
    """The same 40 epochs of spec edits and informer events (one generator per epoch, seeded alike) on each side."""
    out = []
    for side in sides:
        gen, counter = [2], [0]

        def step(epoch, side=side, gen=gen, counter=counter):
            r = np.random.default_rng(1000 * seed + epoch)
            spec_edits(r, side, gen, int(r.integers(1, 4)))
            events(r, side, counter, structural=False)
        out.append(stream(side, oracle_mod, 40, step))
    return out


@pytest.mark.parametrize("seed", [1, 2])
def test_stream_through_the_native_packer(seed, oracle_mod):
    clusters, pods, jobs = objects(seed, big=True)
    pks = [Packer(**PACKER_CAPS, spec_rows=on) for on in (True, False)]
    try:
        assert pks[0].engine.get_option(abi.OPT_SPEC_ROWS) == 1 and pks[1].engine.get_option(abi.OPT_SPEC_ROWS) == 0
        ms = [Mirror(copy.deepcopy(clusters), copy.deepcopy(pods), jobs, pk) for pk in pks]
        for pk, m in zip(pks, ms):
            pk.flush()
            packer_check(m, oracle_mod, lean=True)
        (gots_on, modes_on), (gots_off, modes_off) = _twin_streams(seed, ms, oracle_mod, packer_stream)
        for epoch, (mode_on, mode_off, got_on, got_off) in enumerate(zip(modes_on, modes_off, gots_on, gots_off)):
            assert mode_on & abi.PACK_SPEC_ROWS and not mode_on & abi.PART_JSON, (epoch, mode_on)
            assert mode_off & abi.PART_JSON and not mode_off & abi.PACK_SPEC_ROWS, (epoch, mode_off)
            assert not got_off.diff(got_on), epoch
        modes = [device_incremental(g) for g in gots_on]
        assert sum(modes) >= 36, modes
    finally:
        for pk in pks:
            pk.close()


@pytest.mark.parametrize("seed", [1, 2])
def test_stream_through_the_live_arena(seed, oracle_mod):
    clusters, pods, jobs = objects(seed, big=True)
    arenas = [LiveArena(copy.deepcopy(clusters), copy.deepcopy(pods), jobs, spare_rows=64, spec_rows=on) for on in (True, False)]
    try:
        gots_on, gots_off = _twin_streams(seed, arenas, oracle_mod, arena_stream)
        for epoch, (got_on, got_off) in enumerate(zip(gots_on, gots_off)):
            assert not got_off.diff(got_on), epoch
        inc = [device_incremental(g) for g in gots_on]
        assert arenas[0].engine.get_option(abi.OPT_SPEC_ROWS) == 1
        assert sum(inc) >= 34 and arenas[0].stats["rebase"] <= 2, (inc, arenas[0].stats)
    finally:
        for a in arenas:
            a.close()

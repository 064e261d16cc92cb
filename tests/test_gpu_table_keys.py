"""The engine's hash tables under colliding, wrapping and full-range ids (tests/table_keys.py builds the snapshots).

K1 puts about 480 RayCluster keys, orphan Pods' and RayJobs' absent keys and swapped or shared halves in one probe chain that starts in
the last slot of the cluster table and wraps; K2 does the same for about 3 000 workersToDelete names (Bloom bitmap at its cap, decoy
Pods that pass both Bloom bits and miss); K3 puts 60 head Pods at pod rows that share the last slot of the head-aux table; K4 runs
the differential fuzz seeds and C2 / C5 with every id moved across the whole u32 domain.  Every pass must equal the oracle, and a
pass over a relabelled snapshot must return the records of the original with their ids mapped."""
import numpy as np
import pytest

import fuzz_objects
from harness import OBJ_COLS, REBUILD, Driver, flip_ready, lists_of, members, run, workers_of
from kuberay_b200 import abi, synthetic
from kuberay_b200.engine import Engine
from kuberay_b200.snapshot import Snapshot
from table_keys import hash_pair, ids_in, k1, k2, k3, map_results, random_map, relabel

pytestmark = pytest.mark.gpu

OPTS = dict(large_clusters=True, wide_clusters=True, huge_clusters=True)
ENV = {"radix": "KR_FORCE_RADIX", "no_bucket": "KR_NO_BUCKET", "no_graph": "KR_NO_GRAPH"}
FETCH = {"bucket": 0, "lists": 1, "radix": 1, "no_bucket": 0, "no_graph": 0}


@pytest.fixture(scope="module")
def cases():
    return {"K1": k1(), "K2": k2(), "K3": k3()}


def _copy(snap):
    out = Snapshot(**{"n_" + k if k != "json" else "json_bytes": v for k, v in snap.dims.items()})
    for name in snap.cols:
        out.cols[name][:] = snap.cols[name]
    return out


def _flags(flags, fetch):
    f = abi.kr_flags.from_buffer_copy(flags)
    f.fetch_pod_lists = fetch
    return f


@pytest.mark.parametrize("variant", list(FETCH))
@pytest.mark.parametrize("name", ["K1", "K2", "K3"])
def test_full_pass(name, variant, cases, oracle_mod, monkeypatch):
    k = cases[name]
    if variant in ENV:
        monkeypatch.setenv(ENV[variant], "1")
    flags = _flags(k.kflags, FETCH[variant])
    got, _, stride = run(k.snap, flags, **OPTS)
    if variant == "bucket":
        assert stride != 0
    d = oracle_mod.run(k.snap, flags, threads=8).diff(got)
    assert not d, (name, variant, d[:8])
    if variant in ("bucket", "lists"):   # the engine's records over the relabelled snapshot are its records over the original, mapped
        base, _, _ = run(k.orig, _flags(k.flags, FETCH[variant]), **OPTS)
        d = map_results(base, k.f).diff(got)
        assert not d, (name, variant, "relabelled", d[:8])


def _k4(snap, flags, seed, oracle_mod, threads=1):
    f = random_map(ids_in(snap, flags), np.random.default_rng(seed))
    rs, rf = relabel(snap, flags, f)
    want = oracle_mod.run(rs, rf, threads=threads)
    eng = Engine.for_snapshot(rs, max_creates=1 << 16)
    try:
        eng.load(rs)
        got = eng.reconcile(_flags(rf, 1))
        lean = eng.reconcile(_flags(rf, 0))
    finally:
        eng.close()
    for what, res in (("lists", got), ("compact", lean)):
        d = want.diff(res)
        assert not d, (seed, what, d[:8])
    return got


@pytest.mark.parametrize("seed0", [0, 100, 200, 300])
def test_full_range_ids_fuzz(seed0, oracle_mod):
    """K4: the seeds of test_fuzz_adversarial_snapshots under random bijections of their ids onto [2, 0xFFFFFFFE]."""
    for seed in range(seed0, seed0 + 100, 2):
        snap, flags = fuzz_objects.snapshot(seed, big=(seed % 10 == 0))
        _k4(snap, flags, seed, oracle_mod)


@pytest.mark.parametrize("cfg", ["C2", "C5"])
def test_full_range_ids_configs(cfg, oracle_mod):
    snap, flags = synthetic.generate(synthetic.config(cfg, wtd_group_frac=0.3, jobs=True))
    got = _k4(snap, flags, 7, oracle_mod, threads=8)
    assert got.n_actions > 0


# ------------------------------------------------------------------------------------------------ incremental epochs
def _driver(k, wtd_room=512, **opts):
    """Fixed layout with room for the workersToDelete lists to grow, KR_OPT_WTD_EDITS on."""
    return Driver(_copy(k.snap), _flags(k.kflags, 0), wtd_room=wtd_room, **opts, wtd_edits=True)


def test_epochs_in_the_cluster_chain(cases, oracle_mod):
    """K1: status updates of Pods in the chain (rewritten in place through cl_probe), Pods moved between two colliding RayClusters and
    onto colliding absent keys and back, group rows of colliding RayClusters through kr_snapshot_commit_object_rows."""
    k = cases["K1"]
    rng = np.random.default_rng(11)
    dr = _driver(k, **OPTS)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        s = dr.snap
        owned = np.concatenate([members(s, c) for c in range(s.dims["clusters"])])
        rows = rng.choice(owned, 300, replace=False)
        flip_ready(s, rows)
        dr.commit_rows(rows)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        assert got.changed_clusters is not None and got.changed_clusters.size > 100
        # Pods of RayClusters of the shared namespace move to their neighbours, and onto absent keys of the chain
        ns = k.absent[0][0]
        cs = np.flatnonzero((s.c_ns_id == ns) & (s.c_group_cnt > 0))
        moved, back = [], {}
        for a, b in zip(cs[10:30], cs[11:31]):
            w = workers_of(s, int(s.c_group_off[a]))[:2]
            for r in w:
                back[int(r)] = (int(s.p_cluster_name_id[r]), int(s.p_group_name_id[r]))
            s.p_cluster_name_id[w], s.p_group_name_id[w] = s.c_name_id[b], s.g_name_id[int(s.c_group_off[b])]
            moved += w.tolist()
        for (ns_, z), a in zip(k.absent, cs[40:]):
            w = workers_of(s, int(s.c_group_off[a]))[:2]
            for r in w:
                back[int(r)] = (int(s.p_cluster_name_id[r]), int(s.p_group_name_id[r]))
            assert ns_ == ns
            s.p_cluster_name_id[w] = z
            moved += w.tolist()
        dr.commit_rows(moved)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        assert got.n_orphans >= 16 + len(k.orphans)
        for r, (cn, gn) in back.items():
            s.p_cluster_name_id[r], s.p_group_name_id[r] = cn, gn
        dr.commit_rows(list(back))
        dr.check(oracle_mod, expect_incremental=True)
        # group rows of colliding RayClusters (replicas, expectations), row-granular
        edit = [int(c) for c in cs[:12]] + [k.large, k.wide]
        for c in edit:
            g = slice(int(s.c_group_off[c]), int(s.c_group_off[c] + s.c_group_cnt[c]))
            s.g_replicas[g] += 1
            s.g_flags[g] ^= np.uint32(abi.GF_EXPECT_OK)
        for col in OBJ_COLS:
            np.copyto(dr.views[col], s.cols[col])
        dr.eng.commit_object_rows(edit, [])
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        assert set(edit) <= set(got.changed_clusters.tolist())
    finally:
        dr.close()


def test_epochs_in_the_workers_to_delete_chain(cases, oracle_mod):
    """K2: workersToDelete renames among colliding names (the name table rebuilt on the device), onto decoys, and back; status updates
    of named Pods and decoys."""
    k = cases["K2"]
    rng = np.random.default_rng(12)
    dr = _driver(k, wtd_room=64)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        s = dr.snap
        old = lists_of(s)
        lists = [list(x) for x in old]
        ns_of = s.c_ns_id[s.g_cluster_idx]
        decoy_ns = s.p_ns_id[k.decoys]
        gs = [g for g in range(s.dims["groups"]) if lists[g]]
        for g in rng.choice(gs, 60, replace=False).tolist():
            same = [x for h in range(max(0, g - 40), min(len(lists), g + 40)) if ns_of[h] == ns_of[g] for x in old[h]]
            dec = k.decoys[decoy_ns == ns_of[g]]
            lists[g][0] = int(s.p_name_id[dec[0]]) if dec.size and rng.random() < 0.5 else same[int(rng.integers(len(same)))]
        dr.set_wtd_lists(lists)
        got, names = dr.check(oracle_mod, expect_incremental=True, profiled=True)
        assert set(REBUILD) <= set(names), names
        rows = np.concatenate([np.flatnonzero(np.isin(s.p_name_id, s.w_name_id))[:200], k.decoys[:100]])
        flip_ready(dr.snap, rows)
        dr.commit_rows(rows)
        dr.check(oracle_mod, expect_incremental=True)
        dr.set_wtd_lists(old)
        dr.check(oracle_mod, expect_incremental=True)
    finally:
        dr.close()


def test_epochs_with_heads_at_colliding_rows(cases, oracle_mod):
    """K3: head Pods leave colliding rows and come back at other colliding rows, under other RayClusters (the head-aux table is rebuilt
    with every key in one wrapping chain); status updates of the heads."""
    k = cases["K3"]
    dr = _driver(k)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        s = dr.snap
        spare = [int(r) for r in k.spare]
        for step in range(3):
            rows = []
            for i in range(4):
                src, dst = int(k.hot[8 * step + i + 10]), spare.pop()
                t = int(np.flatnonzero(s.h_pod_idx == src)[0])
                for name in (c for c, _dt, _m, dim in abi.COLUMNS if dim == "pods"):
                    s.cols[name][dst] = s.cols[name][src]
                    s.cols[name][src] = 0
                s.p_packed[src] = abi.PP_TOMBSTONE
                other = int(np.flatnonzero(s.h_pod_idx == int(k.hot[8 * step + i + 40]))[0])   # now under another colliding RayCluster
                s.p_ns_id[dst], s.p_cluster_name_id[dst] = s.p_ns_id[s.h_pod_idx[other]], s.p_cluster_name_id[s.h_pod_idx[other]]
                s.h_pod_idx[t] = dst
                rows += [src, dst]
            dr.commit_objects()
            dr.commit_rows(rows)
            dr.check(oracle_mod, expect_incremental=True)
        heads = s.h_pod_idx.copy()
        flip_ready(s, heads)
        dr.commit_rows(heads)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        assert (got.clusters["n_heads"] == 2).any() and (got.clusters["n_heads"] == 0).any()
    finally:
        dr.close()


def test_chain_keys_really_collide_in_the_engine_tables(cases):
    """The constructions mean what they claim for the layouts the engine picks (cluster table >= 2 x clusters, power of two)."""
    s = cases["K1"].snap
    mask = (1 << int(np.ceil(np.log2(2 * s.dims["clusters"])))) - 1
    home = hash_pair(s.c_ns_id, s.c_name_id) & np.uint32(mask)
    assert (home == mask).sum() >= 470

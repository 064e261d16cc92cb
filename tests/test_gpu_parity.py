"""GPU parity: the CUDA engine (through the C ABI) vs the CPU oracle on the same seeded snapshots. Bit-exact."""
import numpy as np
import pytest

from harness import b32, compact, kernels, parity
from kuberay_b200 import abi, synthetic
from kuberay_b200.engine import Engine

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cfg", ["C1", "C2"])
def test_parity_small_configs(cfg, oracle_mod):
    snap, flags = synthetic.generate(synthetic.config(cfg))
    parity(snap, flags, oracle_mod)


def test_parity_c3_headline(oracle_mod):
    snap, flags = synthetic.generate(synthetic.config("C3"))
    got = parity(snap, flags, oracle_mod)
    assert got.n_actions > 0 and got.n_create_total > 0


def test_parity_multi_group(oracle_mod):
    snap, flags = synthetic.generate(synthetic.config("C2", groups=3, pods_per_cluster=40))
    parity(snap, flags, oracle_mod)


def test_parity_many_groups_spill(oracle_mod):
    # > 32 worker groups per cluster: accumulators spill from shared memory to global scratch
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=50, pods_per_cluster=200, groups=40))
    parity(snap, flags, oracle_mod)


def test_parity_multihost_groups(oracle_mod, monkeypatch):
    # numOfHosts=4 groups with replica-name labels, incomplete / unhealthy / scale-down replicas in the mix
    params = synthetic.SynthParams(n_clusters=400, pods_per_cluster=41, groups=2, multihost_frac=0.5)
    snap, flags = synthetic.generate(params)
    got = parity(snap, flags, oracle_mod)
    acts = set(np.unique(got.sorted_action).tolist())
    assert {abi.ACT_DELETE_MH_UNHEALTHY, abi.ACT_DELETE_MH_INCOMPLETE} & acts
    assert (got.groups["flags"] & abi.GR_MULTIHOST).any()
    monkeypatch.setenv("KR_FORCE_RADIX", "1")
    parity(snap, flags, oracle_mod)


def test_parity_flag_variants(oracle_mod):
    snap, flags = synthetic.generate(synthetic.config("C2"))
    for kw in (dict(env_random_pod_delete=1), dict(gate_status_conditions=0), dict(gate_multihost_indexing=0)):
        f = abi.default_flags(id_head_not_found_reason=flags.id_head_not_found_reason, id_head_not_found_msg=flags.id_head_not_found_msg, **kw)
        parity(snap, f, oracle_mod)


def test_parity_big_bucket_falls_back_to_radix(oracle_mod):
    # one RayCluster with 3000 pods: the fast pipeline's in-warp sort takes <= 1024 per bucket, the engine must switch
    # to the radix pipeline by itself and still be bit-exact
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=20, pods_per_cluster=3000, groups=2))
    parity(snap, flags, oracle_mod)


def test_many_orphans_stay_on_the_fast_pipeline(oracle_mod):
    # 20 % of the pods name a RayCluster that is not in the snapshot: the orphan bucket (5000 pods) is ordered without a sort
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=500, pods_per_cluster=50, groups=1, orphan_frac=0.2))
    got = parity(snap, flags, oracle_mod)
    assert got.n_orphans == 5000
    names = kernels(snap, flags)
    assert any(k.startswith("k_place") for k in names) and "k_scatter" not in names


def test_parity_radix_pipeline_forced(oracle_mod, monkeypatch):
    monkeypatch.setenv("KR_FORCE_RADIX", "1")
    snap, flags = synthetic.generate(synthetic.config("C2", groups=2))
    parity(snap, flags, oracle_mod)
    snap, flags = synthetic.generate(synthetic.config("C3"))
    parity(snap, flags, oracle_mod)


@pytest.mark.parametrize("ppc", [1, 2, 33, 41, 63, 64, 65, 127])
def test_parity_odd_cluster_sizes_both_pipelines(ppc, oracle_mod, monkeypatch):
    params = synthetic.SynthParams(n_clusters=257, pods_per_cluster=ppc, groups=1)
    snap, flags = synthetic.generate(params)
    parity(snap, flags, oracle_mod)
    monkeypatch.setenv("KR_FORCE_RADIX", "1")
    parity(snap, flags, oracle_mod)


def test_parity_unfused_scan_kernels(oracle_mod, monkeypatch):
    # large snapshots use separate chained-scan kernels instead of the shared-memory fused ones: force that path
    monkeypatch.setenv("KR_NO_FUSE", "1")
    snap, flags = synthetic.generate(synthetic.config("C2", groups=2, orphan_frac=0.05))
    parity(snap, flags, oracle_mod)
    snap, flags = synthetic.generate(synthetic.config("C3"))
    parity(snap, flags, oracle_mod)


def test_parity_rayjob_rollup_c4(oracle_mod):
    snap, flags = synthetic.generate(synthetic.config("C4"))
    got = parity(snap, flags, oracle_mod)
    assert got.jobs["status_changed"].sum() > 0 and (got.jobs["cluster_idx"] < 0).sum() > 0


def test_parity_without_cuda_graph(oracle_mod, monkeypatch):
    monkeypatch.setenv("KR_NO_GRAPH", "1")
    snap, flags = synthetic.generate(synthetic.config("C2"))
    parity(snap, flags, oracle_mod)


def test_repeated_passes_are_identical(oracle_mod):
    snap, flags = synthetic.generate(synthetic.config("C2"))
    eng = Engine.for_snapshot(snap)
    try:
        eng.load(snap)
        first = eng.reconcile(flags)
        for _ in range(3):
            again = eng.reconcile(flags)
            assert not first.diff(again)
        eng.commit()
        assert not first.diff(eng.reconcile(flags))
    finally:
        eng.close()


def test_partial_commit_columns_only(oracle_mod):
    """kr_snapshot_commit_parts(KR_PART_COLUMNS): pod statuses move, the spec-JSON arena stays resident; results must equal
    a full pass over the mutated snapshot."""
    snap, flags = synthetic.generate(synthetic.config("C2"))
    eng = Engine.for_snapshot(snap)
    try:
        with pytest.raises(Exception):
            eng.begin(snap.sizes()); eng.commit(abi.PART_COLUMNS)        # needs a full commit of this layout first
        views = eng.load(snap)
        eng.reconcile(flags)
        rng = np.random.default_rng(3)
        flip = rng.choice(snap.dims["pods"], 500, replace=False)
        snap.p_packed[flip] = (snap.p_packed[flip] & ~np.uint32(7 << abi.PP_PHASE_SHIFT)) | np.uint32(abi.PHASE_FAILED << abi.PP_PHASE_SHIFT)
        np.copyto(views["p_packed"], snap.p_packed)
        views["json"][:] = 0                                               # host copy of the JSON is NOT re-uploaded ...
        eng.commit(abi.PART_COLUMNS)
        got = eng.reconcile(flags)
    finally:
        eng.close()
    want = oracle_mod.run(snap, flags, threads=8)                          # ... so the hashes still match the real specs
    assert not want.diff(got)


def test_incremental_pod_rows(oracle_mod):
    """kr_snapshot_commit_pod_rows: only rewritten pod rows cross PCIe; results equal a full pass over the mutated snapshot."""
    snap, flags = synthetic.generate(synthetic.config("C2", groups=2))
    eng = Engine.for_snapshot(snap)
    try:
        views = eng.load(snap)
        eng.reconcile(flags)
        rng = np.random.default_rng(11)
        for epoch in range(3):
            rows = rng.choice(snap.dims["pods"], 300, replace=False).astype(np.uint32)
            snap.p_packed[rows] ^= np.uint32(abi.PHASE_RUNNING << abi.PP_PHASE_SHIFT) ^ np.uint32(abi.PHASE_FAILED << abi.PP_PHASE_SHIFT)
            snap.p_group_name_id[rows[:20]] = snap.p_group_name_id[rows[20:40]]          # relabelled pods move between groups
            for name in ("p_packed", "p_group_name_id"):
                np.copyto(views[name], snap.cols[name])
            eng.commit_pod_rows(np.concatenate([rows, rows[:5]]))                      # duplicates are fine
            got = eng.reconcile(flags)
            want = oracle_mod.run(snap, flags, threads=8)
            assert not want.diff(got), epoch
    finally:
        eng.close()


def test_compact_action_list_without_pod_lists(oracle_mod):
    """kr_flags.fetch_pod_lists = 0: only the compact action list comes back; it must equal the oracle's."""
    snap, flags = synthetic.generate(synthetic.config("C2", groups=2))
    flags.fetch_pod_lists = 0
    eng = Engine.for_snapshot(snap)
    try:
        eng.load(snap)
        got = eng.reconcile(flags)
    finally:
        eng.close()
    want = oracle_mod.run(snap, flags, threads=8)
    assert got.sorted_pod_idx.size == 0 and got.n_actions == want.n_actions > 0
    assert not want.diff(got)
    # the list is exactly the non-KEEP entries of the full lists, cluster by cluster
    keep = (want.sorted_action != abi.ACT_KEEP) & (want.sorted_action != abi.ACT_ORPHAN)
    own = abi._gather_owned(got.act_start[:-1], got.act_cnt)  # cluster c owns [act_start[c], act_start[c] + act_cnt[c])
    assert np.array_equal(got.act_pod_idx[own], want.sorted_pod_idx[keep]) and np.array_equal(got.act_code[own], want.sorted_action[keep])
    assert np.array_equal(got.act_cnt.astype(np.int64), np.add.reduceat(keep.astype(np.int64), want.clusters["pod_start"].astype(np.int64))
                          if snap.dims["clusters"] else [])
    # one run per cluster, anywhere in the list, never overlapping (RayClusters whose Recreate gate waited for the digest reserved
    # their whole bucket: the list's extent is at least the count)
    assert got.act_pod_idx.size >= got.n_actions and np.unique(own).size == own.size


def test_bucket_pipeline_is_taken_and_widens_its_stride(oracle_mod):
    """fetch_pod_lists = 0 on a qualifying snapshot runs k_match2 + k_decide2 and nothing of the sort pipeline.  A RayCluster
    larger than the first stride voids the attempt: the engine widens the stride (64 -> 128 -> 256), then leaves for the sort
    pipeline (here: a 300-pod cluster), every time bit-exact."""
    snap, flags = synthetic.generate(synthetic.config("C3"))
    names = kernels(snap, compact(flags))
    assert {"k_match2", "k_decide2", "k_hash"} <= set(names) and not any(k.startswith(("k_place", "k_creates", "k_decide_small")) for k in names)
    names = kernels(snap, flags)
    assert "k_match2" not in names and "k_decide_small" in names
    for big in (100, 200, 300):
        # 300 RayClusters x 20 pods; the pods of clusters 1 .. k are relabelled into cluster 0 (same namespace), which then
        # lists `big` pods (and several heads), while clusters 1 .. k list none
        both, f = synthetic.generate(synthetic.SynthParams(n_clusters=300, pods_per_cluster=20, groups=1))
        k = big // 20 - 1
        moved = np.isin(both.p_cluster_name_id, both.c_name_id[1:k + 1])
        both.p_cluster_name_id[moved] = both.c_name_id[0]
        parity(both, f, oracle_mod)
        names = kernels(both, compact(f))   # (a fresh engine starts at the narrow stride again and ends where the ladder ends)
        assert ("k_match2" in names) == (big <= 256), (big, names)


def test_bucket_pipeline_long_delete_prefix_and_delete_all(oracle_mod):
    """The ordered pieces of k_decide2 off their common path: scale-downs by tens of pods (counting rank instead of the
    min-extraction), whole-cluster deletions (suspension, Recreate: action list = the sorted bucket), three worker groups."""
    params = synthetic.SynthParams(n_clusters=600, pods_per_cluster=90, groups=3, suspended_frac=0.1, recreate_frac=0.3, autoscaling_frac=0.2)
    snap, flags = synthetic.generate(params)
    rng = np.random.default_rng(5)
    shrink = rng.random(snap.dims["groups"]) < 0.5
    snap.g_replicas[shrink] = rng.integers(0, 8, int(shrink.sum()))
    snap.g_min[shrink] = 0
    snap.g_flags[shrink] &= ~np.uint32(abi.GF_REPLICAS_NIL | abi.GF_MIN_NIL)
    flags.env_random_pod_delete = 1
    got = parity(snap, flags, oracle_mod)
    assert (got.groups["diff"] < -8).sum() > 50 and (got.clusters["path"] == abi.PATH_RECREATE_DELETE_ALL).sum() > 5


def test_hash_batch_matches_hashlib():
    rng = np.random.default_rng(1)
    msgs = [b"", b"abc", b"a" * 55, b"a" * 56, b"a" * 63, b"a" * 64, b"a" * 65, b"a" * 119, b"a" * 120, b"a" * 127, b"a" * 128]
    msgs += [rng.integers(0, 256, int(n), dtype=np.uint8).tobytes() for n in rng.integers(0, 9000, 300)]
    eng = Engine(0, max_clusters=1)
    try:
        got = eng.hash_batch(msgs)
    finally:
        eng.close()
    want = [b32(m).decode() for m in msgs]
    assert got == want
    from oracle import oracle as _oracle
    assert got[:40] == [_oracle.hash32(m) for m in msgs[:40]]      # and the oracle's own SHA-1 / base32hex (kr_oracle_hash32) agrees with both


def test_hash_batch_and_passes_share_an_engine(oracle_mod):
    """kr_hash_batch (the RayService callers' entry point) between passes of the same engine: its staging buffers grow
    without disturbing the pass's own pinned buffers (a stray free there once corrupted the totals record)."""
    snap, flags = synthetic.generate(synthetic.config("C2"))
    eng = Engine.for_snapshot(snap)
    try:
        eng.load(snap)
        want = oracle_mod.run(snap, flags, threads=8)
        for size in (10, 1000, 40000):
            msgs = [bytes([i % 251]) * (i % 700) for i in range(size // 10)]
            assert eng.hash_batch(msgs) == [b32(m).decode() for m in msgs]
            assert not want.diff(eng.reconcile(flags)), size
    finally:
        eng.close()


def _per_cluster_case(snap, arm, seed):
    """The fuzz snapshot carried into the per-cluster kernels of the bucket pipeline (kr_large.cuh) -> (snapshot, the RayCluster
    grown past 256 pods or None), or None when the seed has no candidate.
      wide:  worker group 0 of every RayCluster that has a group split into 33..64 groups;
      large: the non-head pods of one RayCluster (adversarial phases and labels included) cloned into appended rows under fresh
             names until it lists 257..1200 pods — as far as the layout's first stride, which holds 1.25x the mean cluster, stays
             at 256 or below (past that the pass never tries the bucket pipeline)."""
    from kuberay_b200.snapshot import Snapshot
    from oracle import oracle
    rng = np.random.default_rng(seed ^ 0xC1A55)
    grown = None
    if arm == "wide":
        cs = np.flatnonzero(snap.c_group_cnt >= 1)
        if not cs.size:
            return None
        out = synthetic.widen_clusters(snap, cs, int(rng.integers(33, 65)))
    else:
        ckey = (snap.c_ns_id.astype(np.uint64) << np.uint64(32)) | snap.c_name_id.astype(np.uint64)
        pkey = (snap.p_ns_id.astype(np.uint64) << np.uint64(32)) | snap.p_cluster_name_id.astype(np.uint64)
        head = ((snap.p_packed >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_HEAD
        cands = [(c, np.flatnonzero((pkey == ckey[c]) & ~head & (snap.p_cluster_name_id != 0))) for c in range(snap.dims["clusters"])]
        cands = [(c, m) for c, m in cands if m.size]
        if not cands:
            return None
        grown, src = cands[int(rng.integers(len(cands)))]
        members = int(np.sum(pkey == ckey[grown]))
        d = snap.dims
        most = min(1200, members + (256 * d["clusters"] * 4) // 5 - d["pods"])
        if members > most or most < 257:
            return None
        extra = np.resize(src, int(rng.integers(max(257, members), most + 1)) - members)
        out = Snapshot(d["clusters"], d["groups"], d["wtd"], d["pods"] + extra.size, d["heads"], d["jobs"], d["json"])
        for name, _dt, _m, dim in abi.COLUMNS:
            out.cols[name][:] = np.concatenate([snap.cols[name], snap.cols[name][extra]]) if dim == "pods" else snap.cols[name]
        out.p_name_id[d["pods"]:] = np.uint32(max(int(snap.p_name_id.max(initial=0)), 0x10000) + 1) + np.arange(extra.size, dtype=np.uint32)
    # split replicas times numOfHosts can reach billions of pods to create (and an expected count near -2^31 wraps expected - running):
    # a capacity error on both sides, not a parity case (fuzz_objects.generate keeps |expected| <= 300 for the same reason)
    L = oracle.lib()
    big = any(abs(L.kr_oracle_desired_replicas(int(out.g_replicas[g]), int(out.g_min[g]), int(out.g_max[g]), int(out.g_num_hosts[g]),
                                               int(out.g_flags[g]))) > 300 for g in range(out.dims["groups"]))
    return None if big else (out, grown)


FUZZ_ARMS = [pytest.param(s0, None, id=str(s0)) for s0 in (0, 100, 200, 300)] + \
            [pytest.param(s0, arm, id=f"{arm}-{s0}") for arm in ("wide", "large") for s0 in (0, 100, 200)]


@pytest.mark.parametrize("seed0,arm", FUZZ_ARMS)
def test_fuzz_adversarial_snapshots(seed0, arm, oracle_mod, monkeypatch):
    """Differential fuzz: tiny snapshots drawn from the whole input domain (tests/fuzz_objects.py), packed like the golden
    scenarios, engine vs oracle byte for byte.  Every fourth seed also runs the radix / unfused pipeline.
    The wide and large arms carry the same contents into the per-cluster kernels of the bucket pipeline (KR_OPT_WIDE_CLUSTERS and
    KR_OPT_LARGE_CLUSTERS on, compact results): the first (captured) full pass == oracle == engine with both options off; then a
    profiled epoch shows the per-cluster kernels on the list, and in the large arm the grown RayCluster past the stride, i.e. in its
    region of the large-cluster arena."""
    import fuzz_objects
    if arm:
        cases = regions = 0
        for seed in range(seed0, seed0 + 100):
            snap, flags = fuzz_objects.snapshot(seed, big=(seed % 10 == 0))
            case = _per_cluster_case(snap, arm, seed)
            if case is None:
                continue
            snap, grown = case
            cases += 1
            flags = compact(flags)
            want = oracle_mod.run(snap, flags, threads=1)
            runs = []
            for on in (True, False):
                eng = Engine.for_snapshot(snap, large_clusters=on, wide_clusters=on, max_creates=1 << 16)
                try:
                    eng.load(snap)
                    got = eng.reconcile(flags)
                    names = {k for k, _ in eng.reconcile_profiled(flags)["kernels"]} if on else set()
                    runs.append((got, names, eng.get_option(abi.OPT_BUCKET_STRIDE)))
                finally:
                    eng.close()
            (got, names, stride), (off, _, _) = runs
            d = want.diff(got)
            assert not d, (arm, seed, d[:8])
            d = off.diff(got)
            assert not d, (arm, "options off", seed, d[:8])
            assert "k_decide_large" in names and stride, (arm, seed, sorted(names), stride)
            if grown is not None:
                n = int(np.sum((snap.p_ns_id == snap.c_ns_id[grown]) & (snap.p_cluster_name_id == snap.c_name_id[grown])))
                regions += n > stride
        assert cases >= 50 and (arm != "large" or regions >= 50), (cases, regions)
        return
    for seed in range(seed0, seed0 + 100):
        snap, flags = fuzz_objects.snapshot(seed, big=(seed % 10 == 0))
        want = oracle_mod.run(snap, flags, threads=1)
        eng = Engine.for_snapshot(snap)
        try:
            eng.load(snap)
            got = eng.reconcile(flags)
            lean = eng.reconcile(compact(flags))
        finally:
            eng.close()
        d = want.diff(got)
        assert not d, (seed, d[:8])
        d = want.diff(lean)
        assert not d, ("compact", seed, d[:8])
    monkeypatch.setenv("KR_FORCE_RADIX", "1")
    monkeypatch.setenv("KR_NO_FUSE", "1")
    for seed in range(seed0, seed0 + 100, 4):
        snap, flags = fuzz_objects.snapshot(seed)
        want = oracle_mod.run(snap, flags, threads=1)
        eng = Engine.for_snapshot(snap)
        try:
            eng.load(snap)
            got = eng.reconcile(flags)
        finally:
            eng.close()
        d = want.diff(got)
        assert not d, ("radix", seed, d[:8])


def test_double_buffered_epochs_two_engines(oracle_mod):
    """Two engines on one GPU used alternately (bench.py's e2e loop): the asynchronous commit of epoch k+1 is issued before the
    blocking reconcile of epoch k.  Each epoch carries a different snapshot; every result must match the oracle."""
    snaps = [synthetic.generate(synthetic.config("C2", seed=synthetic.SEED + i)) for i in range(4)]
    big = max((s for s, _ in snaps), key=lambda s: s.nbytes())
    engines = [Engine.for_snapshot(big, slack=1.3), Engine.for_snapshot(big, slack=1.3)]
    try:
        def stage(i):
            eng, (snap, _f) = engines[i & 1], snaps[i]
            eng.fill(eng.begin(snap.sizes()), snap)
            eng.commit()
        stage(0)
        for i in range(len(snaps)):
            if i + 1 < len(snaps):
                stage(i + 1)
            got = engines[i & 1].reconcile(snaps[i][1])
            want = oracle_mod.run(snaps[i][0], snaps[i][1], threads=8)
            assert not want.diff(got), i
    finally:
        for eng in engines:
            eng.close()


def test_parity_c5_autoscaling_sharded_over_8(oracle_mod):
    """C5 (BASELINE.json configs[4]): 1 000 autoscaling RayClusters x 100 pods, UID-hash sharded 8 ways (SURVEY §8(e)).
    Every shard goes through the engine; its records must equal the global CPU pass restricted to the shard's clusters —
    the path needs no exchange between GPUs."""
    snap, flags = synthetic.generate(synthetic.config("C5", wtd_group_frac=0.3))
    glob = oracle_mod.run(snap, flags, threads=8)
    world, seen = 8, 0
    for rank in range(world):
        sh = synthetic.shard_by_uid(snap, rank, world)
        got = parity(sh, flags, oracle_mod)
        keep = (snap.c_uid_hash % np.uint64(world)) == np.uint64(rank)
        for fld in ("path", "head_action", "err_kind", "err_arg", "n_pods", "new_state", "needs_status_write", "counts", "cond_status"):
            assert np.array_equal(got.clusters[fld], glob.clusters[keep][fld]), (rank, fld)
        assert np.array_equal(got.hash, glob.hash[keep])
        gkeep = keep[snap.g_cluster_idx]
        for fld in ("expected", "n_running", "diff", "n_create", "flags"):
            assert np.array_equal(got.groups[fld], glob.groups[gkeep][fld]), (rank, fld)
        seen += sh.dims["clusters"]
    assert seen == snap.dims["clusters"]
    assert (glob.groups["flags"] & abi.GR_WTD_EXECUTED).any()


def test_error_paths_return_codes_not_crashes(oracle_mod):
    """The C ABI never throws across the boundary: misuse and capacity overruns come back as KR_E_* codes with a message
    (kr_last_error), and the engine stays usable afterwards — the Go side falls back to the per-object path for that epoch."""
    from kuberay_b200.engine import EngineError
    snap, flags = synthetic.generate(synthetic.config("C1"))
    eng = Engine.for_snapshot(snap, max_creates=1024)
    try:
        # a snapshot larger than the capacities given to kr_engine_create
        big, _ = synthetic.generate(synthetic.config("C2"))
        with pytest.raises(EngineError) as ei:
            eng.begin(big.sizes())
        assert ei.value.code == abi.KR_E_CAPACITY
        # partial / incremental commits before this layout was ever fully uploaded
        views = eng.begin(snap.sizes())
        eng.fill(views, snap)
        for call in (lambda: eng.commit(abi.PART_COLUMNS), lambda: eng.commit(abi.PART_OBJECTS), lambda: eng.commit_pod_rows(np.array([0], dtype=np.uint32))):
            with pytest.raises(EngineError) as ei:
                call()
            assert ei.value.code == abi.KR_E_STATE
        # broken invariants are caught on the host at commit: misaligned JSON offset, groups out of cluster order
        views["c_json_off"][1] += 1
        with pytest.raises(EngineError) as ei:
            eng.commit()
        assert ei.value.code == abi.KR_E_INVALID and "16-byte" in str(ei.value)
        views["c_json_off"][1] -= 1
        views["c_group_off"][2] += 1
        with pytest.raises(EngineError) as ei:
            eng.commit()
        assert ei.value.code == abi.KR_E_INVALID
        views["c_group_off"][2] -= 1
        eng.commit()
        # a pod row outside the arena
        with pytest.raises(EngineError) as ei:
            eng.commit_pod_rows(np.array([snap.dims["pods"]], dtype=np.uint32))
        assert ei.value.code == abi.KR_E_INVALID
        # more pods to create than kr_config.max_creates: the pass runs, the fetch reports the overrun
        views["g_replicas"][:] = 500
        views["g_max"][:] = 2 ** 31 - 1
        views["g_flags"][:] &= ~np.uint32(abi.GF_REPLICAS_NIL | abi.GF_MAX_NIL)
        eng.commit()
        with pytest.raises(EngineError) as ei:
            eng.reconcile(flags)
        assert ei.value.code == abi.KR_E_CAPACITY and "max_creates" in str(ei.value)
        # ... and the engine is still usable
        eng.fill(views, snap)
        eng.commit()
        got = eng.reconcile(flags)
        assert not oracle_mod.run(snap, flags).diff(got)
    finally:
        eng.close()


def test_fixed_layout_keeps_addresses_and_resident_data(oracle_mod):
    """KR_OPT_FIXED_LAYOUT: arenas laid out for the capacities.  begin() with other row counts returns the same pointers, the
    spec-JSON arena stays resident across it, and the pass (graph parameters updated in place) matches the oracle."""
    snaps = [synthetic.generate(synthetic.config("C2", seed=synthetic.SEED + i)) for i in range(3)]
    eng = Engine.for_snapshot(snaps[0][0], slack=1.3)
    eng.set_fixed_layout(True)
    try:
        addr = None
        for i, (snap, flags) in enumerate(snaps):
            views = eng.begin(snap.sizes())
            here = {k: v.ctypes.data for k, v in views.items() if v.size}
            assert addr is None or all(addr[k] == p for k, p in here.items() if k in addr), "a column moved"
            addr = here if addr is None else addr
            eng.fill(views, snap)
            # the JSON arena is the same for every seed of this config: after the first epoch only the columns travel
            eng.commit(abi.PART_ALL if i == 0 else abi.PART_COLUMNS)
            assert i == 0 or eng.last_profile()["h2d_bytes"] < 1.35 * (snap.nbytes() - snap.dims["json"])  # (small columns travel capacity-long)
            got = eng.reconcile(flags)
            assert not oracle_mod.run(snap, flags, threads=8).diff(got), i
        with pytest.raises(Exception):
            eng.set_fixed_layout(False)  # only before the first begin
    finally:
        eng.close()


@pytest.mark.parametrize("seed", [1, 2, 3, 4, 5, 6])
def test_parity_stressed_distributions(seed, oracle_mod, monkeypatch):
    """Medium snapshots with the rare branches made common: a third of the clusters suspended / on the Recreate gate (large
    phase-1 list) / waiting on expectations, half of the groups multi-host or carrying workersToDelete, many orphans."""
    rng = np.random.default_rng(seed)
    params = synthetic.SynthParams(
        n_clusters=int(rng.integers(500, 3000)), pods_per_cluster=int(rng.integers(5, 130)), groups=int(rng.integers(1, 5)),
        clusters_per_namespace=int(rng.integers(1, 200)), autoscaling_frac=float(rng.random()), suspended_frac=float(rng.random() * 0.3),
        recreate_frac=float(rng.random() * 0.4), expect_pending_frac=float(rng.random() * 0.3), wtd_group_frac=float(rng.random() * 0.6),
        orphan_frac=float(rng.random() * 0.1), multihost_frac=float(rng.random() * 0.6), steady_frac=float(rng.random()), jobs=bool(seed % 2),
        seed=synthetic.SEED + seed)
    snap, flags = synthetic.generate(params)
    flags.env_random_pod_delete = seed % 2
    got = parity(snap, flags, oracle_mod)
    assert got.n_actions > 0
    if seed % 3 == 0:
        monkeypatch.setenv("KR_FORCE_RADIX", "1")
        parity(snap, flags, oracle_mod)


def test_remaining_entry_points(oracle_mod):
    """kr_reconcile_device_only + kr_results_fetch (the split the benchmark's value leg uses), kr_reconcile_batch_profiled,
    kr_group_results_device / _copy (the multi-GPU all-gather's source) and kr_algorithmic_bytes."""
    import torch
    snap, flags = synthetic.generate(synthetic.config("C2", groups=2, jobs=True))
    want = oracle_mod.run(snap, flags, threads=8)
    eng = Engine.for_snapshot(snap)
    try:
        eng.load(snap)
        with pytest.raises(Exception):
            eng.fetch()                                   # nothing has run on this snapshot yet
        eng.reconcile_device_only(flags)                  # kernels only, results stay in HBM
        assert eng.last_profile()["kernels_ms"] > 0
        assert not want.diff(eng.fetch())                 # ... until they are asked for
        prof = eng.reconcile_profiled(flags)              # serialised, one event pair per kernel
        names = [k for k, _ in prof["kernels"]]
        assert {"k_clear", "k_build_tables", "k_match", "k_decide_small", "k_hash", "k_jobs"} <= set(names) and all(ms > 0 for _, ms in prof["kernels"])
        assert not want.diff(eng.fetch())
        ptr, nbytes = eng.group_results_device()
        assert ptr and nbytes == 32 * snap.dims["groups"]
        buf = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
        eng.group_results_copy(buf.data_ptr(), buf.numel())
        assert np.array_equal(buf.cpu().numpy().view(abi.group_result_dtype), want.groups)
        with pytest.raises(Exception):
            eng.group_results_copy(buf.data_ptr(), nbytes - 1)   # destination too small: KR_E_CAPACITY, no partial copy
        alg = eng.algorithmic_bytes()
        d = snap.dims
        # SURVEY §8(d): 144 B/cluster (32 of them the digest, counted with the hash) + 56 B/group + 4 B/workersToDelete name + 33 B/pod + L
        assert alg["hash"] == int(snap.c_json_len.sum()) + 32 * d["clusters"]
        assert alg["match"] == 112 * d["clusters"] + 56 * d["groups"] + 4 * d["wtd"] + 33 * d["pods"]
        assert alg["pass"] == alg["hash"] + alg["match"]
    finally:
        eng.close()

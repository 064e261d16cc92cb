"""The engine across the size thresholds where it changes kernel or code path, against hashlib, the CPU oracle and a few lines of
plain Python: the throughput-regime hash (k_hash2<4, 1>) and its grid-stride trips, replica-index windows past the first 1024,
the 32-worker-group and 64 / 128 / 256-pod limits of the bucket pipeline, and incremental epochs that run out of arena.

Every threshold is derived from the device's SM count in `Regimes`, the way the engine derives it; a test that claims to cross
one asserts that its sizes fall on each side of it."""
import numpy as np
import pytest

from harness import Driver, b32, compact, flip_ready, incremental, kernels, parity, set_phase, spec_bytes
from kuberay_b200 import abi, synthetic
from kuberay_b200.engine import Engine, EngineError

pytestmark = pytest.mark.gpu


class Regimes:
    """The engine's size thresholds for this device.  Mirrors launch_hash in kuberay_b200/csrc/kr_engine.cu, which the full
    pass, the incremental pass's re-hash after a JSON commit and kr_hash_batch all call: k_hash3 while
    `(n + 31) / 32 <= sm_count * 4` and k_hash2<4, 1> above; k_hash2's grid is capped at sm_count * hash_ctas_per_sm
    (2, KR_HASH_CTAS) CTAs of 128 lanes in a pass and at sm_count * 4 CTAs in kr_hash_batch, so more messages than that make
    its grid-stride loop take a second trip.
    KR_SMEM_GROUPS (kr_decide.cuh) is the widest RayCluster the bucket pipeline takes; 256 pods is the widest bucket stride."""

    def __init__(self):
        import torch
        self.sms = torch.cuda.get_device_properties(0).multi_processor_count
        self.latency_max = 32 * 4 * self.sms        # most messages hashed by k_hash3
        self.pass_trip = 128 * 2 * self.sms         # messages per grid-stride trip of k_hash2<4, 1> in a pass
        self.batch_trip = 128 * 4 * self.sms        # ... in kr_hash_batch
        self.smem_groups = 32
        self.max_stride = 256

    def throughput(self, n):
        return (n + 31) // 32 > 4 * self.sms


@pytest.fixture(scope="module")
def regimes():
    return Regimes()


# ------------------------------------------------------------------------------------------------ hash, throughput regime

def _hash_messages(n, rng):
    """n messages, mostly short: every length 0..200 (every padding and length-word position), the block edges, some up to
    9 KB.  kr_hash_batch orders them by block count, so the many classes of a few messages each put mixed warps at every
    class boundary."""
    lens = [i % 201 for i in range(n)]
    edges = [55, 56, 63, 64, 119, 120, 127, 128]
    pos = rng.permutation(n)
    for k, p in enumerate(pos[:400]):
        lens[p] = edges[k % len(edges)]
    for p in pos[400:700]:
        lens[p] = int(rng.integers(129, 9 * 1024 + 1))
    blob = rng.integers(0, 256, max(lens) + n, dtype=np.uint8).tobytes()
    return [blob[i % n:i % n + ln] for i, ln in enumerate(lens)]


def test_hash_batch_on_both_sides_of_the_throughput_threshold(regimes):
    rng = np.random.default_rng(31)
    sizes = (regimes.latency_max, regimes.latency_max + 1, regimes.batch_trip + 777)
    assert not regimes.throughput(sizes[0]) and regimes.throughput(sizes[1]) and regimes.throughput(sizes[2])
    assert sizes[1] <= regimes.batch_trip < sizes[2]          # one grid-stride trip, then two
    eng = Engine(0, max_clusters=1)
    try:
        for n in sizes:
            msgs = _hash_messages(n, rng)
            got = eng.hash_batch(msgs)
            bad = [i for i, (m, h) in enumerate(zip(msgs, got)) if b32(m).decode() != h]
            assert not bad, (n, len(bad), [len(msgs[i]) for i in bad[:10]])
    finally:
        eng.close()


def _throughput_snapshot(n_clusters, seed=7):
    """n_clusters x 4 pods, 30 % on the Recreate gate.  Each spec is shortened inside the slot the generator laid out (offsets
    stay 16-aligned, ranges inside the arena; the bytes after the new end are stale JSON the kernel must not hash): every length
    0..200, the block edges, random lengths up to the template's.  Half of the Recreate heads carry the true digest of the
    shortened spec."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=n_clusters, pods_per_cluster=4, groups=1, recreate_frac=0.3, seed=seed))
    rng = np.random.default_rng(seed)
    old = snap.c_json_len.astype(np.int64)
    sel = rng.random(n_clusters)
    new = np.where(sel < 0.4, np.arange(n_clusters) % 201, (rng.random(n_clusters) * (old + 1)).astype(np.int64))
    edge = sel > 0.95
    new[edge] = np.array([55, 56, 63, 64, 119, 120, 127, 128])[np.arange(int(edge.sum())) % 8]
    assert (new <= old).all()
    snap.c_json_len[:] = new.astype(np.uint32)
    gate = np.flatnonzero(((snap.c_flags & abi.CF_UPGRADE_RECREATE) != 0) & (snap.h_annot_state == abi.ANNOT_HASH32))
    ah = snap.h_annot_hash.reshape(-1, 32)                     # head-aux row c is cluster c's head (generator order)
    for i, c in enumerate(gate):
        h = b32(spec_bytes(snap, c))
        ah[c] = np.frombuffer(h if i % 2 == 0 else h[::-1], dtype=np.uint8)
    return snap, flags


def _check_digests(snap, res):
    want = np.frombuffer(b"".join(b32(spec_bytes(snap, c)) for c in range(snap.dims["clusters"])), dtype=np.uint8).reshape(-1, 32)
    bad = np.flatnonzero((res.hash != want).any(axis=1))
    assert not bad.size, (bad.size, bad[:10].tolist(), [int(snap.c_json_len[c]) for c in bad[:10]])


@pytest.mark.parametrize("trips", [1, 2])
def test_full_pass_in_the_throughput_regime(trips, regimes, oracle_mod, monkeypatch):
    """Digests against hashlib and full parity on both pipelines; the bucket pipeline's Recreate-gate warps wait for digests of
    k_hash2<4, 1> inside the decide kernel (spin), and, with KR_NO_HASH_SPIN=1, on the two-phase schedule."""
    n = regimes.latency_max + 3000 if trips == 1 else regimes.pass_trip + 1500
    assert regimes.throughput(n) and (n <= regimes.pass_trip) == (trips == 1)
    snap, flags = _throughput_snapshot(n)
    got, lean = parity(snap, flags, oracle_mod, both=True)
    _check_digests(snap, got)
    _check_digests(snap, lean)
    rec = (snap.c_flags & abi.CF_UPGRADE_RECREATE) != 0
    paths = got.clusters["path"][rec]
    assert (paths == abi.PATH_RECREATE_DELETE_ALL).sum() > 100 and (paths == abi.PATH_NORMAL).sum() > 100
    assert _bucket_taken(snap, flags)
    monkeypatch.setenv("KR_NO_HASH_SPIN", "1")
    got, lean = parity(snap, flags, oracle_mod, both=True)
    _check_digests(snap, lean)


def test_incremental_json_recommit_in_the_throughput_regime(regimes, oracle_mod):
    """A JSON commit between device-side epochs re-hashes every spec with k_hash2<4, 1> and re-reads every Recreate gate.  Specs
    are edited in place (same lengths): gates that matched stop matching, and gates armed with the digest of the edited spec
    start to match."""
    n = regimes.latency_max + 2000
    assert regimes.throughput(n)
    snap, flags = _throughput_snapshot(n, seed=11)
    rng = np.random.default_rng(11)
    ah = snap.h_annot_hash.reshape(-1, 32)
    cand = np.flatnonzero(((snap.c_flags & abi.CF_UPGRADE_RECREATE) != 0) & ((snap.c_flags & abi.CF_SKIP) == 0) & (snap.h_annot_state == abi.ANNOT_HASH32)
                          & (snap.h_version_state == abi.VER_CURRENT) & (snap.c_json_len > 0))
    path = oracle_mod.run(snap, flags, threads=8).clusters["path"]
    match = np.array([c for c in cand if bytes(ah[c]) == b32(spec_bytes(snap, c))])
    spoil = rng.choice(match[path[match] == abi.PATH_NORMAL], 60, replace=False)
    miss = np.setdiff1d(cand, match)
    arm = rng.choice(miss[path[miss] == abi.PATH_RECREATE_DELETE_ALL], 60, replace=False)
    edit = {int(c): int(snap.c_json_off[c]) + int(rng.integers(0, int(snap.c_json_len[c]))) for c in np.concatenate([spoil, arm])}
    for c in arm:                                              # the annotation already names the spec as it will be edited
        b = bytearray(spec_bytes(snap, c))
        b[edit[int(c)] - int(snap.c_json_off[c])] ^= 0x20
        ah[c] = np.frombuffer(b32(bytes(b)), dtype=np.uint8)
    dr = Driver(snap, flags)
    try:
        first, _ = dr.check(oracle_mod, expect_incremental=False)
        gated = first.clusters["path"]
        assert (gated[spoil] == abi.PATH_NORMAL).all() and (gated[arm] == abi.PATH_RECREATE_DELETE_ALL).all()
        for p in edit.values():
            snap.json[p] ^= 0x20
        np.copyto(dr.views["json"], snap.json)
        dr.eng.commit(abi.PART_JSON)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        assert (got.clusters["path"][spoil] == abi.PATH_RECREATE_DELETE_ALL).all() and (got.clusters["path"][arm] == abi.PATH_NORMAL).all()
        _check_digests(snap, got)
    finally:
        dr.close()


# ------------------------------------------------------------------------------------------------ replica-index windows

def _group_members(snap):
    """Worker pod rows by group row (pods keyed to their RayCluster and worker group)."""
    ckey = {(int(snap.c_ns_id[c]), int(snap.c_name_id[c])): c for c in range(snap.dims["clusters"])}
    gkey = {(int(snap.g_cluster_idx[g]), int(snap.g_name_id[g])): g for g in range(snap.dims["groups"])}
    out = {}
    worker = ((snap.p_packed >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER
    for p in np.flatnonzero(worker):
        c = ckey.get((int(snap.p_ns_id[p]), int(snap.p_cluster_name_id[p])))
        g = gkey.get((c, int(snap.p_group_name_id[p]))) if c is not None else None
        if g is not None:
            out.setdefault(g, []).append(int(p))
    return out


def _set_labels(snap, rows, labels):
    """labels[i] is the ray.io/worker-group-replica-index of rows[i]; None: the pod carries no such label."""
    for i, (p, v) in enumerate(zip(rows, labels)):
        if v is None:
            snap.p_packed[p] &= ~np.uint32(abi.PP_HAS_REPLICA_IDX)
            snap.p_replica_index[p] = i                        # a low value, which would be in use if the column counted without the flag
        else:
            snap.p_packed[p] |= np.uint32(abi.PP_HAS_REPLICA_IDX)
            snap.p_replica_index[p] = v


def _set_replicas(snap, g, replicas):
    """Group row g asks for `replicas`, no maximum (its minimum, suspension and expectations stay as they are)."""
    snap.g_replicas[g] = replicas
    snap.g_max[g] = 2 ** 31 - 1
    snap.g_flags[g] &= ~np.uint32(abi.GF_REPLICAS_NIL | abi.GF_MAX_NIL)


def _lowest_free(used, n):
    """The first n non-negative integers not in `used`."""
    out, i = [], 0
    while len(out) < n:
        if i not in used:
            out.append(i)
        i += 1
    return out


def _check_creates(snap, res, members):
    """Every group's creates against the plain rule: the lowest labels not held by its kept, labelled pods."""
    acted = set()
    for c in range(snap.dims["clusters"]):
        acted.update(res.actions_of(c)[0].tolist())
    checked = 0
    for g in range(snap.dims["groups"]):
        n = int(res.groups["n_create"][g])
        if not n:
            continue
        used = {int(snap.p_replica_index[p]) for p in members.get(g, []) if p not in acted and snap.p_packed[p] & abi.PP_HAS_REPLICA_IDX}
        got = res.creates_of(g)
        assert got.tolist() == _lowest_free(used, n), (g, n, got[:8].tolist())
        checked += n
    return checked


# (replicas, labels of the group's 20 workers) — in-use labels at the window edges 1023 / 1024 / 2047 / 2048, duplicates,
# negatives, labels at or above the bound n_running + n_create, unlabelled members, bounds ending inside a 32-bit word
_WINDOW_CASES = [
    (3000, [1023, 1024, 2047, 2048] + list(range(16))),                     # bound 3000 = 93 words + 24 bits
    (1024, list(range(19, -1, -1))),                                         # bound ends exactly at the first window's end
    (1025, [1024] + list(range(19))),                                        # ... one bit into the second: 1024 is in use but out of bounds
    (3001, [5, 5, 5, -1, -7, -2 ** 31, 1024, 1024, 31, 32, 63, 64, 2 ** 31 - 1, 3000, 3001, 0, 1, 2, None, None]),
    (1100, [None] * 10 + list(range(10, 20))),                               # unlabelled members free their values 0..9
    (5000, [1000 + 32 * i for i in range(20)]),                              # five windows, bound 5000 = 156 words + 8 bits
    (4100, [4095, 4096, 4097, 1023, 1024, 2047, 2048, 3071, 3072] + list(range(100, 111))),
    (2070, list(range(2040, 2060))),                                         # bound 2070 inside a word of window 2
    (2049, [2048, 2047, 1024, 1023] + list(range(40, 56))),
    (1057, list(range(1024, 1044))),
]


def _window_snapshot():
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=64, pods_per_cluster=41, groups=2, healthy=True, seed=3))
    members = _group_members(snap)
    assert all(len(members[g]) == 20 for g in range(snap.dims["groups"]))
    cases = {}
    for i, (replicas, labels) in enumerate(_WINDOW_CASES):
        for g in (5 * i + 1, 5 * i + 66):                                    # two groups per case, in different RayClusters
            _set_replicas(snap, g, replicas)
            _set_labels(snap, members[g], labels)
            cases[g] = replicas
    return snap, flags, members, cases


def test_replica_index_windows_on_every_pipeline(oracle_mod, monkeypatch):
    snap, flags, members, cases = _window_snapshot()
    cap = 1 << 17
    got, lean = parity(snap, flags, oracle_mod, both=True, max_creates=cap)
    assert _bucket_taken(snap, flags, max_creates=cap)
    for res in (got, lean):
        for g in cases:
            assert res.groups["n_create"][g] > 0, g
        assert _check_creates(snap, res, members) > 40000
    monkeypatch.setenv("KR_FORCE_RADIX", "1")
    got, lean = parity(snap, flags, oracle_mod, both=True, max_creates=cap)
    for res in (got, lean):
        _check_creates(snap, res, members)


def test_replica_index_windows_with_the_gate_off(oracle_mod):
    snap, flags, _, _ = _window_snapshot()
    flags.gate_multihost_indexing = 0
    got, lean = parity(snap, flags, oracle_mod, both=True, max_creates=1 << 17)
    for res in (got, lean):
        own = abi._gather_owned(res.groups["create_off"], res.groups["n_create"])
        assert own.size > 40000 and (res.create_idx[own] == -1).all()


def test_replica_index_window_filled_by_one_group(oracle_mod, monkeypatch):
    """Groups of 1100 workers (sort, then radix pipeline; the bucket pipeline leaves such a RayCluster to them): the in-use
    labels fill the whole second window, or the whole first one."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=6, pods_per_cluster=1101, groups=1, healthy=True, seed=4))
    members = _group_members(snap)
    _set_replicas(snap, 0, 2100)
    _set_labels(snap, members[0], list(range(1024, 2048)) + list(range(76)))      # free: 76..1023, then 2048..2099
    _set_replicas(snap, 1, 1150)
    _set_labels(snap, members[1], list(range(1100)))                             # free from 1100 on
    _set_replicas(snap, 2, 1500)
    _set_labels(snap, members[2], list(range(0, 2200, 2))[:1100])                # every even label below 2200
    got, lean = parity(snap, flags, oracle_mod, both=True, max_creates=1 << 14)
    for res in (got, lean):
        _check_creates(snap, res, members)
    assert got.creates_of(0)[[0, 947, 948, 999]].tolist() == [76, 1023, 2048, 2099]
    assert got.creates_of(1)[[0, 49]].tolist() == [1100, 1149]
    monkeypatch.setenv("KR_FORCE_RADIX", "1")
    for res in parity(snap, flags, oracle_mod, both=True, max_creates=1 << 14):
        _check_creates(snap, res, members)


def test_replica_index_windows_multihost(oracle_mod):
    """numOfHosts = 4: a replica's index is in use when its first pod (List order) belongs to a healthy replica; creates count
    replicas.  Both pipelines against the oracle."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=64, pods_per_cluster=41, groups=2, healthy=True, multihost_frac=1.0, seed=5))
    assert (snap.g_num_hosts == 4).all()
    members = _group_members(snap)
    cases = [(3000, [1023, 1024, 2047, 2048, 0]), (1500, [5, 5, -1, 1024, 7]), (4100, [4095, 4096, 4097, 0, 1]), (1025, [1024, 0, 1, 2, 3]),
             (2050, [2049, 2048, 2047, 1024, 1023])]
    rng = np.random.default_rng(5)
    for i, (replicas, labels) in enumerate(cases):
        for g in (3 * i + 1, 3 * i + 70):
            _set_replicas(snap, g, replicas)
            rows = members[g]
            names = np.unique(snap.p_replica_name_id[rows])
            assert names.size == 5
            for name, v in zip(names, labels):
                in_rep = [p for p in rows if snap.p_replica_name_id[p] == name]
                _set_labels(snap, in_rep, [v] * len(in_rep))
                if i == 1:                                     # a replica whose first pod carries another label than the rest
                    _set_labels(snap, [min(in_rep)], [int(rng.integers(1000, 1100))])
    got, lean = parity(snap, flags, oracle_mod, both=True, max_creates=1 << 16)
    assert _bucket_taken(snap, flags, max_creates=1 << 16)
    scaled = [g for i in range(len(cases)) for g in (3 * i + 1, 3 * i + 70)]
    for res in (got, lean):
        assert (res.groups["flags"][scaled] & abi.GR_MULTIHOST).all() and res.groups["n_create"].sum() > 20000
        assert res.creates_of(1).tolist()[:4] == [1, 2, 3, 4] and 1023 not in res.creates_of(1) and 1024 not in res.creates_of(1)


def _bucket_taken(snap, flags, **kw):
    """Whether a compact-results pass over `snap` runs the bucket pipeline (k_match2 + k_decide2)."""
    return {"k_match2", "k_decide2"} <= set(kernels(snap, compact(flags), **kw))


# ------------------------------------------------------------------------------------------------ pipeline limits

def _last_slot(n_groups):
    return min(31, n_groups - 1)


def _wide_snapshot(n_groups, multihost_frac=0.0, seed=9):
    """60 RayClusters of `n_groups` worker groups; the group slot 31 (30 of 31 groups, and 32 of 33) holds pods and asks for
    creates in every other RayCluster and a scale-down in the rest."""
    per = 4 if multihost_frac else 2
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=60, pods_per_cluster=1 + per * n_groups + (0 if multihost_frac else 3), groups=n_groups,
                                                           multihost_frac=multihost_frac, seed=seed))
    for slot in sorted({_last_slot(n_groups), 32} & set(range(n_groups))):
        g = snap.c_group_off.astype(np.int64) + slot
        up = np.arange(g.size) % 2 == 0
        snap.g_replicas[g[up]] = (3 if not multihost_frac else 2)
        snap.g_replicas[g[~up]] = 0
        snap.g_min[g] = 0
        snap.g_max[g] = 200
        snap.g_flags[g] &= ~np.uint32(abi.GF_REPLICAS_NIL | abi.GF_MIN_NIL | abi.GF_MAX_NIL)
    return snap, flags


@pytest.mark.parametrize("n_groups", [31, 32, 33])
def test_widest_cluster_at_the_worker_group_limit(n_groups, regimes, oracle_mod):
    snap, flags = _wide_snapshot(n_groups)
    assert int(snap.c_group_cnt.max()) == n_groups
    got = parity(snap, flags, oracle_mod)
    g31 = snap.c_group_off.astype(np.int64) + _last_slot(n_groups)
    assert (got.groups["n_create"][g31] > 0).any() and (got.groups["diff"][g31] < 0).any()
    assert _bucket_taken(snap, flags) == (n_groups <= regimes.smem_groups)
    if n_groups == regimes.smem_groups:
        mh, mflags = _wide_snapshot(n_groups, multihost_frac=0.3)
        slot31 = mh.c_group_off.astype(np.int64) + 31
        assert (mh.g_num_hosts[slot31] > 1).any()
        got = parity(mh, mflags, oracle_mod)
        assert (got.groups["flags"][slot31] & abi.GR_MULTIHOST).any()
        assert _bucket_taken(mh, mflags)


def test_incremental_epochs_touch_group_slot_31(oracle_mod):
    snap, flags = _wide_snapshot(32)
    members = _group_members(snap)
    slot31 = (snap.c_group_off.astype(np.int64) + 31).tolist()
    dr = Driver(snap, flags)
    try:
        dr.check(oracle_mod, expect_incremental=False)
        rows = [p for g in slot31[:20] for p in members.get(g, [])]
        assert rows
        flip_ready(snap, rows[::2]); set_phase(snap, rows[1::2], abi.PHASE_FAILED)
        dr.commit_rows(rows)
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        assert got.changed_clusters is not None and np.isin(snap.g_cluster_idx[slot31[:20]], got.changed_clusters).all()
        snap.g_replicas[slot31[20:40]] = 5
        dr.commit_objects()
        got, _ = dr.check(oracle_mod, expect_incremental=True)
        assert (got.groups["n_create"][slot31[20:40]] > 0).any()
    finally:
        dr.close()


def _one_cluster_of(size, multihost=False):
    """300 RayClusters x 20 pods (the mean picks the 64-pod stride); worker pods of clusters 1.. move into cluster 0 until it
    lists exactly `size` pods."""
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=300, pods_per_cluster=20, groups=1, seed=12))
    key0 = (snap.c_ns_id[0], snap.c_name_id[0])
    in0 = (snap.p_ns_id == key0[0]) & (snap.p_cluster_name_id == key0[1])
    worker = ((snap.p_packed >> abi.PP_NODE_TYPE_SHIFT) & 3) == abi.NT_WORKER
    move = np.flatnonzero(worker & ~in0)[:size - int(in0.sum())]
    snap.p_ns_id[move], snap.p_cluster_name_id[move], snap.p_group_name_id[move] = key0[0], key0[1], snap.g_name_id[0]
    in0 = (snap.p_ns_id == key0[0]) & (snap.p_cluster_name_id == key0[1])
    assert int(in0.sum()) == size
    if multihost:
        ws = np.flatnonzero(in0 & worker)
        snap.g_num_hosts[0] = 4
        snap.p_replica_name_id[ws] = np.uint32(0x7D000000) + (np.arange(ws.size) // 4).astype(np.uint32)
        _set_labels(snap, ws, (np.arange(ws.size) // 4).tolist())
        _set_replicas(snap, 0, ws.size // 4 + 2)
    return snap, flags


@pytest.mark.parametrize("multihost", [False, True])
def test_one_cluster_at_each_bucket_stride_edge(multihost, regimes, oracle_mod):
    for size in (64, 65, 128, 129, 256, 257):
        snap, flags = _one_cluster_of(size, multihost)
        n, c = snap.dims, snap.dims["clusters"]
        assert (n["pods"] * 5 // 4 + c - 1) // c <= 64                 # the commit's stride: 64 (kr_snapshot_begin)
        got = parity(snap, flags, oracle_mod)
        assert got.clusters["n_pods"][0] == size
        if multihost:
            assert got.groups["flags"][0] & abi.GR_MULTIHOST
        assert _bucket_taken(snap, flags) == (size <= regimes.max_stride), size


@pytest.mark.parametrize("multihost", [False, True])
def test_one_cluster_at_each_bucket_stride_edge_with_lists(multihost, regimes, oracle_mod):
    """KR_OPT_BUCKET_POD_LISTS fetching the lists: one Pod past a stride voids the attempt (k_lists_owner then leaves every owner
    unset) and the stride widens, and past 256 Pods the pass leaves the bucket pipeline; the lists fetched are those of the attempt
    that stood.  Then a second pass on the same engine, incremental wherever the first stayed on the bucket pipeline."""
    strides = (64, 128, 256)
    assert strides[-1] == regimes.max_stride
    for size in (64, 65, 128, 129, 256, 257):
        snap, flags = _one_cluster_of(size, multihost)
        flags.fetch_pod_lists = 1
        want = oracle_mod.run(snap, flags)
        eng = Engine.for_snapshot(snap, bucket_pod_lists=True)
        try:
            eng.load(snap)
            for kind in ("full", "incremental"):
                got = eng.reconcile(flags)
                rep = eng.last_pass()
                d = want.diff(got)
                assert not d, (size, kind, d[:6])
                assert got.sorted_pod_idx.size == snap.dims["pods"] and got.clusters["n_pods"][0] == size
                if size > regimes.max_stride:
                    assert rep["pipeline"] != "bucket" and rep["kind"] == "full", (size, rep)
                    continue
                stride = next(s for s in strides if size <= s)
                assert rep["pipeline"] == "bucket" and rep["kind"] == kind and rep["stride"] == stride, (size, rep)
                assert kind != "full" or rep["attempts"] == strides.index(stride), (size, rep)
        finally:
            eng.close()


# ------------------------------------------------------------------------------------------------ incremental arena exhaustion

def test_incremental_epochs_that_run_out_of_arena(oracle_mod):
    """A tight max_creates: re-decided RayClusters that outgrow their create runs take new ones at the cursor, and unhealthy
    pods grow action runs; once a cursor passes its end the epoch is void and a full pass packs the arenas again."""
    _arena_epochs(oracle_mod, lists=False)


def test_incremental_epochs_that_run_out_of_arena_with_lists(oracle_mod):
    """The same with KR_OPT_BUCKET_POD_LISTS fetching the lists every epoch: the void incremental attempt builds no lists, and
    the full pass after it does."""
    _arena_epochs(oracle_mod, lists=True)


def _arena_epochs(oracle_mod, lists):
    snap, flags = synthetic.generate(synthetic.SynthParams(n_clusters=400, pods_per_cluster=12, groups=1, healthy=True, seed=14))
    nc = snap.dims["clusters"]
    members = _group_members(snap)
    cap = 600
    dr = Driver(snap, flags, max_creates=cap, bucket_pod_lists=lists)
    dr.flags.fetch_pod_lists = int(lists)

    def check(expect_incremental=None):
        got, _ = dr.check(oracle_mod, expect_incremental)
        rep = dr.eng.last_pass()
        assert rep["pipeline"] == "bucket" and rep["kind"] == ("incremental" if incremental(got, nc) else "full"), rep
        assert got.sorted_pod_idx.size == (snap.dims["pods"] if lists else 0) and "POD_LISTS" not in rep["why"], rep
        return got, _

    try:
        got, _ = check(expect_incremental=False)
        assert got.n_create_total == 0
        base = snap.g_replicas.copy()
        kinds, prev_up, prev_bad = [], np.zeros(0, np.int64), []
        for epoch in range(12):
            up = np.arange(40 * epoch, 40 * epoch + 40) % nc                   # a rotating set of RayClusters scales up ...
            snap.g_replicas[prev_up] = base[prev_up]                          # ... and the previous one back down
            snap.g_replicas[up] = base[up] + 3
            set_phase(snap, prev_bad, abi.PHASE_RUNNING)
            bad = [members[int(g)][k] for g in (up + 200) % nc for k in (0, 1)][:40]   # pods of other RayClusters fail
            set_phase(snap, bad, abi.PHASE_FAILED)
            dr.commit_objects()
            dr.commit_rows(list(bad) + list(prev_bad))
            got, _ = check()
            inc = incremental(got, nc)
            full = got.changed_clusters is None and got.n_changed == nc
            assert inc != full
            kinds.append(inc)
            prev_up, prev_bad = up, bad
            if len(kinds) >= 2 and not kinds[-2] and kinds[-1]:
                break
        assert len(kinds) >= 2 and not kinds[-2] and kinds[-1], kinds     # a full pass, then incremental again
        # more creates than the arena holds: the epoch reports KR_E_CAPACITY, and the engine is usable afterwards
        snap.g_replicas[:] = base + 2
        dr.commit_objects()
        with pytest.raises(EngineError) as ei:
            dr.eng.reconcile(dr.flags)
        assert ei.value.code == abi.KR_E_CAPACITY and "max_creates" in str(ei.value)
        snap.g_replicas[:] = base
        set_phase(snap, prev_bad, abi.PHASE_RUNNING)
        dr.commit_objects()
        dr.commit_rows(prev_bad)
        dr.prev = None
        check(expect_incremental=False)   # (the overrun left runs unwritten: this pass starts over)
        flip_ready(snap, bad)
        dr.commit_rows(bad)
        check(expect_incremental=True)
    finally:
        dr.close()

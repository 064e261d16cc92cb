"""The engine's hash tables under keys built to collide (CPU half; tests/test_gpu_table_keys.py runs the engine on them).

Every join of the engine goes through an open-addressing table keyed by interned ids: (namespace, ray.io/cluster) -> RayCluster,
(namespace, pod name) -> workersToDelete entries (behind a Bloom bitmap) and pod row -> head-aux row.  The packers hand out small
dense ids, so the tables' probe chains stay short.  tests/table_keys.py restates the hashes and builds snapshots in which
those chains are long, start in the last slot and wrap, and whose ids cover the whole u32 domain; this file pins the hashes to
kr_common.cuh and checks the constructions and the oracle on them:

  * collide(a, u): the name id b with hash_pair(a, b) == mix32(u) (the multiplier of b is odd, so it has an inverse mod 2^32);
    U[k] = mix32^-1(k << 20 | 0xFFFFF), so every key built from a U[k] lands in the last slot of every table of up to 2^20 slots;
  * relabel(snap, flags, f): the same snapshot under a bijection f of the ids (0 and 1 stay fixed); the results of a pass map
    through f as well, which the oracle must honour (its own map hashes with mix64, so these keys do not collide there);
  * K1 / K2 / K3: one long RayCluster chain, one long workersToDelete chain with the Bloom bitmap at its cap, head Pods at pod rows
    that all hash to the last slot of the head-aux table.
"""
import re
from pathlib import Path

import numpy as np
import pytest

from harness import members
from kuberay_b200 import abi, synthetic
from table_keys import (BLOOM, FLAG_IDS, HEAD_ROWS, ID_COLUMNS, LAST, M32, MIX, PAIR, RESULT_IDS, U, bloom2, collide, hash_pair, ids_in, in_chain,
                        k1, k2, k3, map_results, mix32, mix32_inv, node_type, random_map, relabel)

CSRC = Path(__file__).resolve().parents[1] / "kuberay_b200" / "csrc"


def _source(name):
    return " ".join((CSRC / name).read_text().split())


def test_hashes_match_the_kernel_source():
    src = _source("kr_common.cuh")
    body = re.search(r"uint32_t mix32\(uint32_t x\) \{ (.*?) return x; \}", src).group(1)
    ops = [int(sh) if sh else int(mul, 16) for sh, mul in re.findall(r"x \^= x >> (\d+);|x \*= (0x[0-9a-fA-F]+)u;", body)]
    assert tuple(ops) == MIX, body
    m = re.search(r"uint32_t hash_pair\(uint32_t a, uint32_t b\) \{ return mix32\(a \* (0x\w+)u \^ \(b \* (0x\w+)u \+ (0x\w+)u\)\); \}", src)
    assert m and tuple(int(x, 16) for x in m.groups()) == PAIR
    m = re.search(r"uint32_t bloom2\(uint32_t hk\) \{ return \(hk \* (0x\w+)u\) >> (\d+); \}", src)
    assert m and (int(m.group(1), 16), int(m.group(2))) == BLOOM
    assert "#define KR_EMPTY64 0xFFFFFFFFFFFFFFFFull" in src and "#define KR_EMPTY32 0xFFFFFFFFu" in src
    # what the constructions below rely on besides the hashes: tables of at least 2n slots (a power of two, probed with `& mask`),
    # the Bloom bitmap capped at 2^17 bits, the head-aux table hashed with mix32 of the pod row
    eng = _source("kr_engine.cu")
    for t in ("n_clusters", "n_wtd", "n_heads"):
        assert f"pow2_at_least(2ull * n.{t})" in eng
    assert "bits < (1ull << 17)" in eng
    for f in ("kr_match.cuh", "kr_incr.cuh"):
        assert "mix32(p) & sc.aux_mask" in _source(f)


def test_restated_hashes_known_values():
    # bit-exact restatement of the C expressions with Python integers
    def ref_mix(x):
        x ^= x >> 16; x = (x * MIX[1]) & M32; x ^= x >> 15; x = (x * MIX[3]) & M32; x ^= x >> 16   # noqa: E702
        return x
    rng = np.random.default_rng(0)
    xs = rng.integers(0, 1 << 32, 2000, dtype=np.uint64).tolist() + [0, 1, M32, 0x80000000]
    assert mix32(xs).tolist() == [ref_mix(x) for x in xs]
    assert mix32_inv(mix32(xs)).tolist() == xs
    a, b = xs[:1000], xs[1000:2000]
    assert hash_pair(a, b).tolist() == [ref_mix(((x * PAIR[0]) & M32) ^ (((y * PAIR[1]) + PAIR[2]) & M32)) for x, y in zip(a, b)]
    assert bloom2(a).tolist() == [((x * BLOOM[0]) & M32) >> BLOOM[1] for x in a]


def test_constructor_collides():
    assert np.unique(U).size == U.size == 4096
    assert ((mix32(U) & np.uint32(LAST)) == LAST).all()
    for a in (2, 3, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE, 123456789):
        b = collide(a, U)
        h = hash_pair(a, b)
        assert (h == mix32(U)).all() and np.unique(b).size == b.size      # all 32 bits, distinct names inside one namespace
        for mask in (1, 0xFF, 0xFFF, 0xFFFF, LAST):
            assert ((h & np.uint32(mask)) == mask).all()                     # the last slot of every table up to 2^20 slots
    # one inner value, five namespaces: five different names with one and the same 32-bit hash (and Bloom bits)
    ns = np.array([2, 0x1234, 0x80000000, 0xDEADBEEF, 0xFFFFFFFE])
    bs = collide(ns, np.full(ns.size, U[7]))
    assert np.unique(bs).size == 5 and np.unique(hash_pair(ns, bs)).size == 1
    assert HEAD_ROWS.size == 76 and ((mix32(HEAD_ROWS) & np.uint32(0xFFF)) == 0xFFF).all()


def test_relabel_covers_every_id_column():
    want = {"c_ns_id", "c_name_id", "c_ext_err_msg_id", "c_old_cond_reason_id", "c_old_cond_msg_id", "c_old_head_ids", "c_svc_ip_id",
            "c_svc_name_id", "c_summary_id", "g_name_id", "w_name_id", "p_ns_id", "p_cluster_name_id", "p_group_name_id", "p_name_id",
            "p_replica_name_id", "h_ready_reason_id", "h_ready_msg_id", "h_pod_ip_id", "j_ns_id", "j_cluster_name_id", "j_summary_id"}
    assert set(ID_COLUMNS) == want == set(synthetic._ID_COLUMNS)
    assert FLAG_IDS == ("id_head_not_found_reason", "id_head_not_found_msg")
    assert set(RESULT_IDS) == {"head_ready_reason_id", "head_ready_msg_id", "head_ids"}
    assert not [n for dt in (abi.group_result_dtype, abi.job_result_dtype) for n in dt.names if n.endswith(("_id", "_ids"))]
    snap, flags = synthetic.generate(synthetic.config("C1", jobs=True, wtd_group_frac=1.0, autoscaling_frac=1.0))
    f = random_map(ids_in(snap, flags), np.random.default_rng(1))
    out, fl = relabel(snap, flags, f)
    for name, _dt, _m, _d in abi.COLUMNS:
        a, b = snap.cols[name], out.cols[name]
        if name in ID_COLUMNS:
            assert np.array_equal(b, f(a)) and np.array_equal(f.inverse()(b), a), name
            assert np.array_equal(a <= 1, b <= 1), name                    # 0 and 1 stay, nothing else maps onto them
        else:
            assert np.array_equal(a, b), name
    assert (fl.id_head_not_found_reason, fl.id_head_not_found_msg) == (f.one(flags.id_head_not_found_reason), f.one(flags.id_head_not_found_msg))
    v = f.dst[2:]
    assert (v >= 2).all() and (v <= 0xFFFFFFFE).all() and (v >= 1 << 31).sum() > v.size // 4 and 0xFFFFFFFE in v.tolist()


@pytest.fixture(scope="module")
def cases():
    return {"K1": k1(), "K2": k2(), "K3": k3()}


def test_k_snapshots_have_their_shape(cases):
    K1, K2, K3 = cases["K1"], cases["K2"], cases["K3"]
    s = K1.snap
    h = hash_pair(s.c_ns_id, s.c_name_id)
    assert ((h & np.uint32(LAST)) == LAST).sum() >= 470 and in_chain(h).all()
    assert np.unique(s.c_ns_id).size >= 45 and np.unique(s.c_ns_id, return_counts=True)[1].max() >= 140
    a, b, c = K1.swapped
    assert (s.c_ns_id[a], s.c_name_id[a]) == (s.c_name_id[b], s.c_ns_id[b])
    for c in K1.shared:   # same name as a RayCluster of another namespace, both keys in the chain
        assert ((s.c_name_id == s.c_name_id[c]) & (s.c_ns_id != s.c_ns_id[c])).sum() == 1
    ck = set(zip(s.c_ns_id.tolist(), s.c_name_id.tolist()))
    po = K1.orphans
    assert in_chain(hash_pair(s.p_ns_id[po], s.p_cluster_name_id[po])).all()
    assert not ck & set(zip(s.p_ns_id[po].tolist(), s.p_cluster_name_id[po].tolist()))
    assert members(s, K1.large).size > 256 and s.c_group_cnt[K1.wide] > 32
    assert (s.g_num_hosts > 1).any() and (s.c_flags & abi.CF_UPGRADE_RECREATE).any()
    assert (s.c_ns_id >= 1 << 31).any() and (s.p_name_id == 0xFFFFFFFE).any() | (s.c_ns_id == 0xFFFFFFFE).any()
    s = K2.snap
    assert s.dims["wtd"] > 2048
    wns = np.repeat(s.c_ns_id[s.g_cluster_idx], s.g_wtd_cnt)
    assert ((hash_pair(wns, s.w_name_id) & np.uint32(LAST)) == LAST).all()
    assert np.unique(s.w_name_id).size < s.dims["wtd"]                       # duplicates
    listed = set(hash_pair(wns, s.w_name_id).tolist())
    dk = hash_pair(s.p_ns_id[K2.decoys], s.p_name_id[K2.decoys])
    assert all(x in listed for x in dk.tolist())                              # same 32-bit hash as a listed name: both Bloom bits set
    assert not np.isin(s.p_name_id[K2.decoys], s.w_name_id).any()
    s = K3.snap
    assert ((mix32(s.h_pod_idx) & np.uint32(0xFFF)) == 0xFFF).sum() == K3.hot.size == 60 and np.isin(K3.hot, s.h_pod_idx).all()
    hk = (s.p_ns_id[K3.hot].astype(np.uint64) << np.uint64(32)) | s.p_cluster_name_id[K3.hot]
    assert sorted(np.unique(np.unique(hk, return_counts=True)[1]).tolist()) == [1, 2]        # RayClusters with 2 heads ...
    assert 0 < (node_type(s)[s.h_pod_idx] == abi.NT_HEAD).sum() and any(                        # ... and with none
        not (node_type(s)[members(s, c)] == abi.NT_HEAD).any() for c in range(5))


def _same(a, b, what):
    d = a.diff(b)
    assert not d, (what, d[:8])


@pytest.mark.parametrize("seed0", [0, 100])
def test_oracle_is_relabelling_invariant_fuzz(seed0, oracle_mod):
    import fuzz_objects
    for seed in range(seed0, seed0 + 60):
        snap, flags = fuzz_objects.snapshot(seed, big=(seed % 10 == 0))
        f = random_map(ids_in(snap, flags), np.random.default_rng(seed))
        rs, rf = relabel(snap, flags, f)
        _same(oracle_mod.run(rs, rf), map_results(oracle_mod.run(snap, flags), f), seed)


@pytest.mark.parametrize("name", ["K1", "K2", "K3"])
def test_oracle_is_relabelling_invariant_k(name, cases, oracle_mod):
    k = cases[name]
    want = oracle_mod.run(k.orig, k.flags, threads=4)
    got = oracle_mod.run(k.snap, k.kflags, threads=4)
    _same(got, map_results(want, k.f), name)
    assert got.n_actions > 0

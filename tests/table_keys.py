"""Snapshots whose keys collide in the engine's hash tables (tests/test_table_keys.py checks them and the oracle on them,
tests/test_gpu_table_keys.py runs the engine on them).

Every join of the engine goes through an open-addressing table keyed by interned ids: (namespace, ray.io/cluster) -> RayCluster,
(namespace, pod name) -> workersToDelete entries (behind a Bloom bitmap) and pod row -> head-aux row.  The packers hand out small
dense ids, so the tables' probe chains stay short.  This module restates the hashes (test_table_keys.py pins them to
kr_common.cuh) and builds snapshots in which those chains are long, start in the last slot and wrap, and whose ids cover the whole u32 domain:

  * collide(a, u): the name id b with hash_pair(a, b) == mix32(u) (the multiplier of b is odd, so it has an inverse mod 2^32);
    U[k] = mix32^-1(k << 20 | 0xFFFFF), so every key built from a U[k] lands in the last slot of every table of up to 2^20 slots;
  * relabel(snap, flags, f): the same snapshot under a bijection f of the ids (0 and 1 stay fixed); the results of a pass map
    through f as well, which the oracle must honour (its own map hashes with mix64, so these keys do not collide there);
  * K1 / K2 / K3: one long RayCluster chain, one long workersToDelete chain with the Bloom bitmap at its cap, head Pods at pod rows
    that all hash to the last slot of the head-aux table.
"""
import copy
from types import SimpleNamespace

import numpy as np

from harness import members, with_wtd_lists
from kuberay_b200 import abi, synthetic
from kuberay_b200.snapshot import Snapshot

M32 = 0xFFFFFFFF
MIX = (16, 0x7FEB352D, 15, 0x846CA68B, 16)          # mix32: x ^= x >> 16; x *= ..; x ^= x >> 15; x *= ..; x ^= x >> 16
PAIR = (0x9E3779B1, 0x85EBCA77, 0x165667B1)         # hash_pair(a, b) = mix32(a * P0 ^ (b * P1 + P2))
BLOOM = (0x9E3779B1, 9)                             # bloom2(hk) = (hk * B0) >> B1
LAST = 0xFFFFF                                      # low 20 bits of every constructed hash
WINDOW = 16                                         # keys homed in slots 0..15 also sit in a wrapped chain


def _u(x):
    return np.array(x, dtype=np.uint64, ndmin=1) & np.uint64(M32)


def mix32(x):
    x = _u(x)
    x ^= x >> np.uint64(MIX[0])
    x = (x * np.uint64(MIX[1])) & np.uint64(M32)
    x ^= x >> np.uint64(MIX[2])
    x = (x * np.uint64(MIX[3])) & np.uint64(M32)
    x ^= x >> np.uint64(MIX[4])
    return x.astype(np.uint32)


def mix32_inv(y):
    x = _u(y)
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(pow(MIX[3], -1, 1 << 32))) & np.uint64(M32)
    x ^= (x >> np.uint64(15)) ^ (x >> np.uint64(30))
    x = (x * np.uint64(pow(MIX[1], -1, 1 << 32))) & np.uint64(M32)
    x ^= x >> np.uint64(16)
    return x.astype(np.uint32)


def hash_pair(a, b):
    a, b = _u(a), _u(b)
    return mix32(((a * np.uint64(PAIR[0])) & np.uint64(M32)) ^ (((b * np.uint64(PAIR[1])) + np.uint64(PAIR[2])) & np.uint64(M32)))


def bloom2(hk):
    return (((_u(hk) * np.uint64(BLOOM[0])) & np.uint64(M32)) >> np.uint64(BLOOM[1])).astype(np.uint32)


def collide(a, u):
    """The name id b with hash_pair(a, b) == mix32(u), for every namespace id a."""
    a, u = _u(a), _u(u)
    inner = ((u ^ ((a * np.uint64(PAIR[0])) & np.uint64(M32))) + np.uint64((1 << 32) - PAIR[2])) & np.uint64(M32)
    return ((inner * np.uint64(pow(PAIR[1], -1, 1 << 32))) & np.uint64(M32)).astype(np.uint32)


U = mix32_inv((np.arange(4096, dtype=np.uint64) << np.uint64(20)) | np.uint64(LAST))   # distinct inner values, all homed in the last slot
HEAD_ROWS = np.flatnonzero((mix32(np.arange(300000)) & 0xFFF) == 0xFFF)                 # last slot of every head-aux table of <= 4096 slots


def in_chain(h):
    """Keys homed in the last slot or in the first WINDOW slots of any table of up to 2^20 slots (the run of a wrapped chain)."""
    low = np.asarray(h, dtype=np.uint32) & np.uint32(LAST)
    return (low == LAST) | (low < WINDOW)


# ------------------------------------------------------------------------------------------------ relabelling
ID_COLUMNS = tuple(name for name, dt, _m, _d in abi.COLUMNS if dt is np.uint32 and name.endswith(("_id", "_ids")))
FLAG_IDS = tuple(name for name, _t in abi.kr_flags._fields_ if name.startswith("id_"))
RESULT_IDS = tuple(name for name in abi.cluster_result_dtype.names if name.endswith(("_id", "_ids")))


class IdMap:
    """A bijection of ids: 0 and 1 fixed, `src[i]` -> `dst[i]`.  Applying it to an id outside its domain is an error."""

    def __init__(self, src, dst):
        src = np.concatenate([[0, 1], np.asarray(src, dtype=np.uint64)]).astype(np.uint32)
        dst = np.concatenate([[0, 1], np.asarray(dst, dtype=np.uint64)]).astype(np.uint32)
        order = np.argsort(src)
        self.src, self.dst = src[order], dst[order]
        assert np.unique(self.src).size == self.src.size and np.unique(self.dst).size == self.dst.size, "not a bijection"
        assert not (self.dst == np.uint32(M32)).any(), "0xFFFFFFFF is not an id"

    def __call__(self, a):
        a = np.asarray(a, dtype=np.uint32)
        i = np.minimum(np.searchsorted(self.src, a), self.src.size - 1)
        assert (self.src[i] == a).all(), "id outside the map's domain"
        return self.dst[i]

    def inverse(self):
        return IdMap(self.dst[2:], self.src[2:])

    def one(self, x):
        return int(self(np.array([x], dtype=np.uint32))[0])


def ids_in(snap, flags):
    parts = [snap.cols[c].ravel() for c in ID_COLUMNS] + [np.array([getattr(flags, k) for k in FLAG_IDS], dtype=np.uint32)]
    ids = np.unique(np.concatenate(parts))
    return ids[ids > 1]


def relabel(snap, flags, f):
    """A copy of (snap, flags) with every id column and id flag mapped through f."""
    out = Snapshot(**{"n_" + k if k != "json" else "json_bytes": v for k, v in snap.dims.items()})
    for name, _dt, _m, _d in abi.COLUMNS:
        out.cols[name][:] = f(snap.cols[name]) if name in ID_COLUMNS else snap.cols[name]
    fl = abi.kr_flags.from_buffer_copy(flags)
    for k in FLAG_IDS:
        setattr(fl, k, int(f(getattr(flags, k))))
    return out, fl


def map_results(res, f):
    """The records a pass over relabel(snap, f) must return, given the records of the pass over snap."""
    out = copy.copy(res)
    out.clusters = res.clusters.copy()
    for name in RESULT_IDS:
        out.clusters[name] = f(res.clusters[name])
    return out


def random_map(ids, rng):
    """A random bijection of `ids` onto [2, 0xFFFFFFFE]: about half of the values at 2^31 and above, 0xFFFFFFFE itself taken."""
    col = Collider(rng)
    return col.finish(ids)


class Collider:
    """Builds a bijection f of the ids under which chosen (namespace, name) keys all hash to the last slot."""

    NS_VALUES = (0xFFFFFFFE, 0x80000000, 0x7FFFFFFF, 2, 0xFFFFFFFD, 0x80000001)  # the first namespaces' images

    def __init__(self, rng):
        self.rng = rng
        self.f = {}
        self.used = {0, 1, M32}
        self.ks = {}        # namespace image -> inner-value indexes taken in it
        self.order = {}     # namespace image -> the order in which it hands out inner values (its own permutation)
        self.n_ns = 0

    def _take(self, old, new):
        assert old not in self.f and new not in self.used, (old, new)
        self.f[old] = new
        self.used.add(new)

    def _fresh(self):
        while True:
            v = int(self.rng.integers(2, M32))
            if v not in self.used:
                return v

    def ns(self, old):
        """f(old) for a namespace id (one of NS_VALUES for the first few, random after that)."""
        if old not in self.f:
            v = self.NS_VALUES[self.n_ns] if self.n_ns < len(self.NS_VALUES) and self.NS_VALUES[self.n_ns] not in self.used else self._fresh()
            self.n_ns += 1
            self._take(old, v)
        return self.f[old]

    def chain(self, ns, name, k=None):
        """Give `name` the image that puts (ns, name) in the last slot, through inner value U[k] (the next free one of the namespace by
        default).  -> k, or None when `name` has an image already."""
        a = self.ns(ns)
        if name in self.f:
            return None
        taken = self.ks.setdefault(a, set())
        if a not in self.order:
            self.order[a] = self.rng.permutation(len(U)).tolist()
        for kk in ([k] if k is not None else self.order[a]):
            if kk in taken:
                continue
            b = int(collide(a, U[kk])[0])
            if b in self.used:
                continue
            taken.add(kk)
            self._take(name, b)
            return kk
        raise ValueError("no inner value left in this namespace")

    def search_ns(self, old, name, k=None):
        """A fresh namespace image for `old` with (old, name) in the chain's run.  With `k`, `name` gets the image collide(f(old), U[k])
        and the key (name, old) — the halves swapped — must sit in the run instead."""
        cand = self.rng.integers(2, M32, 1 << 21, dtype=np.uint64)
        if k is None:
            ok = in_chain(hash_pair(cand, self.f[name]))
        else:
            ok = in_chain(hash_pair(collide(cand, U[k]), cand))
        for a in cand[ok].tolist():
            b = int(collide(a, U[k])[0]) if k is not None else None
            if a not in self.used and (b is None or (b not in self.used and b != a)):
                self._take(old, a)
                self.ks[a] = set()
                if k is not None:
                    self.ks[a].add(k)
                    self._take(name, b)
                return a
        raise ValueError("no namespace image found")

    def finish(self, ids):
        ids = [int(i) for i in np.unique(np.asarray(list(ids), dtype=np.uint64)) if i > 1]
        rest = [i for i in ids if i not in self.f]
        if 0xFFFFFFFE not in self.used and rest:
            self._take(rest.pop(), 0xFFFFFFFE)
        cand = self.rng.integers(2, M32, 2 * len(rest) + 64, dtype=np.uint64)
        _, first = np.unique(cand, return_index=True)
        cand = cand[np.sort(first)]
        cand = cand[~np.isin(cand, np.fromiter(self.used, dtype=np.uint64))][:len(rest)]
        assert cand.size == len(rest)
        for old, new in zip(rest, cand.tolist()):
            self.f[old] = new
        self.used.update(cand.tolist())
        src = np.fromiter(self.f.keys(), dtype=np.uint64)
        return IdMap(src, np.fromiter((self.f[k] for k in src.tolist()), dtype=np.uint64, count=src.size))


# ------------------------------------------------------------------------------------------------ snapshot surgery (dense ids)
def node_type(snap):
    return (snap.p_packed >> abi.PP_NODE_TYPE_SHIFT) & 3


def move_key(snap, c, ns=None, name=None):
    """RayCluster c under the key (ns, name), with every Pod and RayJob that named its old key."""
    ons, onm = int(snap.c_ns_id[c]), int(snap.c_name_id[c])
    ns, name = ons if ns is None else ns, onm if name is None else name
    pm = (snap.p_ns_id == ons) & (snap.p_cluster_name_id == onm)
    snap.p_ns_id[pm], snap.p_cluster_name_id[pm] = ns, name
    jm = (snap.j_ns_id == ons) & (snap.j_cluster_name_id == onm)
    snap.j_ns_id[jm], snap.j_cluster_name_id[jm] = ns, name
    snap.c_ns_id[c], snap.c_name_id[c] = ns, name


class Fresh:
    def __init__(self, snap, flags):
        self.n = int(max(ids_in(snap, flags).max(initial=1), 1)) + 1

    def __call__(self, k=None):
        if k is None:
            self.n += 1
            return self.n - 1
        out = np.arange(self.n, self.n + k, dtype=np.uint32)
        self.n += k
        return out


def _case(orig, flags, col, extra_ids=(), **extra):
    f = col.finish(np.concatenate([ids_in(orig, flags), np.asarray(extra_ids, dtype=np.uint32)]))
    snap, kflags = relabel(orig, flags, f)
    return SimpleNamespace(orig=orig, flags=flags, f=f, snap=snap, kflags=kflags, **extra)


# ------------------------------------------------------------------------------------------------ K1: one wrapping RayCluster chain
def k1(seed=1):
    """About 480 RayClusters whose keys all start in the last slot: three namespaces of about 145, forty in namespaces of their own,
    eight sharing a name with a RayCluster of another namespace, one pair with swapped halves ((a, b) and (b, a)) and one whose
    swap only Pods name.  One of them lists 300 Pods, one has 40 worker groups, some have multi-host groups or a Recreate gate.
    Orphan Pods and RayJobs name absent keys of the same chain; `absent` holds spare absent keys for epochs (images)."""
    rng = np.random.default_rng(seed)
    p = synthetic.SynthParams(n_clusters=480, pods_per_cluster=12, groups=2, clusters_per_namespace=160, jobs=True, multihost_frac=0.1,
                              recreate_frac=0.05, autoscaling_frac=0.5, wtd_group_frac=0.3, seed=synthetic.SEED + seed)
    s, flags = synthetic.generate(p)
    large, wide = 300, 310
    synthetic.grow_clusters(s, [large], 300)
    s = synthetic.widen_clusters(s, [wide], 40)
    fresh = Fresh(s, flags)
    col = Collider(rng)
    A, B, C = int(s.c_ns_id[200]), int(s.c_ns_id[400]), int(s.c_ns_id[100])
    # swapped halves: (A, B) and (B, A) both present; (A, C) present while only Pods name (C, A)
    move_key(s, 200, name=B)
    move_key(s, 400, name=A)
    move_key(s, 201, name=C)
    strays = members(s, 202)[node_type(s)[members(s, 202)] == abi.NT_WORKER][:3]
    s.p_ns_id[strays], s.p_cluster_name_id[strays] = C, A
    col.search_ns(A, B, k=0)
    col.chain(A, C)
    # RayClusters in namespaces of their own, and RayClusters sharing a name with one of namespace C
    for c in range(40):
        move_key(s, c, ns=fresh())
    shared = []
    for i in range(8):
        y, n = fresh(), int(s.c_name_id[100 + i])
        move_key(s, 40 + i, ns=y, name=n)
        col.chain(C, n)
        col.search_ns(y, n)
        shared.append(40 + i)
    for c in range(s.dims["clusters"]):
        col.chain(int(s.c_ns_id[c]), int(s.c_name_id[c]))
    # orphans labelled for absent keys of the chain, RayJobs naming absent keys
    workers = np.flatnonzero(node_type(s) == abi.NT_WORKER)
    orph = rng.choice(workers[~np.isin(workers, strays)], 40, replace=False)
    for r in orph:
        z = fresh()
        s.p_cluster_name_id[r] = z
        col.chain(int(s.p_ns_id[r]), z)
    for j in range(0, min(20, s.dims["jobs"])):
        z = fresh()
        s.j_cluster_name_id[j] = z
        col.chain(int(s.j_ns_id[j]), z)
    spare = [(C, fresh()) for _ in range(8)]
    for ns, z in spare:
        col.chain(ns, z)
    case = _case(s.validate(), flags, col, extra_ids=[z for _, z in spare], large=large, wide=wide, shared=shared, swapped=(200, 400, 201),
                 orphans=orph)
    case.absent = [(case.f.one(ns), case.f.one(z)) for ns, z in spare]
    return case


# ------------------------------------------------------------------------------------------------ K2: one long workersToDelete chain
def k2(seed=2):
    """1 200 RayClusters of two worker groups whose workersToDelete lists hold about 3 000 names (the Bloom bitmap at its cap), every
    listed (namespace, name) key homed in the last slot: names of the group's own workers, of the other group's, of a RayCluster of
    the same namespace, of nothing, and duplicates.  `decoys` are Pods of other namespaces whose keys hash exactly like a listed
    name (both Bloom bits set) without being listed."""
    rng = np.random.default_rng(seed)
    p = synthetic.SynthParams(n_clusters=1200, pods_per_cluster=12, groups=2, clusters_per_namespace=100, autoscaling_frac=1.0, wtd_group_frac=0.0,
                              seed=synthetic.SEED + seed)
    s, flags = synthetic.generate(p)
    fresh = Fresh(s, flags)
    worker = node_type(s) == abi.NT_WORKER
    by_group = {}
    gkey = {}
    for g in range(s.dims["groups"]):
        c = int(s.g_cluster_idx[g])
        m = members(s, c)
        by_group[g] = m[worker[m] & (s.p_group_name_id[m] == s.g_name_id[g])]
        gkey[g] = c
    lists = []
    for g in range(s.dims["groups"]):
        c = gkey[g]
        other_g = int(s.c_group_off[c]) + (1 - (g - int(s.c_group_off[c])))
        same_ns = np.flatnonzero(s.c_ns_id == s.c_ns_id[c])
        other_c = int(same_ns[(np.searchsorted(same_ns, c) + 1) % same_ns.size])
        lst = []
        for _ in range(int(rng.integers(0, 4))):
            kind = rng.random()
            if kind < 0.5 and by_group[g].size:
                lst.append(int(s.p_name_id[rng.choice(by_group[g])]))
            elif kind < 0.65 and by_group[other_g].size:
                lst.append(int(s.p_name_id[rng.choice(by_group[other_g])]))
            elif kind < 0.8 and other_c != c:
                lst.append(int(s.p_name_id[rng.choice(members(s, other_c))]))
            else:
                prev = lst + (lists[g - 1] if g and s.c_ns_id[gkey[g - 1]] == s.c_ns_id[c] else [])
                lst.append(int(prev[int(rng.integers(len(prev)))]) if kind >= 0.9 and prev else fresh())
        lists.append(lst)
    s = with_wtd_lists(s, lists)
    col = Collider(rng)
    ns_of_w = np.repeat(s.c_ns_id[s.g_cluster_idx], s.g_wtd_cnt)
    for ns, nm in zip(ns_of_w.tolist(), s.w_name_id.tolist()):
        col.chain(ns, nm)
    listed = np.isin(s.p_name_id, s.w_name_id)
    decoys = rng.choice(np.flatnonzero(~listed), 400, replace=False)
    images = [(b, sorted(ks)) for b, ks in col.ks.items()]
    for r in decoys:
        a = col.ns(int(s.p_ns_id[r]))
        other = [(b, ks) for b, ks in images if b != a]
        b, ks = other[int(rng.integers(len(other)))]
        free = sorted(k for k in ks if k not in col.ks.setdefault(a, set()))
        col.chain(int(s.p_ns_id[r]), int(s.p_name_id[r]), k=free[int(rng.integers(len(free)))])
    return _case(s, flags, col, decoys=decoys)


# ------------------------------------------------------------------------------------------------ K3: head Pods at colliding rows
def k3(seed=3, n_hot=60):
    """1 600 RayClusters in 300 000 pod rows: the head Pods of the first 60 sit at pod rows that all hash to the last slot of the
    head-aux table (HEAD_ROWS), every other row holds a worker, another head, an orphan or nothing (a free row); five RayClusters lost
    their head to another one (0 and 2 heads).  `spare` are colliding rows left free for head Pods to come to."""
    rng = np.random.default_rng(seed)
    base, flags = synthetic.generate(synthetic.SynthParams(n_clusters=1600, pods_per_cluster=8, groups=1, clusters_per_namespace=100,
                                                           recreate_frac=0.1, seed=synthetic.SEED + seed))
    heads = np.flatnonzero(node_type(base) == abi.NT_HEAD)
    assert heads.size == base.dims["heads"]
    hot = np.array([int(heads[np.isin(heads, members(base, c))][0]) for c in range(n_hot)])
    for i in range(5):   # the head Pod of RayCluster i now names RayCluster i + 5 (same namespace)
        base.p_cluster_name_id[hot[i]] = base.c_name_id[i + 5]
    n, rows = 300000, HEAD_ROWS
    assert rows.size >= n_hot + 8 and rows[-1] < n
    new_row = np.zeros(base.dims["pods"], dtype=np.int64)
    new_row[hot] = rows[:n_hot]
    others = np.setdiff1d(np.arange(base.dims["pods"]), hot)
    free = np.setdiff1d(np.arange(n), rows)
    new_row[others] = np.sort(rng.choice(free, others.size, replace=False))
    d = base.dims
    s = Snapshot(d["clusters"], d["groups"], d["wtd"], n, d["heads"], d["jobs"], d["json"])
    for name, _dt, _m, dim in abi.COLUMNS:
        if dim != "pods":
            s.cols[name][:] = base.cols[name]
    s.p_packed[:] = abi.PP_TOMBSTONE
    for name in (c for c, _dt, _m, dim in abi.COLUMNS if dim == "pods"):
        s.cols[name][new_row] = base.cols[name]
    s.h_pod_idx[:] = new_row[base.h_pod_idx].astype(np.uint32)
    fresh = Fresh(base, flags)
    empty = np.setdiff1d(free, new_row[others])
    orph = np.sort(rng.choice(empty, empty.size // 3, replace=False))
    nss = np.unique(base.c_ns_id)
    s.p_ns_id[orph] = nss[rng.integers(0, nss.size, orph.size)]
    s.p_cluster_name_id[orph] = fresh(16)[rng.integers(0, 16, orph.size)]
    s.p_group_name_id[orph] = base.g_name_id[0]
    s.p_name_id[orph] = fresh(orph.size)
    s.p_packed[orph] = (abi.NT_WORKER << abi.PP_NODE_TYPE_SHIFT) | (abi.PHASE_RUNNING << abi.PP_PHASE_SHIFT) | (abi.COND_TRUE << abi.PP_READY_SHIFT)
    col = Collider(rng)
    return _case(s.validate(), flags, col, hot=rows[:n_hot], spare=rows[n_hot:])

"""ctypes binding of the C-ABI library libkrengine.so (include/kr_engine.h) — the product path.

There is NO CPU fallback: if the CUDA library is missing or no device is visible, construction raises.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from . import abi
from .snapshot import Snapshot

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("KR_ENGINE_LIB") or os.path.join(_HERE, "libkrengine.so")  # KR_ENGINE_LIB: development builds (tools/)
_LIB = None


class EngineError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"kr_engine error {code}: {msg}")
        self.code = code


def build(force: bool = False) -> str:
    """Compile libkrengine.so for sm_90a in-tree (nvcc cross-compiles without a GPU)."""
    src = os.path.join(_HERE, "csrc")
    deps = [os.path.join(src, f) for f in os.listdir(src) if f.endswith((".cu", ".cuh", ".cpp"))] + [os.path.join(_HERE, "..", "include", "kr_engine.h")]
    stale = force or not os.path.exists(LIB_PATH) or any(os.path.getmtime(d) > os.path.getmtime(LIB_PATH) for d in deps)
    if stale:
        subprocess.check_call(["make", "-s", "-C", src, "-B", "NVCCFLAGS=-O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC"])
    return LIB_PATH


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError(f"{LIB_PATH} is missing — run `python -c 'import __graft_entry__ as g; g.build()'`; there is no CPU fallback")
        host_only = os.environ.get("KR_HOST_ONLY_LIB")  # development aid (tools/host_sanitize.sh): an ASan / UBSan build of the host-side builders alone
        if host_only:
            L = C.CDLL(host_only)
            L.kr_spec_json_emit.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
            L.kr_quantity_canonical.argtypes = [C.c_char_p, C.c_char_p, C.c_uint64]
            L.kr_spec_json_emit_arena.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
            L.kr_spec_json_last_error.restype = C.c_char_p
            _LIB = L
            return _LIB
        L = C.CDLL(LIB_PATH)
        P = C.POINTER
        L.kr_device_count.restype = C.c_int
        L.kr_engine_create.argtypes = [P(abi.kr_config), P(C.c_void_p)]
        L.kr_engine_destroy.argtypes = [C.c_void_p]
        L.kr_engine_destroy.restype = None
        L.kr_snapshot_begin.argtypes = [C.c_void_p, P(abi.kr_sizes), P(abi.kr_snapshot_bufs)]
        L.kr_snapshot_commit.argtypes = [C.c_void_p]
        L.kr_snapshot_commit_parts.argtypes = [C.c_void_p, C.c_uint32]
        L.kr_snapshot_commit_pod_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
        L.kr_snapshot_commit_pod_values.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
        L.kr_snapshot_commit_object_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
        L.kr_snapshot_commit_spec_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
        L.kr_snapshot_commit_json_moves.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
        L.kr_engine_set_option.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64]
        L.kr_engine_get_option.argtypes = [C.c_void_p, C.c_uint32, P(C.c_uint64)]
        L.kr_reconcile_batch.argtypes = [C.c_void_p, P(abi.kr_flags), P(abi.kr_results_view)]
        L.kr_reconcile_device_only.argtypes = [C.c_void_p, P(abi.kr_flags)]
        L.kr_reconcile_batch_profiled.argtypes = [C.c_void_p, P(abi.kr_flags), P(abi.kr_profile)]
        L.kr_results_fetch.argtypes = [C.c_void_p, P(abi.kr_results_view)]
        L.kr_hash_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
        L.kr_last_profile.argtypes = [C.c_void_p, P(abi.kr_profile)]
        L.kr_last_pass.argtypes = [C.c_void_p, P(abi.kr_pass_report)]
        L.kr_group_results_device.argtypes = [C.c_void_p, P(C.c_void_p), P(C.c_uint64)]
        L.kr_group_results_copy.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        L.kr_last_error.argtypes = [C.c_void_p]
        L.kr_last_error.restype = C.c_char_p
        L.kr_algorithmic_bytes.argtypes = [C.c_void_p, P(C.c_uint64), P(C.c_uint64), P(C.c_uint64)]
        L.kr_spec_json_emit.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64, P(C.c_uint64)]
        L.kr_spec_json_emit_arena.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, P(C.c_uint64), P(C.c_uint64), P(C.c_uint32)]
        L.kr_quantity_canonical.argtypes = [C.c_char_p, C.c_char_p, C.c_uint64]
        L.kr_spec_json_last_error.restype = C.c_char_p
        L.kr_hash_compare_batch.argtypes = [C.c_void_p, P(abi.kr_hash_compare_row), C.c_uint32, C.c_void_p, C.c_void_p]
        L.kr_group_create.argtypes = [P(abi.kr_config), C.c_void_p, C.c_uint32, P(C.c_void_p)]
        L.kr_group_destroy.argtypes = [C.c_void_p]
        L.kr_group_destroy.restype = None
        L.kr_group_size.argtypes = [C.c_void_p]
        L.kr_group_size.restype = C.c_uint32
        L.kr_group_engine.argtypes = [C.c_void_p, C.c_uint32]
        L.kr_group_engine.restype = C.c_void_p
        L.kr_group_device.argtypes = [C.c_void_p, C.c_uint32]
        L.kr_group_shard_of_uid.argtypes = [C.c_void_p, C.c_uint64]
        L.kr_group_shard_of_uid.restype = C.c_uint32
        L.kr_group_route.argtypes = [C.c_void_p, P(abi.kr_snapshot_bufs), P(abi.kr_sizes), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.kr_group_commit.argtypes = [C.c_void_p, C.c_uint32]
        L.kr_group_reconcile.argtypes = [C.c_void_p, P(abi.kr_flags), C.c_void_p]
        L.kr_group_allgather_group_results.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, P(C.c_uint64), P(C.c_int)]
        L.kr_group_last_error.argtypes = [C.c_void_p]
        L.kr_group_last_error.restype = C.c_char_p
        L.kr_shard_of_key.argtypes = [abi.kr_str, abi.kr_str, C.c_uint32]
        L.kr_shard_of_key.restype = C.c_uint32
        L.kr_group_packer_create.argtypes = [P(abi.kr_config), C.c_void_p, C.c_uint32, P(C.c_void_p)]
        L.kr_group_packer_destroy.argtypes = [C.c_void_p]
        L.kr_group_packer_destroy.restype = None
        L.kr_group_packer_size.argtypes = [C.c_void_p]
        L.kr_group_packer_size.restype = C.c_uint32
        L.kr_group_packer_shard.argtypes = [C.c_void_p, C.c_uint32]
        L.kr_group_packer_shard.restype = C.c_void_p
        L.kr_group_packer_group.argtypes = [C.c_void_p]
        L.kr_group_packer_group.restype = C.c_void_p
        L.kr_group_packer_pod_upsert.argtypes = [C.c_void_p, P(abi.kr_pod_obj)]
        L.kr_group_packer_pod_delete.argtypes = [C.c_void_p, abi.kr_str, abi.kr_str]
        L.kr_group_packer_cluster_upsert.argtypes = [C.c_void_p, P(abi.kr_cluster_obj)]
        L.kr_group_packer_cluster_delete.argtypes = [C.c_void_p, abi.kr_str, abi.kr_str]
        L.kr_group_packer_job_upsert.argtypes = [C.c_void_p, P(abi.kr_job_obj)]
        L.kr_group_packer_job_delete.argtypes = [C.c_void_p, abi.kr_str, abi.kr_str]
        L.kr_group_packer_flush.argtypes = [C.c_void_p, C.c_void_p]
        L.kr_group_packer_reconcile.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.kr_group_packer_last_error.argtypes = [C.c_void_p]
        L.kr_group_packer_last_error.restype = C.c_char_p
        for name in abi.ENGINE_SYMBOLS + abi.ENGINE_HANDLE_SYMBOLS:
            getattr(L, name)  # raises AttributeError if the header and the library drifted apart
        _LIB = L
    return _LIB


def spec_json_emit(spec_json: bytes, muted: bool = True) -> bytes:
    """kr_spec_json_emit: canonical json.Marshal(mute(spec)) bytes of a RayClusterSpec given as JSON text (host code, no GPU)."""
    L = lib()
    need = C.c_uint64()
    cap = 2 * len(spec_json) + 256
    for _ in range(2):
        out = C.create_string_buffer(cap)
        rc = L.kr_spec_json_emit(spec_json, len(spec_json), 0 if muted else abi.SPEC_JSON_UNMUTED, out, cap, C.byref(need))
        if rc == abi.KR_E_CAPACITY:
            cap = need.value
            continue
        if rc != 0:
            raise EngineError(rc, L.kr_spec_json_last_error().decode())
        return out.raw[:need.value]
    raise EngineError(abi.KR_E_CAPACITY, "kr_spec_json_emit: output does not fit")


def quantity_canonical(text: str) -> str:
    L = lib()
    out = C.create_string_buffer(128)
    rc = L.kr_quantity_canonical(text.encode(), out, 128)
    if rc != 0:
        raise EngineError(rc, L.kr_spec_json_last_error().decode())
    return out.value.decode()


def _np_view(ptr: int, dtype, count: int) -> np.ndarray:
    if count == 0 or not ptr:
        return np.zeros(0, dtype=dtype)
    dt = np.dtype(dtype)
    buf = (C.c_uint8 * (dt.itemsize * count)).from_address(ptr)
    return np.frombuffer(buf, dtype=dt, count=count)


class Group:
    """kr_group: one engine per shard behind the multi-GPU coordinator of the C ABI (UID-hash sharding, SURVEY §8(e))."""

    def __init__(self, per_shard: abi.kr_config, devices: list[int]):
        self._L = lib()
        if self._L.kr_device_count() <= 0:
            raise EngineError(abi.KR_E_NO_DEVICE, "no CUDA device visible (this engine has no CPU fallback)")
        self.n = len(devices)
        dv = (C.c_int32 * self.n)(*devices)
        self._h = C.c_void_p()
        rc = self._L.kr_group_create(C.byref(per_shard), dv, self.n, C.byref(self._h))
        if rc != 0:
            raise EngineError(rc, "kr_group_create failed")
        self.engines = []
        for i in range(self.n):  # Engine views over the group's engines (not owned: close() is the group's)
            e = Engine.__new__(Engine)
            e._L, e._h, e.sizes, e.cfg = self._L, C.c_void_p(self._L.kr_group_engine(self._h, i)), None, per_shard
            self.engines.append(e)

    def _check(self, rc: int):
        if rc != 0:
            raise EngineError(rc, self._L.kr_group_last_error(self._h).decode())

    def route(self, snap: Snapshot):
        """kr_group_route: -> (shard sizes, cluster shard, cluster row, pod shard, pod row)."""
        d = snap.dims
        sizes, bufs = snap.sizes(), snap.bufs()
        ss = (abi.kr_sizes * self.n)()
        cs, cr = np.zeros(d["clusters"], np.uint32), np.zeros(d["clusters"], np.uint32)
        ps, pr = np.zeros(d["pods"], np.uint32), np.zeros(d["pods"], np.uint32)
        self._check(self._L.kr_group_route(self._h, C.byref(bufs), C.byref(sizes), ss, cs.ctypes.data, cr.ctypes.data, ps.ctypes.data, pr.ctypes.data))
        for i, e in enumerate(self.engines):
            e.sizes = abi.kr_sizes.from_buffer_copy(ss[i])
        return [abi.kr_sizes.from_buffer_copy(s) for s in ss], cs, cr, ps, pr

    def commit(self, parts: int = abi.PART_ALL):
        self._check(self._L.kr_group_commit(self._h, parts))

    def reconcile(self, flags: abi.kr_flags, copy: bool = True) -> list[abi.Results]:
        views = (abi.kr_results_view * self.n)()
        self._check(self._L.kr_group_reconcile(self._h, C.byref(flags), views))
        return [e._results(views[i], copy) for i, e in enumerate(self.engines)]

    def allgather_group_results(self) -> tuple[np.ndarray, int, bool]:
        """-> (device 0's gathered records [n_shards, slot/32] of group_result_dtype, slot bytes, used NCCL)."""
        slot, used = C.c_uint64(), C.c_int()
        self._check(self._L.kr_group_allgather_group_results(self._h, None, 0, C.byref(slot), C.byref(used)))
        out = np.zeros(max(slot.value * self.n, 32), dtype=np.uint8)
        self._check(self._L.kr_group_allgather_group_results(self._h, out.ctypes.data, out.size, C.byref(slot), C.byref(used)))
        return out[:slot.value * self.n].view(abi.group_result_dtype).reshape(self.n, -1), slot.value, bool(used.value)

    def close(self):
        if self._h:
            for e in self.engines:
                e._h = C.c_void_p()
            self._L.kr_group_destroy(self._h)
            self._h = C.c_void_p()


class Engine:
    """One engine == one GPU.  Mirrors the C ABI call sequence: begin -> (fill) -> commit -> reconcile."""

    def __init__(self, device: int = 0, max_clusters=0, max_groups=0, max_wtd=0, max_pods=0, max_heads=0, max_jobs=0,
                 max_creates=0, max_json_bytes=0):
        self._L = lib()
        n = self._L.kr_device_count()
        if n <= 0:
            raise EngineError(abi.KR_E_NO_DEVICE, "no CUDA device visible (this engine has no CPU fallback)")
        self.cfg = abi.kr_config(device, max_clusters, max_groups, max_wtd, max_pods, max_heads, max_jobs, max_creates, max_json_bytes)
        self._h = C.c_void_p()
        rc = self._L.kr_engine_create(C.byref(self.cfg), C.byref(self._h))
        if rc != 0:
            raise EngineError(rc, "kr_engine_create failed")
        self.sizes = None

    @classmethod
    def for_snapshot(cls, snap: Snapshot, device: int = 0, max_creates: int | None = None, slack: float = 1.0,
                     large_clusters: bool = False, wide_clusters: bool = False, huge_clusters: bool = False,
                     wtd_edits: bool = False, spec_rows: bool = False, cluster_creates: bool = False,
                     cluster_deletes: bool = False, group_edits: bool = False, large_growth: bool = False,
                     large_moves: bool = False, bucket_pod_lists: bool = False, json_moves: bool = False,
                     huge_growth: bool = False) -> "Engine":
        d = snap.dims
        up = lambda x: int(x * slack) + 1  # noqa: E731
        if max_creates is None:
            max_creates = max(1024, d["pods"] // 2)
        eng = cls(device, up(d["clusters"]), up(d["groups"]), up(d["wtd"]), up(d["pods"]), up(d["heads"]), up(d["jobs"]),
                  max_creates, up(d["json"]))
        if large_clusters:
            eng.set_large_clusters(True)
        if wide_clusters:
            eng.set_wide_clusters(True)
        if huge_clusters:
            eng.set_huge_clusters(True)
        if wtd_edits:
            eng.set_wtd_edits(True)
        if spec_rows:
            eng.set_spec_rows(True)
        if cluster_creates:
            eng.set_cluster_creates(True)
        if cluster_deletes:
            eng.set_cluster_deletes(True)
        if group_edits:
            eng.set_group_edits(True)
        if large_growth:
            eng.set_large_growth(True)
        if large_moves:
            eng.set_large_moves(True)
        if bucket_pod_lists:
            eng.set_bucket_pod_lists(True)
        if json_moves:
            eng.set_json_moves(True)
        if huge_growth:
            eng.set_huge_growth(True)
        return eng

    def _check(self, rc: int):
        if rc != 0:
            raise EngineError(rc, self._L.kr_last_error(self._h).decode())

    def close(self):
        if self._h:
            self._L.kr_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- snapshot
    def set_fixed_layout(self, on: bool = True):
        """KR_OPT_FIXED_LAYOUT: lay the arenas out for the capacities once; begin() then only sets the live row counts."""
        self._check(self._L.kr_engine_set_option(self._h, abi.OPT_FIXED_LAYOUT, 1 if on else 0))

    def set_incremental(self, on: bool = True):
        """KR_OPT_INCREMENTAL: allow (default) or forbid device-side incremental passes; off = every pass is a full pass."""
        self._check(self._L.kr_engine_set_option(self._h, abi.OPT_INCREMENTAL, 1 if on else 0))

    def set_large_clusters(self, on: bool = True):
        """KR_OPT_LARGE_CLUSTERS: keep RayClusters of 257..LARGE_MAX_PODS pods on the bucket pipeline (their own regions) instead of
        widening every cluster's bucket or leaving the pipeline; takes effect at the next full pass."""
        self._check(self._L.kr_engine_set_option(self._h, abi.OPT_LARGE_CLUSTERS, 1 if on else 0))

    def set_wide_clusters(self, on: bool = True):
        """KR_OPT_WIDE_CLUSTERS: keep RayClusters of more than 32 worker groups on the bucket pipeline (one CTA decides each) instead
        of sending every pass to the sort pipeline; takes effect at the next full pass."""
        self._check(self._L.kr_engine_set_option(self._h, abi.OPT_WIDE_CLUSTERS, 1 if on else 0))

    def set_huge_clusters(self, on: bool = True):
        """KR_OPT_HUGE_CLUSTERS: with set_large_clusters, keep RayClusters of more than LARGE_MAX_PODS pods on the bucket pipeline
        too (their pods are sorted tile by tile and merged) instead of sending every pass to the sort pipeline; no effect without
        it; takes effect at the next full pass."""
        self._check(self._L.kr_engine_set_option(self._h, abi.OPT_HUGE_CLUSTERS, 1 if on else 0))

    def set_wtd_edits(self, on: bool = True):
        """KR_OPT_WTD_EDITS: keep incremental epochs across scaleStrategy.workersToDelete edits (renames always, list length changes
        under the fixed layout) instead of taking a full pass; read at each object commit."""
        self._check(self._L.kr_engine_set_option(self._h, abi.OPT_WTD_EDITS, 1 if on else 0))

    def set_spec_rows(self, on: bool = True):
        """KR_OPT_SPEC_ROWS: the native packer (and LiveArena) commit re-emitted specs row by row (kr_snapshot_commit_spec_rows)
        instead of re-sending the whole JSON arena; commit_spec_rows itself works either way."""
        self._check(self._L.kr_engine_set_option(self._h, abi.OPT_SPEC_ROWS, 1 if on else 0))

    def set_cluster_creates(self, on: bool = True):
        """KR_OPT_CLUSTER_CREATES: under the fixed layout, keep incremental epochs when RayClusters are appended after the last row or
        RayJobs are created or deleted (commit the object part, then the new RayClusters' specs with commit_spec_rows); read at each
        begin and object commit."""
        self._check(self._L.kr_engine_set_option(self._h, abi.OPT_CLUSTER_CREATES, 1 if on else 0))

    def set_cluster_deletes(self, on: bool = True):
        """KR_OPT_CLUSTER_DELETES: under the fixed layout, keep incremental epochs when RayClusters are deleted by swap-remove (begin
        with the new counts, commit the object part; with cluster_creates the same epoch may create RayClusters in vacated rows); read
        at each begin and object commit."""
        self._check(self._L.kr_engine_set_option(self._h, abi.OPT_CLUSTER_DELETES, 1 if on else 0))

    def set_group_edits(self, on: bool = True):
        """KR_OPT_GROUP_EDITS: under the fixed layout, keep incremental epochs when a RayCluster's worker groups are appended, removed,
        renamed or reordered (begin with the new counts, commit the object part, and a re-emitted spec as a spec row); read at each begin
        and object commit."""
        self._check(self._L.kr_engine_set_option(self._h, abi.OPT_GROUP_EDITS, 1 if on else 0))

    def set_large_growth(self, on: bool = True):
        """KR_OPT_LARGE_GROWTH: with set_large_clusters, a RayCluster that outgrows its bucket or region in an incremental epoch (it
        scaled up) gets a new region in that epoch instead of making the pass a full one; read at each incremental pass."""
        self._check(self._L.kr_engine_set_option(self._h, abi.OPT_LARGE_GROWTH, 1 if on else 0))

    def set_large_moves(self, on: bool = True):
        """KR_OPT_LARGE_MOVES: with set_large_clusters under the fixed layout, set_cluster_deletes and set_group_edits also keep
        incremental epochs when a large RayCluster (one with a region) is deleted, moved by swap-remove or regrouped: a moved or
        regrouped one carries its region; read at each object commit."""
        self._check(self._L.kr_engine_set_option(self._h, abi.OPT_LARGE_MOVES, 1 if on else 0))

    def set_huge_growth(self, on: bool = True):
        """KR_OPT_HUGE_GROWTH: with set_large_clusters, set_huge_clusters and set_large_growth, a RayCluster that grows past
        LARGE_MAX_PODS Pods in an incremental epoch (or a huge one that outgrows its region) gets a region and tiles in that epoch
        instead of making the pass a full one; read at each incremental pass."""
        self._check(self._L.kr_engine_set_option(self._h, abi.OPT_HUGE_GROWTH, 1 if on else 0))

    def set_bucket_pod_lists(self, on: bool = True):
        """KR_OPT_BUCKET_POD_LISTS: fetch_pod_lists only asks for the lists; the pass keeps its pipeline and its incremental epoch, and
        the bucket pipeline builds the same sorted_pod_idx, sorted_action and pod_start as the sort pipeline; read at each pass."""
        self._check(self._L.kr_engine_set_option(self._h, abi.OPT_BUCKET_POD_LISTS, 1 if on else 0))

    def set_json_moves(self, on: bool = True):
        """KR_OPT_JSON_MOVES: with KR_OPT_SPEC_ROWS, the native packer commits a compaction of its JSON arena as moves inside the device
        arena (commit_json_moves) instead of re-sending the arena; commit_json_moves itself works either way."""
        self._check(self._L.kr_engine_set_option(self._h, abi.OPT_JSON_MOVES, 1 if on else 0))

    def get_option(self, option: int) -> int:
        """kr_engine_get_option: an option's current value, or the read-only OPT_BUCKET_STRIDE (0: the sort pipeline) or OPT_SM_COUNT
        (the SM count the SM-sized grids are laid out for: the device's, or a lower KR_SM_COUNT)."""
        v = C.c_uint64()
        self._check(self._L.kr_engine_get_option(self._h, option, C.byref(v)))
        return v.value

    def begin(self, sizes: abi.kr_sizes) -> dict[str, np.ndarray]:
        """kr_snapshot_begin: returns numpy views over the engine-owned pinned arenas, keyed by column name."""
        bufs = abi.kr_snapshot_bufs()
        self._check(self._L.kr_snapshot_begin(self._h, C.byref(sizes), C.byref(bufs)))
        self.sizes = abi.kr_sizes.from_buffer_copy(sizes)
        dims = {"clusters": sizes.n_clusters, "groups": sizes.n_groups, "wtd": sizes.n_wtd, "pods": sizes.n_pods,
                "heads": sizes.n_heads, "jobs": sizes.n_jobs, "json": sizes.json_bytes}
        views = {}
        for name, dt, mult, dim in abi.COLUMNS:
            ptr = C.cast(getattr(bufs, name), C.c_void_p).value
            views[name] = _np_view(ptr, dt, dims[dim] * mult)
        return views

    def fill(self, views: dict[str, np.ndarray], snap: Snapshot):
        """Host-side packing stand-in: copy pre-packed columns into the pinned arenas."""
        for name, *_ in abi.COLUMNS:
            if views[name].size:
                np.copyto(views[name], snap.cols[name])

    def commit(self, parts: int = abi.PART_ALL):
        self._check(self._L.kr_snapshot_commit_parts(self._h, parts))

    def commit_pod_rows(self, rows: np.ndarray):
        """Incremental epoch: upload only the pod rows the caller rewrote in the pinned arenas."""
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        self._check(self._L.kr_snapshot_commit_pod_rows(self._h, rows.ctypes.data, rows.size))

    def commit_pod_values(self, rows: np.ndarray, values: np.ndarray):
        """Incremental epoch, journal style: hand over the new rows themselves (values[i] = the 7 pod columns of rows[i])."""
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        values = np.ascontiguousarray(values, dtype=np.uint32).reshape(-1, 7)
        assert values.shape[0] == rows.size
        self._check(self._L.kr_snapshot_commit_pod_values(self._h, rows.ctypes.data, values.ctypes.data, rows.size))

    def commit_object_rows(self, cluster_rows=(), head_rows=()):
        """kr_snapshot_commit_object_rows: only the rewritten RayCluster (+ their groups') and head-aux rows travel."""
        cr = np.ascontiguousarray(cluster_rows, dtype=np.uint32)
        hr = np.ascontiguousarray(head_rows, dtype=np.uint32)
        self._check(self._L.kr_snapshot_commit_object_rows(self._h, cr.ctypes.data if cr.size else None, cr.size, hr.ctypes.data if hr.size else None, hr.size))

    def commit_spec_rows(self, rows):
        """kr_snapshot_commit_spec_rows: only the rewritten muted-spec JSON ranges (and c_json_off / c_json_len) of these RayClusters
        travel; the next pass re-hashes only them.  Call before the epoch's object commit."""
        r = np.ascontiguousarray(rows, dtype=np.uint32)
        self._check(self._L.kr_snapshot_commit_spec_rows(self._h, r.ctypes.data if r.size else None, r.size))

    def commit_json_moves(self, rows):
        """kr_snapshot_commit_json_moves: these RayClusters' unchanged specs now sit at the ranges c_json_off gives; the device moves
        its copies there (no spec byte crosses PCIe, no digest is recomputed).  Call before the epoch's spec-row and object commits."""
        r = np.ascontiguousarray(rows, dtype=np.uint32)
        self._check(self._L.kr_snapshot_commit_json_moves(self._h, r.ctypes.data if r.size else None, r.size))

    def load(self, snap: Snapshot):
        views = self.begin(snap.sizes())
        self.fill(views, snap)
        self.commit()
        return views

    # -- passes
    def reconcile(self, flags: abi.kr_flags, copy: bool = True) -> abi.Results:
        view = abi.kr_results_view()
        self._check(self._L.kr_reconcile_batch(self._h, C.byref(flags), C.byref(view)))
        return self._results(view, copy)

    def reconcile_device_only(self, flags: abi.kr_flags):
        self._check(self._L.kr_reconcile_device_only(self._h, C.byref(flags)))

    def reconcile_profiled(self, flags: abi.kr_flags) -> dict:
        prof = abi.kr_profile()
        self._check(self._L.kr_reconcile_batch_profiled(self._h, C.byref(flags), C.byref(prof)))
        return self._profile_dict(prof, kernels=True)

    def fetch(self, copy: bool = True) -> abi.Results:
        view = abi.kr_results_view()
        self._check(self._L.kr_results_fetch(self._h, C.byref(view)))
        return self._results(view, copy)

    def last_profile(self) -> dict:
        prof = abi.kr_profile()
        self._check(self._L.kr_last_profile(self._h, C.byref(prof)))
        return self._profile_dict(prof, kernels=False)

    def last_pass(self) -> dict:
        """kr_last_pass: what the last pass that returned KR_OK was — kind ("incremental" / "full"), pipeline ("bucket" / "sort" /
        "radix"), attempts, hash_wait, stride — and why it was not incremental: why_full (the KR_FULL_* bits) and why (their names)."""
        rep = abi.kr_pass_report()
        self._check(self._L.kr_last_pass(self._h, C.byref(rep)))
        return {"kind": {abi.PASSK_INCREMENTAL: "incremental", abi.PASSK_FULL: "full"}.get(rep.kind, rep.kind),
                "pipeline": {abi.PIPE_BUCKET: "bucket", abi.PIPE_SORT: "sort", abi.PIPE_RADIX: "radix"}.get(rep.pipeline, rep.pipeline),
                "attempts": rep.attempts, "hash_wait": bool(rep.hash_wait), "stride": rep.stride,
                "why_full": rep.why_full, "why": abi.full_names(rep.why_full)}

    @staticmethod
    def _profile_dict(prof: abi.kr_profile, kernels: bool) -> dict:
        d = {"h2d_ms": prof.h2d_ms, "kernels_ms": prof.kernels_ms, "d2h_ms": prof.d2h_ms, "n_kernels": prof.n_kernels,
             "h2d_bytes": prof.h2d_bytes, "d2h_bytes": prof.d2h_bytes}
        if kernels:
            k = min(prof.n_kernels, abi.MAX_KERNEL_TIMES)
            d["kernels"] = [((prof.kernel_name[i] or b"?").decode(), prof.kernel_ms[i]) for i in range(k)]
        return d

    def algorithmic_bytes(self) -> dict:
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        self._check(self._L.kr_algorithmic_bytes(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return {"pass": a.value, "hash": b.value, "match": c.value}

    def group_results_device(self) -> tuple[int, int]:
        p, n = C.c_void_p(), C.c_uint64()
        self._check(self._L.kr_group_results_device(self._h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def group_results_copy(self, dst_device_ptr: int, capacity_bytes: int):
        self._check(self._L.kr_group_results_copy(self._h, C.c_void_p(dst_device_ptr), capacity_bytes))

    def hash_batch(self, messages: list[bytes]) -> list[str]:
        n = len(messages)
        if n == 0:
            return []
        offs = np.zeros(n + 1, dtype=np.uint64)
        offs[1:] = np.cumsum([len(m) for m in messages])
        blob = np.frombuffer(b"".join(messages) or b"\0", dtype=np.uint8)
        out = np.zeros(32 * n, dtype=np.uint8)
        self._check(self._L.kr_hash_batch(self._h, blob.ctypes.data, offs.ctypes.data, n, out.ctypes.data))
        return [bytes(out[32 * i:32 * i + 32]).decode("ascii") for i in range(n)]

    def hash_compare_batch(self, rows: list[tuple[bytes, str | None, str | None, bool]]) -> tuple[list[bool], list[str]]:
        """kr_hash_compare_batch — batched isClusterSpecHashEqual (rayservice_controller.go:1130-1157).
        rows: (goal .spec.rayClusterSpec as JSON text, cluster hash annotation, num-worker-groups annotation, partial).
        -> (equal flags, goal hashes ("" where the reference leaves the goal hash empty))."""
        n = len(rows)
        arr = (abi.kr_hash_compare_row * max(n, 1))()
        keep = []
        for i, (spec, chash, nwg, partial) in enumerate(rows):
            cb = chash.encode() if chash is not None else None
            nb = nwg.encode() if nwg is not None else None
            keep += [spec, cb, nb]
            arr[i].goal_spec_json, arr[i].goal_spec_len = spec, len(spec)
            arr[i].cluster_hash, arr[i].cluster_hash_len = cb, len(cb) if cb is not None else 0
            arr[i].num_worker_groups, arr[i].num_worker_groups_len = nb, len(nb) if nb is not None else 0
            arr[i].partial = 1 if partial else 0
        eq = np.zeros(max(n, 1), dtype=np.uint8)
        hs = np.zeros(32 * max(n, 1), dtype=np.uint8)
        self._check(self._L.kr_hash_compare_batch(self._h, arr, n, eq.ctypes.data, hs.ctypes.data))
        return [bool(x) for x in eq[:n]], [bytes(hs[32 * i:32 * i + 32]).rstrip(b"\0").decode("ascii") for i in range(n)]

    def _results(self, view: abi.kr_results_view, copy: bool) -> abi.Results:
        s = self.sizes
        res = abi.Results.__new__(abi.Results)
        res.clusters = _np_view(view.clusters, abi.cluster_result_dtype, s.n_clusters)
        res.hash = _np_view(view.hash, np.uint8, 32 * s.n_clusters).reshape(s.n_clusters, 32)
        res.groups = _np_view(view.groups, abi.group_result_dtype, s.n_groups)
        res.wtd_pod_idx = _np_view(view.wtd_pod_idx, np.int32, s.n_wtd)
        res.sorted_pod_idx = _np_view(view.sorted_pod_idx, np.uint32, s.n_pods if view.sorted_pod_idx else 0)
        res.sorted_action = _np_view(view.sorted_action, np.uint8, s.n_pods if view.sorted_action else 0)
        res.act_start = _np_view(view.act_start, np.uint32, s.n_clusters + 1)
        res.act_cnt = _np_view(view.act_cnt, np.uint32, s.n_clusters)
        res.act_pod_idx = _np_view(view.act_pod_idx, np.uint32, view.act_extent)
        res.act_code = _np_view(view.act_code, np.uint8, view.act_extent)
        res.create_idx = _np_view(view.create_idx, np.int32, view.create_extent)
        res.jobs = _np_view(view.jobs, abi.job_result_dtype, s.n_jobs)
        res.n_create_total, res.n_orphans, res.n_actions = view.n_create_total, view.n_orphans, view.n_actions
        # incremental epochs: the records the pass recomputed (None: a full pass, every record)
        res.n_changed = view.n_changed
        res.changed_clusters = _np_view(view.changed_clusters, np.uint32, view.n_changed).copy() if view.changed_clusters else None
        if copy:
            for name in abi.Results.FIELDS:
                setattr(res, name, getattr(res, name).copy())
        return res

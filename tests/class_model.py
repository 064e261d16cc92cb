"""A host model of the engine's classification of RayClusters on the bucket pipeline (no test_ prefix: pytest does not collect it).
Imports nothing that needs a GPU; tests/test_class_model.py pins its constants and formulas to the sources.

Model restates kr_engine.cu's first_stride, run_pass's ladder through after_bucket_void, upload_lg's list and kr_engine_set_option,
plus what the structural options decide in an incremental epoch:
  * KR_OPT_LARGE_GROWTH (k_inc_admit's grow list and spill, k_inc_grow): a RayCluster whose records outgrow its bucket and region
    gets a region at the cursor in the same epoch, sized by large_region_cap of its peak (its records before the epoch plus the
    Pods that joined it), unless one of the limits in grow() sends the epoch to the full pass;
  * the row maps of KR_OPT_CLUSTER_CREATES / _DELETES / _GROUP_EDITS (commit_map): a gone row (deleted, moved from or regrouped)
    that has a region voids the epoch, as do more than kMapMax rows and adoption by more than kAdoptMax new RayClusters.  Kept rows
    keep their regions; the rows at or past a smaller RayCluster count lose theirs before the pass (run_pass), and a row below the
    count keeps its region for whichever RayCluster takes the row;
  * KR_OPT_WIDE_CLUSTERS: a wide RayCluster is on the per-cluster list by its group count and never forces a full pass."""
import numpy as np

from kuberay_b200 import abi

SMEM_GROUPS = 32  # KR_SMEM_GROUPS (kr_decide.cuh)
GROW_MAX, GROW_LIST_MIN, GROW_LIST_DIV, GROW_SPILL = 64, 64, 64, 16384  # include/kr_engine.h
MAP_MAX = ADOPT_MAX = 4096  # kMapMax, kAdoptMax (kr_engine.cu)


def large_region_cap(count, stride):
    """kr_bucket2.cuh: 1.25 x the count rounded up to 32 records, capped at KR_LARGE_MAX_PODS unless the count is past it, less the
    stride (unsigned: wraps below 0 as the C expression does)."""
    want = (count + count // 4 + 31) // 32 * 32
    return ((want if count > abi.LARGE_MAX_PODS else min(want, abi.LARGE_MAX_PODS)) - stride) & 0xFFFFFFFF


def region_arena(max_pods):
    """Records of the region arena an engine of kr_config.max_pods allocates (kr_engine_set_option)."""
    return max_pods * 5 // 4 + 32 * (max_pods // 257 + 1)


def owners(snap):
    """The RayCluster every pod row belongs to (-1: none), matched on (namespace, ray.io/cluster) as k_match2 does."""
    ckey = (snap.c_ns_id.astype(np.uint64) << np.uint64(32)) | snap.c_name_id.astype(np.uint64)
    order = np.argsort(ckey)
    pkey = (snap.p_ns_id.astype(np.uint64) << np.uint64(32)) | snap.p_cluster_name_id.astype(np.uint64)
    if not order.size:
        return np.full(pkey.size, -1, dtype=np.int64)
    pos = np.minimum(np.searchsorted(ckey[order], pkey), order.size - 1)
    return np.where((ckey[order][pos] == pkey) & (snap.p_cluster_name_id != 0), order[pos], -1)


def counts(snap, own):
    return np.bincount(own[own >= 0], minlength=snap.dims["clusters"])


class Model:
    """The engine's host-side classification and the capacities an incremental epoch is checked against on the device.  caps / offs:
    region capacity and offset by row; cursor: the region arena's first entry past every region in use; valid: the last full pass
    ended on the bucket pipeline."""

    def __init__(self, n_clusters, n_pods, large, wide, huge=False, arena=None):
        self.nc, self.n_pods, self.large, self.wide, self.huge = n_clusters, n_pods, large, wide, huge
        self.arena = arena
        self.reset()

    def first_stride(self):
        st, want = 64, (self.n_pods * 5 // 4 + self.nc - 1) // self.nc
        while st < want and st < 512:
            st <<= 1
        return st if st <= 256 else 0

    def reset(self):
        """An option changed: the next full pass starts from the layout's first stride, without regions."""
        self.stride, self.caps, self.offs, self.cursor, self.valid = self.first_stride(), {}, {}, 0, False

    def limits(self):
        lim = np.full(self.nc, self.stride, dtype=np.int64)
        for c, cap in self.caps.items():
            if c < self.nc:
                lim[c] += cap
        return lim

    def bucket(self, groups):
        return self.stride != 0 and (groups.max(initial=0) <= SMEM_GROUPS or self.wide)

    def full_pass(self, counts, groups):
        """A full pass over `counts`: the ladder of voided bucket attempts.  -> whether it ended on the bucket pipeline."""
        self.shrink(counts.size)
        for _ in range(5):
            if not self.bucket(groups) or not (counts > self.limits()).any():
                break
            self._after_void(counts)
        self.valid = self.bucket(groups)
        return self.valid

    def shrink(self, n):
        """The RayCluster count is n: the regions of rows at or past it go (run_pass, ahead of the pass)."""
        self.nc = n
        for c in [c for c in self.caps if c >= n]:
            del self.caps[c], self.offs[c]

    def _after_void(self, counts):
        if not self.large:
            self.stride = self.stride * 2 if self.stride * 2 <= 256 else 0
            return
        self.caps, self.offs, self.cursor = {}, {}, 0
        if not self.huge and counts.max(initial=0) > abi.LARGE_MAX_PODS:
            self.stride = 0
            return
        big = np.flatnonzero(counts > 256)
        if not big.size:
            self.stride = self.stride * 2 if self.stride * 2 <= 256 else 0
            return
        most, st = int(counts[counts <= 256].max(initial=0)), self.stride
        while st < most and st * 2 <= 256:
            st <<= 1
        if st < most:
            self.stride = 0
            return
        off = 0
        for c in big.tolist():
            self.caps[c], self.offs[c] = large_region_cap(int(counts[c]), st), off
            off += self.caps[c]
        if self.arena is not None and off > self.arena:
            self.caps, self.offs, self.stride = {}, {}, 0
            return
        self.stride, self.cursor = st, off

    def per_cluster_list(self, groups):
        wide = set(np.flatnonzero(groups > SMEM_GROUPS).tolist()) if self.wide else set()
        return set(self.caps) | wide

    def row_map(self, gone, n_rows, n_created, adopt):
        """An object commit's row map (gone: old rows deleted, moved from or regrouped; n_rows: the rows it lists, gone + moved +
        created + regrouped).  -> why the epoch takes the full pass (None: the resident state follows the map)."""
        if any(int(o) in self.caps for o in gone):
            return "large gone row"
        if n_rows > MAP_MAX:
            return "map cap"
        if adopt and n_created > ADOPT_MAX:
            return "adoption cap"
        return None

    def grow(self, peak, groups):
        """An incremental epoch's records against the room of every RayCluster (peak: records before the epoch plus the Pods that
        joined).  -> why the epoch takes the full pass, or None; without a cause the grown RayClusters have their new regions."""
        over = np.flatnonzero(peak > self.limits())
        if not over.size:
            return None
        if len(over) > GROW_MAX:
            return "grow list"
        if int((peak[over] - self.limits()[over]).sum()) > GROW_SPILL:
            return "spill"
        if (peak[over] > abi.LARGE_MAX_PODS).any():
            return "past 8192 pods"
        caps = {int(c): large_region_cap(int(peak[c]), self.stride) for c in over}
        if self.arena is not None and self.cursor + sum(caps.values()) > self.arena:
            return "arena"
        wide = groups > SMEM_GROUPS if self.wide else np.zeros(groups.size, dtype=bool)
        listed = sum(1 for c in caps if c not in self.caps and not wide[c])
        if listed and len(self.per_cluster_list(groups)) + listed > max(GROW_LIST_MIN, self.nc // GROW_LIST_DIV):
            return "list cap"
        for c in sorted(caps):
            self.caps[c], self.offs[c] = caps[c], self.cursor
            self.cursor += caps[c]
        return None

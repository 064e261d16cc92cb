// kr_decide.cuh — the decision kernels: reconcilePods + calculateStatus per RayCluster (one warp each), multi-host groups, status roll-up.
// Part of the sm_90a kernel set of the batched reconcile engine; see kr_kernels.cuh for the pipeline overview.
#pragma once

#include "kr_bucket.cuh"

namespace kr {

// ------------------------------------------------------------------------------------------------ k_decide

#define KR_SMEM_GROUPS 32  // clusters with more worker groups than this spill their accumulators to global scratch
static constexpr int kDecideWarps = 4;

// group processing modes (internal)
enum { GM_UNPROCESSED = 0, GM_SKIP = 1, GM_SUSPENDED = 2, GM_UNHEALTHY = 3, GM_NORMAL = 4, GM_MULTIHOST = 5 };

// first index i in [0,n) with a[i] >= v; warp-cooperative 32-ary search, result uniform across the warp
__device__ __forceinline__ uint32_t warp_lower_bound(const uint32_t *__restrict__ a, uint32_t n, uint32_t v, uint32_t lane) {
  uint32_t lo = 0, hi = n;  // answer in [lo, hi]
  while (hi - lo > 32) {
    uint32_t step = (hi - lo + 31) / 32;  // probe points lo + (l+1)*step - 1
    uint32_t idx = lo + (lane + 1) * step - 1;
    bool ge = (idx >= hi) ? true : (__ldg(&a[idx]) >= v);
    uint32_t b = __ballot_sync(0xFFFFFFFFu, ge);
    if (b == 0) return hi;  // every probe (the last one sits at hi-1 at the earliest) is < v: the answer is hi itself
    uint32_t first = __ffs(b) - 1;
    uint32_t nlo = lo + first * step, nhi = min(hi, lo + (first + 1) * step - 1);
    lo = nlo; hi = nhi;
  }
  uint32_t idx = lo + lane;
  bool ge = (idx >= hi) ? true : (__ldg(&a[idx]) >= v);
  uint32_t b = __ballot_sync(0xFFFFFFFFu, ge);
  return b ? lo + (__ffs(b) - 1) : hi;
}

struct DecideArgs {
  SnapDev s; ScratchDev sc; ResDev r; Sizes n; kr_flags f;
  const uint32_t *sorted_keys;  // radix pipeline: cluster idx per sorted position
  const uint32_t *unsorted;     // fast pipeline: pods bucketed by cluster in arrival order (sorted per bucket here)
  int fast;
  int phase;                    // 0: everything that does not need the hash; 1: only clusters deferred by phase 0
};

// Where status_rollup finds a RayCluster's inputs: straight in the snapshot columns (sort / radix pipelines: scalar code on
// lane 0) ...
struct ColumnsCI {
  const SnapDev &s; uint32_t c;
  __device__ __forceinline__ uint32_t flags() const { return s.c_flags[c]; }
  __device__ __forceinline__ uint8_t ext_err_kind() const { return s.c_ext_err_kind[c]; }
  __device__ __forceinline__ uint32_t ext_err_msg() const { return s.c_ext_err_msg_id[c]; }
  __device__ __forceinline__ uint8_t cond_status(int k) const { return s.c_old_cond_status[5 * (size_t)c + k]; }
  __device__ __forceinline__ uint8_t cond_variant(int k) const { return s.c_old_cond_variant[5 * (size_t)c + k]; }
  __device__ __forceinline__ uint32_t reason() const { return s.c_old_cond_reason_id[c]; }
  __device__ __forceinline__ uint32_t msg(int k) const { return s.c_old_cond_msg_id[2 * (size_t)c + k]; }
  __device__ __forceinline__ uint32_t group_cnt() const { return s.c_group_cnt[c]; }
  __device__ __forceinline__ uint32_t group_off() const { return s.c_group_off[c]; }
  __device__ __forceinline__ uint8_t svc_count() const { return s.c_svc_count[c]; }
  __device__ __forceinline__ uint8_t svc_ip_kind() const { return s.c_svc_ip_kind[c]; }
  __device__ __forceinline__ uint32_t svc_ip() const { return s.c_svc_ip_id[c]; }
  __device__ __forceinline__ uint32_t svc_name() const { return s.c_svc_name_id[c]; }
  __device__ __forceinline__ uint8_t old_state() const { return s.c_old_state[c]; }
  __device__ __forceinline__ uint8_t suspend_status() const { return s.c_suspend_status[c]; }
  __device__ __forceinline__ int32_t old_count(int k) const { return s.c_old_counts[5 * (size_t)c + k]; }
  __device__ __forceinline__ uint32_t old_head(int k) const { return s.c_old_head_ids[4 * (size_t)c + k]; }
  // worker group 0's scalars may come with the cluster's record; here every group is read from the columns
  __device__ __forceinline__ bool has_group0() const { return false; }
  __device__ __forceinline__ uint32_t g0_flags() const { return 0; }
  __device__ __forceinline__ int32_t g0_rep() const { return 0; }
  __device__ __forceinline__ int32_t g0_min() const { return 0; }
  __device__ __forceinline__ int32_t g0_max() const { return 0; }
  __device__ __forceinline__ int32_t g0_hosts() const { return 0; }
};
// ... or in the 128-byte cl_in record the warp loaded with one access (lane i storing word i) into its own shared-memory slot
// (bucket pipeline: every lane runs the roll-up, uniformly, and each field is one broadcast load away — no shuffle, and no
// register holds the record).
struct RecordCI {
  const uint32_t *rec;  // the warp's 32-word slot in shared memory
  __device__ __forceinline__ uint32_t w(int i) const { return rec[i]; }
  __device__ __forceinline__ uint8_t byte(int i, int b) const { return (uint8_t)(w(i) >> (8 * b)); }
  __device__ __forceinline__ uint32_t flags() const { return w(KR_CI_FLAGS); }
  __device__ __forceinline__ uint8_t ext_err_kind() const { return byte(KR_CI_B0, 1); }
  __device__ __forceinline__ uint32_t ext_err_msg() const { return w(KR_CI_EXT_MSG); }
  __device__ __forceinline__ uint8_t cond_status(int k) const { return k < 3 ? byte(KR_CI_B1, 1 + k) : byte(KR_CI_B2, k - 3); }
  __device__ __forceinline__ uint8_t cond_variant(int k) const { return k < 2 ? byte(KR_CI_B2, 2 + k) : byte(KR_CI_B3, k - 2); }
  __device__ __forceinline__ uint32_t reason() const { return w(KR_CI_REASON); }
  __device__ __forceinline__ uint32_t msg(int k) const { return w(KR_CI_MSG + k); }
  __device__ __forceinline__ uint32_t group_cnt() const { return w(KR_CI_GCNT); }
  __device__ __forceinline__ uint32_t group_off() const { return w(KR_CI_GOFF); }
  __device__ __forceinline__ uint8_t svc_count() const { return byte(KR_CI_B0, 3); }
  __device__ __forceinline__ uint8_t svc_ip_kind() const { return byte(KR_CI_B1, 0); }
  __device__ __forceinline__ uint32_t svc_ip() const { return w(KR_CI_SVC_IP); }
  __device__ __forceinline__ uint32_t svc_name() const { return w(KR_CI_SVC_NAME); }
  __device__ __forceinline__ uint8_t old_state() const { return byte(KR_CI_B0, 2); }
  __device__ __forceinline__ uint8_t suspend_status() const { return byte(KR_CI_B0, 0); }
  __device__ __forceinline__ int32_t old_count(int k) const { return (int32_t)w(KR_CI_CNT + k); }
  __device__ __forceinline__ uint32_t old_head(int k) const { return w(KR_CI_HEAD + k); }
  __device__ __forceinline__ bool has_group0() const { return true; }
  __device__ __forceinline__ uint32_t g0_flags() const { return w(KR_CI_G0_FLAGS); }
  __device__ __forceinline__ int32_t g0_rep() const { return (int32_t)w(KR_CI_G0_REP); }
  __device__ __forceinline__ int32_t g0_min() const { return (int32_t)w(KR_CI_G0_MIN); }
  __device__ __forceinline__ int32_t g0_max() const { return (int32_t)w(KR_CI_G0_MAX); }
  __device__ __forceinline__ int32_t g0_hosts() const { return (int32_t)w(KR_CI_G0_HOSTS); }
};

// calculateStatus (raycluster_controller.go:1552-1719) + InconsistentRayClusterStatus (utils/consistency.go:16-34).
// Scalar code: executed by lane 0 only (ColumnsCI) or by every lane uniformly (RecordCI, with cr a volatile reference to the
// warp's shared slot: every lane stores the same value).  aux = head-aux row of the first head pod (-1: none / not in the table).
template <class CI, class CR>
__device__ __forceinline__ void status_rollup(const SnapDev &s, const kr_flags &f, const CI &ci, CR &cr, uint32_t P, uint32_t n_heads,
                                              int32_t head_pod, int32_t aux, uint32_t head_name_id, int32_t ready, int32_t available, bool all_running) {
  const uint32_t cf = ci.flags();
  const bool gate = f.gate_status_conditions != 0;
  const bool reconcile_err = cr.err_kind != KR_ERR_NONE;
  const uint8_t ek = ci.ext_err_kind();
  uint8_t cst[KR_NUM_CONDS], cvr[KR_NUM_CONDS];
#pragma unroll
  for (int k = 0; k < KR_NUM_CONDS; k++) { cst[k] = ci.cond_status(k); cvr[k] = ci.cond_variant(k); }
  uint32_t hpr_reason = ci.reason(), hpr_msg = ci.msg(0), rf_msg = ci.msg(1);
  if (gate) {  // :1563-1577
    if (reconcile_err) {
      if (ek >= KR_EXT_ERR_FAILED_DELETE_ALL_PODS && ek <= KR_EXT_ERR_FAILED_CREATE_WORKER_POD) {
        cst[KR_COND_REPLICA_FAILURE] = KR_COND_TRUE; cvr[KR_COND_REPLICA_FAILURE] = ek; rf_msg = ci.ext_err_msg();
      }
    } else {
      cst[KR_COND_REPLICA_FAILURE] = KR_COND_ABSENT; cvr[KR_COND_REPLICA_FAILURE] = KR_CV_NONE; rf_msg = 0;
    }
  }
  int32_t desired = 0, minr = 0; long long maxr = 0;  // utils/util.go:407-442
  const uint32_t G = ci.group_cnt(), g0 = ci.group_off();
  for (uint32_t gi = 0; gi < G; gi++) {
    const uint32_t g = g0 + gi;
    const bool rec = gi == 0 && ci.has_group0();
    const uint32_t gf = rec ? ci.g0_flags() : s.g_flags[g];
    const int32_t hosts = rec ? ci.g0_hosts() : s.g_num_hosts[g], g_rep = rec ? ci.g0_rep() : s.g_replicas[g];
    const int32_t g_mn = rec ? ci.g0_min() : s.g_min[g], g_mx = rec ? ci.g0_max() : s.g_max[g];
    desired = (int32_t)((uint32_t)desired + (uint32_t)desired_replicas(g_rep, g_mn, g_mx, hosts, gf));
    if (gf & KR_GF_SUSPEND) continue;
    int32_t mn = (gf & KR_GF_MIN_NIL) ? 0 : g_mn;
    int32_t mx = (gf & KR_GF_MAX_NIL) ? INT32_MAX : g_mx;
    minr = (int32_t)((uint32_t)minr + (uint32_t)mn * (uint32_t)hosts);
    maxr += (long long)mx * (long long)hosts;
  }
  int32_t maxc = maxr > INT32_MAX ? INT32_MAX : (maxr < INT32_MIN ? INT32_MIN : (int32_t)maxr);  // utils/util.go:284-292

  cr.n_pods = (int32_t)P; cr.n_heads = (int32_t)n_heads; cr.head_pod_idx = head_pod;
  uint8_t serr = KR_SERR_NONE;  // :1608-1611, :1785-1806, :1721-1745
  const uint8_t svc_count = ci.svc_count(), svc_ip_kind = ci.svc_ip_kind();
  if (n_heads > 1) serr = KR_SERR_MULTIPLE_HEADS;
  else if (svc_count == 0) serr = KR_SERR_NO_HEAD_SERVICE;
  else if (svc_count > 1) serr = KR_SERR_MULTIPLE_HEAD_SERVICES;
  else if (svc_ip_kind == KR_SVCIP_EMPTY) serr = KR_SERR_EMPTY_SERVICE_IP;
  cr.status_err = serr;
  if (serr != KR_SERR_NONE) return;

  const uint8_t old_state = ci.old_state();
  uint8_t new_state = old_state;
  bool reason_cleared = false;
  if (!reconcile_err && (long long)P == (long long)desired + 1 && all_running) { new_state = KR_STATE_READY; reason_cleared = true; }  // :1599-1604

  uint32_t head_pod_ip = 0, head_pod_name = 0;
  if (n_heads != 1) aux = -1;
  if (n_heads == 1) {
    head_pod_ip = aux >= 0 ? s.h_pod_ip_id[aux] : 0;
    head_pod_name = head_name_id;
  }
  if (gate) {
    if (n_heads == 0) {  // :1613-1619
      cst[KR_COND_HEAD_POD_READY] = KR_COND_FALSE; cvr[KR_COND_HEAD_POD_READY] = KR_CV_HEAD_NOT_FOUND;
      hpr_reason = f.id_head_not_found_reason; hpr_msg = f.id_head_not_found_msg;
    } else {             // :1621-1622
      cst[KR_COND_HEAD_POD_READY] = aux >= 0 ? s.h_ready_status[aux] : (uint8_t)KR_COND_FALSE;
      cvr[KR_COND_HEAD_POD_READY] = KR_CV_HEAD_FROM_POD;
      hpr_reason = aux >= 0 ? s.h_ready_reason_id[aux] : 0; hpr_msg = aux >= 0 ? s.h_ready_msg_id[aux] : 0;
    }
    const uint8_t ss = ci.suspend_status();
    if (cst[KR_COND_PROVISIONED] != KR_COND_TRUE && ss != KR_SUSPEND_SUSPENDED) {  // :1625-1644
      if (all_running) { cst[KR_COND_PROVISIONED] = KR_COND_TRUE; cvr[KR_COND_PROVISIONED] = KR_CV_PROV_ALL_READY; }
      else { cst[KR_COND_PROVISIONED] = KR_COND_FALSE; cvr[KR_COND_PROVISIONED] = KR_CV_PROV_PROVISIONING; }
    }
    if (ss == KR_SUSPEND_SUSPENDING) {  // :1646-1693
      if (P == 0) {
        cst[KR_COND_PROVISIONED] = KR_COND_FALSE; cvr[KR_COND_PROVISIONED] = KR_CV_PROV_SUSPENDED;
        cst[KR_COND_SUSPENDING] = KR_COND_FALSE; cvr[KR_COND_SUSPENDING] = KR_CV_CANONICAL;
        cst[KR_COND_SUSPENDED] = KR_COND_TRUE; cvr[KR_COND_SUSPENDED] = KR_CV_CANONICAL;
      }
    } else if (ss == KR_SUSPEND_SUSPENDED) {
      if (cf & KR_CF_SUSPEND_SET_FALSE) { cst[KR_COND_SUSPENDED] = KR_COND_FALSE; cvr[KR_COND_SUSPENDED] = KR_CV_CANONICAL; }
    } else {
      cst[KR_COND_SUSPENDED] = KR_COND_FALSE; cvr[KR_COND_SUSPENDED] = KR_CV_CANONICAL;
      cst[KR_COND_SUSPENDING] = (cf & KR_CF_SUSPEND) ? KR_COND_TRUE : KR_COND_FALSE; cvr[KR_COND_SUSPENDING] = KR_CV_CANONICAL;
    }
  }
  if ((cf & KR_CF_SUSPEND) && P == 0) new_state = KR_STATE_SUSPENDED;  // :1696-1698

  uint32_t svc_ip = ci.svc_ip();
  if (svc_ip_kind == KR_SVCIP_NONE) svc_ip = (n_heads == 1) ? head_pod_ip : 0;  // :1732-1742
  uint32_t head_ids[4] = {head_pod_ip, svc_ip, head_pod_name, ci.svc_name()};

  cr.new_state = new_state;
  cr.state_changed = new_state != old_state;
  cr.status_flags = (reason_cleared ? KR_SF_READY_BRANCH : 0u) | (all_running ? KR_SF_ALL_PODS_RUNNING : 0u);
  cr.counts[0] = ready; cr.counts[1] = available; cr.counts[2] = desired; cr.counts[3] = minr; cr.counts[4] = maxc;
#pragma unroll
  for (int k = 0; k < KR_NUM_CONDS; k++) { cr.cond_status[k] = cst[k]; cr.cond_variant[k] = cvr[k]; }
  cr.head_ready_reason_id = hpr_reason; cr.head_ready_msg_id = hpr_msg;
#pragma unroll
  for (int k = 0; k < 4; k++) cr.head_ids[k] = head_ids[k];

  bool inc = new_state != old_state;  // utils/consistency.go:16-34
  if (reason_cleared && (cf & KR_CF_OLD_REASON_NONEMPTY)) inc = true;
#pragma unroll
  for (int k = 0; k < 5; k++) if (ci.old_count(k) != cr.counts[k]) inc = true;
  if (cf & KR_CF_ENDPOINTS_CHANGED) inc = true;
#pragma unroll
  for (int k = 0; k < 4; k++) if (ci.old_head(k) != head_ids[k]) inc = true;
  // (the old conditions are read from ci again and the new ones from cr: no copy of either is held through the roll-up)
#pragma unroll
  for (int k = 0; k < KR_NUM_CONDS; k++) {
    const uint8_t st = cr.cond_status[k];
    if (ci.cond_status(k) != st) { inc = true; continue; }
    if (st == KR_COND_ABSENT) continue;
    if (k == KR_COND_HEAD_POD_READY) {
      if (ci.reason() != cr.head_ready_reason_id || ci.msg(0) != cr.head_ready_msg_id) inc = true;
    } else if (k == KR_COND_REPLICA_FAILURE) {
      if (ci.cond_variant(k) != cr.cond_variant[k] || ci.msg(1) != rf_msg) inc = true;
    } else if (ci.cond_variant(k) != cr.cond_variant[k]) inc = true;
  }
  cr.needs_status_write = inc ? 1 : 0;
}

// reconcileMultiHostWorkerGroup (raycluster_controller.go:963-1125) for one worker group, by one warp.
// Replicas (pods sharing ray.io/worker-group-replica-name) are identified by the list position of their first pod, so
// "first appearance in list order" — the deterministic stand-in for the reference's Go-map iteration (SURVEY Appendix
// A.5) — is simply ascending position.  Cost O(pods x replicas / 32); every sweep is a coalesced 4-byte column read.
// Returns the KR_ERR_* kind (0 = nil).
#define KR_MH_NONE 0xFFFFFFFFu        // not a member of this group
#define KR_MH_UNASSIGNED 0xFFFFFFFEu  // member with a replica-name label, replica not identified yet
#define KR_MH_NOREP 0xFFFFFFFDu       // member without the label: belongs to no replica
#define KR_MHF_DELETED 1u
#define KR_MHF_WTD 2u
#define KR_MHF_SCALE 4u
__device__ int decide_multihost(const DecideArgs &a, uint32_t slot, uint32_t seg0, uint32_t seg1, int32_t expected, int32_t H,
                                bool delete_allowed, uint32_t wtd_cnt, kr_group_result &gr, int32_t &err_arg, uint32_t lane) {
  uint32_t *rep = a.sc.mh_rep, *name = a.sc.mh_name, *meta = a.sc.mh_meta, *cnt = a.sc.mh_cnt, *flg = a.sc.mh_flg;
  uint8_t *act = a.sc.mh_act, *headv = a.sc.mh_head;
  const uint32_t lt = lanemask_lt();
  // 0. per-position columns of this group (valid only while this group is being decided)
  for (uint32_t b = seg0; b < seg1; b += 32) {
    uint32_t i = b + lane;
    if (i < seg1) {
      uint4 row = a.sc.rows[a.r.sorted_pod_idx[i]];
      bool member = (row.w >> 16) == slot;
      rep[i] = member ? (row.y ? KR_MH_UNASSIGNED : KR_MH_NOREP) : KR_MH_NONE;
      if (member) { name[i] = row.y; meta[i] = row.w & 0xFFFFu; act[i] = KR_ACT_KEEP; headv[i] = 0; }
    }
  }
  __syncwarp();
  // 1. replicaMap (:967-972): peel replicas off in order of first appearance
  uint32_t cursor = seg0, first_incomplete = KR_MH_NONE, m_empty = KR_MH_NONE;
  int32_t incomplete_cnt = 0;
  while (true) {
    uint32_t m = KR_MH_NONE;
    for (uint32_t b = cursor; b < seg1; b += 32) {
      uint32_t i = b + lane;
      uint32_t bal = __ballot_sync(0xFFFFFFFFu, i < seg1 && rep[i] == KR_MH_UNASSIGNED);
      if (bal) { m = b + (__ffs(bal) - 1); break; }
    }
    if (m == KR_MH_NONE) break;
    const uint32_t nm = name[m];
    uint32_t count = 0;
    for (uint32_t b = m; b < seg1; b += 32) {
      uint32_t i = b + lane;
      bool hit = i < seg1 && rep[i] == KR_MH_UNASSIGNED && name[i] == nm;
      if (hit) rep[i] = m;
      count += __popc(__ballot_sync(0xFFFFFFFFu, hit));
    }
    if (lane == 0) { cnt[m] = count; flg[m] = 0; }
    if (nm == KR_ID_EMPTY_STRING) m_empty = m;
    if ((int64_t)count < (int64_t)H && first_incomplete == KR_MH_NONE) { first_incomplete = m; incomplete_cnt = (int32_t)count; }
    cursor = m + 1;
    __syncwarp();
  }
  // 2. incomplete replica groups (:975-984)
  if (first_incomplete != KR_MH_NONE) {
    for (uint32_t b = seg0; b < seg1; b += 32) { uint32_t i = b + lane; if (i < seg1 && rep[i] == first_incomplete) act[i] = KR_ACT_DELETE_MH_INCOMPLETE; }
    gr.flags |= KR_GR_ABORTED; err_arg = incomplete_cnt;
    __syncwarp();
    return KR_ERR_MH_INCOMPLETE;
  }
  // 3. unhealthy replica groups (:987-1007): a pod marks its replica; unlabelled pods resolve to the "" replica if one exists
  for (uint32_t b = seg0; b < seg1; b += 32) {
    uint32_t i = b + lane;
    if (i < seg1 && rep[i] != KR_MH_NONE && should_delete(meta[i])) {
      uint32_t r = rep[i] == KR_MH_NOREP ? m_empty : rep[i];
      if (r != KR_MH_NONE) atomicOr(&flg[r], KR_MHF_DELETED);
    }
  }
  __syncwarp();
  int32_t n_unh = 0;
  for (uint32_t b = seg0; b < seg1; b += 32) {
    uint32_t i = b + lane;
    bool hit = i < seg1 && rep[i] < KR_MH_NOREP && (flg[rep[i]] & KR_MHF_DELETED);
    if (hit) act[i] = KR_ACT_DELETE_MH_UNHEALTHY;
    n_unh += __popc(__ballot_sync(0xFFFFFFFFu, hit));
  }
  gr.n_unhealthy = n_unh;
  // 4. explicit deletions from the autoscaler (:1010-1038)
  if (wtd_cnt > 0) {
    for (uint32_t b = seg0; b < seg1; b += 32) {
      uint32_t i = b + lane;
      if (i < seg1 && rep[i] != KR_MH_NONE && (meta[i] & KR_ROW_WTD_OWN)) {
        uint32_t r = rep[i] == KR_MH_NOREP ? m_empty : rep[i];
        if (r != KR_MH_NONE) atomicOr(&flg[r], KR_MHF_WTD);
      }
    }
    __syncwarp();
    int32_t n_del = 0;
    for (uint32_t b = seg0; b < seg1; b += 32) {
      uint32_t i = b + lane;
      bool hit = i < seg1 && rep[i] < KR_MH_NOREP && (flg[rep[i]] & KR_MHF_WTD);
      if (hit && act[i] == KR_ACT_KEEP) act[i] = KR_ACT_DELETE_MH_WTD;
      n_del += __popc(__ballot_sync(0xFFFFFFFFu, hit));
    }
    gr.flags |= KR_GR_WTD_EXECUTED;
    if (n_del > 0) { gr.flags |= KR_GR_ABORTED; err_arg = n_del; __syncwarp(); return KR_ERR_MH_WTD; }
  }
  // 5. diff by replica (:1042-1064)
  int32_t running = 0;
  for (uint32_t b = seg0; b < seg1; b += 32) {
    uint32_t i = b + lane;
    bool ok = i < seg1 && rep[i] == i && !(flg[i] & KR_MHF_DELETED);  // first pod of a healthy, complete replica
    if (ok) headv[i] = 1;
    running += __popc(__ballot_sync(0xFFFFFFFFu, ok));
  }
  gr.n_running = running;
  if (expected % H != 0) { gr.flags |= KR_GR_ABORTED; err_arg = expected; __syncwarp(); return KR_ERR_MH_NOT_MULTIPLE; }
  const int32_t to_create = expected / H - running;
  gr.diff = to_create;
  if (to_create > 0) gr.n_create = (uint32_t)to_create;  // one replica index per new replica group; k_create_fill allocates them
  else if (to_create < 0) {
    if (delete_allowed) {  // :1104-1118 — the first -to_create valid replicas in first-appearance order
      int32_t seen = 0;
      const int32_t remove = -to_create;
      for (uint32_t b = seg0; b < seg1 && seen < remove; b += 32) {
        uint32_t i = b + lane;
        bool ok = i < seg1 && rep[i] == i && !(flg[i] & KR_MHF_DELETED);
        uint32_t bal = __ballot_sync(0xFFFFFFFFu, ok);
        if (ok && seen + (int32_t)__popc(bal & lt) < remove) flg[i] |= KR_MHF_SCALE;
        seen += __popc(bal);
      }
      __syncwarp();
      for (uint32_t b = seg0; b < seg1; b += 32) {
        uint32_t i = b + lane;
        if (i < seg1 && rep[i] < KR_MH_NOREP && (flg[rep[i]] & KR_MHF_SCALE)) act[i] = KR_ACT_DELETE_MH_SCALE_DOWN;
      }
    } else gr.flags |= KR_GR_RANDOM_DELETE_OFF;
  }
  __syncwarp();
  return KR_ERR_NONE;
}

#define LDG(x) __ldg(&(x))

// Bitonic sort of 32*K values held K per lane, STRIPED (element g = k*32 + lane), ascending.  Striped order is what the
// chunked scans of k_decide want: register k of lane l is list position k*32+l, and loads/stores are fully coalesced.
template <int K>
__device__ __forceinline__ void warp_bitonic_sort_striped(uint32_t (&v)[K], uint32_t lane) {
#pragma unroll
  for (int size = 2; size <= 32 * K; size <<= 1) {
#pragma unroll
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      if (stride < 32) {
        const bool lower = (lane & stride) == 0;
#pragma unroll
        for (int k = 0; k < K; k++) {
          uint32_t o = __shfl_xor_sync(0xFFFFFFFFu, v[k], stride);
          bool asc = ((k * 32 + lane) & size) == 0;
          v[k] = (asc == lower) ? min(v[k], o) : max(v[k], o);
        }
      } else {
        const int ks = stride / 32;
#pragma unroll
        for (int k = 0; k < K; k++) {
          if ((k & ks) == 0) {
            const bool asc = ((k * 32) & size) == 0;  // size >= 64 here: the lane bits do not reach it
            uint32_t lo = min(v[k], v[k + ks]), hi = max(v[k], v[k + ks]);
            v[k] = asc ? lo : hi; v[k + ks] = asc ? hi : lo;
          }
        }
      }
    }
  }
}

// The scalar middle of reconcilePods for one RayCluster, by one warp (uniformly; lane 0 stores), from the scan-1 counters
// (acc_list / acc_unh / acc_wtd per worker group): the path, the head decision and every worker group's record, n_create and mode
// and delete-prefix length (g_mode / g_prefix, or gacc when those are null).  all_action: the action of every pod (delete-all
// paths).  Shared by the warp decide (decide_cluster) and the block decide (decide_cluster_block).  -> false when phase 0 defers
// the cluster to phase 1 (its Recreate gate needs the digest).
template <bool kMH>
__device__ __forceinline__ bool decide_cluster_scalar(const DecideArgs &a, const uint32_t c, const uint32_t seg0, const uint32_t seg1, const uint32_t cf,
                                                      const uint32_t G, const uint32_t g0, const uint8_t suspend_status, const uint8_t ext_err,
                                                      const uint8_t old_prov, const int32_t n_heads, const int32_t head_pod, const int32_t *acc_list,
                                                      const int32_t *acc_unh, const int32_t *acc_wtd, int32_t *g_mode, int32_t *g_prefix,
                                                      kr_cluster_result &cr, uint32_t &head_name, uint8_t &all_action, bool &head_delete,
                                                      bool &run_groups, const uint32_t lane) {
  const SnapDev &s = a.s;
  const bool gate = a.f.gate_status_conditions != 0;
  uint32_t head_flags = 0; head_name = 0;
  if (n_heads > 0) { uint4 hrow = __ldg(&a.sc.rows[head_pod]); head_flags = hrow.w & 0xFFFFu; head_name = hrow.x; }

  {
    uint32_t *z = reinterpret_cast<uint32_t *>(&cr);
#pragma unroll
    for (int k = 0; k < (int)(sizeof(cr) / 4); k++) z[k] = 0;
  }
  cr.head_pod_idx = -1; cr.stop_after_group = -1; cr.pod_start = seg0;
  all_action = KR_ACT_KEEP;
  head_delete = false;
  run_groups = false;

  if (cf & KR_CF_SKIP) {
    cr.path = KR_PATH_SKIPPED;
  } else if (ext_err != KR_EXT_ERR_NONE) {
    cr.path = KR_PATH_SKIPPED;  // :308-314
    cr.err_kind = ext_err == KR_EXT_ERR_STATUS_ONLY_NIL ? KR_ERR_NONE : KR_ERR_EXTERNAL;
  } else if (suspend_status == KR_SUSPEND_SUSPENDING || (!gate && (cf & KR_CF_SUSPEND))) {
    cr.path = KR_PATH_SUSPENDING_DELETE_ALL; all_action = KR_ACT_DELETE_ALL_SUSPEND;  // :629-644
  } else if (gate && (suspend_status == KR_SUSPEND_SUSPENDED || (cf & KR_CF_SUSPEND))) {
    cr.path = KR_PATH_SUSPENDED_NOOP;  // :646-654
  } else {
    bool recreate = false;
    if ((cf & KR_CF_UPGRADE_RECREATE) && n_heads > 0) {  // shouldRecreatePodsForUpgrade :1132-1171
      int32_t aux = aux_lookup(a.sc, (uint32_t)head_pod);
      uint8_t ver = aux >= 0 ? s.h_version_state[aux] : (uint8_t)KR_VER_EMPTY;
      uint8_t ast = aux >= 0 ? s.h_annot_state[aux] : (uint8_t)KR_ANNOT_EMPTY;
      if (ver == KR_VER_DIFFERENT) cr.head_update_annotations = 1;
      else if (ast == KR_ANNOT_OTHER) recreate = true;
      else if (ast == KR_ANNOT_HASH32 && !a.f.skip_hash) {
        if (a.phase == 0) {  // the hash kernel runs concurrently on another stream: decide this cluster in phase 1
          if (lane == 0) a.sc.deferred_list[atomicAdd(&a.r.totals[4], 1u)] = c;
          return false;
        }
        const uint8_t *ah = s.h_annot_hash + 32 * (size_t)aux;
        const char *hh = a.r.hash + 32 * (size_t)c;
        bool ne = ah[lane] != (uint8_t)hh[lane];
        recreate = __any_sync(0xFFFFFFFFu, ne);
      }
    }
    if (recreate) {
      cr.path = KR_PATH_RECREATE_DELETE_ALL; all_action = KR_ACT_DELETE_ALL_RECREATE;  // :657-670
    } else {
      cr.path = KR_PATH_NORMAL;
      // head (:673-748)
      if (!(cf & KR_CF_HEAD_EXPECT_OK)) { cr.head_action = KR_HEAD_EXPECT_PENDING; run_groups = true; }
      else if (n_heads == 1) {
        if (should_delete(head_flags)) { cr.head_action = KR_HEAD_DELETE; cr.err_kind = KR_ERR_HEAD_DELETED; head_delete = true; }
        else run_groups = true;
      } else if (n_heads == 0) {
        if (old_prov == KR_COND_TRUE && (cf & KR_CF_SKIP_HEAD_RESTART)) cr.head_action = KR_HEAD_SKIP_RESTART;
        else { cr.head_action = KR_HEAD_CREATE; run_groups = true; }
      } else {
        cr.head_action = KR_HEAD_MULTIPLE; cr.err_kind = KR_ERR_MULTIPLE_HEADS; cr.err_arg = n_heads;
      }
    }
  }

  // worker groups in spec order (:751-933): O(1) per group from the scan-1 counters
  if (run_groups) {
    const bool autoscaling = (cf & KR_CF_AUTOSCALING) != 0;
    cr.stop_after_group = (int32_t)G;
    for (uint32_t gi = 0; gi < G; gi++) {
      const uint32_t g = g0 + gi, gf = LDG(s.g_flags[g]);
      const int32_t hosts = LDG(s.g_num_hosts[g]), g_rep = LDG(s.g_replicas[g]), g_mn = LDG(s.g_min[g]), g_mx = LDG(s.g_max[g]);
      kr_group_result gr;
      gr.expected = 0; gr.n_list = 0; gr.n_unhealthy = 0; gr.n_running = 0; gr.diff = 0; gr.n_create = 0; gr.create_off = 0;
      gr.flags = KR_GR_PROCESSED;
      int32_t mode = GM_SKIP, prefix = 0;
      bool abort_here = false;
      if (!(gf & KR_GF_EXPECT_OK)) {
        gr.flags |= KR_GR_EXPECT_PENDING;
      } else {
        const int32_t expected = desired_replicas(g_rep, g_mn, g_mx, hosts, gf);
        const int32_t n_list = acc_list[gi], n_unh = acc_unh[gi], n_wtd = acc_wtd[gi];
        gr.expected = expected; gr.n_list = n_list;
        if (gf & KR_GF_SUSPEND) { gr.flags |= KR_GR_SUSPENDED; mode = GM_SUSPENDED; }
        else if (kMH && hosts > 1 && a.f.gate_multihost_indexing) {  // :777-784 (clusters with such groups never reach the <.., false> instantiations)
          gr.flags |= KR_GR_MULTIHOST; mode = GM_MULTIHOST;
          int32_t earg = 0;
          int ek = decide_multihost(a, gi, seg0, seg1, expected, hosts, !autoscaling || a.f.env_random_pod_delete, LDG(s.g_wtd_cnt[g]), gr, earg, lane);
          if (ek != KR_ERR_NONE) { cr.err_kind = (uint8_t)ek; cr.err_arg = earg; abort_here = true; }
        }
        else if (n_unh > 0) {  // :786-812
          gr.n_unhealthy = n_unh; gr.flags |= KR_GR_ABORTED; mode = GM_UNHEALTHY;
          cr.err_kind = KR_ERR_UNHEALTHY_WORKERS; cr.err_arg = n_unh; abort_here = true;
        } else {
          gr.flags |= KR_GR_WTD_EXECUTED; mode = GM_NORMAL;  // :814-849
          const int32_t running = n_list - n_wtd;
          const int32_t diff = expected - running;
          gr.n_running = running; gr.diff = diff;
          if (diff > 0) gr.n_create = (uint32_t)diff;
          else if (diff < 0) {
            if (!autoscaling || a.f.env_random_pod_delete) {  // :898-928
              long long remove = -(long long)diff;
              if (remove > running) {  // expected < 0: the Go loop would index past runningPods (:917)
                prefix = running; gr.flags |= KR_GR_ABORTED;
                cr.err_kind = KR_ERR_NEGATIVE_EXPECTED; cr.err_arg = expected; abort_here = true;
              } else prefix = (int32_t)remove;
            } else gr.flags |= KR_GR_RANDOM_DELETE_OFF;
          }
        }
      }
      __syncwarp();  // every lane has read this group's counters before lane 0 recycles their cells
      if (lane == 0) {
        if (g_mode) { g_mode[gi] = mode; g_prefix[gi] = prefix; }
        else { a.sc.gacc[g] = mode; a.sc.gacc[a.n.n_groups + g] = prefix; }
        a.r.groups[g] = gr;
        a.sc.gcreate[g] = gr.n_create;
      }
      if (abort_here) { cr.stop_after_group = (int32_t)gi; break; }
    }
  }
  // groups never reached keep an all-zero record
  {
    const int32_t reached = ((cf & KR_CF_SKIP) || !run_groups) ? 0 : (cr.stop_after_group == (int32_t)G ? (int32_t)G : cr.stop_after_group + 1);
    for (uint32_t gi = reached + lane; gi < G; gi += 32) {
      kr_group_result z; z.expected = 0; z.n_list = 0; z.n_unhealthy = 0; z.n_running = 0; z.diff = 0; z.n_create = 0; z.create_off = 0; z.flags = 0;
      a.r.groups[g0 + gi] = z;
      a.sc.gcreate[g0 + gi] = 0;
      if (!g_mode) { a.sc.gacc[g0 + gi] = GM_UNPROCESSED; a.sc.gacc[a.n.n_groups + g0 + gi] = 0; }
    }
  }
  __syncwarp();
  return true;
}

// The RayCluster's record (calculateStatus on top of the decisions, except for a skipped cluster) and its action count.  Lane 0.
__device__ __forceinline__ void decide_cluster_record(const DecideArgs &a, const uint32_t c, const uint32_t cf, kr_cluster_result &cr, const uint32_t P,
                                                      const int32_t n_heads, const int32_t head_pod, const uint32_t head_name, const int32_t ready,
                                                      const int32_t available, const bool all_running, const uint32_t n_act) {
  if (!(cf & KR_CF_SKIP))
    status_rollup(a.s, a.f, ColumnsCI{a.s, c}, cr, P, (uint32_t)n_heads, head_pod, n_heads == 1 ? aux_lookup(a.sc, (uint32_t)head_pod) : -1, head_name, ready, available, all_running);
  a.r.clusters[c] = cr;
  a.sc.cact[c] = n_act;
  if (n_act) atomicAdd(&a.r.totals[2], n_act);
}

// reconcilePods (raycluster_controller.go:619-935) + calculateStatus for one RayCluster, by one warp.
// K > 0: the cluster's bucket (<= 32*K pods) is sorted and kept in registers — pod index pidx[k] and row word pw[k] of list
// position k*32+lane — so the two scans below touch no memory.  K == 0: positions are read from sorted_pod_idx / rows
// (radix pipeline, buckets larger than 256 pods, and phase 1).
template <int K, bool kMH>
__device__ __forceinline__ void decide_cluster(const DecideArgs &a, const uint32_t c, const uint32_t seg0, const uint32_t seg1,
                                               uint32_t (&pidx)[K ? K : 1], uint32_t (&pw)[K ? K : 1],
                                               int32_t (&s_acc)[4][KR_SMEM_GROUPS], int32_t (&s_mode)[2][KR_SMEM_GROUPS], const uint32_t lane) {
  const SnapDev &s = a.s;
  const uint32_t lt = lanemask_lt();
  const uint32_t P = seg1 - seg0;
  const uint32_t nchunks = (P + 31) / 32;
  // cluster scalars: independent read-only loads, issued together
  const uint32_t cf = LDG(s.c_flags[c]);
  const uint32_t G = LDG(s.c_group_cnt[c]), g0 = LDG(s.c_group_off[c]);
  const uint8_t suspend_status = LDG(s.c_suspend_status[c]);
  const uint8_t ext_err = LDG(s.c_ext_err_kind[c]);
  const uint8_t old_prov = LDG(s.c_old_cond_status[5 * (size_t)c + KR_COND_PROVISIONED]);

  // accumulators: shared memory for the common case, global scratch for clusters with many groups
  int32_t *acc_list, *acc_unh, *acc_wtd, *acc_rank, *g_mode, *g_prefix;
  if (G <= KR_SMEM_GROUPS) {
    acc_list = s_acc[0]; acc_unh = s_acc[1]; acc_wtd = s_acc[2]; acc_rank = s_acc[3];
    g_mode = s_mode[0]; g_prefix = s_mode[1];
    if (lane < KR_SMEM_GROUPS) { acc_list[lane] = 0; acc_unh[lane] = 0; acc_wtd[lane] = 0; acc_rank[lane] = 0; g_mode[lane] = GM_UNPROCESSED; g_prefix[lane] = 0; }
  } else {
    const uint32_t Ng = a.n.n_groups;
    acc_list = a.sc.gacc + g0; acc_unh = a.sc.gacc + Ng + g0; acc_wtd = a.sc.gacc + 2 * (size_t)Ng + g0; acc_rank = a.sc.gacc + 3 * (size_t)Ng + g0;
    g_mode = nullptr; g_prefix = nullptr;  // modes recycle the n_list / n_unhealthy cells once they are consumed
    for (uint32_t gi = lane; gi < G; gi += 32) { acc_list[gi] = 0; acc_unh[gi] = 0; acc_wtd[gi] = 0; acc_rank[gi] = 0; }
  }
  __syncwarp();

  // ---------------- scan 1: counts over the cluster's pods (list order)
  int32_t ready = 0, available = 0, n_heads = 0;
  bool all_running = P > 0;  // CheckAllPodsRunning (utils/util.go:584-603)
  int32_t head_pod = -1;     // first head in list order
#pragma unroll
  for (int k = 0; k < (K ? K : 1 << 30); k++) {
    if ((uint32_t)k >= nchunks) break;
    const uint32_t i = seg0 + k * 32 + lane;
    const bool valid = i < seg1;
    uint32_t pod, w;
    if (K) { pod = pidx[K ? k : 0]; w = pw[K ? k : 0]; }
    else { pod = valid ? LDG(a.r.sorted_pod_idx[i]) : 0u; w = valid ? reinterpret_cast<const uint32_t *>(a.sc.rows)[4 * (size_t)pod + 3] : 0u; }
    const uint32_t fl = w & 0xFFFFu, slot = valid ? (w >> 16) : KR_ROW_NO_GROUP;
    const uint32_t nt = pp_node_type(fl), ph = pp_phase(fl), rd = pp_ready(fl);
    const bool w_run = valid && nt == KR_NT_WORKER && ph == KR_PHASE_RUNNING;
    available += __popc(__ballot_sync(0xFFFFFFFFu, w_run));
    ready += __popc(__ballot_sync(0xFFFFFFFFu, w_run && rd == KR_COND_TRUE));
    const bool not_ok = valid && (ph != KR_PHASE_RUNNING || rd == KR_COND_FALSE || rd == KR_COND_UNKNOWN);
    if (__any_sync(0xFFFFFFFFu, not_ok)) all_running = false;
    const uint32_t hb = __ballot_sync(0xFFFFFFFFu, valid && nt == KR_NT_HEAD);
    if (hb) { if (n_heads == 0) head_pod = (int32_t)__shfl_sync(0xFFFFFFFFu, pod, __ffs(hb) - 1); n_heads += __popc(hb); }
    // warp-ballot group-by on the group slot
    const uint32_t gkey = (slot < G) ? slot : KR_ROW_NO_GROUP;
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, gkey);
    if (gkey != KR_ROW_NO_GROUP) {
      const uint32_t ub = __ballot_sync(peers, should_delete(fl));
      const uint32_t wb = __ballot_sync(peers, (fl & KR_ROW_WTD_OWN) != 0);
      if ((peers & lt) == 0) {  // leader of its group in this chunk
        acc_list[gkey] += __popc(peers);
        acc_unh[gkey] += __popc(ub & peers);
        acc_wtd[gkey] += __popc(wb & peers);
      }
    }
    __syncwarp();
  }

  // ---------------- scalar decisions (uniform across the warp)
  kr_cluster_result cr;
  uint32_t head_name;
  uint8_t all_action;  // action applied to every pod of the cluster (delete-all paths)
  bool head_delete, run_groups;
  if (!decide_cluster_scalar<kMH>(a, c, seg0, seg1, cf, G, g0, suspend_status, ext_err, old_prov, n_heads, head_pod, acc_list, acc_unh, acc_wtd,
                                  g_mode, g_prefix, cr, head_name, all_action, head_delete, run_groups, lane))
    return;
  const int32_t *mode_arr = g_mode ? g_mode : a.sc.gacc + g0;
  const int32_t *prefix_arr = g_prefix ? g_prefix : a.sc.gacc + a.n.n_groups + g0;

  // ---------------- scan 2: per-pod actions in list order
  uint32_t n_act = 0;
#pragma unroll
  for (int k = 0; k < (K ? K : 1 << 30); k++) {
    if ((uint32_t)k >= nchunks) break;
    const uint32_t i = seg0 + k * 32 + lane;
    const bool valid = i < seg1;
    uint32_t pod, w = 0;
    if (K) { pod = pidx[K ? k : 0]; w = pw[K ? k : 0]; }
    else {
      pod = valid ? LDG(a.r.sorted_pod_idx[i]) : 0u;
      if (valid && run_groups) w = reinterpret_cast<const uint32_t *>(a.sc.rows)[4 * (size_t)pod + 3];
    }
    uint8_t act = KR_ACT_KEEP;
    uint32_t gkey = KR_ROW_NO_GROUP;
    const uint32_t fl = w & 0xFFFFu;
    if (valid && run_groups && (w >> 16) < G) gkey = w >> 16;
    const int32_t mode = (gkey != KR_ROW_NO_GROUP) ? mode_arr[gkey] : GM_UNPROCESSED;
    bool candidate = false;  // running pod of a group in normal mode: subject to the ordered delete prefix
    if (all_action != KR_ACT_KEEP) act = valid ? all_action : (uint8_t)KR_ACT_KEEP;
    else if (head_delete) { if (valid && (int32_t)pod == head_pod) act = KR_ACT_DELETE_HEAD; }
    else if (mode == GM_SUSPENDED) act = KR_ACT_DELETE_GROUP_SUSPEND;
    else if (kMH && mode == GM_MULTIHOST) act = a.sc.mh_act[i];
    else if (mode == GM_UNHEALTHY) { if (should_delete(fl)) act = KR_ACT_DELETE_UNHEALTHY; }
    else if (mode == GM_NORMAL) {
      if (fl & KR_ROW_WTD_OWN) act = KR_ACT_DELETE_WTD;
      else candidate = true;
    }
    // stable rank among the running pods of the same group: ballot group-by + per-group cursor
    const uint32_t ckey = candidate ? gkey : KR_ROW_NO_GROUP;
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, ckey);
    if (candidate) {
      const int32_t cur = acc_rank[ckey];
      __syncwarp(peers);
      const int32_t rank = cur + __popc(peers & lt);
      if ((peers & lt) == 0) acc_rank[ckey] = cur + __popc(peers);
      if (rank < prefix_arr[ckey]) act = KR_ACT_DELETE_RANDOM;  // runningPods.Items[0 .. -diff) (:916-919)
    }
    __syncwarp();
    if (valid) a.r.sorted_action[i] = act;
    // the cluster's action list, compacted while the pods are still in registers (k_creates_fused / k_compact_actions only move it)
    const uint32_t abal = __ballot_sync(0xFFFFFFFFu, valid && act != KR_ACT_KEEP);
    if (valid && act != KR_ACT_KEEP) {
      const size_t o = (size_t)seg0 + n_act + __popc(abal & lt);
      a.sc.act_tmp_idx[o] = pod; a.sc.act_tmp_code[o] = act;
    }
    n_act += __popc(abal);
  }

  // ---------------- status roll-up + record
  if (lane == 0) decide_cluster_record(a, c, cf, cr, P, n_heads, head_pod, head_name, ready, available, all_running, n_act);
}

// Shared memory of decide_cluster_block.
template <int kWarps>
struct BlockDecideSmem {
  int32_t w_cnt[3][kWarps][KR_SMEM_GROUPS];  // per warp and worker group (scan 1): pods, unhealthy pods, workersToDelete-owned pods
  int32_t acc[3][KR_SMEM_GROUPS];            // ... summed over the warps
  int32_t mode[2][KR_SMEM_GROUPS];           // per worker group: mode, delete-prefix length
  int32_t rank[kWarps][KR_SMEM_GROUPS];      // per warp and worker group: running-rank cursor of scan 2
  uint32_t w_red[kWarps][5];                 // per warp (scan 1): ready, available, heads, position of its first head, not all running
  uint32_t w_act[kWarps];                    // per warp (scan 2): pods with an action
  uint32_t plan[2];                          // all_action | head_delete << 8 | run_groups << 9; the first head's pod index
};

// reconcilePods + calculateStatus for one RayCluster of at most KR_SMEM_GROUPS worker groups whose List-ordered pods are
// sorted_pod_idx[seg0, seg1), by all kWarps warps of the CTA (every thread calls it), with the results of decide_cluster<0, true>.
// Warp w owns the positions [seg0 + w * per, seg0 + (w + 1) * per) (per: P / kWarps rounded up to whole chunks of 32), so List
// order inside a warp's range is kept:
//   scan 1  each warp counts its range: ready, available, heads and its first one, all running, and per worker group its pods,
//           unhealthy pods and workersToDelete-owned pods.  A group's pods that are not workersToDelete-owned are exactly its
//           candidates for the ordered delete prefix of normal mode, so their exclusive prefix over the warps is each warp's rank
//           base in scan 2;
//   scalar  warp 0 sums the counters (the first head is the first warp's that has one) and runs decide_cluster_scalar; a
//           multi-host group's decide_multihost sweeps the whole cluster on warp 0 while the other warps wait at the barrier;
//   scan 2  each warp decides its pods (stable rank: its base + the rank inside the warp) and counts its actions; after the block
//           prefix of those counts, a warp with actions compacts them at seg0 + its base, so the run stays in List order.
// sorted_pod_idx and the rows come through the read-only cache (an earlier grid wrote them); what this call writes and reads
// back (mh_act, sorted_action) takes plain loads after a barrier.  Phase 1 only (a.phase: nothing is deferred).
template <int kWarps>
__device__ __forceinline__ void decide_cluster_block(const DecideArgs &a, const uint32_t c, const uint32_t seg0, const uint32_t seg1,
                                                     BlockDecideSmem<kWarps> &sm, const uint32_t warp, const uint32_t lane) {
  static_assert(kWarps <= 32 && KR_SMEM_GROUPS == 32, "one lane per warp and per worker group");
  const SnapDev &s = a.s;
  const uint32_t lt = lanemask_lt();
  const uint32_t P = seg1 - seg0;
  const uint32_t G = LDG(s.c_group_cnt[c]);
  const uint32_t per = ((P + kWarps - 1) / kWarps + 31) & ~31u;
  const uint32_t r0 = seg0 + min(warp * per, P), r1 = seg0 + min(warp * per + per, P);
  int32_t *w_list = sm.w_cnt[0][warp], *w_unh = sm.w_cnt[1][warp], *w_wtd = sm.w_cnt[2][warp];
  w_list[lane] = 0; w_unh[lane] = 0; w_wtd[lane] = 0;
  __syncwarp();

  // ---------------- scan 1: this warp's counts
  int32_t ready = 0, available = 0, n_heads = 0;
  uint32_t first_head = KR_EMPTY32;
  bool not_ok_any = false;
  for (uint32_t b = r0; b < r1; b += 32) {
    const uint32_t i = b + lane;
    const bool valid = i < r1;
    const uint32_t pod = valid ? LDG(a.r.sorted_pod_idx[i]) : 0u;
    const uint32_t w = valid ? reinterpret_cast<const uint32_t *>(a.sc.rows)[4 * (size_t)pod + 3] : 0u;
    const uint32_t fl = w & 0xFFFFu, slot = valid ? (w >> 16) : KR_ROW_NO_GROUP;
    const uint32_t nt = pp_node_type(fl), ph = pp_phase(fl), rd = pp_ready(fl);
    const bool w_run = valid && nt == KR_NT_WORKER && ph == KR_PHASE_RUNNING;
    available += __popc(__ballot_sync(0xFFFFFFFFu, w_run));
    ready += __popc(__ballot_sync(0xFFFFFFFFu, w_run && rd == KR_COND_TRUE));
    const bool not_ok = valid && (ph != KR_PHASE_RUNNING || rd == KR_COND_FALSE || rd == KR_COND_UNKNOWN);
    if (__any_sync(0xFFFFFFFFu, not_ok)) not_ok_any = true;
    const uint32_t hb = __ballot_sync(0xFFFFFFFFu, valid && nt == KR_NT_HEAD);
    if (hb) { if (n_heads == 0) first_head = b + __ffs(hb) - 1; n_heads += __popc(hb); }
    const uint32_t gkey = (slot < G) ? slot : KR_ROW_NO_GROUP;
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, gkey);
    if (gkey != KR_ROW_NO_GROUP) {
      const uint32_t ub = __ballot_sync(peers, should_delete(fl));
      const uint32_t wb = __ballot_sync(peers, (fl & KR_ROW_WTD_OWN) != 0);
      if ((peers & lt) == 0) {  // leader of its group in this chunk
        w_list[gkey] += __popc(peers);
        w_unh[gkey] += __popc(ub & peers);
        w_wtd[gkey] += __popc(wb & peers);
      }
    }
    __syncwarp();
  }
  if (lane == 0) { sm.w_red[warp][0] = ready; sm.w_red[warp][1] = available; sm.w_red[warp][2] = n_heads; sm.w_red[warp][3] = first_head; sm.w_red[warp][4] = not_ok_any; }
  __syncthreads();

  // ---------------- scalar decisions (warp 0), while the other warps find their rank bases
  kr_cluster_result cr;
  uint32_t cf = 0, head_name = 0;
  int32_t head_pod = -1;
  bool all_running = false;
  if (warp == 0) {
    cf = LDG(s.c_flags[c]);
    const uint32_t g0 = LDG(s.c_group_off[c]);
    const uint8_t suspend_status = LDG(s.c_suspend_status[c]);
    const uint8_t ext_err = LDG(s.c_ext_err_kind[c]);
    const uint8_t old_prov = LDG(s.c_old_cond_status[5 * (size_t)c + KR_COND_PROVISIONED]);
    const bool mine = lane < (uint32_t)kWarps;
    ready = (int32_t)__reduce_add_sync(0xFFFFFFFFu, mine ? sm.w_red[lane][0] : 0u);
    available = (int32_t)__reduce_add_sync(0xFFFFFFFFu, mine ? sm.w_red[lane][1] : 0u);
    n_heads = (int32_t)__reduce_add_sync(0xFFFFFFFFu, mine ? sm.w_red[lane][2] : 0u);
    all_running = P > 0 && !__any_sync(0xFFFFFFFFu, mine && sm.w_red[lane][4]);
    const uint32_t hw = __ballot_sync(0xFFFFFFFFu, mine && sm.w_red[lane][2] != 0);
    if (hw) head_pod = (int32_t)LDG(a.r.sorted_pod_idx[sm.w_red[__ffs(hw) - 1][3]]);
    int32_t l = 0, u = 0, t = 0;
    for (int w = 0; w < kWarps; w++) { l += sm.w_cnt[0][w][lane]; u += sm.w_cnt[1][w][lane]; t += sm.w_cnt[2][w][lane]; }
    sm.acc[0][lane] = l; sm.acc[1][lane] = u; sm.acc[2][lane] = t;
    sm.mode[0][lane] = GM_UNPROCESSED; sm.mode[1][lane] = 0;
    sm.rank[0][lane] = 0;
    __syncwarp();
    uint8_t all_action;
    bool head_delete, run_groups;
    decide_cluster_scalar<true>(a, c, seg0, seg1, cf, G, g0, suspend_status, ext_err, old_prov, n_heads, head_pod, sm.acc[0], sm.acc[1], sm.acc[2],
                                sm.mode[0], sm.mode[1], cr, head_name, all_action, head_delete, run_groups, lane);
    if (lane == 0) { sm.plan[0] = all_action | (head_delete ? 0x100u : 0u) | (run_groups ? 0x200u : 0u); sm.plan[1] = (uint32_t)head_pod; }
  } else {
    int32_t base = 0;
    for (uint32_t w = 0; w < warp; w++) base += sm.w_cnt[0][w][lane] - sm.w_cnt[2][w][lane];
    sm.rank[warp][lane] = base;
  }
  __syncthreads();

  // ---------------- scan 2: this warp's per-pod actions
  const uint32_t plan = sm.plan[0];
  const uint8_t all_action = (uint8_t)(plan & 0xFFu);
  const bool head_delete = (plan & 0x100u) != 0, run_groups = (plan & 0x200u) != 0;
  const int32_t head = (int32_t)sm.plan[1];
  int32_t *acc_rank = sm.rank[warp];
  const int32_t *mode_arr = sm.mode[0], *prefix_arr = sm.mode[1];
  uint32_t n_act = 0;
  for (uint32_t b = r0; b < r1; b += 32) {
    const uint32_t i = b + lane;
    const bool valid = i < r1;
    const uint32_t pod = valid ? LDG(a.r.sorted_pod_idx[i]) : 0u;
    uint32_t w = 0;
    if (valid && run_groups) w = reinterpret_cast<const uint32_t *>(a.sc.rows)[4 * (size_t)pod + 3];
    uint8_t act = KR_ACT_KEEP;
    uint32_t gkey = KR_ROW_NO_GROUP;
    const uint32_t fl = w & 0xFFFFu;
    if (valid && run_groups && (w >> 16) < G) gkey = w >> 16;
    const int32_t mode = (gkey != KR_ROW_NO_GROUP) ? mode_arr[gkey] : GM_UNPROCESSED;
    bool candidate = false;
    if (all_action != KR_ACT_KEEP) act = valid ? all_action : (uint8_t)KR_ACT_KEEP;
    else if (head_delete) { if (valid && (int32_t)pod == head) act = KR_ACT_DELETE_HEAD; }
    else if (mode == GM_SUSPENDED) act = KR_ACT_DELETE_GROUP_SUSPEND;
    else if (mode == GM_MULTIHOST) act = a.sc.mh_act[i];
    else if (mode == GM_UNHEALTHY) { if (should_delete(fl)) act = KR_ACT_DELETE_UNHEALTHY; }
    else if (mode == GM_NORMAL) {
      if (fl & KR_ROW_WTD_OWN) act = KR_ACT_DELETE_WTD;
      else candidate = true;
    }
    const uint32_t ckey = candidate ? gkey : KR_ROW_NO_GROUP;
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, ckey);
    if (candidate) {
      const int32_t cur = acc_rank[ckey];
      __syncwarp(peers);
      const int32_t rank = cur + __popc(peers & lt);
      if ((peers & lt) == 0) acc_rank[ckey] = cur + __popc(peers);
      if (rank < prefix_arr[ckey]) act = KR_ACT_DELETE_RANDOM;  // runningPods.Items[0 .. -diff) (:916-919)
    }
    __syncwarp();
    if (valid) a.r.sorted_action[i] = act;
    n_act += __popc(__ballot_sync(0xFFFFFFFFu, valid && act != KR_ACT_KEEP));
  }
  if (lane == 0) sm.w_act[warp] = n_act;
  __syncthreads();

  // ---------------- the cluster's action list, in List order
  const uint32_t v = lane < (uint32_t)kWarps ? sm.w_act[lane] : 0u;
  const uint32_t before = __reduce_add_sync(0xFFFFFFFFu, lane < warp ? v : 0u);
  if (n_act) {
    uint32_t o = seg0 + before;
    for (uint32_t b = r0; b < r1; b += 32) {
      const uint32_t i = b + lane;
      const uint8_t act = i < r1 ? a.r.sorted_action[i] : (uint8_t)KR_ACT_KEEP;
      const uint32_t abal = __ballot_sync(0xFFFFFFFFu, act != KR_ACT_KEEP);
      if (act != KR_ACT_KEEP) {
        const size_t p = (size_t)o + __popc(abal & lt);
        a.sc.act_tmp_idx[p] = LDG(a.r.sorted_pod_idx[i]); a.sc.act_tmp_code[p] = act;
      }
      o += __popc(abal);
    }
  }
  if (warp == 0) {
    const uint32_t total = __reduce_add_sync(0xFFFFFFFFu, v);
    if (lane == 0) decide_cluster_record(a, c, cf, cr, P, n_heads, head_pod, head_name, ready, available, all_running, total);
  }
}

// Sort a bucket of <= 32*K pod indices in registers, publish it (sorted_pod_idx), gather the row words, decide.
template <int K>
__device__ __forceinline__ void decide_cluster_regs(const DecideArgs &a, uint32_t c, uint32_t seg0, uint32_t seg1,
                                                    int32_t (&s_acc)[4][KR_SMEM_GROUPS], int32_t (&s_mode)[2][KR_SMEM_GROUPS], uint32_t lane) {
  uint32_t pidx[K], pw[K];
  const uint32_t P = seg1 - seg0;
  if (a.phase == 0) {
#pragma unroll
    for (int k = 0; k < K; k++) { uint32_t g = k * 32 + lane; pidx[k] = g < P ? LDG(a.unsorted[seg0 + g]) : 0xFFFFFFFFu; }
    warp_bitonic_sort_striped<K>(pidx, lane);
  } else {  // phase 1: phase 0 sorted and published this bucket before it deferred the cluster
#pragma unroll
    for (int k = 0; k < K; k++) { uint32_t g = k * 32 + lane; pidx[k] = g < P ? a.r.sorted_pod_idx[seg0 + g] : 0xFFFFFFFFu; }
  }
#pragma unroll
  for (int k = 0; k < K; k++) {
    uint32_t g = k * 32 + lane;
    pw[k] = 0;
    if (g < P) { if (a.phase == 0) a.r.sorted_pod_idx[seg0 + g] = pidx[k]; pw[k] = reinterpret_cast<const uint32_t *>(a.sc.rows)[4 * (size_t)pidx[k] + 3]; }
    else pidx[k] = 0;
  }
  __syncwarp();  // sorted_pod_idx of this bucket is visible to the whole warp (decide_multihost re-reads it)
  decide_cluster<K, false>(a, c, seg0, seg1, pidx, pw, s_acc, s_mode, lane);
}

// Is this cluster decided by k_decide_small (bucket sorted and kept in registers)?  Fast pipeline, at most 256 pods, no
// multi-host worker group (those need the memory-resident sweeps of decide_multihost).  Both phases: the clusters phase 0
// deferred (Recreate gate waiting for the hash) keep their shape, so phase 1 splits them between the same two kernels.
__device__ __forceinline__ bool small_path(const DecideArgs &a, uint32_t c, uint32_t P) {
  return a.fast && P <= 256 && !(a.f.gate_multihost_indexing && (__ldg(&a.sc.cl_rec[c]).w & 1u));
}

// Common case: one warp per RayCluster with <= 256 pods, everything after the bucket load stays in registers.
__global__ void __launch_bounds__(kDecideWarps * 32, 8) k_decide_small(DecideArgs a) {
  KR_TL(a.phase ? 12 : 3);
  __shared__ int32_t s_acc[kDecideWarps][4][KR_SMEM_GROUPS];  // n_list, n_unhealthy, n_wtd_own, running-rank cursor
  __shared__ int32_t s_mode[kDecideWarps][2][KR_SMEM_GROUPS]; // mode, delete-prefix length
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t c = blockIdx.x * kDecideWarps + warp;
  pdl_wait(); pdl_trigger();
  if (a.phase == 1) {  // compact list of the clusters phase 0 deferred
    if (c >= a.r.totals[4]) return;
    c = a.sc.deferred_list[c];
  } else if (c >= a.n.n_clusters) return;
  const uint32_t attempt = KR_ATTEMPT_WORD(a.r.totals);
  const uint32_t seg0 = LDG(a.sc.cstart[c]), seg1 = LDG(a.sc.cstart[c + 1]);
  if (KR_WORD_VOID(attempt)) return;
  const uint32_t P = seg1 - seg0;
  if (!small_path(a, c, P)) return;
  if (P <= 128) decide_cluster_regs<4>(a, c, seg0, seg1, s_acc[warp], s_mode[warp], lane);
  else decide_cluster_regs<8>(a, c, seg0, seg1, s_acc[warp], s_mode[warp], lane);
}

// General case: radix pipeline (all clusters), big buckets, clusters with multi-host groups, phase 1, the orphan bucket.
__global__ void __launch_bounds__(kDecideWarps * 32) k_decide(DecideArgs a) {
  KR_TL(4 + a.phase);
  __shared__ int32_t s_acc[kDecideWarps][4][KR_SMEM_GROUPS];
  __shared__ int32_t s_mode[kDecideWarps][2][KR_SMEM_GROUPS];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t Nc = a.n.n_clusters, Np = a.n.n_pods;
  if (a.fast && KR_ATTEMPT_VOID(a.r.totals)) return;
  uint32_t c = blockIdx.x * kDecideWarps + warp;
  if (a.phase == 0) {
    // The orphans' segment: pods whose (namespace, ray.io/cluster) names no RayCluster in the snapshot, and the free rows of an
    // incrementally maintained arena (KR_PP_TOMBSTONE; there can be many).  Every warp of the grid labels a strided share — the
    // warps past the last cluster of the rounded-up grid as well, so this comes before their early return.
    const uint32_t o0 = a.fast ? LDG(a.sc.cstart[Nc]) : warp_lower_bound(a.sorted_keys, Np, Nc, lane);
    const uint32_t gw = blockIdx.x * kDecideWarps + warp, nw = gridDim.x * kDecideWarps;
    uint32_t real = 0;
    for (uint32_t i = o0 + gw * 32 + lane; i < Np; i += nw * 32) {
      const uint32_t pod = a.fast ? LDG(a.unsorted[i]) : a.r.sorted_pod_idx[i];  // k_match/k_place put this segment in List order already
      if (a.fast) a.r.sorted_pod_idx[i] = pod;
      const bool tomb = reinterpret_cast<const uint32_t *>(a.sc.rows)[4 * (size_t)pod + 3] & KR_PP_TOMBSTONE;
      a.r.sorted_action[i] = tomb ? KR_ACT_TOMBSTONE : KR_ACT_ORPHAN;
      real += tomb ? 0u : 1u;
    }
    real = __reduce_add_sync(0xFFFFFFFFu, real);
    if (lane == 0 && real) atomicAdd(&a.r.totals[1], real);
  }
  if (a.phase == 1) {  // compact list of the clusters phase 0 deferred
    if (c >= a.r.totals[4]) return;
    c = a.sc.deferred_list[c];
  } else if (c > Nc) return;

  uint32_t seg0, seg1;
  if (a.fast) { seg0 = LDG(a.sc.cstart[c]); seg1 = LDG(a.sc.cstart[c + 1]); }
  else {
    seg0 = warp_lower_bound(a.sorted_keys, Np, c, lane);
    seg1 = (c == Nc) ? Np : warp_lower_bound(a.sorted_keys, Np, c + 1, lane);
  }
  const uint32_t P = seg1 - seg0;
  if (c == Nc) return;
  if (small_path(a, c, P)) return;  // k_decide_small owns it
  // fast pipeline, phase 0: informer List order inside the bucket = ascending pod index (phase 1 finds it already sorted)
  if (a.fast && a.phase == 0 && P <= KR_FAST_MAX_BUCKET) { warp_sort_dispatch(a.unsorted + seg0, a.r.sorted_pod_idx + seg0, P, lane); __syncwarp(); }
  uint32_t d0[1] = {0}, d1[1] = {0};
  decide_cluster<0, true>(a, c, seg0, seg1, d0, d1, s_acc[warp], s_mode[warp], lane);
}

}  // namespace kr

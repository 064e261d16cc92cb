/*
 * kr_engine.h — C ABI of the batched RayCluster reconcile engine (H100 / sm_90a).
 *
 * This is the drop-in boundary a cgo shim binds (see INTEGRATION.md).  Plain C,
 * plain pointers and sizes, no callbacks, no C++ exceptions across the boundary.
 * Every entry point cites the reference interface (ray-project/kuberay, paths
 * relative to the reference root) whose *decision half* it replaces; the Go
 * side keeps performing the side effects (Create/Delete/Eventf/ExpectScalePod/
 * Status().Update) in the recorded order.
 *
 * Data model: one *snapshot* = every watched RayCluster, its worker groups and
 * every cached Pod, packed as little-endian SoA columns.  Strings are interned
 * to u32 ids host-side (id 0 = absent; the empty string is a normal id).
 * Pod order in the snapshot IS the informer List order and is honoured
 * (reference deletes "the first -diff items in List order",
 * ray-operator/controllers/ray/raycluster_controller.go:916-918).
 */
#ifndef KR_ENGINE_H_
#define KR_ENGINE_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Interner convention: id 0 = "absent" (label/annotation/field not present), id 1 = the empty string "".
 * In HeadInfo-like fields (pod IP, names, service IP) the empty string MUST be encoded as 0.
 * Id domain: every other id is an opaque u32 in [2, 0xFFFFFFFE]; the engine compares ids only for equality, so any assignment of
 * distinct values gives the same decisions.  0xFFFFFFFF is not an id: the engine's join tables and the oracle's map mark an empty
 * slot with the all-ones key, so a (namespace, name) pair of two 0xFFFFFFFF ids would read as an empty slot.  The packers never
 * produce it. */
#define KR_ID_ABSENT 0u
#define KR_ID_EMPTY_STRING 1u

/* ------------------------------------------------------------------ enums */

/* clusters.flags bits */
enum {
  KR_CF_SUSPEND            = 1u << 0,  /* spec.suspend != nil && *spec.suspend            (raycluster_controller.go:632,651,1680,1696) */
  KR_CF_SUSPEND_SET_FALSE  = 1u << 1,  /* spec.suspend != nil && !*spec.suspend           (:1667) */
  KR_CF_AUTOSCALING        = 1u << 2,  /* utils.IsAutoscalingEnabled(&spec)                (:898) */
  KR_CF_UPGRADE_RECREATE   = 1u << 3,  /* spec.upgradeStrategy.type == Recreate            (:1134) */
  KR_CF_SKIP_HEAD_RESTART  = 1u << 4,  /* annotation ray.io/disable-provisioned-head-restart == "true" (:1127) */
  KR_CF_HEAD_EXPECT_OK     = 1u << 5,  /* rayClusterScaleExpectation.IsSatisfied(ns,name,HeadGroup) (:689) — evaluated in Go */
  KR_CF_SKIP               = 1u << 6,  /* deletionTimestamp set / managed by external controller / validation failed: no decisions, no status (:152-185,290) */
  KR_CF_ENDPOINTS_CHANGED  = 1u << 7,  /* host evaluated updateEndpoints (:1747-1783) and the map differs from old status */
  KR_CF_OLD_REASON_NONEMPTY= 1u << 8   /* old status.reason != ""                           (consistency.go:17) */
};

/* clusters.suspend_status: utils.FindRayClusterSuspendStatus (utils/util.go:153-162), evaluated host-side */
enum { KR_SUSPEND_NONE = 0, KR_SUSPEND_SUSPENDING = 1, KR_SUSPEND_SUSPENDED = 2 };

/* clusters.ext_err_kind: error returned by a sub-reconciler that ran BEFORE reconcilePods
 * (raycluster_controller.go:296-314) or, in status-only re-evaluation after an API failure,
 * one of the ErrFailed* markers (utils/constant.go:322-334).  != 0 => decisions are skipped. */
enum {
  KR_EXT_ERR_NONE = 0,
  KR_EXT_ERR_PLAIN = 1,
  KR_EXT_ERR_FAILED_DELETE_ALL_PODS = 2,
  KR_EXT_ERR_FAILED_DELETE_HEAD_POD = 3,
  KR_EXT_ERR_FAILED_CREATE_HEAD_POD = 4,
  KR_EXT_ERR_FAILED_DELETE_WORKER_POD = 5,
  KR_EXT_ERR_FAILED_CREATE_WORKER_POD = 6,
  KR_EXT_ERR_STATUS_ONLY_NIL = 7   /* status-only evaluation with reconcileErr == nil: decisions skipped (replays calculateStatus(ctx, instance, nil)) */
};

/* condition status codes (metav1.ConditionStatus) */
enum { KR_COND_ABSENT = 0, KR_COND_TRUE = 1, KR_COND_FALSE = 2, KR_COND_UNKNOWN = 3 };

/* condition slots (apis/ray/v1/raycluster_types.go:362-374) */
enum {
  KR_COND_PROVISIONED = 0,
  KR_COND_HEAD_POD_READY = 1,
  KR_COND_REPLICA_FAILURE = 2,
  KR_COND_SUSPENDING = 3,
  KR_COND_SUSPENDED = 4,
  KR_NUM_CONDS = 5
};

/* condition (reason,message) variants the controller itself writes; anything else is KR_CV_OTHER */
enum {
  KR_CV_NONE = 0,
  KR_CV_PROV_ALL_READY = 1,        /* AllPodRunningAndReadyFirstTime / "All Ray Pods are ready for the first time" (:1630-1635) */
  KR_CV_PROV_PROVISIONING = 2,     /* RayClusterPodsProvisioning / "RayCluster Pods are being provisioned for first time" (:1637-1642) */
  KR_CV_PROV_SUSPENDED = 3,        /* RayClusterPodsProvisioning / "RayCluster has been suspended" (:1649-1654) */
  KR_CV_CANONICAL = 4,             /* Suspending/Suspended: reason == type, empty message (:1655-1691) */
  KR_CV_HEAD_FROM_POD = 5,         /* HeadPodReady copied from the head pod (reason/message ids in the record) (:1621-1622) */
  KR_CV_HEAD_NOT_FOUND = 6,        /* HeadPodNotFound / "Head Pod not found" (:1613-1619) */
  /* ReplicaFailure slot: variant = the KR_EXT_ERR_FAILED_* kind (2..6) that names the reason (:1564-1571) */
  KR_CV_OTHER = 255
};

/* cluster state (apis/ray/v1/raycluster_types.go:268-274) */
enum { KR_STATE_EMPTY = 0, KR_STATE_READY = 1, KR_STATE_FAILED = 2, KR_STATE_SUSPENDED = 3, KR_STATE_OTHER = 4 };

/* groups.flags bits */
enum {
  KR_GF_SUSPEND       = 1u << 0,   /* worker.Suspend != nil && *worker.Suspend (:766; utils/util.go:391) */
  KR_GF_EXPECT_OK     = 1u << 1,   /* IsSatisfied(ns, cluster, groupName) (:752) — evaluated in Go */
  KR_GF_REPLICAS_NIL  = 1u << 2,
  KR_GF_MIN_NIL       = 1u << 3,
  KR_GF_MAX_NIL       = 1u << 4
};

/* pods.packed bit fields */
#define KR_PP_NODE_TYPE_SHIFT 0   /* 2 bits: 0 none/other, 1 head, 2 worker, 3 redis-cleanup (label ray.io/node-type) */
#define KR_PP_PHASE_SHIFT     2   /* 3 bits: 0 "", 1 Pending, 2 Running, 3 Succeeded, 4 Failed, 5 Unknown */
#define KR_PP_READY_SHIFT     5   /* 2 bits: PodReady condition: 0 absent, 1 True, 2 False, 3 Unknown */
#define KR_PP_RESTART_NEVER   (1u << 7)   /* spec.restartPolicy == Never */
#define KR_PP_RAY_TERMINATED  (1u << 8)   /* getRayContainerStateTerminated(pod) != nil (:1237-1248) */
#define KR_PP_HAS_DELETION_TS (1u << 9)
#define KR_PP_HAS_REPLICA_IDX (1u << 10)  /* label ray.io/worker-group-replica-index present AND strconv.Atoi succeeded (:857-860) */
#define KR_PP_TOMBSTONE       (1u << 12)  /* free row of an incrementally maintained arena (a Pod that left the informer cache, or spare
                                             capacity): the shim writes ns_id = cluster_name_id = 0 with this bit; the row matches no
                                             RayCluster, is reported as KR_ACT_TOMBSTONE after the orphans' segment and is not counted */
enum { KR_NT_NONE = 0, KR_NT_HEAD = 1, KR_NT_WORKER = 2, KR_NT_REDIS = 3 };
enum { KR_PHASE_EMPTY = 0, KR_PHASE_PENDING = 1, KR_PHASE_RUNNING = 2, KR_PHASE_SUCCEEDED = 3, KR_PHASE_FAILED = 4, KR_PHASE_UNKNOWN = 5 };

/* per-pod action codes (results) */
enum {
  KR_ACT_KEEP = 0,
  KR_ACT_DELETE_ALL_SUSPEND = 1,     /* deleteAllPods on suspension (:633) */
  KR_ACT_DELETE_ALL_RECREATE = 2,    /* deleteAllPods on Recreate upgrade (:659) */
  KR_ACT_DELETE_HEAD = 3,            /* unhealthy head (:701) */
  KR_ACT_DELETE_GROUP_SUSPEND = 4,   /* suspended worker group (:767) */
  KR_ACT_DELETE_UNHEALTHY = 5,       /* shouldDeletePod worker (:796) */
  KR_ACT_DELETE_WTD = 6,             /* named in scaleStrategy.workersToDelete and listed in its group (:822) */
  KR_ACT_DELETE_RANDOM = 7,          /* list-prefix "random" delete (:917-919) */
  KR_ACT_DELETE_MH_INCOMPLETE = 8,   /* multi-host: incomplete replica cleanup (:978) */
  KR_ACT_DELETE_MH_UNHEALTHY = 9,    /* multi-host: unhealthy replica (:999) */
  KR_ACT_DELETE_MH_WTD = 10,         /* multi-host: autoscaler scale-down request (:1030) */
  KR_ACT_DELETE_MH_SCALE_DOWN = 11,  /* multi-host: scaling down (:1114) */
  KR_ACT_TOMBSTONE = 254,            /* free row (KR_PP_TOMBSTONE) — listed among the orphans, not counted in n_orphans */
  KR_ACT_ORPHAN = 255                /* pod matched no RayCluster in the snapshot */
};

/* cluster_results.path */
enum {
  KR_PATH_NORMAL = 0,
  KR_PATH_SKIPPED = 1,               /* KR_CF_SKIP or ext_err_kind != 0 */
  KR_PATH_SUSPENDING_DELETE_ALL = 2, /* :631-644 */
  KR_PATH_SUSPENDED_NOOP = 3,        /* :646-654 */
  KR_PATH_RECREATE_DELETE_ALL = 4    /* :657-670 */
};

/* cluster_results.head_action */
enum {
  KR_HEAD_NONE = 0,
  KR_HEAD_EXPECT_PENDING = 1,        /* :689-690 */
  KR_HEAD_DELETE = 2,                /* :700-711, reconcile aborts with error */
  KR_HEAD_CREATE = 3,                /* :735 */
  KR_HEAD_SKIP_RESTART = 4,          /* :714-732, reconcile returns nil early */
  KR_HEAD_MULTIPLE = 5               /* :738-747, error */
};

/* cluster_results.err_kind: which plain error reconcilePods returned (never an ErrFailed* marker:
 * those arise only from API-call failures, SURVEY Appendix A.3) */
enum {
  KR_ERR_NONE = 0,
  KR_ERR_HEAD_DELETED = 1,           /* errstd.New(reason) :711 */
  KR_ERR_MULTIPLE_HEADS = 2,         /* :747; err_arg = count */
  KR_ERR_UNHEALTHY_WORKERS = 3,      /* "delete %d unhealthy worker Pods" :811; err_arg = count */
  KR_ERR_MH_INCOMPLETE = 4,          /* :982 */
  KR_ERR_MH_WTD = 5,                 /* :1034; err_arg = pods deleted */
  KR_ERR_MH_NOT_MULTIPLE = 6,        /* :1060 */
  KR_ERR_EXTERNAL = 7,               /* ext_err_kind != 0 */
  KR_ERR_NEGATIVE_EXPECTED = 8       /* expected < 0 with delete allowed: the Go code would index out of range (:917); engine refuses */
};

/* cluster_results.status_err: calculateStatus returned an error => no status write (:1608-1611,1704-1706,1721-1745) */
enum {
  KR_SERR_NONE = 0,
  KR_SERR_MULTIPLE_HEADS = 1,        /* common/association.go:192-194 */
  KR_SERR_NO_HEAD_SERVICE = 2,
  KR_SERR_MULTIPLE_HEAD_SERVICES = 3,
  KR_SERR_EMPTY_SERVICE_IP = 4
};

/* cluster_results.status_flags */
enum {
  KR_SF_READY_BRANCH = 1u << 0,      /* State = ready and Reason = "" were assigned this pass (:1599-1604) */
  KR_SF_ALL_PODS_RUNNING = 1u << 1   /* utils.CheckAllPodsRunning(runtimePods) (utils/util.go:584-603) */
};

/* group_results.flags */
enum {
  KR_GR_PROCESSED       = 1u << 0,   /* loop body reached this group */
  KR_GR_EXPECT_PENDING  = 1u << 1,   /* :752-755 */
  KR_GR_SUSPENDED       = 1u << 2,   /* :766-775 */
  KR_GR_MULTIHOST       = 1u << 3,   /* :777-784 */
  KR_GR_WTD_EXECUTED    = 1u << 4,   /* the WorkersToDelete loop (:817-835) ran: every resolved wtd entry is a Delete call */
  KR_GR_ABORTED         = 1u << 5,   /* reconcilePods returned from inside this group */
  KR_GR_RANDOM_DELETE_OFF = 1u << 6, /* diff<0 but autoscaler owns deletions (:929-931) */
  KR_GR_CREATE_TRUNCATED = 1u << 7   /* create arena exhausted: n_create was clipped (engine limit, not reference behaviour) */
};

/* heads.annot_state / heads.version_state (raycluster_controller.go:1153-1168) */
enum { KR_ANNOT_EMPTY = 0, KR_ANNOT_HASH32 = 1, KR_ANNOT_OTHER = 2 };
enum { KR_VER_EMPTY = 0, KR_VER_CURRENT = 1, KR_VER_DIFFERENT = 2 };

/* head service ip kind (raycluster_controller.go:1726-1744) */
enum { KR_SVCIP_NORMAL = 0, KR_SVCIP_EMPTY = 1, KR_SVCIP_NONE = 2 /* "None": headless => head pod IP */ };

/* error codes */
enum {
  KR_OK = 0,
  KR_E_INVALID = -1,
  KR_E_CAPACITY = -2,
  KR_E_CUDA = -3,
  KR_E_STATE = -4,
  KR_E_NO_DEVICE = -5
};

/* -------------------------------------------------------------- config */

typedef struct kr_engine kr_engine;

typedef struct kr_config {
  int32_t  device;          /* CUDA ordinal */
  uint32_t max_clusters;
  uint32_t max_groups;
  uint32_t max_wtd;         /* total scaleStrategy.workersToDelete names */
  uint32_t max_pods;
  uint32_t max_heads;       /* rows of the head-aux table */
  uint32_t max_jobs;        /* RayJob roll-up rows */
  uint32_t max_creates;     /* capacity of the replica-index arena (ints) */
  uint64_t max_json_bytes;  /* muted-spec JSON arena */
} kr_config;

/* process-level switches read at reconcile time in the reference */
typedef struct kr_flags {
  uint8_t  gate_status_conditions;   /* features.RayClusterStatusConditions (pkg/features/features.go:56-62), default 1 */
  uint8_t  gate_multihost_indexing;  /* features.RayMultiHostIndexing, default 1 */
  uint8_t  env_random_pod_delete;    /* strings.ToLower(os.Getenv("ENABLE_RANDOM_POD_DELETE")) == "true" (:905) */
  uint8_t  skip_hash;                /* 1 => do not run the hash kernel (hash[] zeroed; Recreate gate treats hash as unknown) — test/bench knob only */
  uint8_t  fetch_pod_lists;          /* 1 => the pass also builds every RayCluster's full pod list in List order (sorted_pod_idx,
                                        sorted_action: 5 B/pod; cluster_result.pod_start) and kr_reconcile_batch / kr_results_fetch copy
                                        it back — verification and debugging; 0 => only the compact action list (act_*) is produced,
                                        which is all the shim consumes, and the pass takes the bucket pipeline (no per-cluster sort;
                                        pod_start is then 0) */
  uint8_t  reserved_[3];
  uint32_t id_head_not_found_reason; /* interned id of "HeadPodNotFound" */
  uint32_t id_head_not_found_msg;    /* interned id of "Head Pod not found" */
} kr_flags;

typedef struct kr_sizes {
  uint32_t n_clusters, n_groups, n_wtd, n_pods, n_heads, n_jobs;
  uint64_t json_bytes;
} kr_sizes;

/* ------------------------------------------------- snapshot (host arenas) */

/* All pointers below are engine-owned pinned host memory (cudaHostAlloc) sized
 * for kr_config capacities; the caller fills the first kr_sizes entries.
 * Go fills them through unsafe.Slice, so C never retains a Go pointer. */
typedef struct kr_snapshot_bufs {
  /* clusters [n_clusters]  — apis/ray/v1/raycluster_types.go:13-53, 277-348 */
  uint32_t *c_ns_id, *c_name_id;
  uint64_t *c_uid_hash;            /* sharding key (SURVEY §8(e)) */
  uint32_t *c_flags;               /* KR_CF_* */
  uint8_t  *c_suspend_status;      /* KR_SUSPEND_* */
  uint8_t  *c_ext_err_kind;        /* KR_EXT_ERR_* */
  uint32_t *c_ext_err_msg_id;
  uint32_t *c_group_off, *c_group_cnt;   /* worker groups in spec order */
  uint64_t *c_json_off;            /* offset into json[]; must be 16-byte aligned */
  uint32_t *c_json_len;
  /* old status (the copy taken at raycluster_controller.go:188) */
  uint8_t  *c_old_state;           /* KR_STATE_* */
  int32_t  *c_old_counts;          /* [5*n]: ready, available, desired, min, max */
  uint8_t  *c_old_cond_status;     /* [5*n]: KR_COND_* per slot */
  uint8_t  *c_old_cond_variant;    /* [5*n]: KR_CV_* per slot (ReplicaFailure: KR_EXT_ERR_* kind or KR_CV_OTHER) */
  uint32_t *c_old_cond_reason_id;  /* [n]: HeadPodReady reason */
  uint32_t *c_old_cond_msg_id;     /* [2*n]: [0]=HeadPodReady message, [1]=ReplicaFailure message */
  uint32_t *c_old_head_ids;        /* [4*n]: podIP, serviceIP, podName, serviceName (HeadInfo, :376-386) */
  /* head Service (raycluster_controller.go:1721-1745) */
  uint8_t  *c_svc_count;           /* 0, 1, 2 (= more than one) */
  uint8_t  *c_svc_ip_kind;         /* KR_SVCIP_* */
  uint32_t *c_svc_ip_id, *c_svc_name_id;

  /* groups [n_groups] — WorkerGroupSpec, raycluster_types.go:157-207 */
  uint32_t *g_cluster_idx, *g_name_id;
  int32_t  *g_replicas, *g_min, *g_max, *g_num_hosts;
  uint32_t *g_flags;               /* KR_GF_* */
  uint32_t *g_wtd_off, *g_wtd_cnt;

  /* workersToDelete names [n_wtd], grouped by group in spec order */
  uint32_t *w_name_id;

  /* pods [n_pods] in informer List order */
  uint32_t *p_ns_id, *p_cluster_name_id, *p_group_name_id, *p_name_id, *p_packed;
  int32_t  *p_replica_index;
  uint32_t *p_replica_name_id;

  /* head-aux rows [n_heads]: one per pod whose node-type label is head */
  uint32_t *h_pod_idx;
  uint8_t  *h_ready_status;        /* FindHeadPodReadyCondition(...).Status as KR_COND_* (utils/util.go:81-124) */
  uint32_t *h_ready_reason_id, *h_ready_msg_id;
  uint32_t *h_pod_ip_id;
  uint8_t  *h_annot_state;         /* KR_ANNOT_* of ray.io/upgrade-strategy-recreate-hash */
  uint8_t  *h_version_state;       /* KR_VER_* of ray.io/kuberay-version vs utils.KUBERAY_VERSION */
  uint8_t  *h_annot_hash;          /* [32*n]: the annotation's 32 chars when KR_ANNOT_HASH32 */

  /* RayJob roll-up rows [n_jobs] — rayjob_controller.go:203-216,343,880-905 */
  uint32_t *j_ns_id, *j_cluster_name_id;
  uint32_t *j_summary_id;          /* interned id of the canonical encoding of the job's current status.rayClusterStatus compare-fields */
  uint32_t *c_summary_id;          /* [n_clusters]: same encoding of the RayCluster's stored status */

  /* muted-spec JSON arena (bytes produced by Go json.Marshal, utils/util.go:629,645-661) */
  uint8_t  *json;
} kr_snapshot_bufs;

/* ------------------------------------------------------------- results */

typedef struct kr_cluster_result {      /* 96 bytes */
  uint8_t  path;                 /* KR_PATH_* */
  uint8_t  head_action;          /* KR_HEAD_* */
  uint8_t  err_kind;             /* KR_ERR_* : reconcileErr != nil iff != 0 */
  uint8_t  status_err;           /* KR_SERR_* */
  uint8_t  new_state;            /* KR_STATE_* */
  uint8_t  state_changed;        /* StateTransitionTimes[new_state] = now (:1711-1716) */
  uint8_t  needs_status_write;   /* InconsistentRayClusterStatus(old,new) (utils/consistency.go:16-34) && status_err == 0 */
  uint8_t  head_update_annotations; /* KubeRay version changed: re-annotate head pod (:1155-1162) */
  int32_t  stop_after_group;     /* group index inside which reconcilePods returned; group_cnt if it ran through; -1 if it returned before the worker loop */
  int32_t  err_arg;
  int32_t  n_pods;               /* len(runtimePods.Items) (:1583) */
  int32_t  n_heads;
  int32_t  head_pod_idx;         /* first head pod in list order, -1 if none */
  int32_t  counts[5];            /* ready, available, desired, min, max (utils/util.go:407-474) */
  uint8_t  cond_status[8];       /* [KR_NUM_CONDS] KR_COND_* after calculateStatus; rest padding */
  uint8_t  cond_variant[8];      /* [KR_NUM_CONDS] KR_CV_* */
  uint32_t head_ready_reason_id, head_ready_msg_id;
  uint32_t head_ids[4];          /* podIP, serviceIP, podName, serviceName */
  uint32_t pod_start;            /* this cluster's pods are sorted_pod_idx[pod_start .. pod_start+n_pods) in list order */
  uint32_t status_flags;         /* KR_SF_* */
} kr_cluster_result;

typedef struct kr_group_result {        /* 32 bytes */
  int32_t  expected;             /* int(GetWorkerGroupDesiredReplicas) (utils/util.go:386-404) */
  int32_t  n_list;               /* len(workerPods.Items) (:761) */
  int32_t  n_unhealthy;          /* :794 */
  int32_t  n_running;            /* len(runningPods.Items) (:837-842); multi-host: valid replica groups (:1055) */
  int32_t  diff;                 /* :849 (Go int, saturated at INT32_MIN); multi-host: replicasToCreate (:1064) */
  uint32_t n_create;             /* entries of create_idx this group owns: pods to create; for a KR_GR_MULTIHOST group REPLICA GROUPS to create
                                    (each one is NumOfHosts pods with one generated replica name, raycluster_controller.go:1081-1094) */
  uint32_t create_off;           /* first replica index of this group in create_idx[] (one entry per pod; multi-host: per replica) */
  uint32_t flags;                /* KR_GR_* */
} kr_group_result;

typedef struct kr_job_result {          /* 8 bytes */
  int32_t  cluster_idx;          /* -1: RayCluster not in snapshot */
  uint8_t  cluster_state;        /* KR_STATE_* of the stored RayCluster status */
  uint8_t  not_ready;            /* rayCluster.Status.State != Ready (rayjob_controller.go:209) */
  uint8_t  status_changed;       /* InconsistentRayClusterStatus(job.status.rayClusterStatus, cluster.status) (:885) */
  uint8_t  reserved;
} kr_job_result;

/* Engine-owned pinned host arenas, valid until the next kr_snapshot_begin. */
typedef struct kr_results_view {
  const kr_cluster_result *clusters;   /* [n_clusters] */
  const char              *hash;       /* [32*n_clusters] base32hex(sha1(json)) (utils/util.go:628-640) */
  const kr_group_result   *groups;     /* [n_groups] */
  const int32_t           *wtd_pod_idx;/* [n_wtd]: pod (same namespace, same name) the Delete call resolves to, -1 = NotFound */
  const uint32_t          *sorted_pod_idx; /* [n_pods]: pods bucketed by cluster, list order kept; orphans last.  NULL unless kr_flags.fetch_pod_lists */
  const uint8_t           *sorted_action;  /* [n_pods]: KR_ACT_* aligned with sorted_pod_idx.  NULL unless kr_flags.fetch_pod_lists */
  const int32_t           *create_idx; /* [n_create_total] replica indices (:869-881,1081-1094) */
  const kr_job_result     *jobs;       /* [n_jobs] */
  /* compact action list: every pod whose action != KEEP (orphans excluded), one contiguous run per cluster, List order inside
   * a run; cluster c owns entries [act_start[c], act_start[c] + act_cnt[c]).  This is all the Go shim needs to issue the Delete
   * calls.  The ORDER of the runs inside the list is unspecified when kr_flags.fetch_pod_lists == 0 (each RayCluster reserves
   * its run with one atomic; a RayCluster whose Recreate gate was still waiting for the digest reserves its whole bucket and
   * may use less), and is cluster order with act_start[c + 1] == act_start[c] + act_cnt[c] when it is 1.  The same holds for
   * create_idx: group g owns [create_off, create_off + n_create).  act_start[n_clusters] is only meaningful in the second case. */
  const uint32_t          *act_start;  /* [n_clusters + 1] */
  const uint32_t          *act_cnt;    /* [n_clusters] */
  const uint32_t          *act_pod_idx;/* [act_extent] */
  const uint8_t           *act_code;   /* [act_extent] KR_ACT_* */
  uint32_t n_create_total;         /* sum of group_results.n_create (= pods to create when no multi-host group is creating) */
  uint32_t n_orphans;
  uint32_t n_actions;              /* pods with action != KEEP (orphans excluded) = sum of act_cnt */
  uint32_t create_extent;          /* entries of create_idx in use (>= n_create_total) */
  uint32_t act_extent;             /* entries of act_pod_idx / act_code in use (>= n_actions) */
  /* Incremental epochs: after a full pass on the bucket pipeline (kr_flags.fetch_pod_lists == 0) the engine keeps its join tables,
   * per-cluster pod buckets, digests and results resident on the device.  While the commits that follow are
   * kr_snapshot_commit_pod_rows / _values and kr_snapshot_commit_parts(KR_PART_OBJECTS and/or KR_PART_JSON) — the informer's Pod and
   * RayCluster events — and the flags stay the same, the next pass re-matches only the touched pod rows, re-decides only the
   * RayClusters they (or changed object rows) belong to and returns only those records; every array of this view is still
   * complete and bit-identical to what a full pass would return.  n_changed / changed_clusters name the records that were
   * recomputed: n_changed == n_clusters and changed_clusters == NULL after a full pass.  Anything the resident state cannot
   * absorb (a changed table key or CSR offset, wholesale column commits, different flags, an overflowing bucket) silently
   * takes the full pass (with KR_OPT_LARGE_GROWTH, a RayCluster that outgrows its bucket or region gets a new region in the
   * incremental pass instead).  Snapshots with multi-host worker groups (numOfHosts > 1) keep incremental epochs, and so does an edit of
   * numOfHosts; so does an edit of a workersToDelete list with KR_OPT_WTD_EDITS (a length change only under KR_OPT_FIXED_LAYOUT).  Every pass is a full one on the sort pipeline — no resident state — while the caller fetches the full pod lists
   * (fetch_pod_lists = 1), while some RayCluster lists more than 256 pods (more than KR_LARGE_MAX_PODS with KR_OPT_LARGE_CLUSTERS,
   * unless KR_OPT_HUGE_CLUSTERS) or has more than 32 worker groups (unless KR_OPT_WIDE_CLUSTERS is set), or when KR_NO_INCR=1 is set in the environment. */
  uint32_t n_changed;
  const uint32_t          *changed_clusters; /* [n_changed] cluster rows, unordered */
} kr_results_view;

/* Per-kernel device times of the last kr_reconcile_batch (CUDA events on the engine's streams). */
#define KR_MAX_KERNEL_TIMES 24
typedef struct kr_profile {
  float    h2d_ms, kernels_ms, d2h_ms;      /* whole phases */
  uint32_t n_kernels;                       /* kernels launched by the last batch (our own, not library) */
  float    kernel_ms[KR_MAX_KERNEL_TIMES];  /* valid only after kr_reconcile_batch_profiled */
  const char *kernel_name[KR_MAX_KERNEL_TIMES];
  uint64_t h2d_bytes, d2h_bytes;            /* bytes uploaded by the commits since the previous pass (after a pass: plus the hash order it
                                               uploaded itself) / moved by the last results fetch */
} kr_profile;

/* --------------------------------------------------------- entry points */

/* Number of CUDA devices visible; <0 on error. */
int kr_device_count(void);

/* Create/destroy an engine bound to one device.  Replaces nothing in the reference;
 * a cgo shim calls it once from main() next to ctrl.NewManager (ray-operator/main.go:239-243). */
int  kr_engine_create(const kr_config *cfg, kr_engine **out);
void kr_engine_destroy(kr_engine *e);

/* Begin filling a snapshot: returns the pinned arenas.  Replaces the per-object
 * r.Get / cached r.List reads (raycluster_controller.go:114,674,761,1583; common/association.go:83-130,184). */
int kr_snapshot_begin(kr_engine *e, const kr_sizes *sizes, kr_snapshot_bufs *out);

/* Upload the filled snapshot (host -> HBM).  Asynchronous: the copies are queued on the engine's copy stream and the next
 * pass waits for them on the device; the arenas must not be rewritten before that pass (or kr_snapshot_begin) returns. */
int kr_snapshot_commit(kr_engine *e);

/* Upload only some parts of the arenas; the rest keeps what the previous commit of the SAME layout (same kr_sizes, and for
 * KR_PART_JSON the same c_json_off/c_json_len) put in HBM.  Typical epoch: pod statuses moved but no spec did — commit
 * KR_PART_COLUMNS and keep the spec-JSON arena resident (the hash is still recomputed from it every pass). */
enum {
  KR_PART_COLUMNS = 1,  /* every column */
  KR_PART_JSON = 2,     /* the muted-spec JSON arena.  Without KR_PART_OBJECTS / KR_PART_COLUMNS the c_json_off / c_json_len
                           columns stay behind: the RayClusters whose range moved need an object commit of their rows. */
  KR_PART_ALL = 3,
  KR_PART_OBJECTS = 4   /* every column except the seven per-pod ones: RayCluster / group / workersToDelete / head-aux / RayJob
                           rows (about 2 MB at C3).  Together with kr_snapshot_commit_pod_rows this is an incremental epoch. */
};
/* Every row is checked before anything moves: KR_E_INVALID (KR_E_CAPACITY for a RayCluster of 65 535 or more worker groups) for
 * groups out of cluster order or naming another RayCluster in g_cluster_idx, workersToDelete names out of group order or past
 * n_wtd, a JSON offset that is not 16-byte aligned or a range past json_bytes, a head-aux row whose h_pod_idx is not below n_pods;
 * KR_E_STATE for a partial commit before a full commit of the layout.  An invalid call commits nothing. */
int kr_snapshot_commit_parts(kr_engine *e, uint32_t parts);

/* Incremental epoch (SURVEY §8(f) rank 1): the caller has rewritten the 7 pod columns of `rows[0..n)` in the pinned arenas;
 * upload just those rows (rows may repeat; `rows` itself is copied before the call returns).  Informer events map to rows:
 * Update -> the Pod's row rewritten; Delete -> the row becomes a free row (every id 0, p_packed = KR_PP_TOMBSTONE);
 * Add -> a free row filled in (an arena is created with spare free rows; List order = row order, which is as arbitrary as the
 * informer cache's own order).  Combine with kr_snapshot_commit_parts(KR_PART_OBJECTS) for the RayCluster / group / head /
 * RayJob rows.  The rows are read from the arenas asynchronously (the device pulls them over PCIe): like after
 * kr_snapshot_commit, do not rewrite the arenas until the next pass has returned.  A change that moves a table's row
 * count (kr_sizes) needs kr_snapshot_begin + a full commit. */
int kr_snapshot_commit_pod_rows(kr_engine *e, const uint32_t *rows, uint32_t n);

/* The same epoch, journal style: the caller hands over the new rows themselves instead of writing them into the arenas —
 * values[7*i + k] is column k (p_ns_id, p_cluster_name_id, p_group_name_id, p_name_id, p_packed, p_replica_index,
 * p_replica_name_id) of pod row rows[i]; the rows[] entries must be distinct.  One contiguous upload of 32 bytes per row
 * (both arrays are copied before the call returns); the device scatters the values into the resident columns.  The pinned
 * arenas are NOT touched: a caller that may later take the full-commit path writes the row there as well (its handler has the
 * values in hand either way).  Faster than kr_snapshot_commit_pod_rows, whose rows the device pulls over PCIe one 32-byte
 * sector at a time. */
int kr_snapshot_commit_pod_values(kr_engine *e, const uint32_t *rows, const uint32_t *values, uint32_t n);

/* Row-granular object commit: the caller rewrote, in the arenas, the rows of `cluster_rows` (every per-RayCluster column and the rows
 * of those clusters' worker groups — same group count, same names, same workersToDelete lists as before) and the head-aux rows
 * `head_rows` (same row count as before).  Only those rows travel (packed) and are applied by the on-device object diff.  It is
 * purely an optimisation of kr_snapshot_commit_parts(KR_PART_OBJECTS) — the informer's RayCluster status / replica / expectation
 * updates and head Pod status updates at a few hundred bytes per object instead of the whole object part: whenever the engine has
 * no resident state, or a Recreate gate, a JSON range or the number of head rows changed, it commits the whole object part itself.
 * That includes a range an earlier KR_PART_JSON-only commit moved (an arena compaction moves every range): unless every such
 * RayCluster is among `cluster_rows`, the whole object part is committed.  Whichever path it takes, the named rows are checked as
 * kr_snapshot_commit_parts checks them, and a row >= n_clusters or a head-aux row >= n_heads is KR_E_INVALID; an invalid call
 * commits nothing. */
int kr_snapshot_commit_object_rows(kr_engine *e, const uint32_t *cluster_rows, uint32_t n_cluster_rows, const uint32_t *head_rows, uint32_t n_head_rows);

/* Row-granular spec commit: the caller rewrote, in the pinned arenas, the muted-spec JSON of the RayClusters `cluster_rows` — in
 * place or at a new 16-byte aligned range inside the live json_bytes — and their c_json_off / c_json_len.  Only those ranges
 * (padded to 16 bytes) and those two column entries travel; the next pass re-hashes only these messages and re-decides only those
 * of them whose Recreate gate reads the digest.  Results equal kr_snapshot_commit_parts(KR_PART_JSON).  Rows may repeat and may be
 * given in several calls per epoch (the engine takes the union); `cluster_rows` is copied before the call returns.  The device
 * pulls the ranges from the arenas asynchronously: do not rewrite them until the next pass has returned.  Call it BEFORE the
 * epoch's object commit (kr_snapshot_commit_parts(KR_PART_OBJECTS) / kr_snapshot_commit_object_rows): an object commit that finds a
 * moved range re-hashes every RayCluster — correct, only slower.  A whole-arena commit (KR_PART_JSON) in the same epoch wins.
 * A row listed again before the pass that hashes it is pulled once per pass in between (after a skip_hash pass, which leaves the rows
 * pending, the caller may have rewritten it) and hashed once.  kr_profile.h2d_bytes counts 16 B per pulled row (row id, offset,
 * length) plus its padded range, and, at the pass that hashes them, 4 B per row for their hash order (the pending rows sorted by
 * SHA-1 block count, uploaded once).
 * KR_E_STATE before a full commit of the layout; KR_E_INVALID for a row >= n_clusters, an offset that is not 16-byte aligned or a
 * range past json_bytes (nothing is committed then). */
int kr_snapshot_commit_spec_rows(kr_engine *e, const uint32_t *cluster_rows, uint32_t n);

/* Run the whole decision + status pass over the committed snapshot and copy the results back.
 * Replaces the decision halves of reconcilePods (raycluster_controller.go:619-935), reconcileMultiHostWorkerGroup
 * (:963-1125), shouldRecreatePodsForUpgrade (:1132-1171), shouldDeletePod (:1181-1231), calculateStatus (:1552-1719),
 * GetWorkerGroupDesiredReplicas/Calculate*Replicas (utils/util.go:386-474), CheckAllPodsRunning (:584-603),
 * GenerateHashWithoutReplicasAndWorkersToDelete (:642-665, SHA-1 + base32hex half) and
 * InconsistentRayClusterStatus (utils/consistency.go:16-34); RayJob roll-up rayjob_controller.go:209-216,343,885. */
int kr_reconcile_batch(kr_engine *e, const kr_flags *flags, kr_results_view *out);

/* Same pass, kernels only: no D2H copy, results stay in HBM (bench "value" leg; also used under ncu). */
int kr_reconcile_device_only(kr_engine *e, const kr_flags *flags);

/* Same as kr_reconcile_device_only but serialises the kernels and brackets each with CUDA events. */
int kr_reconcile_batch_profiled(kr_engine *e, const kr_flags *flags, kr_profile *prof);

/* Copy results of the last device-only pass to the host arenas. */
int kr_results_fetch(kr_engine *e, kr_results_view *out);

/* Stand-alone batched hash: base32hex(sha1(bytes[offsets[i]..offsets[i+1]))) for i<n into out32xN
 * (32 chars per message, no terminator).  Replaces utils.GenerateJsonHash's digest half (utils/util.go:634-637);
 * also used by rayservice_controller.go:1130-1157,1244 callers.  Host buffers; copies included. */
int kr_hash_batch(kr_engine *e, const uint8_t *bytes, const uint64_t *offsets, uint32_t n, char *out32xN);

/* Batched isClusterSpecHashEqual (rayservice_controller.go:1130-1157; callers :1121-1127, :1179-1186 and the rollback check
 * :2064-2094): for every row, does the RayCluster's ray.io/hash-without-replicas-and-workers-to-delete annotation equal the hash
 * of the RayService's goal spec?  The goal specs are canonicalised on the host (kr_spec_json_emit) and hashed in ONE GPU batch.
 *   partial == 0: goal hash = hash(mute(goal spec)); a goal spec that does not parse hashes to "" (the reference drops the error).
 *   partial != 0: n = strconv.Atoi(num-worker-groups annotation); failure => equal (the reference returns true); with at least n
 *                 goal worker groups the hash is taken over the first n only, with fewer the goal hash stays "" (:1143-1153).
 *                 (A negative n panics in the reference — slice bounds; here it counts as an Atoi failure.)
 * equal_out[i] = 1 / 0; goal_hash_out32xN (optional) receives the 32 characters of every goal hash, zero bytes when it is "". */
typedef struct kr_hash_compare_row {
  const uint8_t *goal_spec_json;      /* RayService .spec.rayClusterSpec as JSON text, any key order */
  uint64_t       goal_spec_len;
  const char    *cluster_hash;        /* the annotation's value; NULL / len 0 when absent */
  uint32_t       cluster_hash_len;
  const char    *num_worker_groups;   /* annotation ray.io/num-worker-groups (only read when partial) */
  uint32_t       num_worker_groups_len;
  uint8_t        partial;
  uint8_t        reserved_[7];
} kr_hash_compare_row;
int kr_hash_compare_batch(kr_engine *e, const kr_hash_compare_row *rows, uint32_t n, uint8_t *equal_out, char *goal_hash_out32xN);

/* Timings of the last batch. */
int kr_last_profile(kr_engine *e, kr_profile *prof);

/* Engine options (call before the first kr_snapshot_begin).
 * KR_OPT_FIXED_LAYOUT = 1: lay the arenas out once, for the capacities given to kr_engine_create, instead of per snapshot.
 *   Column addresses then never move: kr_snapshot_begin(sizes) only sets the live row counts (<= capacities) and returns the
 *   same pointers, and what is resident in HBM stays valid across begins.  A head Pod appearing or going, or a Pod appended after
 *   the last row, is still an incremental epoch: kr_snapshot_begin(new counts) + KR_PART_OBJECTS + kr_snapshot_commit_pod_rows/
 *   _values.  So are workersToDelete lists that grow or shrink, with KR_OPT_WTD_EDITS, and RayClusters appended after the last row
 *   or RayJobs created or deleted, with KR_OPT_CLUSTER_CREATES, RayClusters deleted by swap-remove, with KR_OPT_CLUSTER_DELETES,
 *   and worker groups added to or removed from a RayCluster, with KR_OPT_GROUP_EDITS.  Any other change of a row count (one of these
 *   without its option) makes the next pass a full one. */
enum {
  KR_OPT_FIXED_LAYOUT = 1,
  KR_OPT_INCREMENTAL = 2,  /* 1 (default): passes after a full bucket-pipeline pass are incremental on the device whenever the commits in
                              between allow it (kr_results_view docs); 0: every pass is a full pass (benchmarks of the full pass, tests).
                              May be changed at any time. */
  KR_OPT_LARGE_CLUSTERS = 3,  /* 1: RayClusters listing more than 256 and at most KR_LARGE_MAX_PODS pods stay on the bucket pipeline
                              (DESIGN §4.1): a bucket attempt that meets one gives it a region of its own instead of widening the stride
                              of the whole fleet or leaving the pipeline, so such a fleet keeps its incremental epochs.  Results are the
                              same as with 0 (the default: one such RayCluster sends every pass to the sort pipeline).  May be set at any
                              time; takes effect at the next full pass.  A RayCluster of more than KR_LARGE_MAX_PODS pods still sends
                              the pass to the sort / radix pipelines, unless KR_OPT_HUGE_CLUSTERS.  A RayCluster that outgrows its
                              bucket or region in an incremental epoch makes that epoch a full pass, unless KR_OPT_LARGE_GROWTH.
                              Turning it on allocates the region arena once, for the
                              capacities: about 11 B per max_pods + 20 B per max_clusters of device memory. */
  KR_OPT_BUCKET_STRIDE = 4,   /* read only (kr_engine_get_option): records per RayCluster bucket of the current layout (64 / 128 / 256);
                              0 = the passes take the sort pipeline */
  KR_OPT_WIDE_CLUSTERS = 5,   /* 1: RayClusters with more than 32 worker groups stay on the bucket pipeline (DESIGN §4.1): one CTA per
                              such RayCluster decides it beside the warp-per-cluster decide of the others, so such a fleet keeps its
                              incremental epochs.  Results are the same as with 0 (the default: one such RayCluster sends every pass to
                              the sort pipeline).  May be set at any time; takes effect at the next full pass.  A wide RayCluster of more
                              than 256 pods is treated like any other such RayCluster: with KR_OPT_LARGE_CLUSTERS it gets a region,
                              without it the stride widens or the pass leaves the bucket pipeline.  Turning it on allocates 20 B per
                              max_clusters of device memory once (shared with KR_OPT_LARGE_CLUSTERS). */
  KR_OPT_HUGE_CLUSTERS = 6,   /* 1, together with KR_OPT_LARGE_CLUSTERS: RayClusters of more than KR_LARGE_MAX_PODS pods also stay on
                              the bucket pipeline (DESIGN §4.1): they get regions like the large ones, and their pods are put in List
                              order tile by tile and merged on the device, so no RayCluster is too large for incremental epochs.  No
                              effect while KR_OPT_LARGE_CLUSTERS is 0.  Results are the same as with 0 (the default: one such RayCluster
                              sends every pass to the sort / radix pipelines).  May be set at any time; takes effect at the next full
                              pass.  Turning it on allocates the tile scratch once, for the capacities: about 18 B per max_pods of device
                              memory (at least 128 KB). */
  KR_OPT_WTD_EDITS = 7,       /* 1: an edit of a scaleStrategy.workersToDelete list (a name renamed, a list grown or shrunk, as the
                              autoscaler writes on every scale-down and clears once the Pods are gone) keeps the incremental epoch: the
                              next pass rebuilds the name table on the device and re-decides only the RayClusters whose Pods were named
                              before or are named now.  A list whose length changes moves n_wtd, which needs KR_OPT_FIXED_LAYOUT (without
                              it every new row count is a full pass); a rename does not.  Results are the same as with 0 (the default:
                              any such edit makes the next pass a full one).  May be set at any time; read at each object commit.
                              kr_snapshot_commit_object_rows still expects unchanged lists: with this option, rows whose lists changed
                              are committed as the whole object part. */
  KR_OPT_SPEC_ROWS = 8,       /* 1: the native packer (kr_packer_flush) commits re-emitted specs with kr_snapshot_commit_spec_rows and
                              reports KR_PACK_SPEC_ROWS instead of KR_PART_JSON (a flush that compacts the JSON arena still sends
                              KR_PART_JSON).  The engine call itself needs no option.  Results are the same as with 0 (the default). */
  KR_OPT_CLUSTER_CREATES = 9, /* 1, together with KR_OPT_FIXED_LAYOUT: RayClusters appended after the last row (every existing
                              RayCluster keeps its row, its groups and its workersToDelete names, and the new groups and names come after
                              all the old ones), and RayJobs created or deleted, keep the incremental epoch: kr_snapshot_begin(new
                              counts), the object part (KR_PART_OBJECTS), then the new RayClusters' specs with
                              kr_snapshot_commit_spec_rows.  The next pass hashes only those specs, inserts the new RayClusters into
                              the resident tables, moves the resident Pods labelled for them out of the orphans and into their buckets,
                              and returns them among changed_clusters.  A RayCluster deleted, a worker group added to an existing one
                              (unless KR_OPT_GROUP_EDITS), fewer RayClusters than before, or a RayCluster the resident state cannot hold (more Pods than its bucket
                              without KR_OPT_LARGE_CLUSTERS, more than 32 worker groups without KR_OPT_WIDE_CLUSTERS) still takes the
                              full pass.  Results are the same as with 0 (the default: every such event makes the next pass a full
                              one).  May be set at any time; read at each kr_snapshot_begin and object commit.  No effect without
                              KR_OPT_FIXED_LAYOUT.  The native packer's flush takes this path by itself when the engine has the option
                              and a flush only appended RayClusters or created and deleted RayJobs.  Deleting a RayCluster is
                              KR_OPT_CLUSTER_DELETES. */
  KR_OPT_CLUSTER_DELETES = 10, /* 1, together with KR_OPT_FIXED_LAYOUT: RayClusters deleted by swap-remove keep the incremental epoch:
                              kr_snapshot_begin(new counts), then the object part (KR_PART_OBJECTS), where every surviving RayCluster
                              either keeps its row or moves from a row at or past the new n_clusters into a row a deleted RayCluster
                              vacated, keeps its worker-group count (unless KR_OPT_GROUP_EDITS), and groups and workersToDelete names
                              stay in row order.  With
                              KR_OPT_CLUSTER_CREATES the same epoch may also create RayClusters, in vacated rows or after the last one
                              (their specs then follow with kr_snapshot_commit_spec_rows).  The next pass releases the deleted
                              RayClusters' Pods (orphans from then on), brings every moved RayCluster's Pods to its new row, moves its
                              digest when its spec range stayed, shifts the per-group results, and re-decides only the moved and created
                              RayClusters, which it returns among changed_clusters.  Still full passes: another renumbering, a surviving
                              RayCluster whose group count changed (without KR_OPT_GROUP_EDITS), a deleted or moved key that another row also holds, more than 4 096
                              RayClusters deleted, moved or created at once, a deleted or moved RayCluster that is large
                              (KR_OPT_LARGE_CLUSTERS: one with a region) unless KR_OPT_LARGE_MOVES, and, within one epoch, a renumbering after an object
                              commit that appended RayClusters, or any object commit after a renumbering that changes a row count or
                              renumbers again.  With KR_OPT_WIDE_CLUSTERS, RayClusters of more than 32 worker groups are followed too.
                              Results are the same as with 0 (the default: every deletion makes the next pass a full one).  May be set
                              at any time; read at each kr_snapshot_begin and object commit.  No effect without KR_OPT_FIXED_LAYOUT.
                              The native packer's flush takes this path by itself when the engine has the option (the specs it placed
                              travel as spec rows unless it compacted the JSON arena). */
  KR_OPT_GROUP_EDITS = 11,    /* 1, together with KR_OPT_FIXED_LAYOUT: a RayCluster whose list of worker groups changed (groups appended,
                              as a RayService in-place update does, removed, renamed or reordered) keeps the incremental epoch:
                              kr_snapshot_begin(new counts; n_groups and n_wtd may move either way), then the object part
                              (KR_PART_OBJECTS), with the RayCluster's spec, when it was re-emitted, as a spec row before or after it.
                              The RayCluster is released and initialised again in its own row: the next pass touches its Pods and matches
                              them against its new groups (a Pod of a removed group stays among its Pods, in no group), shifts the
                              per-group results of the RayClusters after it, keeps its digest unless its spec range moved, and
                              re-decides it, returning it among changed_clusters with the RayClusters whose Pods a rebuilt
                              workersToDelete name table touched.  With KR_OPT_CLUSTER_DELETES a RayCluster moved by swap-remove may
                              change its group count in the same epoch, and with KR_OPT_CLUSTER_CREATES the epoch may create
                              RayClusters as well.  Still full passes: a regrouped RayCluster that is large (KR_OPT_LARGE_CLUSTERS: one
                              with a region) unless KR_OPT_LARGE_MOVES, one of more than 32 worker groups without
                              KR_OPT_WIDE_CLUSTERS, more than 4 096 RayClusters deleted, moved, created or regrouped at once, the rules
                              of KR_OPT_CLUSTER_DELETES for two object commits in one epoch, and group edits committed with
                              kr_snapshot_commit_object_rows (a changed group count falls back to the whole object part; a renamed
                              group there is structural).  Results are the same as with 0 (the default: every such edit makes the
                              next pass a full one).  May be set at any time; read at each kr_snapshot_begin and object commit (the
                              first object commit with it on records the group names, the next ones compare against them).  No effect
                              without KR_OPT_FIXED_LAYOUT.  The native packer's flush takes this path by itself when the engine has the
                              option: the regrouped RayClusters' specs travel as spec rows. */
  KR_OPT_LARGE_GROWTH = 12,   /* 1, together with KR_OPT_LARGE_CLUSTERS: a RayCluster that outgrows its room in an incremental epoch (an
                              ordinary one its bucket, a large one its region, as Pods join it when it scales up) keeps the incremental
                              epoch: the pass gives it a region of the size a full pass would (1.25x its Pods rounded up to 32, at
                              most KR_LARGE_MAX_PODS, less the stride) past the regions in use, copies a large one's old region into it,
                              places the records that did not fit and decides it with the per-cluster kernels in the same pass.  The
                              stride does not move, and the grown RayClusters are among changed_clusters.  This also covers a
                              RayCluster KR_OPT_CLUSTER_CREATES creates and that adopts more resident orphan Pods than its bucket holds.
                              Still full passes: more than KR_GROW_MAX RayClusters outgrowing their room at once, promotions that
                              would take the per-cluster list past max(KR_GROW_LIST_MIN, n_clusters / KR_GROW_LIST_DIV) RayClusters (a
                              regrowth alone adds no one to the list and is never held back by it), a RayCluster of more than
                              KR_LARGE_MAX_PODS Pods (a huge one needs tiles) unless KR_OPT_HUGE_GROWTH, a full region arena (regions a
                              regrowth abandons are reclaimed by the next full pass that reclassifies) and more than KR_GROW_SPILL Pods
                              joining grown RayClusters in one epoch.  Results are the same as with 0 (the default: each such epoch is
                              a full pass that widens the stride or reclassifies the fleet).  May be set at any time; read at each
                              incremental pass.  No effect without KR_OPT_LARGE_CLUSTERS.  Turning it on allocates about 0.5 MB of
                              device memory and 1 KB of pinned host memory once. */
  KR_OPT_LARGE_MOVES = 13,    /* 1, together with KR_OPT_LARGE_CLUSTERS and KR_OPT_FIXED_LAYOUT: KR_OPT_CLUSTER_DELETES and
                              KR_OPT_GROUP_EDITS also follow large RayClusters (those with a region, huge ones included) incrementally.
                              A deleted large RayCluster's Pods are released, bucket and region, and become orphans; its region is
                              abandoned until the next full pass that reclassifies the fleet.  A large RayCluster moved by swap-remove
                              carries its region (offset and capacity) and, a huge one, its tiles to its new row, and its Pods are
                              admitted there again.  A regrouped large RayCluster keeps its region and is initialised again in place.
                              Either one is re-decided by the per-cluster kernels in the same pass and returned among changed_clusters.
                              Still full passes with it: the other rules of KR_OPT_CLUSTER_DELETES and KR_OPT_GROUP_EDITS (more than
                              4 096 RayClusters in one map, two object commits in one epoch), and a moved or regrouped large RayCluster
                              that joins more Pods than its carried region holds, unless KR_OPT_LARGE_GROWTH gives it a new region in
                              the same pass (one that grows past KR_LARGE_MAX_PODS Pods also needs KR_OPT_HUGE_GROWTH: its carried
                              tiles are retired and new ones appended).  Results are the same as with 0 (the default: every such
                              epoch is a full pass).  May be set at any time; read at each object commit.  No effect without
                              KR_OPT_LARGE_CLUSTERS and KR_OPT_FIXED_LAYOUT. */
  KR_OPT_HUGE_GROWTH = 14     /* 1, together with KR_OPT_LARGE_CLUSTERS, KR_OPT_HUGE_CLUSTERS and KR_OPT_LARGE_GROWTH: a RayCluster that
                              grows past KR_LARGE_MAX_PODS Pods in an incremental epoch (a large one that scales past it, an ordinary
                              one that jumps past it, or a huge one that outgrows its region) keeps the incremental epoch: the pass
                              gives it a region of the size a full pass would (1.25x its Pods rounded up to 32, less the stride),
                              appends its tiles to the KR_HUGE_GROW_TILES reserve entries of the tile table (retiring a huge one's
                              old tiles), and sorts and decides it with the tile kernels in the same pass.  The stride does not move,
                              and the grown RayClusters are among changed_clusters.  Still full passes: more tiles than
                              KR_HUGE_GROW_TILES appended in one epoch (a RayCluster regrown to about 200 000 Pods or more), more
                              resident tiles than the engine's capacities hold, and the limits of KR_OPT_LARGE_GROWTH: more than
                              KR_GROW_SPILL Pods waiting for new regions, a full region arena, the per-cluster list cap and more than
                              KR_GROW_MAX RayClusters growing at once.  Results are the same as with 0 (the default: each such epoch
                              is a full pass that lays every region out again).  May be set at any time; read at each incremental
                              pass.  No effect without the three other options.  Turning it on allocates the tile scratch with
                              KR_HUGE_GROW_TILES more tiles (64 KB of device memory each); an engine whose KR_OPT_HUGE_CLUSTERS had
                              allocated it reallocates it. */
};
enum { KR_LARGE_MAX_PODS = 8192 };  /* largest RayCluster KR_OPT_LARGE_CLUSTERS keeps on the bucket pipeline */
/* KR_OPT_LARGE_GROWTH: at most KR_GROW_MAX RayClusters get a region in one incremental epoch, and an epoch that puts RayClusters on
 * the per-cluster kernels' list may leave it at most max(KR_GROW_LIST_MIN, n_clusters / KR_GROW_LIST_DIV) long (BASELINE.md: k_decide_large over promoted
 * RayClusters); beyond either, the epoch is a full pass, so a fleet that grows as a whole still widens its stride.  At most
 * KR_GROW_SPILL records of grown RayClusters wait for their new regions in one epoch. */
enum { KR_GROW_MAX = 64, KR_GROW_LIST_MIN = 64, KR_GROW_LIST_DIV = 64, KR_GROW_SPILL = 16384 };
/* KR_OPT_HUGE_GROWTH: tile-table entries kept free past the resident tiles for the RayClusters an incremental epoch makes huge or
 * regrows (KR_LARGE_MAX_PODS arrival ranks each: 262 144 in all). */
enum { KR_HUGE_GROW_TILES = 32 };
int kr_engine_set_option(kr_engine *e, uint32_t option, uint64_t value);
/* Current value of an option (KR_OPT_*), and the read-only KR_OPT_BUCKET_STRIDE. */
int kr_engine_get_option(kr_engine *e, uint32_t option, uint64_t *value);

/* Device pointer + byte size of the per-group delta records (kr_group_result[n_groups]) of the last pass:
 * the payload of the optional cross-GPU all-gather (SURVEY §8(e)); the caller owns the collective. */
int kr_group_results_device(kr_engine *e, const void **dev_ptr, uint64_t *bytes);

/* Copy those records device-to-device into a caller-owned device buffer (e.g. a torch tensor handed to
 * torch.distributed.all_gather over NCCL); synchronises the engine stream before returning. */
int kr_group_results_copy(kr_engine *e, void *dst_device, uint64_t dst_capacity_bytes);

/* ---- spec JSON (SURVEY §8(f) rank 2): the step BEFORE the hash, host code (no device needed).
 * Canonical bytes of json.Marshal(mute(RayClusterSpec)) — what utils.GenerateHashWithoutReplicasAndWorkersToDelete hashes
 * (ray-operator/controllers/ray/utils/util.go:642-665, types apis/ray/v1/raycluster_types.go:13-225) — from the spec as JSON
 * text in any key order (e.g. `.spec` of the watch event, whose keys the API server sorts alphabetically).  Replaces the
 * per-reconcile DeepCopy + reflective json.Marshal of the reference: the shim calls it once per metadata.generation.
 * flags: KR_SPEC_JSON_UNMUTED = plain json.Marshal(spec) without the muting (utils.GenerateJsonHash callers).
 * Returns KR_E_INVALID on malformed input, KR_E_CAPACITY (with *out_len = the size needed) when out is too small. */
enum { KR_SPEC_JSON_UNMUTED = 1 };
int kr_spec_json_emit(const uint8_t *spec_json, uint64_t len, uint32_t flags, uint8_t *out, uint64_t out_cap, uint64_t *out_len);

/* Same, written straight into a JSON arena (kr_snapshot_bufs.json): the bytes go to the next 16-byte aligned offset at or after
 * *cursor, zero-padded to 16 bytes; *off_out / *len_out are the values for c_json_off / c_json_len; *cursor moves past them. */
int kr_spec_json_emit_arena(const uint8_t *spec_json, uint64_t len, uint8_t *arena, uint64_t arena_cap, uint64_t *cursor,
                            uint64_t *off_out, uint32_t *len_out);

/* resource.Quantity's canonical string ("1000m" -> "1", "1.5Gi" -> "1536Mi", "0.5" -> "500m"; k8s.io/apimachinery
 * pkg/api/resource Quantity.String), NUL-terminated into out.  Used by the emitter for ResourceList values. */
int kr_quantity_canonical(const char *text, char *out, uint64_t out_cap);

/* Error text of the last failing kr_spec_json_* / kr_quantity_canonical call on this thread (never NULL). */
const char *kr_spec_json_last_error(void);

/* ---- multi-GPU coordinator (SURVEY §8(b) "one engine per device + a coordinator", §8(e)).  One process, one engine per shard,
 * each driven by its own host thread bound to its GPU's NUMA node (the thread also creates the engine: node-local pinned arenas).
 * A RayCluster's decisions depend only on its own objects (common/association.go:83-130), so the snapshot shards by
 * uid_hash64 % n with no data-path collective; the only exchange is the optional all-gather of the per-group delta records.
 * devices[i] = CUDA ordinal of shard i (NULL: i % device count; a device may repeat — several shards on one GPU).
 * The group's calls are made from ONE coordinator thread; the engines stay reachable (kr_group_engine) for the per-shard calls
 * (kr_snapshot_commit_pod_rows, kr_results_fetch, ...), which the caller may issue from any one thread at a time per engine. */
typedef struct kr_group kr_group;
int       kr_group_create(const kr_config *per_shard_capacities, const int32_t *devices, uint32_t n, kr_group **out);
void      kr_group_destroy(kr_group *g);
uint32_t  kr_group_size(kr_group *g);
kr_engine *kr_group_engine(kr_group *g, uint32_t shard);
int       kr_group_device(kr_group *g, uint32_t shard);
uint32_t  kr_group_shard_of_uid(kr_group *g, uint64_t uid_hash);   /* uid_hash64 % n */
/* Route a GLOBAL snapshot (host columns in `global`, row counts in `n`) into the shards' pinned arenas — kr_snapshot_begin +
 * fill of every engine, natively: clusters by UID hash, pods through the (namespace, ray.io/cluster) -> cluster table (orphans by
 * a hash of that key), head-aux rows after their pod, RayJobs after their RayCluster; List order is kept inside every shard and
 * every index column is rewritten.  The optional outputs say where each global cluster / pod row went ([n_clusters] / [n_pods]):
 * the shim maps the shards' result rows back through them.  Follow with kr_group_commit. */
int       kr_group_route(kr_group *g, const kr_snapshot_bufs *global, const kr_sizes *n, kr_sizes *shard_sizes_out,
                         uint32_t *cluster_shard_out, uint32_t *cluster_row_out, uint32_t *pod_shard_out, uint32_t *pod_row_out);
int       kr_group_commit(kr_group *g, uint32_t parts);                                           /* kr_snapshot_commit_parts on every shard, in parallel */
int       kr_group_reconcile(kr_group *g, const kr_flags *flags, kr_results_view *views /* [n] */); /* kr_reconcile_batch on every shard, in parallel */
/* The optional exchange step: every device receives every shard's kr_group_result records.  *slot_bytes_out = bytes per shard
 * slot (32 * the largest shard's n_groups, rounded up to 256; shorter shards are zero padded); host_out (optional, >= n slots)
 * receives device 0's gathered copy.  NCCL (ncclAllGather from the coordinator thread) when every shard has its own device and
 * libnccl is loadable, peer copies otherwise; *used_nccl_out says which. */
int       kr_group_allgather_group_results(kr_group *g, void *host_out, uint64_t host_cap, uint64_t *slot_bytes_out, int *used_nccl_out);
const char *kr_group_last_error(kr_group *g);

/* ---- native event-driven packer / interner (SURVEY §8(f) rank 1: the step BEFORE the path; host code).
 * The shim's informer handlers (watch set raycluster_controller.go:1525-1533, cache universe internal/managercache/cache.go:16-36)
 * call the upsert / delete entry points as events arrive; kr_packer_flush brings the device copy up to date before an epoch:
 * only the pod rows the events touched, the small RayCluster / group / head / RayJob tables when one of them changed, and the
 * muted-spec JSON (kr_spec_json_emit, re-emitted only when metadata.generation moved) cross PCIe.  The packer owns an engine
 * created with KR_OPT_FIXED_LAYOUT for the given capacities; kr_packer_engine() is the handle for kr_reconcile_batch etc.
 * Strings are interned here (kr_packer_string turns a result's id back into bytes).  One caller thread at a time. */
typedef struct kr_str { const char *p; uint32_t n; } kr_str;   /* not NUL-terminated; p == NULL: absent (label / annotation / field not there) */
typedef struct kr_pod_obj {            /* what the path reads of a *corev1.Pod (SURVEY Appendix A.1) */
  kr_str ns, name;
  kr_str cluster, group, replica_name, replica_index;  /* labels ray.io/cluster, ray.io/group, ray.io/worker-group-replica-name / -index (text; strconv.Atoi here) */
  uint8_t node_type, phase, ready_cond;  /* KR_NT_*, KR_PHASE_*, PodReady condition as KR_COND_* */
  uint8_t restart_never, ray_terminated, has_deletion_ts;
  uint8_t head_ready_status, reserved_;  /* the rest is read only for node_type == KR_NT_HEAD */
  kr_str head_ready_reason, head_ready_msg;  /* FindHeadPodReadyCondition (utils/util.go:81-124) */
  kr_str pod_ip, recreate_hash, kuberay_version;  /* status.podIP; annotations ray.io/upgrade-strategy-recreate-hash, ray.io/kuberay-version */
} kr_pod_obj;
typedef struct kr_group_obj {          /* WorkerGroupSpec (apis/ray/v1/raycluster_types.go:157-207) + its expectation bit */
  kr_str name;
  int32_t replicas, min_replicas, max_replicas, num_hosts;
  uint32_t flags;                      /* KR_GF_* */
  const kr_str *workers_to_delete; uint32_t n_workers_to_delete;
} kr_group_obj;
typedef struct kr_cluster_obj {
  kr_str ns, name, uid;
  uint64_t resource_version, generation;  /* epoch keys (SURVEY §8(b)); the spec JSON is re-emitted only when generation moves */
  uint32_t flags;                      /* KR_CF_* */
  uint8_t suspend_status, ext_err_kind, old_state, svc_count, svc_ip_kind;
  uint8_t spec_json_verbatim;          /* 1: spec_json already IS json.Marshal(mute(spec)) (marshalled by the Go side): stored as is */
  uint8_t reserved_[2];
  kr_str ext_err_msg;
  int32_t old_counts[5];
  uint8_t old_cond_status[5], old_cond_variant[5], reserved2_[6];
  kr_str old_head_ready_reason, old_head_ready_msg, old_replica_failure_msg;
  kr_str old_head[4];                  /* podIP, serviceIP, podName, serviceName */
  kr_str svc_ip, svc_name, status_summary;
  const kr_group_obj *groups; uint32_t n_groups;
  const uint8_t *spec_json; uint64_t spec_json_len;  /* .spec as JSON text, any key order */
} kr_cluster_obj;
typedef struct kr_job_obj { kr_str ns, name, cluster_name, status_summary; } kr_job_obj;
typedef struct kr_packer kr_packer;
enum { KR_PACK_POD_ROWS = 8, KR_PACK_FULL = 16, KR_PACK_OBJECT_ROWS = 32, KR_PACK_SPEC_ROWS = 64 };  /* kr_packer_flush mode bits, beside KR_PART_OBJECTS / KR_PART_JSON (OBJECT_ROWS: kr_snapshot_commit_object_rows instead of the whole object part; SPEC_ROWS: kr_snapshot_commit_spec_rows instead of KR_PART_JSON, with KR_OPT_SPEC_ROWS) */
int        kr_packer_create(const kr_config *capacities, kr_packer **out);
void       kr_packer_destroy(kr_packer *p);
kr_engine *kr_packer_engine(kr_packer *p);
int        kr_packer_set_kuberay_version(kr_packer *p, kr_str version);  /* utils.KUBERAY_VERSION; default "nightly" */
int        kr_packer_pod_upsert(kr_packer *p, const kr_pod_obj *pod);      /* Add / Update */
int        kr_packer_pod_delete(kr_packer *p, kr_str ns, kr_str name);
int        kr_packer_cluster_upsert(kr_packer *p, const kr_cluster_obj *c);
int        kr_packer_cluster_delete(kr_packer *p, kr_str ns, kr_str name);
int        kr_packer_job_upsert(kr_packer *p, const kr_job_obj *j);
int        kr_packer_job_delete(kr_packer *p, kr_str ns, kr_str name);
int        kr_packer_flush(kr_packer *p, uint32_t *mode_out);
int        kr_packer_sizes(kr_packer *p, kr_sizes *out);
int        kr_packer_bufs(kr_packer *p, kr_snapshot_bufs *out);            /* the arenas the packer maintains (read-only for the caller) */
uint32_t   kr_packer_intern(kr_packer *p, kr_str s);                       /* e.g. kr_flags.id_head_not_found_reason */
int        kr_packer_string(kr_packer *p, uint32_t id, kr_str *out);
int64_t    kr_packer_cluster_row(kr_packer *p, kr_str ns, kr_str name);    /* -1: not packed */
int64_t    kr_packer_pod_row(kr_packer *p, kr_str ns, kr_str name);
int        kr_packer_pod_key(kr_packer *p, uint32_t row, kr_str *ns, kr_str *name);  /* act_pod_idx -> the Pod to delete */
/* The epoch a record belongs to: Reconcile(req) trusts the record of `req` only if its own cache read of the RayCluster shows the
 * resourceVersion packed here and no Pod event arrived since the flush (podset version) — else it takes the per-object Go path. */
int        kr_packer_epoch(kr_packer *p, uint64_t *epoch, uint64_t *podset_version);
int        kr_packer_cluster_epoch(kr_packer *p, uint32_t cluster_row, uint64_t *resource_version, uint64_t *generation);
const char *kr_packer_last_error(kr_packer *p);

/* ---- group packer: the native packer sharded over GPUs (DESIGN §6).  One kr_packer per shard behind one handle; each is created
 * on its shard's worker thread of a kr_group (NUMA-local pinned arenas), and flush / reconcile run every shard on its worker in
 * parallel, each on the single-device incremental path.
 * Routing key (namespace, RayCluster name): a RayCluster by its own name, a Pod by its ray.io/cluster label, a RayJob by its
 * cluster name; shard = kr_shard_of_key.  A Pod therefore always sits on the shard of every RayCluster its label can match
 * (common/association.go:83-130): an orphan needs no move when its RayCluster arrives, and a RayCluster deleted and re-created
 * under its name (a new UID) lands where its old Pods are.  kr_group_route / kr_group_shard_of_uid keep UID routing for the
 * global-snapshot path; a RayCluster's decisions depend only on its own objects, so the key that shards changes no result.
 * Event calls run on the caller thread (O(1) plus at most n Pod-table lookups, no hop to a worker).  A Pod whose label changed, or
 * a RayJob whose cluster name changed, is upserted on its new shard and deleted from its old one; deleting an unknown key is KR_OK.
 * kr_group_packer_shard(i) is shard i's kr_packer for reads and per-shard settings (kr_packer_string / _pod_key / _cluster_row /
 * _epoch / _intern / _set_kuberay_version, options through kr_packer_engine — they are not forwarded); kr_group_packer_group is
 * the kr_group over the shards' engines (kr_group_engine / _device / _allgather_group_results; kr_group_route / _commit /
 * _reconcile do not belong to a group packer).  On an error the first failing shard's code is returned and
 * kr_group_packer_last_error names that shard with its packer's message.  One caller thread at a time for the whole handle. */
typedef struct kr_group_packer kr_group_packer;
uint32_t   kr_shard_of_key(kr_str ns, kr_str cluster_name, uint32_t n);  /* FNV-1a 64 over ns "/" name, % n (an absent name hashes as ""); no handle, no device */
int        kr_group_packer_create(const kr_config *per_shard_capacities, const int32_t *devices, uint32_t n, kr_group_packer **out);  /* devices as kr_group_create */
void       kr_group_packer_destroy(kr_group_packer *gp);
uint32_t   kr_group_packer_size(kr_group_packer *gp);
kr_packer *kr_group_packer_shard(kr_group_packer *gp, uint32_t shard);
kr_group  *kr_group_packer_group(kr_group_packer *gp);
int        kr_group_packer_pod_upsert(kr_group_packer *gp, const kr_pod_obj *pod);
int        kr_group_packer_pod_delete(kr_group_packer *gp, kr_str ns, kr_str name);
int        kr_group_packer_cluster_upsert(kr_group_packer *gp, const kr_cluster_obj *c);
int        kr_group_packer_cluster_delete(kr_group_packer *gp, kr_str ns, kr_str name);
int        kr_group_packer_job_upsert(kr_group_packer *gp, const kr_job_obj *j);
int        kr_group_packer_job_delete(kr_group_packer *gp, kr_str ns, kr_str name);
int        kr_group_packer_flush(kr_group_packer *gp, uint32_t *modes_out /* [n], optional: each shard's kr_packer_flush mode */);
/* flags[i] for shard i (id_head_not_found_* are ids of shard i's interner: kr_packer_intern on kr_group_packer_shard(i)) */
int        kr_group_packer_reconcile(kr_group_packer *gp, const kr_flags *flags /* [n] */, kr_results_view *views /* [n] */);
const char *kr_group_packer_last_error(kr_group_packer *gp);

/* ------------------------------------------------------------------------------------------------------------------------------
 * Pod metadata builder (SURVEY §8 f3, first part): what createHeadPod / createWorkerPodWithIndex put into the new Pod's
 * ObjectMeta — the part of buildHeadPod / buildWorkerPod that depends on the engine's create tuples (group, replica index,
 * host index).  Host-side; no GPU.  Replaces, for the metadata only:
 *   utils.PodName            (controllers/ray/utils/util.go:198-215)   kr_pod_name
 *   utils.CheckName          (util.go:217-240)                          kr_check_name
 *   utils.CheckLabel         (util.go:247-265)                          kr_check_label
 *   utils.GenerateRayWorkerReplicaGroupName (util.go:375-379)           kr_pod_creates_expand (names "<group>-<5 chars>")
 *   mergeLabels + labelPod   (common/pod.go:1276-1283, 775-799)         kr_pod_meta_build
 *   replica index / name / host index labels (common/pod.go:430-439)    kr_pod_meta_build
 *   Name | GenerateName, Namespace (common/pod.go:170-178, 353-357)     kr_pod_meta_build
 *   initTemplateAnnotations, ray.io/ft-enabled, ray.io/external-storage-namespace (common/pod.go:67-75, 85-87, 105-114)
 *   ray.io/serve label for RayService-owned clusters (common/pod.go:583-588)
 *   recreate-hash + kuberay-version annotations of the head (raycluster_controller.go:1313-1316)
 *   the controller ownerReference (raycluster_controller.go:1407, 1429: controllerutil.SetControllerReference)
 * The container / env / command part of BuildPod (common/pod.go:575-760) is NOT here: it does not depend on the create tuple and
 * stays in Go (INTEGRATION.md). */
typedef struct kr_kv { kr_str key, value; } kr_kv;
enum { KR_CRD_RAYCLUSTER = 0, KR_CRD_RAYJOB = 1, KR_CRD_RAYSERVICE = 2 };  /* utils.GetCRDType(instance.Labels[ray.io/originated-from-crd]) */
typedef struct kr_podmeta_cluster {
  kr_str name, ns, uid;
  kr_str cluster_hash;            /* createHeadPod's clusterHash; absent or "": no hash / version stamps (:1313) */
  kr_str kuberay_version;         /* utils.KUBERAY_VERSION */
  kr_str storage_ns_annotation;   /* instance.Annotations[ray.io/external-storage-namespace]; p == NULL: not set */
  kr_str storage_ns_option;       /* spec.gcsFaultToleranceOptions.externalStorageNamespace; absent or "": not set */
  uint8_t overwrite_container_cmd;  /* isOverwriteRayContainerCmd(instance) (common/pod.go:62-65) */
  uint8_t ft_enabled;               /* utils.IsGCSFaultToleranceEnabled (util.go:753-756) */
  uint8_t crd_type;                 /* KR_CRD_* */
  uint8_t deterministic_head_name;  /* utils.IsDeterministicHeadPodNameEnabled() (util.go:895-897) */
  uint8_t gate_multihost_indexing;  /* features.RayMultiHostIndexing */
  uint8_t reserved[3];
} kr_podmeta_cluster;
typedef struct kr_podmeta_group {   /* HeadGroupSpec or one WorkerGroupSpec, as far as the metadata reads it */
  kr_str group_name;                /* ignored for the head ("headgroup") */
  int32_t num_of_hosts;             /* ignored for the head */
  uint32_t n_template_labels, n_group_labels, n_template_annotations;
  const kr_kv *template_labels;     /* spec.template.metadata.labels */
  const kr_kv *group_labels;        /* the group's top-level `labels` (they win, common/pod.go:1276-1283) */
  const kr_kv *template_annotations;/* spec.template.metadata.annotations */
} kr_podmeta_group;
typedef struct kr_podmeta_create {  /* one Pod to create */
  int32_t group;                    /* -1: the head; else index into the worker groups */
  int32_t replica_index, host_index;/* createWorkerPodWithIndex(..., replicaIndex, hostIndex) (:1363) */
  kr_str replica_name;              /* replicaGrpName; "" for single-host groups */
} kr_podmeta_create;

/* Each returns the length of the result (which may exceed cap: nothing is written past cap) or a negative KR_E_*; an empty
 * input to kr_check_name / kr_check_label is KR_E_INVALID (the reference indexes s[0] and panics). */
int64_t kr_pod_name(kr_str prefix, uint8_t node_type /* KR_NT_HEAD | KR_NT_WORKER */, uint8_t is_generate_name, char *out, uint64_t cap);
int64_t kr_check_name(kr_str s, char *out, uint64_t cap);
int64_t kr_check_label(kr_str s, char *out, uint64_t cap);

/* One JSON object per create, written back to back into out[]; create i owns out[off[i] .. off[i+1]).  Each object is the
 * ObjectMeta patch in Go's field order and map encoding (keys sorted, strings escaped as encoding/json does):
 *   {"name"|"generateName":…,"namespace":…,"labels":{…},"annotations":{…},"ownerReferences":[{…}]}
 * *need = bytes required; KR_E_CAPACITY when cap is too small (off[] is still filled in, so the caller can size and retry). */
int kr_pod_meta_build(const kr_podmeta_cluster *cluster, const kr_podmeta_group *head, const kr_podmeta_group *groups, uint32_t n_groups,
                      const kr_podmeta_create *creates, uint32_t n_creates, uint8_t *out, uint64_t cap, uint64_t *off, uint64_t *need);

/* Engine results -> create tuples for ONE RayCluster, in the order the reference issues the Create calls: the head first when
 * head_create != 0 (:692-699), then group by group (:869-889; multi-host :1081-1094: for every new replica index one generated
 * replica name and hosts 0..NumOfHosts-1).  group_results / groups are the cluster's n_groups rows, create_idx the engine's arena.
 * Replica names take 5 characters of the apimachinery rand.String alphabet from a splitmix64 stream seeded with `seed`; they live
 * in name_buf.  *n_out = tuples required; KR_E_CAPACITY when cap or name_cap is too small. */
int kr_pod_creates_expand(const kr_group_result *group_results, const kr_podmeta_group *groups, uint32_t n_groups, const int32_t *create_idx,
                          uint8_t head_create, uint8_t gate_multihost_indexing, uint64_t seed, kr_podmeta_create *out, uint32_t cap,
                          char *name_buf, uint64_t name_cap, uint32_t *n_out);
const char *kr_pod_meta_last_error(void);

/* `ray start` command builder (SURVEY §8 f3, second part): what DefaultHeadPodTemplate / DefaultWorkerPodTemplate and BuildPod do to a
 * group's rayStartParams and to the Ray container's command line — once per group and reconcile, it does not depend on the create
 * tuple.  Host-side; no GPU.  Replaces:
 *   updateRayStartParamsResources / updateRayStartParamsLabels   (common/pod.go:1219-1276)    KR_RS_UPDATE_RESOURCES / _LABELS
 *   setMissingRayStartParams + the head's no-monitor             (common/pod.go:935-978, 196-200)  KR_RS_SET_MISSING
 *   generateRayStartCommand, addWellKnownAcceleratorResources, convertParamMap (common/pod.go:980-1135)  KR_RS_GENERATE
 *   the container command / args assembly of BuildPod            (common/pod.go:617-650; utils.GetContainerCommand util.go:884-892)
 * (env vars, probes, volumes, GCS-FT / token-auth additions, the autoscaler sidecar and the init container: the entry points below) */
enum { KR_RS_UPDATE_RESOURCES = 1, KR_RS_UPDATE_LABELS = 2, KR_RS_SET_MISSING = 4, KR_RS_GENERATE = 8 };
typedef struct kr_raystart_in {
  uint8_t node_type;                /* KR_NT_HEAD | KR_NT_WORKER */
  uint8_t autoscaling_enabled;      /* utils.IsAutoscalingEnabled(&instance.Spec): the head gets no-monitor=true */
  uint8_t overwrite_container_cmd;  /* podTemplate annotation ray.io/overwrite-container-cmd == "true" (common/pod.go:631-634) */
  uint8_t login_shell;              /* strings.ToLower(os.Getenv("ENABLE_LOGIN_SHELL")) == "true" */
  uint32_t steps;                   /* KR_RS_* mask; 0 = all of them, in the reference's order */
  kr_str head_port;                 /* GetHeadPort(instance.Spec.HeadGroupSpec.RayStartParams); absent: "6379" */
  kr_str fqdn_ray_ip;               /* utils.GenerateFQDNServiceName(...): the worker's default address is <fqdn>:<head port> */
  const kr_kv *ray_start_params;    uint32_t n_ray_start_params;   /* the group's rayStartParams */
  const kr_kv *group_labels;        uint32_t n_group_labels;       /* the group's top-level `labels` */
  const kr_kv *group_resources;     uint32_t n_group_resources;    /* the group's top-level `resources` (name -> quantity text) */
  const kr_kv *container_limits;    uint32_t n_container_limits;   /* Ray container resources.limits (name -> quantity text) */
  const kr_kv *container_requests;  uint32_t n_container_requests; /* Ray container resources.requests */
  const kr_str *command;            uint32_t n_command;            /* Ray container command / args from the template */
  const kr_str *args;               uint32_t n_args;
} kr_raystart_in;
/* Writes one JSON object (Go map / string encoding):
 *   {"rayStartParams":{...final params, keys sorted...},"rayStartCommand":"ray start ...","generated":true|false,"command":[...],"args":[...]}
 * generated == false: the container keeps the template's command / args (overwrite annotation, or they already contain "ray start").
 * *need = bytes required; KR_E_CAPACITY when cap is too small. */
int kr_ray_start_command(const kr_raystart_in *in, uint8_t *out, uint64_t cap, uint64_t *need);
/* The environment variables BuildPod appends to the Ray container (setContainerEnvVars, common/pod.go:815-933) or to an init container
 * (setInitContainerEnvVars, :801-813), in its order: a JSON array of corev1.EnvVar in Go's encoding.  `existing` = the names the template's
 * container already carries (the "already set by the user" checks read them and everything appended so far). */
typedef struct kr_rayenv_in {
  uint8_t node_type;        /* KR_NT_HEAD | KR_NT_WORKER (ignored for an init container) */
  uint8_t crd_type;         /* KR_CRD_*: RayService clusters get three extra timeouts; the head's usage tag names the CRD */
  uint8_t init_container;   /* 1: setInitContainerEnvVars (FQ_RAY_IP, RAY_IP) */
  uint8_t reserved;
  kr_str fqdn_ray_ip, head_port, ray_start_cmd, kuberay_version;
  const kr_str *existing;       uint32_t n_existing;
  const kr_kv *default_envs;    uint32_t n_default_envs;   /* the operator configuration's DefaultContainerEnvs (name -> value) */
} kr_rayenv_in;
int kr_ray_container_env(const kr_rayenv_in *in, uint8_t *out, uint64_t cap, uint64_t *need);
/* The liveness / readiness probes BuildPod injects into the Ray container when the template has none (initLivenessAndReadinessProbe,
 * common/pod.go:477-573; ENABLE_PROBES_INJECTION is the caller's business): {"livenessProbe":{...},"readinessProbe":{...}} in corev1.Probe's
 * encoding, only the ones to inject.  Ray >= 2.53.0 (supportsUnifiedHealthCheck, :466-475) gets one HTTP check, older / unparsable versions the
 * wget commands; a RayService worker's readiness probe always adds the Serve proxy check by exec. */
typedef struct kr_rayprobe_in {
  uint8_t node_type, crd_type;                       /* KR_NT_*, KR_CRD_* */
  uint8_t has_liveness_probe, has_readiness_probe;   /* the template's Ray container already defines it: left alone */
  int32_t serving_port;                              /* utils.FindContainerPort(rayContainer, "serve", 8000); <= 0: 8000 */
  kr_str ray_version;                                /* spec.rayVersion */
  const kr_kv *ray_start_params; uint32_t n_ray_start_params;  /* dashboard-agent-listen-port / dashboard-port are read from here */
} kr_rayprobe_in;
int kr_ray_probes(const kr_rayprobe_in *in, uint8_t *out, uint64_t cap, uint64_t *need);
/* The emptyDir volumes BuildPod adds and their mounts (common/pod.go:600-615, 1137-1217): {"volumes":[..],"rayContainerVolumeMounts":[..],
 * "autoscalerVolumeMounts":[..]} — corev1.Volume / corev1.VolumeMount objects to APPEND.  /dev/shm ("shared-mem", memory medium, sizeLimit =
 * the Ray container's memory limit, else request, in resource.Quantity's canonical form) unless rayStartParams sets plasma-directory;
 * /tmp/ray ("ray-logs") on the Ray and the autoscaler container when the head runs the autoscaler sidecar.  A path already mounted or a
 * volume name already present is left alone. */
typedef struct kr_rayvol_in {
  uint8_t node_type, autoscaling_enabled, plasma_directory_set, reserved;
  kr_str memory_limit, memory_request;                                  /* Ray container resources (quantity text; absent: p == NULL) */
  const kr_str *volume_names;           uint32_t n_volume_names;          /* pod.Spec.Volumes[*].Name */
  const kr_str *ray_mount_paths;        uint32_t n_ray_mount_paths;       /* Ray container VolumeMounts[*].MountPath */
  const kr_str *autoscaler_mount_paths; uint32_t n_autoscaler_mount_paths;/* autoscaler container VolumeMounts[*].MountPath */
} kr_rayvol_in;
int kr_ray_volumes(const kr_rayvol_in *in, uint8_t *out, uint64_t cap, uint64_t *need);
/* resource.Quantity as the builder reads it: Value() (rounded up), AsApproximateFloat64(), IsZero(); KR_E_INVALID: not a quantity. */
int64_t kr_quantity_value(kr_str text, int64_t *value_out, double *approx_out, uint8_t *is_zero_out);
const char *kr_ray_start_last_error(void);

/* ------------------------------------------------------------------------------------------------------------------------------
 * Pod template surgery (SURVEY §8 f3, last part): the remaining pieces DefaultHeadPodTemplate / DefaultWorkerPodTemplate bolt onto the
 * group's template before BuildPod — once per group and reconcile; host-side, no GPU.  Fragments of corev1 objects the caller already
 * holds (an EnvVarSource, ResourceRequirements, a SecurityContext, env / envFrom / volumeMount lists) travel as RAW JSON text in Go's
 * encoding (json.Marshal on the Go side) and are spliced into the output unchanged; p == NULL, "" or "null" means absent, and "[]"
 * an empty list.  Every function writes ONE JSON document; *need = bytes required, KR_E_CAPACITY when cap is too small. */

/* configureGCSFaultTolerance (common/pod.go:77-163): {"env":[...EnvVars to APPEND to the Ray container...],"rayStartParams":{...entries
 * to SET on the head group's rayStartParams: redis-username / redis-password...}}.  The two annotations it writes are part of
 * kr_pod_meta_build.  ft_enabled == 0 gives {"env":[],"rayStartParams":{}}. */
typedef struct kr_rayft_in {
  uint8_t node_type;                 /* KR_NT_HEAD | KR_NT_WORKER */
  uint8_t ft_enabled;                /* utils.IsGCSFaultToleranceEnabled (util.go:753-756) */
  uint8_t has_options;               /* spec.gcsFaultToleranceOptions != nil */
  uint8_t has_redis_username, has_redis_password;   /* options.RedisUsername / RedisPassword != nil */
  uint8_t reserved[3];
  kr_str cluster_uid;                /* string(instance.UID): the default external storage namespace */
  kr_str storage_ns_annotation;      /* instance.Annotations[ray.io/external-storage-namespace]; p == NULL: not set */
  kr_str storage_ns_option;          /* options.ExternalStorageNamespace; absent or "": not set */
  kr_str redis_address;              /* options.RedisAddress */
  kr_str redis_username_value, redis_username_value_from;   /* RedisCredential.Value, .ValueFrom (raw EnvVarSource JSON) */
  kr_str redis_password_value, redis_password_value_from;
  kr_str head_redis_password_param;  /* head rayStartParams["redis-password"]; p == NULL: the key is absent (no-options path, :148-159) */
  const kr_str *existing;  uint32_t n_existing;    /* the Ray container's env names */
} kr_rayft_in;
int kr_ray_ft_env(const kr_rayft_in *in, uint8_t *out, uint64_t cap, uint64_t *need);

/* SetContainerTokenAuthEnvVars + AddRayTokenVolume (common/pod.go:254-335) for ONE container (the Ray container, the wait-gcs-ready init
 * container or the autoscaler sidecar): {"env":[..],"volumeMounts":[..],"volumes":[..]} — objects to APPEND to the container's env /
 * volumeMounts and to the pod's volumes (the projected service-account token, once per pod). */
typedef struct kr_rayauth_in {
  uint8_t k8s_token_auth;            /* utils.IsK8sAuthEnabled(authOptions) (util.go:763-765) */
  uint8_t reserved[3];
  kr_str cluster_name;               /* the default Secret is utils.CheckName(clusterName) */
  kr_str secret_name;                /* authOptions.SecretName; absent or "": the default */
  const kr_str *existing_env;          uint32_t n_existing_env;           /* container.Env[*].Name */
  const kr_str *existing_mount_names;  uint32_t n_existing_mount_names;   /* container.VolumeMounts[*].Name */
  const kr_str *existing_volume_names; uint32_t n_existing_volume_names;  /* podSpec.Volumes[*].Name */
} kr_rayauth_in;
int kr_ray_auth(const kr_rayauth_in *in, uint8_t *out, uint64_t cap, uint64_t *need);

/* The autoscaler sidecar of the head Pod (common/pod.go:194-220: BuildAutoscalerContainer :673-724, token auth on it, then
 * mergeAutoscalerOverrides :727-751, setAutoscalerV2EnvVars :242-251):
 *   {"container":{...corev1.Container...},"serviceAccountName":"...","rayContainerEnv":[...],"restartPolicy":"Never"|""}
 * rayContainerEnv / restartPolicy carry the autoscaler-v2 additions (empty / "" for v1).  With k8s token auth the sidecar mounts
 * "ray-token"; the volume itself comes from kr_ray_auth on the Ray container (configureTokenAuth runs later, :234-236). */
typedef struct kr_rayautoscaler_in {
  uint8_t login_shell;               /* ENABLE_LOGIN_SHELL == "true" (utils.GetContainerCommand) */
  uint8_t autoscaler_v2;             /* utils.IsAutoscalingV2Enabled(&instance.Spec) */
  uint8_t auth_enabled;              /* utils.IsAuthEnabled(&instance.Spec) */
  uint8_t k8s_token_auth;            /* utils.IsK8sAuthEnabled(authOptions) */
  uint8_t has_options;               /* spec.autoscalerOptions != nil */
  uint8_t reserved[3];
  kr_str cluster_name, secret_name;  /* as kr_rayauth_in */
  kr_str head_service_account;       /* head template spec.serviceAccountName; absent or "": the cluster's name (util.go:575-581) */
  kr_str ray_image;                  /* the Ray head container's image: the sidecar's default */
  kr_str image, image_pull_policy;   /* options.Image / ImagePullPolicy; p == NULL: not set (a set-but-empty string IS an override) */
  kr_str resources_json;             /* options.Resources (raw ResourceRequirements); absent: 500m / 512Mi */
  kr_str env_json, env_from_json, volume_mounts_json;   /* options.Env / EnvFrom / VolumeMounts (raw arrays) */
  kr_str security_context_json;      /* options.SecurityContext (raw) */
} kr_rayautoscaler_in;
int kr_ray_autoscaler_container(const kr_rayautoscaler_in *in, uint8_t *out, uint64_t cap, uint64_t *need);

/* The worker's wait-gcs-ready init container (common/pod.go:359-415; ENABLE_INIT_CONTAINER_INJECTION is the caller's business): one
 * corev1.Container.  env / volumeMounts / securityContext are the Ray container's, copied. */
typedef struct kr_rayinit_in {
  uint8_t login_shell, reserved[3];
  kr_str image, image_pull_policy;   /* the Ray container's */
  kr_str fqdn_ray_ip, head_port;
  kr_str env_json, volume_mounts_json, security_context_json;   /* the Ray container's Env / VolumeMounts / SecurityContext (raw) */
} kr_rayinit_in;
int kr_ray_init_container(const kr_rayinit_in *in, uint8_t *out, uint64_t cap, uint64_t *need);
const char *kr_ray_template_last_error(void);

/* ------------------------------------------------------------------------------------------------------------------------------
 * The whole Pod (SURVEY §8 f3, assembled): buildHeadPod / buildWorkerPod (raycluster_controller.go:1387-1433) = DefaultHeadPodTemplate /
 * DefaultWorkerPodTemplate (common/pod.go:166-239, 352-464) + BuildPod (:577-669) + the controller ownerReference, for every create
 * tuple of ONE RayCluster in one call.  Host-side; no GPU.  The container half of a manifest depends only on the group, so it is
 * built once per group and call; the ObjectMeta varies per tuple (kr_pod_meta_build).
 *   cluster_json: the RayCluster as JSON — {"metadata":{"name","namespace","uid","labels","annotations"},"spec":{...}}, keys in any
 *     order (what the API server serves, or json.Marshal(instance)).
 *   out: one corev1.Pod per create, back to back (create i owns out[off[i] .. off[i+1])):
 *     {"kind":"Pod","apiVersion":"v1","metadata":{...},"spec":{...},"status":{}} — struct fields in Go's declaration order, omitempty
 *     honoured, maps sorted, quantities canonical; it decodes into the corev1.Pod the reference hands to client.Create.
 * *need = bytes required; KR_E_CAPACITY when cap is too small (off[] is still filled in). */
typedef struct kr_podbuild_env {       /* the operator process's contribution */
  kr_str kuberay_version;              /* utils.KUBERAY_VERSION */
  kr_str cluster_domain;               /* CLUSTER_DOMAIN; absent or "": cluster.local */
  kr_str cluster_hash;                 /* createHeadPod's clusterHash (head annotations); absent or "": none */
  uint8_t deterministic_head_name;     /* utils.IsDeterministicHeadPodNameEnabled() */
  uint8_t gate_multihost_indexing;     /* features.RayMultiHostIndexing */
  uint8_t login_shell;                 /* ENABLE_LOGIN_SHELL == "true" */
  uint8_t no_init_container_injection; /* ENABLE_INIT_CONTAINER_INJECTION == "false" */
  uint8_t no_probes_injection;         /* ENABLE_PROBES_INJECTION == "false" */
  uint8_t reserved[3];
  const kr_kv *default_envs; uint32_t n_default_envs;          /* configuration DefaultContainerEnvs */
  kr_str head_sidecars_json, worker_sidecars_json;             /* configuration Head / WorkerSidecarContainers (raw []corev1.Container) */
} kr_podbuild_env;
int kr_pod_build(const uint8_t *cluster_json, uint64_t len, const kr_podbuild_env *env, const kr_podmeta_create *creates, uint32_t n_creates,
                 uint8_t *out, uint64_t cap, uint64_t *off, uint64_t *need);
const char *kr_pod_build_last_error(void);

/* Last error text for this engine (never NULL). */
const char *kr_last_error(kr_engine *e);

/* Algorithmic bytes of one pass over the committed snapshot (SURVEY §8(d): 144/cluster + 56/group + 4/wtd
 * + 33/pod + json bytes), and of the hash kernel alone (json bytes + 32/cluster). */
int kr_algorithmic_bytes(kr_engine *e, uint64_t *pass_bytes, uint64_t *hash_bytes, uint64_t *match_bytes);

#ifdef __cplusplus
}
#endif
#endif /* KR_ENGINE_H_ */

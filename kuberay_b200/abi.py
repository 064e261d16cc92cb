"""ctypes / numpy mirror of include/kr_engine.h (the C ABI of the reconcile engine).

Keep this file in lock-step with the header: tests/test_abi.py checks struct sizes and that the
built library exports every declared symbol.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

# ---------------------------------------------------------------- enums (include/kr_engine.h)
ID_ABSENT, ID_EMPTY_STRING = 0, 1

CF_SUSPEND = 1 << 0
CF_SUSPEND_SET_FALSE = 1 << 1
CF_AUTOSCALING = 1 << 2
CF_UPGRADE_RECREATE = 1 << 3
CF_SKIP_HEAD_RESTART = 1 << 4
CF_HEAD_EXPECT_OK = 1 << 5
CF_SKIP = 1 << 6
CF_ENDPOINTS_CHANGED = 1 << 7
CF_OLD_REASON_NONEMPTY = 1 << 8

SUSPEND_NONE, SUSPEND_SUSPENDING, SUSPEND_SUSPENDED = 0, 1, 2

(EXT_ERR_NONE, EXT_ERR_PLAIN, EXT_ERR_FAILED_DELETE_ALL_PODS, EXT_ERR_FAILED_DELETE_HEAD_POD,
 EXT_ERR_FAILED_CREATE_HEAD_POD, EXT_ERR_FAILED_DELETE_WORKER_POD, EXT_ERR_FAILED_CREATE_WORKER_POD,
 EXT_ERR_STATUS_ONLY_NIL) = range(8)

COND_ABSENT, COND_TRUE, COND_FALSE, COND_UNKNOWN = 0, 1, 2, 3
COND_PROVISIONED, COND_HEAD_POD_READY, COND_REPLICA_FAILURE, COND_SUSPENDING, COND_SUSPENDED = range(5)
NUM_CONDS = 5

CV_NONE, CV_PROV_ALL_READY, CV_PROV_PROVISIONING, CV_PROV_SUSPENDED, CV_CANONICAL, CV_HEAD_FROM_POD, CV_HEAD_NOT_FOUND = range(7)
CV_OTHER = 255

STATE_EMPTY, STATE_READY, STATE_FAILED, STATE_SUSPENDED, STATE_OTHER = range(5)

GF_SUSPEND = 1 << 0
GF_EXPECT_OK = 1 << 1
GF_REPLICAS_NIL = 1 << 2
GF_MIN_NIL = 1 << 3
GF_MAX_NIL = 1 << 4

PP_NODE_TYPE_SHIFT, PP_PHASE_SHIFT, PP_READY_SHIFT = 0, 2, 5
PP_RESTART_NEVER = 1 << 7
PP_RAY_TERMINATED = 1 << 8
PP_HAS_DELETION_TS = 1 << 9
PP_HAS_REPLICA_IDX = 1 << 10
PP_TOMBSTONE = 1 << 12
NT_NONE, NT_HEAD, NT_WORKER, NT_REDIS = range(4)
PHASE_EMPTY, PHASE_PENDING, PHASE_RUNNING, PHASE_SUCCEEDED, PHASE_FAILED, PHASE_UNKNOWN = range(6)

(ACT_KEEP, ACT_DELETE_ALL_SUSPEND, ACT_DELETE_ALL_RECREATE, ACT_DELETE_HEAD, ACT_DELETE_GROUP_SUSPEND,
 ACT_DELETE_UNHEALTHY, ACT_DELETE_WTD, ACT_DELETE_RANDOM, ACT_DELETE_MH_INCOMPLETE, ACT_DELETE_MH_UNHEALTHY,
 ACT_DELETE_MH_WTD, ACT_DELETE_MH_SCALE_DOWN) = range(12)
ACT_TOMBSTONE = 254
ACT_ORPHAN = 255

PATH_NORMAL, PATH_SKIPPED, PATH_SUSPENDING_DELETE_ALL, PATH_SUSPENDED_NOOP, PATH_RECREATE_DELETE_ALL = range(5)
HEAD_NONE, HEAD_EXPECT_PENDING, HEAD_DELETE, HEAD_CREATE, HEAD_SKIP_RESTART, HEAD_MULTIPLE = range(6)
(ERR_NONE, ERR_HEAD_DELETED, ERR_MULTIPLE_HEADS, ERR_UNHEALTHY_WORKERS, ERR_MH_INCOMPLETE, ERR_MH_WTD,
 ERR_MH_NOT_MULTIPLE, ERR_EXTERNAL, ERR_NEGATIVE_EXPECTED) = range(9)
SERR_NONE, SERR_MULTIPLE_HEADS, SERR_NO_HEAD_SERVICE, SERR_MULTIPLE_HEAD_SERVICES, SERR_EMPTY_SERVICE_IP = range(5)

SF_READY_BRANCH, SF_ALL_PODS_RUNNING = 1, 2

GR_PROCESSED = 1 << 0
GR_EXPECT_PENDING = 1 << 1
GR_SUSPENDED = 1 << 2
GR_MULTIHOST = 1 << 3
GR_WTD_EXECUTED = 1 << 4
GR_ABORTED = 1 << 5
GR_RANDOM_DELETE_OFF = 1 << 6
GR_CREATE_TRUNCATED = 1 << 7

ANNOT_EMPTY, ANNOT_HASH32, ANNOT_OTHER = 0, 1, 2
VER_EMPTY, VER_CURRENT, VER_DIFFERENT = 0, 1, 2
SVCIP_NORMAL, SVCIP_EMPTY, SVCIP_NONE = 0, 1, 2

PART_COLUMNS, PART_JSON, PART_ALL, PART_OBJECTS = 1, 2, 3, 4
OPT_FIXED_LAYOUT = 1
OPT_INCREMENTAL = 2
OPT_LARGE_CLUSTERS = 3
OPT_BUCKET_STRIDE = 4
OPT_WIDE_CLUSTERS = 5
OPT_HUGE_CLUSTERS = 6
OPT_WTD_EDITS = 7
OPT_SPEC_ROWS = 8
OPT_CLUSTER_CREATES = 9
OPT_CLUSTER_DELETES = 10
OPT_GROUP_EDITS = 11
OPT_LARGE_GROWTH = 12
OPT_LARGE_MOVES = 13
OPT_HUGE_GROWTH = 14
OPT_SM_COUNT = 15
OPT_BUCKET_POD_LISTS = 16
OPT_JSON_MOVES = 17
HUGE_GROW_TILES = 32
LARGE_MAX_PODS = 8192
SPEC_JSON_UNMUTED = 1
KR_OK, KR_E_INVALID, KR_E_CAPACITY, KR_E_CUDA, KR_E_STATE, KR_E_NO_DEVICE = 0, -1, -2, -3, -4, -5
MAX_KERNEL_TIMES = 24

# ---------------------------------------------------------------- snapshot columns
# (field, numpy dtype, per-row multiplicity, dimension)   — order == struct kr_snapshot_bufs
u8, u32, i32, u64 = np.uint8, np.uint32, np.int32, np.uint64
COLUMNS = [
    ("c_ns_id", u32, 1, "clusters"), ("c_name_id", u32, 1, "clusters"), ("c_uid_hash", u64, 1, "clusters"),
    ("c_flags", u32, 1, "clusters"), ("c_suspend_status", u8, 1, "clusters"), ("c_ext_err_kind", u8, 1, "clusters"),
    ("c_ext_err_msg_id", u32, 1, "clusters"), ("c_group_off", u32, 1, "clusters"), ("c_group_cnt", u32, 1, "clusters"),
    ("c_json_off", u64, 1, "clusters"), ("c_json_len", u32, 1, "clusters"),
    ("c_old_state", u8, 1, "clusters"), ("c_old_counts", i32, 5, "clusters"),
    ("c_old_cond_status", u8, 5, "clusters"), ("c_old_cond_variant", u8, 5, "clusters"),
    ("c_old_cond_reason_id", u32, 1, "clusters"), ("c_old_cond_msg_id", u32, 2, "clusters"),
    ("c_old_head_ids", u32, 4, "clusters"),
    ("c_svc_count", u8, 1, "clusters"), ("c_svc_ip_kind", u8, 1, "clusters"),
    ("c_svc_ip_id", u32, 1, "clusters"), ("c_svc_name_id", u32, 1, "clusters"),
    ("g_cluster_idx", u32, 1, "groups"), ("g_name_id", u32, 1, "groups"),
    ("g_replicas", i32, 1, "groups"), ("g_min", i32, 1, "groups"), ("g_max", i32, 1, "groups"), ("g_num_hosts", i32, 1, "groups"),
    ("g_flags", u32, 1, "groups"), ("g_wtd_off", u32, 1, "groups"), ("g_wtd_cnt", u32, 1, "groups"),
    ("w_name_id", u32, 1, "wtd"),
    ("p_ns_id", u32, 1, "pods"), ("p_cluster_name_id", u32, 1, "pods"), ("p_group_name_id", u32, 1, "pods"),
    ("p_name_id", u32, 1, "pods"), ("p_packed", u32, 1, "pods"), ("p_replica_index", i32, 1, "pods"),
    ("p_replica_name_id", u32, 1, "pods"),
    ("h_pod_idx", u32, 1, "heads"), ("h_ready_status", u8, 1, "heads"), ("h_ready_reason_id", u32, 1, "heads"),
    ("h_ready_msg_id", u32, 1, "heads"), ("h_pod_ip_id", u32, 1, "heads"), ("h_annot_state", u8, 1, "heads"),
    ("h_version_state", u8, 1, "heads"), ("h_annot_hash", u8, 32, "heads"),
    ("j_ns_id", u32, 1, "jobs"), ("j_cluster_name_id", u32, 1, "jobs"), ("j_summary_id", u32, 1, "jobs"),
    ("c_summary_id", u32, 1, "clusters"),
    ("json", u8, 1, "json"),
]
DIMS = ["clusters", "groups", "wtd", "pods", "heads", "jobs", "json"]
_CT = {np.uint8: C.c_uint8, np.uint32: C.c_uint32, np.int32: C.c_int32, np.uint64: C.c_uint64}


class kr_config(C.Structure):
    _fields_ = [("device", C.c_int32), ("max_clusters", C.c_uint32), ("max_groups", C.c_uint32), ("max_wtd", C.c_uint32),
                ("max_pods", C.c_uint32), ("max_heads", C.c_uint32), ("max_jobs", C.c_uint32), ("max_creates", C.c_uint32),
                ("max_json_bytes", C.c_uint64)]


class kr_flags(C.Structure):
    _fields_ = [("gate_status_conditions", C.c_uint8), ("gate_multihost_indexing", C.c_uint8), ("env_random_pod_delete", C.c_uint8),
                ("skip_hash", C.c_uint8), ("fetch_pod_lists", C.c_uint8), ("reserved_", C.c_uint8 * 3),
                ("id_head_not_found_reason", C.c_uint32), ("id_head_not_found_msg", C.c_uint32)]


class kr_sizes(C.Structure):
    _fields_ = [("n_clusters", C.c_uint32), ("n_groups", C.c_uint32), ("n_wtd", C.c_uint32), ("n_pods", C.c_uint32),
                ("n_heads", C.c_uint32), ("n_jobs", C.c_uint32), ("json_bytes", C.c_uint64)]


class kr_snapshot_bufs(C.Structure):
    _fields_ = [(name, C.POINTER(_CT[dt])) for (name, dt, _m, _d) in COLUMNS]


cluster_result_dtype = np.dtype([
    ("path", u8), ("head_action", u8), ("err_kind", u8), ("status_err", u8), ("new_state", u8), ("state_changed", u8),
    ("needs_status_write", u8), ("head_update_annotations", u8),
    ("stop_after_group", i32), ("err_arg", i32), ("n_pods", i32), ("n_heads", i32), ("head_pod_idx", i32),
    ("counts", i32, (5,)), ("cond_status", u8, (8,)), ("cond_variant", u8, (8,)),
    ("head_ready_reason_id", u32), ("head_ready_msg_id", u32), ("head_ids", u32, (4,)), ("pod_start", u32), ("status_flags", u32),
], align=True)
group_result_dtype = np.dtype([
    ("expected", i32), ("n_list", i32), ("n_unhealthy", i32), ("n_running", i32), ("diff", i32),
    ("n_create", u32), ("create_off", u32), ("flags", u32),
], align=True)
job_result_dtype = np.dtype([
    ("cluster_idx", i32), ("cluster_state", u8), ("not_ready", u8), ("status_changed", u8), ("reserved", u8),
], align=True)
assert cluster_result_dtype.itemsize == 96 and group_result_dtype.itemsize == 32 and job_result_dtype.itemsize == 8


class kr_results_view(C.Structure):
    _fields_ = [("clusters", C.c_void_p), ("hash", C.c_void_p), ("groups", C.c_void_p), ("wtd_pod_idx", C.c_void_p),
                ("sorted_pod_idx", C.c_void_p), ("sorted_action", C.c_void_p), ("create_idx", C.c_void_p), ("jobs", C.c_void_p),
                ("act_start", C.c_void_p), ("act_cnt", C.c_void_p), ("act_pod_idx", C.c_void_p), ("act_code", C.c_void_p),
                ("n_create_total", C.c_uint32), ("n_orphans", C.c_uint32), ("n_actions", C.c_uint32),
                ("create_extent", C.c_uint32), ("act_extent", C.c_uint32), ("n_changed", C.c_uint32), ("changed_clusters", C.c_void_p)]


class kr_str(C.Structure):
    _fields_ = [("p", C.c_char_p), ("n", C.c_uint32)]


class kr_pod_obj(C.Structure):
    _fields_ = [("ns", kr_str), ("name", kr_str), ("cluster", kr_str), ("group", kr_str), ("replica_name", kr_str), ("replica_index", kr_str),
                ("node_type", C.c_uint8), ("phase", C.c_uint8), ("ready_cond", C.c_uint8), ("restart_never", C.c_uint8), ("ray_terminated", C.c_uint8),
                ("has_deletion_ts", C.c_uint8), ("head_ready_status", C.c_uint8), ("reserved_", C.c_uint8),
                ("head_ready_reason", kr_str), ("head_ready_msg", kr_str), ("pod_ip", kr_str), ("recreate_hash", kr_str), ("kuberay_version", kr_str)]


class kr_group_obj(C.Structure):
    _fields_ = [("name", kr_str), ("replicas", C.c_int32), ("min_replicas", C.c_int32), ("max_replicas", C.c_int32), ("num_hosts", C.c_int32),
                ("flags", C.c_uint32), ("workers_to_delete", C.POINTER(kr_str)), ("n_workers_to_delete", C.c_uint32)]


class kr_cluster_obj(C.Structure):
    _fields_ = [("ns", kr_str), ("name", kr_str), ("uid", kr_str), ("resource_version", C.c_uint64), ("generation", C.c_uint64), ("flags", C.c_uint32),
                ("suspend_status", C.c_uint8), ("ext_err_kind", C.c_uint8), ("old_state", C.c_uint8), ("svc_count", C.c_uint8), ("svc_ip_kind", C.c_uint8),
                ("spec_json_verbatim", C.c_uint8), ("reserved_", C.c_uint8 * 2), ("ext_err_msg", kr_str), ("old_counts", C.c_int32 * 5), ("old_cond_status", C.c_uint8 * 5),
                ("old_cond_variant", C.c_uint8 * 5), ("reserved2_", C.c_uint8 * 6), ("old_head_ready_reason", kr_str), ("old_head_ready_msg", kr_str),
                ("old_replica_failure_msg", kr_str), ("old_head", kr_str * 4), ("svc_ip", kr_str), ("svc_name", kr_str), ("status_summary", kr_str),
                ("groups", C.POINTER(kr_group_obj)), ("n_groups", C.c_uint32), ("spec_json", C.c_char_p), ("spec_json_len", C.c_uint64)]


class kr_job_obj(C.Structure):
    _fields_ = [("ns", kr_str), ("name", kr_str), ("cluster_name", kr_str), ("status_summary", kr_str)]


PACK_POD_ROWS, PACK_FULL, PACK_OBJECT_ROWS, PACK_SPEC_ROWS, PACK_JSON_MOVES = 8, 16, 32, 64, 128


class kr_kv(C.Structure):
    _fields_ = [("key", kr_str), ("value", kr_str)]


CRD_RAYCLUSTER, CRD_RAYJOB, CRD_RAYSERVICE = 0, 1, 2


class kr_podmeta_cluster(C.Structure):
    _fields_ = [("name", kr_str), ("ns", kr_str), ("uid", kr_str), ("cluster_hash", kr_str), ("kuberay_version", kr_str),
                ("storage_ns_annotation", kr_str), ("storage_ns_option", kr_str), ("overwrite_container_cmd", C.c_uint8), ("ft_enabled", C.c_uint8),
                ("crd_type", C.c_uint8), ("deterministic_head_name", C.c_uint8), ("gate_multihost_indexing", C.c_uint8), ("reserved", C.c_uint8 * 3)]


class kr_podmeta_group(C.Structure):
    _fields_ = [("group_name", kr_str), ("num_of_hosts", C.c_int32), ("n_template_labels", C.c_uint32), ("n_group_labels", C.c_uint32),
                ("n_template_annotations", C.c_uint32), ("template_labels", C.POINTER(kr_kv)), ("group_labels", C.POINTER(kr_kv)),
                ("template_annotations", C.POINTER(kr_kv))]


class kr_raystart_in(C.Structure):
    _fields_ = [("node_type", C.c_uint8), ("autoscaling_enabled", C.c_uint8), ("overwrite_container_cmd", C.c_uint8), ("login_shell", C.c_uint8),
                ("steps", C.c_uint32), ("head_port", kr_str), ("fqdn_ray_ip", kr_str),
                ("ray_start_params", C.POINTER(kr_kv)), ("n_ray_start_params", C.c_uint32), ("group_labels", C.POINTER(kr_kv)), ("n_group_labels", C.c_uint32),
                ("group_resources", C.POINTER(kr_kv)), ("n_group_resources", C.c_uint32), ("container_limits", C.POINTER(kr_kv)), ("n_container_limits", C.c_uint32),
                ("container_requests", C.POINTER(kr_kv)), ("n_container_requests", C.c_uint32),
                ("command", C.POINTER(kr_str)), ("n_command", C.c_uint32), ("args", C.POINTER(kr_str)), ("n_args", C.c_uint32)]


RS_UPDATE_RESOURCES, RS_UPDATE_LABELS, RS_SET_MISSING, RS_GENERATE = 1, 2, 4, 8


class kr_rayvol_in(C.Structure):
    _fields_ = [("node_type", C.c_uint8), ("autoscaling_enabled", C.c_uint8), ("plasma_directory_set", C.c_uint8), ("reserved", C.c_uint8),
                ("memory_limit", kr_str), ("memory_request", kr_str), ("volume_names", C.POINTER(kr_str)), ("n_volume_names", C.c_uint32),
                ("ray_mount_paths", C.POINTER(kr_str)), ("n_ray_mount_paths", C.c_uint32), ("autoscaler_mount_paths", C.POINTER(kr_str)), ("n_autoscaler_mount_paths", C.c_uint32)]


class kr_rayft_in(C.Structure):
    _fields_ = [("node_type", C.c_uint8), ("ft_enabled", C.c_uint8), ("has_options", C.c_uint8), ("has_redis_username", C.c_uint8), ("has_redis_password", C.c_uint8),
                ("reserved", C.c_uint8 * 3), ("cluster_uid", kr_str), ("storage_ns_annotation", kr_str), ("storage_ns_option", kr_str), ("redis_address", kr_str),
                ("redis_username_value", kr_str), ("redis_username_value_from", kr_str), ("redis_password_value", kr_str), ("redis_password_value_from", kr_str),
                ("head_redis_password_param", kr_str), ("existing", C.POINTER(kr_str)), ("n_existing", C.c_uint32)]


class kr_rayauth_in(C.Structure):
    _fields_ = [("k8s_token_auth", C.c_uint8), ("reserved", C.c_uint8 * 3), ("cluster_name", kr_str), ("secret_name", kr_str),
                ("existing_env", C.POINTER(kr_str)), ("n_existing_env", C.c_uint32), ("existing_mount_names", C.POINTER(kr_str)), ("n_existing_mount_names", C.c_uint32),
                ("existing_volume_names", C.POINTER(kr_str)), ("n_existing_volume_names", C.c_uint32)]


class kr_rayautoscaler_in(C.Structure):
    _fields_ = [("login_shell", C.c_uint8), ("autoscaler_v2", C.c_uint8), ("auth_enabled", C.c_uint8), ("k8s_token_auth", C.c_uint8), ("has_options", C.c_uint8),
                ("reserved", C.c_uint8 * 3), ("cluster_name", kr_str), ("secret_name", kr_str), ("head_service_account", kr_str), ("ray_image", kr_str),
                ("image", kr_str), ("image_pull_policy", kr_str), ("resources_json", kr_str), ("env_json", kr_str), ("env_from_json", kr_str),
                ("volume_mounts_json", kr_str), ("security_context_json", kr_str)]


class kr_rayinit_in(C.Structure):
    _fields_ = [("login_shell", C.c_uint8), ("reserved", C.c_uint8 * 3), ("image", kr_str), ("image_pull_policy", kr_str), ("fqdn_ray_ip", kr_str), ("head_port", kr_str),
                ("env_json", kr_str), ("volume_mounts_json", kr_str), ("security_context_json", kr_str)]


class kr_podbuild_env(C.Structure):
    _fields_ = [("kuberay_version", kr_str), ("cluster_domain", kr_str), ("cluster_hash", kr_str), ("deterministic_head_name", C.c_uint8),
                ("gate_multihost_indexing", C.c_uint8), ("login_shell", C.c_uint8), ("no_init_container_injection", C.c_uint8), ("no_probes_injection", C.c_uint8),
                ("reserved", C.c_uint8 * 3), ("default_envs", C.POINTER(kr_kv)), ("n_default_envs", C.c_uint32), ("head_sidecars_json", kr_str), ("worker_sidecars_json", kr_str)]


class kr_rayprobe_in(C.Structure):
    _fields_ = [("node_type", C.c_uint8), ("crd_type", C.c_uint8), ("has_liveness_probe", C.c_uint8), ("has_readiness_probe", C.c_uint8),
                ("serving_port", C.c_int32), ("ray_version", kr_str), ("ray_start_params", C.POINTER(kr_kv)), ("n_ray_start_params", C.c_uint32)]


class kr_rayenv_in(C.Structure):
    _fields_ = [("node_type", C.c_uint8), ("crd_type", C.c_uint8), ("init_container", C.c_uint8), ("reserved", C.c_uint8),
                ("fqdn_ray_ip", kr_str), ("head_port", kr_str), ("ray_start_cmd", kr_str), ("kuberay_version", kr_str),
                ("existing", C.POINTER(kr_str)), ("n_existing", C.c_uint32), ("default_envs", C.POINTER(kr_kv)), ("n_default_envs", C.c_uint32)]


class kr_podmeta_create(C.Structure):
    _fields_ = [("group", C.c_int32), ("replica_index", C.c_int32), ("host_index", C.c_int32), ("replica_name", kr_str)]


class kr_hash_compare_row(C.Structure):
    _fields_ = [("goal_spec_json", C.c_char_p), ("goal_spec_len", C.c_uint64), ("cluster_hash", C.c_char_p), ("cluster_hash_len", C.c_uint32),
                ("num_worker_groups", C.c_char_p), ("num_worker_groups_len", C.c_uint32), ("partial", C.c_uint8), ("reserved_", C.c_uint8 * 7)]


class kr_profile(C.Structure):
    _fields_ = [("h2d_ms", C.c_float), ("kernels_ms", C.c_float), ("d2h_ms", C.c_float), ("n_kernels", C.c_uint32),
                ("kernel_ms", C.c_float * MAX_KERNEL_TIMES), ("kernel_name", C.c_char_p * MAX_KERNEL_TIMES),
                ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64)]


# kr_last_pass (kr_pass_report): what the last pass was and which KR_FULL_* rules kept it from being an incremental epoch
PASSK_INCREMENTAL, PASSK_FULL = 1, 2
PIPE_BUCKET, PIPE_SORT, PIPE_RADIX = 1, 2, 3
FULL_BITS = {  # name -> KR_FULL_* bit, in bit order
    "FIRST": 1 << 0, "CAPACITY": 1 << 1, "DISABLED": 1 << 2, "FLAGS": 1 << 3, "POD_LISTS": 1 << 4, "LARGE": 1 << 5, "WIDE": 1 << 6,
    "OPTION": 1 << 7, "COLUMNS": 1 << 8, "SIZES": 1 << 9, "STRUCTURAL": 1 << 10, "ROW_MAP": 1 << 11, "OVERFLOW": 1 << 12,
    "GROW_LIMIT": 1 << 13, "ARENA": 1 << 14, "EPOCH_WRAP": 1 << 15,
}
globals().update({"FULL_" + k: v for k, v in FULL_BITS.items()})


def full_names(why: int) -> list[str]:
    """The KR_FULL_* names of a why_full bit set, in bit order (an unknown bit reads as BIT<n>)."""
    names = [k for k, v in FULL_BITS.items() if why & v]
    known = sum(FULL_BITS.values())
    names += [f"BIT{i}" for i in range(32) if (why & ~known) >> i & 1]
    return names


class kr_pass_report(C.Structure):
    _fields_ = [("kind", C.c_uint8), ("pipeline", C.c_uint8), ("attempts", C.c_uint8), ("hash_wait", C.c_uint8),
                ("stride", C.c_uint32), ("why_full", C.c_uint32), ("reserved_", C.c_uint32)]


assert C.sizeof(kr_pass_report) == 16


class kr_oracle_out(C.Structure):  # oracle/kr_oracle.h (test infrastructure; declared here only for layout sharing)
    _fields_ = [("clusters", C.c_void_p), ("hash", C.c_void_p), ("groups", C.c_void_p), ("wtd_pod_idx", C.c_void_p),
                ("sorted_pod_idx", C.c_void_p), ("sorted_action", C.c_void_p), ("create_idx", C.c_void_p), ("jobs", C.c_void_p),
                ("act_start", C.c_void_p), ("act_cnt", C.c_void_p), ("act_pod_idx", C.c_void_p), ("act_code", C.c_void_p),
                ("create_cap", C.c_uint32), ("n_create_total", C.c_uint32), ("n_orphans", C.c_uint32), ("n_actions", C.c_uint32)]


# every symbol include/kr_engine.h declares
ENGINE_SYMBOLS = [
    "kr_device_count", "kr_engine_create", "kr_engine_destroy", "kr_snapshot_begin", "kr_snapshot_commit", "kr_snapshot_commit_parts", "kr_snapshot_commit_pod_rows", "kr_snapshot_commit_pod_values", "kr_snapshot_commit_object_rows", "kr_snapshot_commit_spec_rows", "kr_snapshot_commit_json_moves", "kr_engine_set_option", "kr_engine_get_option",
    "kr_reconcile_batch", "kr_reconcile_device_only", "kr_reconcile_batch_profiled", "kr_results_fetch",
    "kr_hash_batch", "kr_last_profile", "kr_last_pass", "kr_group_results_device", "kr_group_results_copy", "kr_last_error", "kr_algorithmic_bytes",
    "kr_spec_json_emit", "kr_spec_json_emit_arena", "kr_quantity_canonical", "kr_spec_json_last_error", "kr_hash_compare_batch",
    "kr_group_create", "kr_group_destroy", "kr_group_size", "kr_group_engine", "kr_group_device", "kr_group_shard_of_uid", "kr_group_route",
    "kr_group_commit", "kr_group_reconcile", "kr_group_allgather_group_results", "kr_group_last_error",
    "kr_packer_create", "kr_packer_destroy", "kr_packer_engine", "kr_packer_set_kuberay_version", "kr_packer_pod_upsert", "kr_packer_pod_delete",
    "kr_packer_cluster_upsert", "kr_packer_cluster_delete", "kr_packer_job_upsert", "kr_packer_job_delete", "kr_packer_flush", "kr_packer_sizes", "kr_packer_bufs",
    "kr_packer_intern", "kr_packer_string", "kr_packer_cluster_row", "kr_packer_pod_row", "kr_packer_pod_key", "kr_packer_epoch",
    "kr_packer_cluster_epoch", "kr_packer_last_error",
    "kr_shard_of_key", "kr_group_packer_create", "kr_group_packer_destroy", "kr_group_packer_size", "kr_group_packer_pod_upsert",
    "kr_group_packer_pod_delete", "kr_group_packer_cluster_upsert", "kr_group_packer_cluster_delete", "kr_group_packer_job_upsert",
    "kr_group_packer_job_delete", "kr_group_packer_flush", "kr_group_packer_reconcile", "kr_group_packer_last_error",
    "kr_pod_name", "kr_check_name", "kr_check_label", "kr_pod_meta_build", "kr_pod_creates_expand", "kr_pod_meta_last_error",
    "kr_ray_start_command", "kr_ray_container_env", "kr_ray_probes", "kr_ray_volumes", "kr_quantity_value", "kr_ray_start_last_error",
    "kr_pod_build", "kr_pod_build_last_error", "kr_ray_ft_env", "kr_ray_auth", "kr_ray_autoscaler_container", "kr_ray_init_container", "kr_ray_template_last_error",
]

# declared with a handle return type (kr_packer * / kr_group *): exported as well
ENGINE_HANDLE_SYMBOLS = ["kr_group_packer_shard", "kr_group_packer_group"]


def default_flags(**kw) -> kr_flags:
    """Process-level switches at their reference defaults (pkg/features/features.go:56-62; env unset)."""
    f = kr_flags()
    f.gate_status_conditions = 1
    f.gate_multihost_indexing = 1
    f.env_random_pod_delete = 0
    f.skip_hash = 0
    f.fetch_pod_lists = 1
    f.id_head_not_found_reason = 0
    f.id_head_not_found_msg = 0
    for k, v in kw.items():
        setattr(f, k, v)
    return f


class Results:
    """Owned numpy copy of one pass's results (engine or oracle) — same fields as kr_results_view."""

    FIELDS = ["clusters", "hash", "groups", "wtd_pod_idx", "sorted_pod_idx", "sorted_action", "create_idx", "jobs",
              "act_start", "act_cnt", "act_pod_idx", "act_code"]

    def __init__(self, sizes: kr_sizes, create_cap: int):
        self.clusters = np.zeros(sizes.n_clusters, dtype=cluster_result_dtype)
        self.hash = np.zeros((sizes.n_clusters, 32), dtype=np.uint8)
        self.groups = np.zeros(sizes.n_groups, dtype=group_result_dtype)
        self.wtd_pod_idx = np.zeros(sizes.n_wtd, dtype=np.int32)
        self.sorted_pod_idx = np.zeros(sizes.n_pods, dtype=np.uint32)
        self.sorted_action = np.zeros(sizes.n_pods, dtype=np.uint8)
        self.create_idx = np.zeros(max(create_cap, 1), dtype=np.int32)
        self.jobs = np.zeros(sizes.n_jobs, dtype=job_result_dtype)
        self.act_start = np.zeros(sizes.n_clusters + 1, dtype=np.uint32)
        self.act_cnt = np.zeros(sizes.n_clusters, dtype=np.uint32)
        self.act_pod_idx = np.zeros(max(sizes.n_pods, 1), dtype=np.uint32)
        self.act_code = np.zeros(max(sizes.n_pods, 1), dtype=np.uint8)
        self.n_create_total = 0
        self.n_orphans = 0
        self.n_actions = 0
        self.n_changed = sizes.n_clusters   # records recomputed by the pass (engine: fewer after an incremental epoch)
        self.changed_clusters = None

    def hash_strings(self):
        return [bytes(r).decode("ascii", "replace") for r in self.hash]

    def actions_of(self, c: int):
        """(pod idx, action) pairs of cluster c, List order."""
        a, n = int(self.act_start[c]), int(self.act_cnt[c])
        return self.act_pod_idx[a:a + n], self.act_code[a:a + n]

    def creates_of(self, g: int):
        a, n = int(self.groups["create_off"][g]), int(self.groups["n_create"][g])
        return self.create_idx[a:a + n]

    def diff(self, other: "Results") -> list[str]:
        """Field-by-field comparison; returns human-readable mismatches (empty == bit-exact parity).

        The two variable-length arenas (action list, replica indices) are compared owner by owner through their
        (offset, count) pairs: the engine may leave reserved-but-unused places in them (kr_results_view docs), so raw offsets
        are layout, not results.  pod_start / sorted_* only mean something when the full pod lists were fetched."""
        out = []
        for k in ("n_create_total", "n_orphans", "n_actions"):
            if getattr(self, k) != getattr(other, k):
                out.append(f"{k}: {getattr(self, k)} != {getattr(other, k)}")
        lists = self.sorted_pod_idx.size != 0 and other.sorted_pod_idx.size != 0
        for name in self.FIELDS:
            a, b = getattr(self, name), getattr(other, name)
            if name in ("create_idx", "act_pod_idx", "act_code", "act_start"):
                continue  # compared through their owners below
            if name in ("sorted_pod_idx", "sorted_action") and not lists:
                continue  # one side did not fetch the full pod lists (kr_flags.fetch_pod_lists == 0)
            if a.shape != b.shape:
                out.append(f"{name}: shape {a.shape} != {b.shape}")
                continue
            if a.dtype.names:
                for fld in a.dtype.names:
                    if fld == "reserved" or fld == "create_off" or (fld == "pod_start" and not lists):
                        continue
                    neq = a[fld] != b[fld]
                    if neq.ndim > 1:
                        neq = neq.any(axis=tuple(range(1, neq.ndim)))
                    if neq.any():
                        i = int(np.flatnonzero(neq)[0])
                        out.append(f"{name}.{fld}: {int(neq.sum())} rows differ, first at [{i}]: {a[fld][i]} != {b[fld][i]}")
            else:
                neq = a != b
                if neq.ndim > 1:
                    neq = neq.any(axis=1)
                if neq.any():
                    i = int(np.flatnonzero(neq)[0])
                    out.append(f"{name}: {int(neq.sum())} entries differ, first at [{i}]: {a[i]} != {b[i]}")
        if self.act_cnt.shape == other.act_cnt.shape and not (self.act_cnt != other.act_cnt).any():
            sa, sb = _gather_owned(self.act_start[:-1], self.act_cnt), _gather_owned(other.act_start[:-1], other.act_cnt)
            for res, idx in ((self, sa), (other, sb)):
                if np.unique(idx).size != idx.size or (idx.size and int(idx.max()) >= res.act_pod_idx.size):
                    out.append("act_start / act_cnt: two clusters' runs overlap or leave the list")
            for name in ("act_pod_idx", "act_code"):
                neq = getattr(self, name)[sa] != getattr(other, name)[sb]
                if neq.any():
                    i = int(np.flatnonzero(neq)[0])
                    out.append(f"{name}: {int(neq.sum())} entries differ, first at action #{i}: {getattr(self, name)[sa][i]} != {getattr(other, name)[sb][i]}")
        if self.groups.shape == other.groups.shape and not (self.groups["n_create"] != other.groups["n_create"]).any():
            sa, sb = _gather_owned(self.groups["create_off"], self.groups["n_create"]), _gather_owned(other.groups["create_off"], other.groups["n_create"])
            bad = False
            for res, idx in ((self, sa), (other, sb)):
                if np.unique(idx).size != idx.size or (idx.size and int(idx.max()) >= res.create_idx.size):
                    out.append("create_off / n_create: two groups' runs overlap or leave the list")
                    bad = True
            neq = np.zeros(0, dtype=bool) if bad else self.create_idx[sa] != other.create_idx[sb]
            if neq.any():
                i = int(np.flatnonzero(neq)[0])
                out.append(f"create_idx: {int(neq.sum())} entries differ, first at create #{i}: {self.create_idx[sa][i]} != {other.create_idx[sb][i]}")
        return out


def _gather_owned(start: np.ndarray, cnt: np.ndarray) -> np.ndarray:
    """Indices [start[i], start[i] + cnt[i]) of every owner i, concatenated in owner order."""
    cnt = cnt.astype(np.int64)
    tot = int(cnt.sum())
    if tot == 0:
        return np.zeros(0, dtype=np.int64)
    owner = np.repeat(np.arange(cnt.size), cnt)
    first = np.cumsum(cnt) - cnt
    return start.astype(np.int64)[owner] + (np.arange(tot) - first[owner])

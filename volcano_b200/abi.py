"""ctypes mirror of include/vcalloc.h (the C ABI of libvcalloc.so).

Only plain C types cross this boundary; numpy arrays are passed as host pointers.
A `Snapshot` (volcano_b200.snapshot) owns the numpy arrays and builds these structs.
"""
from __future__ import annotations

import ctypes as C

VC_ABI_VERSION = 7
VC_MAX_DIMS = 16
VC_MAX_KDIMS = 4
VC_MAX_WORDS = 4
VC_MAX_TERMS = 4
VC_MAX_PLUGINS = 16
VC_MAX_JOB_ROLES = 64
VC_MAX_TIERS = 8

VC_OK = 0
VC_EINVAL = -1
VC_ENODEV = -2
VC_ECUDA = -3
VC_EUNSUPPORTED = -4
VC_ENOMEM = -5

VC_NODE_UNSCHEDULABLE = 1
VC_CLASS_REVOCABLE = 1
VC_CLASS_TOLERATES_UNSCHEDULABLE = 2
VC_JOB_PENDING_PHASE = 1
VC_JOB_PREEMPTABLE = 2
VC_JOB_UNSUPPORTED = 4
VC_ROLE_EMPTY_NAME = 1
VC_ROLE_IN_MIN_MAP = 2
VC_QUEUE_OPEN = 1
VC_QUEUE_NOT_RECLAIMABLE = 2
VC_RES_HAS_ANY = 0x80000000

VC_PLUGIN_PRIORITY = 1
VC_PLUGIN_GANG = 2
VC_PLUGIN_DRF = 3
VC_PLUGIN_PROPORTION = 4
VC_PLUGIN_PREDICATES = 5
VC_PLUGIN_NODEORDER = 6
VC_PLUGIN_BINPACK = 7
VC_PLUGIN_TDM = 8
VC_PLUGIN_NETWORK_TOPOLOGY_AWARE = 9
VC_PLUGIN_CONFORMANCE = 10
VC_PLUGIN_PDB = 11
VC_PLUGIN_CDP = 12
VC_PLUGIN_OTHER = 99
PLUGIN_IDS = {
    "priority": VC_PLUGIN_PRIORITY,
    "gang": VC_PLUGIN_GANG,
    "drf": VC_PLUGIN_DRF,
    "proportion": VC_PLUGIN_PROPORTION,
    "predicates": VC_PLUGIN_PREDICATES,
    "nodeorder": VC_PLUGIN_NODEORDER,
    "binpack": VC_PLUGIN_BINPACK,
    "tdm": VC_PLUGIN_TDM,
    "network-topology-aware": VC_PLUGIN_NETWORK_TOPOLOGY_AWARE,
    "conformance": VC_PLUGIN_CONFORMANCE,
    "pdb": VC_PLUGIN_PDB,
    "cdp": VC_PLUGIN_CDP,
}

VC_EN_JOB_ORDER = 0x001
VC_EN_JOB_READY = 0x002
VC_EN_JOB_PIPELINED = 0x004
VC_EN_TASK_ORDER = 0x008
VC_EN_QUEUE_ORDER = 0x010
VC_EN_PREDICATE = 0x020
VC_EN_NODE_ORDER = 0x040
VC_EN_BEST_NODE = 0x080
VC_EN_OVERUSED = 0x100
VC_EN_ALLOCATABLE = 0x200
VC_EN_PREEMPTABLE = 0x400
VC_EN_RECLAIMABLE = 0x800
VC_EN_JOB_STARVING = 0x1000
VC_EN_PREEMPTIVE = 0x2000
VC_EN_ALL = 0x3FFF
# conf.PluginOption field name -> flag (conf/scheduler_conf.go:60-107)
ENABLE_FLAGS = {
    "EnabledJobOrder": VC_EN_JOB_ORDER,
    "EnabledJobReady": VC_EN_JOB_READY,
    "EnabledJobPipelined": VC_EN_JOB_PIPELINED,
    "EnabledTaskOrder": VC_EN_TASK_ORDER,
    "EnabledQueueOrder": VC_EN_QUEUE_ORDER,
    "EnabledPredicate": VC_EN_PREDICATE,
    "EnabledNodeOrder": VC_EN_NODE_ORDER,
    "EnabledBestNode": VC_EN_BEST_NODE,
    "EnabledOverused": VC_EN_OVERUSED,
    "EnabledAllocatable": VC_EN_ALLOCATABLE,
    "EnabledPreemptable": VC_EN_PREEMPTABLE,
    "EnabledReclaimable": VC_EN_RECLAIMABLE,
    "EnabledJobStarving": VC_EN_JOB_STARVING,
    "EnablePreemptive": VC_EN_PREEMPTIVE,
}

VC_PRED_NODE_AFFINITY = 1
VC_PRED_TAINT_TOLERATION = 2

VC_OP_ALLOCATE = 0
VC_OP_PIPELINE = 1
VC_OP_EVICT = 2
VC_COMM_HANDLE_BYTES = 64
VC_RT_PREEMPTABLE, VC_RT_RUNNING, VC_RT_BOUND, VC_RT_BEST_EFFORT, VC_RT_CRITICAL = 1, 2, 4, 8, 16
VC_TASK_PREEMPT_NEVER = 1
VC_VISIT_COMMIT = 0
VC_VISIT_KEEP = 1
VC_VISIT_DISCARD = 2

_dp = C.POINTER(C.c_double)
_i32p = C.POINTER(C.c_int32)
_i64p = C.POINTER(C.c_int64)
_u32p = C.POINTER(C.c_uint32)
_u64p = C.POINTER(C.c_uint64)
_u8p = C.POINTER(C.c_uint8)


class vc_dims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "n_nodes", "n_tasks", "n_jobs", "n_queues", "n_classes", "n_roles", "n_dims", "n_kdims",
        "label_words", "taint_words", "n_zones", "pods_dim")]


class vc_nodes(C.Structure):
    _fields_ = [
        ("allocatable", _dp), ("idle", _dp), ("used", _dp), ("releasing", _dp), ("pipelined", _dp),
        ("k8s_allocatable", _dp), ("k8s_requested", _dp), ("k8s_nonzero_requested", _dp),
        ("max_tasks", _i32p), ("pod_count", _i32p),
        ("label_bits", _u64p), ("taint_hard", _u64p), ("taint_soft", _u64p),
        ("flags", _u32p), ("revocable_zone", _i32p), ("zone_active", _u8p),
    ]


class vc_tasks(C.Structure):
    _fields_ = [
        ("resreq", _dp), ("req_has", _u32p), ("k8s_req", _dp), ("k8s_nonzero_req", _dp),
        ("job", _i32p), ("klass", _i32p), ("role", _i32p), ("priority", _i32p),
        ("pod_index", _i64p), ("creation_ts", _i64p), ("uid_rank", _u32p),
    ]


class vc_classes(C.Structure):
    _fields_ = [
        ("selector", _u64p), ("n_affinity", _i32p), ("affinity", _u64p),
        ("tolerated_hard", _u64p), ("tolerated_soft", _u64p),
        ("n_preferred", _i32p), ("preferred", _u64p), ("preferred_weight", _i32p), ("flags", _u32p),
    ]


class vc_jobs(C.Structure):
    _fields_ = [
        ("queue", _i32p), ("min_available", _i32p), ("priority", _i32p), ("creation_ts", _i64p),
        ("uid_rank", _u32p), ("flags", _u32p), ("n_tasks_total", _i32p), ("ready_num", _i32p),
        ("waiting_num", _i32p), ("pending_besteffort", _i32p), ("valid_num", _i32p),
        ("task_min_total", _i32p), ("role_off", _i32p), ("allocated", _dp),
        ("role_min", _i32p), ("role_occupied", _i32p), ("role_pipelined", _i32p),
        ("role_pending_other", _i32p), ("role_valid", _i32p), ("role_flags", _u32p),
    ]


class vc_queues(C.Structure):
    _fields_ = [
        ("weight", _i32p), ("priority", _i32p), ("creation_ts", _i64p), ("uid_rank", _u32p), ("flags", _u32p),
        ("capability", _dp), ("capability_has", _u32p), ("guarantee", _dp), ("guarantee_has", _u32p),
        ("allocated", _dp), ("request", _dp), ("request_has", _u32p), ("allocated_has", _u32p),
    ]


class vc_plugin_option(C.Structure):
    _fields_ = [("plugin", C.c_int32), ("tier", C.c_int32), ("enabled", C.c_uint32)]


class vc_conf(C.Structure):
    _fields_ = [
        ("n_plugins", C.c_int32),
        ("plugins", vc_plugin_option * VC_MAX_PLUGINS),
        ("binpack_weight", C.c_int32),
        ("binpack_dim_weight", C.c_int32 * VC_MAX_DIMS),
        ("w_least", C.c_int32), ("w_most", C.c_int32), ("w_balanced", C.c_int32),
        ("w_node_affinity", C.c_int32), ("w_taint_toleration", C.c_int32),
        ("kdim_dim", C.c_int32 * VC_MAX_KDIMS),
        ("predicates_enable", C.c_uint32),
        ("enable_predicate_error_cache", C.c_int32),
        ("enqueue_action_enabled", C.c_int32),
        ("percentage_nodes_to_find", C.c_int32),
        ("min_nodes_to_find", C.c_int32),
        ("min_percentage_nodes_to_find", C.c_int32),
        ("last_processed_node_index", C.c_int32),
        ("nta_weight", C.c_int32),
        ("nta_dim_weight", C.c_int32 * VC_MAX_DIMS),
        ("nta_normal_pod_enable", C.c_int32),
        ("nta_fading", C.c_double),
    ]


class vc_hypernodes(C.Structure):
    _fields_ = [("n_hypernodes", C.c_int32), ("min_tier", C.c_int32), ("max_tier", C.c_int32),
                ("member", C.POINTER(C.c_int32)), ("tier", C.POINTER(C.c_int32)), ("parent", C.POINTER(C.c_int32)),
                ("job_soft", C.POINTER(C.c_uint8)), ("job_allocated", C.POINTER(C.c_int32)),
                ("job_placed_off", C.POINTER(C.c_int32)), ("job_placed_node", C.POINTER(C.c_int32))]


class vc_hdrf(C.Structure):
    _fields_ = [("path_off", _i32p), ("path_name", _i32p), ("n_weights", _i32p), ("weight", _dp),
                ("job_request", _dp)]


class vc_running_tasks(C.Structure):
    _fields_ = [("n_tasks", C.c_int32), ("node", _i32p), ("job", _i32p), ("role", _i32p), ("priority", _i32p),
                ("pod_index", _i64p), ("creation_ts", _i64p), ("uid_rank", C.POINTER(C.c_uint32)), ("resreq", _dp),
                ("req_has", C.POINTER(C.c_uint32)), ("k8s_req", _dp), ("k8s_nonzero_req", _dp),
                ("flags", C.POINTER(C.c_uint32))]


VC_START_TIME_UNSET = -(2 ** 63)


class vc_preempt_options(C.Structure):
    _fields_ = [("topology_aware", C.c_int32), ("min_candidate_nodes_percentage", C.c_int32),
                ("min_candidate_nodes_absolute", C.c_int32), ("max_candidate_nodes_absolute", C.c_int32),
                ("offset_seed", C.c_uint64), ("now_ns", C.c_int64), ("n_running", C.c_int32),
                ("rt_pod_priority", _i32p), ("rt_start_ns", _i64p)]


VC_COOLDOWN_NONE = -(2 ** 63)
VC_GUARD_NO_LABELS = 1


class vc_victim_guards(C.Structure):
    _fields_ = [("n_running", C.c_int32), ("n_pdb", C.c_int32), ("pdb_allowed", _i32p), ("rt_pdb_off", _i32p),
                ("rt_pdb", _i32p), ("rt_flags", _u32p), ("rt_cooldown_until_ns", _i64p), ("now_ns", C.c_int64)]


class vc_decision(C.Structure):
    _fields_ = [("task", C.c_int32), ("node", C.c_int32), ("kind", C.c_int32), ("visit", C.c_int32),
                ("score", C.c_double)]


class vc_visit(C.Structure):
    _fields_ = [("job", C.c_int32), ("outcome", C.c_int32), ("first_op", C.c_int32), ("n_ops", C.c_int32)]


VC_KERNEL_GENERAL, VC_KERNEL_INCREMENTAL = 0, 1


class vc_stats(C.Structure):
    _fields_ = [("upload_ms", C.c_double), ("commit_ms", C.c_double), ("download_ms", C.c_double),
                ("total_ms", C.c_double), ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64),
                ("kernel_launches", C.c_int32), ("n_steps", C.c_int32), ("prof_cycles", C.c_int64 * 8),
                ("last_processed_node_index", C.c_int32), ("commit_kernel", C.c_int32),
                ("group_reentry", C.c_int32 * 4)]


# every symbol include/vcalloc.h declares: name -> (restype, argtypes)
_vp = C.c_void_p
SYMBOLS = {
    "vc_abi_version": (C.c_int, []),
    "vc_last_error": (C.c_char_p, []),
    "vc_init": (C.c_int, [C.c_int]),
    "vc_debug_option": (C.c_int, [C.c_char_p, C.c_int]),
    "vc_snapshot_create": (C.c_int, [C.POINTER(vc_dims), C.POINTER(_vp)]),
    "vc_snapshot_destroy": (None, [_vp]),
    "vc_snapshot_upload": (C.c_int, [_vp, C.POINTER(vc_nodes), C.POINTER(vc_tasks), C.POINTER(vc_classes),
                                     C.POINTER(vc_jobs), C.POINTER(vc_queues), C.POINTER(vc_conf)]),
    "vc_snapshot_update_nodes": (C.c_int, [_vp, C.c_int32, _i32p, C.POINTER(vc_nodes)]),
    "vc_snapshot_set_topology": (C.c_int, [_vp, C.POINTER(vc_hypernodes)]),
    "vc_snapshot_set_hdrf": (C.c_int, [_vp, C.POINTER(vc_hdrf)]),
    "vc_snapshot_set_backfill": (C.c_int, [_vp, C.c_int32, C.POINTER(vc_tasks)]),
    "vc_snapshot_set_running": (C.c_int, [_vp, C.POINTER(vc_running_tasks), C.POINTER(C.c_uint32)]),
    "vc_snapshot_set_nominated": (C.c_int, [_vp, C.POINTER(C.c_int32)]),
    "vc_snapshot_set_preempt_options": (C.c_int, [_vp, C.POINTER(vc_preempt_options)]),
    "vc_snapshot_set_victim_guards": (C.c_int, [_vp, C.POINTER(vc_victim_guards)]),
    "vc_comm_create": (C.c_int, [_vp, C.c_int, C.c_int, C.c_void_p]),
    "vc_comm_attach": (C.c_int, [_vp, C.c_void_p]),
    "vc_comm_prepare": (C.c_int, [_vp]),
    "vc_snapshot_set_shard": (C.c_int, [_vp, C.c_int32, C.c_int32]),
    "vc_allocate_run": (C.c_int, [_vp, C.POINTER(_vp)]),
    "vc_backfill_run": (C.c_int, [_vp, C.POINTER(_vp)]),
    "vc_preempt_run": (C.c_int, [_vp, C.POINTER(_vp)]),
    "vc_reclaim_run": (C.c_int, [_vp, C.POINTER(_vp)]),
    "vc_score_matrix": (C.c_int, [_vp, _u64p, _dp, _dp, _i32p]),
    "vc_score_matrix_device": (C.c_int, [_vp, C.c_int, _dp, _i64p]),
    "vc_dense_begin": (C.c_int, [_vp]),
    "vc_dense_stats": (C.c_int, [_vp, C.POINTER(_i32p), C.POINTER(C.c_int32)]),
    "vc_dense_finish": (C.c_int, [_vp, C.c_int]),
    "vc_dense_best": (C.c_int, [_vp, C.POINTER(_dp), C.POINTER(_i32p)]),
    "vc_dense_fetch": (C.c_int, [_vp, _u64p, _dp, _dp, _i32p]),
    "vc_queue_deserved": (C.c_int, [_vp, _dp, _dp]),
    "vc_result_num_decisions": (C.c_size_t, [_vp]),
    "vc_result_decisions": (C.POINTER(vc_decision), [_vp]),
    "vc_result_num_visits": (C.c_size_t, [_vp]),
    "vc_result_visits": (C.POINTER(vc_visit), [_vp]),
    "vc_result_num_fit_errors": (C.c_size_t, [_vp]),
    "vc_result_fit_errors": (_i32p, [_vp]),
    "vc_result_stats": (C.POINTER(vc_stats), [_vp]),
    "vc_result_job_allocated_hypernodes": (_i32p, [_vp, C.POINTER(C.c_size_t)]),
    "vc_result_free": (None, [_vp]),
}


def bind(lib: C.CDLL, symbols=SYMBOLS) -> C.CDLL:
    """Attach restype/argtypes; raises AttributeError if the library lacks a symbol."""
    for name, (res, args) in symbols.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib

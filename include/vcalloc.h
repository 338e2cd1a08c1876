/*
 * vcalloc.h — C ABI of libvcalloc.so: the GPU-native replacement for Volcano's
 * per-cycle `allocate` hot path.
 *
 * Every entry point below is what a cgo shim inside the reference would bind
 * (INTEGRATION.md shows the shim).  Citations are into volcano's pkg/scheduler
 * unless a full path is given.
 *
 *   reference interface replaced                         entry point here
 *   ---------------------------------------------------  ---------------------------
 *   framework.OpenSession  (framework/framework.go:34,   vc_snapshot_create +
 *     framework/session.go:166-282: Snapshot -> Session)   vc_snapshot_upload
 *   Action.Execute for "allocate"                        vc_allocate_run
 *     (actions/allocate/allocate.go:122-140, :283-348,
 *      :558-694, :709-824; framework/interface.go:41-51)
 *   Action.Execute for "backfill"                        vc_snapshot_set_backfill +
 *     (actions/backfill/backfill.go:58-116, :118-199)      vc_backfill_run
 *   Action.Execute for "preempt"                         vc_snapshot_set_running +
 *     (actions/preempt/preempt.go:101-434)                 vc_preempt_run
 *   Action.Execute for "reclaim"                         vc_snapshot_set_running +
 *     (actions/reclaim/reclaim.go:56-258)                  vc_reclaim_run
 *   util.PredicateNodes + util.PrioritizeNodes for one    vc_score_matrix
 *     task over []*NodeInfo, i.e. what a PredicateFn /
 *     BatchNodeOrderFn / BestNodeFn plugin would serve
 *     (util/predicate_helper.go:43-140,
 *      util/scheduler_helper.go:76-138,191-206;
 *      framework/session_plugins.go:70-108)
 *   Statement operations the shim replays through          vc_result_* accessors
 *     Statement.Allocate/Pipeline/Commit/Discard
 *     (framework/statement.go:146-412)
 *   CloseSession (framework/framework.go:61-69)           vc_result_free / vc_snapshot_destroy
 *
 * Conventions: plain C types only; every pointer in an input struct is HOST memory
 * owned by the caller and is copied during the call (pinned staging inside); return 0 on
 * success or a negative VC_E* code, with vc_last_error() giving the message for the
 * calling thread; no callbacks; results are library-owned until vc_result_free.
 * There is NO CPU fallback: without a CUDA device vc_init fails with VC_ENODEV.
 *
 * Layout conventions ("SoA"): resource vectors are dimension-major double arrays,
 * X[d * count + i] for dimension d of entity i.  Dimension 0 = cpu (milli), 1 = memory
 * (bytes), 2.. = scalar resources sorted by name (milli units, except "pods" = count) —
 * the units of api.NewResource (api/resource_info.go:86-127).  All values are
 * integer-valued doubles exactly as in the reference (Appendix A-2 of SURVEY.md).
 */
#ifndef VCALLOC_H
#define VCALLOC_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VC_ABI_VERSION 7
#define VC_MAX_DIMS 16   /* R  */
#define VC_MAX_KDIMS 4   /* dims seen by the upstream kube-scheduler scorers (cpu, memory, nvidia.com/gpu, ...) */
#define VC_MAX_WORDS 4   /* 64-bit words per label / taint bitset */
#define VC_MAX_TERMS 4   /* required-affinity terms and preferred-affinity terms per class */
#define VC_MAX_PLUGINS 16
#define VC_MAX_JOB_ROLES 64
#define VC_MAX_TIERS 8   /* HyperNode tiers incl. the cluster top tier */

/* error codes */
#define VC_OK 0
#define VC_EINVAL (-1)       /* malformed input (message in vc_last_error) */
#define VC_ENODEV (-2)       /* no CUDA device / extension unusable: the product has no CPU path */
#define VC_ECUDA (-3)        /* CUDA runtime error */
#define VC_EUNSUPPORTED (-4) /* snapshot uses a feature outside the hot-path scope (see DESIGN.md) */
#define VC_ENOMEM (-5)

/* ---- sizes ------------------------------------------------------------------------ */
typedef struct vc_dims {
  int32_t n_nodes;     /* N: len(ssn.NodeList), NodeList order (framework/session.go:237) */
  int32_t n_tasks;     /* T: Pending, non-BestEffort, non-gated tasks (allocate.go:255-271) */
  int32_t n_jobs;      /* J: len(ssn.Jobs) */
  int32_t n_queues;    /* Q: len(ssn.Queues) */
  int32_t n_classes;   /* C: distinct (nodeSelector, affinity, tolerations, revocable) tuples */
  int32_t n_roles;     /* total rows of the per-job role tables (vc_jobs.role_off[J]) */
  int32_t n_dims;      /* R */
  int32_t n_kdims;     /* K <= VC_MAX_KDIMS; kdim 0 = cpu, 1 = memory */
  int32_t label_words; /* Wl */
  int32_t taint_words; /* Wt */
  int32_t n_zones;     /* tdm revocable zones */
  int32_t pods_dim;    /* index of the "pods" scalar in [2,R) or -1 (api/resource_info.go:219) */
} vc_dims;

/* ---- api.NodeInfo (api/node_info.go:51-100) ---------------------------------------- */
#define VC_NODE_UNSCHEDULABLE 1u /* node.Spec.Unschedulable (upstream NodeUnschedulable filter) */
typedef struct vc_nodes {
  const double *allocatable;           /* [R][N] NodeInfo.Allocatable */
  const double *idle;                  /* [R][N] NodeInfo.Idle */
  const double *used;                  /* [R][N] NodeInfo.Used */
  const double *releasing;             /* [R][N] NodeInfo.Releasing */
  const double *pipelined;             /* [R][N] NodeInfo.Pipelined */
  const double *k8s_allocatable;       /* [K][N] k8s NodeInfo.Allocatable in upstream units (cpu milli, memory
                                          bytes, extended resources as plain counts) */
  const double *k8s_requested;         /* [K][N] k8s NodeInfo.Requested of ssn.NodeMap (framework/util.go:226-234) */
  const double *k8s_nonzero_requested; /* [K][N] k8s NodeInfo.NonZeroRequested (rows >= 2 unused) */
  const int32_t *max_tasks;            /* [N] Allocatable.MaxTaskNum (api/resource_info.go:95-97) */
  const int32_t *pod_count;            /* [N] len(k8s NodeInfo.Pods) (plugins/predicates/predicates.go:662) */
  const uint64_t *label_bits;          /* [Wl][N] bit b: node satisfies label requirement b */
  const uint64_t *taint_hard;          /* [Wt][N] NoSchedule / NoExecute taints */
  const uint64_t *taint_soft;          /* [Wt][N] PreferNoSchedule taints */
  const uint32_t *flags;               /* [N] VC_NODE_* */
  const int32_t *revocable_zone;       /* [N] zone id or -1 (NodeInfo.RevocableZone) */
  const uint8_t *zone_active;          /* [Z] tdm availableRevocableZone() evaluated by the host once per cycle
                                          (plugins/tdm/tdm.go:118-137 uses time.Now()) */
} vc_nodes;

/* ---- api.TaskInfo (api/job_info.go:117-154) ---------------------------------------- */
typedef struct vc_tasks {
  const double *resreq;          /* [R][T] Resreq (== InitResreq, api/job_info.go:185-186) */
  const uint32_t *req_has;       /* [T] bit d (d>=2): scalar d is a key of Resreq.ScalarResources */
  const double *k8s_req;         /* [K][T] pod request as upstream computes it (Requested flavour) */
  const double *k8s_nonzero_req; /* [K][T] NonZero flavour (cpu 100m / memory 200Mi defaults) */
  const int32_t *job;            /* [T] job index */
  const int32_t *klass;          /* [T] class index */
  const int32_t *role;           /* [T] row in the job's role tables (TaskRole == "" has its own row,
                                    flagged VC_ROLE_EMPTY_NAME) */
  const int32_t *priority;       /* [T] TaskInfo.Priority */
  const int64_t *pod_index;      /* [T] numeric suffix of the pod name or -1
                                    (pkg/controllers/job/helpers/helpers.go:44-52) */
  const int64_t *creation_ts;    /* [T] Pod.CreationTimestamp */
  const uint32_t *uid_rank;      /* [T] rank of TaskInfo.UID in byte-string order */
} vc_tasks;

/* ---- scheduling constraints shared by tasks ("class") ------------------------------ */
#define VC_CLASS_REVOCABLE 1u             /* len(task.RevocableZone) > 0 */
#define VC_CLASS_TOLERATES_UNSCHEDULABLE 2u
typedef struct vc_classes {
  const uint64_t *selector;     /* [C][Wl] nodeSelector: all bits required */
  const int32_t *n_affinity;    /* [C] number of required nodeAffinity terms (0 = none) */
  const uint64_t *affinity;     /* [C][VC_MAX_TERMS][Wl] OR of AND-masks */
  const uint64_t *tolerated_hard; /* [C][Wt] */
  const uint64_t *tolerated_soft; /* [C][Wt] tolerations with effect PreferNoSchedule or empty */
  const int32_t *n_preferred;   /* [C] preferred nodeAffinity terms */
  const uint64_t *preferred;    /* [C][VC_MAX_TERMS][Wl] */
  const int32_t *preferred_weight; /* [C][VC_MAX_TERMS] */
  const uint32_t *flags;        /* [C] VC_CLASS_* */
} vc_classes;

/* ---- api.JobInfo (api/job_info.go:341-386) ----------------------------------------- */
#define VC_JOB_PENDING_PHASE 1u /* JobInfo.IsPending() (api/job_info.go:1181-1185) */
#define VC_JOB_PREEMPTABLE 2u   /* JobInfo.Preemptable (tdm jobOrderFn) */
#define VC_ROLE_EMPTY_NAME 1u    /* TaskRole == "": no predicate-error cache (util/predicate_helper.go:47-52),
                                   TaskHasFitErrors is always false (api/job_info.go:894-902) */
#define VC_ROLE_IN_MIN_MAP 2u    /* role is a key of JobInfo.TaskMinAvailable */
#define VC_JOB_UNSUPPORTED 4u   /* hard topology / subjob policy: run returns VC_EUNSUPPORTED */
typedef struct vc_jobs {
  const int32_t *queue;            /* [J] queue index or -1 when ssn.Queues lacks it (allocate.go:171) */
  const int32_t *min_available;    /* [J] JobInfo.MinAvailable */
  const int32_t *priority;         /* [J] JobInfo.Priority */
  const int64_t *creation_ts;      /* [J] */
  const uint32_t *uid_rank;        /* [J] rank of JobID string */
  const uint32_t *flags;           /* [J] VC_JOB_* */
  const int32_t *n_tasks_total;    /* [J] len(ji.Tasks), every status */
  const int32_t *ready_num;        /* [J] ReadyTaskNum() at open (api/job_info.go:844-853) */
  const int32_t *waiting_num;      /* [J] WaitingTaskNum() at open */
  const int32_t *pending_besteffort; /* [J] PendingBestEffortTaskNum() */
  const int32_t *valid_num;        /* [J] ValidTaskNum() (api/job_info.go:1100-1113) */
  const int32_t *task_min_total;   /* [J] TaskMinAvailableTotal */
  const int32_t *role_off;         /* [J+1] rows [role_off[j], role_off[j+1]) of the role tables */
  const double *allocated;         /* [R][J] sum Resreq over AllocatedStatus tasks at open (drf.go:196-203) */
  /* role tables, one row per (job, TaskRole) incl. roles that only appear in TaskMinAvailable */
  const int32_t *role_min;         /* [NR] TaskMinAvailable[role] (0 if absent) */
  const int32_t *role_occupied;    /* [NR] getJobAllocatedRoles() at open (api/job_info.go:969-990) */
  const int32_t *role_pipelined;   /* [NR] tasks of the role in Pipelined status at open */
  const int32_t *role_pending_other; /* [NR] Pending tasks of the role NOT in vc_tasks (best-effort, gated) */
  const int32_t *role_valid;       /* [NR] CheckTaskValid's `actual` at open (api/job_info.go:993-1019) */
  const uint32_t *role_flags;      /* [NR] VC_ROLE_* */
} vc_jobs;

/* ---- api.QueueInfo (api/queue_info.go:36-51) + proportion inputs ------------------- */
#define VC_QUEUE_OPEN 1u
#define VC_QUEUE_NOT_RECLAIMABLE 2u /* !QueueInfo.Reclaimable(): Queue.Spec.Reclaimable == false (api/queue_info.go) */
#define VC_RES_HAS_ANY 0x80000000u /* in a *_has word: the ResourceList itself is non-empty */
typedef struct vc_queues {
  const int32_t *weight;        /* [Q] */
  const int32_t *priority;      /* [Q] Queue.Spec.Priority */
  const int64_t *creation_ts;   /* [Q] */
  const uint32_t *uid_rank;     /* [Q] */
  const uint32_t *flags;        /* [Q] VC_QUEUE_* */
  const double *capability;     /* [R][Q] Queue.Spec.Capability */
  const uint32_t *capability_has; /* [Q] bit d: dim d present; VC_RES_HAS_ANY: len(Capability) != 0 */
  const double *guarantee;      /* [R][Q] Queue.Spec.Guarantee.Resource */
  const uint32_t *guarantee_has;/* [Q] */
  const double *allocated;      /* [R][Q] proportion attr.allocated at open (proportion.go:143-149) */
  const double *request;        /* [R][Q] proportion attr.request at open (allocated + ALL Pending tasks) */
  const uint32_t *request_has;  /* [Q] scalar keys present in attr.request */
  const uint32_t *allocated_has;/* [Q] scalar keys present in attr.allocated */
} vc_queues;

/* ---- conf.SchedulerConfiguration (conf/scheduler_conf.go:28-107) ------------------- */
enum vc_plugin {
  VC_PLUGIN_PRIORITY = 1,
  VC_PLUGIN_GANG = 2,
  VC_PLUGIN_DRF = 3,
  VC_PLUGIN_PROPORTION = 4,
  VC_PLUGIN_PREDICATES = 5,
  VC_PLUGIN_NODEORDER = 6,
  VC_PLUGIN_BINPACK = 7,
  VC_PLUGIN_TDM = 8,
  VC_PLUGIN_NETWORK_TOPOLOGY_AWARE = 9,
  VC_PLUGIN_CONFORMANCE = 10, /* evictableFn: never evict critical pods (plugins/conformance/conformance.go:46-66) */
  VC_PLUGIN_PDB = 11, /* PreemptableFn / ReclaimableFn: PodDisruptionBudgets (plugins/pdb/pdb.go:65-137), vc_victim_guards */
  VC_PLUGIN_CDP = 12, /* PreemptableFn / ReclaimableFn: cooldown protection (plugins/cdp/cdp.go:56-110), vc_victim_guards */
  VC_PLUGIN_OTHER = 99 /* overcommit, ...: no effect on this path */
};
/* PluginOption enable flags (conf/scheduler_conf.go:60-107); nil == false unless
   ApplyPluginConfDefaults ran (plugins/defaults.go:29-55) — the caller resolves that. */
#define VC_EN_JOB_ORDER 0x001u
#define VC_EN_JOB_READY 0x002u
#define VC_EN_JOB_PIPELINED 0x004u
#define VC_EN_TASK_ORDER 0x008u
#define VC_EN_QUEUE_ORDER 0x010u
#define VC_EN_PREDICATE 0x020u
#define VC_EN_NODE_ORDER 0x040u
#define VC_EN_BEST_NODE 0x080u
#define VC_EN_OVERUSED 0x100u
#define VC_EN_ALLOCATABLE 0x200u
#define VC_EN_PREEMPTABLE 0x400u
#define VC_EN_RECLAIMABLE 0x800u
#define VC_EN_JOB_STARVING 0x1000u
#define VC_EN_PREEMPTIVE 0x2000u /* EnablePreemptive: ssn.Preemptive (reclaim.go:145), proportion.go:376-380 */
#define VC_EN_ALL 0x3fffu
typedef struct vc_plugin_option {
  int32_t plugin;   /* enum vc_plugin */
  int32_t tier;     /* 0-based tier index; options are listed in tier, then plugin order */
  uint32_t enabled; /* VC_EN_* */
} vc_plugin_option;

/* predicates plugin switches (plugins/predicates/predicates.go:126-151) */
#define VC_PRED_NODE_AFFINITY 1u
#define VC_PRED_TAINT_TOLERATION 2u
typedef struct vc_conf {
  int32_t n_plugins;
  vc_plugin_option plugins[VC_MAX_PLUGINS];
  /* binpack arguments (plugins/binpack/binpack.go:94-158) */
  int32_t binpack_weight;
  int32_t binpack_dim_weight[VC_MAX_DIMS]; /* -1: resource not in BinPackingResources */
  /* nodeorder arguments (plugins/nodeorder/nodeorder.go:131-171) */
  int32_t w_least, w_most, w_balanced, w_node_affinity, w_taint_toleration;
  int32_t kdim_dim[VC_MAX_KDIMS]; /* volcano dim index of each k8s-scored dim */
  /* predicates arguments */
  uint32_t predicates_enable; /* VC_PRED_* */
  /* allocate action + server options */
  int32_t enable_predicate_error_cache; /* allocate.go:107-120, default 1 */
  int32_t enqueue_action_enabled;       /* conf.EnabledActionMap["enqueue"] (allocate.go:154-164) */
  int32_t percentage_nodes_to_find;     /* options.go:48-54; 100 = parity mode (SURVEY §8c) */
  int32_t min_nodes_to_find;            /* 100 */
  int32_t min_percentage_nodes_to_find; /* 5 */
  int32_t last_processed_node_index;    /* util.lastProcessedNodeIndex (util/scheduler_helper.go:50) carried over from
                                           the previous cycle; only read when the sampling above is in force */
  /* network-topology-aware arguments (plugins/network-topology-aware/network_topology_aware.go:155-229) */
  int32_t nta_weight;                   /* "weight", default 1 */
  int32_t nta_dim_weight[VC_MAX_DIMS];  /* hypernode.binpack.{cpu,memory,resources.*}; -1: not in the weight map */
  int32_t nta_normal_pod_enable;        /* hypernode.binpack.normal-pod.enable, default 1 */
  double nta_fading;                    /* hypernode.binpack.normal-pod.fading, default 0.8 */
} vc_conf;

/* ---- HyperNode tree (ssn.HyperNodesSetByTier / ssn.RealNodesSet, framework/session.go:239-245) -----
   Consumed by network-topology-aware's hypernode-level binpacking of pods without a network topology
   (batchNodeOrderFnForNormalPods, network_topology_aware.go:462-496). The cluster top hypernode that
   Session open adds above the highest real tier (session.go:285-313) is part of the table. */
typedef struct vc_hypernodes {
  int32_t n_hypernodes;  /* H */
  int32_t min_tier;      /* hyperNodesTier.init, network_topology_aware.go:97-104 */
  int32_t max_tier;      /* max_tier - min_tier + 1 <= VC_MAX_TIERS */
  const int32_t *member; /* [max_tier-min_tier+1][N]: index in [0,H) of the hypernode of tier min_tier+l whose
                            RealNodesSet holds node n, -1 when no hypernode of that tier does */
  const int32_t *tier;   /* [H] HyperNodeInfo.Tier() */
  const int32_t *parent; /* [H] HyperNodeInfo.Parent as an index, -1 for the cluster top hypernode */
  /* Jobs whose default subJob carries a soft-mode network topology (SubJobInfo.IsSoftTopologyMode,
     api/sub_job_info.go:94-99): their tasks are scored by batchNodeOrderFnForNetworkAwarePods
     (network_topology_aware.go:541-571). All four may be NULL when the session has none. */
  const uint8_t *job_soft;          /* [J] 1 = soft-mode topology job */
  const int32_t *job_allocated;     /* [J] subJob.AllocatedHyperNode at open as an index, -1 = "" */
  const int32_t *job_placed_off;    /* [J+1] CSR over job_placed_node */
  const int32_t *job_placed_node;   /* node index of every task of the job that carries a NodeName at open
                                       (FindJobTaskNumOfHyperNode counts subJob.Tasks by NodeName) */
} vc_hypernodes;

/* ---- hierarchical drf (drf's enableHierarchy, plugins/drf/drf.go:45-184,458-560): the queue annotations
   volcano.sh/hierarchy and volcano.sh/hierarchy-weights (QueueInfo.Hierarchy / Weights, api/queue_info.go:60-61), split
   on "/" with the first segment (the root) dropped. The library builds the tree (first-creator weights, clamp to 1). ---- */
typedef struct vc_hdrf {
  const int32_t *path_off;  /* [Q+1] CSR over path_name: queue q names the segments [path_off[q], path_off[q+1]) */
  const int32_t *path_name; /* interned segment names (equal ids = equal strings) */
  const int32_t *n_weights; /* [Q] segments of the weights string after the first (len(split(Weights)) - 1) */
  const double *weight;     /* laid out like path_name: strconv.ParseFloat of the weight segment at the same depth, the
                               value ParseFloat returns even with an error (0 for a syntax error, +-Inf out of range);
                               entries at depths >= n_weights[q] are ignored */
  const double *job_request; /* [R][J] JobInfo.TotalRequest: Resreq summed over every task of the job, any status */
} vc_hdrf;

/* ---- node.Tasks: the pods that occupy nodes (api/node_info.go:88) — candidate victims of the preempt and
   reclaim actions. Their resources are already part of vc_nodes.{idle,used,...}; this table adds what victim
   selection reads per task. Index space of its own ("running task" r). ---- */
#define VC_RT_PREEMPTABLE 1u  /* TaskInfo.Preemptable (volcano.sh/preemptable annotation / label) */
#define VC_RT_RUNNING 2u      /* Status == Running */
#define VC_RT_BOUND 4u        /* Status == Bound (api.PreemptableStatus: Bound | Running, api/helpers.go:70-77) */
#define VC_RT_BEST_EFFORT 8u  /* TaskInfo.BestEffort */
#define VC_RT_CRITICAL 16u    /* conformance: system-cluster-critical / system-node-critical PriorityClassName or
                                 namespace kube-system (plugins/conformance/conformance.go:50-56) */
typedef struct vc_running_tasks {
  int32_t n_tasks;
  const int32_t *node;           /* [n] node index (TaskInfo.NodeName) */
  const int32_t *job;            /* [n] job index, -1 when ssn.Jobs lacks it */
  const int32_t *role;           /* [n] row in the job's role tables (or -1 with job == -1) */
  const int32_t *priority;       /* [n] TaskInfo.Priority */
  const int64_t *pod_index;      /* [n] as vc_tasks.pod_index */
  const int64_t *creation_ts;    /* [n] */
  const uint32_t *uid_rank;      /* [n] rank of TaskInfo.UID among the running tasks */
  const double *resreq;          /* [R][n] TaskInfo.Resreq */
  const uint32_t *req_has;       /* [n] */
  const double *k8s_req;         /* [K][n] what the predicates plugin's event handler subtracts on eviction */
  const double *k8s_nonzero_req; /* [K][n] (rows >= 2 unused) */
  const uint32_t *flags;         /* [n] VC_RT_* */
} vc_running_tasks;
#define VC_TASK_PREEMPT_NEVER 1u /* pod.Spec.PreemptionPolicy == Never (preempt.go:437-441, reclaim.go:140-143) */

/* ---- the preempt action's arguments (actions/preempt/preempt.go:50-99) and what its topology-aware reading reads per
   running task. Defaults (vc_snapshot_set_preempt_options(s, NULL)): topology_aware 0, 10 / 1 / 100.
   Determinism contract of the topology-aware reading:
   - predicateNodes are in NodeList order; node.Tasks in ascending running-task index;
   - the k-th dry run of one vc_preempt_run (k counts from 0 the preemptors that reach findCandidates with at least one
     predicate node) starts at offset = splitmix64(offset_seed + k) % len(predicateNodes), where
       splitmix64(x): z = x + 0x9E3779B97F4A7C15; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;
                      z = (z ^ (z >> 27)) * 0x94D049BB133111EB; return z ^ (z >> 31)   (uint64 arithmetic);
   - the 16 workers with early cancel read as one: the candidates are the first numCandidates nodes with victims in scan
     order from the offset, wrapping around; ties of pickOneNodeForPreemption go to the earlier candidate of that order;
   - a victim without Pod.Status.StartTime starts at now_ns (one time.Now() per run);
   - topologyAwarePreemptWorkerNum is accepted by the callers and ignored. ---- */
#define VC_START_TIME_UNSET INT64_MIN /* rt_start_ns: Pod.Status.StartTime == nil */
typedef struct vc_preempt_options {
  int32_t topology_aware;                 /* enableTopologyAwarePreemption */
  int32_t min_candidate_nodes_percentage; /* minCandidateNodesPercentage */
  int32_t min_candidate_nodes_absolute;   /* minCandidateNodesAbsolute */
  int32_t max_candidate_nodes_absolute;   /* maxCandidateNodesAbsolute */
  uint64_t offset_seed;                   /* replaces rand.Intn (see above) */
  int64_t now_ns;                         /* replaces time.Now() for victims without a StartTime, ns since the epoch */
  int32_t n_running;                      /* length of the two arrays: vc_preempt_run checks it against vc_running_tasks */
  const int32_t *rt_pod_priority;         /* [n_running] PodPriority: Pod.Spec.Priority, 0 when nil (not TaskInfo.Priority) */
  const int64_t *rt_start_ns;             /* [n_running] Pod.Status.StartTime in ns, VC_START_TIME_UNSET when nil */
} vc_preempt_options;

/* ---- what the victim votes of the pdb and cdp plugins read per running task. The caller matches selectors and parses
   durations; the library walks the budgets and compares the times. Determinism contract of both votes:
   - the preemptees of one ssn.Preemptable / ssn.Reclaimable call are walked in ascending running-task index (node.Tasks);
   - PDB status (DisruptionsAllowed, DisruptedPods) is read once, at session open;
   - every vote starts from DisruptionsAllowed again (pdb.go:75-79): evictions earlier in the session do not use up a budget;
   - one now_ns per session stands for every time.Now() of cdp. ---- */
#define VC_COOLDOWN_NONE INT64_MIN /* rt_cooldown_until_ns: cdp cannot protect the pod */
#define VC_GUARD_NO_LABELS 1u      /* rt_flags: len(pod.Labels) == 0 — pdb skips the pod, so it never returns it */
typedef struct vc_victim_guards {
  int32_t n_running;                    /* checked against vc_running_tasks */
  int32_t n_pdb;                        /* PodDisruptionBudgets of the session, any order */
  const int32_t *pdb_allowed;           /* [n_pdb] Status.DisruptionsAllowed */
  const int32_t *rt_pdb_off;            /* [n_running + 1] CSR over rt_pdb */
  const int32_t *rt_pdb;                /* the PDBs that count task r, each once: same namespace, a non-empty selector
                                           (metav1.LabelSelectorAsSelector without error) that matches the labels, the pod's
                                           name not in Status.DisruptedPods. Ignored for a task flagged VC_GUARD_NO_LABELS */
  const uint32_t *rt_flags;             /* [n_running] VC_GUARD_* */
  const int64_t *rt_cooldown_until_ns;  /* [n_running] LastTransitionTime of the first PodScheduled=True condition plus
                                           the volcano.sh/cooldown-time duration (label first, then annotation, by
                                           time.ParseDuration; an invalid label disables it), for a Running pod; else
                                           VC_COOLDOWN_NONE. cdp protects the pod while this is after now_ns */
  int64_t now_ns;                       /* time.Now() of the session, ns since the epoch */
} vc_victim_guards;

/* ---- results ----------------------------------------------------------------------- */
#define VC_OP_ALLOCATE 0 /* Statement.Allocate (framework/statement.go:242-302) */
#define VC_OP_PIPELINE 1 /* Statement.Pipeline (framework/statement.go:146-200) */
#define VC_OP_EVICT 2    /* Statement.Evict (framework/statement.go:72-99): decision.task indexes vc_running_tasks */
typedef struct vc_decision {
  int32_t task;
  int32_t node;
  int32_t kind;  /* VC_OP_* */
  int32_t visit; /* index into the visit list */
  double score;  /* score of the chosen node (0 when it was the only candidate, allocate.go:757) */
} vc_decision;

#define VC_VISIT_COMMIT 0  /* stmt != nil && JobReady: stmt.Commit() (allocate.go:330-331) */
#define VC_VISIT_KEEP 1    /* stmt != nil, job only pipelined: operations stay in the session */
#define VC_VISIT_DISCARD 2 /* stmt.Discard() (allocate.go:692) — its operations are not reported */
typedef struct vc_visit {
  int32_t job;
  int32_t outcome; /* VC_VISIT_* */
  int32_t first_op;
  int32_t n_ops;
} vc_visit;

typedef struct vc_stats {
  double upload_ms;   /* host->device copies + session-open kernels */
  double commit_ms;   /* the persistent commit kernel (CUDA events) */
  double download_ms; /* device->host result copy */
  double total_ms;
  int64_t h2d_bytes, d2h_bytes;
  int32_t kernel_launches;
  int32_t n_steps;    /* node sweeps executed */
  int64_t prof_cycles[8]; /* commit kernel phase timers (SM cycles of CTA 0): 0 queue/job control, 1 task fetch +
                             gates, 2 node sweep, 3 mailbox exchange, 4 apply + bookkeeping */
  int32_t last_processed_node_index; /* util.lastProcessedNodeIndex after the cycle (to carry into the next one) */
  int32_t commit_kernel; /* which instance of the commit kernel served the cycle: VC_KERNEL_* (diagnostic) */
  int32_t group_reentry[4]; /* VC_PROF instance of the incremental kernel: 0 group switches served by a full sweep, 1 those
                               served from the per-group verdict table (control program of CTA 0); 2 rows re-evaluated on
                               re-entry, 3 re-entries of a CTA past its changed-row threshold (both summed over CTAs) */
} vc_stats;
#define VC_KERNEL_GENERAL 0      /* k_commit: full sweep + all-gather per placement */
#define VC_KERNEL_INCREMENTAL 1  /* k_commit_fast: verdict cache, single-record publications, run-length batches */

typedef struct vc_snapshot vc_snapshot;
typedef struct vc_result vc_result;

/* ---- entry points ------------------------------------------------------------------ */
int vc_abi_version(void);
const char *vc_last_error(void);

/* Bind the calling process to CUDA device `device` (one process per GPU). The diagnostic switches (environment
   variables VC_PROF, VC_COMMIT_GENERIC, ... listed in README.md) are read here, once, never per cycle. */
int vc_init(int device);
/* Set one diagnostic switch by its environment-variable name at run time (tests, tools/). Switches select
   instrumented or alternative kernel instances; none changes a result. VC_EINVAL for an unknown name. */
int vc_debug_option(const char *name, int value);

/* Device memory for one scheduling session of the given size. */
int vc_snapshot_create(const vc_dims *dims, vc_snapshot **out);
void vc_snapshot_destroy(vc_snapshot *s);

/* Upload the session snapshot (host SoA -> HBM) and run the session-open reductions
   (ssn.TotalResource, drf shares, proportion deserved, class x node predicate mask). */
int vc_snapshot_upload(vc_snapshot *s, const vc_nodes *nodes, const vc_tasks *tasks,
                       const vc_classes *classes, const vc_jobs *jobs, const vc_queues *queues,
                       const vc_conf *conf);

/* Incremental upload (SURVEY §8f-2): the rows of the nodes whose NodeInfo changed since the last upload of this snapshot
   — the caller keeps the NodeInfo.Generation it uploaded per node (api/node_info.go:95-99) and lists the nodes whose
   generation moved. `rows` holds the SAME arrays as vc_nodes but compact, [dim][n_dirty] instead of [dim][N], for the
   accounting fields only: idle, used, releasing, pipelined, k8s_requested, k8s_nonzero_requested, pod_count (the other
   pointers are ignored; a change of Allocatable, labels, taints or flags needs vc_snapshot_upload). Tasks, jobs, queues
   and the configuration stay as uploaded: the session-open results that depend only on them (task / job order, groups,
   proportion's deserved) are kept, so a cycle that re-runs on a moved cluster state costs the dirty rows, not the
   snapshot. The session is reset to its (new) opening state. VC_EUNSUPPORTED: sessions with the topology tables
   (hypernode `used` sums are part of session open) and a row that would move the session between the commit kernels
   (first Releasing / Pipelined resource): do a full upload then. */
int vc_snapshot_update_nodes(vc_snapshot *s, int32_t n_dirty, const int32_t *node_idx, const vc_nodes *rows);

/* Optional, before vc_snapshot_upload: the HyperNode tree of the session. Without it a configured
   network-topology-aware plugin scores against the cluster top hypernode only (no HyperNode CRs). */
int vc_snapshot_set_topology(vc_snapshot *s, const vc_hypernodes *topo);

/* Optional, before vc_snapshot_upload: the queue hierarchy of drf's enableHierarchy (passing it means the option is set;
   NULL clears it). The table is copied; the tree is built at upload: children in first-insertion order with jobs inserted
   in index order, so the node's creator (and its weight) is the first job's queue; a weight < 1 or unparsable becomes 1.
   The allocate action then orders queues with hdrf's compareQueues in the tier chain of ssn.QueueOrderFn (when drf has
   EnabledQueueOrder) on a Go heap re-evaluated at every Push / Pop, as util.PriorityQueue does, and backfill's pick
   order uses the same chain on the state allocate left. VC_EINVAL at upload: drf not configured, a job outside ssn.Queues, a queue with jobs whose weights string
   has fewer segments than its path (the reference crashes on both), non-integral task requests or job allocations.
   vc_preempt_run / vc_reclaim_run return VC_EUNSUPPORTED with the table present (hdrf's reclaimFn is not built). Calling
   this after vc_snapshot_upload requires a new upload. */
int vc_snapshot_set_hdrf(vc_snapshot *s, const vc_hdrf *hdrf);

/* Optional, before vc_snapshot_upload: the BestEffort pending tasks of the session (TaskInfo.BestEffort,
   api/job_info.go:188: Resreq empty but for pods:1; not scheduling-gated) — the tasks the backfill action
   places (backfill.go:140-151). Same SoA as vc_tasks with its own index space [0, n_tasks); job / klass / role
   index the session's job, class and role tables; uid_rank ranks within this list. They are NOT part of
   vc_dims.n_tasks (allocate skips them, allocate.go:255-271) but stay counted in vc_jobs.pending_besteffort. The list is
   copied; it stays in effect for later uploads of this snapshot until replaced (n_tasks = 0 clears it). */
int vc_snapshot_set_backfill(vc_snapshot *s, int32_t n_tasks, const vc_tasks *tasks);

/* Optional, before vc_snapshot_upload: Pod.Status.NominatedNodeName of the pending tasks (set by a preemption of an earlier
   cycle) as node indices, [vc_dims.n_tasks], -1 = none or a node that is not in the session. allocate tries such a node first
   (actions/allocate/allocate.go:624-634): if InitResreq <= its FutureIdle, ph.PredicateNodes runs on that one node, and a pass
   makes it the task's only candidate. NULL clears the list. Sessions that carry a nominated task run on the general commit
   kernel. vc_reclaim_run runs them: reclaim never reads the nominated node (it checks PreemptionPolicy only,
   reclaim.go:140-143). vc_preempt_run refuses them (taskEligibleToPreempt's nominated-node rules, preempt.go:436-470, are
   not modelled). The list is copied and stays in effect for later uploads until replaced. */
int vc_snapshot_set_nominated(vc_snapshot *s, const int32_t *nominated_node);

/* Optional, before vc_snapshot_upload: the tasks that occupy nodes (victim candidates of preempt / reclaim) and,
   per pending task of vc_tasks, VC_TASK_* flags (task_flags may be NULL = all zero). Copied; stays in effect for
   later uploads until replaced (rt == NULL or n_tasks == 0 clears it). */
int vc_snapshot_set_running(vc_snapshot *s, const vc_running_tasks *rt, const uint32_t *task_flags);

/* Optional, any time before vc_preempt_run: the preempt action's arguments. Copied (arrays included); NULL restores the
   defaults, under which the action runs its normal reading. VC_EINVAL: arrays missing with n_running > 0. The reclaim
   action ignores them. */
int vc_snapshot_set_preempt_options(vc_snapshot *s, const vc_preempt_options *opts);

/* Optional, any time before vc_preempt_run / vc_reclaim_run: the table the pdb and cdp victim votes read (see
   vc_victim_guards). Copied; NULL clears it. VC_EINVAL: arrays missing, a bad CSR, a PDB index out of range or listed twice
   for one task. vc_preempt_run / vc_reclaim_run return VC_EINVAL when pdb or cdp votes in the action and no table is set,
   or when its n_running differs from vc_running_tasks. */
int vc_snapshot_set_victim_guards(vc_snapshot *s, const vc_victim_guards *g);

/* ONE session across the GPUs of a node (SURVEY §8e), one process per GPU: the exact allocate loop with the node axis cut
   over the CTAs of all ranks. Every rank uploads the same snapshot and runs the same replicated control program; a CTA's
   per-step records (its best (score, node); the publication of a run of placements) are written into EVERY rank's mailbox
   / ring through peer-mapped memory (CUDA IPC over NVLink) and polled locally. Rank 0 returns the decisions; the other
   ranks return empty results. Incremental commit kernel only (VC_EUNSUPPORTED otherwise, at upload).
     vc_comm_create   before vc_snapshot_upload: allocate this rank's slab, return its CUDA IPC handle (64 bytes)
     vc_comm_attach   map the slabs of all ranks: handles = world x 64 bytes in rank order (exchanged by the caller, e.g.
                      with torch.distributed.all_gather)
     vc_comm_prepare  before EVERY vc_allocate_run: clear this rank's slab. The caller then barriers across the ranks
                      (no rank may write into a slab that is still being cleared), calls vc_allocate_run on every rank,
                      and barriers again before the next prepare.
   A poll that sees nothing for ~10 s (a peer that never launched, diverged ranks) aborts the kernel with a CUDA error. */
#define VC_COMM_HANDLE_BYTES 64
int vc_comm_create(vc_snapshot *s, int world, int rank, void *handle_out);
int vc_comm_attach(vc_snapshot *s, const void *handles);
int vc_comm_prepare(vc_snapshot *s);

/* Restrict the node axis of this process to [node_begin, node_end) for node-sharded
   multi-GPU runs (SURVEY §8e); tasks/jobs/queues stay replicated. Default: all nodes.
   A non-empty shard begins at a multiple of 64 (one mask word per shard); an empty one may begin anywhere. */
int vc_snapshot_set_shard(vc_snapshot *s, int32_t node_begin, int32_t node_end);

/* The allocate action on the uploaded snapshot: exact sequential greedy assignment. VC_EUNSUPPORTED: feasible-node
   sampling with min_nodes_to_find below 1 where numNodesToFind of the node list is 0 (the reference then finds no node
   and advances lastProcessedNodeIndex by an amount that depends on its 16 workers). */
int vc_allocate_run(vc_snapshot *s, vc_result **out);

/* The backfill action (actions/backfill/backfill.go:58-116) on the session state vc_allocate_run left (or the
   opening state when allocate was not run): pickUpPendingTasks order (queues by QueueOrderFn, jobs by
   JobOrderFn, tasks by TaskOrderFn, all evaluated once at the start), then per task the plugin predicates
   (no resource fit), util.PrioritizeNodes + arg-max over every feasible node (skipped when there is exactly
   one), and Session.Allocate (framework/session.go:746-796) at once. In the result, decision.task indexes
   the BACKFILL task list; there is one visit per job in pick order, outcome VC_VISIT_COMMIT when ssn.JobReady
   held (the tasks were dispatched to the binder) else VC_VISIT_KEEP (Allocated in the session only); tasks
   without a feasible node are listed in fit_errors. Feasible-node sampling continues from the lastProcessedNodeIndex
   the allocate run left (vc_stats.last_processed_node_index of this result carries it on). VC_EUNSUPPORTED: the
   network-topology-aware plugin weighs a resource BestEffort pods request ("pods" in hypernode.binpack.resources), and
   numNodesToFind 0 as for vc_allocate_run. */
int vc_backfill_run(vc_snapshot *s, vc_result **out);

/* The preempt action (actions/preempt/preempt.go:101-283, normalPreempt :333-434, or topologyAwarePreempt :475-1015 when
   vc_preempt_options.topology_aware is set) and the reclaim action (actions/reclaim/reclaim.go:56-258) on the session state the preceding
   actions left (vc_allocate_run, each other). Preemptors are the tasks of vc_tasks that are still Pending.
   Split: per preemptor the device evaluates EVERY node at once — plugin predicates in their preempt reading
   (ssn.PredicateForPreemptAction, framework/session.go:679-697: only unresolvable failures reject a node, the pod-count cap
   does not), the util.PrioritizeNodes total, and exact necessary conditions of the attempt (util.ValidateVictims over every
   task that could be a victim; the queue's Allocatable gate with all of them gone) — and hands out the surviving nodes in
   the action's order (util.SortNodes for preempt, NodeList for reclaim). The victim selection on the node under trial
   (ssn.Preemptable / ssn.Reclaimable tier votes, victim queue order, evict until the preemptor fits) is O(tasks on that
   node) and runs in the library's host control loop, as on the reference's action goroutine; attempts that fail leave no
   trace (nodeStmt.Discard, preempt.go:400-430). Canonical order of node.Tasks (a Go map): ascending running-task index.
   Result: decisions of kind VC_OP_EVICT (task = running-task index) and VC_OP_PIPELINE (task = vc_tasks index) in
   statement order; one visit per Statement (preempt: per preemptor job, then per intra-job preemptor; reclaim: per job),
   VC_VISIT_COMMIT or VC_VISIT_DISCARD (discarded operations are not reported).
   Topology-aware reading (vc_preempt_options): per preemptor one device pass runs SelectVictimsOnNode as a dry run on every
   predicate node at once (victims from the tier votes and ValidateVictims, popped in victim-queue order until
   SimulateAllocatableFn and the FutureIdle fit hold, then reprieved last-popped first, on proportion's simulated queue
   state) and one single-block pass keeps the first numCandidates successes from the offset and picks the winner
   (SelectCandidate); the winner's victims are evicted in list order, then the preemptor is pipelined. The determinism
   contract is listed at vc_preempt_options. VC_EINVAL: its arrays do not match vc_running_tasks, or the arguments give a
   negative numCandidates for a preemptor (the reference panics in make; 0 is kept: no node is ever picked).
   Feasible-node sampling (a session where numNodesToFind(N) < N): every PredicateNodes call of both actions follows this
   determinism contract; without sampling predicateNodes are every passing node in NodeList order and the index is untouched.
   - the scanned list: a pending task that allocate left a NodesFitErrors entry with node errors (its predicate failed on
     every node; not a task skipped through TaskHasFitErrors) scans the nodes passing the static predicate in NodeList
     order (FilterOutUnschedulableAndUnresolvableNodesForTask); any other task scans the NodeList; P is its length;
   - numNodesToFind comes from P; the scan visits list[(start + i) % P] from start = util.lastProcessedNodeIndex and keeps
     the first numNodesToFind nodes that pass ssn.PredicateForPreemptAction (the 16 workers read as one); processed is the
     scan position of the last one kept + 1, or P when fewer pass; the index becomes (start + processed) % P, and an
     empty list leaves it alone;
   - the index is one value for the cycle: vc_allocate_run -> vc_preempt_run (both phases, every preemptor that reaches
     PredicateNodes, failed ones included; PreemptionPolicy Never does not) -> vc_reclaim_run; vc_stats.last_processed_node_index
     of each result reports it. Before any action of the cycle ran, vc_conf's value is taken as it is, not modulo N;
   - predicateNodes keep scan order: SortNodes' equal scores go to the lower scan position, reclaim walks scan order, and
     the topology-aware offset and candidate order count positions in scan order.
   PreferNoSchedule taints under TaintToleration's batch score order preempt's normal reading: the count of intolerable
   ones is normalised by its maximum over predicateNodes (every node passing the static predicate, or under sampling the
   sampled list), candidates or not; reclaim and the topology-aware reading do not score nodes.
   network-topology-aware (hypernode binpacking of normal pods, hypernode.binpack.normal-pod.enable): preempt's normal
   reading adds the plugin's node score to util.PrioritizeNodes' total (batchNodeOrderFnForNormalPods + scaleFinalScore,
   network_topology_aware.go:461-498), read from hyperNodeResourceCache.used as the session stands: the opening rows,
   then allocate's kept operations in order, then every Statement Evict (-Resreq), Pipeline (+Resreq) and Discard (the
   inverse, in reverse order) of preempt and reclaim, on every hypernode that holds the node, cpu, memory and the
   task's present scalars. The sums are exact for integer-valued requests (the node rows follow the same rule). A node's
   hypernode at a tier is the one of vc_hypernodes.member (where hypernodes of one tier overlap, the reference breaks out
   of a Go map walk; the encoder keeps the lowest name); node.Tasks are walked in ascending running-task index. Jobs with
   a (soft-mode) network topology never preempt, in either phase or reading (preempt.go:132-137); they reclaim, and their
   pods are victims like any other. Reclaim and the topology-aware reading do not score nodes.
   VC_EUNSUPPORTED: BestEffort pending tasks in the session (vc_snapshot_set_backfill), the tdm plugin; under sampling,
   enablePredicateErrorCache with a job
   whose named roles span several (class, request) groups, and min_nodes_to_find below 1 (numNodesToFind of a list can
   then be 0; a session whose numNodesToFind(N) is 0 is refused too, although allocate runs it without sampling). */
int vc_preempt_run(vc_snapshot *s, vc_result **out);
int vc_reclaim_run(vc_snapshot *s, vc_result **out);

/* Dense task x node pass on the opening snapshot: feasibility bit (allocate.predicate,
   allocate.go:816-824), total score (util.PrioritizeNodes) of every feasible pair and
   per-task best (score, node) under the canonical tie-break (lowest NodeList index).
   All outputs are HOST buffers (any may be NULL):
     mask_out  [T][ceil(N/64)] uint64, bit n of row t
     score_out [T][N] double (0.0 where infeasible)
     best_score[T] double, best_node[T] int32 (-1 = no feasible node)          */
int vc_score_matrix(vc_snapshot *s, uint64_t *mask_out, double *score_out, double *best_score,
                    int32_t *best_node);
/* Same pass with the outputs kept in HBM, run `repeats` times; returns CUDA-event times measured on the
   launching stream: kernel_ms_out[0] = mean of the whole dense pass (K1a + best + K1b),
   kernel_ms_out[1] = mean of the materialising kernel K1b alone; *algorithmic_bytes_out = the bytes of
   SURVEY.md §8(d): T*N*(8 + 1/8) + per-task and per-node operand bytes. */
int vc_score_matrix_device(vc_snapshot *s, int repeats, double *kernel_ms_out, int64_t *algorithmic_bytes_out);

/* Node-sharded dense pass (SURVEY §8e), one process per GPU, tasks replicated:
     vc_dense_begin   K1a on this shard (per group: any idle-fit / future-fit node, max soft-taint count)
     vc_dense_stats   device pointer to those int32 counters so the caller can MAX-all-reduce them (NCCL)
     vc_dense_finish  per-task best (score,node) of this shard [+ materialised shard of the matrix]
     vc_dense_best    device pointers to best_score[T] (f64) / best_node[T] (i32; -1 none) for the
                      cross-shard arg-max (all-gather + fold, or two all-reduces)            */
int vc_dense_begin(vc_snapshot *s);
int vc_dense_stats(vc_snapshot *s, int32_t **stats_dev_out, int32_t *count_out);
int vc_dense_finish(vc_snapshot *s, int materialize);
int vc_dense_best(vc_snapshot *s, double **best_score_dev_out, int32_t **best_node_dev_out);
/* copy the materialised matrix of the last vc_dense_finish(.,1) to host buffers (any may be NULL) */
int vc_dense_fetch(vc_snapshot *s, uint64_t *mask_out, double *score_out, double *best_score, int32_t *best_node);

/* proportion's per-queue deserved / share after session open (plugins/proportion/
   proportion.go:197-264), for parity checks: [R][Q] and [Q]. */
int vc_queue_deserved(vc_snapshot *s, double *deserved_out, double *share_out);

size_t vc_result_num_decisions(const vc_result *r);
const vc_decision *vc_result_decisions(const vc_result *r);
size_t vc_result_num_visits(const vc_result *r);
const vc_visit *vc_result_visits(const vc_result *r);
/* tasks for which job.NodesFitErrors was recorded (allocate.go:600-607,651) */
size_t vc_result_num_fit_errors(const vc_result *r);
const int32_t *vc_result_fit_errors(const vc_result *r);
const vc_stats *vc_result_stats(const vc_result *r);
/* subJob.AllocatedHyperNode of every job after the run (index into the hypernode table, -1 = ""): what
   allocate.go:681-686 stores for soft-mode topology jobs. NULL / 0 when the session has no such job. */
const int32_t *vc_result_job_allocated_hypernodes(const vc_result *r, size_t *n_jobs);
void vc_result_free(vc_result *r);

#ifdef __cplusplus
}
#endif
#endif /* VCALLOC_H */

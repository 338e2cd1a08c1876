"""Seeded synthetic session snapshots of the BASELINE.json configs (SURVEY.md §8d).

Generates the structure-of-arrays directly (no per-pod Python objects) so that the
10k x 100k and 50k x 1M shapes build in seconds.  All resource values are integer-valued
(milli-cpu, bytes, milli-scalars, pod counts) exactly like api.NewResource produces.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import numpy as np

from . import abi
from .snapshot import PluginOption, SchedulerConf, Snapshot, build_conf

DIMS = ["cpu", "memory", "ephemeral-storage", "example.com/foo", "hugepages-2Mi", "nvidia.com/gpu", "pods", "rdma/hca"]
D_CPU, D_MEM, D_EPH, D_FOO, D_HUGE, D_GPU, D_PODS, D_RDMA = range(8)
KDIMS = ("cpu", "memory", "nvidia.com/gpu")
GI = 1 << 30
MI = 1 << 20
DEFAULT_SEED = 20260921


@dataclass
class SynthConfig:
    name: str
    n_nodes: int
    n_tasks: int
    n_queues: int = 1
    plugins: str = "gang+predicates+nodeorder+binpack"  # '+'-separated
    utilisation: float = 0.6   # initial Used ~ U(min_util, utilisation) * Allocatable
    min_util: float = 0.0
    n_classes: int = 64
    seed: int = DEFAULT_SEED
    releasing_frac: float = 0.0  # fraction of nodes with Releasing resources (exercises the FutureIdle gradient)
    soft_taint_p: float = 0.0    # per-bit probability of PreferNoSchedule taints (normalising TaintToleration scorer)
    mixed_roles: bool = False    # two roles with different requests per job + TaskMinAvailable (role minima, error cache)
    topology: Optional[tuple] = None  # HyperNode tree fan-outs below the single root, e.g. (32, 40): 32 tier-2 x 40 tier-1 each
    topology_scatter: float = 0.0     # fraction of nodes assigned to a random leaf / left outside the tree (tests)
    soft_topology_frac: float = 0.0   # fraction of jobs whose PodGroup carries a soft-mode network topology
    n_besteffort: int = 0             # extra BestEffort pending pods spread over the jobs (the backfill action's tasks)
    besteffort_jobs: int = 0          # > 0: the BestEffort pods go into that many random jobs only (long same-group runs
                                      # in backfill's pick order); 0: spread over all jobs
    hetero: int = 0                   # > 0: every task draws its own request from `hetero` distinct cpu / memory sizes
                                      # (heterogeneous pods: the (class, request) groups of the dense pass approach T)
    hdrf: Optional[tuple] = None      # (departments, teams): drf's enableHierarchy over a root -> department -> team tree


CONFIGS = {
    # BASELINE.json configs[0]: plumbing-size case the CPU oracle runs instantly
    "cfg1": SynthConfig("cfg1", 128, 1024, 1, "gang+predicates+binpack"),
    # configs[1]: the headline single-GPU workload
    "cfg2": SynthConfig("cfg2", 10_000, 100_000, 1, "priority+gang+predicates+nodeorder+binpack"),
    # cfg2 with terminating pods on 30 % of the nodes (Releasing resources: the FutureIdle gradient exists, most placements
    # still land on idle resources) and a nearly full cluster where many tasks can only be pipelined
    "cfg2_fut": SynthConfig("cfg2_fut", 10_000, 100_000, 1, "priority+gang+predicates+nodeorder+binpack", releasing_frac=0.3),
    "cfg2_fut_tight": SynthConfig("cfg2_fut_tight", 10_000, 100_000, 1, "priority+gang+predicates+nodeorder+binpack",
                                  utilisation=0.97, min_util=0.8, releasing_frac=0.5),
    # cfg2 with PreferNoSchedule taints (the normalising TaintToleration batch scorer), alone and with terminating pods
    "cfg2_soft": SynthConfig("cfg2_soft", 10_000, 100_000, 1, "priority+gang+predicates+nodeorder+binpack", soft_taint_p=0.05),
    "cfg2_fut_soft": SynthConfig("cfg2_fut_soft", 10_000, 100_000, 1, "priority+gang+predicates+nodeorder+binpack",
                                 utilisation=0.9, min_util=0.5, releasing_frac=0.4, soft_taint_p=0.05),
    "mid_soft": SynthConfig("mid_soft", 2_000, 20_000, 2, "priority+gang+drf+predicates+proportion+nodeorder+binpack", soft_taint_p=0.08,
                            utilisation=0.95, min_util=0.6, releasing_frac=0.4),
    "mid_fut": SynthConfig("mid_fut", 2_000, 20_000, 1, "priority+gang+predicates+nodeorder+binpack", releasing_frac=0.3),
    "cfg3_fut": SynthConfig("cfg3_fut", 10_000, 100_000, 16, "priority+gang+drf+predicates+proportion+nodeorder+binpack",
                            utilisation=0.9, min_util=0.5, releasing_frac=0.4),
    # configs[2]: + DRF + proportion over 16 queues
    "cfg3": SynthConfig("cfg3", 10_000, 100_000, 16, "priority+gang+drf+predicates+proportion+nodeorder+binpack"),
    # cfg3 with hierarchical drf: its 16 queues as 4 departments x 4 teams, unequal weights
    "cfg3_hdrf": SynthConfig("cfg3_hdrf", 10_000, 100_000, 16, "priority+gang+drf+predicates+proportion+nodeorder+binpack",
                             hdrf=(4, 4)),
    # configs[3]: 3-tier HyperNode tree (root -> 32 -> 40 each -> ~39 nodes), network-topology-aware weight 10
    # (hypernode-level binpacking of pods without a network topology; topology-constrained jobs are not generated)
    "cfg4": SynthConfig("cfg4", 50_000, 1_000_000, 16,
                        "priority+gang+drf+predicates+proportion+nodeorder+binpack+network-topology-aware", topology=(32, 40),
                        soft_topology_frac=0.1),
    # the same shape without the topology plugin (incremental commit kernel)
    "cfg4_flat": SynthConfig("cfg4_flat", 50_000, 1_000_000, 16, "priority+gang+drf+predicates+proportion+nodeorder+binpack"),
    # small shapes for tests
    "tiny": SynthConfig("tiny", 64, 300, 3, "priority+gang+drf+predicates+proportion+nodeorder+binpack", n_classes=12),
    "small": SynthConfig("small", 700, 4000, 4, "priority+gang+drf+predicates+proportion+nodeorder+binpack", n_classes=24),
    # general-kernel shapes: Releasing resources (pipelining) and PreferNoSchedule taints
    "tiny_fut": SynthConfig("tiny_fut", 64, 300, 3, "priority+gang+drf+predicates+proportion+nodeorder+binpack", n_classes=12,
                            utilisation=0.99, min_util=0.9, releasing_frac=0.6),
    "small_soft": SynthConfig("small_soft", 300, 1500, 2, "priority+gang+predicates+nodeorder+binpack", n_classes=16,
                              soft_taint_p=0.08),
    "small_fut_soft": SynthConfig("small_fut_soft", 300, 1500, 4, "priority+gang+drf+predicates+proportion+nodeorder+binpack",
                                  n_classes=16, utilisation=0.99, min_util=0.88, releasing_frac=0.5, soft_taint_p=0.08),
    # cfg4's plugin set on a size that profiles in seconds
    "mid_topo": SynthConfig("mid_topo", 20_000, 40_000, 16,
                            "priority+gang+drf+predicates+proportion+nodeorder+binpack+network-topology-aware", topology=(16, 20),
                            soft_topology_frac=0.1),
    "tiny_topo": SynthConfig("tiny_topo", 96, 400, 2, "priority+gang+drf+predicates+proportion+nodeorder+binpack+network-topology-aware",
                             n_classes=8, topology=(2, 3), topology_scatter=0.1, soft_topology_frac=0.3),
    "small_topo": SynthConfig("small_topo", 600, 3000, 3, "priority+gang+predicates+nodeorder+binpack+network-topology-aware",
                              n_classes=16, topology=(4, 6), topology_scatter=0.15, soft_topology_frac=0.2),
    "small_topo_fut_soft": SynthConfig("small_topo_fut_soft", 300, 1500, 3,
                                       "priority+gang+drf+predicates+proportion+nodeorder+binpack+network-topology-aware",
                                       n_classes=12, utilisation=0.99, min_util=0.88, releasing_frac=0.5, soft_taint_p=0.08,
                                       topology=(3, 4), topology_scatter=0.1, soft_topology_frac=0.3),
    # hypernode binpacking only (no topology-constrained jobs)
    "small_topo_normal": SynthConfig("small_topo_normal", 600, 3000, 3, "priority+gang+predicates+nodeorder+binpack+network-topology-aware",
                                     n_classes=16, topology=(4, 6), topology_scatter=0.15),
    # allocate + backfill: BestEffort pods next to the regular ones
    "tiny_bf": SynthConfig("tiny_bf", 64, 300, 3, "priority+gang+drf+predicates+proportion+nodeorder+binpack", n_classes=12,
                           n_besteffort=150),
    "small_bf": SynthConfig("small_bf", 700, 4000, 4, "priority+gang+drf+predicates+proportion+nodeorder+binpack", n_classes=24,
                            n_besteffort=3000),
    "small_soft_bf": SynthConfig("small_soft_bf", 300, 1500, 2, "priority+gang+predicates+nodeorder+binpack", n_classes=16,
                                 soft_taint_p=0.08, n_besteffort=1200),
    "small_topo_bf": SynthConfig("small_topo_bf", 600, 3000, 3, "priority+gang+predicates+nodeorder+binpack+network-topology-aware",
                                 n_classes=16, topology=(4, 6), topology_scatter=0.15, soft_topology_frac=0.2, n_besteffort=2500),
    "cfg2_bf": SynthConfig("cfg2_bf", 10_000, 100_000, 1, "priority+gang+predicates+nodeorder+binpack", n_besteffort=20_000),
    "small_roles": SynthConfig("small_roles", 200, 1200, 2, "priority+gang+predicates+nodeorder+binpack", n_classes=8,
                               utilisation=0.85, mixed_roles=True),
}


def scheduler_conf(cfg: SynthConfig) -> SchedulerConf:
    names = cfg.plugins.split("+")
    args = {
        "binpack": {"binpack.weight": 10, "binpack.cpu": 5, "binpack.memory": 1,
                    "binpack.resources": "nvidia.com/gpu", "binpack.resources.nvidia.com/gpu": 2},
        "nodeorder": {},  # default weights: least 1, balanced 1, nodeaffinity 2, tainttoleration 3
        "network-topology-aware": {"weight": 10, "hypernode.binpack.cpu": 5, "hypernode.binpack.memory": 1,
                                   "hypernode.binpack.resources": "nvidia.com/gpu",
                                   "hypernode.binpack.resources.nvidia.com/gpu": 2},
    }
    tier1 = [PluginOption.defaults(n, args.get(n)) for n in names if n in ("priority", "gang")]
    tier2 = [PluginOption.defaults(n, args.get(n)) for n in names if n not in ("priority", "gang")]
    return SchedulerConf(tiers=[t for t in (tier1, tier2) if t],
                         actions=("allocate", "backfill") if cfg.n_besteffort > 0 else ("allocate",))


def make_snapshot(cfg: SynthConfig | str, seed: Optional[int] = None) -> Snapshot:
    if isinstance(cfg, str):
        cfg = CONFIGS[cfg]
    rng = np.random.default_rng(cfg.seed if seed is None else seed)
    N, T, Q, R = cfg.n_nodes, cfg.n_tasks, cfg.n_queues, len(DIMS)

    # ---- jobs: Zipf gang sizes, minAvailable = size (70 %) or size/2 (30 %) ------------------
    sizes = np.array([1, 2, 4, 8, 16, 64, 256])
    pz = 1.0 / np.arange(1, len(sizes) + 1)
    pz /= pz.sum()
    job_sizes: List[int] = []
    tot = 0
    while tot < T:
        sz = int(rng.choice(sizes, p=pz))
        sz = min(sz, T - tot)
        job_sizes.append(sz)
        tot += sz
    job_sizes_a = np.array(job_sizes, np.int64)
    J = len(job_sizes_a)
    C_ = cfg.n_classes
    s = Snapshot(N, T, J, Q, C_, J, R, K=len(KDIMS), Wl=1, Wt=1, Z=0, pods_dim=D_PODS, B=cfg.n_besteffort)
    s.dim_names = list(DIMS)
    s.node_names = [f"node-{i:06d}" for i in range(N)] if N <= 20000 else []
    s.queue_names = [f"q{i:02d}" for i in range(Q)]

    # ---- nodes: 4 SKUs 40/30/20/10 % ---------------------------------------------------------
    sku = rng.choice(4, size=N, p=[0.4, 0.3, 0.2, 0.1])
    cpu = np.array([32, 64, 96, 128])[sku] * 1000.0
    mem = np.array([128, 256, 768, 1024])[sku] * float(GI)
    maxpods = np.array([110, 110, 110, 250])[sku]
    gpus = np.array([0, 0, 8, 8])[sku]
    a = s.n_allocatable
    a[D_CPU], a[D_MEM] = cpu, mem
    a[D_EPH] = np.array([1, 2, 4, 8])[sku] * 1e12 * 1000.0       # ephemeral-storage in milli-bytes
    a[D_FOO] = 16 * 1000.0
    a[D_HUGE] = np.array([0, 4, 16, 64])[sku] * float(GI) * 1000.0
    a[D_GPU] = gpus * 1000.0
    a[D_PODS] = maxpods
    a[D_RDMA] = np.where(gpus > 0, 4, 0) * 1000.0
    u = rng.uniform(cfg.min_util, cfg.utilisation, size=(R, N))
    used = np.zeros((R, N))
    used[D_CPU] = np.floor(u[D_CPU] * cpu / 100.0) * 100.0
    used[D_MEM] = np.floor(u[D_MEM] * mem / (64 * MI)) * (64 * MI)
    used[D_EPH] = np.floor(u[D_EPH] * a[D_EPH] / 1e12) * 1e12
    used[D_GPU] = np.floor(u[D_GPU] * gpus) * 1000.0
    used[D_PODS] = np.floor(u[D_PODS] * maxpods)
    used[D_RDMA] = np.floor(u[D_RDMA] * a[D_RDMA] / 1000.0) * 1000.0
    s.n_used[:] = used
    s.n_idle[:] = a - used
    s.n_max_tasks[:] = maxpods
    s.n_pod_count[:] = used[D_PODS].astype(np.int32)
    kmap = [D_CPU, D_MEM, D_GPU]
    for k, d in enumerate(kmap):
        scale = 1000.0 if d == D_GPU else 1.0
        s.n_k8s_allocatable[k] = a[d] / scale
        s.n_k8s_requested[k] = used[d] / scale
        s.n_k8s_nonzero_requested[k] = used[d] / scale
    # 64 label bits: zone one-hot(16) | sku one-hot(4) | pool one-hot(8) | 36 booleans p=0.1
    zone = rng.integers(0, 16, N)
    pool = rng.integers(0, 8, N)
    lb = (np.uint64(1) << zone.astype(np.uint64)) | (np.uint64(1) << (16 + sku).astype(np.uint64)) | \
         (np.uint64(1) << (20 + pool).astype(np.uint64))
    rb = rng.random((36, N)) < 0.1
    for b in range(36):
        lb |= rb[b].astype(np.uint64) << np.uint64(28 + b)
    s.n_label_bits[0] = lb
    tb = np.zeros(N, np.uint64)
    rt = rng.random((32, N)) < 0.02
    for b in range(32):
        tb |= rt[b].astype(np.uint64) << np.uint64(b)
    s.n_taint_hard[0] = tb
    if cfg.soft_taint_p > 0:
        sb = np.zeros(N, np.uint64)
        rs_ = rng.random((8, N)) < cfg.soft_taint_p
        for b in range(8):
            sb |= rs_[b].astype(np.uint64) << np.uint64(b)
        s.n_taint_soft[0] = sb
    if cfg.releasing_frac > 0:
        # some of the used resources are being released (terminating pods): Releasing <= Used
        relmask = rng.random(N) < cfg.releasing_frac
        frac = rng.uniform(0.2, 0.8, size=N) * relmask
        rel = np.zeros((R, N))
        rel[D_CPU] = np.floor(frac * used[D_CPU] / 100.0) * 100.0
        rel[D_MEM] = np.floor(frac * used[D_MEM] / (64 * MI)) * (64 * MI)
        rel[D_PODS] = np.floor(frac * used[D_PODS])
        rel[D_GPU] = np.floor(frac * used[D_GPU] / 1000.0) * 1000.0
        s.n_releasing[:] = rel

    # ---- classes: 25 % with a nodeSelector on <= 2 label bits, 10 % with tolerations -----------
    for c in range(C_):
        r = rng.random()
        if c > 0 and r < 0.25:
            bits = [int(rng.integers(0, 16))] if rng.random() < 0.5 else [16 + int(rng.integers(0, 4))]
            if rng.random() < 0.5:
                bits.append(20 + int(rng.integers(0, 8)))
            for b in bits:
                s.c_selector[c, 0] |= np.uint64(1) << np.uint64(b)
        if c > 0 and rng.random() < 0.10:
            s.c_tolerated_hard[c, 0] = np.uint64(rng.integers(0, 2**32))
        if cfg.soft_taint_p > 0 and c > 0 and rng.random() < 0.3:
            s.c_tolerated_soft[c, 0] = np.uint64(rng.integers(0, 256))
        if c > 0 and rng.random() < 0.15:
            s.c_n_preferred[c] = 1
            s.c_preferred[c, 0, 0] = np.uint64(1) << np.uint64(int(rng.integers(0, 16)))
            s.c_preferred_weight[c, 0] = int(rng.integers(1, 101))

    # ---- tasks: one request type and one class per job (a gang is homogeneous) ----------------
    types = np.array([
        # cpu(milli), mem(bytes), gpu(count)
        [500, 1 * GI, 0], [1000, 2 * GI, 0], [2000, 8 * GI, 0], [4000, 16 * GI, 0], [8000, 64 * GI, 1], [32000, 256 * GI, 8],
    ], dtype=np.float64)
    job_type = rng.choice(6, size=J, p=[0.30, 0.30, 0.20, 0.10, 0.08, 0.02])
    job_class = rng.integers(0, C_, J)
    job_of_task = np.repeat(np.arange(J), job_sizes_a)
    tt = job_type[job_of_task]
    s.t_resreq[D_CPU] = types[tt, 0]
    s.t_resreq[D_MEM] = types[tt, 1]
    s.t_resreq[D_GPU] = types[tt, 2] * 1000.0
    s.t_resreq[D_PODS] = 1.0
    has = np.full(T, 1 << D_PODS, np.uint32)
    has[types[tt, 2] > 0] |= np.uint32(1 << D_GPU)
    s.t_req_has[:] = has
    for k, col in enumerate((0, 1, 2)):
        s.t_k8s_req[k] = types[tt, col]
        s.t_k8s_nonzero_req[k] = types[tt, col]
    if cfg.hetero > 0:  # heterogeneous pods: per-task cpu in 100m steps, memory in 256Mi steps
        kc = rng.integers(1, cfg.hetero + 1, T).astype(np.float64)
        km = rng.integers(1, cfg.hetero + 1, T).astype(np.float64)
        s.t_resreq[D_CPU] = kc * 100.0
        s.t_resreq[D_MEM] = km * 256.0 * MI
        s.t_resreq[D_GPU] = 0.0
        s.t_req_has[:] = np.uint32(1 << D_PODS)
        for k, d in enumerate((D_CPU, D_MEM)):
            s.t_k8s_req[k] = s.t_resreq[d]
            s.t_k8s_nonzero_req[k] = s.t_resreq[d]
        s.t_k8s_req[2] = 0.0
        s.t_k8s_nonzero_req[2] = 0.0
    s.t_job[:] = job_of_task
    s.t_klass[:] = job_class[job_of_task]
    s.t_role[:] = job_of_task  # one role row per job
    s.t_priority[:] = 1
    starts = np.concatenate([[0], np.cumsum(job_sizes_a)[:-1]])
    s.t_pod_index[:] = np.arange(T) - starts[job_of_task]
    s.t_uid_rank[:] = np.arange(T, dtype=np.uint32)

    # ---- jobs --------------------------------------------------------------------------------
    full = rng.random(J) < 0.7
    s.j_min_available[:] = np.where(full, job_sizes_a, np.maximum(1, job_sizes_a // 2))
    s.j_queue[:] = rng.integers(0, Q, J)
    s.j_priority[:] = rng.integers(0, 3, J)
    s.j_creation_ts[:] = rng.integers(0, 1000, J)
    s.j_uid_rank[:] = np.arange(J, dtype=np.uint32)
    s.j_n_tasks_total[:] = job_sizes_a
    s.j_valid_num[:] = job_sizes_a
    s.j_role_off[:] = np.arange(J + 1)
    s.r_valid[:] = job_sizes_a
    s.r_flags[:] = 0  # named role "worker", not in TaskMinAvailable
    if cfg.mixed_roles:
        # two roles per job: role 0 = even pod index, role 1 = odd pod index with a different request type;
        # jobs with >= 4 tasks declare TaskMinAvailable {role0: 1, role1: 1}
        s2 = Snapshot(N, T, J, Q, C_, 2 * J, R, K=len(KDIMS), Wl=1, Wt=1, Z=0, pods_dim=D_PODS, B=cfg.n_besteffort)
        for k, v in s.__dict__.items():
            if isinstance(v, np.ndarray) and not k.startswith("r_") and k != "j_role_off":
                getattr(s2, k)[...] = v
        s2.dim_names, s2.node_names, s2.queue_names = s.dim_names, s.node_names, s.queue_names
        s = s2
        odd = (s.t_pod_index % 2 == 1)
        s.t_role[:] = 2 * job_of_task + odd.astype(np.int32)
        alt = (tt + 1) % 4
        for col, d in ((0, D_CPU), (1, D_MEM)):
            s.t_resreq[d, odd] = types[alt[odd], col]
        for k, col in enumerate((0, 1)):
            s.t_k8s_req[k, odd] = types[alt[odd], col]
            s.t_k8s_nonzero_req[k, odd] = types[alt[odd], col]
        s.j_role_off[:] = 2 * np.arange(J + 1)
        s.r_valid[0::2] = (job_sizes_a + 1) // 2
        s.r_valid[1::2] = job_sizes_a // 2
        big = job_sizes_a >= 4
        s.r_min[0::2] = np.where(big, 1, 0)
        s.r_min[1::2] = np.where(big, 1, 0)
        s.r_flags[0::2] = np.where(big, abi.VC_ROLE_IN_MIN_MAP, 0)
        s.r_flags[1::2] = np.where(big, abi.VC_ROLE_IN_MIN_MAP, 0)
        s.j_task_min_total[:] = np.where(big, 2, 0)
    s.job_names = []

    # ---- queues ------------------------------------------------------------------------------
    s.q_weight[:] = rng.integers(1, 5, Q)
    s.q_uid_rank[:] = np.arange(Q, dtype=np.uint32)
    if Q >= 4:  # two queues with capability caps
        total = a.sum(axis=1)
        for qi in (1, 3):
            s.q_capability[:, qi] = np.floor(total * 0.03)
            s.q_capability_has[qi] = np.uint32(abi.VC_RES_HAS_ANY | sum(1 << d for d in range(2, R)))
    # proportion request = sum of pending Resreq per queue (nothing allocated at open)
    jq = s.j_queue[job_of_task]
    for d in range(R):
        s.q_request[d] = np.bincount(jq, weights=s.t_resreq[d], minlength=Q)
    for qi in range(Q):
        m = jq == qi
        s.q_request_has[qi] = np.bitwise_or.reduce(has[m]) if m.any() else 0
    sconf = scheduler_conf(cfg)
    s.conf = build_conf(sconf, DIMS, KDIMS)
    s.actions = tuple(sconf.actions)
    if cfg.topology is not None:
        _make_topology(s, cfg, rng)
    if cfg.n_besteffort > 0:
        _make_besteffort(s, cfg, np.random.default_rng((cfg.seed if seed is None else seed) + 7919), job_class)
    if cfg.hdrf is not None:
        depts, teams = cfg.hdrf
        hier = [f"root/dept{(q // teams) % depts}/team{q % teams}" for q in range(Q)]
        wts = [f"1/{1 + (q // teams) % depts}/{1 + 2 * (q % teams)}" for q in range(Q)]
        s.set_hdrf(hier, wts, total_request(s))
    return s


def total_request(s: Snapshot) -> np.ndarray:
    """JobInfo.TotalRequest [R][J] of a synthetic snapshot: allocated at open + every pending task (BestEffort ones too)."""
    treq = s.j_allocated.copy()
    np.add.at(treq.T, s.t_job, s.t_resreq.T)
    if s.B:
        np.add.at(treq.T, s.b_job, s.b_resreq.T)
    return treq


def _make_besteffort(s: Snapshot, cfg: SynthConfig, rng, job_class) -> None:
    """BestEffort pending pods (Resreq = pods:1 only; upstream non-zero defaults 100m / 200Mi for the scorers) attached to
    random jobs: they count in PendingBestEffortTaskNum / the role's occupancy during allocate and are placed by backfill."""
    B, J = cfg.n_besteffort, s.J
    if cfg.besteffort_jobs > 0:
        hosts = rng.choice(J, size=min(cfg.besteffort_jobs, J), replace=False)
        bj = np.sort(hosts[rng.integers(0, len(hosts), B)]).astype(np.int32)
    else:
        bj = np.sort(rng.integers(0, J, B)).astype(np.int32)
    s.b_job[:] = bj
    s.b_klass[:] = job_class[bj]
    s.b_role[:] = s.j_role_off[bj]  # first role row of the job
    s.b_resreq[D_PODS] = 1.0
    s.b_req_has[:] = np.uint32(1 << D_PODS)
    s.b_k8s_nonzero_req[0] = 100.0
    s.b_k8s_nonzero_req[1] = 200.0 * MI
    s.b_priority[:] = rng.integers(1, 4, B)
    s.b_pod_index[:] = 1_000_000 + np.arange(B)
    s.b_uid_rank[:] = rng.permutation(B).astype(np.uint32)
    cnt = np.bincount(bj, minlength=J).astype(np.int32)
    s.j_pending_besteffort[:] = cnt
    s.j_n_tasks_total[:] += cnt
    s.j_valid_num[:] += cnt
    first = s.j_role_off[:-1]
    np.add.at(s.r_valid, first, cnt)
    np.add.at(s.r_occupied, first, cnt)       # occupied counts pending BestEffort tasks (job_info.go:1024-1036)
    np.add.at(s.r_pending_other, first, cnt)


def _make_topology(s: Snapshot, cfg: SynthConfig, rng) -> None:
    """HyperNode tree as the [tier level][node] membership table Session open derives (snapshot.encode_hypernodes):
    tier 1 = leaf hypernodes over contiguous node blocks, tier 2 = their parents, tier 3 = one root, tier 4 = the
    cluster top hypernode.  `topology_scatter` moves some nodes to a random leaf and leaves some outside the tree."""
    N = s.N
    n_mid, per_mid = cfg.topology
    n_leaf = n_mid * per_mid
    block = -(-N // n_leaf)
    leaf = np.minimum(np.arange(N) // block, n_leaf - 1)
    outside = np.zeros(N, bool)
    if cfg.topology_scatter > 0:
        r = rng.random(N)
        moved = r < cfg.topology_scatter
        leaf[moved] = rng.integers(0, n_leaf, int(moved.sum()))
        outside = r > 1.0 - cfg.topology_scatter / 2
    mid = leaf // per_mid
    member = np.full((4, N), -1, np.int32)
    member[0] = np.where(outside, -1, leaf)
    member[1] = np.where(outside, -1, n_leaf + mid)
    member[2] = np.where(outside, -1, n_leaf + n_mid)
    member[3] = n_leaf + n_mid + 1
    s.hn_names = [f"leaf-{i}" for i in range(n_leaf)] + [f"mid-{i}" for i in range(n_mid)] + ["root", "<cluster-top-hypernode>"]
    s.hn_min_tier, s.hn_max_tier = 1, 4
    s.hn_member = np.ascontiguousarray(member)
    H = n_leaf + n_mid + 2
    s.hn_tier = np.concatenate([np.full(n_leaf, 1), np.full(n_mid, 2), [3, 4]]).astype(np.int32)
    s.hn_parent = np.concatenate([n_leaf + np.arange(n_leaf) // per_mid, np.full(n_mid, n_leaf + n_mid), [H - 1, -1]]).astype(np.int32)
    # soft-mode topology jobs: nothing is allocated at open, so AllocatedHyperNode = "" and the node lists are empty
    s.hn_job_soft = (rng.random(s.J) < cfg.soft_topology_frac).astype(np.uint8)
    s.hn_job_allocated = np.full(s.J, -1, np.int32)
    s.hn_job_placed_off = np.zeros(s.J + 1, np.int32)
    s.hn_job_placed_node = np.zeros(1, np.int32)


# ---------------------------------------------------------------------------------------
# BASELINE.json configs[4]: 10k nodes near 85 % utilisation, 32 queues, ~10k pending tasks per cycle, actions
# allocate + preempt + reclaim. One cycle of the churn: the cluster is full of running pods (node.Tasks, the victim
# candidates), part of the jobs are starving (running below minAvailable with pending pods left), new jobs arrive.
# ---------------------------------------------------------------------------------------
CFG5_PLUGINS = "priority+gang+conformance+drf+predicates+proportion+nodeorder+binpack"


def make_cfg5(seed: Optional[int] = None, n_nodes: int = 10_000, n_pending: int = 10_000, n_queues: int = 32,
              utilisation: float = 0.85) -> Snapshot:
    seed = DEFAULT_SEED if seed is None else seed
    rng = np.random.default_rng(seed + 55)
    # capacity of the cluster decides how many running tasks there are: avg task ~2.7 cores
    cores = n_nodes * (0.4 * 32 + 0.3 * 64 + 0.2 * 96 + 0.1 * 128)
    n_all = int(n_pending + utilisation * cores / 2.2)
    base = make_snapshot(SynthConfig("cfg5", n_nodes, n_all, n_queues, CFG5_PLUGINS, utilisation=0.0, seed=seed))
    N, R, K, J, Q = base.N, base.R, base.K, base.J, base.Q
    alloc = base.n_allocatable
    job = base.t_job
    sizes = np.bincount(job, minlength=J)
    # jobs in random order fill the cluster with running pods until the cpu target is reached; the last ones run partially
    order = rng.permutation(J)
    target = utilisation * alloc[D_CPU].sum()
    idle = alloc.copy()
    running = np.zeros(base.T, bool)
    node_of = np.full(base.T, -1, np.int32)
    task_ids = [np.nonzero(job == j)[0] for j in range(J)] if J < 200000 else None
    used_cpu = 0.0
    pend_left = n_pending
    for j in order:
        if used_cpu >= target:
            break
        ts = task_ids[j]
        frac = 1.0 if rng.random() < 0.8 else rng.uniform(0.2, 0.9)  # 20 % of the running jobs are short of pods
        n_run = max(1, int(round(frac * len(ts))))
        for t in ts[:n_run]:
            req = base.t_resreq[:, t]
            for _ in range(32):  # a few random nodes; a task that finds none stays pending
                n = int(rng.integers(0, N))
                if (idle[:, n] >= req).all():
                    idle[:, n] -= req
                    running[t] = True
                    node_of[t] = n
                    used_cpu += req[D_CPU]
                    break
    pending = ~running
    # keep about n_pending pending tasks: whole pending-only jobs beyond the budget are dropped
    keep = pending.copy()
    cnt = 0
    for j in order[::-1]:
        ts = task_ids[j]
        p = ts[pending[ts]]
        if len(p) == 0:
            continue
        if cnt >= n_pending and not running[ts].any():
            keep[p] = False
        else:
            cnt += len(p)
    pend_ids = np.nonzero(keep)[0]
    run_ids = np.nonzero(running)[0]
    T = len(pend_ids)
    s = Snapshot(N, T, J, Q, base.C, J, R, K=K, Wl=1, Wt=1, Z=0, pods_dim=D_PODS, B=0)
    for k, v in base.__dict__.items():
        if isinstance(v, np.ndarray) and not k.startswith(("t_", "b_", "rt_")) and hasattr(s, k) and getattr(s, k).shape == v.shape:
            getattr(s, k)[...] = v
    s.dim_names, s.node_names, s.queue_names, s.job_names = base.dim_names, base.node_names, base.queue_names, []
    for name in ("resreq", "req_has", "k8s_req", "k8s_nonzero_req", "job", "klass", "role", "priority", "pod_index",
                 "creation_ts", "uid_rank"):
        src = getattr(base, "t_" + name)
        getattr(s, "t_" + name)[...] = src[..., pend_ids]
    s.t_uid_rank[:] = np.argsort(np.argsort(s.t_uid_rank)).astype(np.uint32)
    s.t_flags = np.zeros(T, np.uint32)
    # node.Tasks
    RT = len(run_ids)
    s.set_running(RT)
    s.rt_node[:] = node_of[run_ids]
    s.rt_job[:] = base.t_job[run_ids]
    s.rt_role[:] = base.t_role[run_ids]
    s.rt_priority[:] = 1
    s.rt_pod_index[:] = base.t_pod_index[run_ids]
    s.rt_uid_rank[:] = np.arange(RT, dtype=np.uint32)
    s.rt_resreq[:] = base.t_resreq[:, run_ids]
    s.rt_req_has[:] = base.t_req_has[run_ids]
    s.rt_k8s_req[:] = base.t_k8s_req[:, run_ids]
    s.rt_k8s_nonzero_req[:] = base.t_k8s_nonzero_req[:, run_ids]
    s.rt_flags[:] = abi.VC_RT_RUNNING | np.where(rng.random(RT) < 0.7, abi.VC_RT_PREEMPTABLE, 0).astype(np.uint32)
    s.running_task_keys = []
    # node rows
    used = alloc - idle
    s.n_used[:] = used
    s.n_idle[:] = idle
    s.n_pod_count[:] = np.bincount(s.rt_node, minlength=N).astype(np.int32)
    for k in range(K):
        s.n_k8s_requested[k] = np.bincount(s.rt_node, weights=s.rt_k8s_req[k], minlength=N)
        s.n_k8s_nonzero_requested[k] = np.bincount(s.rt_node, weights=s.rt_k8s_nonzero_req[k], minlength=N)
    # jobs / roles / queues as the cache would hand them over
    n_run_j = np.bincount(s.rt_job, minlength=J).astype(np.int32)
    n_pend_j = np.bincount(s.t_job, minlength=J).astype(np.int32)
    total_j = n_run_j + n_pend_j
    s.j_ready_num[:] = n_run_j
    s.j_n_tasks_total[:] = total_j
    s.j_valid_num[:] = total_j
    s.r_valid[:] = total_j
    s.r_occupied[:] = n_run_j
    gang_full = rng.random(J) < 0.5
    s.j_min_available[:] = np.where(gang_full, total_j, np.maximum(1, total_j // 2))
    s.j_priority[:] = rng.choice([0, 10, 100], size=J, p=[0.5, 0.3, 0.2])
    for d in range(R):
        s.j_allocated[d] = np.bincount(s.rt_job, weights=s.rt_resreq[d], minlength=J)
    jq_run, jq_pend = s.j_queue[s.rt_job], s.j_queue[s.t_job]
    s.q_allocated[:] = 0
    for d in range(R):
        s.q_allocated[d] = np.bincount(jq_run, weights=s.rt_resreq[d], minlength=Q)
        s.q_request[d] = s.q_allocated[d] + np.bincount(jq_pend, weights=s.t_resreq[d], minlength=Q)
    for qi in range(Q):
        mr, mp = jq_run == qi, jq_pend == qi
        ah = np.bitwise_or.reduce(s.rt_req_has[mr]) if mr.any() else 0
        s.q_allocated_has[qi] = ah
        s.q_request_has[qi] = ah | (np.bitwise_or.reduce(s.t_req_has[mp]) if mp.any() else 0)
    s.q_capability[:] = 0
    s.q_capability_has[:] = 0
    sconf = scheduler_conf(SynthConfig("cfg5", n_nodes, T, n_queues, CFG5_PLUGINS))
    sconf.actions = ("allocate", "preempt", "reclaim")
    s.conf = build_conf(sconf, DIMS, KDIMS)
    s.actions = tuple(sconf.actions)
    return s

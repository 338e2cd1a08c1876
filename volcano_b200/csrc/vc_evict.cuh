// vc_evict.cuh — device side of the preempt and reclaim actions (actions/preempt/preempt.go, actions/reclaim/reclaim.go).
//
// Per preemptor the node-wide part of the action runs here, one thread per node:
//   k_evict_rank   plugin predicates in their preempt reading (ssn.PredicateForPreemptAction, framework/session.go:
//                  679-697: only the static, unresolvable failures reject a node; the pod-count cap does not), the
//                  util.PrioritizeNodes total of the node, and an exact necessary condition of util.ValidateVictims
//                  (util/scheduler_helper.go:313-329): FutureIdle plus the requests of EVERY task the action's filter
//                  lets through must cover the preemptor — any victim set the plugins return is a subset of those.
//   k_evict_pick   preempt: util.SortNodes' first not-yet-tried candidate = arg-max (score, lowest index); reclaim: the
//                  lowest-index candidate (NodeList order, reclaim.go:180).
//   k_evict_apply  Statement.Evict / Statement.Pipeline on the node rows the ranking reads (Releasing, Pipelined, the
//                  upstream NodeInfo sums of the predicates plugin) once the host committed to a node.
// The victim selection on the one node under trial (tier votes, victim queue order, evict-until-fit) is O(tasks on the
// node) and runs in the host control loop (vc_evict.hpp), like the reference's action goroutine.
#pragma once
#include "vc_device.cuh"
#include "vc_host.hpp"
#include "vc_topo.hpp"

#define EV_MODE_PREEMPT_INTER 0  // victims: other jobs of the preemptor's queue (preempt.go:198-214)
#define EV_MODE_PREEMPT_INTRA 1  // victims: the preemptor's own job (preempt.go:252-268)
#define EV_MODE_RECLAIM 2        // victims: Running tasks of other, reclaimable queues (reclaim.go:184-199)
#define EV_MAX_VICTIMS 256

struct EvictTask {  // the preemptor, staged per launch
  TaskRec rec;
  int klass, job, queue, mode;
  int job_prio, task_prio;
  // ssn.Allocatable of the preemptor's queue (proportion queueAllocatable, proportion.go:333-348) as a bound: with
  // quota_on the queue must admit the preemptor once EVERY candidate of the node is gone (they all sit in that queue)
  int quota_on, quota_open;
  uint32_t qalloc_has, qdes_has;
  double qalloc[VC_MAX_DIMS], qdes[VC_MAX_DIMS];
};
#define EV_PICK_K 32  // candidates one k_evict_pick launch hands to the host, in the action's node order
#define EV_CMD_OFF 80  // the apply command starts at this int of the mapped buffer (after the two sets of pick slots)
struct EvictParams {
  DevDims d;
  DevConf c;
  // node rows: Allocatable / upstream allocatable are inputs; the rest are the working copies the actions share
  const double *alloc, *kalloc;
  double *idle, *used, *rel, *pip, *kreq, *knz;
  int32_t *pod_count;
  const uint32_t *cstat;  // [C][N]
  // node.Tasks as CSR over nodes
  const int32_t *rt_off, *rt_idx;  // [N+1], [RT] running-task ids grouped by node, ascending
  const double *rt_req;            // [R][RT]
  const double *rt_kreq, *rt_knz;  // [K][RT]
  const uint32_t *rt_flags;        // [RT] VC_RT_*
  const int32_t *rt_job;           // [RT]
  uint8_t *rt_evicted;             // [RT] 1 = Releasing (evicted in this session)
  const int32_t *j_queue;          // [J]
  const uint32_t *q_flags;         // [Q]
  const int32_t *rt_prio;          // [RT] TaskInfo.Priority
  const int32_t *j_prio, *j_min;   // [J]
  const int32_t *j_ready;          // [J] ReadyTaskNum as the session stands (the host refreshes it after every eviction)
  const uint8_t *q_over;           // [Q] proportion: !allocated.LessEqual(deserved) as the session stands
  int exact_sums;                  // every request is an integer-valued double: sums of them are exact
  int RT;
  // per-preemptor scratch
  unsigned long long *key;  // [N] order-preserving score key of a candidate
  uint8_t *cand;            // [N] 1 = candidate, 2 = tried
  // pick result (mapped pinned memory): EV_PICK_K nodes in the action's order, -1 = no further candidate
  int32_t *pick_node;
  // feasible-node sampling (k_evict_samp): the sampled nodes in scan order, the only ones the SAMP pick considers
  const int32_t *samp_list, *samp_cnt;
  // apply command (mapped pinned memory): [0] node, [1] n_victims, [2..] victim running-task ids
  const int32_t *cmd;
  // SOFT instances (preempt's normal reading with PreferNoSchedule taints under TaintToleration's batch score): the score
  // is normalised by the largest intolerable-soft-taint count over predicateNodes, so it is final only after a reduction.
  // k_evict_rank then stores the node's order part (the bits of a double) in `key`; soft_word holds
  // (soft_seq << 8) | max — k_evict_rank's grid-wide max when soft_reduce, else k_evict_samp's over its list — and a word
  // whose tag is not soft_seq was left by an earlier ranking and reads as 0. The pick finishes total_score per node.
  unsigned long long *soft_word;
  unsigned long long soft_seq;
  int soft_klass, soft_reduce;
  // GUARD instances (pdb or cdp votes in the action): vct::VCT_GUARD_* bits per running task
  const uint8_t *rt_guard;
  // network-topology-aware with hypernode binpacking of normal pods (DevConf::nta_on): hn_used is the evicting actions'
  // working copy of hyperNodeResourceCache.used, which k_evict_apply books in every action; the NTA instances of
  // k_evict_rank add the plugin's node score to preempt's key. SOFT+NTA: the ranking stores the score per node in
  // nta_term (one array per ranking set) and the pick adds it when it finishes total_score.
  int hn_H;
  const int32_t *hn_member;  // [L][N] hypernode of the node at each tier level, -1 none
  const double *hn_alloc;    // [R][H]
  double *hn_used;           // [R][H]
  const uint32_t *rt_has;    // [RT] resource presence bits of the running tasks (the events book dims 0, 1 and these)
  double *nta_term;          // [N]
};

struct EvNodeView {
  const EvictParams &p;
  int n;
  __device__ __forceinline__ double alloc(int d) const { return p.alloc[(size_t)d * p.d.N + n]; }
  __device__ __forceinline__ double idle(int d) const { return p.idle[(size_t)d * p.d.N + n]; }
  __device__ __forceinline__ double used(int d) const { return p.used[(size_t)d * p.d.N + n]; }
  __device__ __forceinline__ double rel(int d) const { return p.rel[(size_t)d * p.d.N + n]; }
  __device__ __forceinline__ double pip(int d) const { return p.pip[(size_t)d * p.d.N + n]; }
  __device__ __forceinline__ double kalloc(int k) const { return p.kalloc[(size_t)k * p.d.N + n]; }
  __device__ __forceinline__ double kreq(int k) const { return p.kreq[(size_t)k * p.d.N + n]; }
  __device__ __forceinline__ double knz(int k) const { return p.knz[(size_t)k * p.d.N + n]; }
};

__device__ __forceinline__ unsigned long long ev_score_key(double x) {  // monotone double -> u64
  unsigned long long u = (unsigned long long)__double_as_longlong(x);
  return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}

// the soft-taint maximum of the ranking the pick reads (see EvictParams::soft_word)
__device__ __forceinline__ int ev_max_soft(const EvictParams &p) {
  const unsigned long long w = *p.soft_word;
  return (w >> 8) == p.soft_seq ? (int)(w & 0xffull) : 0;
}
// the pick's order key of a node: SOFT adds TaintToleration's normalised score to the stored order part, in total_score's
// operation order (0.0 + order, then + batch: the same double as a single call on the node); NTA adds the stored
// network-topology-aware term as the batch's second addend
template <bool SOFT, bool NTA = false>
__device__ __forceinline__ unsigned long long ev_pick_key(const EvictParams &p, int node, int max_soft) {
  if (!SOFT) return p.key[node];
  const int soft = (int)((p.cstat[(size_t)p.soft_klass * p.d.N + node] >> CS_SOFT_SHIFT) & 0xffu);
  return ev_score_key(total_score(p.c, true, __longlong_as_double((long long)p.key[node]), soft, max_soft,
                                  NTA ? p.nta_term[node] : 0.0));
}

// batchNodeOrderFnForNormalPods + scaleFinalScore (network_topology_aware.go:461-498, :758-764) for node n, on the working
// copy of hyperNodeResourceCache: the same function allocate's dense pass calls (nta_node_score)
__device__ __forceinline__ double ev_nta_score(const EvictParams &p, const TaskRec &t, int n) {
  const int H = p.hn_H;
  return nta_node_score(p.c, [&](int l) {
    const int h = p.hn_member[(size_t)l * p.d.N + n];
    return h < 0 ? 1.0
                 : hn_binpack_score(p.c, p.d.R, t, [&](int d) { return p.hn_used[(size_t)d * H + h]; },
                                    [&](int d) { return p.hn_alloc[(size_t)d * H + h]; });
  });
}

// the action's candidate filter on one task of node.Tasks
__device__ __forceinline__ bool ev_filter(const EvictParams &p, const EvictTask &t, int r) {
  if (p.rt_evicted[r]) return false;
  const uint32_t f = p.rt_flags[r];
  if (!(f & VC_RT_PREEMPTABLE)) return false;
  const int j = p.rt_job[r];
  if (t.mode == EV_MODE_RECLAIM) {
    if (!(f & VC_RT_RUNNING) || j < 0) return false;
    const int q = p.j_queue[j];
    return q >= 0 && q != t.queue && !(p.q_flags[q] & VC_QUEUE_NOT_RECLAIMABLE);
  }
  if (!(f & (VC_RT_RUNNING | VC_RT_BOUND))) return false;
  if (t.mode == EV_MODE_PREEMPT_INTRA) return j == t.job;
  return j >= 0 && j != t.job && p.j_queue[j] == t.queue;
}

// Could task r be among the victims ssn.Preemptable / ssn.Reclaimable returns (session_plugins.go:211-307)? Inside a
// tier the plugins' answers are intersected, but an empty intersection resets the list to nil and the next plugin's answer
// replaces it — so all that is certain about a victim is that it passed the LAST voting plugin of the tier that decided.
// Used here, per voter, is the part of its test that does not depend on the other candidates: conformance (not critical),
// gang (job above minAvailable, gang.go:97-129), priority (lower job / task priority, priority.go:110-148), proportion
// (queue above deserved, proportion.go:286-317); drf's test depends on the walk and counts as a yes. GUARD: cdp (cooldown
// over, exact) and pdb (labelled, and no PDB counting the task allows zero disruptions: the first decrement of such a
// budget already protects it).
template <bool GUARD = false>
__device__ __forceinline__ bool ev_may_be_victim(const EvictParams &p, const EvictTask &t, int r) {
  const bool reclaim = t.mode == EV_MODE_RECLAIM;
  const uint32_t flag = reclaim ? VC_EN_RECLAIMABLE : VC_EN_PREEMPTABLE;
  const int j = p.rt_job[r];
  int i = 0;
  while (i < p.c.n_plugins) {
    const int tier = p.c.tier[i];
    bool any = false, last = false;
    for (; i < p.c.n_plugins && p.c.tier[i] == tier; ++i) {
      if (!(p.c.enabled[i] & flag)) continue;
      const int pl = p.c.plugin[i];
      bool vote;
      if (pl == VC_PLUGIN_CONFORMANCE) vote = !(p.rt_flags[r] & VC_RT_CRITICAL);
      else if (pl == VC_PLUGIN_GANG) vote = j >= 0 && p.j_ready[j] > p.j_min[j];
      else if (pl == VC_PLUGIN_PRIORITY && !reclaim) vote = j >= 0 && (j != t.job ? p.j_prio[j] < t.job_prio : p.rt_prio[r] < t.task_prio);
      else if (pl == VC_PLUGIN_DRF && !reclaim) vote = j >= 0;
      else if (pl == VC_PLUGIN_PROPORTION && reclaim) vote = j >= 0 && p.j_queue[j] >= 0 && p.q_over[p.j_queue[j]];
      else if (GUARD && pl == VC_PLUGIN_PDB) vote = !(p.rt_guard[r] & VCT_GUARD_PDB_NEVER);
      else if (GUARD && pl == VC_PLUGIN_CDP) vote = !(p.rt_guard[r] & VCT_GUARD_CDP);
      else continue;
      any = true;
      last = vote;
    }
    if (any && last) return true;
  }
  return false;
}

// LPN lanes per node (16: two nodes per warp), one lane per entry of node.Tasks (strided when a node runs more pods than
// that): the filters are chains of dependent loads (task -> job -> queue ...), so the walk is latency-bound and the lanes
// overlap it; the requests of the possible victims are then summed per dimension with a shuffle tree inside the group.
// The group's first lane scores the node when it is a candidate. RMAX bounds the resource dimensions (register budget).
// SOFT: the key is the order part only, and with soft_reduce every node passing the static predicate (candidate or not:
// predicateNodes, scheduler_helper.go:76-136) enters the soft-taint maximum, one warp max and at most one atomic per warp.
// GUARD: the pdb and cdp votes take part in ev_may_be_victim.
// NTA: network-topology-aware's node score enters preempt's key (SOFT: it goes to nta_term, the pick adds it).
template <int LPN, int RMAX, bool SOFT = false, bool GUARD = false, bool NTA = false>
__global__ void __launch_bounds__(256) k_evict_rank(EvictParams p, EvictTask t) {
  const size_t gid = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  const int n = (int)(gid / LPN);
  const int gl = (int)(threadIdx.x % LPN);  // lane inside the group
  const int N = p.d.N, R = p.d.R, K = p.d.K;
  const bool live = n < N;
  const uint32_t cs = live ? p.cstat[(size_t)t.klass * N + n] : 0u;
  const bool stat_ok = live && (cs & CS_STATIC_OK);
  double freed[RMAX];
#pragma unroll
  for (int d = 0; d < RMAX; ++d) freed[d] = 0.0;
  int n_pass = 0;
  if (stat_ok) {
    for (int k = p.rt_off[n] + gl; k < p.rt_off[n + 1]; k += LPN) {
      const int r = p.rt_idx[k];
      if (!ev_filter(p, t, r)) continue;
      n_pass += 1;
      if (!ev_may_be_victim<GUARD>(p, t, r)) continue;
#pragma unroll
      for (int d = 0; d < RMAX; ++d)
        if (d < R) freed[d] += p.rt_req[(size_t)d * p.RT + r];
    }
  }
  // sums over the group (every lane of the warp takes part in the shuffles; groups are aligned, xor < LPN stays inside)
#pragma unroll
  for (int o = LPN / 2; o; o >>= 1) {
    n_pass += __shfl_xor_sync(0xffffffffu, n_pass, o);
#pragma unroll
    for (int d = 0; d < RMAX; ++d)
      if (d < R) freed[d] += __shfl_xor_sync(0xffffffffu, freed[d], o);
  }
  if (SOFT && p.soft_reduce) {
    const unsigned sv = (stat_ok && gl == 0) ? ((cs >> CS_SOFT_SHIFT) & 0xffu) : 0u;
    const unsigned long long w = (p.soft_seq << 8) | __reduce_max_sync(0xffffffffu, sv);
    if ((threadIdx.x & 31) == 0 && *reinterpret_cast<volatile unsigned long long *>(p.soft_word) < w) atomicMax(p.soft_word, w);
  }
  if (!live || gl != 0) return;
  uint8_t cand = 0;
  unsigned long long key = 0ull;
  if (stat_ok) {
    // ValidateVictims can only pass when FutureIdle + every possible victim covers the request. The sums above are
    // exact for integer-valued requests (exact_sums); otherwise a relative slack keeps the test a necessary condition
    // whatever the order of the additions.
    const double slack = p.exact_sums ? 0.0 : 1e-9;
    bool fits = true;
#pragma unroll
    for (int d = 0; d < RMAX; ++d) {
      if (d >= R) continue;
      if (d >= 2 && !(t.rec.has & (1u << d))) continue;
      const double pot = (p.idle[(size_t)d * N + n] + p.rel[(size_t)d * N + n]) - p.pip[(size_t)d * N + n];
      const double have = pot + freed[d];
      if (!le_eps(t.rec.req[d], have + fabs(have) * slack)) fits = false;
    }
    if (t.quota_on && p.exact_sums && t.mode != EV_MODE_RECLAIM) {
      // the evict loop ends with ssn.Allocatable(queue, preemptor) (preempt.go:380, :405): even with every possible
      // victim of this node evicted the queue must stay within deserved on the requested dimensions
      if (!t.quota_open) fits = false;
      const uint32_t rq_has = t.rec.has & ~3u;
#pragma unroll
      for (int d = 0; d < RMAX; ++d) {
        if (d >= R) continue;
        const double rq = t.rec.req[d];
        if (!(rq > 0.0)) continue;
        if (d >= 2 && (!(rq_has & (1u << d)) || d == p.d.pods_dim)) continue;
        const double al = (d < 2 || (t.qalloc_has & (1u << d))) ? t.qalloc[d] : 0.0;
        const double de = (d < 2 || (t.qdes_has & (1u << d))) ? t.qdes[d] : 0.0;
        if ((al - freed[d]) + rq > de) fits = false;
      }
    }
    if (fits && (t.mode != EV_MODE_RECLAIM || n_pass > 0)) {
      cand = 1;
      if (t.mode != EV_MODE_RECLAIM) {  // reclaim walks NodeList order, no scores (reclaim.go:172-180)
        const EvNodeView nv{p, n};
        double order = 0.0;
        const bool has_order = node_order(p.c, R, K, t.rec, nv, cs, &order);
        const double nta = NTA ? ev_nta_score(p, t.rec, n) : 0.0;
        if (SOFT) key = (unsigned long long)__double_as_longlong(has_order ? order : 0.0);
        else key = ev_score_key(total_score(p.c, has_order, has_order ? order : 0.0, 0, 0, nta));
        if (SOFT && NTA) p.nta_term[n] = nta;
      }
    }
  }
  p.cand[n] = cand;
  p.key[n] = key;
}

// k_evict_rank with 16 lanes per node, for R <= 8 or up to VC_MAX_DIMS resource dimensions
template <bool SOFT, bool GUARD, bool NTA>
inline void launch_evict_rank(unsigned grid, cudaStream_t st, size_t R, const EvictParams &p, const EvictTask &t) {
  if (R <= 8) k_evict_rank<16, 8, SOFT, GUARD, NTA><<<grid, 256, 0, st>>>(p, t);
  else k_evict_rank<16, VC_MAX_DIMS, SOFT, GUARD, NTA><<<grid, 256, 0, st>>>(p, t);
}

// one block: the next EV_PICK_K candidates in the action's node order (preempt: score descending, lowest index first
// among equals; reclaim: index ascending); the nodes handed out are marked tried. SAMP: the candidates are the nodes of
// k_evict_samp's list and the index is the position in it (scan order). Tournament with incremental repair:
// every thread keeps the best of its own nodes in registers, every warp its best in shared memory; handing out a node
// makes ONE thread rescan its nodes and ONE warp refold, the other 31 entries stay. Used when the keys do not fit in shared
// memory (k_evict_pick below): repairs read the candidate flags and keys from global memory.
// The last store of the launch is `seq` into pick_node[EV_PICK_K] (system scope): the host polls that word of the mapped
// buffer instead of paying a stream synchronisation per hand-out. SOFT: the keys are finished here (ev_pick_key).
template <bool SAMP, bool SOFT = false, bool NTA = false>
__global__ void k_evict_pick_big(EvictParams p, int mode, int seq) {
  __shared__ unsigned long long s_key[32];
  __shared__ int s_node[32];
  __shared__ int s_best;
  __shared__ int s_pick[EV_PICK_K];  // hand-outs, written to the mapped host buffer once at the end (a store to system memory
                                     // per iteration sits on the critical path of the block-wide barriers)
  const int N = SAMP ? *p.samp_cnt : p.d.N;  // SAMP: i walks the sampled list, node_of(i) is the node
  auto node_of = [&](int i) { return SAMP ? p.samp_list[i] : i; };
  const int max_soft = SOFT ? ev_max_soft(p) : 0;
  if (threadIdx.x < EV_PICK_K) s_pick[threadIdx.x] = -1;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  auto better_kn = [](unsigned long long ka, int na, unsigned long long kb, int nb) {
    return na >= 0 && (nb < 0 || ka > kb || (ka == kb && na < nb));
  };
  unsigned long long bk = 0ull;  // this thread's best remaining candidate
  int bn = -1;
  auto rescan = [&](int skip) {
    bk = 0ull; bn = -1;
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
      if (n == skip || p.cand[node_of(n)] != 1) continue;
      const unsigned long long k = mode == EV_MODE_RECLAIM ? 0ull : ev_pick_key<SOFT, NTA>(p, node_of(n), max_soft);
      if (bn < 0 || k > bk) { bk = k; bn = n; }  // ascending n per thread: the first of equal keys stays
    }
  };
  auto warp_fold = [&]() {  // this warp's best into its shared slot
    unsigned long long wk = bk;
    int wn = bn;
    for (int o = 16; o; o >>= 1) {
      const unsigned long long ok = __shfl_xor_sync(0xffffffffu, wk, o);
      const int on = __shfl_xor_sync(0xffffffffu, wn, o);
      if (better_kn(ok, on, wk, wn)) { wk = ok; wn = on; }
    }
    if (lane == 0) { s_key[warp] = wk; s_node[warp] = wn; }
  };
  rescan(-1);
  warp_fold();
  __syncthreads();
  for (int it = 0; it < EV_PICK_K; ++it) {
    if (warp == 0) {
      unsigned long long gk = lane < nw ? s_key[lane] : 0ull;
      int gn = lane < nw ? s_node[lane] : -1;
      for (int o = 16; o; o >>= 1) {
        const unsigned long long ok = __shfl_xor_sync(0xffffffffu, gk, o);
        const int on = __shfl_xor_sync(0xffffffffu, gn, o);
        if (better_kn(ok, on, gk, gn)) { gk = ok; gn = on; }
      }
      if (lane == 0) {
        s_pick[it] = gn >= 0 ? node_of(gn) : -1;
        if (gn >= 0) p.cand[node_of(gn)] = 2;
        s_best = gn;
      }
    }
    __syncthreads();
    const int g = s_best;
    if (g < 0) break;  // exhausted: the remaining slots keep their -1
    if ((g % (int)blockDim.x) >> 5 == warp) {  // the warp of the thread that owned the node
      if (g % (int)blockDim.x == (int)threadIdx.x) rescan(g);  // (cand[g] = 2 was written by another thread: skip g by name)
      warp_fold();
    }
    __syncthreads();
  }
  __syncthreads();
  if (threadIdx.x < EV_PICK_K) {
    *reinterpret_cast<volatile int32_t *>(p.pick_node + threadIdx.x) = s_pick[threadIdx.x];
    __threadfence_system();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    *reinterpret_cast<volatile int32_t *>(p.pick_node + EV_PICK_K) = seq;
  }
}

// k_evict_pick, the common case (the candidates' keys fit in shared memory, N * 8 bytes): two-level selection with two
// block barriers in all. Phase 1, every warp on its own 1/32 of the nodes: EV_PICK_K rounds of a warp arg-max (each lane
// keeps the best of its ~N/1024 nodes in registers, the winner rescans its shared-memory entries) give the warp's first
// EV_PICK_K candidates in order. Phase 2, one warp: a 32-way merge of those sorted lists. Same order as the sequential
// tournament: key descending, node ascending. SOFT: the keys are finished while they are staged (ev_pick_key).
extern __shared__ unsigned long long ev_pick_cache[];
template <bool SAMP, bool SOFT = false, bool NTA = false>
__global__ void __launch_bounds__(1024) k_evict_pick(EvictParams p, int mode, int seq) {
  __shared__ unsigned long long l_key[32][EV_PICK_K];
  __shared__ int l_node[32][EV_PICK_K];
  __shared__ int s_pick[EV_PICK_K];
  const int N = SAMP ? *p.samp_cnt : p.d.N;  // SAMP: n walks the sampled list, node_of(n) is the node
  auto node_of = [&](int i) { return SAMP ? p.samp_list[i] : i; };
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int max_soft = SOFT ? ev_max_soft(p) : 0;
  for (int n = threadIdx.x; n < N; n += blockDim.x)  // key + 1 (never wraps: see ev_score_key), 0 = not a candidate
    ev_pick_cache[n] = p.cand[node_of(n)] == 1 ? (mode == EV_MODE_RECLAIM ? 1ull : ev_pick_key<SOFT, NTA>(p, node_of(n), max_soft) + 1ull)
                                               : 0ull;
  if (threadIdx.x < EV_PICK_K) s_pick[threadIdx.x] = -1;
  __syncwarp();  // a lane only ever reads the entries it wrote
  auto better_kn = [](unsigned long long ka, int na, unsigned long long kb, int nb) {
    return na >= 0 && (nb < 0 || ka > kb || (ka == kb && na < nb));
  };
  unsigned long long bk = 0ull;
  int bn = -1;
  auto rescan = [&]() {
    bk = 0ull; bn = -1;
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
      const unsigned long long k = ev_pick_cache[n];
      if (k == 0ull) continue;
      if (bn < 0 || k > bk) { bk = k; bn = n; }  // ascending n per thread: the first of equal keys stays
    }
  };
  rescan();
  for (int it = 0; it < EV_PICK_K; ++it) {
    unsigned long long wk = bk;
    int wn = bn;
    for (int o = 16; o; o >>= 1) {
      const unsigned long long ok = __shfl_xor_sync(0xffffffffu, wk, o);
      const int on = __shfl_xor_sync(0xffffffffu, wn, o);
      if (better_kn(ok, on, wk, wn)) { wk = ok; wn = on; }
    }
    if (lane == it) { l_key[warp][it] = wk; l_node[warp][it] = wn; }
    if (wn < 0) {  // this warp is out of candidates: the rest of its list says so
      if (lane > it && lane < EV_PICK_K) { l_key[warp][lane] = 0ull; l_node[warp][lane] = -1; }
      break;
    }
    if (bn == wn) { ev_pick_cache[wn] = 0ull; rescan(); }
  }
  __syncthreads();
  if (warp == 0) {
    // lane l walks warp l's list; its head is read at the top of every step (advancing the index and reloading inside the
    // branch below was compiled for sm_90a into a load of the slot after the new head, which dropped candidates)
    int hp = 0;
    for (int it = 0; it < EV_PICK_K; ++it) {
      const int cn = hp < EV_PICK_K ? l_node[lane][hp] : -1;
      unsigned long long gk = hp < EV_PICK_K ? l_key[lane][hp] : 0ull;
      int gn = cn;
      for (int o = 16; o; o >>= 1) {
        const unsigned long long ok = __shfl_xor_sync(0xffffffffu, gk, o);
        const int on = __shfl_xor_sync(0xffffffffu, gn, o);
        if (better_kn(ok, on, gk, gn)) { gk = ok; gn = on; }
      }
      if (gn < 0) break;
      if (lane == 0) { s_pick[it] = node_of(gn); p.cand[node_of(gn)] = 2; }
      if (cn == gn) hp += 1;
    }
  }
  __syncthreads();
  if (threadIdx.x < EV_PICK_K) {
    *reinterpret_cast<volatile int32_t *>(p.pick_node + threadIdx.x) = s_pick[threadIdx.x];
    __threadfence_system();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    *reinterpret_cast<volatile int32_t *>(p.pick_node + EV_PICK_K) = seq;
  }
}

// Statement.Evict for every victim (node.UpdateTask: Releasing += Resreq; predicates DeallocateFunc: RemovePod), then
// Statement.Pipeline of the preemptor (Pipelined += Resreq; predicates AllocateFunc: AddPod) on node cmd[0]
// `undo` != 0: the inverse in Statement.Discard's order (UnPipeline, then unevict the victims in reverse order), so that
// with non-integer requests the rows come back exactly as the reference's discard leaves them.
// With hn_used (nta_on), network-topology-aware's AllocateFunc / DeallocateFunc (network_topology_aware.go:309-340) book
// the request on the hypernode of every tier level that holds the node, dims 0, 1 and the task's present scalars, in
// the same order of events; thread d owns dimension d of every hypernode. Only the NTA instance books them.
template <bool NTA = false>
__global__ void k_evict_apply(EvictParams p, EvictTask t, int undo) {
  const int n = p.cmd[0], nv = p.cmd[1];
  const int N = p.d.N, R = p.d.R, K = p.d.K;
  const int d = threadIdx.x;
  const double sg = undo ? -1.0 : 1.0;
  auto hn_book = [&](double v, uint32_t has) {
    if constexpr (NTA) {
      if (d >= 2 && !(has & (1u << d))) return;
      for (int l = 0; l < p.c.nta_L; ++l) {
        const int h = p.hn_member[(size_t)l * N + n];
        if (h >= 0) p.hn_used[(size_t)d * p.hn_H + h] += v;
      }
    }
  };
  auto pipeline = [&]() {
    if (d < R) p.pip[(size_t)d * N + n] += sg * t.rec.req[d];
    if (NTA && d < R) hn_book(sg * t.rec.req[d], t.rec.has);
    if (p.c.has_predicates) {
      if (d >= 32 && d < 32 + K) p.kreq[(size_t)(d - 32) * N + n] += sg * t.rec.kreq[d - 32];
      if (d >= 48 && d < 50) p.knz[(size_t)(d - 48) * N + n] += sg * t.rec.knz[d - 48];
      if (d == 62) p.pod_count[n] += undo ? nv - 1 : 1 - nv;
    }
  };
  if (undo) pipeline();
  for (int i = 0; i < nv; ++i) {
    const int r = p.cmd[2 + (undo ? nv - 1 - i : i)];
    if (d < R) p.rel[(size_t)d * N + n] += sg * p.rt_req[(size_t)d * p.RT + r];
    if (NTA && d < R) hn_book(-sg * p.rt_req[(size_t)d * p.RT + r], p.rt_has[r]);
    if (p.c.has_predicates) {
      if (d >= 32 && d < 32 + K) p.kreq[(size_t)(d - 32) * N + n] -= sg * p.rt_kreq[(size_t)(d - 32) * p.RT + r];
      if (d >= 48 && d < 50) p.knz[(size_t)(d - 48) * N + n] -= sg * p.rt_knz[(size_t)(d - 48) * p.RT + r];
    }
    if (d == 63) p.rt_evicted[r] = undo ? 0 : 1;
  }
  if (!undo) pipeline();
}

// ---- topology-aware preemption (vc_topo.hpp) -----------------------------------------------------------------------
// k_evict_dryrun: SelectVictimsOnNode as a dry run on every node that passes the preemptor's predicates, one thread per
// node. Node n's scratch is [rt_off[n], rt_off[n+1]) of four slabs over the running tasks, so a node may run any number
// of pods; its victims stay in slab a for k_evict_select. GUARD: the pdb and cdp plugins vote (vct::topo_vote).
struct TopoDry {
  const uint32_t *cstat;  // [C][N]
  int klass;
  int32_t *a, *b;         // [RT]
  uint8_t *f, *g;         // [RT]
  uint8_t *ok;            // [N] 1 = the node is a candidate
  int32_t *nv;            // [N] its victim count
  long long *key;         // [4][N] pickOneNodeForPreemption's scores
  const int32_t *samp_list, *samp_cnt;  // SAMP: thread i runs on the i-th sampled node
};
template <bool SAMP, bool GUARD = false>
__global__ void __launch_bounds__(128) k_evict_dryrun(vct::TopoView v, vct::TopoTask t, TopoDry s) {
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (SAMP) {
    if (n >= *s.samp_cnt) return;
    n = s.samp_list[n];
  } else if (n >= v.N) {
    return;
  }
  uint8_t ok = 0;
  if (SAMP || (s.cstat[(size_t)s.klass * v.N + n] & CS_STATIC_OK)) {
    const int o = v.rt_off[n];
    const vct::TopoResult r = vct::topo_dry_run<GUARD>(v, t, n, s.a + o, s.b + o, s.f + o, s.g + o);
    ok = (uint8_t)r.ok;
    s.nv[n] = r.nv;
    for (int k = 0; k < 4; ++k) s.key[(size_t)k * v.N + n] = r.key[k];
  }
  s.ok[n] = ok;
}

// k_evict_select: one block. The predicate nodes' positions (NodeList order) and the candidates' ranks in scan order
// from the offset come from one block scan; the first numCandidates candidates compete on the four scores, ties going to
// the lower rank. The hand-out goes to mapped pinned memory: [0] node (-1: none), [1] victim count, [2]
// len(predicateNodes), [3] 1 when the victims do not fit the hand-out, [4..] victims in list order; the last store is
// `seq` into [EV_TOPO_SEQ]. SAMP: predicateNodes are k_evict_samp's list, positions are list positions (scan order).
#define EV_TOPO_SEQ (4 + EV_MAX_VICTIMS)
struct TopoSelect {
  const uint32_t *cstat;
  int klass, N;
  const uint8_t *ok;
  const int32_t *nv;
  const long long *key;
  const int32_t *rt_off, *victims;  // victims: slab a of k_evict_dryrun
  unsigned long long seed_k;        // offset_seed + k
  int pct, min_abs, max_abs;
  int32_t *out;
  int seq;
  const int32_t *samp_list, *samp_cnt;
};
template <bool SAMP>
__global__ void __launch_bounds__(1024) k_evict_select(TopoSelect s) {
  __shared__ int sp[1024], ss[1024];
  __shared__ long long wk[32][4];
  __shared__ long long wr[32];
  __shared__ int wn[32];
  __shared__ int s_off;
  const int tid = threadIdx.x, nt = blockDim.x, N = s.N;
  const int D = SAMP ? *s.samp_cnt : N;  // positions n in [0, D), of node node_of(n)
  auto node_of = [&](int n) { return SAMP ? s.samp_list[n] : n; };
  const int chunk = (D + nt - 1) / nt;
  const int lo = min(D, tid * chunk), hi = min(D, lo + chunk);
  auto pred = [&](int n) { return SAMP || (s.cstat[(size_t)s.klass * N + n] & CS_STATIC_OK) != 0; };
  int cp = 0, cs = 0;
  for (int n = lo; n < hi; ++n)
    if (pred(n)) { cp += 1; cs += s.ok[node_of(n)]; }
  sp[tid] = cp; ss[tid] = cs;
  if (tid == 0) s_off = 0;
  __syncthreads();
  for (int o = 1; o < nt; o <<= 1) {  // inclusive scan
    const int a = tid >= o ? sp[tid - o] : 0, b = tid >= o ? ss[tid - o] : 0;
    __syncthreads();
    sp[tid] += a; ss[tid] += b;
    __syncthreads();
  }
  const long long P = sp[nt - 1], S = ss[nt - 1];
  const long long pbase = sp[tid] - cp, sbase = ss[tid] - cs;
  volatile int32_t *out = s.out;
  if (P == 0) {
    if (tid == 0) {
      out[0] = -1; out[1] = 0; out[2] = 0; out[3] = 0;
      __threadfence_system();
      out[EV_TOPO_SEQ] = s.seq;
    }
    return;
  }
  const long long offset = (long long)(vct::splitmix64(s.seed_k) % (unsigned long long)P);
  const long long numc = vct::num_candidates(P, s.pct, s.min_abs, s.max_abs);
  if (numc < 0) {
    if (tid == 0) {
      out[0] = -1; out[1] = 0; out[2] = (int32_t)P; out[3] = 2;
      __threadfence_system();
      out[EV_TOPO_SEQ] = s.seq;
    }
    return;
  }
  int before = 0;  // candidates whose position is below the offset
  {
    long long pi = pbase;
    for (int n = lo; n < hi; ++n)
      if (pred(n)) { if (s.ok[node_of(n)] && pi < offset) before += 1; pi += 1; }
  }
  if (before) atomicAdd(&s_off, before);
  __syncthreads();
  const long long S_off = s_off;
  long long bk[4] = {0, 0, 0, 0}, br = -1;
  int bn = -1;
  {
    long long pi = pbase, si = sbase;
    for (int n = lo; n < hi; ++n) {
      if (!pred(n)) continue;
      const int m = node_of(n);
      if (s.ok[m]) {
        const long long rank = pi >= offset ? si - S_off : (S - S_off) + si;
        if (rank < numc) {
          long long k[4];
          for (int x = 0; x < 4; ++x) k[x] = s.key[(size_t)x * N + m];
          if (vct::topo_better(k, rank, bk, br)) { for (int x = 0; x < 4; ++x) bk[x] = k[x]; br = rank; bn = m; }
        }
        si += 1;
      }
      pi += 1;
    }
  }
  const int lane = tid & 31, warp = tid >> 5;
  for (int o = 16; o; o >>= 1) {
    long long ok[4];
    for (int x = 0; x < 4; ++x) ok[x] = __shfl_xor_sync(0xffffffffu, bk[x], o);
    const long long orr = __shfl_xor_sync(0xffffffffu, br, o);
    const int on = __shfl_xor_sync(0xffffffffu, bn, o);
    if (vct::topo_better(ok, orr, bk, br)) { for (int x = 0; x < 4; ++x) bk[x] = ok[x]; br = orr; bn = on; }
  }
  if (lane == 0) { for (int x = 0; x < 4; ++x) wk[warp][x] = bk[x]; wr[warp] = br; wn[warp] = bn; }
  __syncthreads();
  if (warp == 0) {
    const int nw = (nt + 31) >> 5;
    for (int x = 0; x < 4; ++x) bk[x] = lane < nw ? wk[lane][x] : 0;
    br = lane < nw ? wr[lane] : -1;
    bn = lane < nw ? wn[lane] : -1;
    for (int o = 16; o; o >>= 1) {
      long long ok[4];
      for (int x = 0; x < 4; ++x) ok[x] = __shfl_xor_sync(0xffffffffu, bk[x], o);
      const long long orr = __shfl_xor_sync(0xffffffffu, br, o);
      const int on = __shfl_xor_sync(0xffffffffu, bn, o);
      if (vct::topo_better(ok, orr, bk, br)) { for (int x = 0; x < 4; ++x) bk[x] = ok[x]; br = orr; bn = on; }
    }
    if (lane == 0) wn[0] = bn;
  }
  __syncthreads();
  const int w = wn[0];
  const int nv = w >= 0 ? s.nv[w] : 0;
  if (w >= 0)
    for (int i = tid; i < min(nv, EV_MAX_VICTIMS); i += nt) out[4 + i] = s.victims[s.rt_off[w] + i];
  if (tid == 0) { out[0] = w; out[1] = nv; out[2] = (int32_t)P; out[3] = nv > EV_MAX_VICTIMS ? 1 : 0; }
  __threadfence_system();
  __syncthreads();
  if (tid == 0) {
    __threadfence_system();
    out[EV_TOPO_SEQ] = s.seq;
  }
}

// ---- feasible-node sampling (util/predicate_helper.go:43-140) -------------------------------------------------------
// k_evict_samp: PredicateNodes of one preemptor or reclaimer in the single-worker reading, before the pick (normal
// reading) or the dry runs (topology-aware reading). The scanned list is the NodeList, or with `filtered` (allocate left
// the task a NodesFitErrors entry with node errors) the nodes that pass the static verdict, in NodeList order
// (ssn.FilterOutUnschedulableAndUnresolvableNodesForTask); P is its length. The scan visits list[(start + i) % P] and
// keeps the first numNodesToFind(P) nodes passing the static verdict (ssn.PredicateForPreemptAction). processed is the
// scan position of the last node kept + 1, or P when fewer pass, and the index becomes (start + processed) % P; an empty
// list returns early and leaves the index alone. The kept nodes go to list[0, cnt) in scan order. Only the static bit
// decides the sample: k_evict_rank's necessary conditions prune inside it through the pick.
// One block, as k_evict_select: every thread owns a contiguous chunk of nodes, a block scan gives the positions in the
// scanned list and the ranks among the passing nodes; the rotated rank of a passing node counts from the first passing
// node at or after `start`. idx_in may alias idx_out (read before the first barrier, written after the last).
// SOFT: the largest soft-taint count over the kept nodes (TaintToleration's normalisation set under sampling) goes to
// *soft_word as (soft_seq << 8) | max (EvictParams::soft_word).
struct EvictSamp {
  const uint32_t *cstat;
  int klass, N, filtered;
  int pct, min_nodes, min_pct;  // vc_conf's percentage / minimum node count / minimum percentage to find
  const int32_t *idx_in;
  int32_t *idx_out, *list, *cnt;
  unsigned long long *soft_word;
  unsigned long long soft_seq;
};
template <bool SOFT = false>
__global__ void __launch_bounds__(1024) k_evict_samp(EvictSamp s) {
  __shared__ int sp[1024], ss[1024];
  __shared__ int s_start, s_before, s_proc;
  __shared__ unsigned s_soft;
  const int tid = threadIdx.x, nt = blockDim.x, N = s.N;
  const int chunk = (N + nt - 1) / nt;
  const int lo = min(N, tid * chunk), hi = min(N, lo + chunk);
  auto pass = [&](int n) { return (s.cstat[(size_t)s.klass * N + n] & CS_STATIC_OK) != 0; };
  int cp = 0, cs = 0;
  for (int n = lo; n < hi; ++n) {
    const bool ok = pass(n);
    cp += (ok || !s.filtered) ? 1 : 0;
    cs += ok ? 1 : 0;
  }
  sp[tid] = cp; ss[tid] = cs;
  if (tid == 0) { s_start = *s.idx_in; s_before = 0; s_proc = -1; s_soft = 0u; }
  __syncthreads();
  for (int o = 1; o < nt; o <<= 1) {  // inclusive scan
    const int a = tid >= o ? sp[tid - o] : 0, b = tid >= o ? ss[tid - o] : 0;
    __syncthreads();
    sp[tid] += a; ss[tid] += b;
    __syncthreads();
  }
  const int P = sp[nt - 1], S = ss[nt - 1];
  if (P == 0) {
    if (tid == 0) {
      *s.cnt = 0; *s.idx_out = s_start;
      if (SOFT) *s.soft_word = s.soft_seq << 8;
    }
    return;
  }
  const int start = s_start % P;
  const int tf = vch::num_feasible_nodes_to_find(P, s.pct, s.min_nodes, s.min_pct);
  const int M = min(tf, S);
  int before = 0;  // passing nodes at positions below start
  {
    int pi = sp[tid] - cp;
    for (int n = lo; n < hi; ++n) {
      const bool ok = pass(n);
      if (!ok && s.filtered) continue;
      if (ok && pi < start) before += 1;
      pi += 1;
    }
  }
  if (before) atomicAdd(&s_before, before);
  __syncthreads();
  const int B = s_before;
  {
    int pi = sp[tid] - cp, si = ss[tid] - cs;
    unsigned ms = 0u;
    for (int n = lo; n < hi; ++n) {
      const bool ok = pass(n);
      if (!ok && s.filtered) continue;
      if (ok) {
        const int rank = pi >= start ? si - B : (S - B) + si;
        if (rank < M) {
          s.list[rank] = n;
          if (SOFT) ms = max(ms, (s.cstat[(size_t)s.klass * N + n] >> CS_SOFT_SHIFT) & 0xffu);
        }
        if (rank == tf - 1) s_proc = (pi - start + P) % P + 1;  // the numNodesToFind-th node found: the scan stops there
        si += 1;
      }
      pi += 1;
    }
    if (SOFT && ms) atomicMax(&s_soft, ms);
  }
  __syncthreads();
  if (tid == 0) {
    const int processed = s_proc >= 0 ? s_proc : P;
    *s.cnt = M;
    *s.idx_out = (int)(((long long)start + processed) % P);
    if (SOFT) *s.soft_word = (s.soft_seq << 8) | s_soft;
  }
}

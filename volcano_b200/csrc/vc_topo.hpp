// vc_topo.hpp — the preempt action's topology-aware reading (enableTopologyAwarePreemption, actions/preempt/preempt.go:
// 475-1015): SelectVictimsOnNode as a dry run on one node, and the pieces of the candidate pick. Written once for the host
// and the device: k_evict_dryrun (vc_evict.cuh) runs topo_dry_run on every predicate node at once, and a test shim runs it
// on the CPU. Every floating-point operation is the reference's, in its order (the library builds with -fmad=false).
#pragma once
#include <cstdint>

#include "../../include/vcalloc.h"

#if defined(__CUDACC__)
#define VC_HD __host__ __device__ __forceinline__
#else
#include <cmath>
#define VC_HD inline
#endif

namespace vct {

// the offset of the k-th dry run of one vc_preempt_run: splitmix64(seed + k) mod len(predicateNodes)
VC_HD uint64_t splitmix64(uint64_t x) {
  uint64_t z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// calculateNumCandidates, preempt.go:581-597
VC_HD int64_t num_candidates(int64_t num_nodes, int pct, int min_abs, int max_abs) {
  int64_t n = num_nodes * pct / 100;
  if (n < min_abs) n = min_abs;
  if (n > max_abs) n = max_abs;
  if (n > num_nodes) n = num_nodes;
  return n;
}

VC_HD bool le_eps(double l, double r) { return l < r || fabs(l - r) < 0.1; }  // lessEqualFunc, api/resource_info.go:430-435
VC_HD double share_of(double l, double r) { return r == 0 ? (l == 0 ? 0.0 : 1.0) : l / r; }

// api.Resource with the presence semantics of its ScalarResources map (proportion's simulated queue allocation)
struct TRes {
  double v[VC_MAX_DIMS];
  uint32_t has;
  int nil;
};
VC_HD void tres_add(TRes &a, const double *rq, uint32_t rq_has, int R) {  // Resource.Add :277-290
  a.v[0] += rq[0]; a.v[1] += rq[1];
  for (int d = 2; d < R; ++d)
    if ((rq_has >> d) & 1u) { a.nil = 0; a.has |= 1u << d; a.v[d] += rq[d]; }
}
VC_HD void tres_sub(TRes &a, const double *rq, uint32_t rq_has, int R) {  // Resource.sub :308-320
  a.v[0] -= rq[0]; a.v[1] -= rq[1];
  if (a.nil) return;
  for (int d = 2; d < R; ++d)
    if ((rq_has >> d) & 1u) { a.has |= 1u << d; a.v[d] -= rq[d]; }
}

struct TopoView {  // the session as the dry run reads it; all pointers in one address space
  int R, N, J, RT, pods_dim;
  int n_plugins;
  int32_t plugin[VC_MAX_PLUGINS], tier[VC_MAX_PLUGINS];
  uint32_t enabled[VC_MAX_PLUGINS];
  int task_order_prio;                     // priority has EnabledTaskOrder
  const double *idle, *rel, *pip;          // [R][N] node rows as the session stands
  const int32_t *rt_off, *rt_idx;          // node.Tasks as CSR over nodes, ascending running-task index
  const double *rt_req;                    // [R][RT]
  const uint32_t *rt_has, *rt_flags, *rt_uid;
  const int32_t *rt_job, *rt_prio;         // TaskInfo.Priority
  const int64_t *rt_podidx, *rt_ts;
  const uint8_t *rt_evicted;               // Releasing in this session
  const int32_t *rt_pod_prio;              // PodPriority(pod): Pod.Spec.Priority, 0 when nil
  const int64_t *rt_start;                 // Pod.Status.StartTime in ns, VC_START_TIME_UNSET when nil
  const int32_t *j_queue, *j_prio, *j_min, *j_ready, *j_pbe;
  const uint32_t *j_rank;                  // JobOrderFn's final tie-break (creation time, UID)
  const double *j_alloc, *j_share;         // drf: [R][J] attr.allocated, [J] attr.share
  double total[VC_MAX_DIMS];               // drf.totalResource
  uint32_t total_has;
  // GUARD instances (pdb / cdp vote): vc_victim_guards on the device
  const uint8_t *rt_guard;                 // [RT] VCT_GUARD_* bits
  const int32_t *pdb_off, *pdb, *pdb_allowed;  // its CSR of the PDBs counting each task, DisruptionsAllowed per PDB
};
#define VCT_GUARD_NO_LABELS 1  // pdb skips the pod (pdb.go:87-90)
#define VCT_GUARD_PDB_NEVER 2  // no labels, or a PDB with DisruptionsAllowed <= 0 counts it: pdb never returns it
#define VCT_GUARD_CDP 4        // cdp protects it: cooldown-until after now (cdp.go:87-96)

struct TopoTask {  // the preemptor and what the simulate hooks start from
  int job, queue, intra;                   // intra: victims from the preemptor's own job (preempt.go:252-268)
  int job_prio, task_prio;
  double req[VC_MAX_DIMS];
  uint32_t has;                            // Resreq's scalar keys (bits >= 2)
  int sim_update;                          // proportion has EnabledPreemptable or EnabledAllocatable: remove / add run
  int sim_state;                           // proportion's PrePredicateFn wrote the state (EnabledPredicate)
  int sim_alloc;                           // proportion has EnabledAllocatable: SimulateAllocatableFn reads the state
  int q_exists;                            // the preemptor's queue is in proportion's queueOpts
  TRes qalloc;                             // its attr.allocated when the preemptor is tried
  double qdes[VC_MAX_DIMS];
  uint32_t qdes_has;
  int64_t now_ns;                          // time.Now() for victims without a StartTime
};

struct TopoResult {
  int ok, nv;                              // a candidate with nv victims (victims in the first slab)
  long long key[4];                        // pickOneNodeForPreemption's scores, larger is better
};

VC_HD bool topo_filter(const TopoView &v, const TopoTask &t, int r) {  // the action's filter, preempt.go:198-214 / :252-268
  if (v.rt_evicted[r]) return false;
  const uint32_t f = v.rt_flags[r];
  if (!(f & VC_RT_PREEMPTABLE) || !(f & (VC_RT_RUNNING | VC_RT_BOUND))) return false;
  const int j = v.rt_job[r];
  if (t.intra) return j == t.job;
  return j >= 0 && j != t.job && v.j_queue[j] == t.queue;
}
VC_HD double topo_drf_share(const TopoView &v, const double *a) {  // drf.calculateShare :566-578
  double res = 0;
  for (int d = 0; d < v.R; ++d) {
    if (d >= 2 && !((v.total_has >> d) & 1u)) continue;
    if (!(v.total[d] >= 0.1)) continue;
    const double sh = share_of(a[d], v.total[d]);
    if (sh > res) res = sh;
  }
  return res;
}
// pdb.go:83-124 for candidate a[i]: it is returned unless, for some PDB counting it, the labelled candidates a[0..i] counted
// by that PDB outnumber its DisruptionsAllowed (the budget of the call went below zero at a[i]). Counting needs no state, so
// the dry run's scratch stays one slab entry per task of the node whatever the number of PDBs.
VC_HD bool topo_pdb_returns(const TopoView &v, const int32_t *a, int i) {
  const int r = a[i];
  if (v.rt_guard[r] & VCT_GUARD_NO_LABELS) return false;
  for (int x = v.pdb_off[r]; x < v.pdb_off[r + 1]; ++x) {
    const int q = v.pdb[x];
    int left = v.pdb_allowed[q];
    for (int k = 0; k <= i && left >= 0; ++k) {
      const int rk = a[k];
      if (v.rt_guard[rk] & VCT_GUARD_NO_LABELS) continue;
      for (int y = v.pdb_off[rk]; y < v.pdb_off[rk + 1]; ++y)
        if (v.pdb[y] == q) { left -= 1; break; }
    }
    if (left < 0) return false;
  }
  return true;
}
// one voter of ssn.Preemptable over the candidates a[0..m): g[i] = 1 when it returns a[i]; -> number returned
template <bool GUARD = false>
VC_HD int topo_vote(const TopoView &v, const TopoTask &t, int pl, const int32_t *a, int m, uint8_t *g) {
  int cnt = 0;
  double ls = 0;
  if (pl == VC_PLUGIN_DRF) {
    double la[VC_MAX_DIMS];
    for (int d = 0; d < v.R; ++d) la[d] = v.j_alloc[(size_t)d * v.J + t.job] + t.req[d];
    ls = topo_drf_share(v, la);
  }
  for (int i = 0; i < m; ++i) {
    const int r = a[i], j = v.rt_job[r];
    bool y = false;
    if (pl == VC_PLUGIN_CONFORMANCE) {  // conformance.go:46-63
      y = !(v.rt_flags[r] & VC_RT_CRITICAL);
    } else if (GUARD && pl == VC_PLUGIN_CDP) {
      y = !(v.rt_guard[r] & VCT_GUARD_CDP);
    } else if (GUARD && pl == VC_PLUGIN_PDB) {
      y = !(v.rt_guard[r] & VCT_GUARD_PDB_NEVER) && topo_pdb_returns(v, a, i);
    } else if (j < 0) {
      y = false;
    } else if (pl == VC_PLUGIN_GANG) {  // gang.go:97-129: the job's occupancy drops with every victim it gave
      int occ = v.j_ready[j];
      for (int k = 0; k < i; ++k)
        if (g[k] && v.rt_job[a[k]] == j) occ -= 1;
      y = occ > v.j_min[j];
    } else if (pl == VC_PLUGIN_PRIORITY) {  // priority.go:110-148
      y = j != t.job ? v.j_prio[j] < t.job_prio : v.rt_prio[r] < t.task_prio;
    } else {  // drf.go:222-261: allocations[job].Sub(preemptee.Resreq) for every candidate of the job, in order
      double ra[VC_MAX_DIMS];
      for (int d = 0; d < v.R; ++d) {
        ra[d] = v.j_alloc[(size_t)d * v.J + j];
        for (int k = 0; k <= i; ++k)
          if (v.rt_job[a[k]] == j) ra[d] -= v.rt_req[(size_t)d * v.RT + a[k]];
      }
      const double rs = topo_drf_share(v, ra);
      y = ls < rs || fabs(ls - rs) <= 0.000001;
    }
    g[i] = y ? 1 : 0;
    cnt += y ? 1 : 0;
  }
  return cnt;
}
VC_HD bool topo_run_less(const TopoView &v, int l, int r) {  // TaskOrderFn: priority, then util.LessFn's pod index / time / UID
  if (v.task_order_prio && v.rt_prio[l] != v.rt_prio[r]) return v.rt_prio[l] > v.rt_prio[r];
  const int64_t il = v.rt_podidx[l], ir = v.rt_podidx[r];
  if (il < 0 || ir < 0 || il == ir) {
    if (v.rt_ts[l] == v.rt_ts[r]) return v.rt_uid[l] < v.rt_uid[r];
    return v.rt_ts[l] < v.rt_ts[r];
  }
  return !(il > ir);
}
VC_HD bool topo_job_less(const TopoView &v, int l, int r) {  // JobOrderFn over the tiers
  for (int i = 0; i < v.n_plugins; ++i) {
    if (!(v.enabled[i] & VC_EN_JOB_ORDER)) continue;
    int c = 0;
    if (v.plugin[i] == VC_PLUGIN_PRIORITY) {
      c = v.j_prio[l] > v.j_prio[r] ? -1 : (v.j_prio[l] < v.j_prio[r] ? 1 : 0);
    } else if (v.plugin[i] == VC_PLUGIN_GANG) {
      const bool lr = v.j_ready[l] + v.j_pbe[l] >= v.j_min[l], rr = v.j_ready[r] + v.j_pbe[r] >= v.j_min[r];
      c = (lr && rr) ? 0 : (lr ? 1 : (rr ? -1 : 0));
    } else if (v.plugin[i] == VC_PLUGIN_DRF) {
      c = v.j_share[l] == v.j_share[r] ? 0 : (v.j_share[l] < v.j_share[r] ? -1 : 1);
    }
    if (c != 0) return c < 0;
  }
  return v.j_rank[l] < v.j_rank[r];
}
// the less function of ssn.BuildVictimsPriorityQueue (session_plugins.go:1092-1135). Every victim of this action sits in
// the preemptor's queue, so the queue comparison never decides. It is not a strict weak order (util.LessFn compares pod
// indices when both names carry one and creation times otherwise), so the victims go through the Go heap itself.
VC_HD bool topo_victim_first(const TopoView &v, int l, int r) {
  const int lj = v.rt_job[l], rj = v.rt_job[r];
  if (lj == rj) return !topo_run_less(v, l, r);
  return !topo_job_less(v, lj, rj);
}

// SimulateAllocatableFn(queue, preemptor) && preemptor.InitResreq.LessEqual(node.FutureIdle(), Zero) on the dry-run node
VC_HD bool topo_fits(const TopoView &v, const TopoTask &t, int n, const double *idle, const TRes &qa) {
  if (t.sim_alloc) {  // proportion.go:436-455, LessEqualWithDimensionAndResourcesName(allocated + req, deserved, req)
    if (!t.sim_state || !t.q_exists) return false;
    TRes fu = qa;
    tres_add(fu, t.req, t.has, v.R);
    bool ok = true;
    if (t.req[0] > 0 && fu.v[0] > t.qdes[0]) ok = false;
    if (t.req[1] > 0 && fu.v[1] > t.qdes[1]) ok = false;
    if (!fu.nil)
      for (int d = 2; d < v.R; ++d) {
        if (!((t.has >> d) & 1u) || d == v.pods_dim) continue;
        const double lq = ((fu.has >> d) & 1u) ? fu.v[d] : 0.0, rq = ((t.qdes_has >> d) & 1u) ? t.qdes[d] : 0.0;
        if (t.req[d] > 0 && lq > rq) ok = false;
      }
    if (!ok) return false;
  }
  for (int d = 0; d < v.R; ++d) {
    if (d >= 2 && !((t.has >> d) & 1u)) continue;
    const double fi = (idle[d] + v.rel[(size_t)d * v.N + n]) - v.pip[(size_t)d * v.N + n];
    if (!le_eps(t.req[d], fi)) return false;
  }
  return true;
}

// SelectVictimsOnNode (preempt.go:708-842) on node n. a, b: int scratch, f, g: byte scratch, each with room for the
// node's tasks. On success the victims are a[0..nv) in the reference's list order (reprieve order). GUARD: the pdb and cdp
// plugins vote too.
template <bool GUARD = false>
VC_HD TopoResult topo_dry_run(const TopoView &v, const TopoTask &t, int n, int32_t *a, int32_t *b, uint8_t *f, uint8_t *g) {
  TopoResult res;
  res.ok = 0; res.nv = 0;
  res.key[0] = res.key[1] = res.key[2] = res.key[3] = 0;
  const int R = v.R;
  int m = 0;
  for (int x = v.rt_off[n]; x < v.rt_off[n + 1]; ++x)
    if (topo_filter(v, t, v.rt_idx[x])) a[m++] = v.rt_idx[x];
  // ssn.Preemptable (session_plugins.go:211-259): intersect per tier; an empty answer resets the list to nil
  bool nil = true;
  int i = 0;
  while (i < v.n_plugins) {
    const int tier = v.tier[i];
    for (int x = i; x < v.n_plugins && v.tier[x] == tier; ++x) {
      if (!(v.enabled[x] & VC_EN_PREEMPTABLE)) continue;
      const int pl = v.plugin[x];
      if (pl != VC_PLUGIN_GANG && pl != VC_PLUGIN_CONFORMANCE && pl != VC_PLUGIN_PRIORITY && pl != VC_PLUGIN_DRF &&
          !(GUARD && (pl == VC_PLUGIN_PDB || pl == VC_PLUGIN_CDP)))
        continue;
      if (topo_vote<GUARD>(v, t, pl, a, m, g) == 0) { nil = true; break; }
      int left = 0;
      for (int k = 0; k < m; ++k) {
        f[k] = nil ? g[k] : (uint8_t)(f[k] & g[k]);
        left += f[k];
      }
      nil = left == 0;
    }
    while (i < v.n_plugins && v.tier[i] == tier) ++i;
    if (!nil) break;
  }
  int nv = 0;
  if (!nil)
    for (int k = 0; k < m; ++k)
      if (f[k]) b[nv++] = a[k];
  // util.ValidateVictims (scheduler_helper.go:313-329)
  for (int d = 0; d < R; ++d) {
    double fi = (v.idle[(size_t)d * v.N + n] + v.rel[(size_t)d * v.N + n]) - v.pip[(size_t)d * v.N + n];
    for (int k = 0; k < nv; ++k) fi += v.rt_req[(size_t)d * v.RT + b[k]];
    if (d >= 2 && !((t.has >> d) & 1u)) continue;
    if (!le_eps(t.req[d], fi)) return res;
  }
  // container/heap as util.PriorityQueue uses it, in place: Push in list order (append + up); each Pop swaps the root to
  // the end of the live heap and sifts down, so the k-th popped victim ends at b[nv - 1 - k]
  for (int k = 1; k < nv; ++k)
    for (int j = k; j > 0;) {
      const int i = (j - 1) / 2;
      if (!topo_victim_first(v, b[j], b[i])) break;
      const int x = b[i]; b[i] = b[j]; b[j] = x;
      j = i;
    }
  auto pop = [&](int size) {  // heap of `size` entries -> its root, now at b[size - 1]
    const int n1 = size - 1;
    int x = b[0]; b[0] = b[n1]; b[n1] = x;
    for (int i = 0;;) {
      const int j1 = 2 * i + 1;
      if (j1 >= n1) break;
      int j = j1;
      if (j1 + 1 < n1 && topo_victim_first(v, b[j1 + 1], b[j1])) j = j1 + 1;
      if (!topo_victim_first(v, b[j], b[i])) break;
      x = b[i]; b[i] = b[j]; b[j] = x;
      i = j;
    }
    return b[n1];
  };
  double idle[VC_MAX_DIMS];
  for (int d = 0; d < R; ++d) idle[d] = v.idle[(size_t)d * v.N + n];
  TRes qa = t.qalloc;
  double rq[VC_MAX_DIMS];
  auto load = [&](int r) { for (int d = 0; d < R; ++d) rq[d] = v.rt_req[(size_t)d * v.RT + r]; };
  int popped = 0;
  for (; popped < nv;) {  // pop, removeTask, then test (nothing is tested before the first removal)
    const int r = pop(nv - popped);
    load(r);
    if (t.sim_update) {  // SimulateRemoveTaskFn fails without the state or the queue's attr
      if (!t.sim_state || !t.q_exists) return res;
      tres_sub(qa, rq, v.rt_has[r], R);
    }
    for (int d = 0; d < R; ++d) idle[d] += rq[d];  // NodeInfo.RemoveTask of a Running / Bound task
    popped += 1;
    if (topo_fits(v, t, n, idle, qa)) break;
  }
  if (popped == 0) return res;
  int out = 0;
  for (int k = popped - 1; k >= 0; --k) {  // reprieve, last popped first
    const int r = b[nv - 1 - k];
    load(r);
    if (t.sim_update) tres_add(qa, rq, v.rt_has[r], R);
    for (int d = 0; d < R; ++d) idle[d] -= rq[d];  // NodeInfo.AddTask
    if (!topo_fits(v, t, n, idle, qa)) {
      if (t.sim_update) tres_sub(qa, rq, v.rt_has[r], R);
      for (int d = 0; d < R; ++d) idle[d] += rq[d];
      a[out++] = r;
    }
  }
  if (out == 0) return res;  // "expected at least one victim pod"
  // pickOneNodeForPreemption's scores (preempt.go:910-941) and GetEarliestPodStartTime (:983-1005)
  const int32_t p0 = v.rt_pod_prio[a[0]];
  long long sum = 0, maxp = p0;
  auto start = [&](int r) { return v.rt_start[r] == VC_START_TIME_UNSET ? (long long)t.now_ns : (long long)v.rt_start[r]; };
  long long earliest = start(a[0]);
  for (int k = 0; k < out; ++k) {
    const long long pp = v.rt_pod_prio[a[k]];
    sum += pp + 2147483648ll;
    if (pp == maxp) { if (start(a[k]) < earliest) earliest = start(a[k]); }
    else if (pp > maxp) { maxp = pp; earliest = start(a[k]); }
  }
  res.ok = 1; res.nv = out;
  res.key[0] = -(long long)p0; res.key[1] = -sum; res.key[2] = -(long long)out; res.key[3] = earliest;
  return res;
}

// lexicographic "better" of two candidates: larger keys win, ties go to the earlier position in the scan
VC_HD bool topo_better(const long long *ka, long long pa, const long long *kb, long long pb) {
  if (pb < 0) return pa >= 0;
  if (pa < 0) return false;
  for (int i = 0; i < 4; ++i)
    if (ka[i] != kb[i]) return ka[i] > kb[i];
  return pa < pb;
}

}  // namespace vct

// vc_device.cuh — device-side data layout and the per-(task,node) predicate / score math
// shared by the dense score-matrix kernel (K1) and the persistent commit kernel (K2).
//
// Everything here is fp64 / int arithmetic written in the exact operation order of the
// reference (file:line cited per function, paths relative to volcano's pkg/scheduler);
// the translation unit is compiled with -fmad=false so no mul+add is contracted.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/vcalloc.h"

#define VC_MIN_RESOURCE 0.1  // api/resource_info.go:45-47
#define VC_MAX_NODE_SCORE 100

// cstat word per (class, node): everything of the predicate/score chain that is static
// within a scheduling cycle, precomputed once per session by k_class_static.
#define CS_STATIC_OK 1u        // predicates(static part) && tdm predicate, as enabled in conf
#define CS_TDM_ORDER_ERR 2u    // tdm nodeOrderFn returns an error (inactive zone, tdm.go:181-184)
#define CS_TDM_ORDER_MAX 4u    // tdm nodeOrderFn returns MaxNodeScore (tdm.go:186-191)
#define CS_SOFT_SHIFT 8        // bits 8..15: intolerable PreferNoSchedule taints
#define CS_NAFF_SHIFT 16       // bits 16..31: sum of matching preferred nodeAffinity weights

// internal flag in a group's presence word (bits >= VC_MAX_DIMS are free): the tasks of the group belong to a
// soft-mode topology job, so network-topology-aware scores them as network-aware pods, not by hypernode binpacking
#define VC_HAS_TOPO_TASK 0x40000000u

struct DevConf {
  int n_plugins;
  int plugin[VC_MAX_PLUGINS];
  int tier[VC_MAX_PLUGINS];
  uint32_t enabled[VC_MAX_PLUGINS];
  int binpack_weight;
  int binpack_dim_weight[VC_MAX_DIMS];
  int w_least, w_most, w_balanced, w_node_affinity, w_taint;
  uint32_t predicates_enable;
  int enable_ecache;
  // derived on the host
  int has_gang, has_drf, has_proportion, has_predicates;
  int pred_predicates;  // predicates plugin contributes to ssn.PredicateFn
  int taint_batch;      // nodeorder BatchNodeOrderFn scores TaintToleration
  int batch_any;        // some BatchNodeOrderFn yields entries
  int has_future;       // any Releasing/Pipelined resource at open -> FutureIdle != Idle possible
  int soft_active;      // taint_batch && some node carries a PreferNoSchedule taint
  // feasible-node sampling (util/predicate_helper.go:43-140 with CalculateNumOfFeasibleNodesToFind): stop after
  // `to_find` feasible nodes, scanning from lastProcessedNodeIndex; 0 = every node is evaluated (parity mode)
  int to_find;
  int last_idx0;
  // network-topology-aware, hypernode-level binpacking of pods without a network topology
  int nta_plugin;       // plugin has EnabledNodeOrder (its BatchNodeOrderFn is registered)
  int nta_tables;       // per-CTA hypernode lists are built (nta_on, or soft-mode topology jobs exist)
  int nta_on;           // ... and hypernode.binpack.normal-pod.enable
  int nta_weight;
  int nta_dim_weight[VC_MAX_DIMS];
  int nta_L;            // tier levels min_tier..max_tier (cluster top hypernode included)
  double tier_w[VC_MAX_TIERS];  // math.Pow(fading, tier-1), computed on the host
  double tier_w_total;
};

struct DevDims {
  int N, T, J, Q, C, R, K, Wl, Wt, NR, Z, pods_dim;
  int node_begin, node_end;  // node shard owned by this process
};

__host__ __device__ __forceinline__ bool le_eps(double l, double r) {  // api/resource_info.go:430-435
  return l < r || fabs(l - r) < VC_MIN_RESOURCE;
}

// floor(a / b) for integer-valued doubles 0 <= a, 0 < b (b < 2^52): the int64 divisions of the
// upstream scorers done on the fp64 pipe. a / b is correctly rounded, so trunc() is off by at
// most one; the fma residual is exact for these magnitudes and fixes it.
__device__ __forceinline__ double idiv_floor(double a, double b) {
  double q = trunc(a / b);
  double r = fma(-q, b, a);
  if (r < 0.0) q -= 1.0;
  else if (r >= b) q += 1.0;
  return q;
}

// leastRequestedScore / mostRequestedScore (kube-scheduler v1.35 noderesources, restated)
__device__ __forceinline__ double least_requested_score(double requested, double capacity) {
  if (capacity == 0.0) return 0.0;
  if (requested > capacity) return 0.0;
  return idiv_floor((capacity - requested) * (double)VC_MAX_NODE_SCORE, capacity);
}
__device__ __forceinline__ double most_requested_score(double requested, double capacity) {
  if (capacity == 0.0) return 0.0;
  if (requested > capacity) requested = capacity;
  return idiv_floor(requested * (double)VC_MAX_NODE_SCORE, capacity);
}

// One task's request record, staged in shared memory / registers.
struct TaskRec {
  double req[VC_MAX_DIMS];
  double kreq[VC_MAX_KDIMS];
  double knz[2];
  uint32_t has;
  int klass;
};

// NodeView concept: alloc(d) used(d) idle(d) rel(d) pip(d) kalloc(k) kreq(k) knz(k) max_tasks() pod_count()

// BinPackingScore, plugins/binpack/binpack.go:206-261
template <class NV>
__device__ __forceinline__ double binpack_score(const DevConf &c, int R, const TaskRec &t, const NV &nv) {
  double score = 0.0;
  int weight_sum = 0;
  for (int d = 0; d < R; ++d) {
    double request = t.req[d];
    if (d >= 2 && !(t.has & (1u << d))) continue;
    if (!(request >= VC_MIN_RESOURCE)) continue;  // ResourceNames(), resource_info.go:185-203
    int w = c.binpack_dim_weight[d];
    if (w < 0) continue;
    double allocate = nv.alloc(d);
    double resource_score = 0.0;
    if (!(allocate == 0.0 || w == 0)) {
      double used_finally = request + nv.used(d);
      if (used_finally > allocate) return 0.0;
      resource_score = used_finally * (double)w / allocate;
    }
    score += resource_score;
    weight_sum += w;
  }
  if (weight_sum > 0) score /= (double)weight_sum;
  score *= (double)(VC_MAX_NODE_SCORE * c.binpack_weight);
  return score;
}

// nodeorder NodeOrderFn (plugins/nodeorder/nodeorder.go:314-330): LeastAllocated(cpu 50, mem 50),
// MostAllocated(cpu 1, mem 1), BalancedAllocation(cpu, memory, nvidia.com/gpu), NodeAffinity raw count.
template <class NV>
__device__ __forceinline__ double nodeorder_score(const DevConf &c, int K, const TaskRec &t, const NV &nv,
                                                  uint32_t cstat) {
  double node_score = 0.0;
  if (c.w_least != 0 || c.w_most != 0) {
    double ls = 0.0, ms = 0.0, wl = 0.0, wm = 0.0;
    for (int k = 0; k < 2 && k < K; ++k) {
      double alloc = nv.kalloc(k);
      if (alloc == 0.0) continue;
      double reqv = nv.knz(k) + t.knz[k];
      if (c.w_least != 0) { ls += least_requested_score(reqv, alloc) * 50.0; wl += 50.0; }
      if (c.w_most != 0) { ms += most_requested_score(reqv, alloc) * 1.0; wm += 1.0; }
    }
    if (c.w_least != 0) node_score += (wl == 0.0 ? 0.0 : idiv_floor(ls, wl)) * (double)c.w_least;
    if (c.w_most != 0) node_score += (wm == 0.0 ? 0.0 : idiv_floor(ms, wm)) * (double)c.w_most;
  }
  if (c.w_balanced != 0) {
    double fr[VC_MAX_KDIMS];
    int nf = 0;
    double total = 0.0;
    for (int k = 0; k < K; ++k) {
      double pod_req = t.kreq[k];
      if (k >= 2 && pod_req == 0.0) continue;
      double alloc = nv.kalloc(k);
      if (alloc == 0.0) continue;
      double f = (nv.kreq(k) + pod_req) / alloc;
      if (f > 1.0) f = 1.0;
      total += f;
      fr[nf++] = f;
    }
    double stdv = 0.0;
    if (nf == 2) {
      stdv = fabs((fr[0] - fr[1]) / 2.0);
    } else if (nf > 2) {
      double mean = total / (double)nf;
      double sum = 0.0;
      for (int i = 0; i < nf; ++i) sum = sum + (fr[i] - mean) * (fr[i] - mean);
      stdv = sqrt(sum / (double)nf);
    }
    double bal = (double)__double2ll_rz((1.0 - stdv) * (double)VC_MAX_NODE_SCORE);
    node_score += bal * (double)c.w_balanced;
  }
  if (c.w_node_affinity != 0) node_score += (double)(cstat >> CS_NAFF_SHIFT) * (double)c.w_node_affinity;
  return node_score;
}

// ssn.NodeOrderMapFn order part, framework/session_plugins.go:974-999. Returns false when a
// NodeOrderFn errored (util.PrioritizeNodes then records no order score, scheduler_helper.go:83-87).
template <class NV>
__device__ __forceinline__ bool node_order(const DevConf &c, int R, int K, const TaskRec &t, const NV &nv,
                                           uint32_t cstat, double *out) {
  double priority_score = 0.0;
  for (int i = 0; i < c.n_plugins; ++i) {
    if (!(c.enabled[i] & VC_EN_NODE_ORDER)) continue;
    int pl = c.plugin[i];
    if (pl == VC_PLUGIN_BINPACK) {
      if (c.binpack_weight != 0) priority_score += binpack_score(c, R, t, nv);
    } else if (pl == VC_PLUGIN_NODEORDER) {
      priority_score += nodeorder_score(c, K, t, nv, cstat);
    } else if (pl == VC_PLUGIN_TDM) {
      if (cstat & CS_TDM_ORDER_ERR) return false;
      priority_score += (cstat & CS_TDM_ORDER_MAX) ? (double)VC_MAX_NODE_SCORE : 0.0;
    }
  }
  *out = priority_score;
  return true;
}

// getPodHyperNodeBinPackingScore, plugins/network-topology-aware/network_topology_aware.go:498-539.
// used(d) / alloc(d): the plugin's hyperNodeResourceCache entry of one hypernode.
template <class FU, class FA>
__device__ __forceinline__ double hn_binpack_score(const DevConf &c, int R, const TaskRec &t, FU used, FA alloc) {
  double total_score = 0.0;
  int total_weight = 0;
  for (int d = 0; d < R; ++d) {
    const double request = t.req[d];
    if (d >= 2 && !(t.has & (1u << d))) continue;  // task.Resreq.ResourceNames()
    if (!(request >= VC_MIN_RESOURCE)) continue;
    const int w = c.nta_dim_weight[d];
    if (w < 0) continue;
    const double allocatable = alloc(d), u = used(d);
    if (u + request > allocatable) return 0.0;
    const double score = (u + request) / allocatable;
    total_score += (double)w * score;
    total_weight += w;
  }
  if (total_weight > 0) return total_score / (double)total_weight;
  return 0.0;
}
// batchNodeOrderFnForNormalPods :462-496 + scaleFinalScore :758-764. tier_score(l): binpack score of the
// hypernode holding the node at tier level l, FullScore (1.0) when none does.
template <class FT>
__device__ __forceinline__ double nta_node_score(const DevConf &c, FT tier_score) {
  double total = 0.0;
  for (int l = 0; l < c.nta_L; ++l) total += c.tier_w[l] * tier_score(l);
  const double sc = total / c.tier_w_total;
  return (double)VC_MAX_NODE_SCORE * (double)c.nta_weight * sc;
}

// Total of util.PrioritizeNodes for one node (scheduler_helper.go:117-129): 0.0 + order + batch,
// batch = TaintToleration with DefaultNormalizeScore(reverse) over the scored node set, plus the
// network-topology-aware entry `nta` (two addends: their plugin order does not matter).
__device__ __forceinline__ double total_score(const DevConf &c, bool has_order, double order, int soft, int max_soft,
                                              double nta = 0.0) {
  double score = 0.0;
  if (has_order) score += order;
  if (c.batch_any) {
    double b = 0.0;
    if (c.taint_batch) {
      long long sc = (max_soft == 0) ? (long long)VC_MAX_NODE_SCORE
                                     : (long long)VC_MAX_NODE_SCORE - ((long long)VC_MAX_NODE_SCORE * soft / max_soft);
      sc *= (long long)c.w_taint;
      double node_sc = 0.0;
      node_sc += (double)sc;
      b += node_sc;
    }
    if (c.nta_plugin) b += nta;  // callers pass 0.0 when the plugin's map has no entry for the node
    score += b;
  }
  return score;
}

// Resource fit of the request against Idle / FutureIdle (resource_info.go:429-463, node_info.go:114-116).
// returns 0 = fits Idle, 1 = fits FutureIdle only, 2 = does not fit FutureIdle.
template <class NV>
__device__ __forceinline__ int fit_category(const DevConf &c, int R, const TaskRec &t, const NV &nv) {
  bool fit_idle = true, fit_future = true;
  for (int d = 0; d < R; ++d) {
    if (d >= 2 && !(t.has & (1u << d))) continue;
    double idle = nv.idle(d);
    double rq = t.req[d];
    if (!le_eps(rq, idle)) fit_idle = false;
    if (c.has_future) {
      double fut = (idle + nv.rel(d)) - nv.pip(d);
      if (!le_eps(rq, fut)) fit_future = false;
    }
  }
  if (!c.has_future) return fit_idle ? 0 : 2;
  if (!fit_future) return 2;
  return fit_idle ? 0 : 1;
}

template <bool FUT, class NV>
__device__ __forceinline__ int fit_category_t(int R, const TaskRec &t, const NV &nv) {
  bool fit_idle = true, fit_future = true;
  for (int d = 0; d < R; ++d) {
    if (d >= 2 && !(t.has & (1u << d))) continue;
    double idle = nv.idle(d);
    double rq = t.req[d];
    if (!le_eps(rq, idle)) fit_idle = false;
    if (FUT) {
      double fut = (idle + nv.rel(d)) - nv.pip(d);
      if (!le_eps(rq, fut)) fit_future = false;
    }
  }
  if (!FUT) return fit_idle ? 0 : 2;
  if (!fit_future) return 2;
  return fit_idle ? 0 : 1;
}

// ---------------------------------------------------------------------------------------
// Straight-line evaluator for the commit kernel's common case (no FutureIdle gradient, no normalising
// batch scorer, R <= 8, K <= 4). Same IEEE operations in the same order as the generic functions above,
// but fully unrolled and predicated so the ~12 independent fp64 divisions of one (task, node) pair issue
// back to back instead of one dependency chain after the other (the sweep is latency-bound: one warp per
// SM sub-partition). Adding the 0.0 of a skipped term is exact, so predication does not change results.
// Returns the fit category (0 idle-fit / 2 infeasible) and the total score of util.PrioritizeNodes.
// ---------------------------------------------------------------------------------------
// ORDER_ONLY: *score_out = the NodeOrderFn sum alone (0.0 for a node whose sum was aborted); the caller adds the batch
// scores once the normalisation constants of the candidate set are known.
template <bool ORDER_ONLY = false, class NV>
__device__ __forceinline__ int eval_pair_fast(const DevConf &c, int R, int K, const TaskRec &t, const NV &nv,
                                              uint32_t cs, bool pod_cap_hit, double *score_out) {
  constexpr int RT = 8, KT = VC_MAX_KDIMS;
  // ---- resource fit against Idle (resource_info.go:429-463) ----
  bool fit = (cs & CS_STATIC_OK) != 0 && !pod_cap_hit;
  double usedv[RT], allocv[RT];
#pragma unroll
  for (int d = 0; d < RT; ++d) {
    const bool on = d < R && (d < 2 || (t.has & (1u << d)));
    const double idle = d < R ? nv.idle(d) : 0.0;
    if (on && !le_eps(t.req[d], idle)) fit = false;
    usedv[d] = d < R ? nv.used(d) : 0.0;
    allocv[d] = d < R ? nv.alloc(d) : 0.0;
  }
  // ---- binpack (plugins/binpack/binpack.go:206-261) ----
  double bp_term[RT];
  bool bp_over = false;
  int bp_wsum = 0;
#pragma unroll
  for (int d = 0; d < RT; ++d) {
    const double request = d < R ? t.req[d] : 0.0;
    const int w = c.binpack_dim_weight[d];
    const bool on = d < R && (d < 2 || (t.has & (1u << d))) && request >= VC_MIN_RESOURCE && w >= 0;
    const bool scored = on && !(allocv[d] == 0.0 || w == 0);
    const double used_finally = request + usedv[d];
    if (scored && used_finally > allocv[d]) bp_over = true;
    const double q = used_finally * (double)w / (scored ? allocv[d] : 1.0);
    bp_term[d] = scored ? q : 0.0;
    bp_wsum += on ? w : 0;
  }
  double bp = 0.0;
#pragma unroll
  for (int d = 0; d < RT; ++d) bp += bp_term[d];
  if (bp_wsum > 0) bp /= (double)bp_wsum;
  bp *= (double)(VC_MAX_NODE_SCORE * c.binpack_weight);
  if (bp_over) bp = 0.0;
  // ---- nodeorder NodeOrderFn (plugins/nodeorder/nodeorder.go:314-330) ----
  double ls = 0.0, ms = 0.0, wl = 0.0, wm = 0.0;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const double alloc = nv.kalloc(k);
    const bool on = alloc != 0.0;
    const double a1 = on ? alloc : 1.0;
    const double reqv = nv.knz(k) + t.knz[k];
    const double l = least_requested_score(reqv, a1), m = most_requested_score(reqv, a1);
    ls += on ? l * 50.0 : 0.0; wl += on ? 50.0 : 0.0;
    ms += on ? m * 1.0 : 0.0;  wm += on ? 1.0 : 0.0;
  }
  double fr[KT];
  bool fon[KT];
  int nf = 0;
#pragma unroll
  for (int k = 0; k < KT; ++k) {
    const double pod_req = k < K ? t.kreq[k] : 0.0;
    const double alloc = k < K ? nv.kalloc(k) : 0.0;
    fon[k] = k < K && !(k >= 2 && pod_req == 0.0) && alloc != 0.0;
    double f = ((k < K ? nv.kreq(k) : 0.0) + pod_req) / (fon[k] ? alloc : 1.0);
    if (f > 1.0) f = 1.0;
    fr[k] = f;
    nf += fon[k] ? 1 : 0;
  }
  double total = 0.0;
#pragma unroll
  for (int k = 0; k < KT; ++k) total += fon[k] ? fr[k] : 0.0;
  double stdv = 0.0;
  if (nf == 2) {
    // the two active fractions in dimension order
    double f0 = 0.0, f1 = 0.0;
    int seen = 0;
#pragma unroll
    for (int k = 0; k < KT; ++k)
      if (fon[k]) { if (seen == 0) f0 = fr[k]; else f1 = fr[k]; ++seen; }
    stdv = fabs((f0 - f1) / 2.0);
  } else if (nf > 2) {
    const double mean = total / (double)nf;
    double sum = 0.0;
#pragma unroll
    for (int k = 0; k < KT; ++k)
      if (fon[k]) sum = sum + (fr[k] - mean) * (fr[k] - mean);
    stdv = sqrt(sum / (double)nf);
  }
  const double bal = (double)__double2ll_rz((1.0 - stdv) * (double)VC_MAX_NODE_SCORE);
  double no = 0.0;
  if (c.w_least != 0) no += (wl == 0.0 ? 0.0 : idiv_floor(ls, wl == 0.0 ? 1.0 : wl)) * (double)c.w_least;
  if (c.w_most != 0) no += (wm == 0.0 ? 0.0 : idiv_floor(ms, wm == 0.0 ? 1.0 : wm)) * (double)c.w_most;
  if (c.w_balanced != 0) no += bal * (double)c.w_balanced;
  if (c.w_node_affinity != 0) no += (double)(cs >> CS_NAFF_SHIFT) * (double)c.w_node_affinity;
  // ---- ssn.NodeOrderMapFn sum in plugin order, then util.PrioritizeNodes total ----
  double order = 0.0;
  bool has_order = true;
  for (int i = 0; i < c.n_plugins; ++i) {
    if (!(c.enabled[i] & VC_EN_NODE_ORDER)) continue;
    const int pl = c.plugin[i];
    if (pl == VC_PLUGIN_BINPACK) { if (c.binpack_weight != 0) order += bp; }
    else if (pl == VC_PLUGIN_NODEORDER) order += no;
    else if (pl == VC_PLUGIN_TDM) {
      if (has_order) {
        if (cs & CS_TDM_ORDER_ERR) has_order = false;
        else order += (cs & CS_TDM_ORDER_MAX) ? (double)VC_MAX_NODE_SCORE : 0.0;
      }
    }
  }
  // a NodeOrderFn error aborts the whole NodeOrderMapFn sum for the node (session_plugins.go:984-987)
  *score_out = ORDER_ONLY ? (has_order ? order : 0.0) : total_score(c, has_order, has_order ? order : 0.0, 0, 0);
  return fit ? 0 : 2;
}

// (score, node) ordering of util.SelectBestNodeAndScore with the canonical tie-break.
__host__ __device__ __forceinline__ bool better(double sa, int na, double sb, int nb) {
  return sa > sb || (sa == sb && na < nb);
}

// packed key for a MAX all-reduce across node shards: orderable(score) high, inverted node low
__host__ __device__ __forceinline__ uint64_t order_bits(double x) {
#ifdef __CUDA_ARCH__
  uint64_t u = (uint64_t)__double_as_longlong(x);
#else
  uint64_t u;
  memcpy(&u, &x, 8);
#endif
  return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}

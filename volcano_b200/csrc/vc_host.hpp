// vc_host.hpp — host-side session-open logic of libvcalloc.so (product code, C++17).
//
// What the reference does in plugin OnSessionOpen callbacks and in buildAllocateContext before the
// first task is placed: ssn.TotalResource, drf job shares, proportion's deserved water-filling, gang
// JobValid, the TaskOrderFn order inside each job and the initial JobOrderFn order inside each queue.
// These are O(J + Q + T) scalar passes; the O(T x N) work is on the GPU.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <initializer_list>
#include <limits>
#include <vector>

#include "../../include/vcalloc.h"
#include "vc_hdrf.hpp"

namespace vch {

constexpr double kMinRes = 0.1;
inline bool le_eps(double l, double r) { return l < r || std::fabs(l - r) < kMinRes; }
inline double share_of(double l, double r) { return r == 0 ? (l == 0 ? 0.0 : 1.0) : l / r; }

// api.Resource as a dense vector + key-presence mask + nil-map flag (api/resource_info.go:60-70)
struct HRes {
  double v[VC_MAX_DIMS];
  uint32_t has = 0;
  bool nil = true;
  HRes() { for (double &x : v) x = 0; }
  static HRes load(const double *base, int count, int idx, int R, uint32_t has_bits) {
    HRes r;
    if (!base) return r;
    uint32_t m = has_bits & ~(VC_RES_HAS_ANY | 3u);
    if (R < 32) m &= (1u << R) - 1;
    for (int d = 0; d < R; ++d)
      if (d < 2 || (m & (1u << d))) r.v[d] = base[(size_t)d * count + idx];
    r.has = m;
    r.nil = m == 0;
    return r;
  }
  bool k(int d) const { return (has >> d) & 1u; }
  void add(const HRes &o, int R) {  // Resource.Add :277-290
    v[0] += o.v[0]; v[1] += o.v[1];
    for (int d = 2; d < R; ++d) if (o.k(d)) { v[d] += o.v[d]; has |= 1u << d; nil = false; }
  }
  void multi(double ratio, int R) {  // Resource.Multi :323-330
    v[0] *= ratio; v[1] *= ratio;
    for (int d = 2; d < R; ++d) if (k(d)) v[d] *= ratio;
  }
  void min_dim(const HRes &o, bool inf, int R) {  // MinDimensionResource :939-976
    if (o.v[0] < v[0]) v[0] = o.v[0];
    if (o.v[1] < v[1]) v[1] = o.v[1];
    if (nil) return;
    if (o.nil) { if (!inf) for (int d = 2; d < R; ++d) if (k(d)) v[d] = 0; return; }
    for (int d = 2; d < R; ++d) {
      if (!k(d)) continue;
      if (o.k(d)) v[d] = std::fmin(v[d], o.v[d]);
      else if (!inf) v[d] = 0;
    }
  }
  bool equal(const HRes &o, int R) const {  // equality.Semantic.DeepEqual
    if (v[0] != o.v[0] || v[1] != o.v[1] || has != o.has) return false;
    for (int d = 2; d < R; ++d) if (k(d) && v[d] != o.v[d]) return false;
    return true;
  }
  bool less_equal_zero(const HRes &o, int R) const {  // LessEqual(o, Zero) :429-463
    if (!le_eps(v[0], o.v[0]) || !le_eps(v[1], o.v[1])) return false;
    for (int d = 2; d < R; ++d) if (k(d) && !le_eps(v[d], o.k(d) ? o.v[d] : 0.0)) return false;
    return true;
  }
  bool is_empty(int R, int pods_dim) const {  // IsEmpty :240-255
    if (!(v[0] < kMinRes && v[1] < kMinRes)) return false;
    for (int d = 2; d < R; ++d) if (k(d) && d != pods_dim && v[d] >= kMinRes) return false;
    return true;
  }
};
inline HRes hmax(const HRes &l, const HRes &r, int R) {  // helpers.Max, api/helpers/helpers.go:51-77
  HRes o;
  o.v[0] = std::fmax(l.v[0], r.v[0]); o.v[1] = std::fmax(l.v[1], r.v[1]);
  if (l.nil && r.nil) return o;
  o.nil = false;
  for (int d = 2; d < R; ++d) if (l.k(d) && l.v[d] >= 0) { o.has |= 1u << d; o.v[d] = l.v[d]; }
  for (int d = 2; d < R; ++d) if (r.k(d) && r.v[d] >= 0) { double cur = o.k(d) ? o.v[d] : 0.0; o.has |= 1u << d; o.v[d] = std::fmax(r.v[d], cur); }
  return o;
}
inline void hdiff(const HRes &l, const HRes &r, HRes &inc, HRes &dec, int R) {  // Diff(., Zero) :879-918
  inc = HRes(); dec = HRes();
  inc.nil = dec.nil = false;
  for (int d = 0; d < 2; ++d) { if (l.v[d] > r.v[d]) inc.v[d] = l.v[d] - r.v[d]; else dec.v[d] = r.v[d] - l.v[d]; }
  uint32_t keys = l.has | r.has;
  for (int d = 2; d < R; ++d) {
    if (!((keys >> d) & 1u)) continue;
    double lq = l.k(d) ? l.v[d] : 0.0, rq = r.k(d) ? r.v[d] : 0.0;
    if (lq == -1.0) { inc.has |= 1u << d; inc.v[d] = lq; continue; }
    if (rq == -1.0) { dec.has |= 1u << d; dec.v[d] = rq; continue; }
    if (lq > rq) { inc.has |= 1u << d; inc.v[d] = lq - rq; } else { dec.has |= 1u << d; dec.v[d] = rq - lq; }
  }
}
inline HRes exceeded(const HRes &l, const HRes &r, int R) { HRes a, b; hdiff(l, r, a, b, R); return a; }

struct QAttr {  // proportion.queueAttr, plugins/proportion/proportion.go:57-74
  bool exists = false;
  HRes deserved, allocated, request, capability, real_cap, guarantee;
  double share = 0;
  int32_t weight = 0;
};
inline double queue_share(const QAttr &a, int R) {  // updateQueueAttrShare :590-602
  double res = 0;
  for (int d = 0; d < R; ++d) {
    if (d >= 2 && !a.deserved.k(d)) continue;
    if (!(a.deserved.v[d] >= kMinRes)) continue;
    double al = (d < 2 || a.allocated.k(d)) ? a.allocated.v[d] : 0.0;
    double sh = share_of(al, a.deserved.v[d]);
    if (sh > res) res = sh;
  }
  return res;
}

// proportion OnSessionOpen (plugins/proportion/proportion.go:90-264)
inline void proportion_open(const vc_dims &d, const vc_jobs &jb, const vc_queues &qu, const HRes &total,
                            std::vector<QAttr> &out) {
  const int R = d.n_dims, Q = d.n_queues, J = d.n_jobs;
  out.assign(Q, QAttr());
  HRes total_guar;
  for (int q = 0; q < Q; ++q)
    if (qu.guarantee_has && (qu.guarantee_has[q] & VC_RES_HAS_ANY)) total_guar.add(HRes::load(qu.guarantee, Q, q, R, qu.guarantee_has[q]), R);
  for (int j = 0; j < J; ++j) {
    int q = jb.queue[j];
    if (q < 0 || out[q].exists) continue;
    QAttr &a = out[q];
    a.exists = true;
    a.weight = qu.weight[q];
    bool has_cap = qu.capability_has && (qu.capability_has[q] & VC_RES_HAS_ANY);
    if (has_cap) {
      a.capability = HRes::load(qu.capability, Q, q, R, qu.capability_has[q]);
      if (a.capability.v[0] <= 0) a.capability.v[0] = std::numeric_limits<double>::max();
      if (a.capability.v[1] <= 0) a.capability.v[1] = std::numeric_limits<double>::max();
    }
    if (qu.guarantee_has && (qu.guarantee_has[q] & VC_RES_HAS_ANY)) a.guarantee = HRes::load(qu.guarantee, Q, q, R, qu.guarantee_has[q]);
    a.real_cap = exceeded(total, total_guar, R);
    a.real_cap.add(a.guarantee, R);
    if (has_cap) a.real_cap.min_dim(a.capability, true, R);
    a.allocated = HRes::load(qu.allocated, Q, q, R, qu.allocated_has ? qu.allocated_has[q] : 0);
    a.request = HRes::load(qu.request, Q, q, R, qu.request_has ? qu.request_has[q] : 0);
  }
  HRes remaining = total;
  std::vector<uint8_t> meet(Q, 0);
  for (;;) {
    int64_t tw = 0;
    for (int q = 0; q < Q; ++q) if (out[q].exists && !meet[q]) tw += out[q].weight;
    if (tw == 0) break;
    HRes old_remaining = remaining, increased, decreased;
    for (int q = 0; q < Q; ++q) {
      QAttr &a = out[q];
      if (!a.exists || meet[q]) continue;
      HRes old = a.deserved;
      HRes part = remaining;
      part.multi((double)a.weight / (double)(int32_t)tw, R);
      a.deserved.add(part, R);
      a.deserved.min_dim(a.real_cap, true, R);
      a.deserved.min_dim(a.request, false, R);
      a.deserved = hmax(a.deserved, a.guarantee, R);
      a.share = queue_share(a, R);
      if (a.request.less_equal_zero(a.deserved, R)) meet[q] = 1;
      else if (a.deserved.equal(old, R)) meet[q] = 1;
      HRes inc, dec;
      hdiff(a.deserved, old, inc, dec, R);
      increased.add(inc, R);
      decreased.add(dec, R);
    }
    HRes tmp = remaining;
    tmp.add(decreased, R);
    remaining = exceeded(tmp, increased, R);
    if (remaining.is_empty(R, d.pods_dim) || remaining.equal(old_remaining, R)) break;
  }
}

// math.Pow(x, n) of the Go runtime for a small non-negative integer n (src/math/pow.go: y == 0 -> 1,
// y == 1 -> x, x == 0 -> 0, else binary exponentiation on the Frexp mantissa with the exponent carried
// separately). network-topology-aware derives its tier weights with it (network_topology_aware.go:470-476).
inline double go_pow_uint(double x, unsigned n) {
  if (n == 0 || x == 1.0) return 1.0;
  if (n == 1) return x;
  if (x == 0.0) return 0.0;
  int xe = 0, ae = 0;
  double x1 = std::frexp(x, &xe), a1 = 1.0;
  for (unsigned i = n; i != 0; i >>= 1) {
    if (i & 1u) { a1 *= x1; ae += xe; }
    x1 *= x1;
    xe <<= 1;
    if (x1 < 0.5) { x1 += x1; --xe; }
  }
  return std::ldexp(a1, ae);
}

// CalculateNumOfFeasibleNodesToFind, util/scheduler_helper.go:54-73
VC_HD int32_t num_feasible_nodes_to_find(int32_t num_all, int32_t pct, int32_t min_nodes, int32_t min_pct) {
  if (num_all <= min_nodes || pct >= 100) return num_all;
  int32_t adaptive = pct;
  if (adaptive <= 0) {
    adaptive = 50 - num_all / 125;
    if (adaptive < min_pct) adaptive = min_pct;
  }
  int32_t num = num_all * adaptive / 100;
  if (num < min_nodes) num = min_nodes;
  return num;
}

inline bool has_plugin(const vc_conf &c, int id) {
  for (int i = 0; i < c.n_plugins; ++i) if (c.plugins[i].plugin == id) return true;
  return false;
}
inline bool plugin_enabled(const vc_conf &c, int id, uint32_t flag) {
  for (int i = 0; i < c.n_plugins; ++i) if (c.plugins[i].plugin == id && (c.plugins[i].enabled & flag)) return true;
  return false;
}

// gang validJobFn (plugins/gang/gang.go:58-93) through ssn.JobValid (session_plugins.go:509-524)
inline bool job_valid(const vc_conf &c, const vc_jobs &jb, int j) {
  if (!has_plugin(c, VC_PLUGIN_GANG)) return true;
  if (!(jb.min_available[j] < jb.task_min_total[j])) {
    for (int r = jb.role_off[j]; r < jb.role_off[j + 1]; ++r) {
      if (!(jb.role_flags[r] & VC_ROLE_IN_MIN_MAP) || jb.role_min[r] == 0) continue;
      if (jb.role_valid[r] < jb.role_min[r]) return false;
    }
  }
  return jb.valid_num[j] >= jb.min_available[j];
}

// ssn.TaskOrderFn (session_plugins.go:772-783): priority plugin, then helpers.CompareTask
struct TaskLess {
  const vc_tasks *t;
  bool by_priority;
  bool operator()(int l, int r) const {
    if (by_priority && t->priority[l] != t->priority[r]) return t->priority[l] > t->priority[r];
    bool lerr = t->pod_index[l] < 0, rerr = t->pod_index[r] < 0;
    if (lerr || rerr || t->pod_index[l] == t->pod_index[r]) {
      if (t->creation_ts[l] == t->creation_ts[r]) return t->uid_rank[l] < t->uid_rank[r];
      return t->creation_ts[l] < t->creation_ts[r];
    }
    return !(t->pod_index[l] > t->pod_index[r]);
  }
};

// Pop order of a util.PriorityQueue (container/heap) filled in index order — the order in which
// allocateResourcesForTasks sees the tasks of a job (util/priority_queue.go:30-111).
template <class Less>
inline void go_heap_order(std::vector<int> &items, Less less) {
  std::vector<int> h;
  h.reserve(items.size());
  for (int x : items) {
    h.push_back(x);
    int j = (int)h.size() - 1;
    for (;;) {
      int i = (j - 1) / 2;
      if (i == j || !less(h[j], h[i])) break;
      std::swap(h[i], h[j]);
      j = i;
    }
  }
  size_t out = 0;
  while (!h.empty()) {
    int n = (int)h.size() - 1;
    std::swap(h[0], h[n]);
    int i = 0;
    for (;;) {
      int j1 = 2 * i + 1;
      if (j1 >= n || j1 < 0) break;
      int j = j1;
      if (j1 + 1 < n && less(h[j1 + 1], h[j1])) j = j1 + 1;
      if (!less(h[j], h[i])) break;
      std::swap(h[i], h[j]);
      i = j;
    }
    items[out++] = h.back();
    h.pop_back();
  }
}


// ---------------------------------------------------------------------------------------
// backfill: pickUpPendingTasks (actions/backfill/backfill.go:118-199) on the state the allocate action left
// ---------------------------------------------------------------------------------------
struct BackfillTasks {  // host copy of the BestEffort task list (vc_snapshot_set_backfill)
  int n = 0;
  std::vector<double> req, kreq, knz;
  std::vector<uint32_t> has, uid;
  std::vector<int32_t> job, klass, role, prio;
  std::vector<int64_t> podidx, ts;
};
struct BackfillKeep {  // session-open state the pick order needs, kept at upload when the list is not empty
  std::vector<int32_t> j_queue, j_min, j_prio, j_ready0, j_pbe, j_taskmintotal, j_roleoff, r_min, r_occ0, q_prio, t_role;
  std::vector<uint32_t> j_flags, j_rank, r_flags, q_rank;
  std::vector<uint8_t> j_valid;
  std::vector<double> j_alloc0;  // [R][J]
};
struct BackfillPick {
  std::vector<int32_t> order;             // backfill task ids in visiting order
  std::vector<int> visit_job, visit_begin;  // one visit per job: its slice of `order` is [visit_begin[v], visit_begin[v+1])
  std::vector<int32_t> j_ready, r_occ;    // ReadyTaskNum per job / occupancy per role row after allocate
};
// Exactness precondition of the run-length batches: for dimension-major arrays rows[d][n] (node rows a placement
// updates) and reqs[d][t] (what it adds / subtracts), every value is an integer and max|row_d| + 32 * max|req_d| stays
// below 2^53 — then row -/+ k * req (k <= 32) and the k sequential updates are the same exactly-representable integers.
inline bool max_abs_integral(const double *v, size_t n, double &mx) {
  if (!v) return true;
  for (size_t i = 0; i < n; ++i) {
    const double a = std::fabs(v[i]);
    if (!(a < 9.0e15) || (double)(long long)v[i] != v[i]) return false;  // below 2^63: the conversion is exact iff integral
    if (a > mx) mx = a;
  }
  return true;
}
inline bool runs_exact(size_t D, size_t N, size_t T, std::initializer_list<const double *> rows,
                       std::initializer_list<const double *> reqs) {
  for (size_t d = 0; d < D; ++d) {
    double mrow = 0.0, mreq = 0.0;
    for (const double *r : rows)
      if (!max_abs_integral(r ? r + d * N : nullptr, N, mrow)) return false;
    for (const double *q : reqs)
      if (!max_abs_integral(q ? q + d * T : nullptr, T, mreq)) return false;
    if (!(mrow + 32.0 * mreq < 9.0e15)) return false;
  }
  return true;
}
// FutureIdle = (Idle + Releasing) - Pipelined along a run: every intermediate value stays an exactly representable
// integer when, per node and dimension, |Idle| + |Releasing| + |Pipelined| + 32 * max|req_d| < 2^53
inline bool future_rows_exact(size_t D, size_t N, size_t T, const double *idle, const double *rel, const double *pip,
                              const double *req) {
  if (!rel && !pip) return true;
  for (size_t d = 0; d < D; ++d) {
    double mreq = 0.0, mrel = 0.0, msum = 0.0;
    if (!max_abs_integral(req ? req + d * T : nullptr, T, mreq)) return false;
    if (!max_abs_integral(rel ? rel + d * N : nullptr, N, mrel) || !max_abs_integral(pip ? pip + d * N : nullptr, N, mrel)) return false;
    for (size_t n = 0; n < N; ++n) {
      const double a = std::fabs(idle[d * N + n]) + (rel ? std::fabs(rel[d * N + n]) : 0.0) + (pip ? std::fabs(pip[d * N + n]) : 0.0);
      if (a > msum) msum = a;
    }
    if (!(msum + 32.0 * mreq < 9.0e15)) return false;
  }
  return true;
}
// rank of every object in (CreationTimestamp, UID) order: the fallback of ssn.JobOrderFn / QueueOrderFn
inline void rank_by(const int64_t *ts, const uint32_t *uid, size_t n, std::vector<uint32_t> &rank) {
  std::vector<int> idx(n);
  for (size_t i = 0; i < n; ++i) idx[i] = (int)i;
  std::sort(idx.begin(), idx.end(), [&](int a, int b) { return ts[a] != ts[b] ? ts[a] < ts[b] : uid[a] < uid[b]; });
  rank.resize(n);
  for (size_t r = 0; r < n; ++r) rank[idx[r]] = (uint32_t)r;
}
// hdrf (drf's enableHierarchy) for the pick order: the tree built at upload and TotalRequest [R][J]
struct HdrfPick {
  const HdrfTree *tree;
  const double *job_request;
};
// `ops`: the operations of the preceding allocate action (kept visits only, in order); task_*: allocate's task arrays.
// `alloc_ran`: allocate ran before in this session. Without the enqueue action its buildAllocateContext rewrites the phase of
// every Pending PodGroup to Inqueue (allocate.go:154-164), so job.IsPending() (backfill.go:124) is false afterwards.
inline BackfillPick backfill_pick(const vc_conf &conf, bool alloc_ran, size_t R, size_t T, size_t J, size_t Q, size_t B, bool has_drf,
                                  bool has_proportion, const double *total, uint32_t total_has, const BackfillTasks &bf,
                                  const BackfillKeep &bk, const vc_decision *ops_p, size_t n_ops, const int32_t *task_job,
                                  const double *task_req, const uint32_t *task_has, std::vector<QAttr> qattr,
                                  const HdrfPick *hd = nullptr) {
  struct OpsView { const vc_decision *b, *e; const vc_decision *begin() const { return b; } const vc_decision *end() const { return e; } };
  const OpsView ops{ops_p, ops_p + n_ops};
  // ---- 1. the session state the allocate action left: ready counts, role occupancy, drf / proportion shares ----
  BackfillPick out;
  std::vector<int32_t> &j_ready = out.j_ready, &r_occ = out.r_occ;
  j_ready = bk.j_ready0; r_occ = bk.r_occ0;
  std::vector<double> j_alloc = bk.j_alloc0;
  
  for (const vc_decision &op : ops) {  // Statement.Allocate / Pipeline of every kept visit, in order
    const int t = op.task, j = task_job[t];
    if (op.kind == VC_OP_ALLOCATE) { j_ready[j] += 1; r_occ[bk.t_role[t]] += 1; }
    if (has_drf)  // drf AllocateFunc, drf.go:391-418
      for (size_t d = 0; d < R; ++d) j_alloc[d * J + j] += task_req[d * T + t];
    const int q = bk.j_queue[j];
    if (has_proportion && q >= 0 && qattr[q].exists)  // proportion AllocateFunc, proportion.go:475-497
      qattr[q].allocated.add(HRes::load(task_req, (int)T, t, (int)R, task_has[t]), (int)R);
  }
  std::vector<double> j_share(J, 0.0);
  if (has_drf)
    for (size_t j = 0; j < J; ++j) {  // drf.calculateShare, drf.go:566-578
      double res = 0;
      for (size_t d = 0; d < R; ++d) {
        if (d >= 2 && !((total_has >> d) & 1u)) continue;
        if (!(total[d] >= kMinRes)) continue;
        const double sh = share_of(j_alloc[d * J + j], total[d]);
        if (sh > res) res = sh;
      }
      j_share[j] = res;
    }
  std::vector<double> q_share(Q, 0.0);
  for (size_t q = 0; q < Q; ++q)
    if (qattr[q].exists) q_share[q] = queue_share(qattr[q], (int)R);
  auto is_ready = [&](int j) { return j_ready[j] + bk.j_pbe[j] >= bk.j_min[j]; };  // job_info.go:1169
  auto job_less = [&](int l, int rr) {  // ssn.JobOrderFn, session_plugins.go:660-683
    for (int i = 0; i < conf.n_plugins; ++i) {
      const vc_plugin_option &po = conf.plugins[i];
      if (!(po.enabled & VC_EN_JOB_ORDER)) continue;
      int c = 0;
      switch (po.plugin) {
        case VC_PLUGIN_PRIORITY: c = bk.j_prio[l] > bk.j_prio[rr] ? -1 : (bk.j_prio[l] < bk.j_prio[rr] ? 1 : 0); break;
        case VC_PLUGIN_GANG: {
          const bool lr = is_ready(l), r2 = is_ready(rr);
          c = (lr && r2) ? 0 : (lr ? 1 : (r2 ? -1 : 0));
          break;
        }
        case VC_PLUGIN_DRF: c = j_share[l] == j_share[rr] ? 0 : (j_share[l] < j_share[rr] ? -1 : 1); break;
        case VC_PLUGIN_TDM: {
          const bool lp = bk.j_flags[l] & VC_JOB_PREEMPTABLE, rp = bk.j_flags[rr] & VC_JOB_PREEMPTABLE;
          c = lp == rp ? 0 : (!lp ? -1 : 1);
          break;
        }
        default: break;
      }
      if (c != 0) return c < 0;
    }
    return bk.j_rank[l] < bk.j_rank[rr];
  };
  const bool qorder_prop = plugin_enabled(conf, VC_PLUGIN_PROPORTION, VC_EN_QUEUE_ORDER);
  // hdrf: the tree on the state allocate left (every order function is evaluated before backfill places anything)
  const HdrfOrder hd_ord = hdrf_order(conf);
  const bool hd_on = hd && has_drf && hd_ord.hdrf_on;
  HdrfState hst;
  if (hd_on) hdrf_eval(*hd->tree, (int)R, (int)J, total, total_has, j_alloc.data(), j_share.data(), hd->job_request, hst);
  struct QV {
    const BackfillKeep &bk; const std::vector<double> &q_share;
    int prio(int q) const { return bk.q_prio[q]; }
    double share(int q) const { return q_share[q]; }
    uint32_t rank(int q) const { return bk.q_rank[q]; }
  } qv{bk, q_share};
  auto queue_less = [&](int l, int rr) {  // ssn.QueueOrderFn :709-731; proportion.go:266-284
    if (hd_on)
      return hdrf_queue_less(hd_ord, hd->tree->q_path_off.data(), hd->tree->q_path.data(), hd->tree->weight.data(),
                             hst.n_share.data(), hst.n_sat.data(), qv, l, rr);
    if (qorder_prop) {
      if (bk.q_prio[l] != bk.q_prio[rr]) return bk.q_prio[l] > bk.q_prio[rr];
      if (q_share[l] != q_share[rr]) return q_share[l] < q_share[rr];
    }
    return bk.q_rank[l] < bk.q_rank[rr];
  };

  // ---- 2. pickUpPendingTasks, backfill.go:118-199 ----
  vc_tasks view;
  std::memset(&view, 0, sizeof view);
  view.priority = bf.prio.data(); view.pod_index = bf.podidx.data(); view.creation_ts = bf.ts.data(); view.uid_rank = bf.uid.data();
  const TaskLess task_less{&view, plugin_enabled(conf, VC_PLUGIN_PRIORITY, VC_EN_TASK_ORDER)};
  std::vector<std::vector<int>> job_tasks(J), queue_jobs(Q);
  for (size_t t = 0; t < B; ++t) job_tasks[bf.job[t]].push_back((int)t);
  std::vector<int> queues;
  for (size_t j = 0; j < J; ++j) {
    const bool phase_flipped = alloc_ran && !conf.enqueue_action_enabled;
    if ((bk.j_flags[j] & VC_JOB_PENDING_PHASE) && !phase_flipped) continue;  // job.IsPending(), :124-126
    if (!bk.j_valid[j]) continue;                         // ssn.JobValid, :128-131
    const int q = bk.j_queue[j];
    if (q < 0 || job_tasks[j].empty()) continue;
    if (queue_jobs[q].empty()) queues.push_back(q);
    queue_jobs[q].push_back((int)j);
  }
  go_heap_order(queues, queue_less);
  std::vector<int32_t> &order = out.order;  // backfill task ids in visiting order
  std::vector<int> &visit_job = out.visit_job, &visit_begin = out.visit_begin;
  for (int q : queues) {
    go_heap_order(queue_jobs[q], job_less);
    for (int j : queue_jobs[q]) {
      go_heap_order(job_tasks[j], task_less);
      visit_job.push_back(j);
      visit_begin.push_back((int)order.size());
      for (int t : job_tasks[j]) order.push_back(t);
    }
  }
  visit_begin.push_back((int)order.size());
  return out;
}

}  // namespace vch

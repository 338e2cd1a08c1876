// vc_hdrf.hpp — hierarchical drf (drf's enableHierarchy, plugins/drf/drf.go:45-184,458-560): the weighted queue tree,
// its shares, and ssn.QueueOrderFn with hdrf's compareQueues in the tier chain. Built on the host at session open
// (vc_snapshot_set_hdrf + vc_snapshot_upload); the share update, the comparator and the queue heap run in the control
// program of both commit kernels.
//
// The tree holds inner nodes (0 = the root, a parent before its children) and one leaf per job. With integer-valued
// resources (SURVEY Appendix A-2) every node's state is a pure function of the jobs' drf allocations and of
// totalAllocated, so a replica may recompute it lazily — only the ancestors of the job that changed, or the whole tree
// when the demanding set changed — and still equal what updateHierarchicalShare leaves after every event.
#pragma once
#include <cstdint>
#include <cstdio>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "../../include/vcalloc.h"

#if defined(__CUDACC__)
#define VC_HD __host__ __device__ __forceinline__
#else
#define VC_HD inline
#endif

namespace vch {

// one replica of the tree state: structure (read-only) + shares (mutable), all pointers of one address space
struct HdrfView {
  int R, M, J;
  const int32_t *parent;     // [M] (-1 for the root)
  const int32_t *child_off;  // [M+1] children in first-insertion order: code c < M inner node, else job c - M
  const int32_t *child;
  const int32_t *j_node;     // [J] inner node that holds the job's leaf
  const double *j_req;       // [R][J] JobInfo.TotalRequest
  const double *j_alloc;     // drf attr.allocated of job j, dimension d: j_alloc[j * ja_sj + d * ja_sd]
  long long ja_sj, ja_sd;
  const double *j_share;     // drf attr.share of job j: j_share[j * js_sj]
  long long js_sj;
  const double *total;       // [R] drf.totalResource
  uint32_t total_has;
  double *n_alloc;           // [M][R]
  double *n_share;           // [M]
  int32_t *n_sat;            // [M]
  int32_t *j_sat;            // [J]
  double *tot;               // [R] drf.totalAllocated
  int32_t *dem;              // [1] demanding set of the last update (bit d)
};

// drf.calculateShare over totalResource.ResourceNames() (dims with total >= 0.1), drf.go:566-578
VC_HD double hdrf_share_of(const HdrfView &v, const double *a, long long sd) {
  double res = 0.0;
  for (int d = 0; d < v.R; ++d) {
    if (d >= 2 && !((v.total_has >> d) & 1u)) continue;
    if (!(v.total[d] >= 0.1)) continue;
    const double l = a[d * sd], r = v.total[d];
    const double sh = r == 0 ? (l == 0 ? 0.0 : 1.0) : l / r;
    if (sh > res) res = sh;
  }
  return res;
}
// UpdateHierarchicalShare's demanding set: names of totalResource whose totalAllocated is below the total, drf.go:552-557
VC_HD int32_t hdrf_demanding(const HdrfView &v) {
  int32_t m = 0;
  for (int d = 0; d < v.R; ++d) {
    if (d >= 2 && !((v.total_has >> d) & 1u)) continue;
    if (!(v.total[d] >= 0.1)) continue;
    if (v.tot[d] < v.total[d]) m |= 1 << d;
  }
  return m;
}
// resourceSaturated, drf.go:83-95: over allocated.ResourceNames() (dims with allocated >= 0.1)
VC_HD int32_t hdrf_leaf_sat(const HdrfView &v, int j, int32_t dem) {
  const double *a = v.j_alloc + (long long)j * v.ja_sj;
  for (int d = 0; d < v.R; ++d) {
    const double al = a[d * v.ja_sd];
    if (!(al >= 0.1)) continue;
    const double rq = v.j_req[(long long)d * v.J + j];
    if (al != 0 && rq != 0 && al >= rq) return 1;
    if (!((dem >> d) & 1) && rq != 0) return 1;
  }
  return 0;
}
// updateHierarchicalShare for an inner node whose children are current, drf.go:503-548: mdr over the non-empty,
// unsaturated children; allocated = sum over the non-empty children in canonical order, unsaturated ones scaled by
// mdr / share; saturated when every child is
VC_HD void hdrf_inner(const HdrfView &v, int m) {
  const int c0 = v.child_off[m], c1 = v.child_off[m + 1];
  double mdr = 1.0;
  for (int k = c0; k < c1; ++k) {
    const int c = v.child[k];
    const double sh = c < v.M ? v.n_share[c] : v.j_share[(long long)(c - v.M) * v.js_sj];
    const int32_t sat = c < v.M ? v.n_sat[c] : v.j_sat[c - v.M];
    if (sh != 0 && !sat && sh < mdr) mdr = sh;
  }
  double *acc = v.n_alloc + (long long)m * v.R;
  for (int d = 0; d < v.R; ++d) acc[d] = 0.0;
  int32_t all_sat = 1;
  for (int k = c0; k < c1; ++k) {
    const int c = v.child[k];
    const bool inner = c < v.M;
    const double sh = inner ? v.n_share[c] : v.j_share[(long long)(c - v.M) * v.js_sj];
    const int32_t sat = inner ? v.n_sat[c] : v.j_sat[c - v.M];
    if (!sat) all_sat = 0;
    if (sh == 0) continue;
    const double *a = inner ? v.n_alloc + (long long)c * v.R : v.j_alloc + (long long)(c - v.M) * v.ja_sj;
    const long long sd = inner ? 1 : v.ja_sd;
    if (sat) {
      for (int d = 0; d < v.R; ++d) acc[d] += a[d * sd];
    } else {
      const double ratio = mdr / sh;  // Resource.Multi(mdr / child.attr.share)
      for (int d = 0; d < v.R; ++d) acc[d] += a[d * sd] * ratio;
    }
  }
  v.n_share[m] = hdrf_share_of(v, acc, 1);
  v.n_sat[m] = all_sat;
}
// Bring the replica to the state updateHierarchicalShare leaves after the last event. `job` = the only job whose
// allocation changed since the last call, or -1 for a full recomputation; v.tot must already be current.
VC_HD void hdrf_refresh(const HdrfView &v, int job) {
  const int32_t dem = hdrf_demanding(v);
  if (job < 0 || dem != v.dem[0]) {
    v.dem[0] = dem;
    for (int j = 0; j < v.J; ++j) v.j_sat[j] = v.j_node[j] >= 0 ? hdrf_leaf_sat(v, j, dem) : 0;
    for (int m = v.M - 1; m >= 0; --m) hdrf_inner(v, m);  // children carry larger ids than their parent
    return;
  }
  if (v.j_node[job] < 0) return;
  v.j_sat[job] = hdrf_leaf_sat(v, job, dem);
  for (int m = v.j_node[job]; m >= 0; m = v.parent[m]) hdrf_inner(v, m);
}

// compareQueues, drf.go:160-184, reduced to its sign by hdrf's queueOrderFn (drf.go:266-278): walk both paths from the
// root to the shorter depth; the unsaturated node first, then share / weight; equal values descend one level
VC_HD int hdrf_compare(const int32_t *q_path_off, const int32_t *q_path, const double *weight, const double *n_share,
                       const int32_t *n_sat, int l, int r) {
  const int la = q_path_off[l], ra = q_path_off[r];
  const int ll = q_path_off[l + 1] - la, rl = q_path_off[r + 1] - ra;
  const int depth = ll < rl ? ll : rl;
  for (int i = 0; i < depth; ++i) {
    const int a = q_path[la + i], b = q_path[ra + i];
    if (!n_sat[a] && n_sat[b]) return -1;
    if (n_sat[a] && !n_sat[b]) return 1;
    const double x = n_share[a] / weight[a], y = n_share[b] / weight[b];
    if (x == y) continue;
    const double diff = x - y;
    return diff < 0 ? -1 : (diff > 0 ? 1 : 0);
  }
  return 0;
}

// ssn.QueueOrderFn (session_plugins.go:709-731) with hdrf registered: drf's and proportion's comparators in tier order,
// then (CreationTimestamp, UID). `QV` gives prio(q), share(q) (proportion, proportion.go:266-284) and rank(q).
struct HdrfOrder {
  int hdrf_on;     // drf has EnabledQueueOrder: compareQueues takes part
  int prop_on;     // proportion has EnabledQueueOrder
  int hdrf_first;  // drf's option comes before proportion's
};
#if defined(__CUDACC__)
#pragma nv_exec_check_disable  // instantiated for the host (backfill's pick order) and for the device (commit kernels)
#endif
template <class QV>
VC_HD bool hdrf_queue_less(const HdrfOrder &o, const int32_t *q_path_off, const int32_t *q_path, const double *weight,
                           const double *n_share, const int32_t *n_sat, const QV &qv, int l, int r) {
  for (int k = 0; k < 2; ++k) {
    const bool hd = (k == 0) == (o.hdrf_first != 0);
    if (hd) {
      if (!o.hdrf_on) continue;
      const int c = hdrf_compare(q_path_off, q_path, weight, n_share, n_sat, l, r);
      if (c != 0) return c < 0;
    } else {
      if (!o.prop_on) continue;
      const int pl = qv.prio(l), pr = qv.prio(r);
      if (pl != pr) return pl > pr;
      const double sl = qv.share(l), sr = qv.share(r);
      if (sl != sr) return sl < sr;
    }
  }
  return qv.rank(l) < qv.rank(r);
}

// container/heap over queue ids (util/priority_queue.go): Push = append + up, Pop = swap(0, n-1) + down
template <class Less>
VC_HD void qheap_push(int32_t *h, int &n, int x, const Less &less) {
  h[n] = x;
  int j = n++;
  for (;;) {
    const int i = (j - 1) / 2;
    if (i == j || !less(h[j], h[i])) break;
    const int32_t t = h[i]; h[i] = h[j]; h[j] = t;
    j = i;
  }
}
template <class Less>
VC_HD int qheap_pop(int32_t *h, int &n, const Less &less) {
  const int last = n - 1;
  { const int32_t t = h[0]; h[0] = h[last]; h[last] = t; }
  int i = 0;
  for (;;) {
    const int j1 = 2 * i + 1;
    if (j1 >= last || j1 < 0) break;
    int j = j1;
    if (j1 + 1 < last && less(h[j1 + 1], h[j1])) j = j1 + 1;
    if (!less(h[j], h[i])) break;
    const int32_t t = h[i]; h[i] = h[j]; h[j] = t;
    i = j;
  }
  n = last;
  return h[last];
}

// ---------------------------------------------------------------------------------------
// host: the tree as buildHierarchy leaves it after session open inserted every job (drf.go:186-220,458-500)
// ---------------------------------------------------------------------------------------
struct HdrfTree {
  int M = 0;
  std::vector<int32_t> parent, child_off, child, j_node, q_path_off, q_path;
  std::vector<double> weight;
};
// Jobs are inserted in index order; a node is created by the first job whose queue names it, with that queue's weight
// (ParseFloat value, < 1 -> 1). Returns an empty string or the reason the reference would crash on this input.
inline std::string hdrf_build(int J, int Q, const int32_t *job_queue, const vc_hdrf &h, HdrfTree &t) {
  std::vector<std::map<int32_t, int32_t>> by_name(1);
  std::vector<std::vector<int32_t>> kids(1);  // child codes: >= 0 inner node, -(j+1) job j
  t.parent.assign(1, -1);
  t.weight.assign(1, 1.0);
  t.j_node.assign(J, -1);
  char buf[160];
  for (int j = 0; j < J; ++j) {
    const int q = job_queue[j];
    if (q < 0 || q >= Q) {  // drf.go:216-218 dereferences ssn.Queues[job.Queue]
      std::snprintf(buf, sizeof buf, "job %d: its queue is not in the session (hdrf needs every job's queue)", j);
      return buf;
    }
    const int off = h.path_off[q], len = h.path_off[q + 1] - off;
    if (len < 0) return "hdrf table: path_off not monotone";
    if (h.n_weights[q] < len) {  // weights[i] indexed out of range, drf.go:470
      std::snprintf(buf, sizeof buf, "queue %d: hierarchy-weights has %d segments below the root, hierarchy %d", q, h.n_weights[q], len);
      return buf;
    }
    int node = 0;
    for (int i = 0; i < len; ++i) {
      const int32_t name = h.path_name[off + i];
      auto it = by_name[node].find(name);
      if (it != by_name[node].end()) { node = it->second; continue; }
      double w = h.weight[off + i];
      if (w < 1) w = 1;
      const int m = (int)t.parent.size();
      t.parent.push_back(node);
      t.weight.push_back(w);
      by_name.emplace_back();
      kids.emplace_back();
      by_name[node][name] = m;
      kids[node].push_back(m);
      node = m;
    }
    t.j_node[j] = node;
    kids[node].push_back(-(j + 1));
  }
  t.M = (int)t.parent.size();
  t.child_off.assign(1, 0);
  t.child.clear();
  for (int m = 0; m < t.M; ++m) {
    for (int32_t c : kids[m]) t.child.push_back(c >= 0 ? c : t.M + (-c - 1));
    t.child_off.push_back((int32_t)t.child.size());
  }
  // every queue's chain from the root (a queue without jobs stops where the tree ends; it never enters a heap)
  t.q_path_off.assign(1, 0);
  t.q_path.clear();
  for (int q = 0; q < Q; ++q) {
    int node = 0;
    t.q_path.push_back(0);
    for (int i = h.path_off[q]; i < h.path_off[q + 1]; ++i) {
      auto it = by_name[node].find(h.path_name[i]);
      if (it == by_name[node].end()) break;
      node = it->second;
      t.q_path.push_back(node);
    }
    t.q_path_off.push_back((int32_t)t.q_path.size());
  }
  return std::string();
}
// the comparator chain of ssn.QueueOrderFn as the configuration lists it (options in tier, then plugin order)
inline HdrfOrder hdrf_order(const vc_conf &c) {
  HdrfOrder o{0, 0, 0};
  int first = -1;
  for (int i = 0; i < c.n_plugins; ++i) {
    if (!(c.plugins[i].enabled & VC_EN_QUEUE_ORDER)) continue;
    if (c.plugins[i].plugin == VC_PLUGIN_DRF && !o.hdrf_on) { o.hdrf_on = 1; if (first < 0) first = VC_PLUGIN_DRF; }
    if (c.plugins[i].plugin == VC_PLUGIN_PROPORTION && !o.prop_on) { o.prop_on = 1; if (first < 0) first = VC_PLUGIN_PROPORTION; }
  }
  o.hdrf_first = first == VC_PLUGIN_DRF;
  return o;
}
// The state of every node for given job allocations: a full recomputation on host vectors (backfill's pick order).
struct HdrfState {
  std::vector<double> n_alloc, n_share, tot;
  std::vector<int32_t> n_sat, j_sat;
  int32_t dem = -1;
};
inline void hdrf_eval(const HdrfTree &t, int R, int J, const double *total, uint32_t total_has, const double *j_alloc_rj,
                      const double *j_share, const double *j_req_rj, HdrfState &st) {
  st.n_alloc.assign((size_t)t.M * R, 0.0);
  st.n_share.assign(t.M, 0.0);
  st.n_sat.assign(t.M, 0);
  st.j_sat.assign(J, 0);
  st.tot.assign(VC_MAX_DIMS, 0.0);
  for (int d = 0; d < R; ++d)
    for (int j = 0; j < J; ++j) st.tot[d] += j_alloc_rj[(size_t)d * J + j];
  HdrfView v;
  v.R = R; v.M = t.M; v.J = J;
  v.parent = t.parent.data(); v.child_off = t.child_off.data(); v.child = t.child.data(); v.j_node = t.j_node.data();
  v.j_req = j_req_rj; v.j_alloc = j_alloc_rj; v.ja_sj = 1; v.ja_sd = J; v.j_share = j_share; v.js_sj = 1;
  v.total = total; v.total_has = total_has;
  v.n_alloc = st.n_alloc.data(); v.n_share = st.n_share.data(); v.n_sat = st.n_sat.data(); v.j_sat = st.j_sat.data();
  v.tot = st.tot.data(); v.dem = &st.dem;
  hdrf_refresh(v, -1);
}

}  // namespace vch

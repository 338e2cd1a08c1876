// oracle.cpp — CPU restatement of Volcano's `allocate` hot path.
//
// THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  It exists so that the CUDA path can be
// checked against an independent, straightforward restatement of the reference algorithm.
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
// may load it.  libvcalloc.so never links or calls anything in this directory.
//
// Parity status: the reference is Go (go 1.25, k8s.io/kubernetes v1.35.0 un-vendored) and
// cannot be compiled in this image, so the oracle is pinned against the reference's own
// golden vectors transcribed under tests/golden/ (binpack scores, LessEqual tables,
// feasible-node-count table, allocate placements, proportion/drf orderings) — see
// tests/test_oracle_golden.py.  Upstream kube-scheduler score arithmetic (LeastAllocated,
// MostAllocated, BalancedAllocation, TaintToleration, NodeAffinity) is restated from the
// published v1.35 algorithm and is pinned by the reference only at placement level:
// for those numeric values parity is UNPINNED (SURVEY.md §8c).
//
// Citations are into volcano's pkg/scheduler unless a full path is given.
//
// Canonical determinism contract (SURVEY.md §7.0-2, §8c): tie-break = lowest NodeList index
// among max-score nodes (the reference picks uniformly at random, util/scheduler_helper.go:
// 201-205); map iterations are replaced by index order; scalar dimensions iterate in
// dimension order.
//
// Build: g++ -O2 -std=c++17 -ffp-contract=off -fPIC -shared oracle.cpp -o liboracle.so -lpthread
#include "../include/vcalloc.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <limits>
#include <string>
#include <thread>
#include <vector>

namespace {

constexpr double kMinResource = 0.1;  // api/resource_info.go:45-47
constexpr int64_t kMaxNodeScore = 100; // fwk.MaxNodeScore

// lessEqualFunc, api/resource_info.go:430-435
inline bool le_eps(double l, double r) { return l < r || std::fabs(l - r) < kMinResource; }

// ---------------------------------------------------------------------------------------
// api.Resource with the presence semantics of its ScalarResources map
// (api/resource_info.go:60-70).  Used for the proportion plugin's session-open arithmetic.
// ---------------------------------------------------------------------------------------
struct Res {
  double v[VC_MAX_DIMS];
  uint32_t has = 0;    // bit d (d >= 2): key present in ScalarResources
  bool nilmap = true;  // ScalarResources == nil
  Res() { std::fill(v, v + VC_MAX_DIMS, 0.0); }
};


// Resource.Add, api/resource_info.go:277-290
void res_add(Res &r, const Res &rr, int R) {
  r.v[0] += rr.v[0];
  r.v[1] += rr.v[1];
  for (int d = 2; d < R; ++d)
    if (rr.has & (1u << d)) {
      r.nilmap = false;
      r.has |= 1u << d;
      r.v[d] += rr.v[d];
    }
}
// Resource.Multi, api/resource_info.go:323-330
void res_multi(Res &r, double ratio, int R) {
  r.v[0] *= ratio;
  r.v[1] *= ratio;
  for (int d = 2; d < R; ++d)
    if (r.has & (1u << d)) r.v[d] = r.v[d] * ratio;
}
// Resource.MinDimensionResource, api/resource_info.go:939-976
void res_min_dimension(Res &r, const Res &rr, bool infinity, int R) {
  if (rr.v[0] < r.v[0]) r.v[0] = rr.v[0];
  if (rr.v[1] < r.v[1]) r.v[1] = rr.v[1];
  if (r.nilmap) return;
  if (rr.nilmap) {
    if (infinity) return;
    for (int d = 2; d < R; ++d)
      if (r.has & (1u << d)) r.v[d] = 0;
    return;
  }
  for (int d = 2; d < R; ++d) {
    if (!(r.has & (1u << d))) continue;
    if (rr.has & (1u << d)) {
      r.v[d] = std::fmin(r.v[d], rr.v[d]);
    } else if (!infinity) {
      r.v[d] = 0;
    }
  }
}
// helpers.Max, api/helpers/helpers.go:51-77
Res res_max(const Res &l, const Res &r, int R) {
  Res o;
  o.v[0] = std::fmax(l.v[0], r.v[0]);
  o.v[1] = std::fmax(l.v[1], r.v[1]);
  if (l.nilmap && r.nilmap) return o;
  o.nilmap = false;
  for (int d = 2; d < R; ++d)
    if ((l.has & (1u << d)) && l.v[d] >= 0) {
      o.has |= 1u << d;
      o.v[d] = l.v[d];
    }
  for (int d = 2; d < R; ++d)
    if ((r.has & (1u << d)) && r.v[d] >= 0) {
      double cur = (o.has & (1u << d)) ? o.v[d] : 0.0;
      o.has |= 1u << d;
      o.v[d] = std::fmax(r.v[d], cur);
    }
  return o;
}
// Resource.Diff(rr, Zero), api/resource_info.go:879-918 (+ setDefaultValue :979-1000)
void res_diff_zero(const Res &l, const Res &r, Res &inc, Res &dec, int R) {
  inc = Res();
  dec = Res();
  uint32_t keys = l.has | r.has;
  if (l.v[0] > r.v[0]) inc.v[0] = l.v[0] - r.v[0]; else dec.v[0] = r.v[0] - l.v[0];
  if (l.v[1] > r.v[1]) inc.v[1] = l.v[1] - r.v[1]; else dec.v[1] = r.v[1] - l.v[1];
  inc.nilmap = dec.nilmap = false;  // make(map) in Diff
  for (int d = 2; d < R; ++d) {
    if (!(keys & (1u << d))) continue;
    double lq = (l.has & (1u << d)) ? l.v[d] : 0.0;
    double rq = (r.has & (1u << d)) ? r.v[d] : 0.0;
    if (lq == -1.0) { inc.has |= 1u << d; inc.v[d] = lq; continue; }
    if (rq == -1.0) { dec.has |= 1u << d; dec.v[d] = rq; continue; }
    if (lq > rq) { inc.has |= 1u << d; inc.v[d] = lq - rq; }
    else { dec.has |= 1u << d; dec.v[d] = rq - lq; }
  }
}
// ExceededPart, api/resource_info.go:1075-1086
Res res_exceeded_part(const Res &l, const Res &r, int R) {
  Res inc, dec;
  res_diff_zero(l, r, inc, dec, R);
  return inc;
}
// Resource.LessEqual(rr, Zero), api/resource_info.go:429-463
bool res_less_equal_zero(const Res &l, const Res &r, int R) {
  if (!le_eps(l.v[0], r.v[0])) return false;
  if (!le_eps(l.v[1], r.v[1])) return false;
  for (int d = 2; d < R; ++d) {
    if (!(l.has & (1u << d))) continue;
    double rv = (r.has & (1u << d)) ? r.v[d] : 0.0;
    if (!le_eps(l.v[d], rv)) return false;
  }
  return true;
}
// Resource.IsEmpty, api/resource_info.go:240-255
bool res_is_empty(const Res &r, int R, int pods_dim) {
  if (!(r.v[0] < kMinResource && r.v[1] < kMinResource)) return false;
  for (int d = 2; d < R; ++d) {
    if (!(r.has & (1u << d)) || d == pods_dim) continue;
    if (r.v[d] >= kMinResource) return false;
  }
  return true;
}
// equality.Semantic.DeepEqual on *Resource: same values, same key set (nil == empty map)
bool res_deep_equal(const Res &a, const Res &b, int R) {
  if (a.v[0] != b.v[0] || a.v[1] != b.v[1] || a.has != b.has) return false;
  for (int d = 2; d < R; ++d)
    if ((a.has & (1u << d)) && a.v[d] != b.v[d]) return false;
  return true;
}
// helpers.Share, api/helpers/helpers.go:80-93
inline double share_of(double l, double r) {
  if (r == 0) return l == 0 ? 0.0 : 1.0;
  return l / r;
}

// ---------------------------------------------------------------------------------------
// container/heap as used by util.PriorityQueue (util/priority_queue.go:30-111):
// heap.Push = append + up, heap.Pop = swap(0,n-1) + down + remove last.
// ---------------------------------------------------------------------------------------
struct GoHeap {
  std::vector<int> items;
  std::function<bool(int, int)> less;  // lessFn(items[i], items[j])
  bool empty() const { return items.empty(); }
  size_t size() const { return items.size(); }
  void push(int x) {
    items.push_back(x);
    int j = (int)items.size() - 1;
    for (;;) {
      int i = (j - 1) / 2;
      if (i == j || !less(items[j], items[i])) break;
      std::swap(items[i], items[j]);
      j = i;
    }
  }
  int pop() {
    int n = (int)items.size() - 1;
    std::swap(items[0], items[n]);
    int i = 0;
    for (;;) {
      int j1 = 2 * i + 1;
      if (j1 >= n || j1 < 0) break;
      int j = j1;
      int j2 = j1 + 1;
      if (j2 < n && less(items[j2], items[j1])) j = j2;
      if (!less(items[j], items[i])) break;
      std::swap(items[i], items[j]);
      i = j;
    }
    int x = items.back();
    items.pop_back();
    return x;
  }
};

// ---------------------------------------------------------------------------------------
// A tiny spinning thread pool: mirrors workqueue.ParallelizeUntil(ctx, 16, n, fn)
// (util/predicate_helper.go:133, util/scheduler_helper.go:103) with static chunks.
// ---------------------------------------------------------------------------------------
struct Pool {
  int nthreads = 1;
  std::vector<std::thread> workers;
  std::atomic<uint64_t> gen{0};
  std::atomic<int> done{0};
  std::atomic<bool> stop{false};
  std::function<void(int, int)> job;  // (begin, end)
  int total = 0;
  explicit Pool(int n) : nthreads(std::max(1, n)) {
    for (int w = 1; w < nthreads; ++w)
      workers.emplace_back([this, w] {
        uint64_t seen = 0;
        for (;;) {
          uint64_t g;
          int spins = 0;
          while ((g = gen.load(std::memory_order_acquire)) == seen) {
            if (stop.load(std::memory_order_relaxed)) return;
            if (++spins > 2000) { std::this_thread::yield(); spins = 0; }
          }
          seen = g;
          run_chunk(w);
          done.fetch_add(1, std::memory_order_release);
        }
      });
  }
  ~Pool() {
    stop.store(true);
    for (auto &t : workers) t.join();
  }
  void run_chunk(int w) {
    int per = (total + nthreads - 1) / nthreads;
    int b = std::min(total, w * per), e = std::min(total, b + per);
    if (b < e) job(b, e);
  }
  void parallel_for(int n, std::function<void(int, int)> fn) {
    if (nthreads == 1 || n < 256) { fn(0, n); return; }
    job = std::move(fn);
    total = n;
    done.store(0, std::memory_order_relaxed);
    gen.fetch_add(1, std::memory_order_release);
    run_chunk(0);
    while (done.load(std::memory_order_acquire) < nthreads - 1) {}
  }
};

// ---------------------------------------------------------------------------------------
// Session: the snapshot plus everything the plugins keep (framework/session.go:66-164)
// ---------------------------------------------------------------------------------------
enum TaskStatus : int8_t { kPending = 0, kAllocated = 1, kPipelined = 2, kBinding = 3, kRunning = 4, kBound = 5, kReleasing = 6 };

struct Op { int task; int node; int kind; double score; };  // Statement.operations (framework/statement.go:47-52)

struct QueueAttr {  // proportion.queueAttr (plugins/proportion/proportion.go:57-74)
  bool exists = false;
  Res deserved, allocated, request, capability, realCapability, guarantee;
  double share = 0;
  int32_t weight = 0;
};

struct Session {
  vc_dims d{};
  vc_conf conf{};
  int N = 0, T = 0, J = 0, Q = 0, C = 0, R = 0, K = 0, Wl = 0, Wt = 0, NR = 0;
  int T_alloc = 0;  // tasks [0, T_alloc) are allocate's; [T_alloc, T_run0) the BestEffort tasks of the backfill action
  int T_run0 = -1;  // tasks [T_run0, T) are node.Tasks entries (vc_running_tasks): victim candidates of preempt / reclaim
  std::vector<uint32_t> rt_flags;           // [T - T_run0] VC_RT_*
  std::vector<uint32_t> t_flags;            // [T_alloc] VC_TASK_*
  std::vector<std::vector<int>> node_tasks;  // node.Tasks restricted to those entries, ascending index (canonical order)
  // nodes
  std::vector<double> alloc, idle, used, rel, pip, kalloc, kreq, knz;
  std::vector<int32_t> max_tasks, pod_count, zone;
  std::vector<uint64_t> labels, thard, tsoft;
  std::vector<uint32_t> nflags;
  std::vector<uint8_t> zone_active;
  // tasks
  std::vector<double> req, tkreq, tknz;
  std::vector<uint32_t> req_has, t_uid;
  std::vector<int32_t> t_job, t_class, t_role, t_prio;
  std::vector<int64_t> t_podidx, t_ts;
  std::vector<int8_t> t_status;
  std::vector<int32_t> t_node;
  // classes
  std::vector<uint64_t> c_sel, c_aff, c_tolh, c_tols, c_pref;
  std::vector<int32_t> c_naff, c_npref, c_prefw;
  std::vector<uint32_t> c_flags;
  // jobs
  std::vector<int32_t> j_queue, j_min, j_prio, j_ntasks, j_ready, j_waiting, j_pbe, j_valid, j_taskmintotal,
      j_roleoff;
  std::vector<int64_t> j_ts;
  std::vector<uint32_t> j_uid, j_flags;
  std::vector<double> j_alloc;  // drf attr.allocated [R][J]
  std::vector<double> j_share;  // drf attr.share
  std::vector<int32_t> r_min, r_occ, r_pip, r_pending, r_valid;
  std::vector<uint32_t> r_flags;
  std::vector<uint8_t> r_failed;  // role has an entry in job.NodesFitErrors (FitFailedRoles, job_info.go:881-891)
  // queues
  std::vector<int32_t> q_weight, q_prio;
  std::vector<int64_t> q_ts;
  std::vector<uint32_t> q_uid, q_flags;
  std::vector<Res> q_cap, q_guar, q_alloc0, q_req0;
  std::vector<uint8_t> q_cap_any, q_guar_any;
  std::vector<QueueAttr> qattr;
  Res total;  // ssn.TotalResource (framework/session.go:272-274)
  bool has_plugin[128] = {false};
  // network-topology-aware: hypernode membership per tier level and the plugin's hyperNodeResourceCache
  int hn_H = 0, hn_L = 0, hn_min_tier = 1;
  std::vector<int32_t> hn_member;         // [L][N]
  std::vector<double> hn_alloc, hn_used;  // [R][H]
  double tier_w[VC_MAX_TIERS] = {0};
  double tier_w_total = 0.0;
  bool nta_on = false;      // plugin registered with EnabledNodeOrder and normal-pod binpacking enabled
  bool nta_plugin = false;  // plugin registered with EnabledNodeOrder
  std::vector<int32_t> hn_tier, hn_parent;     // [H]
  std::vector<uint8_t> job_soft;               // [J] default subJob in soft topology mode
  std::vector<int32_t> job_alloc_hn;           // [J] subJob.AllocatedHyperNode (-1 = "")
  std::vector<std::vector<int32_t>> job_placed;  // [J] node of every task of the job that carries a NodeName
  int task_alloc_hn = -1;                      // task.JobAllocatedHyperNode of the task being scored
  // results
  std::vector<vc_decision> decisions;
  std::vector<vc_visit> visits;
  std::vector<int32_t> fit_errors;
  int64_t sweeps = 0;
  int64_t last_processed_node_index = 0;  // util/scheduler_helper.go:50
  std::vector<int32_t> t_nominated;       // [T_alloc] node of Pod.Status.NominatedNodeName or -1; empty: none
  Pool *pool = nullptr;
  ~Session() { delete pool; }
};

inline double &at(std::vector<double> &v, int d, int n, int i) { return v[(size_t)d * n + i]; }
inline double at(const std::vector<double> &v, int d, int n, int i) { return v[(size_t)d * n + i]; }

template <typename Tv>
void copy_in(std::vector<Tv> &dst, const Tv *src, size_t n, Tv fill = Tv()) {
  dst.assign(n, fill);
  if (src && n) std::memcpy(dst.data(), src, n * sizeof(Tv));
}

// ---------------------------------------------------------------------------------------
// JobInfo readiness (api/job_info.go)
// ---------------------------------------------------------------------------------------
// CheckTaskReady, api/job_info.go:1024-1036
bool check_task_ready(const Session &s, int j) {
  if (s.j_min[j] < s.j_taskmintotal[j]) return true;
  for (int r = s.j_roleoff[j]; r < s.j_roleoff[j + 1]; ++r)
    if ((s.r_flags[r] & VC_ROLE_IN_MIN_MAP) && s.r_occ[r] < s.r_min[r]) return false;
  return true;
}
// CheckTaskPipelined, api/job_info.go:1039-1070
bool check_task_pipelined(const Session &s, int j) {
  if (s.j_min[j] < s.j_taskmintotal[j]) return true;
  for (int r = s.j_roleoff[j]; r < s.j_roleoff[j + 1]; ++r)
    if ((s.r_flags[r] & VC_ROLE_IN_MIN_MAP) && s.r_occ[r] + s.r_pip[r] < s.r_min[r]) return false;
  return true;
}
// IsReady / IsPipelined, api/job_info.go:1169-1175
bool is_ready(const Session &s, int j) { return s.j_ready[j] + s.j_pbe[j] >= s.j_min[j]; }
bool is_pipelined(const Session &s, int j) { return s.j_waiting[j] + s.j_ready[j] + s.j_pbe[j] >= s.j_min[j]; }

// ssn.JobReady, framework/session_plugins.go:428-446; gang fn plugins/gang/gang.go:183-189
bool job_ready(const Session &s, int j) {
  for (int i = 0; i < s.conf.n_plugins; ++i) {
    const vc_plugin_option &p = s.conf.plugins[i];
    if (!(p.enabled & VC_EN_JOB_READY)) continue;
    if (p.plugin == VC_PLUGIN_GANG && !(check_task_ready(s, j) && is_ready(s, j))) return false;
  }
  return true;
}
// ssn.JobPipelined, framework/session_plugins.go:450-478 (Permit=1, Abstain=0, Reject=-1)
bool job_pipelined(const Session &s, int j) {
  bool has_found = false;
  int i = 0;
  while (i < s.conf.n_plugins) {
    int tier = s.conf.plugins[i].tier;
    for (; i < s.conf.n_plugins && s.conf.plugins[i].tier == tier; ++i) {
      const vc_plugin_option &p = s.conf.plugins[i];
      if (!(p.enabled & VC_EN_JOB_PIPELINED)) continue;
      int res;
      if (p.plugin == VC_PLUGIN_GANG)  // gang.go:191-197
        res = (check_task_pipelined(s, j) && is_pipelined(s, j)) ? 1 : -1;
      else if (p.plugin == VC_PLUGIN_TDM)  // tdm.go:275-281
        res = is_pipelined(s, j) ? 1 : -1;
      else
        continue;
      if (res < 0) return false;
      if (res > 0) has_found = true;
    }
    if (has_found) return true;
  }
  return true;
}
// ssn.JobValid -> gang validJobFn, plugins/gang/gang.go:58-93; CheckTaskValid job_info.go:993-1019
bool job_valid(const Session &s, int j) {
  if (!s.has_plugin[VC_PLUGIN_GANG]) return true;
  if (!(s.j_min[j] < s.j_taskmintotal[j])) {
    for (int r = s.j_roleoff[j]; r < s.j_roleoff[j + 1]; ++r) {
      if (!(s.r_flags[r] & VC_ROLE_IN_MIN_MAP) || s.r_min[r] == 0) continue;
      if (s.r_valid[r] < s.r_min[r]) return false;  // `!ok || act < minAvailable`
    }
  }
  return s.j_valid[j] >= s.j_min[j];
}

// ---------------------------------------------------------------------------------------
// Ordering functions (framework/session_plugins.go:660-783)
// ---------------------------------------------------------------------------------------
bool job_order_less(const Session &s, int l, int r) {  // ssn.JobOrderFn :660-683
  for (int i = 0; i < s.conf.n_plugins; ++i) {
    const vc_plugin_option &p = s.conf.plugins[i];
    if (!(p.enabled & VC_EN_JOB_ORDER)) continue;
    int c = 0;
    switch (p.plugin) {
      case VC_PLUGIN_PRIORITY:  // priority.go:73-89
        if (s.j_prio[l] > s.j_prio[r]) c = -1;
        else if (s.j_prio[l] < s.j_prio[r]) c = 1;
        break;
      case VC_PLUGIN_GANG: {  // gang.go:131-155
        bool lr = is_ready(s, l), rr = is_ready(s, r);
        if (lr && rr) c = 0;
        else if (lr) c = 1;
        else if (rr) c = -1;
        break;
      }
      case VC_PLUGIN_DRF:  // drf.go:370-388
        if (s.j_share[l] == s.j_share[r]) c = 0;
        else c = s.j_share[l] < s.j_share[r] ? -1 : 1;
        break;
      case VC_PLUGIN_TDM: {  // tdm.go:261-273
        bool lp = (s.j_flags[l] & VC_JOB_PREEMPTABLE) != 0, rp = (s.j_flags[r] & VC_JOB_PREEMPTABLE) != 0;
        if (lp == rp) c = 0;
        else c = !lp ? -1 : 1;
        break;
      }
      default: break;
    }
    if (c != 0) return c < 0;
  }
  if (s.j_ts[l] == s.j_ts[r]) return s.j_uid[l] < s.j_uid[r];
  return s.j_ts[l] < s.j_ts[r];
}
// ssn.QueueOrderFn :709-731; proportion fn plugins/proportion/proportion.go:266-284
bool queue_order_less(const Session &s, int l, int r) {
  for (int i = 0; i < s.conf.n_plugins; ++i) {
    const vc_plugin_option &p = s.conf.plugins[i];
    if (!(p.enabled & VC_EN_QUEUE_ORDER)) continue;
    if (p.plugin == VC_PLUGIN_PROPORTION) {
      if (s.q_prio[l] != s.q_prio[r]) return (s.q_prio[r] - s.q_prio[l]) < 0;
      double ls = s.qattr[l].share, rs = s.qattr[r].share;
      if (ls != rs) return ls < rs;
    }
  }
  if (s.q_ts[l] == s.q_ts[r]) return s.q_uid[l] < s.q_uid[r];
  return s.q_ts[l] < s.q_ts[r];
}
// ssn.TaskOrderFn :772-783: priority plugin (priority.go:50-69) then helpers.CompareTask
// (pkg/controllers/job/helpers/helpers.go:54-69)
bool task_order_less(const Session &s, int l, int r) {
  for (int i = 0; i < s.conf.n_plugins; ++i) {
    const vc_plugin_option &p = s.conf.plugins[i];
    if (!(p.enabled & VC_EN_TASK_ORDER)) continue;
    if (p.plugin == VC_PLUGIN_PRIORITY && s.t_prio[l] != s.t_prio[r]) return s.t_prio[l] > s.t_prio[r];
  }
  bool lerr = s.t_podidx[l] < 0, rerr = s.t_podidx[r] < 0;
  if (lerr || rerr || s.t_podidx[l] == s.t_podidx[r]) {
    if (s.t_ts[l] == s.t_ts[r]) return s.t_uid[l] < s.t_uid[r];
    return s.t_ts[l] < s.t_ts[r];
  }
  return !(s.t_podidx[l] > s.t_podidx[r]);
}

// ---------------------------------------------------------------------------------------
// Plugin state
// ---------------------------------------------------------------------------------------
// drf.calculateShare, plugins/drf/drf.go:566-578 (ResourceNames() = dims with total >= 0.1)
void drf_update_share(Session &s, int j) {
  double res = 0;
  for (int d = 0; d < s.R; ++d) {
    if (d >= 2 && !(s.total.has & (1u << d))) continue;
    if (!(s.total.v[d] >= kMinResource)) continue;
    double sh = share_of(at(s.j_alloc, d, s.J, j), s.total.v[d]);
    if (sh > res) res = sh;
  }
  s.j_share[j] = res;
}
// updateQueueAttrShare, plugins/proportion/proportion.go:590-602
void proportion_update_share(const Session &s, QueueAttr &a) {
  double res = 0;
  for (int d = 0; d < s.R; ++d) {
    if (d >= 2 && !(a.deserved.has & (1u << d))) continue;
    if (!(a.deserved.v[d] >= kMinResource)) continue;
    double al = (d < 2 || (a.allocated.has & (1u << d))) ? a.allocated.v[d] : 0.0;
    double sh = share_of(al, a.deserved.v[d]);
    if (sh > res) res = sh;
  }
  a.share = res;
}

Res task_res(const Session &s, int t) {
  Res r;
  for (int d = 0; d < s.R; ++d) r.v[d] = at(s.req, d, s.T, t);
  r.has = s.req_has[t] & ~3u;
  for (int d = 2; d < s.R; ++d)
    if (!(r.has & (1u << d))) r.v[d] = 0;
  r.nilmap = r.has == 0;
  return r;
}

// proportion OnSessionOpen, plugins/proportion/proportion.go:90-264
void proportion_open(Session &s) {
  const int R = s.R;
  s.qattr.assign(s.Q, QueueAttr());
  if (!s.has_plugin[VC_PLUGIN_PROPORTION]) return;
  Res total_guarantee;  // :95-101, over every queue of the session
  for (int q = 0; q < s.Q; ++q)
    if (s.q_guar_any[q]) res_add(total_guarantee, s.q_guar[q], R);
  // :103-142 — attributes exist only for queues that own at least one job
  for (int j = 0; j < s.J; ++j) {
    int q = s.j_queue[j];
    if (q < 0 || s.qattr[q].exists) continue;
    QueueAttr &a = s.qattr[q];
    a.exists = true;
    a.weight = s.q_weight[q];
    bool has_cap = s.q_cap_any[q];
    if (has_cap) {
      a.capability = s.q_cap[q];
      if (a.capability.v[0] <= 0) a.capability.v[0] = std::numeric_limits<double>::max();
      if (a.capability.v[1] <= 0) a.capability.v[1] = std::numeric_limits<double>::max();
    }
    if (s.q_guar_any[q]) a.guarantee = s.q_guar[q];
    Res real_cap = res_exceeded_part(s.total, total_guarantee, R);
    res_add(real_cap, a.guarantee, R);
    if (has_cap) res_min_dimension(real_cap, a.capability, /*infinity=*/true, R);
    a.realCapability = real_cap;
    a.allocated = s.q_alloc0[q];  // :143-156, summed by the snapshot encoder
    a.request = s.q_req0[q];
  }
  // :197-264 water-filling
  Res remaining = s.total;
  std::vector<uint8_t> meet(s.Q, 0);
  for (;;) {
    int32_t total_weight = 0;
    for (int q = 0; q < s.Q; ++q)
      if (s.qattr[q].exists && !meet[q]) total_weight += s.qattr[q].weight;
    if (total_weight == 0) break;
    Res old_remaining = remaining;
    Res increased, decreased;
    for (int q = 0; q < s.Q; ++q) {
      QueueAttr &a = s.qattr[q];
      if (!a.exists || meet[q]) continue;
      Res old_deserved = a.deserved;
      Res part = remaining;
      res_multi(part, (double)a.weight / (double)total_weight, R);
      res_add(a.deserved, part, R);
      res_min_dimension(a.deserved, a.realCapability, /*infinity=*/true, R);
      res_min_dimension(a.deserved, a.request, /*infinity=*/false, R);
      a.deserved = res_max(a.deserved, a.guarantee, R);
      proportion_update_share(s, a);
      if (res_less_equal_zero(a.request, a.deserved, R)) meet[q] = 1;
      else if (res_deep_equal(a.deserved, old_deserved, R)) meet[q] = 1;
      Res inc, dec;
      res_diff_zero(a.deserved, old_deserved, inc, dec, R);
      res_add(increased, inc, R);
      res_add(decreased, dec, R);
    }
    Res tmp = remaining;
    res_add(tmp, decreased, R);
    remaining = res_exceeded_part(tmp, increased, R);
    if (res_is_empty(remaining, R, s.d.pods_dim) || res_deep_equal(remaining, old_remaining, R)) break;
  }
}

// proportion OverusedFn, plugins/proportion/proportion.go:319-331
bool overused(const Session &s, int q) {
  for (int i = 0; i < s.conf.n_plugins; ++i) {
    const vc_plugin_option &p = s.conf.plugins[i];
    if (!(p.enabled & VC_EN_OVERUSED)) continue;
    if (p.plugin == VC_PLUGIN_PROPORTION) {
      const QueueAttr &a = s.qattr[q];
      if (res_less_equal_zero(a.deserved, a.allocated, s.R)) return true;
    }
  }
  return false;
}
// ssn.Allocatable :350-366 -> proportion queueAllocatable, proportion.go:333-348, using
// LessEqualWithDimensionAndResourcesName with a non-nil req, api/resource_info.go:469-514: only the dimensions `req`
// asks for (> 0) are compared, strictly (no epsilon); `pods` is an ignored scalar (IsIgnoredScalarResource :219)
bool res_less_equal_with_dimension(const Res &l, const Res &r, const Res &req, int R, int pods_dim) {
  bool ok = true;
  if (req.v[0] > 0 && l.v[0] > r.v[0]) ok = false;
  if (req.v[1] > 0 && l.v[1] > r.v[1]) ok = false;
  if (l.nilmap) return ok;  // r.ScalarResources == nil: whatever rr holds, the scalars pass
  for (int d = 2; d < R; ++d) {
    if (!(req.has & (1u << d)) || d == pods_dim) continue;
    double lq = (l.has & (1u << d)) ? l.v[d] : 0.0;
    double rq = (r.has & (1u << d)) ? r.v[d] : 0.0;
    if (req.v[d] > 0 && lq > rq) ok = false;
  }
  return ok;
}
// proportion's AllocatableFn through ssn.Allocatable: queueAllocatable, proportion.go:333-348
bool queue_allocatable(const Session &s, int q, int t) {  // proportion.go:333-348
  if (!(s.q_flags[q] & VC_QUEUE_OPEN)) return false;
  const QueueAttr &a = s.qattr[q];
  Res fu = a.allocated;
  Res rq = task_res(s, t);
  res_add(fu, rq, s.R);
  return res_less_equal_with_dimension(fu, a.deserved, rq, s.R, s.d.pods_dim);
}
bool allocatable(const Session &s, int q, int t) {
  for (int i = 0; i < s.conf.n_plugins; ++i) {
    const vc_plugin_option &p = s.conf.plugins[i];
    if (!(p.enabled & VC_EN_ALLOCATABLE)) continue;
    if (p.plugin != VC_PLUGIN_PROPORTION) continue;
    if (!queue_allocatable(s, q, t)) return false;
  }
  return true;
}
// ssn.Preemptive, framework/session_plugins.go:330-347: proportion's PreemptiveFn is queueAllocatable (proportion.go:376-380)
bool preemptive(const Session &s, int q, int t) {
  for (int i = 0; i < s.conf.n_plugins; ++i) {
    const vc_plugin_option &p = s.conf.plugins[i];
    if (!(p.enabled & VC_EN_PREEMPTIVE)) continue;
    if (p.plugin != VC_PLUGIN_PROPORTION) continue;
    if (!queue_allocatable(s, q, t)) return false;
  }
  return true;
}

// Event handlers fired by Statement.Allocate / Pipeline (AllocateFunc) and by
// unallocate / UnPipeline (DeallocateFunc): drf.go:391-454, proportion.go:475-518,
// predicates.go:212-304 (k8s NodeInfo AddPodInfo / RemovePod).
// ---------------------------------------------------------------------------------------
// network-topology-aware, hypernode-level binpacking of pods without a network topology
// (plugins/network-topology-aware/network_topology_aware.go)
// ---------------------------------------------------------------------------------------
// Go's math.Pow for a non-negative integer exponent (restated from the published Go runtime
// algorithm, src/math/pow.go: special cases, then binary exponentiation on the Frexp mantissa, which is
// the same sequence of fp64 products as on the values themselves). Used for the tier weights :470-476.
double go_pow_uint(double x, unsigned n) {
  if (n == 0 || x == 1.0) return 1.0;
  if (n == 1) return x;
  if (x == 0.0) return 0.0;
  int xe = 0, ae = 0;
  double x1 = std::frexp(x, &xe), a1 = 1.0;
  for (unsigned i = n; i != 0; i >>= 1) {
    if (i & 1u) { a1 *= x1; ae += xe; }
    x1 *= x1;
    xe <<= 1;
    if (x1 < 0.5) { x1 += x1; xe--; }
  }
  return std::ldexp(a1, ae);
}
// hyperNodesTier.init :97-104, initHyperNodeResourceCache :106-125, tier weights :469-476
void nta_init(Session &s, const vc_hypernodes *topo) {
  s.nta_on = s.nta_plugin = false;
  for (int i = 0; i < s.conf.n_plugins; ++i)
    if (s.conf.plugins[i].plugin == VC_PLUGIN_NETWORK_TOPOLOGY_AWARE && (s.conf.plugins[i].enabled & VC_EN_NODE_ORDER)) {
      s.nta_plugin = true;
      if (s.conf.nta_normal_pod_enable) s.nta_on = true;
    }
  s.job_soft.assign(s.J, 0);
  s.job_alloc_hn.assign(s.J, -1);
  s.job_placed.assign(s.J, {});
  if (topo && topo->member) {
    s.hn_H = topo->n_hypernodes;
    s.hn_min_tier = topo->min_tier;
    s.hn_L = topo->max_tier - topo->min_tier + 1;
    s.hn_member.assign(topo->member, topo->member + (size_t)s.hn_L * s.N);
    if (topo->tier) s.hn_tier.assign(topo->tier, topo->tier + s.hn_H);
    if (topo->parent) s.hn_parent.assign(topo->parent, topo->parent + s.hn_H);
    if (topo->job_soft) s.job_soft.assign(topo->job_soft, topo->job_soft + s.J);
    if (topo->job_allocated) s.job_alloc_hn.assign(topo->job_allocated, topo->job_allocated + s.J);
    if (topo->job_placed_off && topo->job_placed_node)
      for (int j = 0; j < s.J; ++j)
        s.job_placed[j].assign(topo->job_placed_node + topo->job_placed_off[j], topo->job_placed_node + topo->job_placed_off[j + 1]);
  } else {  // no HyperNode objects: only the cluster top hypernode, tier 1 (framework/session.go:285-313)
    s.hn_H = 1; s.hn_min_tier = 1; s.hn_L = 1;
    s.hn_member.assign((size_t)s.N, 0);
  }
  s.hn_alloc.assign((size_t)s.R * s.hn_H, 0.0);
  s.hn_used.assign((size_t)s.R * s.hn_H, 0.0);
  for (int l = 0; l < s.hn_L; ++l)
    for (int n = 0; n < s.N; ++n) {
      int h = s.hn_member[(size_t)l * s.N + n];
      if (h < 0) continue;
      for (int d = 0; d < s.R; ++d) {
        at(s.hn_alloc, d, s.hn_H, h) += at(s.alloc, d, s.N, n);
        at(s.hn_used, d, s.hn_H, h) += at(s.used, d, s.N, n);
      }
    }
  s.tier_w_total = 0.0;
  for (int l = 0; l < s.hn_L && l < VC_MAX_TIERS; ++l) {
    int tier = s.hn_min_tier + l;
    s.tier_w[l] = go_pow_uint(s.conf.nta_fading, (unsigned)(tier - 1));
    s.tier_w_total += s.tier_w[l];
  }
}
// getPodHyperNodeBinPackingScore :498-539
double hn_binpack_score(const Session &s, int t, int h) {
  double total_score = 0.0;
  int total_weight = 0;
  for (int d = 0; d < s.R; ++d) {
    double request = at(s.req, d, s.T, t);
    if (d >= 2 && !(s.req_has[t] & (1u << d))) continue;  // task.Resreq.ResourceNames()
    if (!(request >= kMinResource)) continue;
    int w = s.conf.nta_dim_weight[d];
    if (w < 0) continue;  // getBinPackWeight: not found
    double allocatable = at(s.hn_alloc, d, s.hn_H, h);
    double used = at(s.hn_used, d, s.hn_H, h);
    if (used + request > allocatable) return 0.0;
    double score = (used + request) / allocatable;
    total_score += (double)w * score;
    total_weight += w;
  }
  if (total_weight > 0) return total_score / (double)total_weight;
  return 0.0;
}
// batchNodeOrderFnForNormalPods :462-496 + scaleFinalScore :758-764 for one node
double nta_node_score(const Session &s, int t, int n) {
  double total = 0.0;
  for (int l = 0; l < s.hn_L; ++l) {
    int h = s.hn_member[(size_t)l * s.N + n];
    double tier_score = h < 0 ? 1.0 : hn_binpack_score(s, t, h);  // FullScore when no hypernode of the tier holds the node
    total += s.tier_w[l] * tier_score;
  }
  double sc = total / s.tier_w_total;
  return (double)kMaxNodeScore * (double)s.conf.nta_weight * sc;
}
void nta_account(Session &s, int t, int n, double sign) {  // event handlers :374-399
  for (int l = 0; l < s.hn_L; ++l) {
    int h = s.hn_member[(size_t)l * s.N + n];
    if (h < 0) continue;
    for (int d = 0; d < s.R; ++d) {
      if (d >= 2 && !(s.req_has[t] & (1u << d))) continue;
      at(s.hn_used, d, s.hn_H, h) += sign * at(s.req, d, s.T, t);
    }
  }
}

// ---- pods WITH a (soft-mode) network topology: batchNodeOrderFnForNetworkAwarePods :541-571 ----
// HyperNodeInfoMap.GetAncestors (api/hyper_node_info.go:737-758): the hypernode, then its parents upwards
std::vector<int> hn_ancestors(const Session &s, int h) {
  std::vector<int> out;
  while (h >= 0 && std::find(out.begin(), out.end(), h) == out.end()) {
    out.push_back(h);
    h = h < (int)s.hn_parent.size() ? s.hn_parent[h] : -1;
  }
  return out;
}
// GetLCAHyperNode(hypernode, jobHyperNode), api/hyper_node_info.go:787-809
int hn_lca(const Session &s, int hypernode, int job_hypernode) {
  if (hypernode < 0) return job_hypernode;
  if (job_hypernode < 0) return hypernode;
  std::vector<int> a = hn_ancestors(s, hypernode);
  for (int x : hn_ancestors(s, job_hypernode))
    if (std::find(a.begin(), a.end(), x) != a.end()) return x;
  return -1;
}
// util.FindHyperNodeForNode (util/scheduler_helper.go:361-376): only hypernodes of the LOWEST tier are searched
int find_hypernode_for_node(const Session &s, int n) { return s.hn_member[n]; }
// networkTopologyAwareScore :716-733 + scoreHyperNodeWithTier :747-756
double topo_score(const Session &s, int hn, int allocated) {
  if (hn < 0 || allocated < 0) return 0.0;
  if (hn == allocated) return 1.0;
  int lca = hn_lca(s, hn, allocated);
  if (lca < 0) return 0.0;
  const int min_tier = s.hn_min_tier, max_tier = s.hn_min_tier + s.hn_L - 1, tier = s.hn_tier[lca];
  if (min_tier == max_tier) return 1.0;
  if (min_tier <= tier && tier <= max_tier) return (double)(max_tier - tier) / (double)(max_tier - min_tier);
  return 0.0;
}
// scoreWithTaskNum :737-745 -> util.FindJobTaskNumOfHyperNode (scheduler_helper.go:379-393)
double task_num_score(const Session &s, int j, int hn) {
  int cnt = 0;
  if (hn >= 0)
    for (int m : s.job_placed[j])
      if (s.hn_member[m] == hn) ++cnt;
  const int all = s.j_ntasks[j];
  return all > 0 ? (double)cnt / (double)all : 0.0;
}
// the map batchNodeOrderFnForNetworkAwarePods returns for `nodes` (before scaleFinalScore); has[i] = entry present
void topo_node_scores(const Session &s, int t, const std::vector<int> &nodes, std::vector<double> &out,
                      std::vector<uint8_t> &has) {
  out.assign(nodes.size(), 0.0);
  has.assign(nodes.size(), 0);
  const int allocated = s.task_alloc_hn;
  if (allocated < 0) return;  // :544-547: no scores at all
  double max_score = -1.0;
  for (size_t i = 0; i < nodes.size(); ++i) {
    out[i] = topo_score(s, find_hypernode_for_node(s, nodes[i]), allocated);
    has[i] = 1;
    if (out[i] >= max_score) max_score = out[i];
  }
  size_t at_max = 0;
  for (size_t i = 0; i < nodes.size(); ++i) at_max += out[i] == max_score;
  if (at_max > 1)
    for (size_t i = 0; i < nodes.size(); ++i)
      if (out[i] == max_score) out[i] += task_num_score(s, s.t_job[t], find_hypernode_for_node(s, nodes[i]));
}
// allocate.getNewAllocatedHyperNode, actions/allocate/allocate.go:697-707
int new_allocated_hypernode(const Session &s, int best_node, int allocated) {
  int hn = find_hypernode_for_node(s, best_node);
  if (hn >= 0) return allocated < 0 ? hn : hn_lca(s, hn, allocated);
  return allocated;
}
bool topo_task(const Session &s, int t) { return s.nta_plugin && s.job_soft[s.t_job[t]]; }

void on_allocate_event(Session &s, int t, int n) {
  int j = s.t_job[t];
  if (s.has_plugin[VC_PLUGIN_DRF]) {
    for (int d = 0; d < s.R; ++d) at(s.j_alloc, d, s.J, j) += at(s.req, d, s.T, t);
    drf_update_share(s, j);
  }
  if (s.has_plugin[VC_PLUGIN_PROPORTION] && s.j_queue[j] >= 0 && s.qattr[s.j_queue[j]].exists) {
    QueueAttr &a = s.qattr[s.j_queue[j]];
    res_add(a.allocated, task_res(s, t), s.R);
    proportion_update_share(s, a);
  }
  if (s.has_plugin[VC_PLUGIN_NETWORK_TOPOLOGY_AWARE]) nta_account(s, t, n, 1.0);
  if (s.has_plugin[VC_PLUGIN_PREDICATES]) {
    s.pod_count[n] += 1;
    for (int k = 0; k < s.K; ++k) {
      at(s.kreq, k, s.N, n) += at(s.tkreq, k, s.T, t);
      at(s.knz, k, s.N, n) += at(s.tknz, k, s.T, t);
    }
  }
}
void on_deallocate_event(Session &s, int t, int n) {
  int j = s.t_job[t];
  if (s.has_plugin[VC_PLUGIN_DRF]) {
    for (int d = 0; d < s.R; ++d) at(s.j_alloc, d, s.J, j) -= at(s.req, d, s.T, t);
    drf_update_share(s, j);
  }
  if (s.has_plugin[VC_PLUGIN_PROPORTION] && s.j_queue[j] >= 0 && s.qattr[s.j_queue[j]].exists) {
    QueueAttr &a = s.qattr[s.j_queue[j]];
    Res rq = task_res(s, t);  // Resource.Sub -> sub, api/resource_info.go:293-320
    a.allocated.v[0] -= rq.v[0];
    a.allocated.v[1] -= rq.v[1];
    if (!a.allocated.nilmap)
      for (int d = 2; d < s.R; ++d)
        if (rq.has & (1u << d)) {
          a.allocated.has |= 1u << d;
          a.allocated.v[d] -= rq.v[d];
        }
    proportion_update_share(s, a);
  }
  if (s.has_plugin[VC_PLUGIN_NETWORK_TOPOLOGY_AWARE]) nta_account(s, t, n, -1.0);
  if (s.has_plugin[VC_PLUGIN_PREDICATES]) {
    s.pod_count[n] -= 1;
    for (int k = 0; k < s.K; ++k) {
      at(s.kreq, k, s.N, n) -= at(s.tkreq, k, s.T, t);
      at(s.knz, k, s.N, n) -= at(s.tknz, k, s.T, t);
    }
  }
}

// ---------------------------------------------------------------------------------------
// Resource fit: task.InitResreq.LessEqual(x, Zero), api/resource_info.go:429-463
// ---------------------------------------------------------------------------------------
inline double future_idle(const Session &s, int d, int n) {  // NodeInfo.FutureIdle, api/node_info.go:114-116
  return (at(s.idle, d, s.N, n) + at(s.rel, d, s.N, n)) - at(s.pip, d, s.N, n);
}
bool fits_idle(const Session &s, int t, int n) {
  for (int d = 0; d < s.R; ++d) {
    if (d >= 2 && !(s.req_has[t] & (1u << d))) continue;
    if (!le_eps(at(s.req, d, s.T, t), at(s.idle, d, s.N, n))) return false;
  }
  return true;
}
bool fits_future_idle(const Session &s, int t, int n) {
  for (int d = 0; d < s.R; ++d) {
    if (d >= 2 && !(s.req_has[t] & (1u << d))) continue;
    if (!le_eps(at(s.req, d, s.T, t), future_idle(s, d, n))) return false;
  }
  return true;
}

// ---------------------------------------------------------------------------------------
// Predicates (allocate.predicate allocate.go:816-824 -> ssn.PredicateForAllocateAction
// session.go:657-674 -> ssn.PredicateFn session_plugins.go:784-801)
// ---------------------------------------------------------------------------------------
inline bool mask_subset(const uint64_t *need, const std::vector<uint64_t> &bits, int W, int N, int n) {
  for (int w = 0; w < W; ++w)
    if ((bits[(size_t)w * N + n] & need[w]) != need[w]) return false;
  return true;
}
// predicates.Predicate for pods without ports/volumes/pod-affinity/DRA:
// pod-count cap (predicates.go:662-671), then the stable filters NodeUnschedulable,
// NodeAffinity (nodeSelector + required terms), TaintToleration (NoSchedule/NoExecute).
bool predicates_plugin_ok(const Session &s, int t, int n) {
  bool ok = true;
  if (s.max_tasks[n] <= s.pod_count[n]) ok = false;
  int c = s.t_class[t];
  if ((s.nflags[n] & VC_NODE_UNSCHEDULABLE) && !(s.c_flags[c] & VC_CLASS_TOLERATES_UNSCHEDULABLE)) ok = false;
  if (s.conf.predicates_enable & VC_PRED_NODE_AFFINITY) {
    if (!mask_subset(&s.c_sel[(size_t)c * s.Wl], s.labels, s.Wl, s.N, n)) ok = false;
    int na = s.c_naff[c];
    if (na > 0) {
      bool any = false;
      for (int k = 0; k < na && !any; ++k)
        any = mask_subset(&s.c_aff[((size_t)c * VC_MAX_TERMS + k) * s.Wl], s.labels, s.Wl, s.N, n);
      if (!any) ok = false;
    }
  }
  if (s.conf.predicates_enable & VC_PRED_TAINT_TOLERATION) {
    for (int w = 0; w < s.Wt; ++w)
      if (s.thard[(size_t)w * s.N + n] & ~s.c_tolh[(size_t)c * s.Wt + w]) ok = false;
  }
  return ok;
}
// tdm predicateFn, plugins/tdm/tdm.go:146-171
bool tdm_predicate_ok(const Session &s, int t, int n) {
  int z = s.zone[n];
  if (z < 0) return true;
  if (!s.zone_active[z]) return false;
  if (!(s.c_flags[s.t_class[t]] & VC_CLASS_REVOCABLE)) return false;
  return true;
}
bool predicate(const Session &s, int t, int n) {
  if (!fits_future_idle(s, t, n)) return false;
  for (int i = 0; i < s.conf.n_plugins; ++i) {
    const vc_plugin_option &p = s.conf.plugins[i];
    if (!(p.enabled & VC_EN_PREDICATE)) continue;
    if (p.plugin == VC_PLUGIN_PREDICATES && !predicates_plugin_ok(s, t, n)) return false;
    if (p.plugin == VC_PLUGIN_TDM && !tdm_predicate_ok(s, t, n)) return false;
  }
  return true;
}

// ---------------------------------------------------------------------------------------
// Scores
// ---------------------------------------------------------------------------------------
// BinPackingScore / ResourceBinPackingScore, plugins/binpack/binpack.go:206-261
double binpack_score(const Session &s, int t, int n) {
  double score = 0.0;
  int weight_sum = 0;
  for (int d = 0; d < s.R; ++d) {
    double request = at(s.req, d, s.T, t);
    if (d >= 2 && !(s.req_has[t] & (1u << d))) continue;  // ResourceNames(): keys of the map ...
    if (!(request >= kMinResource)) continue;             // ... with amount >= minResource
    if (request == 0) continue;
    int w = s.conf.binpack_dim_weight[d];
    if (w < 0) continue;  // not found in BinPackingResources
    double allocate = at(s.alloc, d, s.N, n);
    double node_used = at(s.used, d, s.N, n);
    double resource_score = 0;
    if (!(allocate == 0 || w == 0)) {
      double used_finally = request + node_used;
      if (used_finally > allocate) return 0;
      resource_score = used_finally * (double)w / allocate;
    }
    score += resource_score;
    weight_sum += w;
  }
  if (weight_sum > 0) score /= (double)weight_sum;
  score *= (double)(kMaxNodeScore * (int64_t)s.conf.binpack_weight);
  return score;
}

// Upstream kube-scheduler v1.35 noderesources scorers (pkg/scheduler/framework/plugins/
// noderesources/{resource_allocation,least_allocated,most_allocated,balanced_allocation}.go),
// restated from the published algorithm; constructed at plugins/nodeorder/nodeorder.go:204-244.
int64_t least_requested_score(int64_t requested, int64_t capacity) {
  if (capacity == 0) return 0;
  if (requested > capacity) return 0;
  return ((capacity - requested) * kMaxNodeScore) / capacity;
}
int64_t most_requested_score(int64_t requested, int64_t capacity) {
  if (capacity == 0) return 0;
  if (requested > capacity) requested = capacity;
  return (requested * kMaxNodeScore) / capacity;
}
int64_t least_allocated(const Session &s, int t, int n) {  // resources cpu:50, memory:50 (nodeorder.go:206-211)
  int64_t node_score = 0, weight_sum = 0;
  for (int k = 0; k < 2 && k < s.K; ++k) {
    int64_t alloc = (int64_t)at(s.kalloc, k, s.N, n);
    int64_t reqv = (int64_t)at(s.knz, k, s.N, n) + (int64_t)at(s.tknz, k, s.T, t);
    if (alloc == 0) continue;
    node_score += least_requested_score(reqv, alloc) * 50;
    weight_sum += 50;
  }
  return weight_sum == 0 ? 0 : node_score / weight_sum;
}
int64_t most_allocated(const Session &s, int t, int n) {  // cpu:1, memory:1 (nodeorder.go:222-227)
  int64_t node_score = 0, weight_sum = 0;
  for (int k = 0; k < 2 && k < s.K; ++k) {
    int64_t alloc = (int64_t)at(s.kalloc, k, s.N, n);
    int64_t reqv = (int64_t)at(s.knz, k, s.N, n) + (int64_t)at(s.tknz, k, s.T, t);
    if (alloc == 0) continue;
    node_score += most_requested_score(reqv, alloc) * 1;
    weight_sum += 1;
  }
  return weight_sum == 0 ? 0 : node_score / weight_sum;
}
int64_t balanced_allocation(const Session &s, int t, int n) {  // cpu, memory, nvidia.com/gpu (nodeorder.go:238-244)
  double fractions[VC_MAX_KDIMS];
  int nf = 0;
  double total_fraction = 0;
  for (int k = 0; k < s.K; ++k) {
    int64_t pod_req = (int64_t)at(s.tkreq, k, s.T, t);
    if (k >= 2 && pod_req == 0) continue;  // extended resource the pod does not request
    int64_t alloc = (int64_t)at(s.kalloc, k, s.N, n);
    if (alloc == 0) continue;
    int64_t reqv = (int64_t)at(s.kreq, k, s.N, n) + pod_req;
    double fraction = (double)reqv / (double)alloc;
    if (fraction > 1) fraction = 1;
    total_fraction += fraction;
    fractions[nf++] = fraction;
  }
  double stdv = 0.0;
  if (nf == 2) {
    stdv = std::fabs((fractions[0] - fractions[1]) / 2);
  } else if (nf > 2) {
    double mean = total_fraction / (double)nf;
    double sum = 0;
    for (int i = 0; i < nf; ++i) sum = sum + (fractions[i] - mean) * (fractions[i] - mean);
    stdv = std::sqrt(sum / (double)nf);
  }
  return (int64_t)((1 - stdv) * (double)kMaxNodeScore);
}
// NodeAffinity.Score without PreScore/NormalizeScore (nodeorder.go:314-330 calls Score only)
int64_t node_affinity_score(const Session &s, int t, int n) {
  int c = s.t_class[t];
  int64_t count = 0;
  for (int k = 0; k < s.c_npref[c]; ++k)
    if (mask_subset(&s.c_pref[((size_t)c * VC_MAX_TERMS + k) * s.Wl], s.labels, s.Wl, s.N, n))
      count += s.c_prefw[(size_t)c * VC_MAX_TERMS + k];
  return count;
}
// nodeorder NodeOrderFn, plugins/nodeorder/nodeorder.go:314-330
double nodeorder_score(const Session &s, int t, int n) {
  double node_score = 0.0;
  if (s.conf.w_least != 0) node_score += (double)least_allocated(s, t, n) * (double)s.conf.w_least;
  if (s.conf.w_most != 0) node_score += (double)most_allocated(s, t, n) * (double)s.conf.w_most;
  if (s.conf.w_balanced != 0) node_score += (double)balanced_allocation(s, t, n) * (double)s.conf.w_balanced;
  if (s.conf.w_node_affinity != 0) node_score += (double)node_affinity_score(s, t, n) * (double)s.conf.w_node_affinity;
  return node_score;
}
// TaintToleration.Score: number of PreferNoSchedule taints the pod does not tolerate
int64_t taint_soft_count(const Session &s, int t, int n) {
  int c = s.t_class[t];
  int64_t cnt = 0;
  for (int w = 0; w < s.Wt; ++w)
    cnt += __builtin_popcountll(s.tsoft[(size_t)w * s.N + n] & ~s.c_tols[(size_t)c * s.Wt + w]);
  return cnt;
}

// ssn.NodeOrderMapFn, framework/session_plugins.go:974-999 (no plugin on this path registers
// a NodeMapFn, so mapScores stays empty).  Returns false when a NodeOrderFn returned an error
// (tdm.go:181-184): util.PrioritizeNodes then records no order score for the node.
bool node_order(const Session &s, int t, int n, double *out) {
  double priority_score = 0.0;
  for (int i = 0; i < s.conf.n_plugins; ++i) {
    const vc_plugin_option &p = s.conf.plugins[i];
    if (!(p.enabled & VC_EN_NODE_ORDER)) continue;
    switch (p.plugin) {
      case VC_PLUGIN_BINPACK:
        if (s.conf.binpack_weight != 0) priority_score += binpack_score(s, t, n);  // binpack.go:192-196
        break;
      case VC_PLUGIN_NODEORDER: priority_score += nodeorder_score(s, t, n); break;
      case VC_PLUGIN_TDM: {  // tdm.go:174-195
        int z = s.zone[n];
        double sc = 0.0;
        if (z >= 0) {
          if (!s.zone_active[z]) return false;
          if (s.c_flags[s.t_class[t]] & VC_CLASS_REVOCABLE) sc = (double)kMaxNodeScore;
        }
        priority_score += sc;
        break;
      }
      default: break;
    }
  }
  *out = priority_score;
  return true;
}
bool batch_enabled(const Session &s) {  // does any BatchNodeOrderFn produce entries?
  for (int i = 0; i < s.conf.n_plugins; ++i) {
    const vc_plugin_option &p = s.conf.plugins[i];
    if ((p.enabled & VC_EN_NODE_ORDER) && (p.plugin == VC_PLUGIN_NODEORDER || p.plugin == VC_PLUGIN_PREDICATES))
      return true;
  }
  return s.nta_plugin;
}
bool taint_batch_enabled(const Session &s) {
  if (s.conf.w_taint_toleration == 0) return false;
  for (int i = 0; i < s.conf.n_plugins; ++i)
    if ((s.conf.plugins[i].enabled & VC_EN_NODE_ORDER) && s.conf.plugins[i].plugin == VC_PLUGIN_NODEORDER) return true;
  return false;
}

// util.PrioritizeNodes (util/scheduler_helper.go:76-138) + util.SelectBestNodeAndScore (:191-206)
// with the canonical tie-break.  `scores_out` (optional) receives the per-node totals.
int prioritize_and_select(Session &s, int t, const std::vector<int> &nodes, double *best_score,
                          std::vector<double> *scores_out) {
  const int m = (int)nodes.size();
  std::vector<double> order(m, 0.0);
  std::vector<uint8_t> has_order(m, 0);
  std::vector<int64_t> tcount(m, 0);
  const bool taint = taint_batch_enabled(s);
  s.pool->parallel_for(m, [&](int b, int e) {
    for (int i = b; i < e; ++i) {
      double o;
      if (node_order(s, t, nodes[i], &o)) { order[i] = o; has_order[i] = 1; }
      if (taint) tcount[i] = taint_soft_count(s, t, nodes[i]);
    }
  });
  // nodeorder BatchNodeOrderFn (nodeorder.go:332-384): TaintToleration through
  // nodescore.CalculatePluginScore (plugins/util/nodescore/score_helper.go:42-109) with
  // DefaultNormalizeScore(MaxNodeScore, reverse=true).
  int64_t max_count = 0;
  if (taint)
    for (int i = 0; i < m; ++i) max_count = std::max(max_count, tcount[i]);
  const bool batch = batch_enabled(s);
  const bool topo = topo_task(s, t);
  std::vector<double> topo_sc;
  std::vector<uint8_t> topo_has;
  if (topo) topo_node_scores(s, t, nodes, topo_sc, topo_has);
  int best = -1;
  double best_sc = -std::numeric_limits<double>::infinity();
  if (scores_out) scores_out->assign(m, 0.0);
  for (int i = 0; i < m; ++i) {
    double score = 0.0;
    if (has_order[i]) score += order[i];
    if (batch) {
      double b = 0.0;  // priorityScore[nodeName] += score, session_plugins.go:946-967
      if (taint) {
        int64_t sc = max_count == 0 ? kMaxNodeScore : kMaxNodeScore - (kMaxNodeScore * tcount[i] / max_count);
        sc *= (int64_t)s.conf.w_taint_toleration;
        double node_sc = 0.0;
        node_sc += (double)sc;  // nodeorder.go:369-381
        b += node_sc;
      }
      // network-topology-aware BatchNodeOrderFn :422-460 (two addends: plugin order is immaterial)
      if (topo) {
        if (topo_has[i]) b += (double)kMaxNodeScore * (double)s.conf.nta_weight * topo_sc[i];
      } else if (s.nta_on) {
        b += nta_node_score(s, t, nodes[i]);
      }
      score += b;
    }
    if (scores_out) (*scores_out)[i] = score;
    if (score > best_sc || (score == best_sc && best >= 0 && nodes[i] < nodes[best])) {
      best_sc = score;
      best = i;
    }
  }
  if (best < 0) return -1;
  *best_score = best_sc;
  return nodes[best];
}

// CalculateNumOfFeasibleNodesToFind, util/scheduler_helper.go:54-73
int32_t num_feasible_nodes_to_find(int32_t num_all, int32_t pct, int32_t min_nodes, int32_t min_pct) {
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

// ---------------------------------------------------------------------------------------
// Statement (framework/statement.go)
// ---------------------------------------------------------------------------------------
void stmt_allocate(Session &s, std::vector<Op> &ops, int t, int n, double score) {  // :242-302
  int j = s.t_job[t], r = s.t_role[t];
  s.t_status[t] = kAllocated;  // job.UpdateTaskStatus(task, Allocated)
  s.r_pending[r] -= 1;
  s.r_occ[r] += 1;
  s.j_ready[j] += 1;
  s.t_node[t] = n;
  for (int d = 0; d < s.R; ++d) {  // node.AddTask default branch, api/node_info.go:467-471
    at(s.idle, d, s.N, n) -= at(s.req, d, s.T, t);
    at(s.used, d, s.N, n) += at(s.req, d, s.T, t);
  }
  on_allocate_event(s, t, n);
  s.job_placed[j].push_back(n);  // task.NodeName = hostname
  ops.push_back({t, n, VC_OP_ALLOCATE, score});
}
void stmt_pipeline(Session &s, std::vector<Op> &ops, int t, int n, double score) {  // :146-200
  int j = s.t_job[t], r = s.t_role[t];
  s.t_status[t] = kPipelined;
  s.r_pending[r] -= 1;
  s.r_pip[r] += 1;
  s.j_waiting[j] += 1;
  s.t_node[t] = n;
  for (int d = 0; d < s.R; ++d) at(s.pip, d, s.N, n) += at(s.req, d, s.T, t);  // node_info.go:457-458
  on_allocate_event(s, t, n);
  s.job_placed[j].push_back(n);
  ops.push_back({t, n, VC_OP_PIPELINE, score});
}
void stmt_discard(Session &s, std::vector<Op> &ops) {  // :357-381
  for (int i = (int)ops.size() - 1; i >= 0; --i) {
    int t = ops[i].task, n = ops[i].node;
    int j = s.t_job[t], r = s.t_role[t];
    if (ops[i].kind == VC_OP_ALLOCATE) {  // unallocate :328-354
      s.t_status[t] = kPending;
      s.r_pending[r] += 1;
      s.r_occ[r] -= 1;
      s.j_ready[j] -= 1;
      for (int d = 0; d < s.R; ++d) {  // node.RemoveTask default branch, node_info.go:507-510
        at(s.idle, d, s.N, n) += at(s.req, d, s.T, t);
        at(s.used, d, s.N, n) -= at(s.req, d, s.T, t);
      }
    } else {  // UnPipeline :205-239
      s.t_status[t] = kPending;
      s.r_pending[r] += 1;
      s.r_pip[r] -= 1;
      s.j_waiting[j] -= 1;
      for (int d = 0; d < s.R; ++d) at(s.pip, d, s.N, n) -= at(s.req, d, s.T, t);
    }
    on_deallocate_event(s, t, n);
    s.job_placed[j].pop_back();  // task.NodeName = "" (ops are undone in reverse order)
    s.t_node[t] = -1;
  }
  ops.clear();
}
void stmt_commit(Session &s, std::vector<Op> &ops) {  // :384-412 -> allocate :309-325
  for (auto &op : ops)
    if (op.kind == VC_OP_ALLOCATE) s.t_status[op.task] = kBinding;  // still counted by ReadyTaskNum
}

// ---------------------------------------------------------------------------------------
// The action (actions/allocate/allocate.go)
// ---------------------------------------------------------------------------------------
// JobInfo.NeedContinueAllocating, api/job_info.go:918-966
bool need_continue_allocating(const Session &s, int j) {
  if (s.j_min[j] == s.j_ntasks[j]) return false;
  if (s.j_min[j] >= s.j_ntasks[j]) return false;  // default SubJob: MinAvailable = job.MinAvailable (:1236-1250)
  if (s.j_min[j] < s.j_taskmintotal[j]) {
    int32_t left = 0;
    for (int r = s.j_roleoff[j]; r < s.j_roleoff[j + 1]; ++r)
      if (!s.r_failed[r]) left += s.r_pending[r];
    return s.j_ready[j] + left >= s.j_min[j];
  }
  for (int r = s.j_roleoff[j]; r < s.j_roleoff[j + 1]; ++r) {
    if (!s.r_failed[r]) continue;
    int32_t mn = (s.r_flags[r] & VC_ROLE_IN_MIN_MAP) ? s.r_min[r] : 0;
    if (mn == 0) continue;
    if (s.r_occ[r] < mn) return false;
  }
  return true;
}

struct PredicateHelper {  // util/predicate_helper.go:38-41, one per allocateResourcesForTasks call
  int role_base = 0;
  std::vector<std::vector<uint8_t>> node_err;  // taskPredicateErrorCache[job/role][node]
  std::vector<uint8_t> exists;
};

// ph.PredicateNodes, util/predicate_helper.go:43-140
void predicate_nodes(Session &s, PredicateHelper &ph, int t, std::vector<int> &out) {
  out.clear();
  const int N = s.N;
  if (N == 0) return;
  int r = s.t_role[t];
  bool enable_cache = s.conf.enable_predicate_error_cache != 0 && !(s.r_flags[r] & VC_ROLE_EMPTY_NAME);
  int lr = r - ph.role_base;
  bool failed_before = ph.exists[lr] != 0;
  if (ph.node_err[lr].empty()) ph.node_err[lr].assign(N, 0);
  std::vector<uint8_t> &cache = ph.node_err[lr];
  int32_t to_find = num_feasible_nodes_to_find(N, s.conf.percentage_nodes_to_find, s.conf.min_nodes_to_find,
                                               s.conf.min_percentage_nodes_to_find);
  s.sweeps++;
  if (to_find >= N) {
    std::vector<uint8_t> ok(N, 0);
    std::atomic<int> any_err{0};
    s.pool->parallel_for(N, [&](int b, int e) {
      bool err = false;
      for (int n = b; n < e; ++n) {
        if (enable_cache && failed_before && cache[n]) continue;
        if (!predicate(s, t, n)) { cache[n] = 1; err = true; continue; }
        ok[n] = 1;
      }
      if (err) any_err.store(1, std::memory_order_relaxed);
    });
    if (any_err.load()) ph.exists[lr] = 1;
    for (int n = 0; n < N; ++n)
      if (ok[n]) out.push_back(n);
    // processedNodes == allNodes -> lastProcessedNodeIndex unchanged modulo N
    return;
  }
  // Sampling mode: the deterministic (single-worker) reading of the early-stop loop.
  int start = (int)s.last_processed_node_index;
  int processed = 0;
  for (int i = 0; i < N && (int)out.size() < to_find; ++i) {
    int n = (start + i) % N;
    processed++;
    if (enable_cache && failed_before && cache[n]) continue;
    if (!predicate(s, t, n)) { cache[n] = 1; ph.exists[lr] = 1; continue; }
    out.push_back(n);
  }
  s.last_processed_node_index = (start + processed) % N;
}

// alloc.prioritizeNodes, allocate.go:709-778 (sharding mode none)
int prioritize_nodes(Session &s, int t, const std::vector<int> &predicate_nodes_v, double *score_out) {
  std::vector<int> idle_c, future_c;
  for (int n : predicate_nodes_v) {
    if (fits_idle(s, t, n)) idle_c.push_back(n);
    else if (fits_future_idle(s, t, n)) future_c.push_back(n);
  }
  int best = -1;
  double highest = 0;
  const std::vector<int> *grads[2] = {&idle_c, &future_c};
  for (int g = 0; g < 2; ++g) {
    const std::vector<int> &nodes = *grads[g];
    if (nodes.empty()) continue;
    if (nodes.size() == 1) {
      best = nodes[0];
    } else {
      double sc;
      best = prioritize_and_select(s, t, nodes, &sc, nullptr);
      if (best >= 0) highest = sc;
    }
    if (best >= 0) break;
  }
  *score_out = highest;
  return best;
}

// alloc.allocateResourcesForTasks, allocate.go:558-694. Returns true when a statement is returned.
bool allocate_resources_for_tasks(Session &s, int j, GoHeap &tasks, std::vector<Op> &ops) {
  int q = s.j_queue[j];
  ops.clear();
  if (s.N == 0) return false;
  PredicateHelper ph;
  ph.role_base = s.j_roleoff[j];
  int nroles = s.j_roleoff[j + 1] - s.j_roleoff[j];
  ph.node_err.resize(nroles);
  ph.exists.assign(nroles, 0);
  std::vector<int> feasible;
  int allocated_hn = s.job_alloc_hn[j];  // allocatedHyperNode := subJob.AllocatedHyperNode, allocate.go:572
  while (!tasks.empty()) {
    int t = tasks.pop();
    if (!allocatable(s, q, t)) continue;
    int r = s.t_role[t];
    // job.TaskHasFitErrors, api/job_info.go:894-902
    if (!(s.r_flags[r] & VC_ROLE_EMPTY_NAME) && s.r_failed[r]) {
      s.fit_errors.push_back(t);
      continue;
    }
    // ssn.PrePredicateFn: nil for pods in scope (predicates PreFilter skip/ok; proportion state clone)
    // Pod.Status.NominatedNodeName, allocate.go:624-634: the nominated node first, alone, when InitResreq <= its FutureIdle
    feasible.clear();
    const int nom = (!s.t_nominated.empty() && t < (int)s.t_nominated.size()) ? s.t_nominated[t] : -1;
    if (nom >= 0 && fits_future_idle(s, t, nom)) {
      // ph.PredicateNodes(task, []*api.NodeInfo{nominatedNodeInfo}, ...), util/predicate_helper.go:43-140 on a one-node list
      const int lr = r - ph.role_base;
      const bool enable_cache = s.conf.enable_predicate_error_cache != 0 && !(s.r_flags[r] & VC_ROLE_EMPTY_NAME);
      if (ph.node_err[lr].empty()) ph.node_err[lr].assign(s.N, 0);
      s.sweeps++;
      if (!(enable_cache && ph.exists[lr] && ph.node_err[lr][nom])) {
        if (predicate(s, t, nom)) feasible.push_back(nom);
        else { ph.node_err[lr][nom] = 1; ph.exists[lr] = 1; }
      }
      s.last_processed_node_index = 0;  // (startIndex + processedNodes) % allNodes with allNodes = 1 (:135-136)
    }
    if (feasible.empty()) predicate_nodes(s, ph, t, feasible);
    if (feasible.empty()) {
      s.fit_errors.push_back(t);
      s.r_failed[r] = 1;
      if (need_continue_allocating(s, j)) continue;
      break;
    }
    double score = 0;
    s.task_alloc_hn = s.job_soft[j] ? allocated_hn : -1;  // task.JobAllocatedHyperNode, allocate.go:658-660
    int best = prioritize_nodes(s, t, feasible, &score);
    if (best < 0) continue;
    // alloc.allocateResourcesForTask, allocate.go:780-814
    if (fits_idle(s, t, best)) stmt_allocate(s, ops, t, best, score);
    else if (fits_future_idle(s, t, best)) stmt_pipeline(s, ops, t, best, score);
    if (s.job_soft[j]) allocated_hn = new_allocated_hypernode(s, best, allocated_hn);  // :672-674
    if (job_ready(s, j)) break;  // ssn.SubJobReady == ssn.JobReady without a subjob policy (:369-372)
  }
  if (job_ready(s, j)) {
    if (s.job_soft[j]) s.job_alloc_hn[j] = allocated_hn;  // :681-686
    return true;
  }
  if (job_pipelined(s, j)) return true;
  stmt_discard(s, ops);
  return false;
}

// Action.Execute -> buildAllocateContext (:142-206) + allocateResources (:283-348)
int allocate_execute(Session &s) {
  for (int j = 0; j < s.J; ++j)
    if (s.j_flags[j] & VC_JOB_UNSUPPORTED) return VC_EUNSUPPORTED;
  std::vector<GoHeap> task_pq(s.J);
  for (int j = 0; j < s.J; ++j) task_pq[j].less = [&s](int l, int r) { return task_order_less(s, l, r); };
  for (int t = 0; t < s.T_alloc; ++t) task_pq[s.t_job[t]].push(t);  // organizeJobWorksheet :208-281
  GoHeap queues;
  queues.less = [&s](int l, int r) { return queue_order_less(s, l, r); };
  std::vector<GoHeap> jobs_by_queue(s.Q);
  std::vector<uint8_t> queue_seen(s.Q, 0);
  for (int q = 0; q < s.Q; ++q) jobs_by_queue[q].less = [&s](int l, int r) { return job_order_less(s, l, r); };
  for (int j = 0; j < s.J; ++j) {
    if (s.j_flags[j] & VC_JOB_PENDING_PHASE) {  // allocate.go:154-164
      if (s.conf.enqueue_action_enabled) continue;
      s.j_flags[j] &= ~VC_JOB_PENDING_PHASE;  // job.PodGroup.Status.Phase = PodGroupInqueue: later actions see it
    }
    if (!job_valid(s, j)) continue;
    int q = s.j_queue[j];
    if (q < 0) continue;
    if (task_pq[j].empty()) continue;  // worksheet.Empty()
    if (!queue_seen[q]) {
      queue_seen[q] = 1;
      queues.push(q);
    }
    jobs_by_queue[q].push(j);
  }
  std::vector<Op> ops;
  while (!queues.empty()) {
    int q = queues.pop();
    if (overused(s, q)) continue;
    GoHeap &jobs = jobs_by_queue[q];
    if (jobs.empty()) continue;
    int j = jobs.pop();
    bool stmt = allocate_resources_for_tasks(s, j, task_pq[j], ops);
    vc_visit v;
    v.job = j;
    v.first_op = (int32_t)s.decisions.size();
    v.n_ops = 0;
    v.outcome = VC_VISIT_DISCARD;
    if (stmt) {
      bool ready = job_ready(s, j);
      v.outcome = ready ? VC_VISIT_COMMIT : VC_VISIT_KEEP;
      v.n_ops = (int32_t)ops.size();
      for (auto &op : ops) {
        vc_decision dcs;
        dcs.task = op.task;
        dcs.node = op.node;
        dcs.kind = op.kind;
        dcs.visit = (int32_t)s.visits.size();
        dcs.score = op.score;
        s.decisions.push_back(dcs);
      }
      if (ready) {
        stmt_commit(s, ops);
        if (task_pq[j].size() > 0) jobs.push(j);
      }
    }
    s.visits.push_back(v);
    queues.push(q);
  }
  return VC_OK;
}

// ---------------------------------------------------------------------------------------
// The backfill action (actions/backfill/backfill.go)
// ---------------------------------------------------------------------------------------
// ssn.PredicateForAllocateAction (framework/session.go:657-674) alone: backfill passes it to PredicateNodes without
// allocate's resource-fit wrapper (backfill.go:66,83)
bool plugin_predicates(const Session &s, int t, int n) {
  for (int i = 0; i < s.conf.n_plugins; ++i) {
    const vc_plugin_option &p = s.conf.plugins[i];
    if (!(p.enabled & VC_EN_PREDICATE)) continue;
    if (p.plugin == VC_PLUGIN_PREDICATES && !predicates_plugin_ok(s, t, n)) return false;
    if (p.plugin == VC_PLUGIN_TDM && !tdm_predicate_ok(s, t, n)) return false;
  }
  return true;
}

// pickUpPendingTasks, backfill.go:118-199: every PQ is filled first and drained afterwards, so the three order
// functions are evaluated on the state the action starts from
std::vector<int> backfill_pick_up_pending_tasks(Session &s, std::vector<int> *job_order) {
  std::vector<GoHeap> task_pq(s.J);
  for (int j = 0; j < s.J; ++j) task_pq[j].less = [&s](int l, int r) { return task_order_less(s, l, r); };
  for (int t = s.T_alloc; t < s.T; ++t)
    if (s.t_status[t] == kPending) task_pq[s.t_job[t]].push(t);
  GoHeap queues;
  queues.less = [&s](int l, int r) { return queue_order_less(s, l, r); };
  std::vector<GoHeap> jobs_by_queue(s.Q);
  std::vector<uint8_t> queue_seen(s.Q, 0);
  for (int q = 0; q < s.Q; ++q) jobs_by_queue[q].less = [&s](int l, int r) { return job_order_less(s, l, r); };
  for (int j = 0; j < s.J; ++j) {
    if (s.j_flags[j] & VC_JOB_PENDING_PHASE) continue;  // job.IsPending() :124-126 — on the phase allocate may have rewritten
    if (!job_valid(s, j)) continue;
    int q = s.j_queue[j];
    if (q < 0) continue;
    if (task_pq[j].empty()) continue;
    if (!queue_seen[q]) {
      queue_seen[q] = 1;
      queues.push(q);
    }
    jobs_by_queue[q].push(j);
  }
  std::vector<int> pending;
  while (!queues.empty()) {
    int q = queues.pop();
    while (!jobs_by_queue[q].empty()) {
      int j = jobs_by_queue[q].pop();
      if (job_order) job_order->push_back(j);
      while (!task_pq[j].empty()) pending.push_back(task_pq[j].pop());
    }
  }
  return pending;
}

// Action.Execute, backfill.go:58-116
int backfill_execute(Session &s) {
  s.decisions.clear(); s.visits.clear(); s.fit_errors.clear();
  if (s.T == s.T_alloc) return VC_OK;
  for (int j = 0; j < s.J; ++j)
    if (s.j_flags[j] & VC_JOB_UNSUPPORTED) return VC_EUNSUPPORTED;
  const int32_t to_find = num_feasible_nodes_to_find(s.N, s.conf.percentage_nodes_to_find, s.conf.min_nodes_to_find,
                                                     s.conf.min_percentage_nodes_to_find);
  std::vector<int> pending = backfill_pick_up_pending_tasks(s, nullptr);
  std::vector<int> feasible;
  int cur_job = -1;
  for (int t : pending) {
    const int j = s.t_job[t], r = s.t_role[t];
    if (j != cur_job) {  // one visit record per job, in pick order
      vc_visit v;
      // ssn.JobReady is invariant under backfill itself (a placed BestEffort task moves from PendingBestEffortTaskNum
      // to ReadyTaskNum, role occupancy counts it either way): COMMIT = the job's placed tasks are dispatched (:785-793)
      v.job = j; v.first_op = (int32_t)s.decisions.size(); v.n_ops = 0;
      v.outcome = job_ready(s, j) ? VC_VISIT_COMMIT : VC_VISIT_KEEP;
      s.visits.push_back(v);
      cur_job = j;
    }
    // ssn.PrePredicateFn: nil for pods in scope.  ph := util.NewPredicateHelper() per task (:71): the error cache is
    // always empty, every node is evaluated
    feasible.clear();
    s.sweeps++;
    if (to_find < s.N) {
      // feasible-node sampling (util/predicate_helper.go:43-140, single-worker reading): scan from
      // lastProcessedNodeIndex, stop after to_find feasible nodes
      const int start = (int)s.last_processed_node_index;
      int processed = 0;
      for (int i = 0; i < s.N && (int)feasible.size() < to_find; ++i) {
        const int n = (start + i) % s.N;
        processed++;
        if (plugin_predicates(s, t, n)) feasible.push_back(n);
      }
      s.last_processed_node_index = (start + processed) % s.N;
    } else {
      std::vector<uint8_t> ok(s.N, 0);
      s.pool->parallel_for(s.N, [&](int b, int e) {
        for (int n = b; n < e; ++n) ok[n] = plugin_predicates(s, t, n) ? 1 : 0;
      });
      for (int n = 0; n < s.N; ++n)
        if (ok[n]) feasible.push_back(n);
    }
    if (feasible.empty()) {  // job.NodesFitErrors[task.UID] = fitErrors :84-87
      s.fit_errors.push_back(t - s.T_alloc);
      continue;
    }
    int node = feasible[0];
    double score = 0.0;
    if (feasible.size() > 1) {  // :90-103 (sharding mode none: one candidate group; ssn.BestNodeFn unregistered)
      s.task_alloc_hn = -1;
      double sc = 0.0;
      int best = prioritize_and_select(s, t, feasible, &sc, nullptr);
      if (best >= 0) { node = best; score = sc; }
    }
    // ssn.Allocate, framework/session.go:746-796
    s.t_status[t] = kAllocated;  // job.UpdateTaskStatus(task, Allocated): leaves PendingBestEffortTaskNum, joins ReadyTaskNum
    s.r_pending[r] -= 1;
    s.j_pbe[j] -= 1;
    s.j_ready[j] += 1;
    s.t_node[t] = node;
    for (int d = 0; d < s.R; ++d) {  // node.AddTask default branch, api/node_info.go:467-471 (Idle may go negative)
      at(s.idle, d, s.N, node) -= at(s.req, d, s.T, t);
      at(s.used, d, s.N, node) += at(s.req, d, s.T, t);
    }
    on_allocate_event(s, t, node);
    s.job_placed[j].push_back(node);
    vc_decision dcs;
    dcs.task = t - s.T_alloc; dcs.node = node; dcs.kind = VC_OP_ALLOCATE;
    dcs.visit = (int32_t)s.visits.size() - 1; dcs.score = score;
    s.decisions.push_back(dcs);
    s.visits.back().n_ops += 1;
    if (job_ready(s, j)) {  // :785-793: every Allocated task of the job is dispatched
      for (int u = 0; u < s.T; ++u)
        if (s.t_job[u] == j && s.t_status[u] == kAllocated) s.t_status[u] = kBinding;
    }
  }
  return VC_OK;
}

// ---------------------------------------------------------------------------------------
// The preempt and reclaim actions (actions/preempt/preempt.go, actions/reclaim/reclaim.go)
//
// Canonical determinism on top of the allocate contract: node.Tasks (a Go map) is walked in ascending
// running-task index; util.SortNodes' buckets of equal score keep NodeList order; reclaim's predicateNodes keep
// NodeList order (the reference's order there is whatever its 16 workers produced).
// ---------------------------------------------------------------------------------------
struct EOp { int kind; int task; int node; };  // VC_OP_EVICT / VC_OP_PIPELINE

// ssn.JobStarving, framework/session_plugins.go:482-506
bool job_starving(const Session &s, int j) {
  bool has_found = false;
  int i = 0;
  while (i < s.conf.n_plugins) {
    const int tier = s.conf.plugins[i].tier;
    for (; i < s.conf.n_plugins && s.conf.plugins[i].tier == tier; ++i) {
      const vc_plugin_option &p = s.conf.plugins[i];
      if (!(p.enabled & VC_EN_JOB_STARVING)) continue;
      bool res;
      if (p.plugin == VC_PLUGIN_GANG) res = s.j_waiting[j] + s.j_ready[j] < s.j_min[j];  // IsStarving, job_info.go:1176-1178
      else if (p.plugin == VC_PLUGIN_PRIORITY) res = s.j_ready[j] + s.j_waiting[j] < s.j_ntasks[j];  // priority.go:151-154
      else continue;
      has_found = true;
      if (!res) return false;
    }
    if (has_found) return true;
  }
  return false;
}
inline bool rt_flag(const Session &s, int t, uint32_t f) { return (s.rt_flags[t - s.T_run0] & f) != 0; }
inline bool preemptable_status(const Session &s, int t) { return s.t_status[t] == kRunning || s.t_status[t] == kBound; }

// Statement.Evict, framework/statement.go:72-99
void stmt_evict(Session &s, std::vector<EOp> &ops, int t) {
  const int j = s.t_job[t], n = s.t_node[t];
  if (j >= 0) {  // job.UpdateTaskStatus(reclaimee, Releasing): leaves ReadyTaskNum / the allocated roles
    s.j_ready[j] -= 1;
    s.r_occ[s.t_role[t]] -= 1;
  }
  s.t_status[t] = kReleasing;
  // node.UpdateTask = RemoveTask + AddTask(Releasing): Idle and Used end where they were, Releasing grows (node_info.go:435-517)
  for (int d = 0; d < s.R; ++d) at(s.rel, d, s.N, n) += at(s.req, d, s.T, t);
  if (j >= 0) on_deallocate_event(s, t, n);
  ops.push_back({VC_OP_EVICT, t, n});
}
// Statement.unevict, framework/statement.go:119-143
void stmt_unevict(Session &s, int t, int8_t status_before) {
  const int j = s.t_job[t], n = s.t_node[t];
  if (j >= 0) {
    s.j_ready[j] += 1;
    s.r_occ[s.t_role[t]] += 1;
  }
  s.t_status[t] = status_before;
  for (int d = 0; d < s.R; ++d) at(s.rel, d, s.N, n) -= at(s.req, d, s.T, t);
  if (j >= 0) on_allocate_event(s, t, n);
}
void estmt_pipeline(Session &s, std::vector<EOp> &ops, int t, int n) {  // Statement.Pipeline :146-200
  std::vector<Op> tmp;
  stmt_pipeline(s, tmp, t, n, 0.0);
  ops.push_back({VC_OP_PIPELINE, t, n});
}
void estmt_discard(Session &s, std::vector<EOp> &ops) {  // Statement.Discard :357-381, reverse order
  for (int i = (int)ops.size() - 1; i >= 0; --i) {
    if (ops[i].kind == VC_OP_EVICT) {
      stmt_unevict(s, ops[i].task, rt_flag(s, ops[i].task, VC_RT_BOUND) ? kBound : kRunning);
    } else {
      std::vector<Op> tmp{{ops[i].task, ops[i].node, VC_OP_PIPELINE, 0.0}};
      stmt_discard(s, tmp);
    }
  }
  ops.clear();
}

// ---- plugin victim functions (candidates in the order given) ----
std::vector<int> gang_victims(const Session &s, const std::vector<int> &cands) {  // gang.go:97-129
  std::vector<int> out;
  std::vector<std::pair<int, int>> occ;  // jobOccupiedMap
  for (int t : cands) {
    const int j = s.t_job[t];
    if (j < 0) continue;
    int *o = nullptr;
    for (auto &e : occ) if (e.first == j) o = &e.second;
    if (!o) { occ.push_back({j, s.j_ready[j]}); o = &occ.back().second; }
    if (*o > s.j_min[j]) { *o -= 1; out.push_back(t); }
  }
  return out;
}
std::vector<int> priority_victims(const Session &s, int preemptor, const std::vector<int> &cands) {  // priority.go:110-148
  std::vector<int> out;
  const int pj = s.t_job[preemptor];
  for (int t : cands) {
    const int j = s.t_job[t];
    if (j < 0) continue;
    if (j != pj) { if (s.j_prio[j] < s.j_prio[pj]) out.push_back(t); }
    else if (s.t_prio[t] < s.t_prio[preemptor]) out.push_back(t);
  }
  return out;
}
double drf_share_of(const Session &s, const std::vector<double> &alloc) {  // drf.calculateShare :566-578
  double res = 0;
  for (int d = 0; d < s.R; ++d) {
    if (d >= 2 && !(s.total.has & (1u << d))) continue;
    if (!(s.total.v[d] >= kMinResource)) continue;
    const double sh = share_of(alloc[d], s.total.v[d]);
    if (sh > res) res = sh;
  }
  return res;
}
std::vector<int> drf_victims(const Session &s, int preemptor, const std::vector<int> &cands) {  // drf.go:222-261
  std::vector<int> out;
  const int pj = s.t_job[preemptor];
  std::vector<double> lalloc(s.R);
  for (int d = 0; d < s.R; ++d) lalloc[d] = at(s.j_alloc, d, s.J, pj) + at(s.req, d, s.T, preemptor);
  const double ls = drf_share_of(s, lalloc);
  std::vector<std::pair<int, std::vector<double>>> allocations;
  for (int t : cands) {
    const int j = s.t_job[t];
    if (j < 0) continue;
    std::vector<double> *ra = nullptr;
    for (auto &e : allocations) if (e.first == j) ra = &e.second;
    if (!ra) {
      allocations.push_back({j, std::vector<double>(s.R)});
      ra = &allocations.back().second;
      for (int d = 0; d < s.R; ++d) (*ra)[d] = at(s.j_alloc, d, s.J, j);
    }
    for (int d = 0; d < s.R; ++d) (*ra)[d] -= at(s.req, d, s.T, t);  // allocations[job].Sub(preemptee.Resreq): mutates the entry
    const double rs = drf_share_of(s, *ra);
    if (ls < rs || std::fabs(ls - rs) <= 0.000001) out.push_back(t);  // shareDelta
  }
  return out;
}
std::vector<int> proportion_victims(const Session &s, const std::vector<int> &cands) {  // proportion.go:286-317
  std::vector<int> out;
  std::vector<std::pair<int, Res>> allocations;
  for (int t : cands) {
    const int j = s.t_job[t];
    if (j < 0) continue;
    const int q = s.j_queue[j];
    if (q < 0 || !s.qattr[q].exists) continue;
    Res *al = nullptr;
    for (auto &e : allocations) if (e.first == q) al = &e.second;
    if (!al) { allocations.push_back({q, s.qattr[q].allocated}); al = &allocations.back().second; }
    if (!res_less_equal_zero(*al, s.qattr[q].deserved, s.R)) {
      const Res rq = task_res(s, t);  // allocated.Sub(reclaimee.Resreq)
      al->v[0] -= rq.v[0]; al->v[1] -= rq.v[1];
      if (!al->nilmap)
        for (int d = 2; d < s.R; ++d)
          if (rq.has & (1u << d)) { al->has |= 1u << d; al->v[d] -= rq.v[d]; }
      out.push_back(t);
    }
  }
  return out;
}
std::vector<int> conformance_victims(const Session &s, const std::vector<int> &cands) {  // conformance.go:46-63
  std::vector<int> out;
  for (int t : cands)
    if (!rt_flag(s, t, VC_RT_CRITICAL)) out.push_back(t);
  return out;
}
// ssn.Preemptable / ssn.Reclaimable, framework/session_plugins.go:211-307: per tier the plugins' candidate lists are
// intersected (a nil list re-initialises from the next plugin; an empty answer voids the tier)
std::vector<int> tier_victims(const Session &s, int preemptor, const std::vector<int> &cands, bool reclaim) {
  std::vector<int> victims;
  bool nil = true;
  int i = 0;
  while (i < s.conf.n_plugins) {
    const int tier = s.conf.plugins[i].tier;
    int k = i;
    for (; k < s.conf.n_plugins && s.conf.plugins[k].tier == tier; ++k) {
      const vc_plugin_option &p = s.conf.plugins[k];
      if (!(p.enabled & (reclaim ? VC_EN_RECLAIMABLE : VC_EN_PREEMPTABLE))) continue;
      std::vector<int> c;
      if (p.plugin == VC_PLUGIN_GANG) c = gang_victims(s, cands);
      else if (p.plugin == VC_PLUGIN_CONFORMANCE) c = conformance_victims(s, cands);
      else if (p.plugin == VC_PLUGIN_PRIORITY && !reclaim) c = priority_victims(s, preemptor, cands);
      else if (p.plugin == VC_PLUGIN_DRF && !reclaim) c = drf_victims(s, preemptor, cands);
      else if (p.plugin == VC_PLUGIN_PROPORTION && reclaim) c = proportion_victims(s, cands);
      else continue;  // no function registered under this name
      if (c.empty()) { victims.clear(); nil = true; break; }
      if (nil) { victims = c; nil = false; }
      else {
        std::vector<int> inter;
        for (int v : victims)
          for (int x : c)
            if (v == x) inter.push_back(v);
        victims = inter;
        nil = inter.empty();  // `var intersection []*TaskInfo` stays nil without an append
      }
    }
    while (i < s.conf.n_plugins && s.conf.plugins[i].tier == tier) ++i;
    if (!nil) return victims;
  }
  return victims;
}
// util.ValidateVictims, util/scheduler_helper.go:313-329
bool validate_victims(const Session &s, int preemptor, int n, const std::vector<int> &victims) {
  for (int d = 0; d < s.R; ++d) {
    double fi = future_idle(s, d, n);
    for (int v : victims) fi += at(s.req, d, s.T, v);
    if (d >= 2 && !(s.req_has[preemptor] & (1u << d))) continue;
    if (!le_eps(at(s.req, d, s.T, preemptor), fi)) return false;
  }
  return true;
}
// the order ssn.BuildVictimsPriorityQueue pops in (framework/session_plugins.go:1092-1135), no VictimQueueOrderFn registered
bool victim_less(const Session &s, int l, int r) {
  const int lj = s.t_job[l], rj = s.t_job[r];
  if (lj == rj) return !task_order_less(s, l, r);
  if (lj < 0 || rj < 0) {
    if (lj < 0 && rj < 0) return !task_order_less(s, l, r);
    return lj < 0;
  }
  if (s.j_queue[lj] != s.j_queue[rj]) return !queue_order_less(s, s.j_queue[lj], s.j_queue[rj]);  // ssn.VictimQueueOrderFn :735-749
  return !job_order_less(s, lj, rj);
}
// plugin predicates as ssn.PredicateForPreemptAction reads them (framework/session.go:679-697): only
// UnschedulableAndUnresolvable / error statuses reject a node; the pod-count cap is Unschedulable and passes
bool preempt_predicate(const Session &s, int t, int n) {
  for (int i = 0; i < s.conf.n_plugins; ++i) {
    const vc_plugin_option &p = s.conf.plugins[i];
    if (!(p.enabled & VC_EN_PREDICATE)) continue;
    if (p.plugin == VC_PLUGIN_PREDICATES) {
      Session &ms = const_cast<Session &>(s);
      const int32_t pc = ms.pod_count[n];
      ms.pod_count[n] = INT32_MIN / 2;  // the cap never binds here
      const bool ok = predicates_plugin_ok(s, t, n);
      ms.pod_count[n] = pc;
      if (!ok) return false;
    }
    if (p.plugin == VC_PLUGIN_TDM && !tdm_predicate_ok(s, t, n)) return false;
  }
  return true;
}
bool preempt_supported(const Session &s) {
  if (s.T_run0 >= 0 && s.T_run0 != s.T_alloc) return false;  // BestEffort pending tasks in the session
  for (int j = 0; j < s.J; ++j)
    if ((s.j_flags[j] & VC_JOB_UNSUPPORTED) || s.job_soft[j]) return false;
  if (s.has_plugin[VC_PLUGIN_TDM] || s.has_plugin[VC_PLUGIN_NETWORK_TOPOLOGY_AWARE]) return false;
  return true;
}
bool task_fits_future_idle(const Session &s, int t, int n) { return fits_future_idle(s, t, n); }

// pmpt.preempt -> normalPreempt, preempt.go:285-434
bool preempt_one(Session &s, std::vector<EOp> &stmt, int preemptor, int phase_job /* -1: inter-job phase */) {
  if (s.t_flags[preemptor] & VC_TASK_PREEMPT_NEVER) return false;  // taskEligibleToPreempt :436-441
  const int pj = s.t_job[preemptor], q = s.j_queue[pj];
  std::vector<int> nodes;
  for (int n = 0; n < s.N; ++n)
    if (preempt_predicate(s, preemptor, n)) nodes.push_back(n);
  if (nodes.empty()) return false;
  std::vector<double> scores;
  double bs;
  s.task_alloc_hn = -1;
  prioritize_and_select(s, preemptor, nodes, &bs, &scores);
  std::vector<int> order(nodes.size());
  for (size_t i = 0; i < order.size(); ++i) order[i] = (int)i;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return scores[a] > scores[b]; });  // util.SortNodes
  for (int oi : order) {
    const int n = nodes[oi];
    std::vector<int> preemptees;
    for (int t : s.node_tasks[n]) {
      if (!preemptable_status(s, t)) continue;
      if (!rt_flag(s, t, VC_RT_PREEMPTABLE)) continue;
      const int j = s.t_job[t];
      if (phase_job < 0) {
        if (j < 0) continue;
        if (!(s.j_queue[j] == q && j != pj)) continue;
      } else if (j != pj) {
        continue;
      }
      preemptees.push_back(t);
    }
    std::vector<int> victims = tier_victims(s, preemptor, preemptees, false);
    if (!validate_victims(s, preemptor, n, victims)) continue;
    std::vector<EOp> node_stmt;
    GoHeap vq;
    vq.less = [&s](int l, int r) { return victim_less(s, l, r); };
    for (int v : victims) vq.push(v);
    while (!vq.empty()) {
      if (allocatable(s, q, preemptor) && task_fits_future_idle(s, preemptor, n)) break;
      stmt_evict(s, node_stmt, vq.pop());
    }
    if (allocatable(s, q, preemptor) && task_fits_future_idle(s, preemptor, n)) {
      estmt_pipeline(s, node_stmt, preemptor, n);
      stmt.insert(stmt.end(), node_stmt.begin(), node_stmt.end());  // stmt.Merge(nodeStmt)
      return true;
    }
    estmt_discard(s, node_stmt);
  }
  return false;
}
void emit_statement(Session &s, int job, const std::vector<EOp> &ops, bool commit) {
  vc_visit v;
  v.job = job; v.first_op = (int32_t)s.decisions.size();
  v.outcome = commit ? VC_VISIT_COMMIT : VC_VISIT_DISCARD;
  v.n_ops = commit ? (int32_t)ops.size() : 0;
  if (commit)
    for (const EOp &op : ops) {
      vc_decision d;
      d.task = op.kind == VC_OP_EVICT ? op.task - s.T_run0 : op.task;
      d.node = op.node; d.kind = op.kind; d.visit = (int32_t)s.visits.size(); d.score = 0.0;
      s.decisions.push_back(d);
    }
  s.visits.push_back(v);
}
// Action.Execute, preempt.go:101-283
void ensure_running_table(Session &s) {  // a session without vc_running_tasks: no task occupies a node
  if (s.T_run0 >= 0) return;
  s.T_run0 = s.T;
  s.node_tasks.assign(s.N, {});
  s.t_flags.assign(s.T_alloc, 0u);
}
int preempt_execute(Session &s) {
  s.decisions.clear(); s.visits.clear(); s.fit_errors.clear();
  ensure_running_table(s);
  if (!preempt_supported(s)) return VC_EUNSUPPORTED;
  std::vector<GoHeap> preemptors(s.Q), ptasks(s.J);
  std::vector<std::vector<int>> under_request(s.Q);
  std::vector<uint8_t> has_q(s.Q, 0);
  for (int q = 0; q < s.Q; ++q) preemptors[q].less = [&s](int l, int r) { return job_order_less(s, l, r); };
  for (int j = 0; j < s.J; ++j) ptasks[j].less = [&s](int l, int r) { return task_order_less(s, l, r); };
  for (int j = 0; j < s.J; ++j) {
    if (s.j_flags[j] & VC_JOB_PENDING_PHASE) continue;
    if (!job_valid(s, j)) continue;
    const int q = s.j_queue[j];
    if (q < 0) continue;
    if (!job_starving(s, j)) continue;
    has_q[q] = 1;
    preemptors[q].push(j);
    under_request[q].push_back(j);
    for (int t = 0; t < s.T_alloc; ++t)
      if (s.t_job[t] == j && s.t_status[t] == kPending) ptasks[j].push(t);
  }
  GoHeap queues;
  queues.less = [&s](int l, int r) { return queue_order_less(s, l, r); };
  for (int q = 0; q < s.Q; ++q)
    if (has_q[q]) queues.push(q);
  while (!queues.empty()) {
    const int q = queues.pop();
    // preemption between jobs within the queue
    while (!preemptors[q].empty()) {
      const int pj = preemptors[q].pop();
      std::vector<EOp> stmt;
      bool assigned = false;
      for (;;) {
        if (!job_starving(s, pj)) break;
        if (ptasks[pj].empty()) break;
        const int preemptor = ptasks[pj].pop();
        assigned = preempt_one(s, stmt, preemptor, -1);
      }
      if (job_pipelined(s, pj)) {
        emit_statement(s, pj, stmt, true);
      } else {
        estmt_discard(s, stmt);
        emit_statement(s, pj, stmt, false);
        continue;
      }
      if (assigned) preemptors[q].push(pj);
    }
    // preemption between tasks within a job
    for (int j : under_request[q]) {
      GoHeap intra;
      intra.less = [&s](int l, int r) { return task_order_less(s, l, r); };
      for (int t = 0; t < s.T_alloc; ++t)
        if (s.t_job[t] == j && s.t_status[t] == kPending) intra.push(t);
      while (!intra.empty()) {
        const int preemptor = intra.pop();
        std::vector<EOp> stmt;
        const bool assigned = preempt_one(s, stmt, preemptor, j);
        if (!assigned) {
          estmt_discard(s, stmt);
          emit_statement(s, j, stmt, false);
          break;
        }
        emit_statement(s, j, stmt, true);
      }
    }
  }
  return VC_OK;
}

// ra.reclaimForTask, reclaim.go:170-258
void reclaim_for_task(Session &s, std::vector<EOp> &stmt, int task, int job) {
  const int jq = s.j_queue[job];
  for (int n = 0; n < s.N; ++n) {
    if (!preempt_predicate(s, task, n)) continue;
    std::vector<int> reclaimees;
    for (int t : s.node_tasks[n]) {
      if (s.t_status[t] != kRunning || !rt_flag(s, t, VC_RT_PREEMPTABLE)) continue;
      const int j = s.t_job[t];
      if (j < 0) continue;
      if (s.j_queue[j] == jq) continue;
      const int q = s.j_queue[j];
      if (q < 0 || (s.q_flags[q] & VC_QUEUE_NOT_RECLAIMABLE)) continue;
      reclaimees.push_back(t);
    }
    if (reclaimees.empty()) continue;
    std::vector<int> victims = tier_victims(s, task, reclaimees, true);
    if (!validate_victims(s, task, n, victims)) continue;
    GoHeap vq;
    vq.less = [&s](int l, int r) { return victim_less(s, l, r); };
    for (int v : victims) vq.push(v);
    std::vector<double> avail(s.R);
    for (int d = 0; d < s.R; ++d) avail[d] = future_idle(s, d, n);
    auto fits = [&]() {
      for (int d = 0; d < s.R; ++d) {
        if (d >= 2 && !(s.req_has[task] & (1u << d))) continue;
        if (!le_eps(at(s.req, d, s.T, task), avail[d])) return false;
      }
      return true;
    };
    std::vector<EOp> node_stmt;
    while (!vq.empty()) {
      if (fits()) break;
      const int v = vq.pop();
      stmt_evict(s, node_stmt, v);
      for (int d = 0; d < s.R; ++d) avail[d] += at(s.req, d, s.T, v);
    }
    if (fits()) {
      estmt_pipeline(s, node_stmt, task, n);
      stmt.insert(stmt.end(), node_stmt.begin(), node_stmt.end());
      return;
    }
    estmt_discard(s, node_stmt);
  }
}
// Action.Execute, reclaim.go:56-168
int reclaim_execute(Session &s) {
  s.decisions.clear(); s.visits.clear(); s.fit_errors.clear();
  ensure_running_table(s);
  if (!preempt_supported(s)) return VC_EUNSUPPORTED;
  GoHeap queues;
  queues.less = [&s](int l, int r) { return queue_order_less(s, l, r); };
  std::vector<uint8_t> q_seen(s.Q, 0);
  std::vector<GoHeap> preemptors(s.Q), ptasks(s.J);
  std::vector<uint8_t> has_pre(s.Q, 0), has_tasks(s.J, 0);
  for (int q = 0; q < s.Q; ++q) preemptors[q].less = [&s](int l, int r) { return job_order_less(s, l, r); };
  for (int j = 0; j < s.J; ++j) ptasks[j].less = [&s](int l, int r) { return task_order_less(s, l, r); };
  for (int j = 0; j < s.J; ++j) {
    if (s.j_flags[j] & VC_JOB_PENDING_PHASE) continue;
    if (!job_valid(s, j)) continue;
    const int q = s.j_queue[j];
    if (q < 0) continue;
    if (!q_seen[q]) { q_seen[q] = 1; queues.push(q); }
    if (job_starving(s, j)) {
      has_pre[q] = 1;
      preemptors[q].push(j);
      has_tasks[j] = 1;
      for (int t = 0; t < s.T_alloc; ++t)
        if (s.t_job[t] == j && s.t_status[t] == kPending) ptasks[j].push(t);
    }
  }
  while (!queues.empty()) {
    const int q = queues.pop();
    if (overused(s, q)) continue;
    for (;;) {
      if (!has_pre[q] || preemptors[q].empty()) break;
      const int job = preemptors[q].pop();
      std::vector<EOp> stmt;
      for (;;) {
        if (!job_starving(s, job)) break;
        if (!has_tasks[job] || ptasks[job].empty()) break;
        const int task = ptasks[job].pop();
        if (s.t_flags[task] & VC_TASK_PREEMPT_NEVER) continue;
        if (!preemptive(s, q, task)) continue;  // ssn.Preemptive(queue, task); ssn.PrePredicateFn: nil for pods in scope
        reclaim_for_task(s, stmt, task, job);
      }
      if (job_pipelined(s, job)) {
        emit_statement(s, job, stmt, true);
      } else {
        estmt_discard(s, stmt);
        emit_statement(s, job, stmt, false);
      }
      if (!preemptors[q].empty()) queues.push(q);
    }
  }
  return VC_OK;
}

// ---------------------------------------------------------------------------------------
// Dense pass on the opening snapshot (the oracle for vc_score_matrix)
// ---------------------------------------------------------------------------------------
void score_matrix(Session &s, uint64_t *mask_out, double *score_out, double *best_score, int32_t *best_node) {
  const int N = s.N, T = s.T_alloc;
  const size_t mw = ((size_t)N + 63) / 64;
  std::vector<int> idle_c, fut_c;
  std::vector<double> sc;
  for (int t = 0; t < T; ++t) {
    idle_c.clear();
    fut_c.clear();
    if (mask_out) std::fill(mask_out + t * mw, mask_out + (t + 1) * mw, 0ull);
    if (score_out) std::fill(score_out + (size_t)t * N, score_out + (size_t)(t + 1) * N, 0.0);
    for (int n = 0; n < N; ++n) {
      if (!predicate(s, t, n)) continue;
      if (mask_out) mask_out[t * mw + n / 64] |= 1ull << (n % 64);
      if (fits_idle(s, t, n)) idle_c.push_back(n);
      else fut_c.push_back(n);  // predicate() already established the FutureIdle fit
    }
    const std::vector<int> &cand = !idle_c.empty() ? idle_c : fut_c;
    double bs = 0;
    int bn = -1;
    if (!cand.empty()) {
      s.task_alloc_hn = s.job_soft[s.t_job[t]] ? s.job_alloc_hn[s.t_job[t]] : -1;
      bn = prioritize_and_select(s, t, cand, &bs, &sc);
      if (score_out)
        for (size_t i = 0; i < cand.size(); ++i) score_out[(size_t)t * N + cand[i]] = sc[i];
    }
    if (best_score) best_score[t] = bn >= 0 ? bs : 0.0;
    if (best_node) best_node[t] = bn;
  }
}

// ---------------------------------------------------------------------------------------
// Load
// ---------------------------------------------------------------------------------------
Res res_from_soa(const double *base, int count, int idx, int R, uint32_t has_bits) {
  Res r;
  if (!base) return r;
  for (int d = 0; d < R; ++d) r.v[d] = base[(size_t)d * count + idx];
  r.has = has_bits & ~(VC_RES_HAS_ANY | 3u) & ((R >= 32) ? ~0u : ((1u << R) - 1));
  for (int d = 2; d < R; ++d)
    if (!(r.has & (1u << d))) r.v[d] = 0.0;
  r.nilmap = r.has == 0;
  return r;
}

Session *load(const vc_dims *dims, const vc_nodes *nd, const vc_tasks *tk, const vc_classes *cl, const vc_jobs *jb,
              const vc_queues *qu, const vc_conf *conf, int threads) {
  Session *sp = new Session();
  Session &s = *sp;
  s.d = *dims;
  s.conf = *conf;
  s.N = dims->n_nodes; s.T = s.T_alloc = dims->n_tasks; s.J = dims->n_jobs; s.Q = dims->n_queues; s.C = dims->n_classes;
  s.R = dims->n_dims; s.K = dims->n_kdims; s.Wl = dims->label_words; s.Wt = dims->taint_words; s.NR = dims->n_roles;
  const size_t N = s.N, T = s.T, J = s.J, Q = s.Q, C = s.C, R = s.R, K = s.K;
  copy_in(s.alloc, nd->allocatable, R * N); copy_in(s.idle, nd->idle, R * N); copy_in(s.used, nd->used, R * N);
  copy_in(s.rel, nd->releasing, R * N); copy_in(s.pip, nd->pipelined, R * N);
  copy_in(s.kalloc, nd->k8s_allocatable, K * N); copy_in(s.kreq, nd->k8s_requested, K * N);
  copy_in(s.knz, nd->k8s_nonzero_requested, K * N);
  copy_in(s.max_tasks, nd->max_tasks, N); copy_in(s.pod_count, nd->pod_count, N);
  copy_in(s.zone, nd->revocable_zone, N, (int32_t)-1);
  copy_in(s.labels, nd->label_bits, (size_t)s.Wl * N); copy_in(s.thard, nd->taint_hard, (size_t)s.Wt * N);
  copy_in(s.tsoft, nd->taint_soft, (size_t)s.Wt * N); copy_in(s.nflags, nd->flags, N);
  copy_in(s.zone_active, nd->zone_active, (size_t)dims->n_zones);
  copy_in(s.req, tk->resreq, R * T); copy_in(s.req_has, tk->req_has, T);
  copy_in(s.tkreq, tk->k8s_req, K * T); copy_in(s.tknz, tk->k8s_nonzero_req, K * T);
  copy_in(s.t_job, tk->job, T); copy_in(s.t_class, tk->klass, T); copy_in(s.t_role, tk->role, T);
  copy_in(s.t_prio, tk->priority, T); copy_in(s.t_podidx, tk->pod_index, T, (int64_t)-1);
  copy_in(s.t_ts, tk->creation_ts, T); copy_in(s.t_uid, tk->uid_rank, T);
  s.t_status.assign(T, kPending);
  s.t_node.assign(T, -1);
  copy_in(s.c_sel, cl->selector, C * s.Wl); copy_in(s.c_naff, cl->n_affinity, C);
  copy_in(s.c_aff, cl->affinity, C * VC_MAX_TERMS * s.Wl); copy_in(s.c_tolh, cl->tolerated_hard, C * s.Wt);
  copy_in(s.c_tols, cl->tolerated_soft, C * s.Wt); copy_in(s.c_npref, cl->n_preferred, C);
  copy_in(s.c_pref, cl->preferred, C * VC_MAX_TERMS * s.Wl); copy_in(s.c_prefw, cl->preferred_weight, C * VC_MAX_TERMS);
  copy_in(s.c_flags, cl->flags, C);
  copy_in(s.j_queue, jb->queue, J); copy_in(s.j_min, jb->min_available, J); copy_in(s.j_prio, jb->priority, J);
  copy_in(s.j_ts, jb->creation_ts, J); copy_in(s.j_uid, jb->uid_rank, J); copy_in(s.j_flags, jb->flags, J);
  copy_in(s.j_ntasks, jb->n_tasks_total, J); copy_in(s.j_ready, jb->ready_num, J);
  copy_in(s.j_waiting, jb->waiting_num, J); copy_in(s.j_pbe, jb->pending_besteffort, J);
  copy_in(s.j_valid, jb->valid_num, J); copy_in(s.j_taskmintotal, jb->task_min_total, J);
  copy_in(s.j_roleoff, jb->role_off, J + 1); copy_in(s.j_alloc, jb->allocated, R * J);
  const size_t NR = s.NR;
  copy_in(s.r_min, jb->role_min, NR); copy_in(s.r_occ, jb->role_occupied, NR); copy_in(s.r_pip, jb->role_pipelined, NR);
  copy_in(s.r_pending, jb->role_pending_other, NR); copy_in(s.r_valid, jb->role_valid, NR);
  copy_in(s.r_flags, jb->role_flags, NR);
  s.r_failed.assign(NR, 0);
  for (size_t t = 0; t < T; ++t) s.r_pending[s.t_role[t]] += 1;  // pending[role], job_info.go:936-939
  copy_in(s.q_weight, qu->weight, Q); copy_in(s.q_prio, qu->priority, Q); copy_in(s.q_ts, qu->creation_ts, Q);
  copy_in(s.q_uid, qu->uid_rank, Q); copy_in(s.q_flags, qu->flags, Q);
  s.q_cap.resize(Q); s.q_guar.resize(Q); s.q_alloc0.resize(Q); s.q_req0.resize(Q);
  s.q_cap_any.assign(Q, 0); s.q_guar_any.assign(Q, 0);
  for (size_t q = 0; q < Q; ++q) {
    uint32_t ch = qu->capability_has ? qu->capability_has[q] : 0, gh = qu->guarantee_has ? qu->guarantee_has[q] : 0;
    s.q_cap_any[q] = (ch & VC_RES_HAS_ANY) != 0;
    s.q_guar_any[q] = (gh & VC_RES_HAS_ANY) != 0;
    s.q_cap[q] = res_from_soa(qu->capability, (int)Q, (int)q, (int)R, ch);
    s.q_guar[q] = res_from_soa(qu->guarantee, (int)Q, (int)q, (int)R, gh);
    s.q_alloc0[q] = res_from_soa(qu->allocated, (int)Q, (int)q, (int)R, qu->allocated_has ? qu->allocated_has[q] : 0);
    s.q_req0[q] = res_from_soa(qu->request, (int)Q, (int)q, (int)R, qu->request_has ? qu->request_has[q] : 0);
  }
  for (int i = 0; i < conf->n_plugins; ++i)
    if (conf->plugins[i].plugin > 0 && conf->plugins[i].plugin < 128) s.has_plugin[conf->plugins[i].plugin] = true;
  // ssn.TotalResource = sum of Allocatable (framework/session.go:272-274); a scalar is a key of the
  // sum when any node carries it (node vectors are dense: every dim is a key of every node)
  for (int d = 0; d < s.R; ++d) {
    double acc = 0;
    for (int n = 0; n < s.N; ++n) acc += at(s.alloc, d, s.N, n);
    s.total.v[d] = acc;
    if (d >= 2 && s.N > 0) { s.total.has |= 1u << d; s.total.nilmap = false; }
  }
  nta_init(s, nullptr);
  s.last_processed_node_index = s.N > 0 ? ((conf->last_processed_node_index % s.N) + s.N) % s.N : 0;
  s.j_share.assign(J, 0.0);
  if (s.has_plugin[VC_PLUGIN_DRF])
    for (int j = 0; j < s.J; ++j) drf_update_share(s, j);  // drf.go:186-214
  proportion_open(s);
  s.pool = new Pool(threads);
  return sp;
}

}  // namespace

// =======================================================================================
// C interface (ctypes)
// =======================================================================================
extern "C" {

void *vco_session_create(const vc_dims *dims, const vc_nodes *nd, const vc_tasks *tk, const vc_classes *cl,
                         const vc_jobs *jb, const vc_queues *qu, const vc_conf *conf, int threads) {
  return load(dims, nd, tk, cl, jb, qu, conf, threads);
}
void vco_session_destroy(void *h) { delete (Session *)h; }
// vc_snapshot_set_backfill for the oracle: the BestEffort tasks are appended to the session's task arrays
int vco_session_set_backfill(void *h, int32_t n, const vc_tasks *bt) {
  Session &s = *(Session *)h;
  if (n <= 0 || !bt || s.T != s.T_alloc) return n == 0 ? VC_OK : VC_EINVAL;
  const size_t T0 = s.T, B = (size_t)n, T1 = T0 + B;
  auto widen = [&](std::vector<double> &v, size_t rows, const double *extra) {
    std::vector<double> w(rows * T1, 0.0);
    for (size_t r = 0; r < rows; ++r) {
      for (size_t t = 0; t < T0; ++t) w[r * T1 + t] = v[r * T0 + t];
      for (size_t t = 0; t < B; ++t) w[r * T1 + T0 + t] = extra ? extra[r * B + t] : 0.0;
    }
    v.swap(w);
  };
  widen(s.req, s.R, bt->resreq); widen(s.tkreq, s.K, bt->k8s_req); widen(s.tknz, s.K, bt->k8s_nonzero_req);
  for (size_t t = 0; t < B; ++t) {
    s.req_has.push_back(bt->req_has[t]); s.t_job.push_back(bt->job[t]); s.t_class.push_back(bt->klass[t]);
    s.t_role.push_back(bt->role[t]); s.t_prio.push_back(bt->priority[t]);
    s.t_podidx.push_back(bt->pod_index ? bt->pod_index[t] : -1); s.t_ts.push_back(bt->creation_ts ? bt->creation_ts[t] : 0);
    s.t_uid.push_back(bt->uid_rank[t]);
    s.t_status.push_back(kPending); s.t_node.push_back(-1);
  }
  s.T = (int)T1;
  return VC_OK;
}
int vco_backfill(void *h) { return backfill_execute(*(Session *)h); }
// vc_snapshot_set_running for the oracle: node.Tasks entries are appended to the session's task arrays
// Pod.Status.NominatedNodeName of the pending tasks as node indices (-1 none); mirrors vc_snapshot_set_nominated
int vco_session_set_nominated(void *h, const int32_t *nominated_node) {
  Session &s = *(Session *)h;
  s.t_nominated.clear();
  if (nominated_node) s.t_nominated.assign(nominated_node, nominated_node + s.T_alloc);
  return VC_OK;
}

int vco_session_set_running(void *h, const vc_running_tasks *rt, const uint32_t *task_flags) {
  Session &s = *(Session *)h;
  if (s.T_run0 >= 0) return VC_EINVAL;
  s.t_flags.assign(s.T_alloc, 0u);
  if (task_flags) s.t_flags.assign(task_flags, task_flags + s.T_alloc);
  const size_t T0 = s.T, B = rt ? (size_t)rt->n_tasks : 0, T1 = T0 + B;
  s.T_run0 = (int)T0;
  s.node_tasks.assign(s.N, {});
  if (B == 0) return VC_OK;
  auto widen = [&](std::vector<double> &v, size_t rows, const double *extra) {
    std::vector<double> w(rows * T1, 0.0);
    for (size_t r = 0; r < rows; ++r) {
      for (size_t t = 0; t < T0; ++t) w[r * T1 + t] = v[r * T0 + t];
      for (size_t t = 0; t < B; ++t) w[r * T1 + T0 + t] = extra ? extra[r * B + t] : 0.0;
    }
    v.swap(w);
  };
  widen(s.req, s.R, rt->resreq); widen(s.tkreq, s.K, rt->k8s_req); widen(s.tknz, s.K, rt->k8s_nonzero_req);
  for (size_t t = 0; t < B; ++t) {
    s.req_has.push_back(rt->req_has[t]); s.t_job.push_back(rt->job[t]); s.t_class.push_back(0);
    s.t_role.push_back(rt->role[t]); s.t_prio.push_back(rt->priority[t]);
    s.t_podidx.push_back(rt->pod_index ? rt->pod_index[t] : -1); s.t_ts.push_back(rt->creation_ts ? rt->creation_ts[t] : 0);
    s.t_uid.push_back(rt->uid_rank[t]);
    s.t_status.push_back((rt->flags[t] & VC_RT_RUNNING) ? kRunning : kBound); s.t_node.push_back(rt->node[t]);
    s.rt_flags.push_back(rt->flags[t]);
    if (rt->node[t] < 0 || rt->node[t] >= s.N) return VC_EINVAL;
    s.node_tasks[rt->node[t]].push_back((int)(T0 + t));
  }
  s.T = (int)T1;
  return VC_OK;
}
int vco_preempt(void *h) { return preempt_execute(*(Session *)h); }
int vco_reclaim(void *h) { return reclaim_execute(*(Session *)h); }
// pickUpPendingTasks order only (backfill_test.go:39-154): indices into the backfill task list
int vco_backfill_pick_order(void *h, int32_t *out) {
  Session &s = *(Session *)h;
  std::vector<int> p = backfill_pick_up_pending_tasks(s, nullptr);
  for (size_t i = 0; i < p.size(); ++i) out[i] = p[i] - s.T_alloc;
  return (int)p.size();
}
// ph.PredicateNodes for one task with a fresh PredicateHelper (util/predicate_helper.go:43-140), for the reference's
// TestPredicateNodes (util/predicate_helper_test.go:31-220): nodes_out = the feasible nodes in scan order, cache_out[n] = the
// node has an entry in taskPredicateErrorCache[job/role], *group_exists = the cache holds that group at all
int vco_predicate_nodes(void *h, int t, int32_t *nodes_out, uint8_t *cache_out, int *group_exists) {
  Session &s = *(Session *)h;
  PredicateHelper ph;
  const int j = s.t_job[t];
  ph.role_base = s.j_roleoff[j];
  const int nroles = s.j_roleoff[j + 1] - s.j_roleoff[j];
  ph.node_err.resize(nroles);
  ph.exists.assign(nroles, 0);
  std::vector<int> feasible;
  predicate_nodes(s, ph, t, feasible);
  const int lr = s.t_role[t] - ph.role_base;
  *group_exists = ph.exists[lr];
  for (int n = 0; n < s.N; ++n) cache_out[n] = (!ph.node_err[lr].empty() && ph.node_err[lr][n]) ? 1 : 0;
  for (size_t i = 0; i < feasible.size(); ++i) nodes_out[i] = feasible[i];
  return (int)feasible.size();
}
int vco_allocate_run(void *h) { return allocate_execute(*(Session *)h); }
// Sampled replay (BASELINE.md §3, config 4: "parity on a 1 % task sample replayed through the oracle"): the caller's
// decision list (any implementation's) is applied in order to this fresh session through Statement.Allocate /
// Pipeline; every decision whose index == offset (mod stride) is first re-derived here on the state reached so
// far — ph.PredicateNodes over all nodes (allocate.go:634) + alloc.prioritizeNodes (:661) — and compared (node,
// kind, score within 1e-6). The role-level predicate-error cache only skips nodes that failed earlier in the same
// visit; node resources only shrink inside a visit, so leaving it out cannot change a verdict. Returns the number
// of sampled decisions that differ; *first_bad = index of the first one (-1 when none).
int64_t vco_replay_check(void *h, const vc_decision *dec, size_t n_dec, const vc_visit *vis, size_t n_vis, int64_t stride,
                         int64_t offset, int64_t *first_bad, int64_t *n_checked) {
  Session &s = *(Session *)h;
  int64_t bad = 0, checked = 0;
  *first_bad = -1;
  std::vector<Op> ops;
  std::vector<int> feasible;
  PredicateHelper ph;
  int cur_visit = -1, allocated_hn = -1;
  for (size_t i = 0; i < n_dec; ++i) {
    const vc_decision &d = dec[i];
    const int t = d.task, j = s.t_job[t];
    if (d.visit != cur_visit) {
      if (cur_visit >= 0 && (size_t)cur_visit < n_vis && vis[cur_visit].outcome == VC_VISIT_COMMIT) {
        const int pj = vis[cur_visit].job;
        if (s.job_soft[pj]) s.job_alloc_hn[pj] = allocated_hn;  // allocate.go:681-686
      }
      cur_visit = d.visit;
      allocated_hn = s.job_alloc_hn[j];  // allocate.go:572
      ops.clear();
    }
    s.task_alloc_hn = s.job_soft[j] ? allocated_hn : -1;
    if (stride > 0 && (int64_t)(i % (size_t)stride) == offset) {
      ph.role_base = s.j_roleoff[j];
      const int nroles = s.j_roleoff[j + 1] - s.j_roleoff[j];
      ph.node_err.assign(nroles, {});
      ph.exists.assign(nroles, 0);
      const int32_t pct = s.conf.percentage_nodes_to_find;
      s.conf.percentage_nodes_to_find = 100;
      predicate_nodes(s, ph, t, feasible);
      s.conf.percentage_nodes_to_find = pct;
      double score = 0;
      const int best = feasible.empty() ? -1 : prioritize_nodes(s, t, feasible, &score);
      const int kind = best >= 0 && !fits_idle(s, t, best) ? VC_OP_PIPELINE : VC_OP_ALLOCATE;
      checked += 1;
      if (best != d.node || kind != d.kind || !(std::fabs(score - d.score) <= 1e-6)) {
        if (*first_bad < 0) *first_bad = (int64_t)i;
        bad += 1;
      }
    }
    if (d.node < 0 || d.node >= s.N) { if (*first_bad < 0) *first_bad = (int64_t)i; return bad + 1; }
    if (d.kind == VC_OP_ALLOCATE) stmt_allocate(s, ops, t, d.node, d.score);
    else stmt_pipeline(s, ops, t, d.node, d.score);
    if (s.job_soft[j]) allocated_hn = new_allocated_hypernode(s, d.node, allocated_hn);  // :672-674
  }
  *n_checked = checked;
  return bad;
}
size_t vco_num_decisions(void *h) { return ((Session *)h)->decisions.size(); }
const vc_decision *vco_decisions(void *h) { return ((Session *)h)->decisions.data(); }
size_t vco_num_visits(void *h) { return ((Session *)h)->visits.size(); }
const vc_visit *vco_visits(void *h) { return ((Session *)h)->visits.data(); }
size_t vco_num_fit_errors(void *h) { return ((Session *)h)->fit_errors.size(); }
const int32_t *vco_fit_errors(void *h) { return ((Session *)h)->fit_errors.data(); }
int64_t vco_num_sweeps(void *h) { return ((Session *)h)->sweeps; }
// HyperNode tree of the session (before any run); mirrors vc_snapshot_set_topology
void vco_session_set_topology(void *h, const vc_hypernodes *topo) { nta_init(*(Session *)h, topo); }
// hyperNodeResourceCache entry (allocatable, used) of hypernode `hn`, for Test_initHyperNodeResourceCache
void vco_hypernode_status(void *h, int hn, double *alloc_out, double *used_out) {
  Session &s = *(Session *)h;
  for (int d = 0; d < s.R; ++d) {
    alloc_out[d] = at(s.hn_alloc, d, s.hn_H, hn);
    used_out[d] = at(s.hn_used, d, s.hn_H, hn);
  }
}
// network-topology-aware BatchNodeOrderFn entry of (task, node); 0 when the map has no entry
double vco_nta_node_score(void *h, int t, int n) {
  Session &s = *(Session *)h;
  return s.nta_on ? nta_node_score(s, t, n) : 0.0;
}
// BatchNodeOrderFn of the plugin for a pod WITH a network topology over `nodes` (scaled); out[i] = 0 when
// the returned map has no entry for the node
void vco_nta_topo_scores(void *h, int t, int allocated_hn, const int32_t *nodes, int n_nodes, double *out) {
  Session &s = *(Session *)h;
  std::vector<int> nv(nodes, nodes + n_nodes);
  std::vector<double> sc;
  std::vector<uint8_t> has;
  s.task_alloc_hn = allocated_hn;
  topo_node_scores(s, t, nv, sc, has);
  for (int i = 0; i < n_nodes; ++i) out[i] = has[i] ? (double)kMaxNodeScore * (double)s.conf.nta_weight * sc[i] : 0.0;
}
int vco_job_allocated_hypernode(void *h, int j) { return ((Session *)h)->job_alloc_hn[j]; }
int64_t vco_last_processed_node_index(void *h) { return ((Session *)h)->last_processed_node_index; }
double vco_go_pow_uint(double x, unsigned n) { return go_pow_uint(x, n); }
void vco_score_matrix(void *h, uint64_t *mask_out, double *score_out, double *best_score, int32_t *best_node) {
  score_matrix(*(Session *)h, mask_out, score_out, best_score, best_node);
}
void vco_queue_deserved(void *h, double *deserved_out, double *share_out) {
  Session &s = *(Session *)h;
  for (int q = 0; q < s.Q; ++q) {
    for (int d = 0; d < s.R; ++d)
      deserved_out[(size_t)d * s.Q + q] = (d < 2 || (s.qattr[q].deserved.has & (1u << d))) ? s.qattr[q].deserved.v[d] : 0.0;
    share_out[q] = s.qattr[q].share;
  }
}
// node state after the run (for round-trip checks): idle/used/pipelined [R][N]
void vco_node_state(void *h, double *idle, double *used, double *pipelined) {
  Session &s = *(Session *)h;
  size_t n = (size_t)s.R * s.N;
  if (idle) std::memcpy(idle, s.idle.data(), n * sizeof(double));
  if (used) std::memcpy(used, s.used.data(), n * sizeof(double));
  if (pipelined) std::memcpy(pipelined, s.pip.data(), n * sizeof(double));
}

// ---- primitives for the reference's known-answer tests ---------------------------------
// Resource.LessEqual (api/resource_info_test.go:609 TestLessEqual)
// Resource.Diff(rr, Zero) and MinDimensionResource(rr, Zero | Infinity) on plain vectors (api/resource_info_test.go:315-487,
// :1562-1693): outputs are value vectors + key-presence masks
int vco_less_equal_with_dimension(const double *l, uint32_t l_has, const double *r, uint32_t r_has, const double *req,
                                  uint32_t req_has, int R, int pods_dim) {
  return res_less_equal_with_dimension(res_from_soa(l, 1, 0, R, l_has), res_from_soa(r, 1, 0, R, r_has),
                                       res_from_soa(req, 1, 0, R, req_has), R, pods_dim) ? 1 : 0;
}
void vco_diff_zero(const double *l, uint32_t l_has, const double *r, uint32_t r_has, int R, double *inc_out, uint32_t *inc_has,
                   double *dec_out, uint32_t *dec_has) {
  Res a = res_from_soa(l, 1, 0, R, l_has), b = res_from_soa(r, 1, 0, R, r_has), inc, dec;
  res_diff_zero(a, b, inc, dec, R);
  for (int d = 0; d < R; ++d) { inc_out[d] = inc.v[d]; dec_out[d] = dec.v[d]; }
  *inc_has = inc.has; *dec_has = dec.has;
}
void vco_min_dimension(const double *l, uint32_t l_has, const double *r, uint32_t r_has, int R, int infinity, double *out,
                       uint32_t *out_has) {
  Res a = res_from_soa(l, 1, 0, R, l_has), b = res_from_soa(r, 1, 0, R, r_has);
  res_min_dimension(a, b, infinity != 0, R);
  for (int d = 0; d < R; ++d) out[d] = a.v[d];
  *out_has = a.has;
}
int vco_less_equal(const double *l, uint32_t l_has, const double *r, uint32_t r_has, int R, int infinity) {
  if (!le_eps(l[0], r[0])) return 0;
  if (!le_eps(l[1], r[1])) return 0;
  if (infinity) {  // :444-450
    for (int d = 2; d < R; ++d)
      if ((r_has & (1u << d)) && !(l_has & (1u << d))) return 0;
  }
  for (int d = 2; d < R; ++d) {
    if (!(l_has & (1u << d))) continue;
    bool ok = (r_has & (1u << d)) != 0;
    if (!ok && infinity) continue;
    double rv = ok ? r[d] : 0.0;
    if (!le_eps(l[d], rv)) return 0;
  }
  return 1;
}
int32_t vco_num_feasible_nodes(int32_t n, int32_t pct, int32_t min_nodes, int32_t min_pct) {
  return num_feasible_nodes_to_find(n, pct, min_nodes, min_pct);
}
int64_t vco_least_requested_score(int64_t requested, int64_t capacity) { return least_requested_score(requested, capacity); }
int64_t vco_most_requested_score(int64_t requested, int64_t capacity) { return most_requested_score(requested, capacity); }
// single (task,node) scores on the opening snapshot
double vco_binpack_score(void *h, int t, int n) { return binpack_score(*(Session *)h, t, n); }
double vco_nodeorder_score(void *h, int t, int n) { return nodeorder_score(*(Session *)h, t, n); }
int64_t vco_least_allocated(void *h, int t, int n) { return least_allocated(*(Session *)h, t, n); }
int64_t vco_most_allocated(void *h, int t, int n) { return most_allocated(*(Session *)h, t, n); }
int64_t vco_balanced_allocation(void *h, int t, int n) { return balanced_allocation(*(Session *)h, t, n); }
int vco_predicate(void *h, int t, int n) { return predicate(*(Session *)h, t, n) ? 1 : 0; }
double vco_job_share(void *h, int j) { return ((Session *)h)->j_share[j]; }
int vco_job_ready(void *h, int j) { return job_ready(*(Session *)h, j) ? 1 : 0; }
// JobInfo.IsReady / IsPipelined (api/job_info.go:1169-1175) on the opening counters
// util.SelectBestNodeAndScore (util/scheduler_helper.go:191-206) with the canonical tie-break, on explicit (score, node)
// pairs; returns the node index or -1 for an empty map
int vco_select_best(const double *scores, const int32_t *nodes, int n, double *best_score) {
  int best = -1;
  double bs = -std::numeric_limits<double>::infinity();
  for (int i = 0; i < n; ++i)
    if (scores[i] > bs || (scores[i] == bs && best >= 0 && nodes[i] < nodes[best])) { bs = scores[i]; best = i; }
  if (best < 0) { *best_score = 0.0; return -1; }
  *best_score = bs;
  return nodes[best];
}
int vco_job_is_ready(void *h, int j) { Session &s = *(Session *)h; return s.j_ready[j] + s.j_pbe[j] >= s.j_min[j]; }
int vco_job_is_pipelined(void *h, int j) {
  Session &s = *(Session *)h;
  return s.j_waiting[j] + s.j_ready[j] + s.j_pbe[j] >= s.j_min[j];
}

}  // extern "C"

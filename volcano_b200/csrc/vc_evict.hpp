// vc_evict.hpp — host control of the preempt and reclaim actions of libvcalloc.so (product code, C++17).
//
// actions/preempt/preempt.go:101-434 and actions/reclaim/reclaim.go:56-258. The action loops (queues, jobs, preemptor
// tasks, statements) and the victim selection on the ONE node under trial run here, as they run on the reference's action
// goroutine; everything that is wide — predicates and scores of every node for the preemptor, the ValidateVictims
// pre-test, the node order — runs on the device (vc_evict.cuh) and is consumed through `Ranker`.
#pragma once
#include <functional>
#include <utility>

#include "vc_host.hpp"
#include "vc_topo.hpp"

namespace vch {

struct RunningTasks {  // host copy of vc_running_tasks + CSR over nodes
  int n = 0;
  std::vector<int32_t> node, job, role, prio, off, idx;
  std::vector<int64_t> podidx, ts;
  std::vector<uint32_t> uid, has, flags;
  std::vector<double> req, kreq, knz;  // [R][n], [K][n], [K][n]
};

struct VictimGuards {  // host copy of vc_victim_guards (the pdb and cdp victim votes)
  int n_running = 0;
  std::vector<int32_t> allowed, off, pdb;
  std::vector<uint32_t> flags;
  std::vector<int64_t> until;
  int64_t now_ns = 0;
  bool cdp_protects(int r) const { return until[r] != VC_COOLDOWN_NONE && until[r] > now_ns; }  // cdp.go:87-96
  // the VCT_GUARD_* bits the device votes read for task r
  uint8_t device_bits(int r) const {
    uint8_t b = 0;
    if (flags[r] & VC_GUARD_NO_LABELS) b |= VCT_GUARD_NO_LABELS | VCT_GUARD_PDB_NEVER;
    for (int x = off[r]; x < off[r + 1]; ++x)
      if (allowed[pdb[x]] <= 0) b |= VCT_GUARD_PDB_NEVER;  // the first decrement already protects the task
    if (cdp_protects(r)) b |= VCT_GUARD_CDP;
    return b;
  }
};

struct EvictKeep {  // session-open state kept at every upload
  std::vector<int32_t> j_queue, j_min, j_prio, j_ntasks, j_ready0, j_waiting0, j_pbe, j_taskmintotal, j_roleoff;
  std::vector<uint32_t> j_flags, j_rank;
  std::vector<uint8_t> j_valid;
  std::vector<double> j_alloc0;  // [R][J]
  std::vector<int32_t> r_min, r_occ0, r_pip0;
  std::vector<uint32_t> r_flags;
  std::vector<int32_t> q_prio;
  std::vector<uint32_t> q_rank, q_flags;
  std::vector<int32_t> t_job, t_role, t_prio, t_class;
  std::vector<int64_t> t_podidx, t_ts;
  std::vector<uint32_t> t_uid, t_has;
  std::vector<double> t_req, t_kreq, t_knz;  // [R][T], [K][T], [K][T]
  std::vector<double> n_idle, n_rel, n_pip;  // [R][N]
};

// container/heap as util.PriorityQueue uses it (util/priority_queue.go:30-111)
struct GoPQ {
  std::vector<int> h;
  std::function<bool(int, int)> less;
  bool empty() const { return h.empty(); }
  void push(int x) {
    h.push_back(x);
    int j = (int)h.size() - 1;
    for (;;) {
      const int i = (j - 1) / 2;
      if (i == j || !less(h[j], h[i])) break;
      std::swap(h[i], h[j]);
      j = i;
    }
  }
  int pop() {
    const int n = (int)h.size() - 1;
    std::swap(h[0], h[n]);
    int i = 0;
    for (;;) {
      const int j1 = 2 * i + 1;
      if (j1 >= n || j1 < 0) break;
      int j = j1;
      if (j1 + 1 < n && less(h[j1 + 1], h[j1])) j = j1 + 1;
      if (!less(h[j], h[i])) break;
      std::swap(h[i], h[j]);
      i = j;
    }
    const int x = h.back();
    h.pop_back();
    return x;
  }
};

struct EvictOp { int kind, task, node; };  // VC_OP_EVICT (task = running-task id) / VC_OP_PIPELINE (task = vc_tasks id)

// Per task: 1 when allocate left job.NodesFitErrors[task] with node errors (allocate.go:599-647), the entries
// ssn.FilterOutUnschedulableAndUnresolvableNodesForTask filters on. Allocate's fit-error list holds, in order, the tasks
// whose predicate failed on every node (an entry with node errors) and the tasks it skipped through job.TaskHasFitErrors
// (an entry without any): a task of a named role is skipped once an earlier task of its role has an entry (FitFailedRoles,
// api/job_info.go:881-902); a task of an unnamed role never is.
inline std::vector<uint8_t> fit_error_node_kinds(const int32_t *fit, size_t n_fit, const int32_t *t_role,
                                                 const uint32_t *r_flags, size_t T) {
  std::vector<uint8_t> out(T, 0);
  std::vector<uint8_t> failed;  // [role] 1: the role has an entry
  for (size_t i = 0; i < n_fit; ++i) {
    const int t = fit[i], r = t_role[t];
    if ((size_t)r >= failed.size()) failed.resize((size_t)r + 1, 0);
    if (!(r_flags[r] & VC_ROLE_EMPTY_NAME) && failed[r]) continue;
    out[t] = 1;
    failed[r] = 1;
  }
  return out;
}

// The device side as the control loop sees it
struct Ranker {
  // rank every node for preemptor `t` under `mode`; then next() yields the candidate nodes in the action's order, -1 at the end
  // optional: the preemptor the control loop will try next if the one passed to the coming begin() fails (the device may
  // rank it ahead; a success in between voids that ranking)
  std::function<void(int t, int mode)> hint = [](int, int) {};
  std::function<int(int t, int mode)> begin;     // returns 0 or a VC_E* code
  std::function<int(int *node)> next;
  std::function<int(int t, int node, const std::vector<int> &victims)> apply;
  std::function<int(int t, int node, const std::vector<int> &victims)> revert;  // the inverse, for a discarded statement
  // topology-aware preemption: dry runs on every predicate node and SelectCandidate for preemptor `t`; -> the chosen node
  // (-1: no candidate) and its victims in eviction order. Set only when the action runs that reading.
  std::function<int(int t, int mode, int *node, std::vector<int> *victims)> topo;
};

struct EvictSession {
  const vc_conf *conf = nullptr;
  const EvictKeep *k = nullptr;
  const RunningTasks *rt = nullptr;
  const std::vector<uint32_t> *t_flags = nullptr;
  const VictimGuards *g = nullptr;  // set when pdb or cdp votes in the action
  int R = 0, K = 0, N = 0, T = 0, J = 0, Q = 0, pods_dim = -1;
  double total[VC_MAX_DIMS] = {0};
  uint32_t total_has = 0;
  // mutable state
  std::vector<int8_t> t_status;  // 0 Pending, 1 Allocated / Binding, 2 Pipelined
  std::vector<int32_t> j_ready, j_waiting, r_occ, r_pip;
  std::vector<double> j_alloc, j_share;
  std::vector<QAttr> qattr;
  std::vector<double> n_idle, n_rel, n_pip;  // [R][N]; Idle moves with allocate's placements, never under Evict / Pipeline
  std::vector<uint8_t> rt_evicted;
  bool phase_flipped = false;  // allocate ran without the enqueue action: Pending PodGroups are Inqueue now

  // ---- plumbing -------------------------------------------------------------------------------------------
  double treq(int d, int t) const { return k->t_req[(size_t)d * T + t]; }
  double rreq(int d, int r) const { return rt->req[(size_t)d * rt->n + r]; }
  HRes task_res(int t) const { return HRes::load(k->t_req.data(), T, t, R, k->t_has[t]); }
  HRes run_res(int r) const { return HRes::load(rt->req.data(), rt->n, r, R, rt->has[r]); }
  bool en(int i, uint32_t f) const { return (conf->plugins[i].enabled & f) != 0; }

  void drf_share(int j) {  // drf.calculateShare, drf.go:566-578
    double res = 0;
    for (int d = 0; d < R; ++d) {
      if (d >= 2 && !((total_has >> d) & 1u)) continue;
      if (!(total[d] >= kMinRes)) continue;
      const double sh = share_of(j_alloc[(size_t)d * J + j], total[d]);
      if (sh > res) res = sh;
    }
    j_share[j] = res;
  }
  // AllocateFunc / DeallocateFunc of drf (drf.go:391-454) and proportion (proportion.go:475-518)
  void on_allocate(int j, const HRes &rq, const double *col, int count, int idx) {
    if (has_plugin(*conf, VC_PLUGIN_DRF)) {
      for (int d = 0; d < R; ++d) j_alloc[(size_t)d * J + j] += col[(size_t)d * count + idx];
      drf_share(j);
    }
    const int q = k->j_queue[j];
    if (has_plugin(*conf, VC_PLUGIN_PROPORTION) && q >= 0 && qattr[q].exists) {
      qattr[q].allocated.add(rq, R);
      qattr[q].share = queue_share(qattr[q], R);
    }
  }
  void on_deallocate(int j, const HRes &rq, const double *col, int count, int idx) {
    if (has_plugin(*conf, VC_PLUGIN_DRF)) {
      for (int d = 0; d < R; ++d) j_alloc[(size_t)d * J + j] -= col[(size_t)d * count + idx];
      drf_share(j);
    }
    const int q = k->j_queue[j];
    if (has_plugin(*conf, VC_PLUGIN_PROPORTION) && q >= 0 && qattr[q].exists) {
      HRes &a = qattr[q].allocated;  // Resource.Sub -> sub, api/resource_info.go:293-320
      a.v[0] -= rq.v[0]; a.v[1] -= rq.v[1];
      if (!a.nil)
        for (int d = 2; d < R; ++d)
          if (rq.k(d)) { a.has |= 1u << d; a.v[d] -= rq.v[d]; }
      qattr[q].share = queue_share(qattr[q], R);
    }
  }

  // ---- readiness (api/job_info.go:1024-1070, :1169-1178) ---------------------------------------------------
  bool is_ready(int j) const { return j_ready[j] + k->j_pbe[j] >= k->j_min[j]; }
  bool is_pipelined(int j) const { return j_waiting[j] + j_ready[j] + k->j_pbe[j] >= k->j_min[j]; }
  bool check_task_pipelined(int j) const {
    if (k->j_min[j] < k->j_taskmintotal[j]) return true;
    for (int r = k->j_roleoff[j]; r < k->j_roleoff[j + 1]; ++r) {
      if (!(k->r_flags[r] & VC_ROLE_IN_MIN_MAP)) continue;
      if (r_occ[r] + r_pip[r] < k->r_min[r]) return false;
    }
    return true;
  }
  bool job_pipelined(int j) const {  // ssn.JobPipelined, session_plugins.go:450-478
    bool has_found = false;
    int i = 0;
    while (i < conf->n_plugins) {
      const int tier = conf->plugins[i].tier;
      for (; i < conf->n_plugins && conf->plugins[i].tier == tier; ++i) {
        if (!en(i, VC_EN_JOB_PIPELINED)) continue;
        int res;
        if (conf->plugins[i].plugin == VC_PLUGIN_GANG) res = (check_task_pipelined(j) && is_pipelined(j)) ? 1 : -1;
        else continue;
        if (res < 0) return false;
        if (res > 0) has_found = true;
      }
      if (has_found) return true;
    }
    return true;
  }
  bool job_starving(int j) const {  // ssn.JobStarving, session_plugins.go:482-506
    bool has_found = false;
    int i = 0;
    while (i < conf->n_plugins) {
      const int tier = conf->plugins[i].tier;
      for (; i < conf->n_plugins && conf->plugins[i].tier == tier; ++i) {
        if (!en(i, VC_EN_JOB_STARVING)) continue;
        bool res;
        if (conf->plugins[i].plugin == VC_PLUGIN_GANG) res = j_waiting[j] + j_ready[j] < k->j_min[j];
        else if (conf->plugins[i].plugin == VC_PLUGIN_PRIORITY) res = j_ready[j] + j_waiting[j] < k->j_ntasks[j];
        else continue;
        has_found = true;
        if (!res) return false;
      }
      if (has_found) return true;
    }
    return false;
  }

  // ---- order functions (session_plugins.go:660-783) ----------------------------------------------------------
  bool job_less(int l, int r) const {
    for (int i = 0; i < conf->n_plugins; ++i) {
      if (!en(i, VC_EN_JOB_ORDER)) continue;
      int c = 0;
      switch (conf->plugins[i].plugin) {
        case VC_PLUGIN_PRIORITY: c = k->j_prio[l] > k->j_prio[r] ? -1 : (k->j_prio[l] < k->j_prio[r] ? 1 : 0); break;
        case VC_PLUGIN_GANG: {
          const bool lr = is_ready(l), rr = is_ready(r);
          c = (lr && rr) ? 0 : (lr ? 1 : (rr ? -1 : 0));
          break;
        }
        case VC_PLUGIN_DRF: c = j_share[l] == j_share[r] ? 0 : (j_share[l] < j_share[r] ? -1 : 1); break;
        default: break;
      }
      if (c != 0) return c < 0;
    }
    return k->j_rank[l] < k->j_rank[r];
  }
  bool queue_less(int l, int r) const {
    for (int i = 0; i < conf->n_plugins; ++i) {
      if (!en(i, VC_EN_QUEUE_ORDER)) continue;
      if (conf->plugins[i].plugin == VC_PLUGIN_PROPORTION) {
        if (k->q_prio[l] != k->q_prio[r]) return k->q_prio[l] > k->q_prio[r];
        if (qattr[l].share != qattr[r].share) return qattr[l].share < qattr[r].share;
      }
    }
    return k->q_rank[l] < k->q_rank[r];
  }
  template <class P, class I, class S, class U>
  bool task_less_v(const P &prio, const I &idx, const S &ts, const U &uid, int l, int r) const {
    if (plugin_enabled(*conf, VC_PLUGIN_PRIORITY, VC_EN_TASK_ORDER) && prio[l] != prio[r]) return prio[l] > prio[r];
    const bool lerr = idx[l] < 0, rerr = idx[r] < 0;
    if (lerr || rerr || idx[l] == idx[r]) {
      if (ts[l] == ts[r]) return uid[l] < uid[r];
      return ts[l] < ts[r];
    }
    return !(idx[l] > idx[r]);
  }
  bool task_less(int l, int r) const { return task_less_v(k->t_prio, k->t_podidx, k->t_ts, k->t_uid, l, r); }
  bool run_less(int l, int r) const { return task_less_v(rt->prio, rt->podidx, rt->ts, rt->uid, l, r); }
  // pop order of ssn.BuildVictimsPriorityQueue (session_plugins.go:1092-1135; no VictimQueueOrderFn on this path)
  bool victim_less(int l, int r) const {
    const int lj = rt->job[l], rj = rt->job[r];
    if (lj == rj) return !run_less(l, r);
    if (lj < 0 || rj < 0) {
      if (lj < 0 && rj < 0) return !run_less(l, r);
      return lj < 0;
    }
    if (k->j_queue[lj] != k->j_queue[rj]) return !queue_less(k->j_queue[lj], k->j_queue[rj]);
    return !job_less(lj, rj);
  }

  // ---- proportion gates (proportion.go:333-348, :376-380) -----------------------------------------------------
  bool queue_allocatable(int q, int t) const {
    if (!(k->q_flags[q] & VC_QUEUE_OPEN)) return false;
    const QAttr &a = qattr[q];
    HRes fu = a.allocated;
    const HRes rq = task_res(t);
    fu.add(rq, R);
    // LessEqualWithDimensionAndResourcesName(deserved, req), api/resource_info.go:469-514
    bool ok = true;
    for (int d = 0; d < 2; ++d)
      if (rq.v[d] > 0 && fu.v[d] > a.deserved.v[d]) ok = false;
    if (fu.nil) return ok;  // r.ScalarResources == nil: whatever rr holds, the scalars pass
    for (int d = 2; d < R; ++d) {
      if (!rq.k(d) || d == pods_dim) continue;
      const double lq = fu.k(d) ? fu.v[d] : 0.0, rqv = a.deserved.k(d) ? a.deserved.v[d] : 0.0;
      if (rq.v[d] > 0 && lq > rqv) ok = false;
    }
    return ok;
  }
  bool gate(uint32_t flag, int q, int t) const {  // ssn.Allocatable / ssn.Preemptive
    for (int i = 0; i < conf->n_plugins; ++i) {
      if (!en(i, flag) || conf->plugins[i].plugin != VC_PLUGIN_PROPORTION) continue;
      if (!queue_allocatable(q, t)) return false;
    }
    return true;
  }
  bool overused(int q) const {  // proportion.go:319-331
    for (int i = 0; i < conf->n_plugins; ++i) {
      if (!en(i, VC_EN_OVERUSED) || conf->plugins[i].plugin != VC_PLUGIN_PROPORTION) continue;
      if (qattr[q].deserved.less_equal_zero(qattr[q].allocated, R)) return true;
    }
    return false;
  }

  // ---- node rows ------------------------------------------------------------------------------------------------
  double future_idle(int d, int n) const {  // node_info.go:114-116
    return (n_idle[(size_t)d * N + n] + n_rel[(size_t)d * N + n]) - n_pip[(size_t)d * N + n];
  }
  bool fits_future_idle(int t, int n) const {
    for (int d = 0; d < R; ++d) {
      if (d >= 2 && !((k->t_has[t] >> d) & 1u)) continue;
      if (!le_eps(treq(d, t), future_idle(d, n))) return false;
    }
    return true;
  }

  // ---- Statement operations (framework/statement.go:72-239) -----------------------------------------------------
  void evict(std::vector<EvictOp> &ops, int r) {
    const int j = rt->job[r], n = rt->node[r];
    if (j >= 0) { j_ready[j] -= 1; r_occ[rt->role[r]] -= 1; }
    rt_evicted[r] = 1;
    for (int d = 0; d < R; ++d) n_rel[(size_t)d * N + n] += rreq(d, r);
    if (j >= 0) on_deallocate(j, run_res(r), rt->req.data(), rt->n, r);
    ops.push_back({VC_OP_EVICT, r, n});
  }
  void unevict(int r) {
    const int j = rt->job[r], n = rt->node[r];
    if (j >= 0) { j_ready[j] += 1; r_occ[rt->role[r]] += 1; }
    rt_evicted[r] = 0;
    for (int d = 0; d < R; ++d) n_rel[(size_t)d * N + n] -= rreq(d, r);
    if (j >= 0) on_allocate(j, run_res(r), rt->req.data(), rt->n, r);
  }
  void pipeline(std::vector<EvictOp> &ops, int t, int n) {
    const int j = k->t_job[t];
    t_status[t] = 2;
    j_waiting[j] += 1; r_pip[k->t_role[t]] += 1;
    for (int d = 0; d < R; ++d) n_pip[(size_t)d * N + n] += treq(d, t);
    on_allocate(j, task_res(t), k->t_req.data(), T, t);
    ops.push_back({VC_OP_PIPELINE, t, n});
  }
  void unpipeline(int t, int n) {
    const int j = k->t_job[t];
    t_status[t] = 0;
    j_waiting[j] -= 1; r_pip[k->t_role[t]] -= 1;
    for (int d = 0; d < R; ++d) n_pip[(size_t)d * N + n] -= treq(d, t);
    on_deallocate(j, task_res(t), k->t_req.data(), T, t);
  }
  void discard(std::vector<EvictOp> &ops) {  // reverse order, statement.go:357-381
    for (int i = (int)ops.size() - 1; i >= 0; --i) {
      if (ops[i].kind == VC_OP_EVICT) unevict(ops[i].task);
      else unpipeline(ops[i].task, ops[i].node);
    }
    ops.clear();
  }

  // stmt.Discard() of a whole statement whose node attempts were already applied on the device: the operations come in
  // groups [evict ..., pipeline] per successful attempt (stmt.Merge, preempt.go:421); undo them last group first
  int discard_applied(const Ranker &rk, std::vector<EvictOp> &ops) {
    struct Group { int task, node; std::vector<int> victims; };
    std::vector<Group> groups;  // last group first
    int end = (int)ops.size();
    while (end > 0) {
      const int pi = end - 1;  // the group's pipeline op
      int b = pi;
      while (b > 0 && ops[b - 1].kind == VC_OP_EVICT) --b;
      Group g{ops[pi].task, ops[pi].node, {}};
      for (int i = b; i < pi; ++i) g.victims.push_back(ops[i].task);
      groups.push_back(std::move(g));
      end = b;
    }
    discard(ops);  // the host state first: the device refresh that follows every revert reads it
    for (const Group &g : groups) {
      const int rc = rk.revert(g.task, g.node, g.victims);
      if (rc) return rc;
    }
    return VC_OK;
  }

  // ---- victim functions of the plugins, candidates in node.Tasks order (ascending running-task id) ---------------
  std::vector<int> gang_victims(const std::vector<int> &c) const {  // gang.go:97-129
    std::vector<int> out;
    std::vector<std::pair<int, int>> occ;
    for (int r : c) {
      const int j = rt->job[r];
      if (j < 0) continue;
      int *o = nullptr;
      for (auto &e : occ) if (e.first == j) o = &e.second;
      if (!o) { occ.push_back({j, j_ready[j]}); o = &occ.back().second; }
      if (*o > k->j_min[j]) { *o -= 1; out.push_back(r); }
    }
    return out;
  }
  std::vector<int> priority_victims(int t, const std::vector<int> &c) const {  // priority.go:110-148
    std::vector<int> out;
    const int pj = k->t_job[t];
    for (int r : c) {
      const int j = rt->job[r];
      if (j < 0) continue;
      if (j != pj) { if (k->j_prio[j] < k->j_prio[pj]) out.push_back(r); }
      else if (rt->prio[r] < k->t_prio[t]) out.push_back(r);
    }
    return out;
  }
  double share_of_alloc(const std::vector<double> &al) const {
    double res = 0;
    for (int d = 0; d < R; ++d) {
      if (d >= 2 && !((total_has >> d) & 1u)) continue;
      if (!(total[d] >= kMinRes)) continue;
      const double sh = share_of(al[d], total[d]);
      if (sh > res) res = sh;
    }
    return res;
  }
  std::vector<int> drf_victims(int t, const std::vector<int> &c) const {  // drf.go:222-261
    std::vector<int> out;
    const int pj = k->t_job[t];
    std::vector<double> la(R);
    for (int d = 0; d < R; ++d) la[d] = j_alloc[(size_t)d * J + pj] + treq(d, t);
    const double ls = share_of_alloc(la);
    std::vector<std::pair<int, std::vector<double>>> allocs;
    for (int r : c) {
      const int j = rt->job[r];
      if (j < 0) continue;
      std::vector<double> *ra = nullptr;
      for (auto &e : allocs) if (e.first == j) ra = &e.second;
      if (!ra) {
        allocs.push_back({j, std::vector<double>(R)});
        ra = &allocs.back().second;
        for (int d = 0; d < R; ++d) (*ra)[d] = j_alloc[(size_t)d * J + j];
      }
      for (int d = 0; d < R; ++d) (*ra)[d] -= rreq(d, r);
      const double rs = share_of_alloc(*ra);
      if (ls < rs || std::fabs(ls - rs) <= 0.000001) out.push_back(r);
    }
    return out;
  }
  std::vector<int> proportion_victims(const std::vector<int> &c) const {  // proportion.go:286-317
    std::vector<int> out;
    std::vector<std::pair<int, HRes>> allocs;
    for (int r : c) {
      const int j = rt->job[r];
      if (j < 0) continue;
      const int q = k->j_queue[j];
      if (q < 0 || !qattr[q].exists) continue;
      HRes *al = nullptr;
      for (auto &e : allocs) if (e.first == q) al = &e.second;
      if (!al) { allocs.push_back({q, qattr[q].allocated}); al = &allocs.back().second; }
      if (!al->less_equal_zero(qattr[q].deserved, R)) {
        const HRes rq = run_res(r);
        al->v[0] -= rq.v[0]; al->v[1] -= rq.v[1];
        if (!al->nil)
          for (int d = 2; d < R; ++d)
            if (rq.k(d)) { al->has |= 1u << d; al->v[d] -= rq.v[d]; }
        out.push_back(r);
      }
    }
    return out;
  }
  // pdb.go:65-126: budgets start from DisruptionsAllowed on every call; each PDB counting a labelled candidate loses one,
  // and a candidate that drives one of them below zero is kept
  std::vector<int> pdb_victims(const std::vector<int> &c) const {
    std::vector<int> out;
    std::vector<std::pair<int, int>> budget;  // PDB -> what is left of its budget in this call
    for (int r : c) {
      if (g->flags[r] & VC_GUARD_NO_LABELS) continue;
      bool violated = false;
      for (int x = g->off[r]; x < g->off[r + 1]; ++x) {
        int *b = nullptr;
        for (auto &e : budget) if (e.first == g->pdb[x]) b = &e.second;
        if (!b) { budget.push_back({g->pdb[x], g->allowed[g->pdb[x]]}); b = &budget.back().second; }
        if (--*b < 0) violated = true;
      }
      if (!violated) out.push_back(r);
    }
    return out;
  }
  // ssn.Preemptable / ssn.Reclaimable, session_plugins.go:211-307
  std::vector<int> tier_victims(int t, const std::vector<int> &c, bool reclaim) const {
    std::vector<int> victims;
    bool nil = true;
    int i = 0;
    while (i < conf->n_plugins) {
      const int tier = conf->plugins[i].tier;
      for (int x = i; x < conf->n_plugins && conf->plugins[x].tier == tier; ++x) {
        if (!en(x, reclaim ? VC_EN_RECLAIMABLE : VC_EN_PREEMPTABLE)) continue;
        const int pl = conf->plugins[x].plugin;
        std::vector<int> cand;
        if (pl == VC_PLUGIN_GANG) cand = gang_victims(c);
        else if (pl == VC_PLUGIN_CONFORMANCE) { for (int r : c) if (!(rt->flags[r] & VC_RT_CRITICAL)) cand.push_back(r); }
        else if (pl == VC_PLUGIN_PRIORITY && !reclaim) cand = priority_victims(t, c);
        else if (pl == VC_PLUGIN_DRF && !reclaim) cand = drf_victims(t, c);
        else if (pl == VC_PLUGIN_PROPORTION && reclaim) cand = proportion_victims(c);
        else if (pl == VC_PLUGIN_PDB) cand = pdb_victims(c);
        else if (pl == VC_PLUGIN_CDP) { for (int r : c) if (!g->cdp_protects(r)) cand.push_back(r); }
        else continue;
        if (cand.empty()) { victims.clear(); nil = true; break; }
        if (nil) { victims = cand; nil = false; }
        else {
          std::vector<int> inter;
          for (int v : victims)
            for (int y : cand)
              if (v == y) inter.push_back(v);
          victims.swap(inter);
          nil = victims.empty();
        }
      }
      while (i < conf->n_plugins && conf->plugins[i].tier == tier) ++i;
      if (!nil) return victims;
    }
    return victims;
  }
  bool validate_victims(int t, int n, const std::vector<int> &victims) const {  // scheduler_helper.go:313-329
    for (int d = 0; d < R; ++d) {
      double fi = future_idle(d, n);
      for (int v : victims) fi += rreq(d, v);
      if (d >= 2 && !((k->t_has[t] >> d) & 1u)) continue;
      if (!le_eps(treq(d, t), fi)) return false;
    }
    return true;
  }
  bool run_filter(int r, int mode, int pj, int q) const {
    if (rt_evicted[r]) return false;
    const uint32_t f = rt->flags[r];
    if (!(f & VC_RT_PREEMPTABLE)) return false;
    const int j = rt->job[r];
    if (mode == 2) {  // reclaim.go:184-199
      if (!(f & VC_RT_RUNNING) || j < 0) return false;
      const int vq = k->j_queue[j];
      return vq >= 0 && vq != q && !(k->q_flags[vq] & VC_QUEUE_NOT_RECLAIMABLE);
    }
    if (!(f & (VC_RT_RUNNING | VC_RT_BOUND))) return false;
    if (mode == 1) return j == pj;
    return j >= 0 && j != pj && k->j_queue[j] == q;
  }

  // ---- one preemptor: normalPreempt (preempt.go:333-434) / reclaimForTask (reclaim.go:170-258) ---------------------
  int try_task(const Ranker &rk, std::vector<EvictOp> &stmt, int t, int mode, bool *assigned) {
    *assigned = false;
    if ((*t_flags)[t] & VC_TASK_PREEMPT_NEVER) return VC_OK;  // preempt.go:436-441 (reclaim checks it in its own loop)
    const int pj = k->t_job[t], q = k->j_queue[pj];
    int rc;
    if (rk.topo && mode != 2) {  // topologyAwarePreempt, preempt.go:475-520
      int n = -1;
      std::vector<int> victims;
      if ((rc = rk.topo(t, mode, &n, &victims)) || n < 0) return rc;
      std::vector<EvictOp> node_stmt;
      for (int v : victims) evict(node_stmt, v);  // prepareCandidate
      pipeline(node_stmt, t, n);
      stmt.insert(stmt.end(), node_stmt.begin(), node_stmt.end());
      if ((rc = rk.apply(t, n, victims))) return rc;
      *assigned = true;
      return VC_OK;
    }
    rc = rk.begin(t, mode);
    if (rc) return rc;
    for (;;) {
      int n = -1;
      if ((rc = rk.next(&n))) return rc;
      if (n < 0) return VC_OK;
      std::vector<int> cands;
      for (int x = rt->off[n]; x < rt->off[n + 1]; ++x)
        if (run_filter(rt->idx[x], mode, pj, q)) cands.push_back(rt->idx[x]);
      if (mode == 2 && cands.empty()) continue;
      std::vector<int> victims = tier_victims(t, cands, mode == 2);
      if (!validate_victims(t, n, victims)) continue;
      GoPQ vq;
      vq.less = [this](int l, int r) { return victim_less(l, r); };
      for (int v : victims) vq.push(v);
      std::vector<EvictOp> node_stmt;
      std::vector<int> evicted;
      bool ok;
      if (mode == 2) {
        std::vector<double> avail(R);
        for (int d = 0; d < R; ++d) avail[d] = future_idle(d, n);
        auto fits = [&]() {
          for (int d = 0; d < R; ++d) {
            if (d >= 2 && !((k->t_has[t] >> d) & 1u)) continue;
            if (!le_eps(treq(d, t), avail[d])) return false;
          }
          return true;
        };
        while (!vq.empty()) {
          if (fits()) break;
          const int v = vq.pop();
          evict(node_stmt, v);
          evicted.push_back(v);
          for (int d = 0; d < R; ++d) avail[d] += rreq(d, v);
        }
        ok = fits();
      } else {
        while (!vq.empty()) {
          if (gate(VC_EN_ALLOCATABLE, q, t) && fits_future_idle(t, n)) break;
          const int v = vq.pop();
          evict(node_stmt, v);
          evicted.push_back(v);
        }
        ok = gate(VC_EN_ALLOCATABLE, q, t) && fits_future_idle(t, n);
      }
      if (ok) {
        pipeline(node_stmt, t, n);
        stmt.insert(stmt.end(), node_stmt.begin(), node_stmt.end());  // stmt.Merge(nodeStmt)
        if ((rc = rk.apply(t, n, evicted))) return rc;
        *assigned = true;
        return VC_OK;
      }
      discard(node_stmt);
    }
  }
};

}  // namespace vch

// topo_oracle.cpp — test infrastructure: the CPU oracle (oracle/oracle.cpp, included unchanged) plus a plain restatement
// of the preempt action's topology-aware reading (enableTopologyAwarePreemption, actions/preempt/preempt.go:475-1015)
// under the determinism contract of include/vcalloc.h (vc_preempt_options). Independent of the library's vc_topo.hpp:
// the node and the cycle state are cloned per dry run, the victims come out of a Go heap, pickOneNodeForPreemption runs
// its score functions one after the other, and proportion's simulated state is kept for every queue.
#include "../../oracle/oracle.cpp"

#include <map>

namespace {

struct TopoOpts {
  vc_preempt_options o{0, 10, 1, 100, 0, 0, 0, nullptr, nullptr};
  std::vector<int32_t> prio;
  std::vector<int64_t> start;
  int k = 0;            // dry runs that met a predicate node
  bool bad = false;     // a negative numCandidates
};
std::map<void *, TopoOpts> g_topo;

uint64_t splitmix64(uint64_t x) {
  uint64_t z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
bool prop_enabled(const Session &s, uint32_t flag) {
  for (int i = 0; i < s.conf.n_plugins; ++i)
    if (s.conf.plugins[i].plugin == VC_PLUGIN_PROPORTION && (s.conf.plugins[i].enabled & flag)) return true;
  return false;
}
void res_sub_plain(Res &r, const Res &rr, int R) {  // Resource.sub
  r.v[0] -= rr.v[0];
  r.v[1] -= rr.v[1];
  if (r.nilmap) return;
  for (int d = 2; d < R; ++d)
    if (rr.has & (1u << d)) { r.has |= 1u << d; r.v[d] -= rr.v[d]; }
}

struct DryRun {  // the clones one dry run works on
  std::vector<double> idle;         // nodeInfoCopy.Idle
  bool have_state = false;          // proportion's PrePredicateFn wrote its state
  std::vector<Res> qalloc;          // state.queueAttrs[*].allocated
};

// SelectVictimsOnNode, preempt.go:708-842
bool select_victims_on_node(Session &s, const TopoOpts &o, DryRun &dr, int preemptor, int phase_job, int n,
                            std::vector<int> &victims) {
  const int pj = s.t_job[preemptor], q = s.j_queue[pj];
  const bool sim_update = prop_enabled(s, VC_EN_PREEMPTABLE) || prop_enabled(s, VC_EN_ALLOCATABLE);
  const bool sim_alloc = prop_enabled(s, VC_EN_ALLOCATABLE);
  auto remove_task = [&](int t) -> bool {
    if (sim_update) {
      const int vq = s.j_queue[s.t_job[t]];
      if (!dr.have_state || vq < 0 || !s.qattr[vq].exists) return false;
      res_sub_plain(dr.qalloc[vq], task_res(s, t), s.R);
    }
    for (int d = 0; d < s.R; ++d) dr.idle[d] += at(s.req, d, s.T, t);
    return true;
  };
  auto add_task = [&](int t) {
    if (sim_update) res_add(dr.qalloc[s.j_queue[s.t_job[t]]], task_res(s, t), s.R);
    for (int d = 0; d < s.R; ++d) dr.idle[d] -= at(s.req, d, s.T, t);
  };
  auto fits = [&]() {
    if (sim_alloc) {
      if (!dr.have_state || !s.qattr[q].exists) return false;
      Res fu = dr.qalloc[q];
      const Res rq = task_res(s, preemptor);
      res_add(fu, rq, s.R);
      if (!res_less_equal_with_dimension(fu, s.qattr[q].deserved, rq, s.R, s.d.pods_dim)) return false;
    }
    for (int d = 0; d < s.R; ++d) {
      if (d >= 2 && !(s.req_has[preemptor] & (1u << d))) continue;
      const double fi = (dr.idle[d] + at(s.rel, d, s.N, n)) - at(s.pip, d, s.N, n);
      if (!le_eps(at(s.req, d, s.T, preemptor), fi)) return false;
    }
    return true;
  };
  std::vector<int> preemptees;
  for (int t : s.node_tasks[n]) {
    if (!preemptable_status(s, t) || !rt_flag(s, t, VC_RT_PREEMPTABLE)) continue;
    const int j = s.t_job[t];
    if (phase_job < 0) {
      if (j < 0 || !(s.j_queue[j] == q && j != pj)) continue;
    } else if (j != pj) {
      continue;
    }
    preemptees.push_back(t);
  }
  const std::vector<int> all = tier_victims(s, preemptor, preemptees, false);
  if (!validate_victims(s, preemptor, n, all)) return false;
  GoHeap vq;
  vq.less = [&s](int l, int r) { return victim_less(s, l, r); };
  for (int v : all) vq.push(v);
  std::vector<int> potential;
  while (!vq.empty()) {
    const int t = vq.pop();
    potential.push_back(t);
    if (!remove_task(t)) return false;
    if (fits()) break;
  }
  if (potential.empty()) return false;
  std::reverse(potential.begin(), potential.end());
  victims.clear();
  for (int t : potential) {
    add_task(t);
    if (!fits()) {
      remove_task(t);
      victims.push_back(t);
    }
  }
  return !victims.empty();
}

// pickOneNodeForPreemption, preempt.go:899-979, over the candidates in their order
int pick_one(const Session &s, const TopoOpts &o, const std::vector<std::pair<int, std::vector<int>>> &cands) {
  auto pp = [&](int t) { return (int64_t)o.prio[t - s.T_run0]; };
  auto start = [&](int t) { const int64_t v = o.start[t - s.T_run0]; return v == VC_START_TIME_UNSET ? o.o.now_ns : v; };
  std::vector<std::function<int64_t(int)>> fs = {
      [&](int c) { return -pp(cands[c].second[0]); },
      [&](int c) { int64_t sum = 0; for (int t : cands[c].second) sum += pp(t) + 2147483648ll; return -sum; },
      [&](int c) { return -(int64_t)cands[c].second.size(); },
      [&](int c) {  // GetEarliestPodStartTime
        const std::vector<int> &v = cands[c].second;
        int64_t earliest = start(v[0]), maxp = pp(v[0]);
        for (int t : v) {
          if (pp(t) == maxp) { if (start(t) < earliest) earliest = start(t); }
          else if (pp(t) > maxp) { maxp = pp(t); earliest = start(t); }
        }
        return earliest;
      }};
  std::vector<int> all(cands.size());
  for (size_t i = 0; i < all.size(); ++i) all[i] = (int)i;
  for (auto &f : fs) {
    std::vector<int> sel;
    int64_t mx = INT64_MIN;
    for (int c : all) {
      const int64_t sc = f(c);
      if (sc > mx) { mx = sc; sel.clear(); }
      if (sc == mx) sel.push_back(c);
    }
    if (sel.size() == 1) return sel[0];
    all = sel;
  }
  return all[0];
}

// pmpt.preempt -> topologyAwarePreempt, preempt.go:293-327, :475-655
bool topo_preempt_one(Session &s, TopoOpts &o, std::vector<EOp> &stmt, int preemptor, int phase_job) {
  if (s.t_flags[preemptor] & VC_TASK_PREEMPT_NEVER) return false;
  std::vector<int> nodes;
  for (int n = 0; n < s.N; ++n)
    if (preempt_predicate(s, preemptor, n)) nodes.push_back(n);
  if (nodes.empty()) return false;
  const int64_t P = (int64_t)nodes.size();
  const int64_t offset = (int64_t)(splitmix64(o.o.offset_seed + (uint64_t)o.k) % (uint64_t)P);
  o.k += 1;
  int64_t numc = P * o.o.min_candidate_nodes_percentage / 100;
  if (numc < o.o.min_candidate_nodes_absolute) numc = o.o.min_candidate_nodes_absolute;
  if (numc > o.o.max_candidate_nodes_absolute) numc = o.o.max_candidate_nodes_absolute;
  if (numc > P) numc = P;
  if (numc < 0) { o.bad = true; return false; }
  const bool have_state = prop_enabled(s, VC_EN_PREDICATE);  // PrePredicateFn
  std::vector<std::pair<int, std::vector<int>>> cands;
  for (int64_t i = 0; i < P && (int64_t)cands.size() < numc; ++i) {
    const int n = nodes[(size_t)((offset + i) % P)];
    DryRun dr;
    dr.idle.resize(s.R);
    for (int d = 0; d < s.R; ++d) dr.idle[d] = at(s.idle, d, s.N, n);
    dr.have_state = have_state;
    dr.qalloc.resize(s.Q);
    for (int q = 0; q < s.Q; ++q) dr.qalloc[q] = s.qattr[q].allocated;
    std::vector<int> victims;
    if (select_victims_on_node(s, o, dr, preemptor, phase_job, n, victims)) cands.push_back({n, victims});
  }
  if (cands.empty()) return false;
  const int c = cands.size() == 1 ? 0 : pick_one(s, o, cands);
  std::vector<EOp> tmp;
  for (int v : cands[c].second) stmt_evict(s, tmp, v);  // prepareCandidate
  estmt_pipeline(s, tmp, preemptor, cands[c].first);
  stmt.insert(stmt.end(), tmp.begin(), tmp.end());  // stmt.Merge(tmpStmt)
  return true;
}

// Action.Execute, preempt.go:101-283, with the topology-aware preempt (a restatement of preempt_execute's loops)
int topo_preempt_execute(Session &s, TopoOpts &o) {
  s.decisions.clear(); s.visits.clear(); s.fit_errors.clear();
  ensure_running_table(s);
  if (!preempt_supported(s)) return VC_EUNSUPPORTED;
  if (o.o.n_running != s.T - s.T_run0) return VC_EINVAL;
  o.k = 0;
  o.bad = false;
  std::vector<GoHeap> preemptors(s.Q), ptasks(s.J);
  std::vector<std::vector<int>> under_request(s.Q);
  std::vector<uint8_t> has_q(s.Q, 0);
  for (int q = 0; q < s.Q; ++q) preemptors[q].less = [&s](int l, int r) { return job_order_less(s, l, r); };
  for (int j = 0; j < s.J; ++j) ptasks[j].less = [&s](int l, int r) { return task_order_less(s, l, r); };
  for (int j = 0; j < s.J; ++j) {
    if (s.j_flags[j] & VC_JOB_PENDING_PHASE) continue;
    if (!job_valid(s, j)) continue;
    const int q = s.j_queue[j];
    if (q < 0 || !job_starving(s, j)) continue;
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
    while (!preemptors[q].empty()) {
      const int pj = preemptors[q].pop();
      std::vector<EOp> stmt;
      bool assigned = false;
      for (;;) {
        if (!job_starving(s, pj) || ptasks[pj].empty()) break;
        assigned = topo_preempt_one(s, o, stmt, ptasks[pj].pop(), -1);
        if (o.bad) return VC_EINVAL;
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
    for (int j : under_request[q]) {
      GoHeap intra;
      intra.less = [&s](int l, int r) { return task_order_less(s, l, r); };
      for (int t = 0; t < s.T_alloc; ++t)
        if (s.t_job[t] == j && s.t_status[t] == kPending) intra.push(t);
      while (!intra.empty()) {
        std::vector<EOp> stmt;
        const bool assigned = topo_preempt_one(s, o, stmt, intra.pop(), j);
        if (o.bad) return VC_EINVAL;
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

}  // namespace

extern "C" {

int vcot_set_preempt_options(void *h, const vc_preempt_options *opts) {
  TopoOpts &o = g_topo[h];
  o = TopoOpts();
  if (!opts) return VC_OK;
  o.o = *opts;
  if (opts->n_running > 0) {
    o.prio.assign(opts->rt_pod_priority, opts->rt_pod_priority + opts->n_running);
    o.start.assign(opts->rt_start_ns, opts->rt_start_ns + opts->n_running);
  }
  return VC_OK;
}
// the preempt action: the topology-aware reading when the options say so, the oracle's normal one otherwise
int vcot_preempt(void *h) {
  auto it = g_topo.find(h);
  if (it == g_topo.end() || !it->second.o.topology_aware) return preempt_execute(*(Session *)h);
  return topo_preempt_execute(*(Session *)h, it->second);
}
void vcot_forget(void *h) { g_topo.erase(h); }

}  // extern "C"

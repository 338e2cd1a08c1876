// samp_evict_oracle.cpp — test infrastructure: the topology oracle (tools/topo_oracle/topo_oracle.cpp, included
// unchanged; it includes the CPU oracle) plus a plain restatement of the preempt and reclaim actions under feasible-node
// sampling, the determinism contract of include/vcalloc.h (vc_preempt_run). Per preemptor / reclaimer that reaches
// PredicateNodes:
//   1. ssn.FilterOutUnschedulableAndUnresolvableNodesForTask: a task that allocate left a NodesFitErrors entry with node
//      errors scans the nodes passing the static predicate, in NodeList order; any other task scans the NodeList;
//   2. numNodesToFind comes from the length P of that list, the scan visits list[(start + i) % P] and stores
//      (start + processed) % P; an empty list returns early and leaves the index alone;
//   3. the predicate is ssn.PredicateForPreemptAction;
//   4. the 16 workers read as one: predicateNodes are the first numNodesToFind passing nodes in scan order;
//   5. the index is one global of the cycle: allocate -> preempt (both phases) -> reclaim;
//   6. predicateNodes keep scan order: SortNodes' ties, reclaim's walk and the topology-aware offset count in it.
// Sessions without sampling keep the oracle's contract: every node passing the predicate, NodeList order, index untouched.
// The per-task entry kind is recorded by a pass of its own over allocate's fit-error list, and every PredicateNodes call
// is logged (task, P, processed, index after, predicateNodes) for the hand-derived tests.
#include "../topo_oracle/topo_oracle.cpp"

namespace {

struct SampState {
  bool init = false;
  std::vector<uint8_t> node_errors;  // [T] 1: allocate left NodesFitErrors[task] with node errors
  int64_t idx = 0;                   // util.lastProcessedNodeIndex as the evicting actions read it
  std::vector<int32_t> log;          // per call: task, P, processed, index after, len, nodes...
};
std::map<void *, SampState> g_samp;

SampState &samp_state(void *h) {
  SampState &st = g_samp[h];
  if (!st.init) {
    const Session &s = *(Session *)h;
    st.init = true;
    st.node_errors.assign(std::max(s.T, 1), 0);
    st.idx = s.conf.last_processed_node_index >= 0 ? s.conf.last_processed_node_index : s.last_processed_node_index;
  }
  return st;
}

bool sampling(const Session &s) {
  return s.N > 0 && num_feasible_nodes_to_find(s.N, s.conf.percentage_nodes_to_find, s.conf.min_nodes_to_find,
                                               s.conf.min_percentage_nodes_to_find) < s.N;
}
// the library refuses sampling with min-nodes-to-find below 1, where numNodesToFind of a list can be 0
bool refused(const Session &s) { return sampling(s) && s.conf.min_nodes_to_find < 1; }

// allocate's fit-error list, in order: a task is an entry with node errors when its predicate failed on every node;
// job.TaskHasFitErrors skips (an entry without node errors) a task of a named role once its role has an entry
void record_entry_kinds(Session &s, SampState &st) {
  std::vector<uint8_t> role_has_entry(s.r_flags.size(), 0);
  st.node_errors.assign(std::max(s.T, 1), 0);
  for (int t : s.fit_errors) {
    const int r = s.t_role[t];
    const bool skipped = !(s.r_flags[r] & VC_ROLE_EMPTY_NAME) && role_has_entry[r];
    if (!skipped) st.node_errors[t] = 1;
    role_has_entry[r] = 1;
  }
}

// FilterOutUnschedulableAndUnresolvableNodesForTask + ph.PredicateNodes(task, nodes, ssn.PredicateForPreemptAction, ...)
std::vector<int> evict_predicate_nodes(Session &s, SampState &st, int t) {
  std::vector<int> out;
  if (!sampling(s)) {
    for (int n = 0; n < s.N; ++n)
      if (preempt_predicate(s, t, n)) out.push_back(n);
    return out;
  }
  std::vector<int> nodes;
  for (int n = 0; n < s.N; ++n)
    if (!st.node_errors[t] || preempt_predicate(s, t, n)) nodes.push_back(n);
  const int64_t P = (int64_t)nodes.size();
  int64_t processed = 0;
  if (P > 0) {
    const int64_t to_find = num_feasible_nodes_to_find((int32_t)P, s.conf.percentage_nodes_to_find,
                                                       s.conf.min_nodes_to_find, s.conf.min_percentage_nodes_to_find);
    const int64_t start = st.idx;
    for (int64_t i = 0; i < P && (int64_t)out.size() < to_find; ++i) {
      const int n = nodes[(size_t)((start + i) % P)];
      processed += 1;
      if (preempt_predicate(s, t, n)) out.push_back(n);
    }
    st.idx = (start + processed) % P;
    s.last_processed_node_index = st.idx;
  }
  st.log.push_back(t);
  st.log.push_back((int32_t)P);
  st.log.push_back((int32_t)processed);
  st.log.push_back((int32_t)st.idx);
  st.log.push_back((int32_t)out.size());
  st.log.insert(st.log.end(), out.begin(), out.end());
  return out;
}

// pmpt.preempt -> normalPreempt, preempt.go:285-434, on predicateNodes in scan order
bool samp_preempt_one(Session &s, SampState &st, std::vector<EOp> &stmt, int preemptor, int phase_job) {
  if (s.t_flags[preemptor] & VC_TASK_PREEMPT_NEVER) return false;  // taskEligibleToPreempt: before PredicateNodes
  const int pj = s.t_job[preemptor], q = s.j_queue[pj];
  const std::vector<int> nodes = evict_predicate_nodes(s, st, preemptor);
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
      if (!preemptable_status(s, t) || !rt_flag(s, t, VC_RT_PREEMPTABLE)) continue;
      const int j = s.t_job[t];
      if (phase_job < 0) {
        if (j < 0 || !(s.j_queue[j] == q && j != pj)) continue;
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
      stmt.insert(stmt.end(), node_stmt.begin(), node_stmt.end());
      return true;
    }
    estmt_discard(s, node_stmt);
  }
  return false;
}

// pmpt.preempt -> topologyAwarePreempt, preempt.go:293-327, :475-655, on predicateNodes in scan order
bool samp_topo_preempt_one(Session &s, SampState &st, TopoOpts &o, std::vector<EOp> &stmt, int preemptor, int phase_job) {
  if (s.t_flags[preemptor] & VC_TASK_PREEMPT_NEVER) return false;
  const std::vector<int> nodes = evict_predicate_nodes(s, st, preemptor);
  if (nodes.empty()) return false;
  const int64_t P = (int64_t)nodes.size();
  const int64_t offset = (int64_t)(splitmix64(o.o.offset_seed + (uint64_t)o.k) % (uint64_t)P);
  o.k += 1;
  int64_t numc = P * o.o.min_candidate_nodes_percentage / 100;
  if (numc < o.o.min_candidate_nodes_absolute) numc = o.o.min_candidate_nodes_absolute;
  if (numc > o.o.max_candidate_nodes_absolute) numc = o.o.max_candidate_nodes_absolute;
  if (numc > P) numc = P;
  if (numc < 0) { o.bad = true; return false; }
  const bool have_state = prop_enabled(s, VC_EN_PREDICATE);
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
  for (int v : cands[c].second) stmt_evict(s, tmp, v);
  estmt_pipeline(s, tmp, preemptor, cands[c].first);
  stmt.insert(stmt.end(), tmp.begin(), tmp.end());
  return true;
}

// Action.Execute of preempt, preempt.go:101-283
int samp_preempt_execute(Session &s, SampState &st, TopoOpts *o) {
  s.decisions.clear(); s.visits.clear(); s.fit_errors.clear();
  ensure_running_table(s);
  if (!preempt_supported(s) || refused(s)) return VC_EUNSUPPORTED;
  const bool topo = o && o->o.topology_aware;
  if (topo) {
    if (o->o.n_running != s.T - s.T_run0) return VC_EINVAL;
    o->k = 0;
    o->bad = false;
  }
  auto try_one = [&](std::vector<EOp> &stmt, int t, int phase_job) {
    return topo ? samp_topo_preempt_one(s, st, *o, stmt, t, phase_job) : samp_preempt_one(s, st, stmt, t, phase_job);
  };
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
    while (!preemptors[q].empty()) {  // between jobs within the queue
      const int pj = preemptors[q].pop();
      std::vector<EOp> stmt;
      bool assigned = false;
      for (;;) {
        if (!job_starving(s, pj) || ptasks[pj].empty()) break;
        assigned = try_one(stmt, ptasks[pj].pop(), -1);
        if (topo && o->bad) return VC_EINVAL;
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
    for (int j : under_request[q]) {  // between tasks within a job
      GoHeap intra;
      intra.less = [&s](int l, int r) { return task_order_less(s, l, r); };
      for (int t = 0; t < s.T_alloc; ++t)
        if (s.t_job[t] == j && s.t_status[t] == kPending) intra.push(t);
      while (!intra.empty()) {
        std::vector<EOp> stmt;
        const bool assigned = try_one(stmt, intra.pop(), j);
        if (topo && o->bad) return VC_EINVAL;
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

// ra.reclaimForTask, reclaim.go:170-258: predicateNodes walked as they come (scan order)
void samp_reclaim_for_task(Session &s, SampState &st, std::vector<EOp> &stmt, int task, int job) {
  const int jq = s.j_queue[job];
  for (int n : evict_predicate_nodes(s, st, task)) {
    std::vector<int> reclaimees;
    for (int t : s.node_tasks[n]) {
      if (s.t_status[t] != kRunning || !rt_flag(s, t, VC_RT_PREEMPTABLE)) continue;
      const int j = s.t_job[t];
      if (j < 0 || s.j_queue[j] == jq) continue;
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

// Action.Execute of reclaim, reclaim.go:56-168
int samp_reclaim_execute(Session &s, SampState &st) {
  s.decisions.clear(); s.visits.clear(); s.fit_errors.clear();
  ensure_running_table(s);
  if (!preempt_supported(s) || refused(s)) return VC_EUNSUPPORTED;
  GoHeap queues;
  queues.less = [&s](int l, int r) { return queue_order_less(s, l, r); };
  std::vector<uint8_t> q_seen(s.Q, 0), has_pre(s.Q, 0);
  std::vector<GoHeap> preemptors(s.Q), ptasks(s.J);
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
        if (!job_starving(s, job) || ptasks[job].empty()) break;
        const int task = ptasks[job].pop();
        if (s.t_flags[task] & VC_TASK_PREEMPT_NEVER) continue;  // before PredicateNodes: the index stays
        if (!preemptive(s, q, task)) continue;
        samp_reclaim_for_task(s, st, stmt, task, job);
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

}  // namespace

extern "C" {

// allocate, then the entry kinds of its fit-error list; the index it leaves is the one preempt starts from
int vcse_allocate(void *h) {
  Session &s = *(Session *)h;
  SampState &st = samp_state(h);
  const int rc = allocate_execute(s);
  if (rc) return rc;
  record_entry_kinds(s, st);
  st.idx = s.last_processed_node_index;
  return VC_OK;
}
// the preempt action: the topology-aware reading when vcot_set_preempt_options asked for it
int vcse_preempt(void *h) {
  auto it = g_topo.find(h);
  return samp_preempt_execute(*(Session *)h, samp_state(h), it == g_topo.end() ? nullptr : &it->second);
}
int vcse_reclaim(void *h) { return samp_reclaim_execute(*(Session *)h, samp_state(h)); }
int64_t vcse_index(void *h) { return samp_state(h).idx; }
void vcse_node_errors(void *h, uint8_t *out) {  // [T] of vc_tasks (the running tasks the session appends have none)
  const SampState &st = samp_state(h);
  std::copy(st.node_errors.begin(), st.node_errors.begin() + ((Session *)h)->T_alloc, out);
}
// the PredicateNodes log: returns its length; copies at most `cap` ints
int64_t vcse_calls(void *h, int32_t *out, int64_t cap) {
  const SampState &st = samp_state(h);
  for (int64_t i = 0; i < cap && i < (int64_t)st.log.size(); ++i) out[i] = st.log[(size_t)i];
  return (int64_t)st.log.size();
}
void vcse_forget(void *h) { g_samp.erase(h); g_topo.erase(h); }

}  // extern "C"

// nta_evict_oracle.cpp — test infrastructure: the guard oracle (tools/guard_oracle/guard_oracle.cpp, included unchanged;
// it includes the sampling, topology and CPU oracles) with preempt and reclaim opened to the network-topology-aware
// plugin and to soft-mode topology jobs:
//   - preempt's preemptor collection skips every job with a network topology (preempt.go:132-137), in both phases
//     (underRequestByQueue is filled in the same loop) and both readings; reclaim has no such skip (reclaim.go:56-168);
//   - the plugin's node score, its AllocateFunc / DeallocateFunc and hyperNodeResourceCache are the CPU oracle's own:
//     util.PrioritizeNodes adds nta_node_score for a preemptor of a job without a topology, and every Statement Evict,
//     Pipeline and Discard goes through on_allocate_event / on_deallocate_event, which call nta_account;
//   - the tdm plugin, hard-mode and subGroupPolicy jobs and BestEffort pending tasks stay refused.
// Everything else (both readings of preempt, sampling, pdb / cdp votes) is the guard oracle's code.
#include "../guard_oracle/guard_oracle.cpp"

namespace {

// preempt_supported without the network-topology-aware refusal
bool nta_evict_supported(const Session &s) {
  if (s.T_run0 >= 0 && s.T_run0 != s.T_alloc) return false;  // BestEffort pending tasks in the session
  for (int j = 0; j < s.J; ++j)
    if (s.j_flags[j] & VC_JOB_UNSUPPORTED) return false;
  return !s.has_plugin[VC_PLUGIN_TDM];
}

// Action.Execute of preempt, preempt.go:101-283 (g_preempt_execute with the topology skip)
int n_preempt_execute(Session &s, SampState &st, TopoOpts *o, const Guards &g) {
  s.decisions.clear(); s.visits.clear(); s.fit_errors.clear();
  ensure_running_table(s);
  if (!nta_evict_supported(s) || refused(s)) return VC_EUNSUPPORTED;
  const bool topo = o && o->o.topology_aware;
  if (topo) {
    if (o->o.n_running != s.T - s.T_run0) return VC_EINVAL;
    o->k = 0;
    o->bad = false;
  }
  auto try_one = [&](std::vector<EOp> &stmt, int t, int phase_job) {
    return topo ? g_topo_preempt_one(s, st, *o, g, stmt, t, phase_job) : g_preempt_one(s, st, g, stmt, t, phase_job);
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
    if (s.job_soft[j]) continue;  // job.ContainsNetworkTopology()
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
    for (int j : under_request[q]) {
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

// Action.Execute of reclaim, reclaim.go:56-168 (g_reclaim_execute; soft-mode topology jobs reclaim like any other)
int n_reclaim_execute(Session &s, SampState &st, const Guards &g) {
  s.decisions.clear(); s.visits.clear(); s.fit_errors.clear();
  ensure_running_table(s);
  if (!nta_evict_supported(s) || refused(s)) return VC_EUNSUPPORTED;
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
        if (s.t_flags[task] & VC_TASK_PREEMPT_NEVER) continue;
        if (!preemptive(s, q, task)) continue;
        g_reclaim_for_task(s, st, g, stmt, task, job);
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

int vcnta_preempt(void *h) {
  Session &s = *(Session *)h;
  const Guards &g = g_guards[h];
  if (votes(s, VC_EN_PREEMPTABLE) && !g.set) return VC_EINVAL;
  auto it = g_topo.find(h);
  return n_preempt_execute(s, samp_state(h), it == g_topo.end() ? nullptr : &it->second, g);
}
int vcnta_reclaim(void *h) {
  Session &s = *(Session *)h;
  const Guards &g = g_guards[h];
  if (votes(s, VC_EN_RECLAIMABLE) && !g.set) return VC_EINVAL;
  return n_reclaim_execute(s, samp_state(h), g);
}

}  // extern "C"

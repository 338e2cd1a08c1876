// guard_oracle.cpp — test infrastructure: the sampling oracle (tools/samp_evict_oracle/samp_evict_oracle.cpp, included
// unchanged; it includes the topology oracle and the CPU oracle) plus a plain restatement of the victim votes of the pdb
// and cdp plugins and of the preempt / reclaim loops that call ssn.Preemptable / ssn.Reclaimable with them:
//   pdb (plugins/pdb/pdb.go:65-126): per call, a budget per PDB starting at DisruptionsAllowed, kept in a map; the
//     preemptees in list order; a pod without labels is skipped (never returned); every PDB that counts a pod loses one,
//     and the pod is returned unless one of them went below zero;
//   cdp (plugins/cdp/cdp.go:56-110): a pod is kept while its cooldown end is after now.
// The tier rule (intersection, an empty answer voids the tier) is restated here; the other plugins' votes are the
// oracle's. Covers the normal and topology-aware readings of preempt and reclaim, with and without sampling.
#include "../samp_evict_oracle/samp_evict_oracle.cpp"

namespace {

struct Guards {  // vc_victim_guards, indexed by running task (oracle task t = T_run0 + r)
  bool set = false;
  std::vector<int32_t> allowed, off, pdb;
  std::vector<uint32_t> flags;
  std::vector<int64_t> until;
  int64_t now = 0;
};
std::map<void *, Guards> g_guards;

std::vector<int> pdb_vote(const Session &s, const Guards &g, const std::vector<int> &preemptees) {
  std::map<int, int> budget;  // PDB -> what is left of DisruptionsAllowed in this call, entered when first met
  std::vector<int> victims;
  for (int t : preemptees) {
    const int r = t - s.T_run0;
    if (g.flags[r] & VC_GUARD_NO_LABELS) continue;
    bool violated = false;
    for (int x = g.off[r]; x < g.off[r + 1]; ++x) {
      auto it = budget.emplace(g.pdb[x], g.allowed[g.pdb[x]]).first;
      it->second -= 1;
      if (it->second < 0) violated = true;
    }
    if (!violated) victims.push_back(t);
  }
  return victims;
}

std::vector<int> cdp_vote(const Session &s, const Guards &g, const std::vector<int> &preemptees) {
  std::vector<int> victims;
  for (int t : preemptees) {
    const int64_t until = g.until[t - s.T_run0];
    const bool protect = until != VC_COOLDOWN_NONE && until > g.now;
    if (!protect) victims.push_back(t);
  }
  return victims;
}

// ssn.Preemptable / ssn.Reclaimable, framework/session_plugins.go:211-307, with pdb and cdp among the voters
std::vector<int> guarded_victims(const Session &s, const Guards &g, int preemptor, const std::vector<int> &cands,
                                 bool reclaim) {
  std::vector<int> victims;
  bool nil = true;
  int i = 0;
  while (i < s.conf.n_plugins) {
    const int tier = s.conf.plugins[i].tier;
    for (int k = i; k < s.conf.n_plugins && s.conf.plugins[k].tier == tier; ++k) {
      const vc_plugin_option &p = s.conf.plugins[k];
      if (!(p.enabled & (reclaim ? VC_EN_RECLAIMABLE : VC_EN_PREEMPTABLE))) continue;
      std::vector<int> c;
      if (p.plugin == VC_PLUGIN_GANG) c = gang_victims(s, cands);
      else if (p.plugin == VC_PLUGIN_CONFORMANCE) c = conformance_victims(s, cands);
      else if (p.plugin == VC_PLUGIN_PRIORITY && !reclaim) c = priority_victims(s, preemptor, cands);
      else if (p.plugin == VC_PLUGIN_DRF && !reclaim) c = drf_victims(s, preemptor, cands);
      else if (p.plugin == VC_PLUGIN_PROPORTION && reclaim) c = proportion_victims(s, cands);
      else if (p.plugin == VC_PLUGIN_PDB) c = pdb_vote(s, g, cands);
      else if (p.plugin == VC_PLUGIN_CDP) c = cdp_vote(s, g, cands);
      else continue;
      if (c.empty()) { victims.clear(); nil = true; break; }
      if (nil) { victims = c; nil = false; continue; }
      std::vector<int> inter;
      for (int v : victims)
        if (std::find(c.begin(), c.end(), v) != c.end()) inter.push_back(v);
      victims = inter;
      nil = inter.empty();
    }
    while (i < s.conf.n_plugins && s.conf.plugins[i].tier == tier) ++i;
    if (!nil) return victims;
  }
  return victims;
}

// the preemptees of node n under the action's filter (preempt.go:198-214 / :252-268)
std::vector<int> preemptees_of(const Session &s, int preemptor, int phase_job, int n) {
  const int pj = s.t_job[preemptor], q = s.j_queue[pj];
  std::vector<int> out;
  for (int t : s.node_tasks[n]) {
    if (!preemptable_status(s, t) || !rt_flag(s, t, VC_RT_PREEMPTABLE)) continue;
    const int j = s.t_job[t];
    if (phase_job < 0) {
      if (j < 0 || !(s.j_queue[j] == q && j != pj)) continue;
    } else if (j != pj) {
      continue;
    }
    out.push_back(t);
  }
  return out;
}

// normalPreempt, preempt.go:333-434, on predicateNodes in scan order
bool g_preempt_one(Session &s, SampState &st, const Guards &g, std::vector<EOp> &stmt, int preemptor, int phase_job) {
  if (s.t_flags[preemptor] & VC_TASK_PREEMPT_NEVER) return false;
  const int q = s.j_queue[s.t_job[preemptor]];
  const std::vector<int> nodes = evict_predicate_nodes(s, st, preemptor);
  if (nodes.empty()) return false;
  std::vector<double> scores;
  double bs;
  s.task_alloc_hn = -1;
  prioritize_and_select(s, preemptor, nodes, &bs, &scores);
  std::vector<int> order(nodes.size());
  for (size_t i = 0; i < order.size(); ++i) order[i] = (int)i;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return scores[a] > scores[b]; });
  for (int oi : order) {
    const int n = nodes[oi];
    std::vector<int> victims = guarded_victims(s, g, preemptor, preemptees_of(s, preemptor, phase_job, n), false);
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

// SelectVictimsOnNode, preempt.go:708-842, on clones of the node and of proportion's queue state
bool g_select_victims(Session &s, const Guards &g, DryRun &dr, int preemptor, int phase_job, int n,
                      std::vector<int> &victims) {
  const int q = s.j_queue[s.t_job[preemptor]];
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
  const std::vector<int> all = guarded_victims(s, g, preemptor, preemptees_of(s, preemptor, phase_job, n), false);
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

// topologyAwarePreempt, preempt.go:475-655, on predicateNodes in scan order
bool g_topo_preempt_one(Session &s, SampState &st, TopoOpts &o, const Guards &g, std::vector<EOp> &stmt, int preemptor,
                        int phase_job) {
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
  std::vector<std::pair<int, std::vector<int>>> cands;
  for (int64_t i = 0; i < P && (int64_t)cands.size() < numc; ++i) {
    const int n = nodes[(size_t)((offset + i) % P)];
    DryRun dr;
    dr.idle.resize(s.R);
    for (int d = 0; d < s.R; ++d) dr.idle[d] = at(s.idle, d, s.N, n);
    dr.have_state = prop_enabled(s, VC_EN_PREDICATE);
    dr.qalloc.resize(s.Q);
    for (int x = 0; x < s.Q; ++x) dr.qalloc[x] = s.qattr[x].allocated;
    std::vector<int> victims;
    if (g_select_victims(s, g, dr, preemptor, phase_job, n, victims)) cands.push_back({n, victims});
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
int g_preempt_execute(Session &s, SampState &st, TopoOpts *o, const Guards &g) {
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

// ra.reclaimForTask, reclaim.go:170-258
void g_reclaim_for_task(Session &s, SampState &st, const Guards &g, std::vector<EOp> &stmt, int task, int job) {
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
    std::vector<int> victims = guarded_victims(s, g, task, reclaimees, true);
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
int g_reclaim_execute(Session &s, SampState &st, const Guards &g) {
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

bool votes(const Session &s, uint32_t flag) {
  for (int i = 0; i < s.conf.n_plugins; ++i)
    if ((s.conf.plugins[i].plugin == VC_PLUGIN_PDB || s.conf.plugins[i].plugin == VC_PLUGIN_CDP) &&
        (s.conf.plugins[i].enabled & flag))
      return true;
  return false;
}

}  // namespace

extern "C" {

// the table of vc_victim_guards (NULL clears it); the pointers are copied
int vcgo_set_victim_guards(void *h, const vc_victim_guards *vg) {
  Guards &g = g_guards[h];
  g = Guards();
  if (!vg) return VC_OK;
  g.set = true;
  g.now = vg->now_ns;
  g.allowed.assign(vg->pdb_allowed, vg->pdb_allowed + vg->n_pdb);
  g.off.assign(vg->rt_pdb_off, vg->rt_pdb_off + vg->n_running + 1);
  g.pdb.assign(vg->rt_pdb, vg->rt_pdb + g.off.back());
  g.flags.assign(vg->rt_flags, vg->rt_flags + vg->n_running);
  g.until.assign(vg->rt_cooldown_until_ns, vg->rt_cooldown_until_ns + vg->n_running);
  return VC_OK;
}
int vcgo_preempt(void *h) {
  Session &s = *(Session *)h;
  const Guards &g = g_guards[h];
  if (votes(s, VC_EN_PREEMPTABLE) && !g.set) return VC_EINVAL;
  auto it = g_topo.find(h);
  return g_preempt_execute(s, samp_state(h), it == g_topo.end() ? nullptr : &it->second, g);
}
int vcgo_reclaim(void *h) {
  Session &s = *(Session *)h;
  const Guards &g = g_guards[h];
  if (votes(s, VC_EN_RECLAIMABLE) && !g.set) return VC_EINVAL;
  return g_reclaim_execute(s, samp_state(h), g);
}
// the votes of one plugin on the running tasks `cands` (oracle order), for the plugin tests: out[i] = 1 when returned
int vcgo_vote(void *h, int plugin, const int32_t *rt, int m, uint8_t *out) {
  Session &s = *(Session *)h;
  ensure_running_table(s);
  const Guards &g = g_guards[h];
  std::vector<int> c;
  for (int i = 0; i < m; ++i) c.push_back(s.T_run0 + rt[i]);
  const std::vector<int> v = plugin == VC_PLUGIN_PDB ? pdb_vote(s, g, c) : cdp_vote(s, g, c);
  for (int i = 0; i < m; ++i) out[i] = std::find(v.begin(), v.end(), c[(size_t)i]) != v.end() ? 1 : 0;
  return (int)v.size();
}
void vcgo_forget(void *h) { g_guards.erase(h); vcse_forget(h); }

}  // extern "C"

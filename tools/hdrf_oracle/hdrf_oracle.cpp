// hdrf_oracle.cpp — test infrastructure: the CPU oracle (oracle/oracle.cpp, included unchanged) plus a plain restatement
// of hierarchical drf (plugins/drf/drf.go:45-184,458-560) and of the allocate action with its queue PQ ordered by it.
//
// Independent of the library's lazy scheme (vc_hdrf.hpp): the tree is a map-like structure of named nodes built by
// buildHierarchy for every job, and updateHierarchicalShare runs over the WHOLE tree, recursively, before every queue-heap
// operation — i.e. the tree every comparison reads is what the reference's event handlers left after the last Allocate /
// Deallocate event. Canonical choices of the determinism contract: children in first-insertion order, jobs inserted in
// index order, queues pushed in the order they first appear over the jobs.
#include "../../oracle/oracle.cpp"

#include <algorithm>
#include <map>
#include <memory>
#include <string>

namespace {

struct HNode {
  HNode *parent = nullptr;
  double weight = 1;
  bool saturated = false;
  bool leaf = false;
  int job = -1;
  double share = 0;
  std::vector<double> allocated, request;
  std::vector<HNode *> order;  // the children in first-insertion order (the map's canonical iteration order)
  std::map<std::string, std::unique_ptr<HNode>> children;
};

struct Hdrf {
  int Q = 0;
  std::vector<std::vector<std::string>> paths;  // per queue: strings.Split(Hierarchy, "/")
  std::vector<std::vector<double>> weights;     // per queue: the ParseFloat values of strings.Split(Weights, "/")
  std::vector<double> job_request;              // [R][J]
  HNode root;
};
std::map<void *, Hdrf> g_hdrf;

double share_of_vec(const Session &s, const std::vector<double> &a) {  // drf.calculateShare
  double res = 0;
  for (int d = 0; d < s.R; ++d) {
    if (d >= 2 && !(s.total.has & (1u << d))) continue;
    if (!(s.total.v[d] >= kMinResource)) continue;
    const double sh = share_of(a[d], s.total.v[d]);
    if (sh > res) res = sh;
  }
  return res;
}
// buildHierarchy, drf.go:458-500 (the job's leaf is replaced by a fresh one, same key)
void build_hierarchy(const Session &s, Hdrf &h, int j) {
  const int q = s.j_queue[j];
  HNode *inode = &h.root;
  const std::vector<std::string> &paths = h.paths[q];
  for (size_t i = 1; i < paths.size(); ++i) {
    auto it = inode->children.find(paths[i]);
    if (it != inode->children.end()) { inode = it->second.get(); continue; }
    double fweight = h.weights[q].at(i);  // the reference indexes weights[i]; a short string is refused at attach
    if (fweight < 1) fweight = 1;
    auto child = std::make_unique<HNode>();
    child->weight = fweight;
    child->parent = inode;
    child->allocated.assign(s.R, 0.0);
    HNode *c = child.get();
    inode->order.push_back(c);
    inode->children[paths[i]] = std::move(child);
    inode = c;
  }
  const std::string key = "\x01job" + std::to_string(j);
  auto leaf = std::make_unique<HNode>();
  leaf->leaf = true;
  leaf->job = j;
  leaf->parent = inode;
  leaf->request.assign(s.R, 0.0);
  for (int d = 0; d < s.R; ++d) leaf->request[d] = h.job_request[(size_t)d * s.J + j];
  auto old = inode->children.find(key);
  if (old == inode->children.end()) inode->order.push_back(leaf.get());
  else std::replace(inode->order.begin(), inode->order.end(), old->second.get(), leaf.get());
  inode->children[key] = std::move(leaf);
}
// updateHierarchicalShare, drf.go:503-548; a leaf's attr is the job's drf attr
void update_share(const Session &s, HNode &node, const std::vector<bool> &demanding) {
  if (node.leaf) {
    node.allocated.assign(s.R, 0.0);
    for (int d = 0; d < s.R; ++d) node.allocated[d] = at(s.j_alloc, d, s.J, node.job);
    node.share = s.j_share[node.job];
    node.saturated = false;  // resourceSaturated, drf.go:83-95
    for (int d = 0; d < s.R; ++d) {
      if (!(node.allocated[d] >= kMinResource)) continue;
      if (node.allocated[d] != 0 && node.request[d] != 0 && node.allocated[d] >= node.request[d]) node.saturated = true;
      if (!demanding[d] && node.request[d] != 0) node.saturated = true;
    }
    return;
  }
  double mdr = 1;
  for (HNode *cp : node.order) {
    HNode &c = *cp;
    update_share(s, c, demanding);
    if (c.share != 0 && !c.saturated) {
      const double rs = share_of_vec(s, c.allocated);
      if (rs < mdr) mdr = rs;
    }
  }
  node.allocated.assign(s.R, 0.0);
  bool saturated = true;
  for (HNode *cp : node.order) {
    HNode &c = *cp;
    if (!c.saturated) saturated = false;
    if (c.share == 0) continue;
    if (c.saturated) {
      for (int d = 0; d < s.R; ++d) node.allocated[d] += c.allocated[d];
    } else {
      const double ratio = mdr / c.share;
      for (int d = 0; d < s.R; ++d) node.allocated[d] += c.allocated[d] * ratio;
    }
  }
  node.share = share_of_vec(s, node.allocated);
  node.saturated = saturated;
}
// UpdateHierarchicalShare, drf.go:550-560: totalAllocated = sum of the jobs' drf allocations
void update_tree(const Session &s, Hdrf &h) {
  std::vector<bool> demanding(s.R, false);
  for (int d = 0; d < s.R; ++d) {
    if (d >= 2 && !(s.total.has & (1u << d))) continue;
    if (!(s.total.v[d] >= kMinResource)) continue;
    double tot = 0;
    for (int j = 0; j < s.J; ++j) tot += at(s.j_alloc, d, s.J, j);
    demanding[d] = tot < s.total.v[d];
  }
  update_share(s, h.root, demanding);
}
// compareQueues, drf.go:160-184
double compare_queues(Hdrf &h, int l, int r) {
  HNode *ln = &h.root, *rn = &h.root;
  const std::vector<std::string> &lp = h.paths[l], &rp = h.paths[r];
  const size_t depth = std::min(lp.size(), rp.size());
  for (size_t i = 0; i < depth; ++i) {
    if (!ln->saturated && rn->saturated) return -1;
    if (ln->saturated && !rn->saturated) return 1;
    if (ln->share / ln->weight == rn->share / rn->weight) {
      if (i < depth - 1) {
        ln = ln->children.at(lp[i + 1]).get();
        rn = rn->children.at(rp[i + 1]).get();
      }
    } else {
      return ln->share / ln->weight - rn->share / rn->weight;
    }
  }
  return 0;
}
// ssn.QueueOrderFn with hdrf's queueOrderFn registered (drf.go:265-278) in the tier chain
bool hdrf_queue_less(const Session &s, Hdrf &h, int l, int r) {
  for (int i = 0; i < s.conf.n_plugins; ++i) {
    const vc_plugin_option &p = s.conf.plugins[i];
    if (!(p.enabled & VC_EN_QUEUE_ORDER)) continue;
    if (p.plugin == VC_PLUGIN_DRF) {
      const double ret = compare_queues(h, l, r);
      if (ret < 0) return true;
      if (ret > 0) return false;
    }
    if (p.plugin == VC_PLUGIN_PROPORTION) {
      if (s.q_prio[l] != s.q_prio[r]) return (s.q_prio[r] - s.q_prio[l]) < 0;
      const double ls = s.qattr[l].share, rs = s.qattr[r].share;
      if (ls != rs) return ls < rs;
    }
  }
  if (s.q_ts[l] == s.q_ts[r]) return s.q_uid[l] < s.q_uid[r];
  return s.q_ts[l] < s.q_ts[r];
}

// allocate_execute (oracle.cpp) with the queue PQ under hdrf: the tree is brought up to date before every Push / Pop
// argmin = true: the same loop with queues.Pop() replaced by an arg-min over the live keys of the queues in the heap —
// NOT the reference; it exists to show where the heap layout changes the result
int hdrf_allocate_execute(Session &s, Hdrf &h, bool argmin) {
  for (int j = 0; j < s.J; ++j)
    if (s.j_flags[j] & VC_JOB_UNSUPPORTED) return VC_EUNSUPPORTED;
  std::vector<GoHeap> task_pq(s.J);
  for (int j = 0; j < s.J; ++j) task_pq[j].less = [&s](int l, int r) { return task_order_less(s, l, r); };
  for (int t = 0; t < s.T_alloc; ++t) task_pq[s.t_job[t]].push(t);
  GoHeap queues;
  queues.less = [&s, &h](int l, int r) { return hdrf_queue_less(s, h, l, r); };
  std::vector<GoHeap> jobs_by_queue(s.Q);
  std::vector<uint8_t> queue_seen(s.Q, 0);
  for (int q = 0; q < s.Q; ++q) jobs_by_queue[q].less = [&s](int l, int r) { return job_order_less(s, l, r); };
  update_tree(s, h);
  for (int j = 0; j < s.J; ++j) {
    if (s.j_flags[j] & VC_JOB_PENDING_PHASE) {
      if (s.conf.enqueue_action_enabled) continue;
      s.j_flags[j] &= ~VC_JOB_PENDING_PHASE;
    }
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
  std::vector<Op> ops;
  while (!queues.empty()) {
    update_tree(s, h);
    int q;
    if (argmin) {
      size_t b = 0;
      for (size_t k = 1; k < queues.items.size(); ++k)
        if (hdrf_queue_less(s, h, queues.items[k], queues.items[b])) b = k;
      q = queues.items[b];
      queues.items.erase(queues.items.begin() + b);
    } else {
      q = queues.pop();
    }
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
        dcs.task = op.task; dcs.node = op.node; dcs.kind = op.kind;
        dcs.visit = (int32_t)s.visits.size(); dcs.score = op.score;
        s.decisions.push_back(dcs);
      }
      if (ready) {
        stmt_commit(s, ops);
        if (task_pq[j].size() > 0) jobs.push(j);
      }
    }
    s.visits.push_back(v);
    update_tree(s, h);
    queues.push(q);
  }
  return VC_OK;
}

// pickUpPendingTasks (backfill.go:118-199) with the queue PQ under hdrf, on the tree the preceding actions left
std::vector<int> hdrf_backfill_pick(Session &s, Hdrf &h) {
  update_tree(s, h);
  std::vector<GoHeap> task_pq(s.J);
  for (int j = 0; j < s.J; ++j) task_pq[j].less = [&s](int l, int r) { return task_order_less(s, l, r); };
  for (int t = s.T_alloc; t < s.T; ++t)
    if (s.t_status[t] == kPending) task_pq[s.t_job[t]].push(t);
  GoHeap queues;
  queues.less = [&s, &h](int l, int r) { return hdrf_queue_less(s, h, l, r); };
  std::vector<GoHeap> jobs_by_queue(s.Q);
  std::vector<uint8_t> queue_seen(s.Q, 0);
  for (int q = 0; q < s.Q; ++q) jobs_by_queue[q].less = [&s](int l, int r) { return job_order_less(s, l, r); };
  for (int j = 0; j < s.J; ++j) {
    if (s.j_flags[j] & VC_JOB_PENDING_PHASE) continue;
    if (!job_valid(s, j)) continue;
    int q = s.j_queue[j];
    if (q < 0 || task_pq[j].empty()) continue;
    if (!queue_seen[q]) { queue_seen[q] = 1; queues.push(q); }
    jobs_by_queue[q].push(j);
  }
  std::vector<int> pending;
  while (!queues.empty()) {
    int q = queues.pop();
    while (!jobs_by_queue[q].empty()) {
      int j = jobs_by_queue[q].pop();
      while (!task_pq[j].empty()) pending.push_back(task_pq[j].pop());
    }
  }
  return pending;
}
// backfill_execute (oracle.cpp) with that pick order; the rest is the same statement by statement
int hdrf_backfill_execute(Session &s, Hdrf &h) {
  s.decisions.clear(); s.visits.clear(); s.fit_errors.clear();
  if (s.T == s.T_alloc) return VC_OK;
  for (int j = 0; j < s.J; ++j)
    if (s.j_flags[j] & VC_JOB_UNSUPPORTED) return VC_EUNSUPPORTED;
  const int32_t to_find = num_feasible_nodes_to_find(s.N, s.conf.percentage_nodes_to_find, s.conf.min_nodes_to_find,
                                                     s.conf.min_percentage_nodes_to_find);
  std::vector<int> pending = hdrf_backfill_pick(s, h);
  std::vector<int> feasible;
  int cur_job = -1;
  for (int t : pending) {
    const int j = s.t_job[t], r = s.t_role[t];
    if (j != cur_job) {
      vc_visit v;
      v.job = j; v.first_op = (int32_t)s.decisions.size(); v.n_ops = 0;
      v.outcome = job_ready(s, j) ? VC_VISIT_COMMIT : VC_VISIT_KEEP;
      s.visits.push_back(v);
      cur_job = j;
    }
    feasible.clear();
    s.sweeps++;
    if (to_find < s.N) {
      const int start = (int)s.last_processed_node_index;
      int processed = 0;
      for (int i = 0; i < s.N && (int)feasible.size() < to_find; ++i) {
        const int n = (start + i) % s.N;
        processed++;
        if (plugin_predicates(s, t, n)) feasible.push_back(n);
      }
      s.last_processed_node_index = (start + processed) % s.N;
    } else {
      for (int n = 0; n < s.N; ++n)
        if (plugin_predicates(s, t, n)) feasible.push_back(n);
    }
    if (feasible.empty()) {
      s.fit_errors.push_back(t - s.T_alloc);
      continue;
    }
    int node = feasible[0];
    double score = 0.0;
    if (feasible.size() > 1) {
      s.task_alloc_hn = -1;
      double sc = 0.0;
      int best = prioritize_and_select(s, t, feasible, &sc, nullptr);
      if (best >= 0) { node = best; score = sc; }
    }
    s.t_status[t] = kAllocated;
    s.r_pending[r] -= 1;
    s.j_pbe[j] -= 1;
    s.j_ready[j] += 1;
    s.t_node[t] = node;
    for (int d = 0; d < s.R; ++d) {
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
    if (job_ready(s, j))
      for (int u = 0; u < s.T; ++u)
        if (s.t_job[u] == j && s.t_status[u] == kAllocated) s.t_status[u] = kBinding;
  }
  return VC_OK;
}

HNode *node_of(Hdrf &h, int q, int level) {
  HNode *n = &h.root;
  for (int i = 1; i <= level; ++i) {
    auto it = n->children.find(h.paths[q].at(i));
    if (it == n->children.end()) return nullptr;
    n = it->second.get();
  }
  return n;
}

}  // namespace

extern "C" {

// drf with enableHierarchy on an oracle session: hierarchy / weights as the annotation strings ("\n"-separated per
// queue) and the ParseFloat values of the weights (`wvals`, laid out per queue by n_weight_segments incl. the first).
// Returns VC_EINVAL for the inputs the reference crashes on (a job outside ssn.Queues, a weights string shorter than
// the path of a queue that has jobs).
int vcoh_attach(void *hp, const char *hierarchy, const int32_t *n_wsegs, const double *wvals, const double *job_request) {
  Session &s = *(Session *)hp;
  Hdrf h;
  h.Q = s.Q;
  std::string all(hierarchy);
  size_t pos = 0, wo = 0;
  for (int q = 0; q < s.Q; ++q) {
    size_t e = all.find('\n', pos);
    std::string line = all.substr(pos, e == std::string::npos ? std::string::npos : e - pos);
    pos = e == std::string::npos ? all.size() : e + 1;
    std::vector<std::string> segs;
    size_t a = 0;
    for (;;) {
      size_t b = line.find('/', a);
      segs.push_back(line.substr(a, b == std::string::npos ? std::string::npos : b - a));
      if (b == std::string::npos) break;
      a = b + 1;
    }
    h.paths.push_back(segs);
    h.weights.emplace_back(wvals + wo, wvals + wo + n_wsegs[q]);
    wo += n_wsegs[q];
  }
  h.job_request.assign(job_request, job_request + (size_t)s.R * s.J);
  h.root.allocated.assign(s.R, 0.0);
  for (int j = 0; j < s.J; ++j) {
    const int q = s.j_queue[j];
    if (q < 0) return VC_EINVAL;
    if (h.weights[q].size() < h.paths[q].size()) return VC_EINVAL;
  }
  for (int j = 0; j < s.J; ++j) build_hierarchy(s, h, j);  // drf.go:186-220, jobs in index order
  update_tree(s, h);
  g_hdrf[hp] = std::move(h);
  return VC_OK;
}
void vcoh_detach(void *hp) { g_hdrf.erase(hp); }
int vcoh_allocate_run(void *hp, int argmin) {
  auto it = g_hdrf.find(hp);
  if (it == g_hdrf.end()) return VC_EINVAL;
  return hdrf_allocate_execute(*(Session *)hp, it->second, argmin != 0);
}
int vcoh_backfill_pick_order(void *hp, int32_t *out) {
  Session &s = *(Session *)hp;
  std::vector<int> p = hdrf_backfill_pick(s, g_hdrf.at(hp));
  for (size_t i = 0; i < p.size(); ++i) out[i] = p[i] - s.T_alloc;
  return (int)p.size();
}
int vcoh_backfill(void *hp) {
  auto it = g_hdrf.find(hp);
  if (it == g_hdrf.end()) return VC_EINVAL;
  return hdrf_backfill_execute(*(Session *)hp, it->second);
}
// compareQueues on the current tree (after the last operation), and the state of the node of queue q at `level`
double vcoh_compare(void *hp, int l, int r) {
  Hdrf &h = g_hdrf.at(hp);
  update_tree(*(Session *)hp, h);
  return compare_queues(h, l, r);
}
int vcoh_node(void *hp, int q, int level, double *share, double *weight, int *saturated, double *allocated) {
  Hdrf &h = g_hdrf.at(hp);
  Session &s = *(Session *)hp;
  update_tree(s, h);
  HNode *n = node_of(h, q, level);
  if (!n) return VC_EINVAL;
  *share = n->share; *weight = n->weight; *saturated = n->saturated;
  for (int d = 0; d < s.R; ++d) allocated[d] = n->allocated[d];
  return VC_OK;
}
// drf AllocateFunc / DeallocateFunc of a task on job j without placing it (hand cases that move one job's allocation)
void vcoh_job_add(void *hp, int j, const double *delta) {
  Session &s = *(Session *)hp;
  for (int d = 0; d < s.R; ++d) at(s.j_alloc, d, s.J, j) += delta[d];
  drf_update_share(s, j);
}

}  // extern "C"

// topo_args.h — one topology-aware dry-run instance as flat host arrays: the argument of the test-only launcher of
// k_evict_dryrun (evict_harness.cu) and of the CPU shim of vct::topo_dry_run (tests/hostshim/topo_shim.cpp).
#pragma once
#include <cstdint>
#include <cstring>

#include "../../volcano_b200/csrc/vc_topo.hpp"

struct EhTopoArgs {
  int N, R, J, RT, pods_dim, n_plugins, task_order_prio;
  const int32_t *plugin, *tier;
  const uint32_t *enabled;
  const double *idle, *rel, *pip;  // [R][N]
  const uint8_t *pred;             // [N] 1 = the node passes the preemptor's predicates
  const int32_t *rt_off, *rt_idx;  // [N+1], [RT]
  const double *rt_req;            // [R][RT]
  const uint32_t *rt_has, *rt_flags, *rt_uid;
  const int32_t *rt_job, *rt_prio, *rt_pod_prio;
  const int64_t *rt_podidx, *rt_ts, *rt_start;
  const uint8_t *rt_evicted;
  const int32_t *j_queue, *j_prio, *j_min, *j_ready, *j_pbe;  // [J]
  const uint32_t *j_rank;
  const double *j_alloc, *j_share;  // [R][J], [J]
  const double *total;              // [R]
  uint32_t total_has;
  // the preemptor
  int job, queue, intra, job_prio, task_prio;
  const double *req;  // [R]
  uint32_t has;
  int sim_update, sim_state, sim_alloc, q_exists;
  const double *qalloc, *qdes;  // [R]
  uint32_t qalloc_has, qdes_has;
  int qalloc_nil;
  int64_t now_ns;
  // results
  uint8_t *ok;         // [N]
  int32_t *nv;         // [N]
  long long *key;      // [4][N]
  int32_t *victims;    // [RT] node n's victims at [rt_off[n], rt_off[n] + nv[n])
};

// the view and preemptor record over the given pointers (host or device copies of the arrays in `a`)
inline void eh_topo_task(const EhTopoArgs &a, vct::TopoTask &t) {
  std::memset(&t, 0, sizeof t);
  t.job = a.job; t.queue = a.queue; t.intra = a.intra; t.job_prio = a.job_prio; t.task_prio = a.task_prio;
  for (int d = 0; d < a.R; ++d) { t.req[d] = a.req[d]; t.qalloc.v[d] = a.qalloc[d]; t.qdes[d] = a.qdes[d]; }
  t.has = a.has; t.sim_update = a.sim_update; t.sim_state = a.sim_state; t.sim_alloc = a.sim_alloc; t.q_exists = a.q_exists;
  t.qalloc.has = a.qalloc_has; t.qalloc.nil = a.qalloc_nil; t.qdes_has = a.qdes_has; t.now_ns = a.now_ns;
}
inline bool eh_topo_check(const EhTopoArgs &a) {  // sizes and indices the routine trusts
  if (a.N < 0 || a.R < 2 || a.R > VC_MAX_DIMS || a.J < 1 || a.RT < 0 || a.pods_dim < -1 || a.pods_dim >= a.R) return false;
  if (a.n_plugins < 0 || a.n_plugins > VC_MAX_PLUGINS || a.job < 0 || a.job >= a.J) return false;
  if (a.N > 0 && (a.rt_off[0] != 0 || a.rt_off[a.N] != a.RT)) return false;
  for (int n = 0; n < a.N; ++n)
    if (a.rt_off[n + 1] < a.rt_off[n]) return false;
  for (int k = 0; k < a.RT; ++k)
    if (a.rt_idx[k] < 0 || a.rt_idx[k] >= a.RT || a.rt_job[k] < -1 || a.rt_job[k] >= a.J) return false;
  return true;
}

// topo_shim.cpp — test shim: the library's per-node dry run of topology-aware preemption (vct::topo_dry_run, the code
// k_evict_dryrun runs on the device) compiled by g++ for tests/test_topo_preempt_host.py.
#include <cstring>
#include <vector>

#include "../../tools/kernels/topo_args.h"

extern "C" int vts_dry_run(const EhTopoArgs *a) {
  if (!a || !eh_topo_check(*a)) return -1;
  vct::TopoView v;
  std::memset(&v, 0, sizeof v);
  v.R = a->R; v.N = a->N; v.J = a->J; v.RT = a->RT; v.pods_dim = a->pods_dim; v.n_plugins = a->n_plugins;
  v.task_order_prio = a->task_order_prio;
  for (int i = 0; i < a->n_plugins; ++i) { v.plugin[i] = a->plugin[i]; v.tier[i] = a->tier[i]; v.enabled[i] = a->enabled[i]; }
  v.idle = a->idle; v.rel = a->rel; v.pip = a->pip; v.rt_off = a->rt_off; v.rt_idx = a->rt_idx; v.rt_req = a->rt_req;
  v.rt_has = a->rt_has; v.rt_flags = a->rt_flags; v.rt_uid = a->rt_uid; v.rt_job = a->rt_job; v.rt_prio = a->rt_prio;
  v.rt_podidx = a->rt_podidx; v.rt_ts = a->rt_ts; v.rt_evicted = a->rt_evicted; v.rt_pod_prio = a->rt_pod_prio;
  v.rt_start = a->rt_start; v.j_queue = a->j_queue; v.j_prio = a->j_prio; v.j_min = a->j_min; v.j_ready = a->j_ready;
  v.j_pbe = a->j_pbe; v.j_rank = a->j_rank; v.j_alloc = a->j_alloc; v.j_share = a->j_share;
  for (int d = 0; d < a->R; ++d) v.total[d] = a->total[d];
  v.total_has = a->total_has;
  vct::TopoTask t;
  eh_topo_task(*a, t);
  const size_t B = (size_t)(a->RT > 0 ? a->RT : 1);
  std::vector<int32_t> sb(B);
  std::vector<uint8_t> sf(B), sg(B);
  for (int n = 0; n < a->N; ++n) {
    a->ok[n] = 0;
    if (!a->pred[n]) continue;
    const int o = a->rt_off[n];
    const vct::TopoResult r = vct::topo_dry_run(v, t, n, a->victims + o, sb.data() + o, sf.data() + o, sg.data() + o);
    a->ok[n] = (uint8_t)r.ok;
    a->nv[n] = r.nv;
    for (int k = 0; k < 4; ++k) a->key[(size_t)k * a->N + n] = r.key[k];
  }
  return 0;
}

// hdrf_shim.cpp — test shim: the library's host-side hdrf logic (vc_hdrf.hpp tree construction and evaluation, the hdrf
// comparator in vch::backfill_pick) compiled by g++ for tests/test_hdrf_host.py.
#include "../../volcano_b200/csrc/vc_host.hpp"

extern "C" {

// the tree after session open: per queue q and level l of its path, the node's (share, weight, saturated); returns M or
// -1 (with the reason in `why`) for the inputs the reference crashes on
int vhh_tree(int R, int J, int Q, const int32_t *job_queue, const vc_hdrf *h, const double *total, uint32_t total_has,
             const double *j_alloc, const double *j_share, int32_t *path_off_out, double *share_out, double *weight_out,
             int32_t *sat_out, char *why, int why_len) {
  vch::HdrfTree t;
  const std::string err = vch::hdrf_build(J, Q, job_queue, *h, t);
  if (!err.empty()) {
    std::snprintf(why, why_len, "%s", err.c_str());
    return -1;
  }
  vch::HdrfState st;
  vch::hdrf_eval(t, R, J, total, total_has, j_alloc, j_share, h->job_request, st);
  for (int q = 0; q <= Q; ++q) path_off_out[q] = t.q_path_off[q];
  for (size_t i = 0; i < t.q_path.size(); ++i) {
    const int m = t.q_path[i];
    share_out[i] = st.n_share[m]; weight_out[i] = t.weight[m]; sat_out[i] = st.n_sat[m];
  }
  return t.M;
}

// pickUpPendingTasks after allocate's kept operations, with the hdrf comparator (the Keep record as vc_snapshot_upload
// fills it; see vh_backfill_pick in host_shim.cpp)
int vhh_backfill_pick(const vc_dims *d, const vc_conf *conf, const vc_nodes *nd, const vc_tasks *tk, const vc_jobs *jb,
                      const vc_queues *qu, const vc_tasks *bt, int n_bf, const vc_decision *ops, int n_ops, const vc_hdrf *h,
                      int32_t *order_out) {
  const size_t R = d->n_dims, K = d->n_kdims, N = d->n_nodes, T = d->n_tasks, J = d->n_jobs, Q = d->n_queues, NR = d->n_roles,
               B = (size_t)n_bf;
  vch::HRes total;
  for (size_t k = 0; k < R; ++k) {
    double acc = 0;
    for (size_t n = 0; n < N; ++n) acc += nd->allocatable[k * N + n];
    total.v[k] = acc;
    if (k >= 2 && N > 0) { total.has |= 1u << k; total.nil = false; }
  }
  const bool has_drf = vch::has_plugin(*conf, VC_PLUGIN_DRF), has_prop = vch::has_plugin(*conf, VC_PLUGIN_PROPORTION);
  std::vector<vch::QAttr> qattr;
  if (has_prop) vch::proportion_open(*d, *jb, *qu, total, qattr);
  else qattr.assign(Q, vch::QAttr());
  vch::BackfillTasks bf;
  bf.n = n_bf;
  bf.req.assign(bt->resreq, bt->resreq + R * B); bf.kreq.assign(bt->k8s_req, bt->k8s_req + K * B);
  bf.knz.assign(bt->k8s_nonzero_req, bt->k8s_nonzero_req + 2 * B);
  bf.has.assign(bt->req_has, bt->req_has + B); bf.uid.assign(bt->uid_rank, bt->uid_rank + B);
  bf.job.assign(bt->job, bt->job + B); bf.klass.assign(bt->klass, bt->klass + B); bf.role.assign(bt->role, bt->role + B);
  bf.prio.assign(bt->priority, bt->priority + B); bf.podidx.assign(bt->pod_index, bt->pod_index + B);
  bf.ts.assign(bt->creation_ts, bt->creation_ts + B);
  vch::BackfillKeep k;
  k.j_queue.assign(jb->queue, jb->queue + J); k.j_min.assign(jb->min_available, jb->min_available + J);
  k.j_prio.assign(jb->priority, jb->priority + J); k.j_ready0.assign(jb->ready_num, jb->ready_num + J);
  k.j_pbe.assign(jb->pending_besteffort, jb->pending_besteffort + J);
  k.j_taskmintotal.assign(jb->task_min_total, jb->task_min_total + J); k.j_roleoff.assign(jb->role_off, jb->role_off + J + 1);
  k.r_min.assign(jb->role_min, jb->role_min + NR); k.r_occ0.assign(jb->role_occupied, jb->role_occupied + NR);
  k.r_flags.assign(jb->role_flags, jb->role_flags + NR);
  k.q_prio.assign(qu->priority, qu->priority + Q); k.t_role.assign(tk->role, tk->role + T);
  k.j_flags.assign(jb->flags, jb->flags + J);
  vch::rank_by(jb->creation_ts, jb->uid_rank, J, k.j_rank);
  vch::rank_by(qu->creation_ts, qu->uid_rank, Q, k.q_rank);
  k.j_valid.resize(J);
  for (size_t j = 0; j < J; ++j) k.j_valid[j] = vch::job_valid(*conf, *jb, (int)j) ? 1 : 0;
  k.j_alloc0.assign(jb->allocated, jb->allocated + R * J);
  vch::HdrfTree tree;
  if (!vch::hdrf_build((int)J, (int)Q, jb->queue, *h, tree).empty()) return -1;
  const vch::HdrfPick hp{&tree, h->job_request};
  vch::BackfillPick p = vch::backfill_pick(*conf, true, R, T, J, Q, B, has_drf, has_prop, total.v, total.has, bf, k, ops,
                                           (size_t)n_ops, tk->job, tk->resreq, tk->req_has, qattr, &hp);
  for (size_t i = 0; i < p.order.size(); ++i) order_out[i] = p.order[i];
  return (int)p.order.size();
}

}  // extern "C"

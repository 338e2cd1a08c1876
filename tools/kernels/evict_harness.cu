// evict_harness.cu — test-only launchers for the preempt / reclaim kernels of volcano_b200/csrc/vc_evict.cuh.
//
// Every launcher takes host arrays and sizes, checks them on the host (sizes within the kernel's limits, every index in
// range) and returns EH_EINVAL without launching when they are not; otherwise it stages the data on the device, builds
// EvictParams / EvictTask / DevConf as vcalloc.cu does, launches with the production geometry and copies the results back.
// The pick hand-outs and the apply command live in mapped pinned memory, as in production.
#include <cstring>
#include <vector>

#include "../../volcano_b200/csrc/vc_evict.cuh"

#define EH_OK 0
#define EH_EINVAL (-1)
#define EH_ECUDA (-3)

#define EH_TRY(x)                                  \
  do {                                             \
    if ((x) != cudaSuccess) return EH_ECUDA;       \
  } while (0)

namespace {

template <class T>
struct DevBuf {  // device copy of a host array (nullptr for an empty one)
  T *d = nullptr;
  ~DevBuf() { if (d) cudaFree(d); }
  cudaError_t put(const T *h, size_t n) {
    if (n == 0) return cudaSuccess;
    cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&d), n * sizeof(T));
    if (e != cudaSuccess) return e;
    return h ? cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice) : cudaMemset(d, 0, n * sizeof(T));
  }
  cudaError_t get(T *h, size_t n) const { return n ? cudaMemcpy(h, d, n * sizeof(T), cudaMemcpyDeviceToHost) : cudaSuccess; }
};

struct Mapped {  // mapped pinned int32 words
  int32_t *h = nullptr, *d = nullptr;
  ~Mapped() { if (h) cudaFreeHost(h); }
  cudaError_t alloc(size_t n) {
    cudaError_t e = cudaHostAlloc(reinterpret_cast<void **>(&h), n * 4, cudaHostAllocMapped);
    if (e != cudaSuccess) return e;
    return cudaHostGetDevicePointer(reinterpret_cast<void **>(&d), h, 0);
  }
};

}  // namespace

// ---- k_evict_pick / k_evict_pick_big --------------------------------------------------------------------------------
// A pick state holds the candidate flags and keys of N nodes on the device; each eh_pick_launch is one production launch
// on that state (cand 1 -> 2 for the nodes handed out), so a test drains it the way the host control loop does.
struct EhPick {
  int N = 0;
  DevBuf<uint8_t> cand;
  DevBuf<unsigned long long> key;
  Mapped pick;  // [0, EV_PICK_K) hand-outs, [EV_PICK_K] sequence word
};

extern "C" int eh_pick_smem_max_nodes() { return 200 * 1024 / 8; }  // vcalloc.cu's switch to k_evict_pick_big

extern "C" int eh_pick_open(int N, const uint8_t *cand, const unsigned long long *key, EhPick **out) {
  if (!out || N < 0 || (N > 0 && (!cand || !key))) return EH_EINVAL;
  for (int n = 0; n < N; ++n)
    if (cand[n] > 2) return EH_EINVAL;
  EhPick *s = new EhPick();
  s->N = N;
  if (s->cand.put(cand, N) != cudaSuccess || s->key.put(key, N) != cudaSuccess || s->pick.alloc(EV_PICK_K + 1) != cudaSuccess) {
    delete s;
    return EH_ECUDA;
  }
  *out = s;
  return EH_OK;
}

extern "C" void eh_pick_close(EhPick *s) { delete s; }

// big = 0: k_evict_pick with N * 8 bytes of dynamic shared memory (N <= eh_pick_smem_max_nodes()); 1: k_evict_pick_big.
// words[0..EV_PICK_K] receive the mapped buffer after the launch (hand-outs, then the sequence word), which is set to
// ~seq before it; cand_out (N bytes, may be null) receives the flags.
extern "C" int eh_pick_launch(EhPick *s, int big, int mode, int seq, int32_t *words, uint8_t *cand_out) {
  if (!s || !words || (big != 0 && big != 1) || mode < EV_MODE_PREEMPT_INTER || mode > EV_MODE_RECLAIM) return EH_EINVAL;
  const size_t smem = (size_t)s->N * 8;
  if (!big && s->N > eh_pick_smem_max_nodes()) return EH_EINVAL;
  EvictParams p;
  std::memset(&p, 0, sizeof p);
  p.d.N = s->N;
  p.cand = s->cand.d;
  p.key = s->key.d;
  p.pick_node = s->pick.d;
  for (int i = 0; i < EV_PICK_K; ++i) s->pick.h[i] = -7;
  s->pick.h[EV_PICK_K] = ~seq;
  if (!big) {
    if (smem > 48 * 1024) EH_TRY(cudaFuncSetAttribute(k_evict_pick<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_evict_pick<false><<<1, 1024, smem>>>(p, mode, seq);
  } else {
    k_evict_pick_big<false><<<1, 1024, 0>>>(p, mode, seq);
  }
  EH_TRY(cudaGetLastError());
  EH_TRY(cudaDeviceSynchronize());
  for (int i = 0; i <= EV_PICK_K; ++i) words[i] = reinterpret_cast<volatile int32_t *>(s->pick.h)[i];
  if (cand_out) EH_TRY(s->cand.get(cand_out, s->N));
  return EH_OK;
}

// ---- k_evict_rank ---------------------------------------------------------------------------------------------------
// One preemptor against N nodes. Only the victim-voting plugins may be enabled (no VC_EN_NODE_ORDER: the harness carries
// no scoring rows), so every candidate's key is ev_score_key(+0.0). Class 0 is the preemptor's; cstat is its row [N].
struct EhRankArgs {
  int N, R, RT, J, Q, pods_dim, exact_sums;
  int n_plugins;
  const int32_t *plugin, *tier;
  const uint32_t *enabled;
  const double *idle, *rel, *pip;  // [R][N]
  const uint32_t *cstat;           // [N]
  const int32_t *rt_off, *rt_idx;  // [N+1], [RT]
  const double *rt_req;            // [R][RT]
  const uint32_t *rt_flags;        // [RT]
  const int32_t *rt_job, *rt_prio; // [RT]
  const uint8_t *rt_evicted;       // [RT]
  const int32_t *j_queue, *j_prio, *j_min, *j_ready;  // [J]
  const uint32_t *q_flags;         // [Q]
  const uint8_t *q_over;           // [Q]
  // the preemptor
  int mode, job, queue, job_prio, task_prio;
  const double *req;  // [R]
  uint32_t has;
  int quota_on, quota_open;
  uint32_t qalloc_has, qdes_has;
  const double *qalloc, *qdes;  // [R]
  // results
  uint8_t *cand;            // [N]
  unsigned long long *key;  // [N]
};

// The SOFT chain of preempt's normal reading (eh_soft_chain): k_evict_rank<.., true>, k_evict_samp<true> under sampling,
// then pick launches until the candidates run out. TaintToleration's batch score (weight w_taint) is the only scorer;
// the soft-taint counts are bits 8..15 of the rank arguments' cstat.
struct EhSoftArgs {
  int w_taint;
  int samp, filtered, pct, min_nodes, min_pct, start;  // samp = 1: one PredicateNodes call between rank and pick
  int big;                                              // 1: k_evict_pick_big, else k_evict_pick
  unsigned long long seq, stale;  // the ranking's tag; the reduction word before the launches (an earlier ranking's)
  int32_t *order;                 // [N] the nodes handed out, in order
  int32_t *n_order;
  unsigned long long *word;       // the reduction word after the launches
};

// network-topology-aware's hypernode binpacking (the NTA instances): the plugin's tables as vcalloc.cu stages them.
// member [L][N] (-1: the node is in no hypernode of that tier level), hn_alloc / hn_used [R][H], the tier weights [L]
// (their total is summed here in level order, as the library does), the plugin's weight and per-dimension weights [R]
// (-1: not weighed). nta_term [N] receives the per-node term the SOFT+NTA ranking stores (0 where it stores none).
struct EhNtaArgs {
  int L, H, weight;
  const int32_t *member;
  const double *hn_alloc, *hn_used, *tier_w;
  const int32_t *dim_weight;
  double *nta_term;
};

static int rank_run(const EhRankArgs *a, const EhSoftArgs *sx, const uint8_t *guard = nullptr, const EhNtaArgs *nx = nullptr);

static bool nta_check(const EhNtaArgs *x, int N, int R) {
  if (!x || x->L < 1 || x->L > VC_MAX_TIERS || x->H < 1 || !x->member || !x->hn_alloc || !x->hn_used || !x->tier_w ||
      !x->dim_weight || !x->nta_term)
    return false;
  for (size_t i = 0; i < (size_t)x->L * N; ++i)
    if (x->member[i] < -1 || x->member[i] >= x->H) return false;
  for (int d = 0; d < R; ++d)
    if (x->dim_weight[d] < -1) return false;
  return true;
}

extern "C" int eh_rank(const EhRankArgs *a) { return rank_run(a, nullptr); }

// The GUARD instance k_evict_rank<16, .., false, true> (sessions where pdb or cdp votes): guard[RT] holds the VCT_GUARD_*
// bits vcalloc.cu derives from the victim-guard table.
extern "C" int eh_rank_guard(const EhRankArgs *a, const uint8_t *guard) {
  if (!a || (a->RT > 0 && !guard)) return EH_EINVAL;
  for (int r = 0; r < a->RT; ++r)
    if (guard[r] & ~(VCT_GUARD_NO_LABELS | VCT_GUARD_PDB_NEVER | VCT_GUARD_CDP)) return EH_EINVAL;
  return rank_run(a, nullptr, guard);
}

extern "C" int eh_soft_chain(const EhRankArgs *a, const EhSoftArgs *sx) {
  if (!a || !sx || !sx->order || !sx->n_order || !sx->word || a->N < 1 || a->mode == EV_MODE_RECLAIM) return EH_EINVAL;
  if ((sx->samp != 0 && sx->samp != 1) || (sx->big != 0 && sx->big != 1) || sx->start < 0) return EH_EINVAL;
  if (!sx->big && a->N > eh_pick_smem_max_nodes()) return EH_EINVAL;
  return rank_run(a, sx);
}

// The NTA instance k_evict_rank<16, .., false, false, true> of preempt's normal reading: cand / key as eh_rank, the key
// carrying the plugin's term (the node-order plugins stay off, so the total is 0.0 + (0.0 + term))
extern "C" int eh_nta_rank(const EhRankArgs *a, const EhNtaArgs *x) {
  if (!a || a->mode == EV_MODE_RECLAIM || !nta_check(x, a->N, a->R)) return EH_EINVAL;
  return rank_run(a, nullptr, nullptr, x);
}

// The SOFT+NTA chain: k_evict_rank<.., true, false, true> (the term goes to nta_term), k_evict_samp<true> under sampling,
// then k_evict_pick / k_evict_pick_big <SAMP, true, true> until the candidates run out
extern "C" int eh_nta_soft_chain(const EhRankArgs *a, const EhSoftArgs *sx, const EhNtaArgs *x) {
  if (!a || !nta_check(x, a->N, a->R)) return EH_EINVAL;
  if (!sx || !sx->order || !sx->n_order || !sx->word || a->N < 1 || a->mode == EV_MODE_RECLAIM) return EH_EINVAL;
  if ((sx->samp != 0 && sx->samp != 1) || (sx->big != 0 && sx->big != 1) || sx->start < 0) return EH_EINVAL;
  if (!sx->big && a->N > eh_pick_smem_max_nodes()) return EH_EINVAL;
  return rank_run(a, sx, nullptr, x);
}

// p / t as rank_run built them (device rows staged, cand / key allocated); rank_run's buffers outlive the call
template <bool NTA>
static int soft_chain(const EhRankArgs *a, const EhSoftArgs &sx, EvictParams p, const EvictTask &t) {
  const int N = a->N;
  p.c.batch_any = 1; p.c.taint_batch = 1; p.c.w_taint = sx.w_taint;
  DevBuf<unsigned long long> word;
  DevBuf<int32_t> list, words;  // words: [0] sampled count, [1] index
  EH_TRY(word.put(&sx.stale, 1));
  EH_TRY(list.put(nullptr, N));
  const int32_t w0[2] = {0, sx.start};
  EH_TRY(words.put(w0, 2));
  p.soft_word = word.d; p.soft_seq = sx.seq; p.soft_klass = 0; p.soft_reduce = sx.samp ? 0 : 1;
  p.samp_list = list.d; p.samp_cnt = words.d;
  launch_evict_rank<true, false, NTA>((unsigned)(((size_t)N * 16 + 255) / 256), 0, (size_t)a->R, p, t);
  EH_TRY(cudaGetLastError());
  if (sx.samp) {
    EvictSamp s;
    s.cstat = p.cstat; s.klass = 0; s.N = N; s.filtered = sx.filtered ? 1 : 0;
    s.pct = sx.pct; s.min_nodes = sx.min_nodes; s.min_pct = sx.min_pct;
    s.idx_in = words.d + 1; s.idx_out = words.d + 1; s.list = list.d; s.cnt = words.d;
    s.soft_word = word.d; s.soft_seq = sx.seq;
    k_evict_samp<true><<<1, 1024>>>(s);
    EH_TRY(cudaGetLastError());
  }
  Mapped pick;
  EH_TRY(pick.alloc(EV_PICK_K + 1));
  p.pick_node = pick.d;
  const size_t smem = (size_t)N * 8;
  auto fn = sx.samp ? k_evict_pick<true, true, NTA> : k_evict_pick<false, true, NTA>;
  auto fn_big = sx.samp ? k_evict_pick_big<true, true, NTA> : k_evict_pick_big<false, true, NTA>;
  if (!sx.big && smem > 48 * 1024) EH_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int n_out = 0;
  for (int seq = 1;; ++seq) {  // as the host control loop drains a ranking: until a batch comes back short
    pick.h[EV_PICK_K] = ~seq;
    if (sx.big) fn_big<<<1, 1024>>>(p, t.mode, seq);
    else fn<<<1, 1024, smem>>>(p, t.mode, seq);
    EH_TRY(cudaGetLastError());
    EH_TRY(cudaDeviceSynchronize());
    const volatile int32_t *h = pick.h;
    if (h[EV_PICK_K] != seq) return EH_ECUDA;
    int got = 0;
    for (; got < EV_PICK_K && h[got] >= 0; ++got) {
      if (n_out >= N) return EH_ECUDA;  // a node handed out twice
      sx.order[n_out++] = h[got];
    }
    if (got < EV_PICK_K) break;
  }
  *sx.n_order = n_out;
  EH_TRY(word.get(sx.word, 1));
  return EH_OK;
}

static int rank_run(const EhRankArgs *a, const EhSoftArgs *sx, const uint8_t *guard, const EhNtaArgs *nx) {
  if (!a) return EH_EINVAL;
  const int N = a->N, R = a->R, RT = a->RT, J = a->J, Q = a->Q;
  if (N < 0 || R < 2 || R > VC_MAX_DIMS || RT < 0 || J < 0 || Q < 0 || a->pods_dim < -1 || a->pods_dim >= R) return EH_EINVAL;
  if (a->n_plugins < 0 || a->n_plugins > VC_MAX_PLUGINS) return EH_EINVAL;
  if (a->mode < EV_MODE_PREEMPT_INTER || a->mode > EV_MODE_RECLAIM || a->job < -1 || a->job >= J || a->queue < -1 || a->queue >= Q)
    return EH_EINVAL;
  if (!a->req || (a->quota_on && (!a->qalloc || !a->qdes)) || !a->cand || !a->key) return EH_EINVAL;
  if (N > 0 && (!a->idle || !a->rel || !a->pip || !a->cstat || !a->rt_off)) return EH_EINVAL;
  if (RT > 0 && (!a->rt_idx || !a->rt_req || !a->rt_flags || !a->rt_job || !a->rt_prio || !a->rt_evicted)) return EH_EINVAL;
  if (J > 0 && (!a->j_queue || !a->j_prio || !a->j_min || !a->j_ready)) return EH_EINVAL;
  if (Q > 0 && (!a->q_flags || !a->q_over)) return EH_EINVAL;
  DevConf c;
  std::memset(&c, 0, sizeof c);
  c.n_plugins = a->n_plugins;
  for (int i = 0; i < a->n_plugins; ++i) {
    if (a->plugin[i] < 0 || (i > 0 && a->tier[i] < a->tier[i - 1]) || (a->enabled[i] & VC_EN_NODE_ORDER)) return EH_EINVAL;
    c.plugin[i] = a->plugin[i]; c.tier[i] = a->tier[i]; c.enabled[i] = a->enabled[i];
  }
  // node.Tasks: CSR over the nodes, every entry a running task, every task's job / queue in range
  if (N > 0 && (a->rt_off[0] != 0 || a->rt_off[N] != RT)) return EH_EINVAL;
  for (int n = 0; n < N; ++n)
    if (a->rt_off[n + 1] < a->rt_off[n]) return EH_EINVAL;
  for (int k = 0; k < RT; ++k) {
    if (a->rt_idx[k] < 0 || a->rt_idx[k] >= RT) return EH_EINVAL;
    if (a->rt_job[k] < -1 || a->rt_job[k] >= J) return EH_EINVAL;
  }
  for (int j = 0; j < J; ++j)
    if (a->j_queue[j] < -1 || a->j_queue[j] >= Q) return EH_EINVAL;

  DevBuf<double> idle, rel, pip, rt_req;
  DevBuf<uint32_t> cstat, rt_flags, q_flags;
  DevBuf<int32_t> rt_off, rt_idx, rt_job, rt_prio, j_queue, j_prio, j_min, j_ready;
  DevBuf<uint8_t> rt_ev, q_over, cand, rt_guard;
  DevBuf<unsigned long long> key;
  const size_t RN = (size_t)R * N;
  if (guard) EH_TRY(rt_guard.put(guard, RT));
  EH_TRY(idle.put(a->idle, RN)); EH_TRY(rel.put(a->rel, RN)); EH_TRY(pip.put(a->pip, RN));
  EH_TRY(cstat.put(a->cstat, N)); EH_TRY(rt_off.put(a->rt_off, N > 0 ? N + 1 : 0));
  EH_TRY(rt_idx.put(a->rt_idx, RT)); EH_TRY(rt_req.put(a->rt_req, (size_t)R * RT)); EH_TRY(rt_flags.put(a->rt_flags, RT));
  EH_TRY(rt_job.put(a->rt_job, RT)); EH_TRY(rt_prio.put(a->rt_prio, RT)); EH_TRY(rt_ev.put(a->rt_evicted, RT));
  EH_TRY(j_queue.put(a->j_queue, J)); EH_TRY(j_prio.put(a->j_prio, J)); EH_TRY(j_min.put(a->j_min, J));
  EH_TRY(j_ready.put(a->j_ready, J)); EH_TRY(q_flags.put(a->q_flags, Q)); EH_TRY(q_over.put(a->q_over, Q));
  EH_TRY(cand.put(nullptr, N)); EH_TRY(key.put(nullptr, N));

  EvictParams p;
  std::memset(&p, 0, sizeof p);
  p.d.N = N; p.d.R = R; p.d.K = 0; p.d.C = 1; p.d.J = J; p.d.Q = Q; p.d.pods_dim = a->pods_dim;
  p.c = c;
  p.idle = idle.d; p.rel = rel.d; p.pip = pip.d; p.cstat = cstat.d;
  p.rt_off = rt_off.d; p.rt_idx = rt_idx.d; p.rt_req = rt_req.d; p.rt_flags = rt_flags.d; p.rt_job = rt_job.d;
  p.rt_prio = rt_prio.d; p.rt_evicted = rt_ev.d; p.j_queue = j_queue.d; p.j_prio = j_prio.d; p.j_min = j_min.d;
  p.j_ready = j_ready.d; p.q_flags = q_flags.d; p.q_over = q_over.d;
  p.exact_sums = a->exact_sums ? 1 : 0;
  p.RT = RT;
  p.key = key.d; p.cand = cand.d;
  p.rt_guard = rt_guard.d;
  EvictTask t;
  std::memset(&t, 0, sizeof t);
  for (int d = 0; d < R; ++d) t.rec.req[d] = a->req[d];
  t.rec.has = a->has; t.rec.klass = 0;
  t.klass = 0; t.job = a->job; t.queue = a->queue; t.mode = a->mode; t.job_prio = a->job_prio; t.task_prio = a->task_prio;
  t.quota_on = a->quota_on ? 1 : 0; t.quota_open = a->quota_open ? 1 : 0;
  t.qalloc_has = a->qalloc_has; t.qdes_has = a->qdes_has;
  if (a->quota_on)
    for (int d = 0; d < R; ++d) { t.qalloc[d] = a->qalloc[d]; t.qdes[d] = a->qdes[d]; }
  DevBuf<int32_t> hn_member;
  DevBuf<double> hn_alloc, hn_used, nta_term;
  if (nx) {  // DevConf's plugin fields as vcalloc.cu derives them for nta_on
    EH_TRY(hn_member.put(nx->member, (size_t)nx->L * N)); EH_TRY(hn_alloc.put(nx->hn_alloc, (size_t)R * nx->H));
    EH_TRY(hn_used.put(nx->hn_used, (size_t)R * nx->H)); EH_TRY(nta_term.put(nullptr, N));
    p.c.batch_any = 1; p.c.nta_plugin = 1; p.c.nta_tables = 1; p.c.nta_on = 1; p.c.nta_weight = nx->weight;
    p.c.nta_L = nx->L; p.c.tier_w_total = 0.0;
    for (int l = 0; l < nx->L; ++l) { p.c.tier_w[l] = nx->tier_w[l]; p.c.tier_w_total += nx->tier_w[l]; }
    for (int d = 0; d < VC_MAX_DIMS; ++d) p.c.nta_dim_weight[d] = d < R ? nx->dim_weight[d] : -1;
    p.hn_H = nx->H; p.hn_member = hn_member.d; p.hn_alloc = hn_alloc.d; p.hn_used = hn_used.d; p.nta_term = nta_term.d;
  }
  if (sx) {
    const int rc = nx ? soft_chain<true>(a, *sx, p, t) : soft_chain<false>(a, *sx, p, t);
    if (rc == EH_OK && nx) EH_TRY(nta_term.get(nx->nta_term, N));
    return rc;
  }
  if (N > 0) {  // the instance vcalloc.cu picks for R
    const unsigned grid = (unsigned)(((size_t)N * 16 + 255) / 256);
    if (nx) {
      launch_evict_rank<false, false, true>(grid, 0, (size_t)R, p, t);
    } else if (guard) {
      if (R <= 8) k_evict_rank<16, 8, false, true><<<grid, 256>>>(p, t);
      else k_evict_rank<16, VC_MAX_DIMS, false, true><<<grid, 256>>>(p, t);
    } else {
      if (R <= 8) k_evict_rank<16, 8><<<grid, 256>>>(p, t);
      else k_evict_rank<16, VC_MAX_DIMS><<<grid, 256>>>(p, t);
    }
    EH_TRY(cudaGetLastError());
  }
  EH_TRY(cudaDeviceSynchronize());
  EH_TRY(cand.get(a->cand, N));
  EH_TRY(key.get(a->key, N));
  if (nx) EH_TRY(nta_term.get(nx->nta_term, N));
  return EH_OK;
}

// ---- k_evict_apply --------------------------------------------------------------------------------------------------
// Statement.Evict of the victims + Statement.Pipeline of the preemptor on one node (undo = 0), or the inverse (undo = 1).
// The rows are updated in place: rel, pip [R][N]; kreq [K][N]; knz [2][N]; pod_count [N]; rt_evicted [RT].
struct EhApplyArgs {
  int N, R, K, RT, has_predicates;
  double *rel, *pip, *kreq, *knz;
  int32_t *pod_count;
  uint8_t *rt_evicted;
  const double *rt_req, *rt_kreq, *rt_knz;  // [R][RT], [K][RT], [2][RT]
  const double *req, *kreq_t, *knz_t;       // the preemptor: [R], [K], [2]
  int node, n_victims;
  const int32_t *victims;
  int undo;
};

// The NTA instance k_evict_apply<true>: hyperNodeResourceCache.used [R][H] booked on every tier level's hypernode of the
// node (member [L][N]), for dims 0, 1 and the present scalars (rt_has [RT] per victim, has for the preemptor); updated in
// place.
struct EhNtaApply {
  int L, H;
  const int32_t *member;
  double *hn_used;
  const uint32_t *rt_has;
  uint32_t has;
};

static int apply_run(const EhApplyArgs *a, const EhNtaApply *x);

extern "C" int eh_apply(const EhApplyArgs *a) { return apply_run(a, nullptr); }

extern "C" int eh_apply_nta(const EhApplyArgs *a, const EhNtaApply *x) {
  if (!a || !x || x->L < 1 || x->L > VC_MAX_TIERS || x->H < 1 || !x->member || !x->hn_used || (a->RT > 0 && !x->rt_has))
    return EH_EINVAL;
  if (a->N < 1) return EH_EINVAL;
  for (size_t i = 0; i < (size_t)x->L * a->N; ++i)
    if (x->member[i] < -1 || x->member[i] >= x->H) return EH_EINVAL;
  return apply_run(a, x);
}

static int apply_run(const EhApplyArgs *a, const EhNtaApply *x) {
  if (!a) return EH_EINVAL;
  const int N = a->N, R = a->R, K = a->K, RT = a->RT;
  if (N < 1 || R < 1 || R > VC_MAX_DIMS || K < 0 || K > VC_MAX_KDIMS || RT < 0) return EH_EINVAL;
  if (a->node < 0 || a->node >= N || a->n_victims < 0 || a->n_victims > EV_MAX_VICTIMS) return EH_EINVAL;
  if (!a->rel || !a->pip || !a->knz || !a->pod_count || !a->req || !a->knz_t || (K > 0 && (!a->kreq || !a->kreq_t))) return EH_EINVAL;
  if (RT > 0 && (!a->rt_evicted || !a->rt_req || !a->rt_knz || (K > 0 && !a->rt_kreq))) return EH_EINVAL;
  if (a->n_victims > 0 && !a->victims) return EH_EINVAL;
  for (int i = 0; i < a->n_victims; ++i)
    if (a->victims[i] < 0 || a->victims[i] >= RT) return EH_EINVAL;
  DevBuf<double> rel, pip, kreq, knz, rt_req, rt_kreq, rt_knz;
  DevBuf<int32_t> pod_count;
  DevBuf<uint8_t> rt_ev;
  EH_TRY(rel.put(a->rel, (size_t)R * N)); EH_TRY(pip.put(a->pip, (size_t)R * N)); EH_TRY(kreq.put(a->kreq, (size_t)K * N));
  EH_TRY(knz.put(a->knz, (size_t)2 * N)); EH_TRY(pod_count.put(a->pod_count, N)); EH_TRY(rt_ev.put(a->rt_evicted, RT));
  EH_TRY(rt_req.put(a->rt_req, (size_t)R * RT)); EH_TRY(rt_kreq.put(a->rt_kreq, (size_t)K * RT));
  EH_TRY(rt_knz.put(a->rt_knz, (size_t)2 * RT));
  Mapped cmd;
  EH_TRY(cmd.alloc(2 + EV_MAX_VICTIMS));
  cmd.h[0] = a->node; cmd.h[1] = a->n_victims;
  for (int i = 0; i < a->n_victims; ++i) cmd.h[2 + i] = a->victims[i];
  EvictParams p;
  std::memset(&p, 0, sizeof p);
  p.d.N = N; p.d.R = R; p.d.K = K;
  p.c.has_predicates = a->has_predicates ? 1 : 0;
  p.rel = rel.d; p.pip = pip.d; p.kreq = kreq.d; p.knz = knz.d; p.pod_count = pod_count.d; p.rt_evicted = rt_ev.d;
  p.rt_req = rt_req.d; p.rt_kreq = rt_kreq.d; p.rt_knz = rt_knz.d; p.RT = RT;
  p.cmd = cmd.d;
  EvictTask t;
  std::memset(&t, 0, sizeof t);
  for (int d = 0; d < R; ++d) t.rec.req[d] = a->req[d];
  for (int k = 0; k < K; ++k) t.rec.kreq[k] = a->kreq_t[k];
  for (int k = 0; k < 2; ++k) t.rec.knz[k] = a->knz_t[k];
  DevBuf<int32_t> hn_member;
  DevBuf<double> hn_used;
  DevBuf<uint32_t> rt_has;
  if (x) {
    EH_TRY(hn_member.put(x->member, (size_t)x->L * N)); EH_TRY(hn_used.put(x->hn_used, (size_t)R * x->H));
    EH_TRY(rt_has.put(x->rt_has, RT));
    p.c.nta_L = x->L; p.hn_H = x->H; p.hn_member = hn_member.d; p.hn_used = hn_used.d; p.rt_has = rt_has.d;
    t.rec.has = x->has;
    k_evict_apply<true><<<1, 64>>>(p, t, a->undo ? 1 : 0);
  } else {
    k_evict_apply<<<1, 64>>>(p, t, a->undo ? 1 : 0);
  }
  EH_TRY(cudaGetLastError());
  EH_TRY(cudaDeviceSynchronize());
  if (x) EH_TRY(hn_used.get(x->hn_used, (size_t)R * x->H));
  EH_TRY(rel.get(a->rel, (size_t)R * N)); EH_TRY(pip.get(a->pip, (size_t)R * N)); EH_TRY(kreq.get(a->kreq, (size_t)K * N));
  EH_TRY(knz.get(a->knz, (size_t)2 * N)); EH_TRY(pod_count.get(a->pod_count, N)); EH_TRY(rt_ev.get(a->rt_evicted, RT));
  return EH_OK;
}

// ---- k_evict_dryrun / k_evict_select (topology-aware preemption) ---------------------------------------------------
#include "topo_args.h"

// The victim-guard table of the GUARD instances, as vcalloc.cu stages it: VCT_GUARD_* bits [RT], the CSR of the PDBs
// counting each task [RT + 1] / [pdb_off[RT]], DisruptionsAllowed [n_pdb].
struct EhGuardArgs {
  int n_pdb;
  const uint8_t *bits;
  const int32_t *pdb_off, *pdb, *pdb_allowed;
};

static int dryrun_run(const EhTopoArgs *a, const EhGuardArgs *g, const int32_t *samp_list, int n_samp);

extern "C" int eh_dryrun(const EhTopoArgs *a) { return dryrun_run(a, nullptr, nullptr, 0); }

// k_evict_dryrun<SAMP, true>: samp_list == nullptr runs the non-sampling instance over every predicate node; otherwise the
// SAMP instance runs on the n_samp listed nodes (k_evict_samp's list: predicate nodes in scan order)
extern "C" int eh_dryrun_guard(const EhTopoArgs *a, const EhGuardArgs *g, const int32_t *samp_list, int n_samp) {
  if (!a || !g || g->n_pdb < 0 || (a->RT > 0 && (!g->bits || !g->pdb_off)) || (g->n_pdb > 0 && !g->pdb_allowed)) return EH_EINVAL;
  if (a->RT > 0) {
    if (g->pdb_off[0] != 0) return EH_EINVAL;
    for (int r = 0; r < a->RT; ++r)
      if (g->pdb_off[r + 1] < g->pdb_off[r]) return EH_EINVAL;
    if (g->pdb_off[a->RT] > 0 && !g->pdb) return EH_EINVAL;
    for (int x = 0; x < g->pdb_off[a->RT]; ++x)
      if (g->pdb[x] < 0 || g->pdb[x] >= g->n_pdb) return EH_EINVAL;
  }
  if (samp_list) {
    if (n_samp < 0 || n_samp > a->N) return EH_EINVAL;
    for (int i = 0; i < n_samp; ++i)
      if (samp_list[i] < 0 || samp_list[i] >= a->N) return EH_EINVAL;
  }
  return dryrun_run(a, g, samp_list, n_samp);
}

static int dryrun_run(const EhTopoArgs *a, const EhGuardArgs *g, const int32_t *samp_list, int n_samp) {
  if (!a || !eh_topo_check(*a)) return EH_EINVAL;
  const int N = a->N, R = a->R, J = a->J, RT = a->RT;
  const size_t B = (size_t)(RT > 0 ? RT : 1);
  DevBuf<double> idle, rel, pip, rt_req, j_alloc, j_share;
  DevBuf<uint32_t> cstat, rt_has, rt_flags, rt_uid, j_rank;
  DevBuf<int32_t> rt_off, rt_idx, rt_job, rt_prio, rt_pp, j_queue, j_prio, j_min, j_ready, j_pbe, sa, sb, nv;
  DevBuf<int64_t> rt_podidx, rt_ts, rt_start;
  DevBuf<uint8_t> rt_ev, sf, sg, ok;
  DevBuf<long long> key;
  std::vector<uint32_t> cs(N);
  for (int n = 0; n < N; ++n) cs[n] = a->pred[n] ? CS_STATIC_OK : 0u;
  const size_t RN = (size_t)R * N;
  EH_TRY(idle.put(a->idle, RN)); EH_TRY(rel.put(a->rel, RN)); EH_TRY(pip.put(a->pip, RN)); EH_TRY(cstat.put(cs.data(), N));
  EH_TRY(rt_off.put(a->rt_off, (size_t)N + 1)); EH_TRY(rt_idx.put(a->rt_idx, RT)); EH_TRY(rt_req.put(a->rt_req, (size_t)R * RT));
  EH_TRY(rt_has.put(a->rt_has, RT)); EH_TRY(rt_flags.put(a->rt_flags, RT)); EH_TRY(rt_uid.put(a->rt_uid, RT));
  EH_TRY(rt_job.put(a->rt_job, RT)); EH_TRY(rt_prio.put(a->rt_prio, RT)); EH_TRY(rt_pp.put(a->rt_pod_prio, RT));
  EH_TRY(rt_podidx.put(a->rt_podidx, RT)); EH_TRY(rt_ts.put(a->rt_ts, RT)); EH_TRY(rt_start.put(a->rt_start, RT));
  EH_TRY(rt_ev.put(a->rt_evicted, RT));
  EH_TRY(j_queue.put(a->j_queue, J)); EH_TRY(j_prio.put(a->j_prio, J)); EH_TRY(j_min.put(a->j_min, J));
  EH_TRY(j_ready.put(a->j_ready, J)); EH_TRY(j_pbe.put(a->j_pbe, J)); EH_TRY(j_rank.put(a->j_rank, J));
  EH_TRY(j_alloc.put(a->j_alloc, (size_t)R * J)); EH_TRY(j_share.put(a->j_share, J));
  EH_TRY(sa.put(nullptr, B)); EH_TRY(sb.put(nullptr, B)); EH_TRY(sf.put(nullptr, B)); EH_TRY(sg.put(nullptr, B));
  EH_TRY(ok.put(nullptr, N)); EH_TRY(nv.put(nullptr, N)); EH_TRY(key.put(nullptr, 4 * (size_t)N));
  DevBuf<uint8_t> g_bits;
  DevBuf<int32_t> g_off, g_pdb, g_allowed, d_list, d_cnt;
  if (g) {
    EH_TRY(g_bits.put(g->bits, RT)); EH_TRY(g_off.put(g->pdb_off, RT > 0 ? (size_t)RT + 1 : 0));
    EH_TRY(g_pdb.put(g->pdb, RT > 0 ? (size_t)g->pdb_off[RT] : 0)); EH_TRY(g_allowed.put(g->pdb_allowed, g->n_pdb));
  }
  if (samp_list) { EH_TRY(d_list.put(samp_list, n_samp)); EH_TRY(d_cnt.put(&n_samp, 1)); }
  vct::TopoView v;
  std::memset(&v, 0, sizeof v);
  v.R = R; v.N = N; v.J = J; v.RT = RT; v.pods_dim = a->pods_dim; v.n_plugins = a->n_plugins;
  v.task_order_prio = a->task_order_prio;
  for (int i = 0; i < a->n_plugins; ++i) { v.plugin[i] = a->plugin[i]; v.tier[i] = a->tier[i]; v.enabled[i] = a->enabled[i]; }
  v.idle = idle.d; v.rel = rel.d; v.pip = pip.d; v.rt_off = rt_off.d; v.rt_idx = rt_idx.d; v.rt_req = rt_req.d;
  v.rt_has = rt_has.d; v.rt_flags = rt_flags.d; v.rt_uid = rt_uid.d; v.rt_job = rt_job.d; v.rt_prio = rt_prio.d;
  v.rt_podidx = rt_podidx.d; v.rt_ts = rt_ts.d; v.rt_evicted = rt_ev.d; v.rt_pod_prio = rt_pp.d; v.rt_start = rt_start.d;
  v.j_queue = j_queue.d; v.j_prio = j_prio.d; v.j_min = j_min.d; v.j_ready = j_ready.d; v.j_pbe = j_pbe.d;
  v.j_rank = j_rank.d; v.j_alloc = j_alloc.d; v.j_share = j_share.d;
  for (int d = 0; d < R; ++d) v.total[d] = a->total[d];
  v.total_has = a->total_has;
  v.rt_guard = g_bits.d; v.pdb_off = g_off.d; v.pdb = g_pdb.d; v.pdb_allowed = g_allowed.d;
  vct::TopoTask t;
  eh_topo_task(*a, t);
  TopoDry s;
  s.cstat = cstat.d; s.klass = 0; s.a = sa.d; s.b = sb.d; s.f = sf.d; s.g = sg.d; s.ok = ok.d; s.nv = nv.d; s.key = key.d;
  s.samp_list = d_list.d; s.samp_cnt = d_cnt.d;
  if (N > 0) {  // the production geometry (vcalloc.cu)
    const unsigned grid = (unsigned)((N + 127) / 128);
    if (!g) k_evict_dryrun<false><<<grid, 128>>>(v, t, s);
    else if (!samp_list) k_evict_dryrun<false, true><<<grid, 128>>>(v, t, s);
    else if (n_samp > 0) k_evict_dryrun<true, true><<<grid, 128>>>(v, t, s);
    EH_TRY(cudaGetLastError());
  }
  EH_TRY(cudaDeviceSynchronize());
  EH_TRY(ok.get(a->ok, N)); EH_TRY(nv.get(a->nv, N)); EH_TRY(key.get(a->key, 4 * (size_t)N)); EH_TRY(sa.get(a->victims, RT));
  return EH_OK;
}

// one k_evict_select launch over per-node dry-run results; words[0..EV_TOPO_SEQ] receive the mapped hand-out
struct EhSelectArgs {
  int N, RT;
  const uint8_t *pred, *ok;        // [N]
  const int32_t *nv;               // [N]
  const long long *key;            // [4][N]
  const int32_t *rt_off, *victims; // [N+1], [RT]
  unsigned long long seed_k;
  int pct, min_abs, max_abs, seq;
  int32_t *words;                  // [EV_TOPO_SEQ + 1]
};

extern "C" int eh_topo_seq_word() { return EV_TOPO_SEQ; }

extern "C" int eh_select(const EhSelectArgs *a) {
  if (!a || a->N < 1 || a->RT < 0 || !a->words || a->rt_off[0] != 0 || a->rt_off[a->N] != a->RT) return EH_EINVAL;
  for (int n = 0; n < a->N; ++n)
    if (a->rt_off[n + 1] < a->rt_off[n] || (a->ok[n] && (!a->pred[n] || a->nv[n] < 1 || a->nv[n] > a->rt_off[n + 1] - a->rt_off[n])))
      return EH_EINVAL;
  const int N = a->N;
  std::vector<uint32_t> cs(N);
  for (int n = 0; n < N; ++n) cs[n] = a->pred[n] ? CS_STATIC_OK : 0u;
  DevBuf<uint32_t> cstat;
  DevBuf<uint8_t> ok;
  DevBuf<int32_t> nv, rt_off, victims;
  DevBuf<long long> key;
  EH_TRY(cstat.put(cs.data(), N)); EH_TRY(ok.put(a->ok, N)); EH_TRY(nv.put(a->nv, N)); EH_TRY(key.put(a->key, 4 * (size_t)N));
  EH_TRY(rt_off.put(a->rt_off, (size_t)N + 1)); EH_TRY(victims.put(a->victims, a->RT));
  Mapped out;
  EH_TRY(out.alloc(EV_TOPO_SEQ + 1));
  for (int i = 0; i <= EV_TOPO_SEQ; ++i) out.h[i] = -7;
  out.h[EV_TOPO_SEQ] = ~a->seq;
  TopoSelect s;
  s.cstat = cstat.d; s.klass = 0; s.N = N; s.ok = ok.d; s.nv = nv.d; s.key = key.d; s.rt_off = rt_off.d; s.victims = victims.d;
  s.seed_k = a->seed_k; s.pct = a->pct; s.min_abs = a->min_abs; s.max_abs = a->max_abs; s.out = out.d; s.seq = a->seq;
  k_evict_select<false><<<1, 1024>>>(s);
  EH_TRY(cudaGetLastError());
  EH_TRY(cudaDeviceSynchronize());
  for (int i = 0; i <= EV_TOPO_SEQ; ++i) a->words[i] = reinterpret_cast<volatile int32_t *>(out.h)[i];
  return EH_OK;
}

// ---- k_evict_samp -----------------------------------------------------------------------------------------------------
// One PredicateNodes call under sampling: static verdicts `pass` of N nodes, the filter flag, vc_conf's three sampling
// arguments and the index the call starts from. Out: list[0, *cnt) the sampled nodes in scan order, *idx the index left.
extern "C" int eh_samp(int N, const uint8_t *pass, int filtered, int pct, int min_nodes, int min_pct, int32_t start,
                       int32_t *list, int32_t *cnt, int32_t *idx) {
  if (N < 1 || !pass || !list || !cnt || !idx || start < 0) return EH_EINVAL;
  std::vector<uint32_t> cs(N);
  for (int n = 0; n < N; ++n) cs[n] = pass[n] ? CS_STATIC_OK : 0u;
  DevBuf<uint32_t> cstat;
  DevBuf<int32_t> d_list, words;  // words: [0] count, [1] index
  EH_TRY(cstat.put(cs.data(), N));
  std::vector<int32_t> fill(N, -7);
  EH_TRY(d_list.put(fill.data(), N));
  const int32_t w0[2] = {-7, start};
  EH_TRY(words.put(w0, 2));
  EvictSamp s;
  s.cstat = cstat.d; s.klass = 0; s.N = N; s.filtered = filtered ? 1 : 0;
  s.pct = pct; s.min_nodes = min_nodes; s.min_pct = min_pct;
  s.idx_in = words.d + 1; s.idx_out = words.d + 1; s.list = d_list.d; s.cnt = words.d;
  k_evict_samp<<<1, 1024>>>(s);
  EH_TRY(cudaGetLastError());
  EH_TRY(cudaDeviceSynchronize());
  int32_t w[2];
  EH_TRY(words.get(w, 2));
  EH_TRY(d_list.get(list, N));
  *cnt = w[0];
  *idx = w[1];
  return EH_OK;
}

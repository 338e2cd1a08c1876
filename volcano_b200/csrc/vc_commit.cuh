// vc_commit.cuh — K2, the persistent cooperative commit kernel.
//
// One launch per scheduling cycle executes the reference's whole allocate action
// (actions/allocate/allocate.go:283-348, :558-694) with its exact sequential semantics:
//
//   * the node axis is partitioned over the CTAs (one CTA per SM); every CTA keeps the mutable state
//     of its nodes (Idle / Used / Pipelined / k8s requested / pod count) in SHARED MEMORY for the
//     whole cycle, one node per thread, dimension-major so a warp reads consecutive banks;
//   * the control state (queue order, job order, gang counters, drf / proportion shares, Statement
//     undo log) is REPLICATED: every CTA runs the same deterministic control code on its own copy, so
//     the only cross-CTA traffic per placement is one all-gather of 48-byte records through an
//     L2-resident mailbox (no grid barrier, no broadcast hop);
//   * per task: every thread evaluates predicate + score of its node, warp-shuffle arg-max, one
//     mailbox exchange, all CTAs derive the same winner, the owner thread mutates its node row.
//
// Bound: latency (mailbox round trip + fp64 dependency chain per step), not HBM — see DESIGN.md.
#pragma once
#include "vc_device.cuh"
#include "vc_hdrf.hpp"

struct HeapEnt {  // a re-pushed job with the key it had when pushed (keys are stable inside the PQ)
  double share;
  int32_t job;
  int32_t prio;
  uint32_t rank;
  uint32_t bits;  // bit0 ready, bit1 preemptable
};

struct HdrfDev {  // device copy (global memory) of the tree (vc_hdrf.hpp), the order inputs and the per-CTA replica slab
  int on;          // the queue PQ is simulated as a Go heap under the hdrf comparator chain
  int M, n_init, R, J, Q;
  vch::HdrfOrder ord;
  const int32_t *parent, *child_off, *child, *j_node, *q_path_off, *q_path, *q_init;
  const double *weight, *j_req;
  const int32_t *q_prio;
  const uint32_t *q_rank;
  double total[VC_MAX_DIMS];
  uint32_t total_has;
  double tot0[VC_MAX_DIMS];  // drf.totalAllocated at open
  unsigned char *rep;
  size_t rep_stride;
};

struct K2Params {
  DevDims d;
  DevConf c;
  int npc;    // nodes per CTA
  int n_cta;  // CTAs that take part in the exchange (== gridDim.x)
  int max_job_tasks;
  // nodes (master copies in HBM; dynamic ones are written back at the end)
  const double *alloc, *rel, *kalloc;
  double *idle, *used, *pip, *kreq, *knz;
  const int32_t *max_tasks;
  int32_t *pod_count;
  const uint32_t *cstat;
  // tasks
  const double *req, *tkreq, *tknz;
  const uint32_t *req_has;
  const int32_t *t_class, *t_role;
  const int32_t *task_order, *job_task_off;
  const int32_t *nominated;  // [T] node index of Pod.Status.NominatedNodeName, -1 none; nullptr: no task has one
  // jobs
  const int32_t *j_queue, *j_min, *j_ntasks, *j_pbe, *j_taskmintotal, *j_roleoff, *j_prio, *j_ready0, *j_waiting0;
  const uint32_t *j_flags, *j_rank;
  const double *j_alloc0, *j_share0;
  const int32_t *r_min, *r_occ0, *r_pip0, *r_pending0;
  const uint32_t *r_flags;
  // queues
  const int32_t *q_prio;
  const uint32_t *q_rank, *q_flags, *q_alloc_has0, *q_des_has, *q_flags2;  // q_flags2: bit0 attr exists, bit1 alloc nil map
  const double *q_alloc0, *q_des, *q_share0;
  const int32_t *qjobs_off, *qjobs;
  double total[VC_MAX_DIMS];
  uint32_t total_has;
  // per-CTA replicas of the mutable control state
  int32_t *rep_i32;
  size_t rep_i32_stride;
  double *rep_f64;
  size_t rep_f64_stride;
  HeapEnt *rep_heap;
  size_t rep_heap_stride;
  // mailbox [2 parity][3 units][n_cta]
  uint4 *mbox;
  uint4 *mbox2;  // same layout: the per-CTA count all-gather of feasible-node sampling
  // outputs
  vc_decision *decisions;
  vc_visit *visits;
  int32_t *fit_errors;
  int32_t *counters;  // 0 n_decisions, 1 n_visits, 2 n_fit_errors, 3 n_steps, 4 error
  long long *prof;    // [8] phase cycle counters of CTA 0
  long long *cta_wait;  // optional [n_cta]: cycles each CTA spent inside the all-gather (the straggler waits least)
  // ---- fast (incremental) kernel ----
  const int4 *tmeta;      // per position of task_order: {task, group, role row, 0}
  int n_groups;
  const double *g_req;    // [R][G] request record of each (class, request) group
  const double *g_kreq;   // [K][G]
  const double *g_knz;    // [2][G]
  const uint32_t *g_has;
  const int32_t *g_class;
  uint4 *ring;            // publication ring, RING_DEPTH entries of RING_STRIDE uint4
  // ---- one session across several GPUs (k_commit_fast only): every rank runs the same control program over its slice
  //      of the node axis; a CTA's records go into EVERY rank's mailbox / ring through peer-mapped memory (NVLink
  //      stores), and are polled locally ----
  int n_ranks;            // 1: single GPU
  int *dbg;               // VC_PROF + VC_WATCHDOG_MS: [n_cta][8] progress words the watchdog prints (nullptr otherwise)
  long long wd_cycles;    // watchdog of the exchange polls (k_commit_fast): SM cycles without an answer before the kernel aborts
  int cta_base;           // global index of this rank's CTA 0; n_cta counts the CTAs of all ranks
  uint4 *peer_mbox[8];    // [n_ranks] the mailbox of every rank (own one included)
  uint4 *peer_ring[8];    // [n_ranks]
  // ---- network-topology-aware (general kernel only) ----
  int hn_H, hn_cap;           // hypernodes; capacity of a CTA's local hypernode list
  const int32_t *hn_member;   // [L][N] global hypernode index per tier level, -1 none
  const int32_t *hn_slot;     // [L][N] position of that hypernode in the owning CTA's local list, -1 none
  const int32_t *cta_hn_off;  // [n_cta+1] local lists: the hypernodes that hold at least one node of the CTA
  const int32_t *cta_hn;
  const int32_t *node_chain;  // [N] position, in the owning CTA's chain list, of the node's tuple of per-tier hypernodes
  const int32_t *cta_chain_off;  // [n_cta+1]
  const int32_t *cta_chain;   // [chains][L] local hypernode slot per tier level (-1 none)
  int chain_cap;              // max chains of one CTA
  const double *hn_alloc;     // [R][H] hyperNodeResourceCache allocatable
  const double *hn_used0;     // [R][H] ... used at session open
  double *rep_hn_used;        // [n_cta][R][hn_cap] per-CTA live copy of `used` for the CTA's local hypernodes
  int hn_smem;                // the CTA's hypernode tables (used, allocatable, ids) fit in shared memory
  // pods with a soft-mode network topology (k_commit<.,.,true>)
  int hn_min_tier;
  const int32_t *hn_up;       // [L][H] ancestor of hypernode h (Parent chain, h included) at tier level l, -1 none
  const int32_t *hn_tier;     // [H]
  const int32_t *hn_parent;   // [H]
  const int32_t *job_soft;    // [J] default subJob is in soft topology mode
  const int32_t *job_alloc0;  // [J] subJob.AllocatedHyperNode at open, -1 = ""
  const int32_t *placed_off;  // [J+1] capacity ranges of the per-job lists of nodes that hold a task of the job
  const int32_t *placed0;     // lists at open
  const int32_t *placed_n0;   // [J] their lengths
  int32_t *rep_placed;        // [n_cta][placed_total] per-CTA live copies
  size_t placed_total;
  int32_t *job_alloc_out;     // [J] subJob.AllocatedHyperNode after the run
  int topo_nval;              // distinct values networkTopologyAwareScore can take, ascending
  double topo_val[VC_MAX_TIERS + 2];
  // ---- hierarchical drf (vc_snapshot_set_hdrf): the queue PQ becomes a simulated Go heap ----
  int hd_on;
  const HdrfDev *hd;  // device memory
};

// Per-CTA replica of the hdrf tree and of the queue heap, and where the kernel's own replica keeps the jobs' drf state
// and the queues' proportion shares (the two kernels lay them out differently). The functions below run on one thread and
// are not inlined: the control program only pays for a call where hdrf is configured.
struct HdrfAcc {
  const double *ja; long long ja_sj, ja_sd;  // job allocation
  const double *js; long long js_sj;         // job share
  const double *qs; long long qs_q;          // proportion share of queue q
};
struct HdrfRep { double *n_alloc, *n_share, *tot; int32_t *n_sat, *j_sat, *heap, *dem; HdrfAcc *acc; };
__device__ __forceinline__ HdrfRep hd_rep(const HdrfDev *h, int lcta) {
  unsigned char *b = h->rep + (size_t)lcta * h->rep_stride;
  HdrfRep r;
  r.acc = reinterpret_cast<HdrfAcc *>(b); b += (sizeof(HdrfAcc) + 15) & ~(size_t)15;
  r.n_alloc = reinterpret_cast<double *>(b); b += (size_t)h->M * h->R * 8;
  r.n_share = reinterpret_cast<double *>(b); b += (size_t)h->M * 8;
  r.tot = reinterpret_cast<double *>(b); b += (size_t)VC_MAX_DIMS * 8;
  r.n_sat = reinterpret_cast<int32_t *>(b); b += (size_t)h->M * 4;
  r.j_sat = reinterpret_cast<int32_t *>(b); b += (size_t)h->J * 4;
  r.heap = reinterpret_cast<int32_t *>(b); b += (size_t)h->Q * 4;
  r.dem = reinterpret_cast<int32_t *>(b);
  return r;
}
__device__ __forceinline__ vch::HdrfView hd_view(const HdrfDev *h, const HdrfRep &r) {
  const HdrfAcc &a = *r.acc;
  vch::HdrfView v;
  v.R = h->R; v.M = h->M; v.J = h->J;
  v.parent = h->parent; v.child_off = h->child_off; v.child = h->child; v.j_node = h->j_node; v.j_req = h->j_req;
  v.j_alloc = a.ja; v.ja_sj = a.ja_sj; v.ja_sd = a.ja_sd; v.j_share = a.js; v.js_sj = a.js_sj;
  v.total = h->total; v.total_has = h->total_has;
  v.n_alloc = r.n_alloc; v.n_share = r.n_share; v.n_sat = r.n_sat; v.j_sat = r.j_sat; v.tot = r.tot; v.dem = r.dem;
  return v;
}
struct HdLess {  // ssn.QueueOrderFn on the replica: the hdrf / proportion chain, then the (CreationTimestamp, UID) rank
  const HdrfDev *h;
  HdrfRep r;
  __host__ __device__ int prio(int q) const { return h->q_prio[q]; }
  __host__ __device__ double share(int q) const { return r.acc->qs[q * r.acc->qs_q]; }
  __host__ __device__ uint32_t rank(int q) const { return h->q_rank[q]; }
  __host__ __device__ bool operator()(int l, int rr) const {
    return vch::hdrf_queue_less(h->ord, h->q_path_off, h->q_path, h->weight, r.n_share, r.n_sat, *this, l, rr);
  }
};
// the tree at session open and queues.Push of every queue of buildAllocateContext (allocate.go:185-188), in the order the
// queues first appear over the jobs; returns the heap size
__device__ __noinline__ int hd_open(const HdrfDev *h, int lcta, const double *ja, long long ja_sj, long long ja_sd,
                                    const double *js, long long js_sj, const double *qs, long long qs_q) {
  const HdrfRep r = hd_rep(h, lcta);
  r.acc->ja = ja; r.acc->ja_sj = ja_sj; r.acc->ja_sd = ja_sd; r.acc->js = js; r.acc->js_sj = js_sj; r.acc->qs = qs; r.acc->qs_q = qs_q;
  for (int d = 0; d < VC_MAX_DIMS; ++d) r.tot[d] = h->tot0[d];
  r.dem[0] = -1;
  vch::hdrf_refresh(hd_view(h, r), -1);
  const HdLess less{h, r};
  int n = 0;
  for (int k = 0; k < h->n_init; ++k) vch::qheap_push(r.heap, n, h->q_init[k], less);
  return n;
}
// queues.Pop() on the heap as it is (the tree is current: nothing changed since the last push)
__device__ __noinline__ int hd_pop(const HdrfDev *h, int lcta, int n) {
  const HdrfRep r = hd_rep(h, lcta);
  const HdLess less{h, r};
  return vch::qheap_pop(r.heap, n, less);
}
// drf.totalAllocated follows a visit's events (integer-valued: exact in any order)
__device__ __noinline__ void hd_tot_add(const HdrfDev *h, int lcta, int d, double delta) { hd_rep(h, lcta).tot[d] += delta; }
// queues.Push(queue) after a visit of `job` (allocate.go:346): bring the tree up to the events of the visit (the replica's
// job records and totalAllocated are already current), then sift up; returns the heap size
__device__ __noinline__ int hd_push(const HdrfDev *h, int lcta, int n, int job, int q) {
  const HdrfRep r = hd_rep(h, lcta);
  vch::hdrf_refresh(hd_view(h, r), job);
  const HdLess less{h, r};
  vch::qheap_push(r.heap, n, q, less);
  return n;
}

// ---------------------------------------------------------------------------------------
// shared-memory resident node slice of one CTA
// ---------------------------------------------------------------------------------------
struct SmemNodes {
  double *alloc, *idle, *used, *rel, *pip, *kalloc, *kreq, *knz;  // [dims][cap]
  int32_t *max_tasks, *pod_count;
  unsigned long long *nerr;  // predicate-error cache bits per role of the current visit
  int cap;
};
struct SmemNodeView {
  const SmemNodes &s;
  int i;
  __device__ __forceinline__ double alloc(int d) const { return s.alloc[d * s.cap + i]; }
  __device__ __forceinline__ double idle(int d) const { return s.idle[d * s.cap + i]; }
  __device__ __forceinline__ double used(int d) const { return s.used[d * s.cap + i]; }
  __device__ __forceinline__ double rel(int d) const { return s.rel[d * s.cap + i]; }
  __device__ __forceinline__ double pip(int d) const { return s.pip[d * s.cap + i]; }
  __device__ __forceinline__ double kalloc(int k) const { return s.kalloc[k * s.cap + i]; }
  __device__ __forceinline__ double kreq(int k) const { return s.kreq[k * s.cap + i]; }
  __device__ __forceinline__ double knz(int k) const { return s.knz[k * s.cap + i]; }
};

// ---------------------------------------------------------------------------------------
// control state of the visit in flight (shared memory, identical in every CTA)
// ---------------------------------------------------------------------------------------
struct Ctl {
  // job under allocation
  int job, queue, cursor, task_end, ready, waiting, pbe, minav, ntasks_total, taskmintotal, role_base, nroles;
  uint32_t jflags;
  double jalloc[VC_MAX_DIMS];
  double jshare;
  int r_occ[VC_MAX_JOB_ROLES], r_pip[VC_MAX_JOB_ROLES], r_pending[VC_MAX_JOB_ROLES], r_min[VC_MAX_JOB_ROLES];
  uint32_t r_flags[VC_MAX_JOB_ROLES];
  uint8_t r_failed[VC_MAX_JOB_ROLES];
  // queue attr (proportion.queueAttr)
  double qalloc[VC_MAX_DIMS], qdes[VC_MAX_DIMS];
  double qshare;
  uint32_t qalloc_has, qdes_has, qflags2, qflags;
  // task under evaluation
  TaskRec trec;
  int task, role_local;
  // soft-mode topology job: allocatedHyperNode of the visit (allocate.go:572), its Parent chain, list length
  int job_soft, topo_A, n_anc, nplaced;
  int anc[VC_MAX_TIERS + 2], anc_lvl[VC_MAX_TIERS + 2];
  int tk[2];
  // feasible-node sampling: util.lastProcessedNodeIndex, per-warp counts of the selection pass, its result
  int last_idx, samp_proc, samp_total, samp_prefA, samp_prefB;
  unsigned seq2;
  int samp_w[4][8][2];   // [row of nodes][warp][segment] feasible counts
  // exchange result
  int cnt[2], best_node[2], max_soft[2];
  double best_score[2];
  // bookkeeping
  int n_ops;
  unsigned seq;
  int n_dec, n_vis, n_fit, n_steps;
  // scratch for CTA-level reductions
  double w_score[2][32];
  int w_node[2][32];
  int w_cnt[2][32];
  int w_soft[2][32];
  long long prof[8];
  long long prof_last;
  int pick;  // scratch for warp0 -> CTA broadcasts
  int pick2;
  // ---- fast (incremental) kernel only ----
  int cmd, sweep_rl, sweep_use_cache, visit_id;
  int cur_group;     // group whose record is staged in trec
  int cache_group;   // group the per-node (cat, score) cache and the slot table describe; -1 = invalid
  int dirty_node;    // node changed by the last placement and not yet re-evaluated for cache_group; -1 none
  unsigned ag;       // all-gathers so far (mailbox parity / tag)
  unsigned pc;       // single-slot publications so far (ring index / tag)
  int since_sync;    // publications since the last all-gather (ring overrun guard)
  int n_full, n_incr;
};

// ---- mailbox --------------------------------------------------------------------------------
__device__ __forceinline__ void mbox_store(uint4 *p, uint4 v) {
  asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 mbox_load(const uint4 *p) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}

struct Local {  // what one CTA (or one lane while folding) contributes per category
  double score[2];
  int node[2];
  int cnt[2];
  int soft[2];
  int proc;   // sampling: rotated position + 1 of the to_find-th feasible node (0 = not in this part)
  int tk[2];  // topology pods: (1 + code of the best networkTopologyAwareScore) << 2 | min(nodes at that score, 2); 0 = none
};
__device__ __forceinline__ int tk_fold(int a, int b) {
  const int ca = a >> 2, cb = b >> 2;
  if (cb > ca) return b;
  if (cb < ca) return a;
  return (ca << 2) | min(2, (a & 3) + (b & 3));
}
__device__ __forceinline__ void local_init(Local &l) {
  l.score[0] = l.score[1] = 0.0;
  l.node[0] = l.node[1] = -1;
  l.cnt[0] = l.cnt[1] = 0;
  l.soft[0] = l.soft[1] = 0;
  l.tk[0] = l.tk[1] = 0;
  l.proc = 0;
}
__device__ __forceinline__ void local_fold(Local &a, const Local &b) {
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    if (b.node[k] >= 0 && (a.node[k] < 0 || better(b.score[k], b.node[k], a.score[k], a.node[k]))) {
      a.score[k] = b.score[k];
      a.node[k] = b.node[k];
    }
    a.cnt[k] += b.cnt[k];
    a.soft[k] = max(a.soft[k], b.soft[k]);
    a.tk[k] = tk_fold(a.tk[k], b.tk[k]);
  }
  a.proc = max(a.proc, b.proc);
}
// Warp-wide fold with the hardware reductions (redux.sync) instead of 5 shuffle rounds over 12 words: the
// (score, node) arg-max goes through an order-preserving 64-bit key reduced as two 32-bit maxima, then the
// lowest node among the lanes that hold the maximum (util.SelectBestNodeAndScore with the canonical tie-break).
// TWO = false skips category 1 (no FutureIdle gradient in this kernel instance).
__device__ __forceinline__ unsigned long long score_key(double x) {
  x += 0.0;  // -0.0 -> +0.0, so equal scores have equal keys
  return order_bits(x);
}
__device__ __forceinline__ double score_of_key(unsigned long long k) {
  const unsigned long long u = (k & 0x8000000000000000ull) ? (k ^ 0x8000000000000000ull) : ~k;
  return __longlong_as_double((long long)u);
}
template <bool TWO = true>
__device__ __forceinline__ void local_warp_reduce(Local &l) {
  constexpr unsigned FULLM = 0xffffffffu;
#pragma unroll
  for (int k = 0; k < (TWO ? 2 : 1); ++k) {
    const bool valid = l.node[k] >= 0;
    const unsigned long long key = valid ? score_key(l.score[k]) : 0ull;
    const unsigned hi = (unsigned)(key >> 32);
    const unsigned mhi = __reduce_max_sync(FULLM, hi);
    const unsigned lo = hi == mhi ? (unsigned)key : 0u;
    const unsigned mlo = __reduce_max_sync(FULLM, lo);
    const unsigned long long mkey = ((unsigned long long)mhi << 32) | mlo;
    const bool is_max = valid && key == mkey;
    const unsigned mnode = __reduce_min_sync(FULLM, is_max ? (unsigned)l.node[k] : 0xffffffffu);
    if (mnode == 0xffffffffu) { l.node[k] = -1; l.score[k] = 0.0; }
    else { l.node[k] = (int)mnode; l.score[k] = score_of_key(mkey); }
    l.cnt[k] = (int)__reduce_add_sync(FULLM, (unsigned)l.cnt[k]);
    // soft-taint maximum and the topology (code, count) pair share one word: soft in bits 0..7, tk above
    const unsigned tcode = (unsigned)l.tk[k] >> 2;
    const unsigned mcode = __reduce_max_sync(FULLM, tcode);
    const unsigned tcnt = __reduce_add_sync(FULLM, tcode == mcode ? ((unsigned)l.tk[k] & 3u) : 0u);
    l.tk[k] = (int)((mcode << 2) | min(2u, tcnt));
    l.soft[k] = (int)__reduce_max_sync(FULLM, (unsigned)l.soft[k]);
  }
  l.proc = (int)__reduce_max_sync(FULLM, (unsigned)l.proc);
}

// All-gather of one Local per CTA through the L2-resident mailbox. Called by warp 0 of every CTA with the
// CTA's folded contribution (identical in all lanes); returns the global fold in all lanes of warp 0.
// Each CTA owns one 256-byte block per parity (blocks of different CTAs hash to different L2 slices, so
// the G x G reads of one step spread over the whole L2 instead of hammering a few slices). A record
// carries its own sequence number, so readers validate each 16-byte unit on its own: no fence needed.
//   FULL = false: one unit  {score0, node0, seq<<2 | min(cnt0,2)}            (no FutureIdle gradient, no
//                                                                              normalising batch scorer)
//   FULL = true : four units {score0,node0,seq} {score1,node1,seq} {cnt0,cnt1,soft0|soft1<<8|tk0<<16|tk1<<24,seq}
//                 {sampling: processed position,0,0,seq}
#define MBOX_STRIDE 16  // uint4 per slot = 256 bytes
// tb_* (optional, category 0 only): every CTA's record is also kept, indexed by CTA, for callers that afterwards
// track single-CTA changes instead of gathering again (k_backfill).
template <bool FULL>
__device__ __forceinline__ Local exchange(const K2Params &p, Local mine, unsigned seq, double *tb_score = nullptr,
                                          int *tb_node = nullptr, int *tb_cnt = nullptr) {
  const int lane = threadIdx.x & 31;
  const int G = p.n_cta;
  uint4 *base = p.mbox + (size_t)(seq & 1u) * G * MBOX_STRIDE;
  if (FULL) {
    if (lane == 3) mbox_store(base + (size_t)blockIdx.x * MBOX_STRIDE + 3, make_uint4((unsigned)mine.proc, 0u, 0u, seq));
    if (lane < 3) {
      uint4 v;
      if (lane < 2) {
        unsigned long long sb = (unsigned long long)__double_as_longlong(mine.score[lane]);
        v = make_uint4((unsigned)sb, (unsigned)(sb >> 32), (unsigned)mine.node[lane], seq);
      } else {
        v = make_uint4((unsigned)mine.cnt[0], (unsigned)mine.cnt[1],
                       (unsigned)mine.soft[0] | ((unsigned)mine.soft[1] << 8) | ((unsigned)mine.tk[0] << 16) |
                           ((unsigned)mine.tk[1] << 24), seq);
      }
      mbox_store(base + (size_t)blockIdx.x * MBOX_STRIDE + lane, v);
    }
  } else if (lane == 0) {
    unsigned long long sb = (unsigned long long)__double_as_longlong(mine.score[0]);
    mbox_store(base + (size_t)blockIdx.x * MBOX_STRIDE,
               make_uint4((unsigned)sb, (unsigned)(sb >> 32), (unsigned)mine.node[0], (seq << 2) | (unsigned)min(mine.cnt[0], 2)));
  }
  Local acc;
  local_init(acc);
  for (int s0 = 0; s0 < G; s0 += 32 * 4) {  // up to 4 slots per lane in flight
    uint4 a[4], b[4], c[4], e[4];
    bool need[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) need[k] = (s0 + k * 32 + lane) < G;
    bool pending;
    do {
      pending = false;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (need[k]) {  // the three units of a slot share one 128-byte line: issue them together
          const uint4 *sl = base + (size_t)(s0 + k * 32 + lane) * MBOX_STRIDE;
          a[k] = mbox_load(sl);
          if (FULL) { b[k] = mbox_load(sl + 1); c[k] = mbox_load(sl + 2); e[k] = mbox_load(sl + 3); }
        }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (!need[k]) continue;
        const bool ok = FULL ? (a[k].w == seq && b[k].w == seq && c[k].w == seq && e[k].w == seq)
                             : ((a[k].w >> 2) == (seq & 0x3fffffffu));
        if (!ok) { pending = true; continue; }
        Local o;
        local_init(o);
        o.score[0] = __longlong_as_double((long long)((unsigned long long)a[k].x | ((unsigned long long)a[k].y << 32)));
        o.node[0] = (int)a[k].z;
        if (FULL) {
          o.score[1] = __longlong_as_double((long long)((unsigned long long)b[k].x | ((unsigned long long)b[k].y << 32)));
          o.node[1] = (int)b[k].z;
          o.cnt[0] = (int)c[k].x; o.cnt[1] = (int)c[k].y;
          o.soft[0] = (int)(c[k].z & 0xffu); o.soft[1] = (int)((c[k].z >> 8) & 0xffu);
          o.tk[0] = (int)((c[k].z >> 16) & 0xffu); o.tk[1] = (int)(c[k].z >> 24);
          o.proc = (int)e[k].x;
        } else {
          o.cnt[0] = (int)(a[k].w & 3u);
        }
        if (tb_score) {
          const int slot = s0 + k * 32 + lane;
          tb_score[slot] = o.score[0]; tb_node[slot] = o.node[0]; tb_cnt[slot] = o.cnt[0];
        }
        local_fold(acc, o);
        need[k] = false;
      }
    } while (pending);
  }
  local_warp_reduce<FULL>(acc);
  if (!FULL) acc.cnt[0] = min(acc.cnt[0], 2);
  return acc;
}

// All-gather of two counts per CTA (feasible nodes at / after the scan start, and before it) for the feasible-node
// sampling: returns in every lane of warp 0 the sums over the CTAs with a lower index, and the totals.
struct CountFold { int prefA, prefB, totA, totB; };
__device__ __forceinline__ CountFold exchange_counts(const K2Params &p, int cA, int cB, unsigned seq) {
  const int lane = threadIdx.x & 31;
  const int G = p.n_cta, me = blockIdx.x;
  uint4 *base = p.mbox2 + (size_t)(seq & 1u) * G * MBOX_STRIDE;
  if (lane == 0) mbox_store(base + (size_t)me * MBOX_STRIDE, make_uint4((unsigned)cA, (unsigned)cB, 0u, seq));
  int pa = 0, pb = 0, ta = 0, tb = 0;
  for (int s = lane; s < G; s += 32) {
    uint4 v;
    do { v = mbox_load(base + (size_t)s * MBOX_STRIDE); } while (v.w != seq);
    ta += (int)v.x; tb += (int)v.y;
    if (s < me) { pa += (int)v.x; pb += (int)v.y; }
  }
  CountFold r;
  r.prefA = (int)__reduce_add_sync(0xffffffffu, (unsigned)pa);
  r.prefB = (int)__reduce_add_sync(0xffffffffu, (unsigned)pb);
  r.totA = (int)__reduce_add_sync(0xffffffffu, (unsigned)ta);
  r.totB = (int)__reduce_add_sync(0xffffffffu, (unsigned)tb);
  return r;
}

// ---- replicated control helpers (executed by every thread on shared Ctl; mutations by thread 0) ----
__device__ __forceinline__ bool ctl_is_ready(const Ctl &s) { return s.ready + s.pbe >= s.minav; }            // job_info.go:1169
__device__ __forceinline__ bool ctl_is_pipelined(const Ctl &s) { return s.waiting + s.ready + s.pbe >= s.minav; }  // :1173
__device__ __forceinline__ bool ctl_check_task_ready(const Ctl &s) {  // job_info.go:1024-1036
  if (s.minav < s.taskmintotal) return true;
  for (int r = 0; r < s.nroles; ++r)
    if ((s.r_flags[r] & VC_ROLE_IN_MIN_MAP) && s.r_occ[r] < s.r_min[r]) return false;
  return true;
}
__device__ __forceinline__ bool ctl_check_task_pipelined(const Ctl &s) {  // job_info.go:1039-1070
  if (s.minav < s.taskmintotal) return true;
  for (int r = 0; r < s.nroles; ++r)
    if ((s.r_flags[r] & VC_ROLE_IN_MIN_MAP) && s.r_occ[r] + s.r_pip[r] < s.r_min[r]) return false;
  return true;
}
__device__ __forceinline__ bool ctl_job_ready(const DevConf &c, const Ctl &s) {  // session_plugins.go:428-446
  for (int i = 0; i < c.n_plugins; ++i)
    if ((c.enabled[i] & VC_EN_JOB_READY) && c.plugin[i] == VC_PLUGIN_GANG)
      if (!(ctl_check_task_ready(s) && ctl_is_ready(s))) return false;
  return true;
}
__device__ __forceinline__ bool ctl_job_pipelined(const DevConf &c, const Ctl &s) {  // session_plugins.go:450-478
  bool has_found = false;
  int i = 0;
  while (i < c.n_plugins) {
    int tier = c.tier[i];
    for (; i < c.n_plugins && c.tier[i] == tier; ++i) {
      if (!(c.enabled[i] & VC_EN_JOB_PIPELINED)) continue;
      int res;
      if (c.plugin[i] == VC_PLUGIN_GANG) res = (ctl_check_task_pipelined(s) && ctl_is_pipelined(s)) ? 1 : -1;
      else if (c.plugin[i] == VC_PLUGIN_TDM) res = ctl_is_pipelined(s) ? 1 : -1;
      else continue;
      if (res < 0) return false;
      if (res > 0) has_found = true;
    }
    if (has_found) return true;
  }
  return true;
}
__device__ __forceinline__ bool ctl_need_continue(const Ctl &s) {  // job_info.go:918-966
  if (s.minav >= s.ntasks_total) return false;
  if (s.minav < s.taskmintotal) {
    int left = 0;
    for (int r = 0; r < s.nroles; ++r)
      if (!s.r_failed[r]) left += s.r_pending[r];
    return s.ready + left >= s.minav;
  }
  for (int r = 0; r < s.nroles; ++r) {
    if (!s.r_failed[r]) continue;
    int mn = (s.r_flags[r] & VC_ROLE_IN_MIN_MAP) ? s.r_min[r] : 0;
    if (mn == 0) continue;
    if (s.r_occ[r] < mn) return false;
  }
  return true;
}
__device__ __forceinline__ double share_of(double l, double r) {  // api/helpers/helpers.go:80-93
  if (r == 0.0) return l == 0.0 ? 0.0 : 1.0;
  return l / r;
}
__device__ __forceinline__ double drf_share(const K2Params &p, const double *jalloc) {  // drf.go:566-578
  double res = 0.0;
  for (int d = 0; d < p.d.R; ++d) {
    if (d >= 2 && !(p.total_has & (1u << d))) continue;
    if (!(p.total[d] >= VC_MIN_RESOURCE)) continue;
    double sh = share_of(jalloc[d], p.total[d]);
    if (sh > res) res = sh;
  }
  return res;
}
__device__ __forceinline__ double queue_share(int R, const double *qalloc, uint32_t alloc_has, const double *qdes,
                                              uint32_t des_has) {  // proportion.go:590-602
  double res = 0.0;
  for (int d = 0; d < R; ++d) {
    if (d >= 2 && !(des_has & (1u << d))) continue;
    if (!(qdes[d] >= VC_MIN_RESOURCE)) continue;
    double al = (d < 2 || (alloc_has & (1u << d))) ? qalloc[d] : 0.0;
    double sh = share_of(al, qdes[d]);
    if (sh > res) res = sh;
  }
  return res;
}
// proportion queueAllocatable (proportion.go:333-348) through ssn.Allocatable (session_plugins.go:350-366)
__device__ __forceinline__ bool ctl_allocatable(const K2Params &p, const Ctl &s) {
  const DevConf &c = p.c;
  for (int i = 0; i < c.n_plugins; ++i) {
    if (!(c.enabled[i] & VC_EN_ALLOCATABLE) || c.plugin[i] != VC_PLUGIN_PROPORTION) continue;
    if (!(s.qflags & VC_QUEUE_OPEN)) return false;
    const TaskRec &t = s.trec;
    bool ok = true;
    if (t.req[0] > 0.0 && s.qalloc[0] + t.req[0] > s.qdes[0]) ok = false;
    if (t.req[1] > 0.0 && s.qalloc[1] + t.req[1] > s.qdes[1]) ok = false;
    const uint32_t rq_has = t.has & ~3u;
    const bool fu_nil = (s.qflags2 & 2u) && rq_has == 0;
    if (!fu_nil) {
      for (int d = 2; d < p.d.R; ++d) {
        if (!(rq_has & (1u << d)) || d == p.d.pods_dim) continue;
        double al = (s.qalloc_has & (1u << d)) ? s.qalloc[d] : 0.0;
        double fu = al + t.req[d];
        double de = (s.qdes_has & (1u << d)) ? s.qdes[d] : 0.0;
        if (t.req[d] > 0.0 && fu > de) ok = false;
      }
    }
    if (!ok) return false;
  }
  return true;
}

// ssn.JobOrderFn (session_plugins.go:660-683) on (static keys, ready, share)
struct JobKey {
  double share;
  int prio;
  uint32_t rank;
  bool ready, preempt;
};
__device__ __forceinline__ bool job_less(const DevConf &c, const JobKey &l, const JobKey &r) {
  for (int i = 0; i < c.n_plugins; ++i) {
    if (!(c.enabled[i] & VC_EN_JOB_ORDER)) continue;
    int cmp = 0;
    switch (c.plugin[i]) {
      case VC_PLUGIN_PRIORITY: cmp = l.prio > r.prio ? -1 : (l.prio < r.prio ? 1 : 0); break;
      case VC_PLUGIN_GANG: cmp = (l.ready && r.ready) ? 0 : (l.ready ? 1 : (r.ready ? -1 : 0)); break;
      case VC_PLUGIN_DRF: cmp = l.share == r.share ? 0 : (l.share < r.share ? -1 : 1); break;
      case VC_PLUGIN_TDM: cmp = l.preempt == r.preempt ? 0 : (!l.preempt ? -1 : 1); break;
      default: break;
    }
    if (cmp != 0) return cmp < 0;
  }
  return l.rank < r.rank;  // (CreationTimestamp, UID) rank precomputed on the host
}
__device__ __forceinline__ JobKey key_of(const HeapEnt &e) {
  JobKey k;
  k.share = e.share; k.prio = e.prio; k.rank = e.rank; k.ready = e.bits & 1u; k.preempt = (e.bits & 2u) != 0;
  return k;
}

// =======================================================================================
// the kernel
// =======================================================================================
extern __shared__ __align__(16) unsigned char k2_smem[];

// phase timers (cycles, CTA 0 / thread 0): 0 queue+job control, 1 task fetch + gates, 2 node sweep,
// 3 mailbox exchange, 4 apply + bookkeeping
#define PROF_MARK(k)                                  \
  do {                                                \
    if (tid == 0 && cta == 0) {                       \
      long long now_ = clock64();                     \
      S.prof[k] += now_ - S.prof_last;                \
      S.prof_last = now_;                             \
    }                                                 \
  } while (0)

template <bool FUT, bool SOFT, bool TOPO = false, bool SAMP = false>
__global__ void __launch_bounds__(256, 1) k_commit(K2Params p) {
  static_assert(!TOPO || (FUT && SOFT), "the topology variant rides on the two-pass, three-unit exchange");
  static_assert(!SAMP || (FUT && SOFT), "the sampling variant rides on the full exchange");
  const DevConf &c = p.c;
  const int R = p.d.R, K = p.d.K, N = p.d.N, J = p.d.J, Q = p.d.Q, NR = p.d.NR, T = p.d.T;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int cta = blockIdx.x;
  const int nbase = p.d.node_begin + cta * p.npc;
  const int nmine = max(0, min(p.npc, p.d.node_end - nbase));
  const int cap = p.npc;

  // ---- carve shared memory ----
  unsigned char *sp = k2_smem;
  Ctl &S = *reinterpret_cast<Ctl *>(sp);
  sp += (sizeof(Ctl) + 15) & ~(size_t)15;
  SmemNodes sn;
  sn.cap = cap;
  auto take = [&](int rows) { double *q = reinterpret_cast<double *>(sp); sp += (size_t)rows * cap * sizeof(double); return q; };
  sn.alloc = take(R); sn.idle = take(R); sn.used = take(R);
  sn.rel = c.has_future ? take(R) : nullptr;
  sn.pip = c.has_future ? take(R) : nullptr;
  sn.kalloc = take(K); sn.kreq = take(K); sn.knz = take(2);
  sn.nerr = reinterpret_cast<unsigned long long *>(sp); sp += (size_t)cap * 8;
  sn.max_tasks = reinterpret_cast<int32_t *>(sp); sp += (size_t)cap * 4;
  sn.pod_count = reinterpret_cast<int32_t *>(sp); sp += (size_t)cap * 4;
  // verdict cache: (fit category, NodeOrderFn sum) of node i for the (class, request) group c_group[i]; an entry dies
  // when the node's state changes (placement / rollback), so a sweep re-evaluates only what a placement touched
  sp = reinterpret_cast<unsigned char *>(((uintptr_t)sp + 7) & ~(uintptr_t)7);
  double *c_order = reinterpret_cast<double *>(sp); sp += (size_t)cap * 8;
  int32_t *c_group = reinterpret_cast<int32_t *>(sp); sp += (size_t)cap * 4;
  uint8_t *c_cat = reinterpret_cast<uint8_t *>(sp); sp += (size_t)cap;
  uint8_t *s_samp = reinterpret_cast<uint8_t *>(sp); sp += (size_t)cap;  // sampling: 1 candidate / feasible, 2 evaluated infeasible, 4 skipped
  for (int i = tid; i < cap; i += blockDim.x) c_group[i] = -1;
  // network-topology-aware: per-step binpack score of each local hypernode for the task under evaluation, and
  // the plugin's score of each distinct per-tier hypernode tuple ("chain") among the CTA's nodes
  sp = reinterpret_cast<unsigned char *>(((uintptr_t)sp + 7) & ~(uintptr_t)7);
  double *hn_score = reinterpret_cast<double *>(sp); sp += (size_t)p.hn_cap * 8;
  double *chain_val = reinterpret_cast<double *>(sp); sp += (size_t)p.chain_cap * 8;
  int32_t *s_chain = reinterpret_cast<int32_t *>(sp); sp += (size_t)cap * 4;  // node -> chain of the CTA
  int32_t *s_chain_slots = reinterpret_cast<int32_t *>(sp);                 // [chain][L] local hypernode slots
  const int chain_base = c.nta_on ? p.cta_chain_off[cta] : 0;
  const int chain_n = c.nta_on ? p.cta_chain_off[cta + 1] - chain_base : 0;
  if (c.nta_on) {
    for (int i = tid; i < nmine; i += blockDim.x) s_chain[i] = p.node_chain[nbase + i];
    for (int k = tid; k < chain_n * c.nta_L; k += blockDim.x) s_chain_slots[k] = p.cta_chain[(size_t)chain_base * c.nta_L + k];
  }
  const int hn_cap = p.hn_cap;
  const int hn_base = c.nta_tables ? p.cta_hn_off[cta] : 0;
  const int hn_n = c.nta_tables ? p.cta_hn_off[cta + 1] - hn_base : 0;
  // live `used` of the CTA's hypernodes: shared memory when the local list is short (the usual tree), else an
  // L2-resident per-CTA replica
  double *hn_used = c.nta_tables ? p.rep_hn_used + (size_t)cta * R * hn_cap : nullptr;
  const double *hn_alloc_l = nullptr;  // [R][hn_cap] allocatable of the local hypernodes (shared-memory copy)
  const int32_t *hn_ids = p.cta_hn + hn_base;
  double *hn_term = nullptr;  // [hn_cap][R] scratch of the per-step hypernode scores
  uint8_t *hn_flag = nullptr;
  if (c.nta_tables && p.hn_smem) {
    sp = reinterpret_cast<unsigned char *>(((uintptr_t)(s_chain_slots + (size_t)p.chain_cap * c.nta_L) + 7) & ~(uintptr_t)7);
    hn_used = reinterpret_cast<double *>(sp); sp += (size_t)R * hn_cap * 8;
    double *al = reinterpret_cast<double *>(sp); sp += (size_t)R * hn_cap * 8;
    int32_t *ids = reinterpret_cast<int32_t *>(sp); sp += (size_t)hn_cap * 4;
    sp = reinterpret_cast<unsigned char *>(((uintptr_t)sp + 7) & ~(uintptr_t)7);
    hn_term = reinterpret_cast<double *>(sp); sp += (size_t)R * hn_cap * 8;
    hn_flag = reinterpret_cast<uint8_t *>(sp);
    for (int k = tid; k < hn_n; k += blockDim.x) {
      const int h = p.cta_hn[hn_base + k];
      ids[k] = h;
      for (int d = 0; d < R; ++d) al[d * hn_cap + k] = p.hn_alloc[(size_t)d * p.hn_H + h];
    }
    hn_alloc_l = al;
    hn_ids = ids;
  }
  for (int k = tid; k < hn_n; k += blockDim.x) {
    const int h = p.cta_hn[hn_base + k];
    for (int d = 0; d < R; ++d) hn_used[d * hn_cap + k] = p.hn_used0[(size_t)d * p.hn_H + h];
  }
  // event handlers of the plugin (network_topology_aware.go:374-399): used += / -= Resreq for every hypernode
  // whose RealNodesSet holds the node; each CTA maintains the entries of its own local list
  auto hn_account = [&](int node, const double *req, size_t req_stride, uint32_t has, double sign) {
    for (int k = tid; k < hn_n; k += blockDim.x) {
      const int h = hn_ids[k];
      bool hit = false;
#pragma unroll
      for (int l = 0; l < VC_MAX_TIERS; ++l)  // independent loads: no short-circuit between the tier levels
        if (l < c.nta_L) hit |= __ldg(&p.hn_member[(size_t)l * N + node]) == h;
      if (!hit) continue;
      for (int d = 0; d < R; ++d) {
        if (d >= 2 && !(has & (1u << d))) continue;
        hn_used[d * hn_cap + k] += sign * req[d * req_stride];
      }
    }
  };

  for (int i = tid; i < nmine; i += blockDim.x) {
    const int n = nbase + i;
    for (int d = 0; d < R; ++d) {
      sn.alloc[d * cap + i] = p.alloc[(size_t)d * N + n];
      sn.idle[d * cap + i] = p.idle[(size_t)d * N + n];
      sn.used[d * cap + i] = p.used[(size_t)d * N + n];
      if (c.has_future) {
        sn.rel[d * cap + i] = p.rel[(size_t)d * N + n];
        sn.pip[d * cap + i] = p.pip[(size_t)d * N + n];
      }
    }
    for (int k = 0; k < K; ++k) {
      sn.kalloc[k * cap + i] = p.kalloc[(size_t)k * N + n];
      sn.kreq[k * cap + i] = p.kreq[(size_t)k * N + n];
    }
    for (int k = 0; k < 2; ++k) sn.knz[k * cap + i] = p.knz[(size_t)k * N + n];
    sn.max_tasks[i] = p.max_tasks[n];
    sn.pod_count[i] = p.pod_count[n];
    sn.nerr[i] = 0ull;
  }

  // ---- per-CTA replica of the control state ----
  int32_t *ri = p.rep_i32 + (size_t)cta * p.rep_i32_stride;
  double *rf = p.rep_f64 + (size_t)cta * p.rep_f64_stride;
  HeapEnt *heap = p.rep_heap + (size_t)cta * p.rep_heap_stride;
  int32_t *j_ready = ri; ri += J;
  int32_t *j_waiting = ri; ri += J;
  int32_t *j_cursor = ri; ri += J;
  int32_t *r_occ = ri; ri += NR;
  int32_t *r_pip = ri; ri += NR;
  int32_t *r_pending = ri; ri += NR;
  int32_t *r_failed = ri; ri += NR;
  int32_t *q_active = ri; ri += Q;      // queue is in the queue PQ
  int32_t *q_scursor = ri; ri += Q;     // cursor into the static, pre-sorted job list of the queue
  int32_t *q_hsize = ri; ri += Q;       // size of the dynamic heap of re-pushed jobs
  uint32_t *q_alloc_has = reinterpret_cast<uint32_t *>(ri); ri += Q;
  uint32_t *q_flags2 = reinterpret_cast<uint32_t *>(ri); ri += Q;
  int32_t *j_alloc_hn = ri; ri += J;    // subJob.AllocatedHyperNode of soft-mode topology jobs
  int32_t *j_nplaced = ri; ri += J;     // length of the job's placed-node list
  int32_t *ops = ri; ri += (size_t)p.max_job_tasks * 3;  // task, node, kind
  double *j_share = rf; rf += J;
  double *j_alloc = rf; rf += (size_t)R * J;
  double *q_alloc = rf; rf += (size_t)R * Q;
  double *q_share = rf; rf += Q;
  double *ops_score = rf; rf += p.max_job_tasks;

  for (int j = tid; j < J; j += blockDim.x) {
    j_ready[j] = p.j_ready0[j];
    j_waiting[j] = p.j_waiting0[j];
    j_cursor[j] = 0;
    j_share[j] = p.j_share0[j];
    for (int d = 0; d < R; ++d) j_alloc[(size_t)d * J + j] = p.j_alloc0[(size_t)d * J + j];
    j_alloc_hn[j] = TOPO ? p.job_alloc0[j] : -1;
    j_nplaced[j] = TOPO ? p.placed_n0[j] : 0;
  }
  int32_t *placed = TOPO ? p.rep_placed + (size_t)cta * p.placed_total : nullptr;
  if (TOPO)
    for (size_t i = tid; i < p.placed_total; i += blockDim.x) placed[i] = p.placed0[i];
  for (int r = tid; r < NR; r += blockDim.x) {
    r_occ[r] = p.r_occ0[r];
    r_pip[r] = p.r_pip0[r];
    r_pending[r] = p.r_pending0[r];
    r_failed[r] = 0;
  }
  for (int q = tid; q < Q; q += blockDim.x) {
    q_active[q] = (p.qjobs_off[q + 1] > p.qjobs_off[q]) ? 1 : 0;  // buildAllocateContext: queues with a job
    q_scursor[q] = 0;
    q_hsize[q] = 0;
    q_alloc_has[q] = p.q_alloc_has0[q];
    q_flags2[q] = p.q_flags2[q];
    q_share[q] = p.q_share0[q];
    for (int d = 0; d < R; ++d) q_alloc[(size_t)d * Q + q] = p.q_alloc0[(size_t)d * Q + q];
  }
  if (tid == 0) {
    S.seq = 0;
    S.seq2 = 0;
    S.last_idx = c.last_idx0;
    S.n_dec = S.n_vis = S.n_fit = S.n_steps = 0;
    for (int k = 0; k < 8; ++k) S.prof[k] = 0;
    S.prof_last = clock64();
  }
  __syncthreads();
  // hdrf: the queue PQ is a simulated Go heap (thread 0), its comparator reads the tree replica
  int hd_n = 0;
  if (p.hd_on && tid == 0) hd_n = hd_open(p.hd, cta, j_alloc, 1, J, j_share, 1, q_share, 1);

  const bool out_cta = (cta == 0);  // CTA 0 writes the result lists
  const bool qorder_prop = [&] {
    for (int i = 0; i < c.n_plugins; ++i)
      if ((c.enabled[i] & VC_EN_QUEUE_ORDER) && c.plugin[i] == VC_PLUGIN_PROPORTION) return true;
    return false;
  }();
  const bool overused_prop = [&] {
    for (int i = 0; i < c.n_plugins; ++i)
      if ((c.enabled[i] & VC_EN_OVERUSED) && c.plugin[i] == VC_PLUGIN_PROPORTION) return true;
    return false;
  }();

  // =====================================================================================
  // allocateResources loop, allocate.go:283-348
  // =====================================================================================
  for (;;) {
    // ---- queues.Pop(): arg-min over the active queues by ssn.QueueOrderFn (session_plugins.go:709-731;
    //      proportion: priority desc, then share asc — proportion.go:266-284; then (ts, uid) rank)
    if (p.hd_on) {
      if (tid == 0) {
        S.pick = hd_n > 0 ? hd_pop(p.hd, cta, hd_n) : -1;
        hd_n = hd_n > 0 ? hd_n - 1 : 0;
      }
    } else if (warp == 0) {
      int bq = -1, bprio = 0;
      double bshare = 0.0;
      uint32_t brank = 0;
      for (int q = lane; q < Q; q += 32) {
        if (!q_active[q]) continue;
        int pr = qorder_prop ? p.q_prio[q] : 0;
        double sh = qorder_prop ? q_share[q] : 0.0;
        uint32_t rk = p.q_rank[q];
        bool lt = bq < 0 || pr > bprio || (pr == bprio && (sh < bshare || (sh == bshare && rk < brank)));
        if (lt) { bq = q; bprio = pr; bshare = sh; brank = rk; }
      }
      for (int o = 16; o; o >>= 1) {
        int oq = __shfl_xor_sync(0xffffffffu, bq, o);
        int opr = __shfl_xor_sync(0xffffffffu, bprio, o);
        double osh = __shfl_xor_sync(0xffffffffu, bshare, o);
        uint32_t ork = __shfl_xor_sync(0xffffffffu, brank, o);
        bool lt = oq >= 0 && (bq < 0 || opr > bprio || (opr == bprio && (osh < bshare || (osh == bshare && ork < brank))));
        if (lt) { bq = oq; bprio = opr; bshare = osh; brank = ork; }
      }
      if (lane == 0) S.pick = bq;
    }
    __syncthreads();
    const int q = S.pick;
    if (q < 0) break;
    __syncthreads();

    // ---- load the queue attr; ssn.Overused (proportion.go:319-331); jobs.Pop() ----
    if (tid == 0) {
      q_active[q] = 0;
      S.queue = q;
      S.qflags = p.q_flags[q];
      S.qflags2 = q_flags2[q];
      S.qalloc_has = q_alloc_has[q];
      S.qdes_has = p.q_des_has[q];
      S.qshare = q_share[q];
      for (int d = 0; d < R; ++d) {
        S.qalloc[d] = q_alloc[(size_t)d * Q + q];
        S.qdes[d] = p.q_des[(size_t)d * Q + q];
      }
      bool over = false;
      if (overused_prop && (S.qflags2 & 1u)) {
        // attr.deserved.LessEqual(attr.allocated, Zero), resource_info.go:429-463
        over = le_eps(S.qdes[0], S.qalloc[0]) && le_eps(S.qdes[1], S.qalloc[1]);
        for (int d = 2; d < R && over; ++d) {
          if (!(S.qdes_has & (1u << d))) continue;
          double rv = (S.qalloc_has & (1u << d)) ? S.qalloc[d] : 0.0;
          if (!le_eps(S.qdes[d], rv)) over = false;
        }
      }
      int j = -1;
      if (!over) {
        // jobs.Pop(): the better of (front of the static sorted list, top of the dynamic heap)
        const int sbeg = p.qjobs_off[q], send = p.qjobs_off[q + 1];
        const int sc = sbeg + q_scursor[q];
        HeapEnt *h = heap + sbeg;
        int hs = q_hsize[q];
        bool have_s = sc < send, have_h = hs > 0;
        bool take_heap = false;
        if (have_s && have_h) {
          int js = p.qjobs[sc];
          JobKey ks;
          ks.share = j_share[js]; ks.prio = p.j_prio[js]; ks.rank = p.j_rank[js];
          ks.ready = j_ready[js] + p.j_pbe[js] >= p.j_min[js];
          ks.preempt = (p.j_flags[js] & VC_JOB_PREEMPTABLE) != 0;
          take_heap = job_less(c, key_of(h[0]), ks);
        } else if (have_h) {
          take_heap = true;
        }
        if (take_heap) {
          j = h[0].job;
          HeapEnt last = h[--hs];
          q_hsize[q] = hs;
          int i = 0;  // sift-down
          for (;;) {
            int l = 2 * i + 1;
            if (l >= hs) break;
            int m = l;
            if (l + 1 < hs && job_less(c, key_of(h[l + 1]), key_of(h[l]))) m = l + 1;
            if (!job_less(c, key_of(h[m]), key_of(last))) break;
            h[i] = h[m];
            i = m;
          }
          if (hs > 0) h[i] = last;
        } else if (have_s) {
          j = p.qjobs[sc];
          q_scursor[q] += 1;
        }
      }
      S.job = j;  // -1: queue dropped (overused, or no jobs left)
      if (j >= 0) {
        S.cursor = p.job_task_off[j] + j_cursor[j];
        S.task_end = p.job_task_off[j + 1];
        S.ready = j_ready[j];
        S.waiting = j_waiting[j];
        S.pbe = p.j_pbe[j];
        S.minav = p.j_min[j];
        S.ntasks_total = p.j_ntasks[j];
        S.taskmintotal = p.j_taskmintotal[j];
        S.jflags = p.j_flags[j];
        S.role_base = p.j_roleoff[j];
        S.nroles = p.j_roleoff[j + 1] - p.j_roleoff[j];
        S.jshare = j_share[j];
        for (int d = 0; d < R; ++d) S.jalloc[d] = j_alloc[(size_t)d * J + j];
        for (int r = 0; r < S.nroles; ++r) {
          int gr = S.role_base + r;
          S.r_occ[r] = r_occ[gr]; S.r_pip[r] = r_pip[gr]; S.r_pending[r] = r_pending[gr];
          S.r_min[r] = p.r_min[gr]; S.r_flags[r] = p.r_flags[gr]; S.r_failed[r] = (uint8_t)r_failed[gr];
        }
        S.n_ops = 0;
        S.job_soft = TOPO ? p.job_soft[j] : 0;
        S.topo_A = TOPO ? j_alloc_hn[j] : -1;  // allocatedHyperNode := subJob.AllocatedHyperNode, allocate.go:572
        S.nplaced = TOPO ? j_nplaced[j] : 0;
      }
    }
    for (int i = tid; i < nmine; i += blockDim.x) sn.nerr[i] = 0ull;  // util.NewPredicateHelper()
    __syncthreads();
    if (S.job < 0) continue;
    const int j = S.job;

    // =================================================================================
    // allocateResourcesForTasks, allocate.go:558-694
    // =================================================================================
    for (;;) {
      if (S.cursor >= S.task_end || N == 0) break;  // tasks.Empty(); no nodes: return nil (allocate.go:563-567)
      PROF_MARK(4);
      // ---- tasks.Pop() + task record ----
      const int t = p.task_order[S.cursor];
      __syncthreads();
      if (tid < R) S.trec.req[tid] = p.req[(size_t)tid * T + t];
      if (tid >= 32 && tid < 32 + K) S.trec.kreq[tid - 32] = p.tkreq[(size_t)(tid - 32) * T + t];
      if (tid >= 64 && tid < 66) S.trec.knz[tid - 64] = p.tknz[(size_t)(tid - 64) * T + t];
      if (tid == 96 % blockDim.x) {
        S.trec.has = p.req_has[t];
        S.trec.klass = p.t_class[t];
        S.task = t;
        S.role_local = p.t_role[t] - S.role_base;
        S.cur_group = p.tmeta[S.cursor].y;
        S.cursor += 1;
      }
      __syncthreads();
      const int rl = S.role_local;
      if (!ctl_allocatable(p, S)) continue;  // allocate.go:575-578
      const bool named_role = !(S.r_flags[rl] & VC_ROLE_EMPTY_NAME);
      if (named_role && S.r_failed[rl]) {  // job.TaskHasFitErrors, allocate.go:600-607
        if (out_cta && tid == 0) p.fit_errors[S.n_fit] = t;
        __syncthreads();
        if (tid == 0) S.n_fit += 1;
        __syncthreads();
        continue;
      }
      const bool use_cache = c.enable_ecache && named_role;
      const int cur_group = S.cur_group;

      // ---- ph.PredicateNodes + alloc.prioritizeNodes over this CTA's nodes ----
      const TaskRec &trec = S.trec;
      const uint32_t *cs_row = p.cstat + (size_t)trec.klass * N + nbase;
      PROF_MARK(1);
      // With a normalising batch scorer (SOFT) two passes are needed: pass 0 = categories, counts and the
      // max soft-taint count of the candidate set; pass 1 = scores.
      int g_soft0 = 0, g_soft1 = 0;
      // pods of a soft-mode topology job are scored by batchNodeOrderFnForNetworkAwarePods (:541-571) with
      // task.JobAllocatedHyperNode = the visit's allocatedHyperNode; no entries at all while that is ""
      const bool topo_task = TOPO && S.job_soft != 0 && c.nta_plugin;
      const bool topo_scored = topo_task && S.topo_A >= 0;
      const int H = p.hn_H;
      if (TOPO && topo_scored) {
        if (tid == 0) {  // GetAncestors(jobAllocatedHyperNode), api/hyper_node_info.go:737-758
          int na = 0;
          for (int h = S.topo_A; h >= 0 && na < VC_MAX_TIERS + 2; h = p.hn_parent[h]) {
            S.anc[na] = h;
            S.anc_lvl[na] = p.hn_tier[h] - p.hn_min_tier;
            ++na;
          }
          S.n_anc = na;
        }
        // FindJobTaskNumOfHyperNode for the CTA's lowest-tier hypernodes: tasks of the job by NodeName
        for (int k = tid; k < hn_n; k += blockDim.x) hn_score[k] = 0.0;
        __syncthreads();
        const int32_t *lst = placed + p.placed_off[j];
        for (int m = tid; m < S.nplaced; m += blockDim.x) {
          const int h = p.hn_member[lst[m]];
          if (h < 0) continue;
          for (int k = 0; k < hn_n; ++k)
            if (hn_ids[k] == h) atomicAdd(&hn_score[k], 1.0);
        }
        __syncthreads();
      }
      // 1 + index into topo_val of networkTopologyAwareScore(FindHyperNodeForNode(node), allocated) :716-756
      auto topo_code = [&](int n) -> int {
        const int hn = p.hn_member[n];  // util.FindHyperNodeForNode: lowest tier only
        double sc = 0.0;
        if (hn >= 0) {
          if (hn == S.topo_A) {
            sc = 1.0;
          } else {  // GetLCAHyperNode: first ancestor of the allocated hypernode that is an ancestor of hn
            for (int i = 0; i < S.n_anc; ++i) {
              if (p.hn_up[(size_t)S.anc_lvl[i] * H + hn] != S.anc[i]) continue;
              const int min_t = p.hn_min_tier, max_t = p.hn_min_tier + c.nta_L - 1, tier = S.anc_lvl[i] + p.hn_min_tier;
              sc = min_t == max_t ? 1.0 : (double)(max_t - tier) / (double)(max_t - min_t);
              break;
            }
          }
        }
        int code = 1;
        for (int v = 0; v < p.topo_nval; ++v)
          if (p.topo_val[v] == sc) code = v + 1;
        return code;
      };
      if (c.nta_on && !topo_task) {  // getPodHyperNodeBinPackingScore(task, hypernode) for the CTA's hypernodes
        if (hn_term) {
          // one thread per (hypernode, resource): the division of every term in parallel, then the terms are
          // summed per hypernode in resource order exactly as the scalar loop does
          for (int idx = tid; idx < hn_n * R; idx += blockDim.x) {
            const int k = idx / R, d = idx - k * R;
            const double request = trec.req[d];
            const int w = c.nta_dim_weight[d];
            const bool on = (d < 2 || (trec.has & (1u << d))) && request >= VC_MIN_RESOURCE && w >= 0;
            double term = 0.0;
            uint8_t flag = 0;
            if (on) {
              const double u = hn_used[d * hn_cap + k], al = hn_alloc_l[d * hn_cap + k];
              if (u + request > al) flag = 3;
              else { flag = 1; term = (double)w * ((u + request) / al); }
            }
            hn_term[idx] = term;
            hn_flag[idx] = flag;
          }
          __syncthreads();
          for (int k = tid; k < hn_n; k += blockDim.x) {
            double total = 0.0;
            int wsum = 0;
            bool over = false;
            for (int d = 0; d < R; ++d) {
              const uint8_t f = hn_flag[k * R + d];
              if (!(f & 1)) continue;
              if (f & 2) { over = true; break; }
              total += hn_term[k * R + d];
              wsum += c.nta_dim_weight[d];
            }
            hn_score[k] = (over || wsum <= 0) ? 0.0 : total / (double)wsum;
          }
        } else {
          for (int k = tid; k < hn_n; k += blockDim.x) {
            const int h = hn_ids[k];
            hn_score[k] = hn_binpack_score(
                c, R, trec, [&](int d) { return hn_used[d * hn_cap + k]; },
                [&](int d) { return hn_alloc_l ? hn_alloc_l[d * hn_cap + k] : p.hn_alloc[(size_t)d * p.hn_H + h]; });
          }
        }
        __syncthreads();
        for (int k = tid; k < chain_n; k += blockDim.x) {  // batchNodeOrderFnForNormalPods per distinct chain
          const int32_t *sl = s_chain_slots + (size_t)k * c.nta_L;
          chain_val[k] = nta_node_score(c, [&](int l) { return sl[l] < 0 ? 1.0 : hn_score[sl[l]]; });
        }
        __syncthreads();
      }
      // cached or fresh (fit category, NodeOrderFn sum) of node i for the staged group
      auto verdict = [&](int i, uint32_t cs, int *cat, bool *has_order, double *order) {
        *cat = 2; *has_order = false; *order = 0.0;
        if (c_group[i] == cur_group) {
          const uint8_t cw = c_cat[i];
          *cat = cw & 3; *has_order = (cw & 0x80) != 0; *order = c_order[i];
          return;
        }
        SmemNodeView nv{sn, i};
        bool ok = (cs & CS_STATIC_OK) != 0;
        if (c.pred_predicates && sn.max_tasks[i] <= sn.pod_count[i]) ok = false;
        const int fc = fit_category_t<FUT>(R, trec, nv);
        if (ok && fc != 2) {
          *cat = fc;
          *has_order = node_order(c, R, K, trec, nv, cs, order);
        }
        c_group[i] = cur_group; c_cat[i] = (uint8_t)(*cat | (*has_order ? 0x80 : 0)); c_order[i] = *order;
      };
      // ---- feasible-node sampling, util/predicate_helper.go:43-140 in its single-worker reading: scan the nodes in
      // index order starting at lastProcessedNodeIndex, stop after `to_find` feasible ones; nodes skipped through the
      // error cache count as processed, predicate failures of processed nodes enter the cache ----
      // ---- Pod.Status.NominatedNodeName (set by a preemption of an earlier cycle), allocate.go:624-634: when the node is in
      //      the session and InitResreq <= its FutureIdle, ph.PredicateNodes runs on that ONE node first; a pass makes it the
      //      only candidate (taken without scoring), anything else falls back to the search over all nodes. With
      //      feasible-node sampling that call also leaves util.lastProcessedNodeIndex at (start + processed) % 1 = 0. ----
      bool nom_hit = false;
      const int nom = p.nominated ? p.nominated[t] : -1;
      if (nom >= 0) {
        if (tid < 32) {  // warp 0: the owner lane evaluates, everybody exchanges
          Local l;
          local_init(l);
          const int i = nom - nbase;
          if (lane == 0 && i >= 0 && i < nmine) {
            SmemNodeView nv{sn, i};
            if (fit_category_t<FUT>(R, trec, nv) != 2) {  // task.InitResreq.LessEqual(nominatedNodeInfo.FutureIdle(), Zero)
              l.proc = 1;                                   // PredicateNodes is called
              if (!(use_cache && ((sn.nerr[i] >> rl) & 1ull))) {
                int cat; bool ho; double od;
                verdict(i, cs_row[i], &cat, &ho, &od);
                if (cat == 2) { if (use_cache) sn.nerr[i] |= (1ull << rl); }
                else { l.cnt[cat] = 1; l.node[cat] = nom; l.score[cat] = 0.0; }
              }
            }
          }
          local_warp_reduce<FUT>(l);
          l.proc = (int)__reduce_max_sync(0xffffffffu, (unsigned)l.proc);
          const unsigned seq = S.seq + 1;
          __syncwarp();
          Local g = exchange<true>(p, l, seq);  // the full record: it carries `proc` (the tags of the two record formats cannot be mistaken for each other)
          if (lane == 0) {
            S.seq = seq;
#pragma unroll
            for (int k = 0; k < 2; ++k) { S.cnt[k] = g.cnt[k]; S.best_node[k] = g.node[k]; S.best_score[k] = g.score[k]; S.max_soft[k] = 0; }
            if (g.proc > 0) S.last_idx = 0;  // (start + processedNodes) % len([nominated]) whatever the sampling mode
          }
        }
        __syncthreads();
        nom_hit = S.cnt[0] + S.cnt[1] > 0;
      }
      const bool sampling = SAMP && c.to_find > 0;
      if (!nom_hit) {
      if (SAMP && sampling) {
        const int start = S.last_idx, Kf = c.to_find;
        const int rows = (cap + (int)blockDim.x - 1) / (int)blockDim.x;
        const unsigned lt = (1u << lane) - 1u;
        for (int row = 0; row < rows; ++row) {
          const int i = row * blockDim.x + tid;
          int flag = 0;
          if (i < nmine) {
            if (use_cache && ((sn.nerr[i] >> rl) & 1ull)) {
              flag = 4;
            } else {
              int cat; bool ho; double od;
              verdict(i, c_group[i] != cur_group ? cs_row[i] : 0u, &cat, &ho, &od);
              flag = cat != 2 ? 1 : 2;
            }
            s_samp[i] = (uint8_t)flag;
          }
          const bool inA = nbase + i >= start;
          const unsigned mA = __ballot_sync(0xffffffffu, flag == 1 && inA), mB = __ballot_sync(0xffffffffu, flag == 1 && !inA);
          if (lane == 0) { S.samp_w[row][warp][0] = __popc(mA); S.samp_w[row][warp][1] = __popc(mB); }
        }
        __syncthreads();
        if (warp == 0) {
          int a = 0, b = 0;
          for (int e = lane; e < rows * nwarps; e += 32) { a += S.samp_w[e / nwarps][e % nwarps][0]; b += S.samp_w[e / nwarps][e % nwarps][1]; }
          a = (int)__reduce_add_sync(0xffffffffu, (unsigned)a);
          b = (int)__reduce_add_sync(0xffffffffu, (unsigned)b);
          const unsigned seq2 = S.seq2 + 1;
          __syncwarp();
          const CountFold f = exchange_counts(p, a, b, seq2);
          if (lane == 0) {
            S.seq2 = seq2;
            S.samp_prefA = f.prefA;            // feasible nodes before this CTA's part of the [start, N) segment
            S.samp_prefB = f.totA + f.prefB;   // ... of the [0, start) segment, which is scanned second
            S.samp_total = f.totA + f.totB;
            S.samp_proc = 0;
          }
        }
        __syncthreads();
        for (int row = 0; row < rows; ++row) {
          const int i = row * blockDim.x + tid;
          const int flag = i < nmine ? s_samp[i] : 0;
          const bool inA = nbase + i >= start;
          const unsigned mA = __ballot_sync(0xffffffffu, flag == 1 && inA), mB = __ballot_sync(0xffffffffu, flag == 1 && !inA);
          if (i >= nmine || flag == 4) continue;
          // feasible nodes scanned before this one: lower-index CTAs, earlier rows / warps of this CTA, lower lanes
          const int seg = inA ? 0 : 1;
          int before = (inA ? S.samp_prefA : S.samp_prefB) + __popc((inA ? mA : mB) & lt);
          for (int r2 = 0; r2 <= row; ++r2)
            for (int w2 = 0; w2 < (r2 < row ? nwarps : warp); ++w2) before += S.samp_w[r2][w2][seg];
          if (flag == 1) {
            const bool cand = before < Kf;
            s_samp[i] = cand ? 1 : 0;
            if (before == Kf - 1) S.samp_proc = (nbase + i - start + N) % N + 1;  // the scan stops here
          } else if (before < Kf && use_cache) {
            sn.nerr[i] |= (1ull << rl);  // a processed node that failed the predicate
          }
        }
        __syncthreads();
      }
      // the first pass is only needed when something is normalised over the candidate set
      const bool two_pass = SOFT && (c.soft_active || (TOPO && topo_scored));
      const int n_pass = two_pass ? 2 : 1;
      for (int pass = 0; pass < n_pass; ++pass) {
        Local mine;
        local_init(mine);
        for (int i = tid; i < nmine; i += blockDim.x) {
          // the class x node word is only needed to (re)evaluate the node or for the soft-taint count
          const uint32_t cs = ((SOFT && c.soft_active) || c_group[i] != cur_group) ? cs_row[i] : 0u;
          int cat = 2;
          bool has_order = false;
          double order = 0.0;
          if (SAMP && sampling) {
            if (s_samp[i] != 1) continue;  // outside the sampled candidate set
            verdict(i, cs, &cat, &has_order, &order);
          } else if (!(use_cache && ((sn.nerr[i] >> rl) & 1ull))) {
            verdict(i, cs, &cat, &has_order, &order);
            if (cat == 2 && use_cache && pass == 0) sn.nerr[i] |= (1ull << rl);
          }
          if (cat == 2) continue;
          const int soft = SOFT ? (int)((cs >> CS_SOFT_SHIFT) & 0xff) : 0;
          const bool c0 = !FUT || cat == 0;
          if (c0) { mine.cnt[0] += 1; mine.soft[0] = max(mine.soft[0], soft); }
          else { mine.cnt[1] += 1; mine.soft[1] = max(mine.soft[1], soft); }
          int tcode = 0;
          if (TOPO && topo_scored) {
            tcode = topo_code(nbase + i);
            if (pass == 0) mine.tk[c0 ? 0 : 1] = tk_fold(mine.tk[c0 ? 0 : 1], (tcode << 2) | 1);
          }
          if (two_pass && pass == 0) continue;
          const int n = nbase + i;
          double nta = 0.0;
          if (TOPO && topo_task) {
            if (topo_scored) {
              const int gk = S.tk[c0 ? 0 : 1];
              double tsc = p.topo_val[tcode - 1];
              if (tcode == (gk >> 2) && (gk & 3) > 1) {  // several nodes share the best score: + taskNum / allTaskNum
                const int k = p.hn_slot[n];
                const double cntv = k < 0 ? 0.0 : hn_score[k];
                if (S.ntasks_total > 0) tsc += cntv / (double)S.ntasks_total;
              }
              nta = (double)VC_MAX_NODE_SCORE * (double)c.nta_weight * tsc;  // scaleFinalScore :758-764
            }
          } else if (c.nta_on) {
            nta = chain_val[s_chain[i]];
          }
          double sc = total_score(c, has_order, order, soft, c0 ? g_soft0 : g_soft1, nta);
          if (c0) {
            if (mine.node[0] < 0 || better(sc, n, mine.score[0], mine.node[0])) { mine.score[0] = sc; mine.node[0] = n; }
          } else {
            if (mine.node[1] < 0 || better(sc, n, mine.score[1], mine.node[1])) { mine.score[1] = sc; mine.node[1] = n; }
          }
        }
        // CTA-level fold
        local_warp_reduce<FUT>(mine);
        if (lane == 0) {
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            S.w_score[k][warp] = mine.score[k]; S.w_node[k][warp] = mine.node[k];
            S.w_cnt[k][warp] = mine.cnt[k]; S.w_soft[k][warp] = mine.soft[k] | (mine.tk[k] << 8);
          }
        }
        __syncthreads();
        PROF_MARK(2);
        if (warp == 0) {
          Local l;
          local_init(l);
          if (lane < nwarps) {
#pragma unroll
            for (int k = 0; k < 2; ++k) {
              l.score[k] = S.w_score[k][lane]; l.node[k] = S.w_node[k][lane];
              l.cnt[k] = S.w_cnt[k][lane]; l.soft[k] = S.w_soft[k][lane] & 0xff; l.tk[k] = S.w_soft[k][lane] >> 8;
            }
          }
          local_warp_reduce<FUT>(l);
          if (SAMP && sampling) l.proc = S.samp_proc;
          const unsigned seq = S.seq + 1;
          __syncwarp();  // every lane has read S.seq before lane 0 advances it below
          const long long tw0 = p.cta_wait ? clock64() : 0;
          Local g = exchange<(FUT || SOFT)>(p, l, seq);
          if (p.cta_wait && lane == 0) p.cta_wait[cta] += clock64() - tw0;
          if (lane == 0) {
            S.seq = seq;
#pragma unroll
            for (int k = 0; k < 2; ++k) {
              S.cnt[k] = g.cnt[k]; S.best_node[k] = g.node[k]; S.best_score[k] = g.score[k]; S.max_soft[k] = g.soft[k];
              if (two_pass && pass == 0) S.tk[k] = g.tk[k];
            }
            if (SAMP && sampling && pass == n_pass - 1) {  // lastProcessedNodeIndex = (start + processedNodes) % N
              const int processed = S.samp_total >= c.to_find ? g.proc : N;
              S.last_idx = (S.last_idx + processed) % N;
            }
          }
          PROF_MARK(3);
        }
        __syncthreads();
        g_soft0 = S.max_soft[0];
        g_soft1 = S.max_soft[1];
        if (S.cnt[0] + S.cnt[1] == 0) break;
      }
      }  // !nom_hit
      if (tid == 0) S.n_steps += 1;

      if (S.cnt[0] + S.cnt[1] == 0) {  // no feasible node, allocate.go:639-659
        if (out_cta && tid == 0) p.fit_errors[S.n_fit] = t;
        __syncthreads();
        if (tid == 0) { S.n_fit += 1; S.r_failed[rl] = 1; }
        __syncthreads();
        if (ctl_need_continue(S)) continue;
        break;
      }
      // ---- gradient choice (allocate.go:750-776) and allocateResourcesForTask (:780-814) ----
      const int cat = S.cnt[0] > 0 ? 0 : 1;
      const int best = S.best_node[cat];
      const double score = S.cnt[cat] == 1 ? 0.0 : S.best_score[cat];
      const int kind = cat == 0 ? VC_OP_ALLOCATE : VC_OP_PIPELINE;
      // owner thread: node.AddTask, api/node_info.go:435-484
      if (best >= nbase && best < nbase + nmine) {
        const int i = best - nbase;
        if ((i % blockDim.x) == tid) {
          c_group[i] = -1;
          if (kind == VC_OP_ALLOCATE) {
            for (int d = 0; d < R; ++d) {
              sn.idle[d * cap + i] -= trec.req[d];
              sn.used[d * cap + i] += trec.req[d];
            }
          } else {
            for (int d = 0; d < R; ++d) sn.pip[d * cap + i] += trec.req[d];
          }
          if (c.has_predicates) {  // predicates AllocateFunc: k8s NodeInfo.AddPodInfo, predicates.go:212-256
            sn.pod_count[i] += 1;
            for (int k = 0; k < K; ++k) sn.kreq[k * cap + i] += trec.kreq[k];
            for (int k = 0; k < 2; ++k) sn.knz[k * cap + i] += trec.knz[k];
          }
        }
      }
      if (c.nta_on) hn_account(best, trec.req, 1, trec.has, 1.0);
      __syncthreads();
      // job.UpdateTaskStatus (job_info.go:651-660) + event handlers (drf.go:391-418, proportion.go:475-497):
      // warp 0, one resource dimension per lane (the same IEEE operations as the scalar helpers drf_share /
      // queue_share: every share is >= 0, so the running `if (sh > res)` maximum is a lane-wise fmax)
      if (warp == 0) {
        if (lane == 0) {
          S.r_pending[rl] -= 1;
          if (kind == VC_OP_ALLOCATE) { S.r_occ[rl] += 1; S.ready += 1; }
          else { S.r_pip[rl] += 1; S.waiting += 1; }
          const int k = S.n_ops;
          ops[k * 3 + 0] = t; ops[k * 3 + 1] = best; ops[k * 3 + 2] = kind;
          ops_score[k] = score;
          S.n_ops = k + 1;
        }
        if (c.has_drf) {
          double sh = 0.0;
          if (lane < R) {
            const double a = S.jalloc[lane] + trec.req[lane];
            S.jalloc[lane] = a;
            if ((lane < 2 || (p.total_has & (1u << lane))) && p.total[lane] >= VC_MIN_RESOURCE) sh = share_of(a, p.total[lane]);
          }
          for (int o = 16; o; o >>= 1) sh = fmax(sh, __shfl_xor_sync(0xffffffffu, sh, o));
          if (lane == 0) S.jshare = sh;
        }
        if (c.has_proportion && (S.qflags2 & 1u)) {
          const uint32_t add_has = trec.has & ~3u & ((R >= 32) ? ~0u : ((1u << R) - 1u));
          const uint32_t new_has = S.qalloc_has | add_has;
          double sh = 0.0;
          if (lane < R) {
            double al = S.qalloc[lane];
            if (lane < 2 || (add_has & (1u << lane))) { al += trec.req[lane]; S.qalloc[lane] = al; }
            if ((lane < 2 || (S.qdes_has & (1u << lane))) && S.qdes[lane] >= VC_MIN_RESOURCE)
              sh = share_of((lane < 2 || (new_has & (1u << lane))) ? al : 0.0, S.qdes[lane]);
          }
          for (int o = 16; o; o >>= 1) sh = fmax(sh, __shfl_xor_sync(0xffffffffu, sh, o));
          __syncwarp();
          if (lane == 0) {
            S.qalloc_has = new_has;
            if (add_has) S.qflags2 &= ~2u;
            S.qshare = sh;
          }
        }
      }
      if (TOPO && tid == 32 && S.job_soft) {
        placed[p.placed_off[j] + S.nplaced] = best;  // task.NodeName = hostname
        S.nplaced += 1;
        // getNewAllocatedHyperNode, allocate.go:697-707
        const int hn = p.hn_member[best];
        if (hn >= 0) {
          if (S.topo_A < 0) {
            S.topo_A = hn;
          } else {
            int lca = -1;
            for (int a = S.topo_A, guard = 0; a >= 0 && guard < VC_MAX_TIERS + 2; a = p.hn_parent[a], ++guard)
              if (p.hn_up[(size_t)(p.hn_tier[a] - p.hn_min_tier) * p.hn_H + hn] == a) { lca = a; break; }
            S.topo_A = lca;
          }
        }
      }
      __syncthreads();
      if (ctl_job_ready(c, S)) break;  // ssn.SubJobReady, allocate.go:676-678
    }

    PROF_MARK(4);
    // ---- statement outcome, allocate.go:681-693 and :330-337 ----
    const bool ready = N != 0 && ctl_job_ready(c, S);
    const bool stmt = N != 0 && (ready || ctl_job_pipelined(c, S));
    const int n_ops = S.n_ops;
    __syncthreads();
    if (!stmt && n_ops > 0) {
      // stmt.Discard(): undo in reverse order (statement.go:357-381)
      for (int k = n_ops - 1; k >= 0; --k) {
        const int ot = ops[k * 3 + 0], on = ops[k * 3 + 1], okind = ops[k * 3 + 2];
        if (c.nta_on) hn_account(on, p.req + ot, (size_t)T, p.req_has[ot], -1.0);
        if (on >= nbase && on < nbase + nmine && ((on - nbase) % blockDim.x) == tid) {
          const int i = on - nbase;
          c_group[i] = -1;
          for (int d = 0; d < R; ++d) {
            double rq = p.req[(size_t)d * T + ot];
            if (okind == VC_OP_ALLOCATE) { sn.idle[d * cap + i] += rq; sn.used[d * cap + i] -= rq; }
            else sn.pip[d * cap + i] -= rq;
          }
          if (c.has_predicates) {
            sn.pod_count[i] -= 1;
            for (int kk = 0; kk < K; ++kk) sn.kreq[kk * cap + i] -= p.tkreq[(size_t)kk * T + ot];
            for (int kk = 0; kk < 2; ++kk) sn.knz[kk * cap + i] -= p.tknz[(size_t)kk * T + ot];
          }
        }
        if (tid == 0) {
          const int orl = p.t_role[ot] - S.role_base;
          S.r_pending[orl] += 1;
          if (okind == VC_OP_ALLOCATE) { S.r_occ[orl] -= 1; S.ready -= 1; }
          else { S.r_pip[orl] -= 1; S.waiting -= 1; }
          if (c.has_drf)
            for (int d = 0; d < R; ++d) S.jalloc[d] -= p.req[(size_t)d * T + ot];
          if (c.has_proportion && (S.qflags2 & 1u)) {
            const uint32_t oh = p.req_has[ot];
            S.qalloc[0] -= p.req[(size_t)0 * T + ot];
            S.qalloc[1] -= p.req[(size_t)1 * T + ot];
            if (!(S.qflags2 & 2u))
              for (int d = 2; d < R; ++d)
                if (oh & (1u << d)) { S.qalloc[d] -= p.req[(size_t)d * T + ot]; S.qalloc_has |= 1u << d; }
          }
        }
      }
      if (tid == 0) {
        if (c.has_drf) S.jshare = drf_share(p, S.jalloc);
        if (c.has_proportion && (S.qflags2 & 1u)) S.qshare = queue_share(R, S.qalloc, S.qalloc_has, S.qdes, S.qdes_has);
        if (TOPO && S.job_soft) S.nplaced -= n_ops;  // unallocate / UnPipeline: task.NodeName = ""
      }
    }
    __syncthreads();
    if (tid == 0) {
      // write the job / queue state back into the replica
      j_ready[j] = S.ready;
      j_waiting[j] = S.waiting;
      j_cursor[j] = S.cursor - p.job_task_off[j];
      j_share[j] = S.jshare;
      if (TOPO) {
        j_nplaced[j] = S.nplaced;
        if (ready && S.job_soft) j_alloc_hn[j] = S.topo_A;  // subJob.AllocatedHyperNode = allocatedHyperNode, :681-686
      }
      if (p.hd_on)
        for (int d = 0; d < R; ++d) hd_tot_add(p.hd, cta, d, S.jalloc[d] - j_alloc[(size_t)d * J + j]);
      for (int d = 0; d < R; ++d) j_alloc[(size_t)d * J + j] = S.jalloc[d];
      for (int r = 0; r < S.nroles; ++r) {
        int gr = S.role_base + r;
        r_occ[gr] = S.r_occ[r]; r_pip[gr] = S.r_pip[r]; r_pending[gr] = S.r_pending[r]; r_failed[gr] = S.r_failed[r];
      }
      for (int d = 0; d < R; ++d) q_alloc[(size_t)d * Q + q] = S.qalloc[d];
      q_alloc_has[q] = S.qalloc_has;
      q_flags2[q] = S.qflags2;
      q_share[q] = S.qshare;
      // results (CTA 0)
      if (out_cta) {
        vc_visit v;
        v.job = j;
        v.outcome = stmt ? (ready ? VC_VISIT_COMMIT : VC_VISIT_KEEP) : VC_VISIT_DISCARD;
        v.first_op = S.n_dec;
        v.n_ops = stmt ? n_ops : 0;
        p.visits[S.n_vis] = v;
      }
      if (stmt) {
        if (out_cta)
          for (int k = 0; k < n_ops; ++k) {
            vc_decision dcs;
            dcs.task = ops[k * 3 + 0]; dcs.node = ops[k * 3 + 1]; dcs.kind = ops[k * 3 + 2];
            dcs.visit = S.n_vis; dcs.score = ops_score[k];
            p.decisions[S.n_dec + k] = dcs;
          }
        S.n_dec += n_ops;
      }
      S.n_vis += 1;
      // jobs.Push(job) when committed and tasks remain (allocate.go:334-336)
      if (stmt && ready && S.cursor < S.task_end) {
        HeapEnt e;
        e.share = S.jshare; e.job = j; e.prio = p.j_prio[j]; e.rank = p.j_rank[j];
        e.bits = (ctl_is_ready(S) ? 1u : 0u) | ((S.jflags & VC_JOB_PREEMPTABLE) ? 2u : 0u);
        HeapEnt *h = heap + p.qjobs_off[q];
        int i = q_hsize[q]++;
        while (i > 0) {  // sift-up
          int par = (i - 1) / 2;
          if (!job_less(c, key_of(e), key_of(h[par]))) break;
          h[i] = h[par];
          i = par;
        }
        h[i] = e;
      }
      q_active[q] = 1;  // queues.Push(queue), allocate.go:346
      if (p.hd_on) hd_n = hd_push(p.hd, cta, hd_n, j, q);
    }
    __syncthreads();
    PROF_MARK(0);
  }

  // ---- epilogue: node state back to HBM, counters ----
  for (int i = tid; i < nmine; i += blockDim.x) {
    const int n = nbase + i;
    for (int d = 0; d < R; ++d) {
      p.idle[(size_t)d * N + n] = sn.idle[d * cap + i];
      p.used[(size_t)d * N + n] = sn.used[d * cap + i];
      if (c.has_future) p.pip[(size_t)d * N + n] = sn.pip[d * cap + i];
    }
    for (int k = 0; k < K; ++k) p.kreq[(size_t)k * N + n] = sn.kreq[k * cap + i];
    for (int k = 0; k < 2; ++k) p.knz[(size_t)k * N + n] = sn.knz[k * cap + i];
    p.pod_count[n] = sn.pod_count[i];
  }
  if (TOPO && out_cta)
    for (int j = tid; j < J; j += blockDim.x) p.job_alloc_out[j] = j_alloc_hn[j];
  if (out_cta && tid == 0) {
    p.counters[0] = S.n_dec;
    p.counters[1] = S.n_vis;
    p.counters[2] = S.n_fit;
    p.counters[3] = S.n_steps;
    p.counters[4] = S.last_idx;
    for (int k = 0; k < 8; ++k) p.prof[k] = S.prof[k];
  }
}

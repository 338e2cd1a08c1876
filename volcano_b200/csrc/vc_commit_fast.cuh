// vc_commit_fast.cuh — K2f, the incremental variant of the persistent commit kernel.
//
// Same exact semantics as k_commit (vc_commit.cuh), for the common session shape: no normalising batch scorer, no
// feasible-node sampling, no hypernode scores, R <= 8. The FUT instance serves sessions with Releasing / Pipelined
// resources (terminating pods, pipelined tasks): a node's verdict is then 0 (fits Idle: allocate), 1 (fits only
// FutureIdle = Idle + Releasing - Pipelined: pipeline) or 2, and a candidate of category 0 beats every candidate of
// category 1 (prioritizeNodes' idle gradient first, allocate.go:750-776). The SOFT instance serves sessions with
// PreferNoSchedule taints and the TaintToleration batch scorer: that score is normalised by the largest count of
// intolerable soft taints over the candidate set (DefaultNormalizeScore, reverse), a constant per category that only
// moves when a node holding the maximum leaves the set; the owner flags that event in its publication and the next
// task takes a full (two-phase) sweep. The SAMP instance serves feasible-node sampling (percentage-nodes-to-find < 100,
// util/predicate_helper.go:43-140 in its single-worker reading): a task's candidates are the first numNodesToFind
// feasible nodes in index order from the rotating start - a window that covers whole CTAs (whose cached bests already
// sit in every CTA's slot table) plus a part of its first and of its last CTA; only those two scan their cache and
// publish, every CTA folds two ring records and a few slots. (Sessions whose jobs need the role-keyed error cache, the
// normalising batch scorer or several GPUs stay on k_commit.) It exploits the one structural fact of the greedy loop: a placement changes ONE node, so between
// two consecutive tasks with the same (class, request) record every other (task, node) verdict and score
// is unchanged. Per CTA it keeps, for the group being placed,
//     c_cat[i], c_score[i], c_cs[i]   verdict, total score, static word of each of its nodes (shared memory)
//     sl_score/node/cnt[cta]          every CTA's current best (score, node) + #candidates   (shared memory)
//     cta best / global best          maintained incrementally, rescanned only when the holder got worse
// and then a step is:
//     group changed  -> full sweep: every thread re-evaluates its node, all-gather of the CTA bests
//     same group     -> the CTA that owns the node changed by the previous placement re-evaluates that one
//                       node and PUBLISHES one 16-byte record into a ring in L2; every other CTA reads that
//                       single record. The owner never waits for anybody, so a run of placements inside one
//                       CTA proceeds at shared-memory speed and the L2 round trip is only paid when the
//                       winner moves to another CTA.
// Control state is replicated exactly as in k_commit, packed in per-job / per-queue records so that one
// visit costs a handful of L2 round trips (lanes of warp 0 load a record in one coalesced access). Only
// warp 0 of each CTA runs the control program; the other warps sleep on the block barrier and serve full
// sweeps / rollbacks on command.
#pragma once
#include "vc_commit.cuh"

#define RING_DEPTH 1024
#define RING_STRIDE 4  // uint4 per ring entry (64 bytes: one entry per cache line)
#define CMD_SWEEP 1
#define CMD_DISCARD 2
#define CMD_EXIT 3
#define CMD_EVAL 4
#define CMD_RUN 5
#define CMD_SWEEP2 6  // SOFT: second phase of a full sweep (totals under the exchanged normalisation constants)
#define RUN_MAX 32  // placements one publication can cover (one lane of the evaluator warp per node state)
#define VC_JOBX_PURE 0x100u  // host-computed: every named role of the job maps to a single group
#define FAST_R 8

struct JobStatic {  // 64 B, read-only
  int32_t min_available, n_tasks_total, pending_besteffort, task_min_total;
  int32_t role_off, n_roles, priority;
  uint32_t flags;
  uint32_t rank;
  int32_t task_off, task_end, queue;
  unsigned long long key_pre, key_post;  // packed static part of the ssn.JobOrderFn key (see HeapKey)
};
struct JobDyn {  // 96 B, per-CTA replica
  int32_t ready, waiting, cursor, pad;
  double share;
  double alloc[FAST_R];
  double pad2;
};
struct RoleStatic { int32_t min; uint32_t flags; };
struct RoleDyn { int32_t occ, pip, pending, failed; };
struct QueueStatic {  // 80 B
  int32_t prio;
  uint32_t rank, flags, des_has;
  double des[FAST_R];
};
struct QueueDyn {  // 96 B
  uint32_t alloc_has, flags2;
  int32_t active, scursor, hsize, pad;
  double share;
  double alloc[FAST_R];
};
static_assert(sizeof(JobStatic) == 64 && sizeof(JobDyn) == 96 && sizeof(QueueStatic) == 80 && sizeof(QueueDyn) == 96, "record layout");

// ssn.JobOrderFn (session_plugins.go:660-683) as one lexicographic integer key: the comparators enabled in
// the conf, in plugin order, packed MSB-first — priority (dense rank of the value, higher first), gang
// readiness bit, drf share (raw bits of a non-negative double), tdm preemptable bit — then the
// (CreationTimestamp, UID) rank. Built on the host for the static parts; the ready bit and the share are
// the only dynamic components and only change while the job is outside the queue.
struct HeapKey {  // 32 B
  unsigned long long pre, share, post;
  int job, pad;
};
__device__ __forceinline__ bool hk_less(const HeapKey &a, const HeapKey &b) {
  if (a.pre != b.pre) return a.pre < b.pre;
  if (a.share != b.share) return a.share < b.share;
  return a.post < b.post;
}

struct FastParams {  // extra kernel arguments of the fast kernel
  const int32_t *heap_off;  // [Q+1] capacity prefix of the per-queue heaps of re-pushed jobs
  int ready_word;           // 0: readiness not compared, 1: bit lives in key.pre, 2: in key.post
  int ready_shift;
  int share_on;             // drf JobOrderFn enabled
  int heap_in_smem;         // the heaps fit in shared memory
  int heap_total;
  const JobStatic *jstat;
  const RoleStatic *rstat;
  const QueueStatic *qstat;
  const double *q_share0;  // [Q]
  int run_max;             // 1: one placement per publication; RUN_MAX: run-length batches (rows integer-valued)
  uint4 *score_log;        // [T] per placement attempt inside a run: (score bits lo, hi, attempt index + 1, 0), written by the
                           // owner CTA as one 16-byte store and polled by CTA 0 - the tag makes a fence before the record unnecessary
  // per-group verdict table (nullptr: the session is over the table's memory budget and re-enters a group with a full
  // sweep): category and score of every (group, node of this rank) as they were when the group's cache was last current
  uint8_t *vt_cat;         // [n_groups][gridDim.x * npc]
  double *vt_score;        // [n_groups][gridDim.x * npc]
  int32_t *vt_gstamp;      // [gridDim.x][n_groups] per-CTA replica of the group stamps (-1: no saved verdicts this cycle)
};
// Above this many changed rows in a CTA, a re-entry evaluates them one per thread (one pass, like a full sweep) instead of
// in warp-cooperative rounds of 2 rows per warp
#define VT_DIRTY_MAX 32

struct FastSmem {
  double *alloc, *idle, *used, *kalloc, *kreq, *knz;
  double *rel, *pip;  // FUT instance only
  int32_t *max_tasks, *pod_count, *nerr_stamp, *c_cat;
  uint32_t *c_cs;
  unsigned long long *nerr;
  double *c_score;
  double *sl_score;
  int32_t *sl_node, *sl_cnt, *sl_cat;
  int32_t *sl_feas;  // SAMP: feasible nodes (category 0 or 1) of every CTA for the cached group
  int32_t *mstamp;   // value of the control program's verdict clock at the last change of each row
  int32_t *dlist;    // rows a re-entry re-evaluates
  int cap;
};
struct FastNodeView {
  const FastSmem &s;
  int i;
  __device__ __forceinline__ double alloc(int d) const { return s.alloc[d * s.cap + i]; }
  __device__ __forceinline__ double idle(int d) const { return s.idle[d * s.cap + i]; }
  __device__ __forceinline__ double used(int d) const { return s.used[d * s.cap + i]; }
  __device__ __forceinline__ double kalloc(int k) const { return s.kalloc[k * s.cap + i]; }
  __device__ __forceinline__ double kreq(int k) const { return s.kreq[k * s.cap + i]; }
  __device__ __forceinline__ double knz(int k) const { return s.knz[k * s.cap + i]; }
};

struct Best {
  double score;
  int node;
  int cnt;  // candidates of category `cat`
  int cat;  // fit category of the candidate: 0 idle-fit, 1 future-idle-fit (always 0 outside the FUT instance)
};
// (cat, score, node) order: the idle gradient first, then the higher score, then the lower node index
__device__ __forceinline__ bool better_c(int cat, double s, int n, int bcat, double bs, int bn) {
  return cat < bcat || (cat == bcat && better(s, n, bs, bn));
}
__device__ __forceinline__ void best_fold(Best &a, double s, int n, int cnt, int cat = 0) {
  if (n < 0) return;
  if (a.node < 0 || cat < a.cat) { a.score = s; a.node = n; a.cnt = cnt; a.cat = cat; return; }
  if (cat > a.cat) return;
  if (better(s, n, a.score, a.node)) { a.score = s; a.node = n; }
  a.cnt += cnt;
}
// warp arg-max with the hardware reductions: order-preserving 64-bit key as two 32-bit maxima, then the lowest
// node among the lanes that hold the maximum (see local_warp_reduce in vc_commit.cuh)
template <bool FUT = false>
__device__ __forceinline__ void best_warp_reduce(Best &b) {
  constexpr unsigned FULLM = 0xffffffffu;
  bool valid = b.node >= 0;
  if (FUT) {  // only the lanes of the lowest category present take part
    const unsigned mc = __reduce_min_sync(FULLM, valid ? (unsigned)b.cat : 3u);
    valid = valid && (unsigned)b.cat == mc;
    if (!valid) b.cnt = 0;
    b.cat = mc == 3u ? 0 : (int)mc;
  }
  const unsigned long long key = valid ? score_key(b.score) : 0ull;
  const unsigned hi = (unsigned)(key >> 32);
  const unsigned mhi = __reduce_max_sync(FULLM, hi);
  const unsigned mlo = __reduce_max_sync(FULLM, hi == mhi ? (unsigned)key : 0u);
  const unsigned long long mkey = ((unsigned long long)mhi << 32) | mlo;
  const unsigned mnode = __reduce_min_sync(FULLM, (valid && key == mkey) ? (unsigned)b.node : 0xffffffffu);
  b.cnt = (int)__reduce_add_sync(FULLM, (unsigned)b.cnt);
  if (mnode == 0xffffffffu) { b.node = -1; b.score = 0.0; }
  else { b.node = (int)mnode; b.score = score_of_key(mkey); }
}
__device__ __forceinline__ uint4 pack_best(const Best &b, unsigned tag) {
  unsigned long long sb = (unsigned long long)__double_as_longlong(b.score);
  return make_uint4((unsigned)sb, (unsigned)(sb >> 32), (unsigned)b.node, (tag << 3) | ((unsigned)b.cat << 2) | (unsigned)min(b.cnt, 2));
}
__device__ __forceinline__ Best unpack_best(const uint4 &v) {
  Best b;
  b.score = __longlong_as_double((long long)((unsigned long long)v.x | ((unsigned long long)v.y << 32)));
  b.node = (int)v.z;
  b.cnt = (int)(v.w & 3u);
  b.cat = (int)((v.w >> 2) & 1u);
  return b;
}

// ring record of a publication: the owner CTA's new best + how many placements the record covers (1..RUN_MAX)
// flag (SOFT): the placement changed the candidate set in a way that may move a normalisation constant
__device__ __forceinline__ uint4 pack_run(const Best &b, unsigned tag, int m, bool flag = false) {
  unsigned long long sb = (unsigned long long)__double_as_longlong(b.score);
  return make_uint4((unsigned)sb, (unsigned)(sb >> 32), (unsigned)b.node,
                    (tag << 10) | (flag ? 0x200u : 0u) | ((unsigned)m << 3) | ((unsigned)b.cat << 2) | (unsigned)min(b.cnt, 2));
}
#define RUN_TAG_MASK 0x3fffffu

// a record into the same slot of every rank's copy (one rank: the plain local store)
__device__ __forceinline__ void store_all(const K2Params &p, uint4 *const *peers, uint4 *local, size_t off, uint4 v) {
  if (p.n_ranks <= 1) { mbox_store(local + off, v); return; }
  for (int r = 0; r < p.n_ranks; ++r) mbox_store(peers[r] + off, v);
}
// a poll that saw nothing for p.wd_cycles (~10 s by default) means a peer never came up or the replicas of the control
// program diverged - abort the kernel (the launch fails with an error) instead of spinning until somebody kills the job
#define WD_EXTRA
#define DBG_STAGE(k, v) do { if (PROF && p.dbg && (threadIdx.x & 31) == 0) ((volatile int *)p.dbg)[(size_t)blockIdx.x * 8 + (k)] = (v); } while (0)
#define PEER_WATCHDOG(spins, t0)                                                                  \
  do {                                                                                            \
    if (((++(spins)) & 0x3ffffu) == 0 && clock64() - (t0) > p.wd_cycles) {                        \
      if ((threadIdx.x & 31) == 0) printf("k_commit_fast watchdog: CTA %d line %d\n", (int)(p.cta_base + blockIdx.x), __LINE__); \
      WD_EXTRA;                                                                                   \
      __trap();                                                                                   \
    }                                                                                             \
  } while (0)

// all-gather of the CTA bests (warp 0 of every CTA); fills the slot table
__device__ __forceinline__ void exchange_all_fast(const K2Params &p, const Best &mine, unsigned ag, FastSmem &fs) {
  const int lane = threadIdx.x & 31;
  const int G = p.n_cta;
  const unsigned tag = (ag + 1u) & 0x1fffffffu;
  const size_t par = (size_t)(ag & 1u) * G * MBOX_STRIDE;
  uint4 *base = p.mbox + par;
  if (lane == 0) store_all(p, p.peer_mbox, p.mbox, par + (size_t)(p.cta_base + blockIdx.x) * MBOX_STRIDE, pack_best(mine, tag));
  unsigned spins = 0;
  const long long t0w = clock64();
  for (int s0 = 0; s0 < G; s0 += 32 * 4) {
    uint4 a[4];
    bool need[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) need[k] = (s0 + k * 32 + lane) < G;
    bool pending;
    do {
      pending = false;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (need[k]) a[k] = mbox_load(base + (size_t)(s0 + k * 32 + lane) * MBOX_STRIDE);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (!need[k]) continue;
        if ((a[k].w >> 3) != tag) { pending = true; continue; }
        const int s = s0 + k * 32 + lane;
        Best b = unpack_best(a[k]);
        fs.sl_score[s] = b.score; fs.sl_node[s] = b.node; fs.sl_cnt[s] = b.cnt; fs.sl_cat[s] = b.cat;
        need[k] = false;
      }
      if (pending) PEER_WATCHDOG(spins, t0w);
    } while (pending);
  }
  __syncwarp();
}

// SAMP: the same all-gather with a second vector per slot: x = feasible nodes of the CTA, y = those at or after the
// rotating start index (meaningful for the CTA that holds it). Fills sl_feas too; returns y of CTA `a_cta`.
__device__ __forceinline__ int exchange_all_samp(const K2Params &p, const Best &mine, int feas, int tail, unsigned ag, FastSmem &fs, int a_cta) {
  const int lane = threadIdx.x & 31;
  const int G = p.n_cta;
  const unsigned tag = (ag + 1u) & 0x1fffffffu;
  const size_t par = (size_t)(ag & 1u) * G * MBOX_STRIDE;
  uint4 *base = p.mbox + par;
  if (lane == 0) mbox_store(base + (size_t)blockIdx.x * MBOX_STRIDE, pack_best(mine, tag));
  if (lane == 1) mbox_store(base + (size_t)blockIdx.x * MBOX_STRIDE + 1, make_uint4((unsigned)feas, (unsigned)tail, 0u, tag << 3));
  unsigned spins = 0;
  const long long t0w = clock64();
  int tail_a = 0;
  for (int s0 = 0; s0 < G; s0 += 32) {
    const int sidx = s0 + lane;
    bool need = sidx < G;
    uint4 a, x;
    bool pending;
    do {
      pending = false;
      if (need) {
        a = mbox_load(base + (size_t)sidx * MBOX_STRIDE);
        x = mbox_load(base + (size_t)sidx * MBOX_STRIDE + 1);
        if ((a.w >> 3) != tag || (x.w >> 3) != tag) pending = true;
        else {
          Best b = unpack_best(a);
          fs.sl_score[sidx] = b.score; fs.sl_node[sidx] = b.node; fs.sl_cnt[sidx] = b.cnt; fs.sl_cat[sidx] = b.cat;
          fs.sl_feas[sidx] = (int)x.x;
          if (sidx == a_cta) tail_a = (int)x.y;
          need = false;
        }
      }
      pending = __any_sync(0xffffffffu, pending);
      if (pending) PEER_WATCHDOG(spins, t0w);
    } while (pending);
  }
  __syncwarp();
  return (int)__reduce_max_sync(0xffffffffu, (unsigned)tail_a);
}

// best of this CTA from its verdict/score cache (a whole warp); cnt = exact number of candidates of the best's category;
// the FUT instance also returns how many nodes sit in each category
template <bool FUT>
__device__ __forceinline__ Best scan_cache(const FastSmem &fs, int nmine, int nbase, int *cnt01 = nullptr) {
  const int lane = threadIdx.x & 31;
  Best b{0.0, -1, 0, 0};
  int n0 = 0, n1 = 0;
  for (int i = lane; i < nmine; i += 32) {
    const int cc = fs.c_cat[i];
    if (cc == 0 || (FUT && cc == 1)) best_fold(b, fs.c_score[i], nbase + i, 1, cc);
    if (FUT) { n0 += cc == 0; n1 += cc == 1; }
  }
  best_warp_reduce<FUT>(b);
  if (FUT && cnt01) {
    cnt01[0] = (int)__reduce_add_sync(0xffffffffu, (unsigned)n0);
    cnt01[1] = (int)__reduce_add_sync(0xffffffffu, (unsigned)n1);
  }
  return b;
}
// arg-max over the slot table (warp 0)
template <bool FUT>
__device__ __forceinline__ Best fold_slots(const FastSmem &fs, int G, int *owner_out) {
  const int lane = threadIdx.x & 31;
  Best g{0.0, -1, 0, 0};
  int owner = -1;
  for (int s = lane; s < G; s += 32) {
    const int before = g.node;
    best_fold(g, fs.sl_score[s], fs.sl_node[s], fs.sl_cnt[s], FUT ? fs.sl_cat[s] : 0);
    if (g.node != before) owner = s;
  }
  const int my_node = g.node;
  best_warp_reduce<FUT>(g);
  // the winning node sits in exactly one slot: the lane whose local best it is knows the owner
  *owner_out = (int)__reduce_max_sync(0xffffffffu, (unsigned)((g.node >= 0 && my_node == g.node) ? owner + 1 : 0)) - 1;
  return g;
}

// lanes of warp 0 copy a record of `words` 32-bit words from global to shared memory in one access
__device__ __forceinline__ void load_record(void *dst_smem, const void *src_global, int words, bool read_only) {
  const int lane = threadIdx.x & 31;
  for (int w = lane; w < words; w += 32) {
    const int *src = reinterpret_cast<const int *>(src_global) + w;
    reinterpret_cast<int *>(dst_smem)[w] = read_only ? __ldg(src) : *src;
  }
}

struct SampWin { int A, B, r, b_lo, total; bool wrap; };  // SAMP: one task's candidate window over the ring of CTAs
#define FAST_MAXQ 64  // queues mirrored in shared memory for the queue scan
struct CtlFast {  // shared-memory state of the fast kernel next to Ctl
  JobStatic js;
  JobDyn jd;
  JobStatic js2;  // head of the queue's static job list (the candidate the heap top is compared with)
  JobDyn jd2;
  double q_share[FAST_MAXQ];
  int q_active[FAST_MAXQ];
  QueueStatic qs;
  QueueDyn qd;
  RoleStatic rs[VC_MAX_JOB_ROLES];
  RoleDyn rd[VC_MAX_JOB_ROLES];
  double cta_best_score, g_best_score;
  int cta_best_node, cta_cnt, g_best_node, g_cnt;
  int cta_best_cat, cta_cnt1;  // FUT: category of the CTA's best; cta_cnt / cta_cnt1 = nodes of category 0 / 1
  // run-ahead results of warp 2, double-buffered by the parity of the CMD_EVAL count
  double spec_sc[2];
  int spec_i[2], spec_group[2], spec_cat[2], spec_kind[2];
  // CMD_EVAL mailbox between warp 0 (control) and warp 1 (evaluator)
  double ev_score;
  int ev_i, ev_ring, ev_node, ev_cnt, ev_cat, cur_group;
  int ev_kind;  // FUT: the placement just applied to row ev_i was an allocation (0) or a pipeline (1)
  uint4 rec[6];  // SAMP: the step's ring records as polled (previous publication, P_B, P_A; two vectors each)
  int ev_feas;  // SAMP: feasible nodes of this CTA after the re-evaluation
  int ev_flag;  // SOFT: the evaluator saw a change of the candidate set that may move g_soft (-> full sweep next)
  int g_soft[2];  // SOFT: largest intolerable-soft-taint count over the candidates of category 0 / 1
  unsigned ev_tag;
  // CMD_RUN: placements the control program allows on node ev_i in a row (run_L), attempt index of the first one,
  // result (run_m placements made), runner-up computed by warp 2
  int run_L, run_att0, run_m;
  // full sweep / re-entry command: group whose cached verdicts are saved to the table first (-1: none), re-entry (1) or
  // full sweep (0), verdicts taken from the table (else the CTA's cache already holds the group), stamp of the saved
  // verdicts, rows found changed; rollback command: stamp of the rows it changes
  int vt_wb, vt_reenter, vt_load, vt_stamp, vt_nd;
  int vt_clock, vt_held, vt_held_stamp;  // control state of the verdict table (see the control program)
  int vt_n[2];  // VC_PROF: group switches served by a full sweep / from saved verdicts
  double ru_score, rl_score;
  int ru_node, rl_node, rl_cnt;
  int ru_cat, rl_cat, rl_cnt0, rl_cnt1;
  double run_sc[RUN_MAX];  // state k of the row (after k further placements): total score, fit category
  int run_cat[RUN_MAX];
};
// node view of row i after `k` further placements of the staged group (k as a double): what eval_pair_fast sees for
// the states a run walks through. Every quantity is integer-valued (checked at upload), so row -/+ k * request is
// exactly what k sequential placements leave (node_info.go:467-471, predicates.go:254-255).
struct RunNodeView {
  const FastSmem &s;
  const TaskRec &t;
  int i;
  double k, kk;  // kk = k when the predicates plugin maintains the upstream NodeInfo, else 0
  __device__ __forceinline__ double alloc(int d) const { return s.alloc[d * s.cap + i]; }
  __device__ __forceinline__ double idle(int d) const { return s.idle[d * s.cap + i] - k * t.req[d]; }
  __device__ __forceinline__ double used(int d) const { return s.used[d * s.cap + i] + k * t.req[d]; }
  __device__ __forceinline__ double rel(int) const { return 0.0; }  // no Releasing / Pipelined resources in this kernel
  __device__ __forceinline__ double pip(int) const { return 0.0; }
  __device__ __forceinline__ double kalloc(int kd) const { return s.kalloc[kd * s.cap + i]; }
  __device__ __forceinline__ double kreq(int kd) const { return s.kreq[kd * s.cap + i] + kk * t.kreq[kd]; }
  __device__ __forceinline__ double knz(int kd) const { return s.knz[kd * s.cap + i] + kk * t.knz[kd]; }
};

// PROF = true keeps the phase / owner-path cycle counters (tools/prof_commit.py, VC_PROF=1); the production
// instance carries no clock reads on the control warp's critical path.
#define FPROF_MARK(k) do { if (PROF) { PROF_MARK(k); } } while (0)
template <bool PROF, bool FUT = false, bool SOFT = false, bool SAMP = false>
__global__ void __launch_bounds__(256, 1) k_commit_fast(K2Params p, FastParams fp) {
  static_assert(!(SAMP && SOFT), "the sampled candidate set changes per task: its normalisation constants are not cacheable");
  const DevConf &c = p.c;
  const int R = p.d.R, K = p.d.K, N = p.d.N, J = p.d.J, Q = p.d.Q, NR = p.d.NR, T = p.d.T;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int lcta = blockIdx.x;            // this rank's buffers are indexed locally
  const int cta = p.cta_base + lcta;      // identity in the exchange: unique over all ranks
  const int nbase = p.d.node_begin + cta * p.npc;
  const int nmine = max(0, min(p.npc, p.d.node_end - nbase));
  const int cap = p.npc;
  const int G = p.n_cta;

  // ---- carve shared memory ----
  unsigned char *sp = k2_smem;
  Ctl &S = *reinterpret_cast<Ctl *>(sp);
  sp += (sizeof(Ctl) + 15) & ~(size_t)15;
  CtlFast &F = *reinterpret_cast<CtlFast *>(sp);
  sp += (sizeof(CtlFast) + 15) & ~(size_t)15;
  FastSmem fs;
  fs.cap = cap;
  auto take = [&](int rows) { double *q = reinterpret_cast<double *>(sp); sp += (size_t)rows * cap * sizeof(double); return q; };
  fs.alloc = take(R); fs.idle = take(R); fs.used = take(R);
  fs.rel = fs.pip = nullptr;
  if (FUT) { fs.rel = take(R); fs.pip = take(R); }
  fs.kalloc = take(K); fs.kreq = take(K); fs.knz = take(2);
  fs.c_score = take(1);
  fs.nerr = reinterpret_cast<unsigned long long *>(sp); sp += (size_t)cap * 8;
  fs.sl_score = reinterpret_cast<double *>(sp); sp += (size_t)G * 8;
  fs.max_tasks = reinterpret_cast<int32_t *>(sp); sp += (size_t)cap * 4;
  fs.pod_count = reinterpret_cast<int32_t *>(sp); sp += (size_t)cap * 4;
  fs.nerr_stamp = reinterpret_cast<int32_t *>(sp); sp += (size_t)cap * 4;
  fs.c_cat = reinterpret_cast<int32_t *>(sp); sp += (size_t)cap * 4;
  fs.c_cs = reinterpret_cast<uint32_t *>(sp); sp += (size_t)cap * 4;
  fs.mstamp = reinterpret_cast<int32_t *>(sp); sp += (size_t)cap * 4;
  fs.dlist = reinterpret_cast<int32_t *>(sp); sp += (size_t)cap * 4;
  fs.sl_node = reinterpret_cast<int32_t *>(sp); sp += (size_t)G * 4;
  fs.sl_cnt = reinterpret_cast<int32_t *>(sp); sp += (size_t)G * 4;
  fs.sl_cat = reinterpret_cast<int32_t *>(sp); sp += (size_t)G * 4;
  fs.sl_feas = reinterpret_cast<int32_t *>(sp); sp += (size_t)G * 4;
  sp = reinterpret_cast<unsigned char *>(((uintptr_t)sp + 15) & ~(uintptr_t)15);
  HeapKey *heap = fp.heap_in_smem ? reinterpret_cast<HeapKey *>(sp)
                                  : reinterpret_cast<HeapKey *>(p.rep_heap) + (size_t)lcta * p.rep_heap_stride;

  for (int i = tid; i < nmine; i += blockDim.x) {
    const int n = nbase + i;
    for (int d = 0; d < R; ++d) {
      fs.alloc[d * cap + i] = p.alloc[(size_t)d * N + n];
      fs.idle[d * cap + i] = p.idle[(size_t)d * N + n];
      fs.used[d * cap + i] = p.used[(size_t)d * N + n];
      if (FUT) { fs.rel[d * cap + i] = p.rel[(size_t)d * N + n]; fs.pip[d * cap + i] = p.pip[(size_t)d * N + n]; }
    }
    for (int k = 0; k < K; ++k) {
      fs.kalloc[k * cap + i] = p.kalloc[(size_t)k * N + n];
      fs.kreq[k * cap + i] = p.kreq[(size_t)k * N + n];
    }
    for (int k = 0; k < 2; ++k) fs.knz[k * cap + i] = p.knz[(size_t)k * N + n];
    fs.max_tasks[i] = p.max_tasks[n];
    fs.pod_count[i] = p.pod_count[n];
    fs.nerr[i] = 0ull;
    fs.nerr_stamp[i] = -1;
    fs.c_cat[i] = 2;
    fs.c_score[i] = 0.0;
    fs.c_cs[i] = 0u;
    fs.mstamp[i] = 0;
  }
  for (int s = tid; s < G; s += blockDim.x) { fs.sl_score[s] = 0.0; fs.sl_node[s] = -1; fs.sl_cnt[s] = 0; fs.sl_cat[s] = 0; fs.sl_feas[s] = 0; }
  // Per-group verdict table (not the SOFT instance: its cached scores carry normalisation constants that move). The table
  // itself is not cleared between cycles: a group's entries count only once its stamp was set in this launch.
  // (entry of row i of group g: g * gridDim.x * npc + blockIdx.x * npc + i; recomputed where used, like VT, to keep
  //  them out of the registers of the control warp)
#define VT (!SOFT && fp.vt_cat != nullptr)
#define VT_AT(g, i) ((size_t)(g) * gridDim.x * p.npc + (size_t)blockIdx.x * p.npc + (i))
#define VT_GSTAMP(g) fp.vt_gstamp[(size_t)blockIdx.x * p.n_groups + (g)]
  if (VT)
    for (int g = tid; g < p.n_groups; g += blockDim.x) VT_GSTAMP(g) = -1;

  // ---- per-CTA replica of the mutable control state, packed records ----
  unsigned char *rb = reinterpret_cast<unsigned char *>(p.rep_f64 + (size_t)lcta * p.rep_f64_stride);
  JobDyn *jdyn = reinterpret_cast<JobDyn *>(rb); rb += (size_t)J * sizeof(JobDyn);
  QueueDyn *qdyn = reinterpret_cast<QueueDyn *>(rb); rb += (size_t)Q * sizeof(QueueDyn);
  RoleDyn *rdyn = reinterpret_cast<RoleDyn *>(rb); rb += (size_t)NR * sizeof(RoleDyn);
  double *ops_score = reinterpret_cast<double *>(rb);
  int32_t *ops = p.rep_i32 + (size_t)lcta * p.rep_i32_stride;  // task, node, kind

  for (int j = tid; j < J; j += blockDim.x) {
    JobDyn jd;
    jd.ready = p.j_ready0[j]; jd.waiting = p.j_waiting0[j]; jd.cursor = 0; jd.pad = 0;
    jd.share = p.j_share0[j];
    for (int d = 0; d < FAST_R; ++d) jd.alloc[d] = d < R ? p.j_alloc0[(size_t)d * J + j] : 0.0;
    jd.pad2 = 0.0;
    jdyn[j] = jd;
  }
  for (int r = tid; r < NR; r += blockDim.x) {
    RoleDyn rd;
    rd.occ = p.r_occ0[r]; rd.pip = p.r_pip0[r]; rd.pending = p.r_pending0[r]; rd.failed = 0;
    rdyn[r] = rd;
  }
  for (int q = tid; q < Q; q += blockDim.x) {
    QueueDyn qd;
    qd.alloc_has = p.q_alloc_has0[q]; qd.flags2 = p.q_flags2[q];
    qd.active = (p.qjobs_off[q + 1] > p.qjobs_off[q]) ? 1 : 0;  // buildAllocateContext: queues with a job
    qd.scursor = 0; qd.hsize = 0; qd.pad = 0;
    qd.share = fp.q_share0[q];
    for (int d = 0; d < FAST_R; ++d) qd.alloc[d] = d < R ? p.q_alloc0[(size_t)d * Q + q] : 0.0;
    qdyn[q] = qd;
    if (q < FAST_MAXQ) { F.q_active[q] = qd.active; F.q_share[q] = qd.share; }
  }
  if (tid == 0) {
    S.seq = 0;
    S.n_dec = S.n_vis = S.n_fit = S.n_steps = 0;
    for (int k = 0; k < 8; ++k) S.prof[k] = 0;
    S.prof_last = clock64();
    S.cmd = 0; S.visit_id = 0; S.cur_group = -1; S.cache_group = -1; S.dirty_node = -1;
    S.ag = 0; S.pc = 0; S.since_sync = 0; S.n_full = 0; S.n_incr = 0;
    F.cta_best_node = -1; F.cta_cnt = 0; F.g_best_node = -1; F.g_cnt = 0; F.cta_best_score = F.g_best_score = 0.0;
    F.cta_best_cat = 0; F.cta_cnt1 = 0; F.ev_kind = 0; F.ev_cat = 0; F.ev_flag = 0; F.g_soft[0] = F.g_soft[1] = 0;
    F.spec_i[0] = F.spec_i[1] = -1;
    F.vt_wb = -1; F.vt_reenter = 0; F.vt_load = 0; F.vt_stamp = -1; F.vt_nd = 0;
    F.vt_clock = 0; F.vt_held = -1; F.vt_held_stamp = -1; F.vt_n[0] = F.vt_n[1] = 0;
  }
  __syncthreads();

  // per-warp result of a sweep: best (score, node, category) and, FUT, how many of the warp's nodes sit in category 0 / 1
  auto post_warp = [&](Best &b, int n0, int n1) {
    best_warp_reduce<FUT>(b);
    if (FUT) {
      n0 = (int)__reduce_add_sync(0xffffffffu, (unsigned)n0);
      n1 = (int)__reduce_add_sync(0xffffffffu, (unsigned)n1);
    }
    if (lane == 0) {
      S.w_score[0][warp] = b.score; S.w_node[0][warp] = b.node; S.w_cnt[0][warp] = FUT ? n0 : b.cnt;
      if (FUT) { S.w_cnt[1][warp] = n1; S.w_node[1][warp] = b.cat; }
    }
  };
  // verdict of row i for the staged group record, one thread (the same operations as eval_dirty, one after the other)
  auto eval_full = [&](int i, uint32_t cs, double *sc) -> int {
    const TaskRec &trec = S.trec;
    FastNodeView nv{fs, i};
    const bool pod_cap = c.pred_predicates && fs.max_tasks[i] <= fs.pod_count[i];
    int cat = eval_pair_fast<SOFT>(c, R, K, trec, nv, cs, pod_cap, sc);
    if (FUT) {
      // alloc.predicate: InitResreq <= FutureIdle (allocate.go:816-824); the idle gradient is the subset that fits
      // Idle as well (:722-733). eval_pair_fast answered 0 exactly when the static part, the pod count AND Idle pass.
      bool fit_future = (cs & CS_STATIC_OK) != 0 && !pod_cap;
      for (int d = 0; d < R; ++d) {
        if (d >= 2 && !(trec.has & (1u << d))) continue;
        const double fut = (fs.idle[d * cap + i] + fs.rel[d * cap + i]) - fs.pip[d * cap + i];
        if (!le_eps(trec.req[d], fut)) fit_future = false;
      }
      cat = !fit_future ? 2 : (cat == 0 ? 0 : 1);
    }
    return cat;
  };
  // before a sweep or a re-entry overwrites the verdict cache: save the verdicts of the group it holds (F.vt_wb) to the
  // table (each thread its own rows, which it overwrites after this)
  auto vt_save = [&]() {
    const int wb = F.vt_wb;
    if (wb < 0) return;
    for (int i = tid; i < nmine; i += blockDim.x) {
      fp.vt_cat[VT_AT(wb, i)] = (uint8_t)fs.c_cat[i];
      fp.vt_score[VT_AT(wb, i)] = fs.c_score[i];
    }
  };

  // full evaluation of this thread's nodes for the staged group record (command CMD_SWEEP)
  auto sweep_part = [&]() {
    const TaskRec &trec = S.trec;
    const uint32_t *cs_row = p.cstat + (size_t)trec.klass * N + nbase;
    const int rl = S.sweep_rl;
    const bool use_cache = S.sweep_use_cache != 0;
    const int vid = S.visit_id;
    Best b{0.0, -1, 0, 0};
    int n0 = 0, n1 = 0;
    if (!SOFT) vt_save();  // (F.vt_wb stays -1 without a table)
    if (SOFT && S.cmd == CMD_SWEEP2) {
      // second phase: TaintToleration's normalised score joins the cached NodeOrderFn sums (scheduler_helper.go:117-129)
      const int gs0 = F.g_soft[0], gs1 = F.g_soft[1];
      for (int i = tid; i < nmine; i += blockDim.x) {
        const int cat = fs.c_cat[i];
        if (cat == 2) continue;
        const int soft = (int)((fs.c_cs[i] >> CS_SOFT_SHIFT) & 0xffu);
        const double sc = total_score(c, true, fs.c_score[i], soft, cat == 0 ? gs0 : gs1);
        fs.c_score[i] = sc;
        best_fold(b, sc, nbase + i, 1, cat);
        if (FUT) { n0 += cat == 0; n1 += cat == 1; }
      }
      post_warp(b, n0, n1);
      return;
    }
    int ms0 = 0, ms1 = 0;  // SOFT, first phase: largest soft-taint count among this thread's candidates per category
    for (int i = tid; i < nmine; i += blockDim.x) {
      const uint32_t cs = __ldg(cs_row + i);
      if (use_cache && fs.nerr_stamp[i] != vid) { fs.nerr[i] = 0ull; fs.nerr_stamp[i] = vid; }
      int cat = 2;
      double sc = 0.0;
      if (!(use_cache && ((fs.nerr[i] >> rl) & 1ull))) {
        cat = eval_full(i, cs, &sc);
        if (cat == 2 && use_cache) fs.nerr[i] |= (1ull << rl);
      }
      fs.c_cat[i] = cat;
      fs.c_score[i] = sc;
      fs.c_cs[i] = cs;
      if (SOFT) {
        const int soft = (int)((cs >> CS_SOFT_SHIFT) & 0xffu);
        if (cat == 0) ms0 = max(ms0, soft);
        if (FUT && cat == 1) ms1 = max(ms1, soft);
        continue;
      }
      if (cat == 0 || (FUT && cat == 1)) best_fold(b, sc, nbase + i, 1, cat);
      if (FUT) { n0 += cat == 0; n1 += cat == 1; }
    }
    if (SOFT) {
      ms0 = (int)__reduce_max_sync(0xffffffffu, (unsigned)ms0);
      ms1 = (int)__reduce_max_sync(0xffffffffu, (unsigned)ms1);
      if (lane == 0) { S.w_soft[0][warp] = ms0; S.w_soft[1][warp] = ms1; }
      return;
    }
    post_warp(b, n0, n1);
  };
  // stmt.Discard() for this thread's nodes (command CMD_DISCARD), statement.go:357-381
  auto discard_part = [&]() {
    const int n_ops = S.n_ops;
    const int vclk = F.vt_clock;
    for (int k = n_ops - 1; k >= 0; --k) {
      const int ot = ops[k * 3 + 0], on = ops[k * 3 + 1];
      const bool was_pipe = FUT && ops[k * 3 + 2] == VC_OP_PIPELINE;
      if (on >= nbase && on < nbase + nmine && ((on - nbase) % blockDim.x) == tid) {
        const int i = on - nbase;
        fs.mstamp[i] = vclk;
        for (int d = 0; d < R; ++d) {
          double rq = p.req[(size_t)d * T + ot];
          if (was_pipe) { fs.pip[d * cap + i] -= rq; continue; }
          fs.idle[d * cap + i] += rq;
          fs.used[d * cap + i] -= rq;
        }
        if (c.has_predicates) {
          fs.pod_count[i] -= 1;
          for (int kk = 0; kk < K; ++kk) fs.kreq[kk * cap + i] -= p.tkreq[(size_t)kk * T + ot];
          for (int kk = 0; kk < 2; ++kk) fs.knz[kk * cap + i] -= p.tknz[(size_t)kk * T + ot];
        }
      }
    }
  };

  // ---- configuration hoisted out of the loops ----
  bool f_qorder_prop = false, f_over_prop = false, f_alloc_prop = false, f_gang_ready = false;
  int ord_n = 0, ord_kind[3] = {0, 0, 0};
  for (int i = 0; i < c.n_plugins; ++i) {
    const int pl = c.plugin[i];
    const uint32_t en = c.enabled[i];
    if ((en & VC_EN_QUEUE_ORDER) && pl == VC_PLUGIN_PROPORTION) f_qorder_prop = true;
    if ((en & VC_EN_OVERUSED) && pl == VC_PLUGIN_PROPORTION) f_over_prop = true;
    if ((en & VC_EN_ALLOCATABLE) && pl == VC_PLUGIN_PROPORTION) f_alloc_prop = true;
    if ((en & VC_EN_JOB_READY) && pl == VC_PLUGIN_GANG) f_gang_ready = true;
    if ((en & VC_EN_NODE_ORDER) && ord_n < 3 &&
        ((pl == VC_PLUGIN_BINPACK && c.binpack_weight != 0) || pl == VC_PLUGIN_NODEORDER || pl == VC_PLUGIN_TDM))
      ord_kind[ord_n++] = pl;
  }
  // ---- lane roles of the warp-cooperative single-node evaluation (see eval_dirty below) ----
  enum { ROLE_NONE = 0, ROLE_BP = 1, ROLE_LEAST = 2, ROLE_MOST = 3, ROLE_BAL = 4 };
  // both half-warps carry the 16 roles: one call evaluates the node in two states (lanes 0-15 / 16-31)
  const int hl = lane & 15, half = lane >> 4;
  const int role = hl < 8 ? ROLE_BP : hl < 10 ? ROLE_LEAST : hl < 12 ? ROLE_MOST : ROLE_BAL;
  const int dk = role == ROLE_BP ? hl : role == ROLE_LEAST ? hl - 8 : role == ROLE_MOST ? hl - 10 : hl - 12;
  const bool lane_valid = (role == ROLE_BP && dk < R) || role == ROLE_LEAST || role == ROLE_MOST || (role == ROLE_BAL && dk < K);
  const int dk_c = lane_valid ? dk : 0;
  const double *a_base = role == ROLE_BP ? fs.used + dk_c * cap : role == ROLE_BAL ? fs.kreq + dk_c * cap : fs.knz + dk_c * cap;
  const double *al_base = role == ROLE_BP ? fs.alloc + dk_c * cap : fs.kalloc + dk_c * cap;
  const double *idle_base = fs.idle + ((hl < 8 && hl < R) ? hl : 0) * cap;
  const double *rel_base = FUT ? fs.rel + ((hl < 8 && hl < R) ? hl : 0) * cap : nullptr;
  const double *pip_base = FUT ? fs.pip + ((hl < 8 && hl < R) ? hl : 0) * cap : nullptr;
  const int w_d = (role == ROLE_BP && lane_valid) ? c.binpack_dim_weight[dk_c] : 0;
  const double mul_const = role == ROLE_BP ? (double)w_d : (role == ROLE_LEAST || role == ROLE_MOST) ? 100.0 : 1.0;
  // per-group lane operands (refreshed when the staged group record changes)
  double b_val = 0.0, req_fit = 0.0;
  bool fit_on = false, on_task = false;
  uint32_t t_has = 0;
  int wsum_g = 0;  // binpack weightSum: depends on the request record only (binpack.go:213-237)
  const double bp_scale = (double)(VC_MAX_NODE_SCORE * c.binpack_weight);
  bool ord_has_tdm = false;
  for (int k = 0; k < ord_n; ++k) ord_has_tdm |= ord_kind[k] == VC_PLUGIN_TDM;

  // Warp-cooperative evaluation of ONE node i of this CTA for the staged group: the same IEEE operations
  // as eval_pair_fast / the generic functions, one division per lane instead of ~17 in a row:
  //   lanes 0-7   fit of dim d against Idle + binpack term of dim d          (binpack.go:213-237)
  //   lanes 8-9   leastRequestedScore of cpu / memory, lanes 10-11 mostRequestedScore
  //   lanes 12-15 BalancedAllocation fraction of upstream dim k
  // then one second-level division (binpack /weightSum, least, most, mean) and the std / sqrt.
  // `extra` = 1 evaluates the node as it will be after ONE more placement of this same group (speculation: under
  // best-fit scoring the node that just won usually wins again); the adds are the same IEEE operations the real
  // placement performs (node_info.go:467-471, predicates.go:254-255), so the speculative score is bit-identical.
  auto eval_dirty = [&](int i0, int i1, int k0, int k1, uint32_t cs, double *score_out, int kind = 0) -> int {
    // lanes 0-15 evaluate row i0 after k0 further placements of this group, lanes 16-31 row i1 after k1 (0 = as it
    // is); cs = the static word of the lane's row; kind (FUT) = those further placements are allocations (0: Idle,
    // Used move) or pipelines (1: only Pipelined moves, node_info.go:457-458) - the upstream NodeInfo follows both
    const int i = half ? i1 : i0;
    const int k = half ? k1 : k0;
    const double kf = (double)k;
    const int hs = half << 4;
    const int kx = c.has_predicates ? k : 0;
    const bool pipe = FUT && kind == 1;
    const bool pod_cap = c.pred_predicates && fs.max_tasks[i] <= fs.pod_count[i] + kx;
    const bool bump = k > 0 && (role == ROLE_BP ? !pipe : c.has_predicates);
    const double a0 = a_base[i], alloc = al_base[i], idle0 = idle_base[i];
    const double a = bump ? a0 + kf * b_val : a0;
    const double idle = (k > 0 && !pipe) ? idle0 - kf * req_fit : idle0;
    const bool bad_fit = fit_on && !le_eps(req_fit, idle);
    bool bad_fut = false;
    if (FUT) {  // FutureIdle = Idle + Releasing - Pipelined, node_info.go:114-116
      const double pip0 = pip_base[i];
      const double pipv = (k > 0 && pipe) ? pip0 + kf * req_fit : pip0;
      const double fut = (idle + rel_base[i]) - pipv;
      bad_fut = fit_on && !le_eps(req_fit, fut);
    }
    const double s = a + b_val;
    const bool nz = alloc != 0.0;
    const bool scored = role == ROLE_BP ? (on_task && nz && w_d != 0) : (on_task && nz);
    const bool over = role == ROLE_BP && scored && s > alloc;
    const bool zero_least = role == ROLE_LEAST && s > alloc;
    const double x = role == ROLE_LEAST ? alloc - s : role == ROLE_MOST ? fmin(s, alloc) : s;
    const double num = x * mul_const;
    const double den = scored ? alloc : 1.0;
    double q = num / den;
    {  // lanes 8-11: floor of the quotient (int64 division of the upstream scorers), exact fma fix-up
      double qq = trunc(q);
      const double r = fma(-qq, den, num);
      qq = r < 0.0 ? qq - 1.0 : (r >= den ? qq + 1.0 : qq);
      if (role == ROLE_LEAST || role == ROLE_MOST) q = zero_least ? 0.0 : qq;
    }
    if (role == ROLE_BAL) q = fmin(q, 1.0);
    const double val = scored ? q : 0.0;
    const unsigned m_bad = (__ballot_sync(0xffffffffu, bad_fit) >> hs) & 0xffffu;
    const unsigned m_over = (__ballot_sync(0xffffffffu, over) >> hs) & 0xffffu;
    const unsigned m_on = (__ballot_sync(0xffffffffu, scored) >> hs) & 0xffffu;
    const bool fit = (cs & CS_STATIC_OK) != 0 && !pod_cap && m_bad == 0;
    bool fit_future = fit;
    if (FUT) {  // (the ballot is evaluated by every lane: the two halves may differ in pod_cap)
      const unsigned m_badf = (__ballot_sync(0xffffffffu, bad_fut) >> hs) & 0xffffu;
      fit_future = (cs & CS_STATIC_OK) != 0 && !pod_cap && m_badf == 0;
    }
    // gather the 16 lane results of this half (adding the 0.0 of an inactive lane is exact)
    double v[16];
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) v[kk] = __shfl_sync(0xffffffffu, val, kk, 16);
    double bp_sum = 0.0;
#pragma unroll
    for (int d = 0; d < 8; ++d) bp_sum += v[d];
    const double on8 = (m_on >> 8) & 1u ? 1.0 : 0.0, on9 = (m_on >> 9) & 1u ? 1.0 : 0.0;
    const double ls = (0.0 + v[8] * 50.0) + v[9] * 50.0;   // inactive lanes carry 0.0
    const double ms = (0.0 + v[10] * 1.0) + v[11] * 1.0;
    const double wl = (on8 + on9) * 50.0, wm = on8 + on9;   // lanes 10,11 are active exactly when 8,9 are
    const unsigned fonm = (m_on >> 12) & 0xfu;
    const double total = ((0.0 + v[12]) + v[13]) + (v[14] + 0.0) * 1.0 + v[15];
    const int nf = __popc(fonm);
    // second-level divisions, one per lane
    const double num2 = hl == 0 ? bp_sum : hl == 1 ? ls : hl == 2 ? ms : total;
    const double den2 = hl == 0 ? (wsum_g > 0 ? (double)wsum_g : 1.0) : hl == 1 ? (wl > 0.0 ? wl : 1.0)
                      : hl == 2 ? (wm > 0.0 ? wm : 1.0) : (nf > 0 ? (double)nf : 1.0);
    double q2 = num2 / den2;
    {
      double qq = trunc(q2);
      const double r = fma(-qq, den2, num2);
      qq = r < 0.0 ? qq - 1.0 : (r >= den2 ? qq + 1.0 : qq);
      if (hl == 1 || hl == 2) q2 = qq;
    }
    double bp = __shfl_sync(0xffffffffu, q2, 0, 16);
    bp = wsum_g > 0 ? bp : bp_sum;
    bp *= bp_scale;
    bp = (m_over & 0xffu) ? 0.0 : bp;
    const double least = wl > 0.0 ? __shfl_sync(0xffffffffu, q2, 1, 16) : 0.0;
    const double most = wm > 0.0 ? __shfl_sync(0xffffffffu, q2, 2, 16) : 0.0;
    const double mean = __shfl_sync(0xffffffffu, q2, 3, 16);
    double stdv = 0.0;
    if (nf == 2) {
      // the two active fractions in dimension order
      const unsigned lo = __ffs(fonm) - 1, hi = 31 - __clz(fonm);
      const double f0 = lo == 0 ? v[12] : lo == 1 ? v[13] : v[14];
      const double f1 = hi == 1 ? v[13] : hi == 2 ? v[14] : v[15];
      stdv = fabs((f0 - f1) / 2.0);
    } else if (nf > 2) {
      double sum = 0.0;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const double dlt = v[12 + kk] - mean;
        sum = ((fonm >> kk) & 1u) ? sum + dlt * dlt : sum;
      }
      stdv = sqrt(sum / (double)nf);
    }
    const double bal = (double)__double2ll_rz((1.0 - stdv) * (double)VC_MAX_NODE_SCORE);
    double no = 0.0;
    if (c.w_least != 0) no += least * (double)c.w_least;
    if (c.w_most != 0) no += most * (double)c.w_most;
    if (c.w_balanced != 0) no += bal * (double)c.w_balanced;
    if (c.w_node_affinity != 0) no += (double)(cs >> CS_NAFF_SHIFT) * (double)c.w_node_affinity;
    const double tdm_sc = (cs & CS_TDM_ORDER_MAX) ? (double)VC_MAX_NODE_SCORE : 0.0;
    double order = 0.0;
#pragma unroll
    for (int kk = 0; kk < 3; ++kk) {
      const int kind = ord_kind[kk];
      const double term = kind == VC_PLUGIN_BINPACK ? bp : kind == VC_PLUGIN_NODEORDER ? no : tdm_sc;
      order = kk < ord_n ? order + term : order;
    }
    const bool has_order = !(ord_has_tdm && (cs & CS_TDM_ORDER_ERR));
    const int cat_r = FUT ? (!fit_future ? 2 : (fit ? 0 : 1)) : (fit ? 0 : 2);
    if (SOFT) *score_out = total_score(c, has_order, has_order ? order : 0.0, (int)((cs >> CS_SOFT_SHIFT) & 0xffu), F.g_soft[cat_r == 1 ? 1 : 0]);
    else *score_out = total_score(c, has_order, has_order ? order : 0.0, 0, 0);
    return cat_r;
  };
  // SOFT: does the row's move from category `oc` to `nc` possibly change a normalisation constant? (conservative)
  auto soft_event = [&](int oc, int nc, uint32_t cs) -> bool {
    if (!SOFT || oc == nc) return false;
    const int soft = (int)((cs >> CS_SOFT_SHIFT) & 0xffu);
    if (oc == 0 && soft > 0 && soft == F.g_soft[0]) return true;            // a holder of the maximum leaves category 0
    if (FUT && oc == 1 && soft > 0 && soft == F.g_soft[1]) return true;     // ... leaves category 1
    if (FUT && nc == 1 && soft > F.g_soft[1]) return true;                  // a larger count enters category 1
    return false;
  };
  // per-lane operands of eval_dirty for the group record staged in S.trec
  auto stage_ops = [&]() {
    t_has = S.trec.has;
    req_fit = hl < 8 && hl < R ? S.trec.req[hl] : 0.0;
    fit_on = hl < R && hl < 8 && (hl < 2 || (t_has & (1u << hl)));
    b_val = !lane_valid ? 0.0 : role == ROLE_BP ? S.trec.req[dk_c] : role == ROLE_BAL ? S.trec.kreq[dk_c] : S.trec.knz[dk_c];
    on_task = role == ROLE_BP ? (lane_valid && (dk_c < 2 || (t_has & (1u << dk_c))) && b_val >= VC_MIN_RESOURCE && w_d >= 0)
            : role == ROLE_BAL ? (lane_valid && !(dk_c >= 2 && b_val == 0.0))
            : (role != ROLE_NONE);
    int wv = (role == ROLE_BP && on_task) ? w_d : 0;
    for (int o = 4; o; o >>= 1) wv += __shfl_xor_sync(0xffffffffu, wv, o);  // lane 0: sum over lanes 0-7 (every 8-lane group sums its own)
    wsum_g = __shfl_sync(0xffffffffu, wv, 0);
  };
  // Re-entry of the staged group (command CMD_SWEEP with F.vt_reenter, every warp, operands staged): rows unchanged since
  // the group's verdicts were saved (stamp <= F.vt_stamp) take them from the table (or keep them, when this CTA's cache
  // still holds the group); the changed ones are re-evaluated - two per worker warp and round, or one per thread past
  // VT_DIRTY_MAX - and the CTA's rows are folded as a sweep folds them. (The control warp takes no round: the
  // warp-cooperative evaluator in its code would cost it registers it does not have to spare.)
  int vt_rows = 0, vt_fallback = 0;  // VC_PROF: rows re-evaluated on re-entry, re-entries past VT_DIRTY_MAX (thread 0)
  auto reenter_part = [&](bool rounds) {
    const int g = F.cur_group, st = F.vt_stamp;
    const bool load = F.vt_load != 0;
    const uint32_t *cs_row = p.cstat + (size_t)S.trec.klass * N + nbase;
    vt_save();
    for (int i = tid; i < nmine; i += blockDim.x) {
      fs.c_cs[i] = __ldg(cs_row + i);
      if (fs.mstamp[i] > st) {
        fs.dlist[atomicAdd(&F.vt_nd, 1)] = i;
      } else if (load) {
        fs.c_cat[i] = fp.vt_cat[VT_AT(g, i)];
        fs.c_score[i] = fp.vt_score[VT_AT(g, i)];
      }
    }
    __syncthreads();
    const int nd = F.vt_nd;
    if (nd > VT_DIRTY_MAX) {
      for (int k = tid; k < nd; k += blockDim.x) {
        const int i = fs.dlist[k];
        double sc = 0.0;
        const int cat = eval_full(i, fs.c_cs[i], &sc);
        fs.c_cat[i] = cat; fs.c_score[i] = sc;
      }
    } else if (rounds) {
      for (int pr = warp - 1; 2 * pr < nd; pr += nwarps - 1) {
        const bool two = 2 * pr + 1 < nd;
        const int i0 = fs.dlist[2 * pr], i1 = two ? fs.dlist[2 * pr + 1] : i0;
        double sc = 0.0;
        const int cat = eval_dirty(i0, i1, 0, 0, fs.c_cs[half ? i1 : i0], &sc);
        if (hl == 0 && (half == 0 || two)) { fs.c_cat[half ? i1 : i0] = cat; fs.c_score[half ? i1 : i0] = sc; }
      }
    }
    if (PROF && tid == 0) { vt_rows += nd; vt_fallback += nd > VT_DIRTY_MAX ? 1 : 0; }
    __syncthreads();
    Best b{0.0, -1, 0, 0};
    int n0 = 0, n1 = 0;
    for (int i = tid; i < nmine; i += blockDim.x) {
      const int cat = fs.c_cat[i];
      if (cat == 0 || (FUT && cat == 1)) best_fold(b, fs.c_score[i], nbase + i, 1, cat);
      if (FUT) { n0 += cat == 0; n1 += cat == 1; }
    }
    post_warp(b, n0, n1);
  };
  // CMD_EVAL (warp 1): re-evaluate node F.ev_i for the cached group, maintain this CTA's best incrementally
  // (rescan only when the holder got worse) and publish the CTA's new best in the ring.
  int n_spec_hit = 0, n_rescan = 0, n_eval = 0;
  unsigned ev_count = 0;  // CMD_EVAL commands seen by this warp (warps 1 and 2 count alike)
  long long ev_acc_pub = 0, ev_acc_spec = 0;
  auto eval_and_publish = [&](int my_group) {
    const long long ev_t0 = PROF ? clock64() : 0;
    const int i = F.ev_i;
    const int dn = nbase + i;
    const int old_cat = fs.c_cat[i];
    double sc = 0.0;
    int cat;
    const int rs = (int)(ev_count & 1u);  // written by warp 2 while the previous command was served
    if (F.spec_i[rs] == i && F.spec_group[rs] == my_group && (!FUT || F.spec_kind[rs] == F.ev_kind)) {
      cat = F.spec_cat[rs]; sc = F.spec_sc[rs]; n_spec_hit += 1;
    } else cat = eval_dirty(i, i, 0, 0, fs.c_cs[i], &sc);
    __syncwarp();
    if (lane == 0) { fs.c_cat[i] = cat; fs.c_score[i] = sc; }
    double bs = F.cta_best_score;
    int bn = F.cta_best_node;
    int bcat = FUT ? F.cta_best_cat : 0;
    int cnt = F.cta_cnt + (cat == 0 ? 1 : 0) - (old_cat == 0 ? 1 : 0);
    int cnt1 = FUT ? F.cta_cnt1 + (cat == 1 ? 1 : 0) - (old_cat == 1 ? 1 : 0) : 0;
    bool rescan = false;
    if (!FUT) {
      if (bn == dn) {
        if (cat == 0 && sc >= bs) bs = sc;
        else rescan = true;
      } else if (cat == 0 && (bn < 0 || better(sc, dn, bs, bn))) {
        bs = sc; bn = dn;
      }
    } else {
      if (bn == dn) {
        if (cat == bcat && sc >= bs) bs = sc;
        else rescan = true;
      } else if (cat != 2 && (bn < 0 || better_c(cat, sc, dn, bcat, bs, bn))) {
        bs = sc; bn = dn; bcat = cat;
      }
    }
    __syncwarp();
    n_eval += 1;
    if (rescan) {
      n_rescan += 1;
      int c01[2] = {0, 0};
      Best r = scan_cache<FUT>(fs, nmine, nbase, c01);
      bs = r.score; bn = r.node; bcat = r.cat;
      if (FUT) { cnt = c01[0]; cnt1 = c01[1]; } else cnt = r.cnt;
    }
    if (lane == 0) {
      F.cta_best_score = bs; F.cta_best_node = bn; F.cta_cnt = cnt;
      if (FUT) { F.cta_best_cat = bcat; F.cta_cnt1 = cnt1; }
      Best nb{bs, bn, (FUT && bcat == 1) ? cnt1 : cnt, bcat};
      const bool flag = soft_event(old_cat, cat, fs.c_cs[i]);
      if (SAMP) {  // second vector of the ring entry: the CTA's feasible-node count
        mbox_store(p.ring + (size_t)F.ev_ring * RING_STRIDE + 1, make_uint4((unsigned)(cnt + cnt1), 0u, 0u, F.ev_tag << 10));
        F.ev_feas = cnt + cnt1;
      }
      store_all(p, p.peer_ring, p.ring, (size_t)F.ev_ring * RING_STRIDE, pack_run(nb, F.ev_tag, 1, flag));
      F.ev_score = bs; F.ev_node = bn; F.ev_cnt = min(nb.cnt, 2); F.ev_cat = bcat; F.run_m = 1;
      if (SOFT) F.ev_flag = flag ? 1 : 0;
    }
    __syncwarp();
    asm volatile("bar.arrive 1, 64;" ::: "memory");  // results ready: warp 0 joins with bar.sync 1, 64
    if (PROF) ev_acc_pub += clock64() - ev_t0;
  };
  // CMD_EVAL (warp 2), concurrently with warp 1: run ahead — the same node after ONE MORE placement of this group. Under
  // best-fit scoring the node that just won usually wins again, and then the next command finds its answer here.
  auto run_ahead = [&](int my_group) {
    const long long t0 = PROF ? clock64() : 0;
    const int i = F.ev_i;
    double sc = 0.0;
    const int kind = FUT ? F.ev_kind : 0;  // one more placement of the kind the row just received
    const int cat = eval_dirty(i, i, 1, 1, fs.c_cs[i], &sc, kind);
    const int ws = (int)((ev_count + 1u) & 1u);
    __syncwarp();
    if (lane == 0) { F.spec_sc[ws] = sc; F.spec_cat[ws] = cat; F.spec_group[ws] = my_group; F.spec_i[ws] = i; F.spec_kind[ws] = kind; }
    if (PROF) ev_acc_spec += clock64() - t0;
  };

  // CMD_RUN (warp 2): the runner-up the run is measured against — the best candidate of this CTA other than node
  // F.ev_i, and the best of every other CTA's slot. Neither changes while placements keep landing on F.ev_i.
  auto run_runner_up = [&]() {
    const int i = F.ev_i;
    Best rl{0.0, -1, 0, 0};
    int n0 = 0, n1 = 0;
    for (int k = lane; k < nmine; k += 32) {
      const int cc = fs.c_cat[k];
      if (k == i) continue;
      if (cc == 0 || (FUT && cc == 1)) best_fold(rl, fs.c_score[k], nbase + k, 1, cc);
      if (FUT) { n0 += cc == 0; n1 += cc == 1; }
    }
    best_warp_reduce<FUT>(rl);
    if (FUT) {
      n0 = (int)__reduce_add_sync(0xffffffffu, (unsigned)n0);
      n1 = (int)__reduce_add_sync(0xffffffffu, (unsigned)n1);
    }
    Best ro{0.0, -1, 0, 0};
    for (int sl = lane; sl < G; sl += 32)
      if (sl != cta) best_fold(ro, fs.sl_score[sl], fs.sl_node[sl], 0, FUT ? fs.sl_cat[sl] : 0);
    best_warp_reduce<FUT>(ro);
    if (lane == 0) {
      F.rl_score = rl.score; F.rl_node = rl.node; F.rl_cnt = rl.cnt; F.rl_cat = rl.cat;
      if (FUT) { F.rl_cnt0 = n0; F.rl_cnt1 = n1; }
      Best ru = rl;
      best_fold(ru, ro.score, ro.node, 0, ro.cat);
      F.ru_score = ru.score; F.ru_node = ru.node; F.ru_cat = ru.cat;
    }
    __syncwarp();
  };
  // CMD_RUN, every worker warp: worker e evaluates states 2e and 2e+1 of the row (warp 2 takes the last pair, after
  // the runner-up), one half-warp per state, with the evaluator of the single-node steps
  auto run_states = [&]() {
    const int L = F.run_L;
    // Evaluation slots in an order that fills the four SM sub-partitions one warp each before doubling up (a warp's
    // sub-partition is warp % 4; an fp64 instruction occupies the sub-partition's pipe whatever the number of
    // active lanes, tools/micro/fp64_latency.cu measures it): warps 1, 3, 6, 4, then 5, 7; warp 2 (runner-up first) comes last.
    int e = warp - 1;
    if (nwarps == 8) e = warp == 1 ? 0 : warp == 3 ? 1 : warp == 6 ? 2 : warp == 4 ? 3 : warp == 5 ? 4 : warp == 7 ? 5 : 6;
    else if (warp == 2) e = nwarps - 2;
    else if (warp > 2) e = warp - 2;
    if (warp == 2) { run_runner_up(); DBG_STAGE(warp, 150); }
    if (2 * e < L) {
      double sc = 0.0;
      const int cat = eval_dirty(F.ev_i, F.ev_i, 2 * e, 2 * e + 1, fs.c_cs[F.ev_i], &sc);
      if (hl == 0) { F.run_sc[2 * e + half] = sc; F.run_cat[2 * e + half] = cat; }
    }
    DBG_STAGE(warp, 180);
    asm volatile("bar.sync 2, %0;" ::"r"((nwarps - 1) * 32) : "memory");  // all worker warps
  };
  // CMD_RUN (warp 1): lane l evaluates node F.ev_i as it will be after l further placements of the staged group
  // (state 0 = the row as the control warp's placement left it), with the sweep's own evaluator. The node keeps
  // winning while its state is feasible and beats the runner-up; the run covers those placements, one publication.
  int n_runs = 0, n_run_place = 0;
  long long run_cycles = 0;
  auto run_eval_and_publish = [&]() {
    const long long run_t0 = clock64();
    const int i = F.ev_i;
    const int dn = nbase + i;
    const int L = F.run_L;  // placements the control program allows in a row, the one already applied included
    const int old_cat = fs.c_cat[i];
    const TaskRec &trec = S.trec;
    // states computed by the worker warps (run_states): lane l holds the row after l further placements
    const double sc = lane < L ? F.run_sc[lane] : 0.0;
    const int cat = lane < L ? F.run_cat[lane] : 2;
    const double ru_s = F.ru_score;
    const int ru_n = F.ru_node;
    // lane l < L-1: does the node still win in state l (i.e. does placement l+1 of the run land on it too)?
    // (runs are made of allocations: the row must stay in the idle gradient, which beats any future-idle runner-up)
    const bool win = lane < L - 1 && cat == 0 && (ru_n < 0 || (FUT && F.ru_cat == 1) || better(sc, dn, ru_s, ru_n));
    const unsigned wmask = __ballot_sync(0xffffffffu, win);
    const int m = min(L, __ffs(~wmask));  // 1 + leading wins; state m-1 is the row after the run
    const double sc_m = __shfl_sync(0xffffffffu, sc, m - 1);
    const int cat_m = __shfl_sync(0xffffffffu, cat, m - 1);
    // scores of placements 1..m-1 of the run (placement j is chosen in state j-1 ... of the row BEFORE it: lane j-1)
    if (lane < m - 1) {  // self-validating entries (the reader, CTA 0 of rank 0, polls the tag): no fence on the owner's path
      const unsigned long long sb = (unsigned long long)__double_as_longlong(sc);
      mbox_store(fp.score_log + F.run_att0 + 1 + lane, make_uint4((unsigned)sb, (unsigned)(sb >> 32), (unsigned)(F.run_att0 + 2 + lane), 0u));
    }
    // the remaining m-1 placements on the row (Statement.Allocate: node_info.go:467-471, predicates.go:254-255)
    const double km = (double)(m - 1);
    if (m > 1) {
      if (lane < R) {
        fs.idle[lane * cap + i] -= km * trec.req[lane];
        fs.used[lane * cap + i] += km * trec.req[lane];
      }
      if (c.has_predicates) {
        if (lane == 16) fs.pod_count[i] += m - 1;
        if (lane >= 17 && lane < 17 + K) fs.kreq[(lane - 17) * cap + i] += km * trec.kreq[lane - 17];
        if (lane >= 24 && lane < 26) fs.knz[(lane - 24) * cap + i] += km * trec.knz[lane - 24];
      }
    }
    __syncwarp();
    if (lane == 0) {
      fs.c_cat[i] = cat_m; fs.c_score[i] = sc_m;
      Best nb{F.rl_score, F.rl_node, F.rl_cnt, FUT ? F.rl_cat : 0};
      if (cat_m == 0 || (FUT && cat_m == 1)) best_fold(nb, sc_m, dn, 1, cat_m);
      F.cta_best_score = nb.score; F.cta_best_node = nb.node;
      if (FUT) {
        F.cta_cnt = F.rl_cnt0 + (cat_m == 0 ? 1 : 0); F.cta_cnt1 = F.rl_cnt1 + (cat_m == 1 ? 1 : 0); F.cta_best_cat = nb.cat;
      } else F.cta_cnt = nb.cnt;
      const bool flag = soft_event(old_cat, cat_m, fs.c_cs[i]);
      store_all(p, p.peer_ring, p.ring, (size_t)F.ev_ring * RING_STRIDE, pack_run(nb, F.ev_tag, m, flag));
      F.ev_score = nb.score; F.ev_node = nb.node; F.ev_cnt = min(nb.cnt, 2); F.ev_cat = nb.cat; F.run_m = m;
      if (SOFT) F.ev_flag = flag ? 1 : 0;
      F.spec_i[0] = -1; F.spec_i[1] = -1;  // whatever was computed ahead describes an older state of the row
    }
    n_runs += 1; n_run_place += m;
    __syncwarp();
    asm volatile("bar.arrive 1, 64;" ::: "memory");  // results ready: warp 0 joins with bar.sync 1, 64
    run_cycles += clock64() - run_t0;
  };

  if (warp != 0) {
    // ---- worker warps: serve block-wide commands ----
    int my_group = -1;
    for (;;) {
      __syncthreads();  // B1: command posted
      const int cmd = S.cmd;
      if (cmd == CMD_EXIT) {
        if (warp == 1 && lane == 0) {
          atomicAdd(&p.counters[8], n_spec_hit); atomicAdd(&p.counters[9], n_rescan); atomicAdd(&p.counters[10], n_eval);
          atomicAdd(&p.counters[13], n_runs); atomicAdd(&p.counters[14], n_run_place);
          atomicAdd(&p.counters[15], (int)(run_cycles >> 10));
          if (PROF && n_eval > 0) atomicAdd(&p.counters[11], (int)(ev_acc_pub >> 10));
        }
        if (PROF && warp == 2 && lane == 0) atomicAdd(&p.counters[12], (int)(ev_acc_spec >> 10));
        break;
      }
      if (!SOFT && cmd == CMD_SWEEP && F.vt_reenter) {
        if (F.cur_group != my_group) { stage_ops(); my_group = F.cur_group; }
        reenter_part(true);
      }
      else if (cmd == CMD_SWEEP || cmd == CMD_SWEEP2) sweep_part();
      else if (cmd == CMD_DISCARD) discard_part();
      else if (cmd == CMD_RUN) {  // all worker warps, joined on named barrier 2; warp 1 signals warp 0 on barrier 1
        if (F.cur_group != my_group) { stage_ops(); my_group = F.cur_group; }
        DBG_STAGE(warp, 100 + F.run_L);
        run_states();
        DBG_STAGE(warp, 200 + F.run_L);
        if (warp == 1) { run_eval_and_publish(); DBG_STAGE(1, 300 + F.run_m); }
        continue;
      }
      else if (cmd == CMD_EVAL) {  // no block-wide B2: warp 1 signals warp 0 on named barrier 1
        if (warp == 1 || warp == 2) {
          if (F.cur_group != my_group) { stage_ops(); my_group = F.cur_group; }
          DBG_STAGE(warp, 400);
          if (warp == 1) eval_and_publish(my_group);
          else run_ahead(my_group);
          DBG_STAGE(warp, 500);
          ev_count += 1;
        }
        continue;
      }
      // sweeps and rollbacks change node state without a CMD_EVAL: whatever was computed ahead is void
      if (warp == 1 && lane == 0) { F.spec_i[0] = -1; F.spec_i[1] = -1; }
      __syncthreads();  // B2: command done
    }
  } else {
    // ===================================================================================
    // warp 0: the replicated control program (allocate.go:283-348, :558-694).
    // All 32 lanes execute it in lock step on REGISTER copies of the control state (identical in every
    // lane); shared memory is used only for records loaded/stored once per visit and for what the worker
    // warps read. Per-dimension vectors (drf / proportion accumulators) live one dimension per lane.
    // ===================================================================================
    const bool out_cta = (cta == 0);
    // hdrf: the queue PQ is a simulated Go heap run by lane 0 on the tree replica; hd_n (its size) is kept in every lane
    int hd_n = 0;
    if (p.hd_on) {
      if (lane == 0)
        hd_n = hd_open(p.hd, lcta, reinterpret_cast<const double *>(reinterpret_cast<const char *>(jdyn) + offsetof(JobDyn, alloc)),
                       sizeof(JobDyn) / 8, 1, reinterpret_cast<const double *>(reinterpret_cast<const char *>(jdyn) + offsetof(JobDyn, share)),
                       sizeof(JobDyn) / 8, reinterpret_cast<const double *>(reinterpret_cast<const char *>(qdyn) + offsetof(QueueDyn, share)),
                       sizeof(QueueDyn) / 8);
      hd_n = __shfl_sync(0xffffffffu, hd_n, 0);
    }
    // ---- register copies of the control state ----
    int cur_group = -1, cache_group = -1, since_sync = 0;
    unsigned ag = 0, pc = 0;
    int n_dec = 0, n_vis = 0, n_fit = 0, n_steps = 0, n_full = 0, n_incr = 0, visit_id = 0, n_owner_change = 0, last_owner = -1;
    double g_best_score = 0.0;
    int g_best_node = -1, g_cnt = 0, g_best_owner = -1;
    // SAMP: util.lastProcessedNodeIndex, feasible nodes of its CTA at or after it (for the cached group), and whether
    // that count is current
    int s_start = SAMP ? c.last_idx0 : 0, s_tail = 0, s_total = 0;  // s_total: feasible nodes over all CTAs
    bool s_tail_valid = false;
    SampWin sp_w{0, 0, 0, 0, 0, false};  // SAMP: the window issued one step ahead, its ring slots
    unsigned sp_pa = 0, sp_pb = 0;
    bool sp_valid = false;
    int g_best_cat = 0, g_cnt1 = 0;  // FUT: g_cnt / g_cnt1 = candidates of category 0 / 1 over all CTAs (each clamped to 2 per CTA)
    bool pub_pending = false;
    long long t_a = 0, t_b = 0, t_c = 0, acc_ab = 0, acc_bc = 0, acc_cp = 0, acc_ja = 0;
    long long t_post = 0, t_join = 0, acc_post_to_joinstart = 0, acc_join_wait = 0, acc_join_to_post = 0; int acc_n = 0;
    int pub_owner = -1, pub_node = -1;
    unsigned pub_pc = 0;
    int n_att = 0;   // placement attempts so far (index into the score log; every task is attempted at most once)
    int pub_m = 1;   // placements covered by the publication resolve() consumed last
    // Per-group verdict table. F.vt_clock: a clock that advances each time a group's cache stops being current (the
    // group's stamp takes its value first); every change of a row stamps the row with it, so the rows a group has to
    // re-evaluate on re-entry are exactly those with a larger stamp. F.vt_held: the group whose verdicts the CTA's cache
    // holds, exact for every row stamped at most F.vt_held_stamp (or current, when it is cache_group). (Shared memory,
    // written by lane 0: the control warp has no registers to spare for them.)
    auto vt_stop = [&]() {
      if (!VT || cache_group < 0) return;
      __syncwarp();
      if (lane == 0) {
        const int clk = F.vt_clock;
        VT_GSTAMP(cache_group) = clk;
        F.vt_held_stamp = clk;
        F.vt_clock = clk + 1;
      }
      __syncwarp();
    };

    // Visit state that survives from one visit to the next: a re-pushed job is usually popped again right away
    // (one task per visit once it is Ready, allocate.go:676), and a session often has few queues — so the queue
    // and job records of the previous visit are kept in registers / shared memory and only reloaded from the
    // L2-resident replica when the queue or the job actually changes.
    const bool q_mirror = Q <= FAST_MAXQ;
    int last_q = -1, last_j = -1, cand_tag = -1, cand_sc = -1, cand_js = -1;
    int sbeg = 0, send = 0, q_scursor = 0, q_hsize = 0;
    uint32_t qflags = 0, qdes_has = 0, qflags2 = 0, qalloc_has = 0;
    double qshare = 0.0, qalloc_l = 0.0, qdes_l = 0.0;
    HeapKey *h = heap;
    int task_off = 0, task_end = 0, role_base = 0, nroles = 0, minav = 0, pbe = 0, taskmintotal = 0, ntasks_total = 0;
    uint32_t jflags = 0;
    unsigned long long jkey_pre = 0, jkey_post = 0;
    int cursor = 0, ready = 0, waiting = 0, n_ops = 0;
    double jshare = 0.0, jalloc_l = 0.0;
    bool role_min_active = false, pure = false;
    int4 meta = make_int4(0, 0, 0, 0);

    for (;;) {
      // ---- queues.Pop(): arg-min by ssn.QueueOrderFn over the active queues ----
      int bq = -1, bprio = 0;
      double bshare = 0.0;
      uint32_t brank = 0;
      if (p.hd_on) {  // hdrf: heap.Pop under the comparator chain on the tree as it is
        int qq = -1;
        if (lane == 0 && hd_n > 0) qq = hd_pop(p.hd, lcta, hd_n);
        bq = __shfl_sync(0xffffffffu, qq, 0);
        hd_n = hd_n > 0 ? hd_n - 1 : 0;
      } else {
      for (int q = lane; q < Q; q += 32) {
        if (!(q_mirror ? F.q_active[q] : qdyn[q].active)) continue;
        int pr = f_qorder_prop ? __ldg(&fp.qstat[q].prio) : 0;
        double sh = f_qorder_prop ? (q_mirror ? F.q_share[q] : qdyn[q].share) : 0.0;
        uint32_t rk = __ldg(&fp.qstat[q].rank);
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
      }
      const int q = bq;
      if (q < 0) break;
      __syncwarp();
      // ---- queue records (one coalesced access each), head of the static job list, heap top ----
      if (q != last_q) {
        load_record(&F.qs, &fp.qstat[q], sizeof(QueueStatic) / 4, true);
        load_record(&F.qd, &qdyn[q], sizeof(QueueDyn) / 4, false);
        sbeg = __ldg(&p.qjobs_off[q]); send = __ldg(&p.qjobs_off[q + 1]);
        h = heap + __ldg(&fp.heap_off[q]);
        __syncwarp();
        qflags = F.qs.flags; qdes_has = F.qs.des_has;
        qflags2 = F.qd.flags2; qalloc_has = F.qd.alloc_has;
        q_scursor = F.qd.scursor; q_hsize = F.qd.hsize;
        qshare = F.qd.share;
        // one dimension per lane
        qalloc_l = lane < R ? F.qd.alloc[lane] : 0.0;
        qdes_l = lane < R ? F.qs.des[lane] : 0.0;
        last_q = q; last_j = -1; cand_tag = -1; cand_sc = -1;
      }
      // ssn.Overused: attr.deserved.LessEqual(attr.allocated, Zero), proportion.go:319-331
      bool over = false;
      if (f_over_prop && (qflags2 & 1u)) {
        bool ok = true;
        if (lane < R && (lane < 2 || (qdes_has & (1u << lane)))) {
          double rv = (lane < 2 || (qalloc_has & (1u << lane))) ? qalloc_l : 0.0;
          ok = le_eps(qdes_l, rv);
        }
        over = __all_sync(0xffffffffu, ok);
      }
      int j = -1;
      bool job_loaded = false;  // F.js / F.jd hold records that differ from the register state
      bool visit_from_heap = false;  // the job of this visit was popped from the heap of re-pushed jobs
      if (!over) {
        const int sc = sbeg + q_scursor;
        const int hs = q_hsize;
        const bool have_s = sc < send, have_h = hs > 0;
        int js = -1;
        if (have_s) {
          if (sc != cand_sc) { cand_js = __ldg(&p.qjobs[sc]); cand_sc = sc; }
          js = cand_js;
        }
        if (have_s && cand_tag != js) {
          // records of the static candidate: needed for the comparison and, if chosen, as the job state; a job
          // at the head of the static list has not been visited yet, so its records cannot go stale
          __syncwarp();
          load_record(&F.js2, &fp.jstat[js], sizeof(JobStatic) / 4, true);
          load_record(&F.jd2, &jdyn[js], sizeof(JobDyn) / 4, false);
          cand_tag = js;
        }
        HeapKey top;
        if (have_h) top = h[0];
        __syncwarp();
        bool from_heap = false;
        if (have_s && have_h) {
          HeapKey ks;
          ks.pre = F.js2.key_pre; ks.post = F.js2.key_post;
          const bool rdy = F.jd2.ready + F.js2.pending_besteffort >= F.js2.min_available;
          if (rdy && fp.ready_word == 1) ks.pre |= 1ull << fp.ready_shift;
          if (rdy && fp.ready_word == 2) ks.post |= 1ull << fp.ready_shift;
          ks.share = fp.share_on ? (unsigned long long)__double_as_longlong(F.jd2.share) : 0ull;
          from_heap = hk_less(top, ks);
        } else if (have_h) {
          from_heap = true;
        }
        visit_from_heap = from_heap;
        if (from_heap) {
          j = top.job;
          if (lane == 0) {  // heap pop: sift-down (only jobs that were re-pushed live here)
            int n = hs - 1;
            const HeapKey last = h[n];
            int i = 0;
            for (;;) {
              int l = 2 * i + 1;
              if (l >= n) break;
              HeapKey cl = h[l];
              if (l + 1 < n) {
                const HeapKey cr = h[l + 1];
                if (hk_less(cr, cl)) { cl = cr; l = l + 1; }
              }
              if (!hk_less(cl, last)) break;
              h[i] = cl;
              i = l;
            }
            if (n > 0) h[i] = last;
          }
          q_hsize = hs - 1;
          __syncwarp();
          if (j != last_j) {  // otherwise the registers still hold this job's state from its previous visit
            load_record(&F.js, &fp.jstat[j], sizeof(JobStatic) / 4, true);
            load_record(&F.jd, &jdyn[j], sizeof(JobDyn) / 4, false);
            job_loaded = true;
          }
        } else if (have_s) {
          j = js;
          q_scursor += 1;
          __syncwarp();
          for (int w = lane; w < (int)(sizeof(JobStatic) / 4); w += 32)
            reinterpret_cast<int *>(&F.js)[w] = reinterpret_cast<const int *>(&F.js2)[w];
          for (int w = lane; w < (int)(sizeof(JobDyn) / 4); w += 32)
            reinterpret_cast<int *>(&F.jd)[w] = reinterpret_cast<const int *>(&F.jd2)[w];
          cand_tag = -1;
          job_loaded = true;
        }
      }
      __syncwarp();
      if (j < 0) {  // queue dropped: overused, or no jobs left (allocate.go:295-305)
        if (lane == 0) {
          qdyn[q].active = 0; qdyn[q].scursor = q_scursor; qdyn[q].hsize = q_hsize;
          if (q_mirror) F.q_active[q] = 0;
        }
        __syncwarp();
        continue;
      }
      // ---- job state into registers; roles into the shared role tables ----
      n_ops = 0;
      int vrun_extra = 0;  // further single-task visits of this (Ready) job folded into this pass of the loop
      if (job_loaded) {
        task_off = F.js.task_off; task_end = F.js.task_end;
        role_base = F.js.role_off; nroles = F.js.n_roles;
        minav = F.js.min_available; pbe = F.js.pending_besteffort; taskmintotal = F.js.task_min_total;
        ntasks_total = F.js.n_tasks_total;
        jflags = F.js.flags;
        jkey_pre = F.js.key_pre; jkey_post = F.js.key_post;
        cursor = task_off + F.jd.cursor; ready = F.jd.ready; waiting = F.jd.waiting;
        jshare = F.jd.share;
        jalloc_l = lane < R ? F.jd.alloc[lane] : 0.0;
        bool role_min_any = false;
        for (int r = lane; r < nroles; r += 32) {
          const RoleStatic rs = fp.rstat[role_base + r];
          const RoleDyn rd = rdyn[role_base + r];
          S.r_occ[r] = rd.occ; S.r_pip[r] = rd.pip; S.r_pending[r] = rd.pending; S.r_failed[r] = (uint8_t)rd.failed;
          S.r_min[r] = rs.min; S.r_flags[r] = rs.flags;
          if (rs.flags & VC_ROLE_IN_MIN_MAP) role_min_any = true;
        }
        role_min_any = __any_sync(0xffffffffu, role_min_any);
        // CheckTaskReady (job_info.go:1024-1036) can only fail when role minima are in force
        role_min_active = role_min_any && !(minav < taskmintotal);
        if (lane == 0) {
          S.minav = minav; S.taskmintotal = taskmintotal; S.nroles = nroles; S.pbe = pbe; S.ntasks_total = ntasks_total;
          S.role_base = role_base;
        }
        pure = (jflags & VC_JOBX_PURE) != 0;
        meta = __ldg(&p.tmeta[cursor]);
      }
      last_j = j;
      visit_id += 1;  // util.NewPredicateHelper(): a fresh error cache per visit
      __syncwarp();
      // ssn.JobReady (session_plugins.go:428-446) on the register state
      auto job_ready_now = [&]() -> bool {
        if (!f_gang_ready) return true;
        if (role_min_active) {
          bool ok = true;
          for (int r = 0; r < nroles; ++r)
            if ((S.r_flags[r] & VC_ROLE_IN_MIN_MAP) && S.r_occ[r] < S.r_min[r]) ok = false;
          if (!ok) return false;
        }
        return ready + pbe >= minav;
      };
      FPROF_MARK(0);
      // Consume the publication of the last placement (made while the verdict cache was valid): the owner CTA
      // joins its evaluator warp (B2 of CMD_EVAL), every other CTA reads the one ring record; then the global
      // best is maintained incrementally (refolded only when its holder got worse).
      auto resolve = [&]() {
        if (!pub_pending) return;
        pub_pending = false;
        const int o = pub_owner;
        if (o != last_owner) { n_owner_change += 1; last_owner = o; }
        Best nb;
        if (o == cta) {
          const long long t0_ = PROF ? clock64() : 0;
          DBG_STAGE(0, (int)(pub_pc << 4) | 4);
          asm volatile("bar.sync 1, 64;" ::: "memory");  // join the evaluator warp
          DBG_STAGE(0, (int)(pub_pc << 4) | 5);
          nb.score = F.ev_score; nb.node = F.ev_node; nb.cnt = F.ev_cnt; nb.cat = FUT ? F.ev_cat : 0; pub_m = F.run_m;
          if (SOFT && F.ev_flag) cache_group = -1;  // a normalisation constant may have moved: full sweep next
          if (PROF && !SAMP) {
            // the barrier blocks lazily: read the clock only after a value that needs it has arrived
            long long tj;
            asm volatile("{ .reg .b32 t; mov.b32 t, %1; mov.u64 %0, %%clock64; }" : "=l"(tj) : "r"(nb.node) : "memory");
            t_join = tj;
            acc_post_to_joinstart += t0_ - t_post; acc_join_wait += t_join - t0_; acc_n += 1;
          }
        } else {
          t_join = 0;
          const unsigned tag = (pub_pc + 1u) & RUN_TAG_MASK;
          const uint4 *ent = p.ring + (size_t)(pub_pc % RING_DEPTH) * RING_STRIDE;
          uint4 v;
          unsigned spins = 0;
          const long long t0w = clock64();
#undef WD_EXTRA
#define WD_EXTRA do { if (PROF && p.dbg && lane == 0) { volatile int *dd = p.dbg + (size_t)(o - p.cta_base) * 8; \
            printf("  waits for pub %u of CTA %d (node %d, ring word %08x); owner stages: ctl %d:%d w1-7 %d %d %d %d %d %d %d\n", pub_pc, o, pub_node, v.w, \
                   dd[0] >> 4, dd[0] & 15, dd[1], dd[2], dd[3], dd[4], dd[5], dd[6], dd[7]); } } while (0)
          do { v = mbox_load(ent); PEER_WATCHDOG(spins, t0w); } while ((v.w >> 10) != tag);
#undef WD_EXTRA
#define WD_EXTRA
          nb = unpack_best(v);
          pub_m = (int)((v.w >> 3) & 0x3fu);
          if (SOFT && (v.w & 0x200u)) cache_group = -1;
          if (SAMP) {
            uint4 x;
            do { x = mbox_load(ent + 1); PEER_WATCHDOG(spins, t0w); } while ((x.w >> 10) != tag);
            // (the count at or after s_start follows when the re-evaluated node lies there)
            if (o == s_start / p.npc && pub_node >= s_start) s_tail += (int)x.x - fs.sl_feas[o];
            s_total += (int)x.x - fs.sl_feas[o];
            __syncwarp();
            if (lane == 0) fs.sl_feas[o] = (int)x.x;
          }
        }
        if (SAMP) {  // the window logic reads the slot table only
          if (o == cta) {
            if (o == s_start / p.npc && pub_node >= s_start) s_tail += F.ev_feas - fs.sl_feas[o];
            s_total += F.ev_feas - fs.sl_feas[o];
            __syncwarp();
            if (lane == 0) fs.sl_feas[o] = F.ev_feas;
          }
          __syncwarp();
          if (lane == 0) { fs.sl_score[o] = nb.score; fs.sl_node[o] = nb.node; fs.sl_cnt[o] = nb.cnt; fs.sl_cat[o] = nb.cat; }
          __syncwarp();
          since_sync += 1;
          return;
        }
        const int old_cnt = fs.sl_cnt[o];
        bool refold = false;
        if (!FUT) {
          g_cnt += nb.cnt - old_cnt;
          if (g_best_owner == o) {
            if (nb.node >= 0 && (better(nb.score, nb.node, g_best_score, g_best_node) ||
                                 (nb.node == g_best_node && nb.score == g_best_score))) {
              g_best_score = nb.score; g_best_node = nb.node;
            } else {
              refold = true;
            }
          } else if (nb.node >= 0 && (g_best_node < 0 || better(nb.score, nb.node, g_best_score, g_best_node))) {
            g_best_score = nb.score; g_best_node = nb.node; g_best_owner = o;
          }
        } else {
          if (fs.sl_cat[o] == 0) g_cnt -= old_cnt; else g_cnt1 -= old_cnt;
          if (nb.cat == 0) g_cnt += nb.cnt; else g_cnt1 += nb.cnt;
          if (g_best_owner == o) {
            if (nb.node >= 0 && (better_c(nb.cat, nb.score, nb.node, g_best_cat, g_best_score, g_best_node) ||
                                 (nb.node == g_best_node && nb.score == g_best_score && nb.cat == g_best_cat))) {
              g_best_score = nb.score; g_best_node = nb.node; g_best_cat = nb.cat;
            } else {
              refold = true;
            }
          } else if (nb.node >= 0 && (g_best_node < 0 || better_c(nb.cat, nb.score, nb.node, g_best_cat, g_best_score, g_best_node))) {
            g_best_score = nb.score; g_best_node = nb.node; g_best_cat = nb.cat; g_best_owner = o;
          }
        }
        __syncwarp();
        if (lane == 0) { fs.sl_score[o] = nb.score; fs.sl_node[o] = nb.node; fs.sl_cnt[o] = nb.cnt; fs.sl_cat[o] = nb.cat; }
        __syncwarp();
        since_sync += 1;
        if (refold) {
          __syncwarp();
          Best g = fold_slots<FUT>(fs, G, &g_best_owner);
          g_best_score = g.score; g_best_node = g.node; g_best_cat = g.cat;
          if (!FUT) g_cnt = g.cnt;  // (FUT: the per-category totals were updated above)
        }
      };

      // full sweep of this CTA's nodes for the staged group (every warp), reduced to the CTA's best and, for the FUT
      // instance, its node counts per category
      // (a pure job's group with verdicts saved this cycle re-enters from them: see reenter_part)
      auto sweep_local = [&](int grp, int rl, bool use_cache, Best &mine, int &c0, int &c1) {
          bool reenter = false;
          if (VT) {
            vt_stop();
            int st = -1;
            if (lane == 0) {
              const int held = F.vt_held;
              if (pure) st = held == grp ? F.vt_held_stamp : VT_GSTAMP(grp);
              F.vt_wb = (held >= 0 && !(st >= 0 && held == grp)) ? held : -1;
              F.vt_reenter = st >= 0 ? 1 : 0; F.vt_load = held != grp ? 1 : 0; F.vt_stamp = st; F.vt_nd = 0;
              F.vt_held = pure ? grp : -1;
            }
            reenter = __shfl_sync(0xffffffffu, st, 0) >= 0;
          }
          if (PROF && lane == 0) F.vt_n[reenter ? 1 : 0] += 1;
          if (lane == 0) { S.cmd = CMD_SWEEP; S.sweep_rl = rl; S.sweep_use_cache = use_cache ? 1 : 0; S.visit_id = visit_id; }
          __syncthreads();  // B1
          if (!SOFT && reenter) reenter_part(false);
          else sweep_part();
          __syncthreads();  // B2
          if (SOFT) {
            // first phase done (verdicts, NodeOrderFn sums, per-warp soft-taint maxima): all-gather the maxima, then the
            // second phase adds the normalised TaintToleration score and folds the bests
            int m0 = lane < nwarps ? S.w_soft[0][lane] : 0, m1 = lane < nwarps ? S.w_soft[1][lane] : 0;
            m0 = (int)__reduce_max_sync(0xffffffffu, (unsigned)m0);
            m1 = (int)__reduce_max_sync(0xffffffffu, (unsigned)m1);
            Best sm{0.0, m0 | (m1 << 8), 0, 0};
            exchange_all_fast(p, sm, ag, fs);
            ag += 1;
            int g0 = 0, g1 = 0;
            for (int sl = lane; sl < G; sl += 32) { g0 = max(g0, fs.sl_node[sl] & 0xff); g1 = max(g1, (fs.sl_node[sl] >> 8) & 0xff); }
            g0 = (int)__reduce_max_sync(0xffffffffu, (unsigned)g0);
            g1 = (int)__reduce_max_sync(0xffffffffu, (unsigned)g1);
            if (lane == 0) { F.g_soft[0] = g0; F.g_soft[1] = g1; S.cmd = CMD_SWEEP2; }
            __syncthreads();  // B1
            sweep_part();
            __syncthreads();  // B2
          }
          FPROF_MARK(2);
          mine = Best{0.0, -1, 0, 0};
          c0 = 0; c1 = 0;
          if (!FUT) {
            if (lane < nwarps) best_fold(mine, S.w_score[0][lane], S.w_node[0][lane], S.w_cnt[0][lane]);
            best_warp_reduce(mine);
          } else {  // per warp: best (score, node, category) + how many of its nodes sit in category 0 / 1
            if (lane < nwarps) {
              best_fold(mine, S.w_score[0][lane], S.w_node[0][lane], 0, S.w_node[1][lane]);
              c0 = S.w_cnt[0][lane]; c1 = S.w_cnt[1][lane];
            }
            best_warp_reduce<true>(mine);
            c0 = (int)__reduce_add_sync(0xffffffffu, (unsigned)c0);
            c1 = (int)__reduce_add_sync(0xffffffffu, (unsigned)c1);
            mine.cnt = mine.node < 0 ? 0 : (mine.cat == 0 ? c0 : c1);
          }
      };
      // ---- allocateResourcesForTasks, allocate.go:558-694 ----
      for (;;) {
        if (cursor >= task_end || N == 0) break;  // no nodes: return nil before touching the tasks (allocate.go:563-567)
        FPROF_MARK(4);
        const int t = meta.x, grp = meta.y, rl = meta.z - role_base;
        cursor += 1;
        if (cursor < task_end) meta = __ldg(&p.tmeta[cursor]);  // prefetch the next task's record
        // ... and, one per lane, the records of the next 32 tasks (run length below); the gates hide the latency
        const int4 mk = (fp.run_max > 1 && cursor + lane < task_end) ? __ldg(&p.tmeta[cursor + lane]) : make_int4(-1, -1, -1, 0);
        if (PROF) t_a = clock64();
        if (grp != cur_group) {  // stage the group's request record (shared: workers read it in sweeps)
          resolve();  // the evaluator works from the record being replaced
          __syncwarp();
          if (lane < R) S.trec.req[lane] = __ldg(&p.g_req[(size_t)lane * p.n_groups + grp]);
          if (lane >= 16 && lane < 16 + K) S.trec.kreq[lane - 16] = __ldg(&p.g_kreq[(size_t)(lane - 16) * p.n_groups + grp]);
          if (lane >= 24 && lane < 26) S.trec.knz[lane - 24] = __ldg(&p.g_knz[(size_t)(lane - 24) * p.n_groups + grp]);
          if (lane == 31) { S.trec.has = __ldg(&p.g_has[grp]); S.trec.klass = __ldg(&p.g_class[grp]); }
          __syncwarp();
          cur_group = grp;
          if (lane == 0) F.cur_group = grp;
          stage_ops();
        }
        const double req_l = lane < R ? S.trec.req[lane] : 0.0;  // request, one dimension per lane
        // ---- ssn.Allocatable -> proportion queueAllocatable (proportion.go:333-348) ----
        if (f_alloc_prop) {
          bool ok = (qflags & VC_QUEUE_OPEN) != 0;
          const uint32_t rq_has = t_has & ~3u;
          const bool fu_nil = (qflags2 & 2u) && rq_has == 0;
          if (lane < R) {
            const int d = lane;
            if (d < 2) {
              if (req_l > 0.0 && qalloc_l + req_l > qdes_l) ok = false;
            } else if (!fu_nil && (rq_has & (1u << d)) && d != p.d.pods_dim) {
              const double al = (qalloc_has & (1u << d)) ? qalloc_l : 0.0;
              const double de = (qdes_has & (1u << d)) ? qdes_l : 0.0;
              if (req_l > 0.0 && al + req_l > de) ok = false;
            }
          }
          if (!__all_sync(0xffffffffu, ok)) continue;
        }
        const uint32_t rflags = S.r_flags[rl];
        const bool named_role = !(rflags & VC_ROLE_EMPTY_NAME);
        if (named_role && S.r_failed[rl]) {  // job.TaskHasFitErrors, allocate.go:600-607
          if (lane == 0 && out_cta) p.fit_errors[n_fit] = t;
          n_fit += 1;
          continue;
        }
        // For a 'pure' job the role-level error cache can never change a verdict (same record, node
        // resources only shrink inside a visit), so it is skipped; other jobs take exact full sweeps.
        const bool use_cache = c.enable_ecache && named_role && !pure;
        FPROF_MARK(1);
        // the gates above do not need the last publication; everything below (global best, sweeps) does
        if (!SAMP) resolve();
        if (PROF) t_b = clock64();

        if (SAMP) {
          // ======== feasible-node sampling: the candidates are the first to_find feasible nodes from s_start ========
          const int Kf = c.to_find, npc_ = p.npc;
          const unsigned lt = (1u << lane) - 1u;
          // feasible nodes of this CTA with local index >= lo, from the verdict cache
          auto count_from = [&](int lo) -> int {
            int n = 0;
            for (int i = lane; i < nmine; i += 32) n += (i >= lo && fs.c_cat[i] != 2) ? 1 : 0;
            return (int)__reduce_add_sync(0xffffffffu, (unsigned)n);
          };
          // all-gather of (best, feasible count, count at or after s_start); fills the slot table and s_tail
          auto sync_exchange = [&](const Best &mine, int feas) {
            const int a_cta = s_start / npc_;
            const int tl = cta == a_cta ? count_from(s_start - nbase) : 0;
            s_tail = exchange_all_samp(p, mine, feas, tl, ag, fs, a_cta);
            int tot = 0;
            for (int sl = lane; sl < G; sl += 32) tot += fs.sl_feas[sl];
            s_total = (int)__reduce_add_sync(0xffffffffu, (unsigned)tot);
            ag += 1; since_sync = 0; s_tail_valid = true;
          };
          bool plain_step = false;  // an incremental step that needed neither a sweep nor a resynchronisation
          if (!(pure && grp == cache_group)) {
            resolve();
            Best mine{0.0, -1, 0, 0};
            int c0 = 0, c1 = 0;
            sweep_local(grp, rl, use_cache, mine, c0, c1);
            const int feas = FUT ? c0 + c1 : mine.cnt;
            if (lane == 0) {
              F.cta_best_score = mine.score; F.cta_best_node = mine.node;
              if (FUT) { F.cta_cnt = c0; F.cta_cnt1 = c1; F.cta_best_cat = mine.cat; } else F.cta_cnt = mine.cnt;
            }
            __syncwarp();
            sync_exchange(mine, feas);
            n_full += 1;
            cache_group = pure ? grp : -1;
          } else {
            if (!s_tail_valid || since_sync >= RING_DEPTH / 2 - 4) {
              resolve();
              Best mine{F.cta_best_score, F.cta_best_node, (FUT && F.cta_best_cat == 1) ? F.cta_cnt1 : F.cta_cnt, FUT ? F.cta_best_cat : 0};
              const int feas = F.cta_cnt + (FUT ? F.cta_cnt1 : 0);
              __syncwarp();
              sync_exchange(mine, feas);
            } else {
              plain_step = true;
            }
            n_incr += 1;
          }
          // ---- the window: CTA A holds s_start, CTA B the to_find-th feasible node; r = how many of B's feasible nodes
          //      (in index order, from local index b_lo) belong to it; wrap = the window runs once around the ring and ends
          //      in A's part before s_start ----
          auto window = [&](SampWin &w) {
            w.A = s_start / npc_;
            w.total = s_total;
            w.B = w.A; w.r = Kf; w.b_lo = s_start - w.A * npc_; w.wrap = false;
            if (w.total < Kf || s_tail >= Kf) return;
            int cum = s_tail;
            bool found = false;
            for (int o0 = 1; o0 < G && !found; o0 += 32) {
              const int off = o0 + lane;
              int sl = w.A + off;
              sl = sl >= G ? sl - G : sl;
              const int f = off < G ? fs.sl_feas[sl] : 0;
              int inc = f;
              for (int d = 1; d < 32; d <<= 1) { const int v = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += v; }
              const unsigned hit = __ballot_sync(0xffffffffu, off < G && cum + inc >= Kf);
              if (hit) {
                const int l = __ffs(hit) - 1;
                const int before = cum + __shfl_sync(0xffffffffu, inc, l) - __shfl_sync(0xffffffffu, f, l);
                w.B = w.A + o0 + l; w.B = w.B >= G ? w.B - G : w.B; w.r = Kf - before; w.b_lo = 0; found = true;
              } else {
                cum += __shfl_sync(0xffffffffu, inc, 31);
              }
            }
            if (!found) { w.B = w.A; w.r = Kf - cum; w.b_lo = 0; w.wrap = true; }
          };
          auto in_window = [&](const SampWin &w, int o) -> bool {  // is CTA o one of the window's CTAs?
            if (w.total < Kf || w.wrap) return true;
            const int d_o = o >= w.A ? o - w.A : o - w.A + G, d_b = w.B >= w.A ? w.B - w.A : w.B - w.A + G;
            return d_o <= d_b;
          };
          // best of this CTA's feasible nodes with local index >= lo, the first `take` of them in index order
          auto scan_part = [&](int lo, int take, Best &b, int &end_local, int &after) {
            b = Best{0.0, -1, 0, 0};
            int base = 0, endl = -1;
            for (int i0 = 0; i0 < nmine; i0 += 32) {
              const int i = i0 + lane;
              const int cc = i < nmine ? fs.c_cat[i] : 2;
              const bool f = i >= lo && cc != 2;
              const unsigned m = __ballot_sync(0xffffffffu, f);
              const int rank = base + __popc(m & lt);
              const bool inc = f && rank < take;
              if (inc) { best_fold(b, fs.c_score[i], nbase + i, 1, cc); endl = i; }
              base += __popc(m);
            }
            best_warp_reduce<FUT>(b);
            end_local = (int)__reduce_max_sync(0xffffffffu, (unsigned)(endl + 1)) - 1;
            after = base - min(base, take);
          };
          auto publish = [&](unsigned slot_pc, const Best &b, int end_local, int after) {
            if (lane == 0) {
              const unsigned tag = (slot_pc + 1u) & RUN_TAG_MASK;
              uint4 *ent = p.ring + (size_t)(slot_pc % RING_DEPTH) * RING_STRIDE;
              mbox_store(ent + 1, make_uint4((unsigned)end_local, (unsigned)after, 0u, tag << 10));
              mbox_store(ent, pack_run(b, tag, 1, false));
            }
          };
          // the two partial CTAs of window w scan their cache and publish (A's part after s_start into slot pa unless the
          // window lies inside A; B's first r feasible nodes into slot pb)
          auto issue = [&](const SampWin &w, unsigned pa, unsigned pb) {
            const bool a_part = !(w.A == w.B && !w.wrap);
            if (cta == w.A && a_part) {
              Best b; int el, af;
              scan_part(s_start - nbase, 0x7fffffff, b, el, af);
              publish(pa, b, el, af);
            }
            if (cta == w.B) {
              Best b; int el, af;
              scan_part(w.b_lo, w.r, b, el, af);
              publish(pb, b, el, af);
            }
          };
          long long tq0 = 0;
#define SAMP_T(acc) do { if (PROF && SAMP) { const long long n_ = clock64(); acc += n_ - tq0; tq0 = n_; } } while (0)
          if (PROF) tq0 = clock64();
          SampWin w;
          unsigned pa = 0, pb = 0;
          // a window issued one step ahead (below) is taken as it is when nothing moved in between
          const bool used_spec = sp_valid && plain_step;
          sp_valid = false;
          if (used_spec) {
            w = sp_w; pa = sp_pa; pb = sp_pb;
          } else {
            window(w);
            if (pub_pending && in_window(w, pub_owner)) {  // the pending publication changes a count the window was built from
              // (its node cannot sit at or after s_start in A: the previous window ended right before s_start, and after
              //  a wrap the step starts with a fresh all-gather)
              resolve();
              window(w);
            }
          }
          FPROF_MARK(2);  // (SAMP profile: 2 = sweep / sync + window, 3 = part scans, poll and fold)
          SAMP_T(acc_post_to_joinstart);  // prof[8]: window (or taking the one issued ahead)
          Best g{0.0, -1, 0, 0};
          int gc0 = 0, gc1 = 0;
          auto add_part = [&](const Best &b) {  // lane-uniform fold of one part's record
            if (b.node < 0) return;
            if (b.cat == 0) gc0 += b.cnt; else gc1 += b.cnt;
            if (g.node < 0 || better_c(b.cat, b.score, b.node, g.cat, g.score, g.node)) { g.score = b.score; g.node = b.node; g.cat = b.cat; }
          };
          if (w.total < Kf) {
            // fewer feasible nodes than wanted: every one of them is a candidate, the scan went once around (processed = N)
            resolve();
            int own = -1;
            g = fold_slots<FUT>(fs, G, &own);
            int t0 = 0, t1 = 0;
            for (int sl = lane; sl < G; sl += 32) { if (fs.sl_cat[sl] == 0) t0 += fs.sl_cnt[sl]; else t1 += fs.sl_cnt[sl]; }
            gc0 = (int)__reduce_add_sync(0xffffffffu, (unsigned)t0);
            gc1 = (int)__reduce_add_sync(0xffffffffu, (unsigned)t1);
            // (s_start stays; should the winner sit at or after it in A, its publication adjusts s_tail when it is consumed)
          } else {
            if (!used_spec) {
              pa = pc; pb = pc + 1u;
              pc += 2; since_sync += 2;
              issue(w, pa, pb);
            }
            SAMP_T(acc_join_wait);  // prof[10]: issue (when not taken from the step before)
            const bool a_part = !(w.A == w.B && !w.wrap);
            // the whole CTAs strictly between A and B (all the others after a wrap): folded from the slot table while the
            // part records are in flight (a pending publication never concerns one of them, see in_window above)
            const int span = w.wrap ? G - 1 : (w.B >= w.A ? w.B - w.A : w.B - w.A + G) - 1;
            if (span > 0) {
              Best mid{0.0, -1, 0, 0};
              int t0 = 0, t1 = 0;
              for (int o = 1 + lane; o <= span; o += 32) {
                int sl = w.A + o;
                sl = sl >= G ? sl - G : sl;
                best_fold(mid, fs.sl_score[sl], fs.sl_node[sl], 0, FUT ? fs.sl_cat[sl] : 0);
                if (fs.sl_node[sl] >= 0) { if (!FUT || fs.sl_cat[sl] == 0) t0 += fs.sl_cnt[sl]; else t1 += fs.sl_cnt[sl]; }
              }
              best_warp_reduce<FUT>(mid);
              gc0 += (int)__reduce_add_sync(0xffffffffu, (unsigned)t0);
              gc1 += (int)__reduce_add_sync(0xffffffffu, (unsigned)t1);
              mid.cnt = 0;
              if (mid.node >= 0) { g.score = mid.score; g.node = mid.node; g.cat = mid.cat; }
            }
            // One poll for everything this step waits for - the previous placement's publication (unless this CTA made
            // it: then its evaluator warp is joined) and the one or two part records, two vectors each: six lanes load
            // one vector each until every tag matches, so the L2 round trips overlap instead of adding up.
            SAMP_T(acc_join_to_post);  // prof[11]: fold of the whole CTAs
            if (pub_pending && pub_owner == cta) resolve();
            const bool po = pub_pending;  // (a foreign owner's record)
            {
              const int which = lane >> 1, vec = lane & 1;  // 0: previous publication, 1: P_B, 2: P_A
              const bool want = lane < 6 && (which == 0 ? po : which == 1 ? true : a_part);
              const unsigned spc = which == 0 ? pub_pc : which == 1 ? pb : pa;
              const unsigned tag = (spc + 1u) & RUN_TAG_MASK;
              const uint4 *ent = p.ring + (size_t)(spc % RING_DEPTH) * RING_STRIDE + vec;
              uint4 v = make_uint4(0u, 0u, 0u, 0u);
              unsigned spins = 0;
              const long long t0w = clock64();
              bool pending;
              do {
                pending = false;
                if (want) { v = mbox_load(ent); pending = (v.w >> 10) != tag; }
                pending = __any_sync(0xffffffffu, pending);
                if (pending) PEER_WATCHDOG(spins, t0w);
              } while (pending);
              if (lane < 6) F.rec[lane] = v;
              __syncwarp();
            }
            SAMP_T(acc_ja);  // prof[12]: poll
            if (po) {  // what resolve() does with a foreign record
              pub_pending = false;
              const int o = pub_owner;
              if (o != last_owner) { n_owner_change += 1; last_owner = o; }
              const Best nb = unpack_best(F.rec[0]);
              const int nf = (int)F.rec[1].x;
              if (o == s_start / npc_ && pub_node >= s_start) s_tail += nf - fs.sl_feas[o];
              s_total += nf - fs.sl_feas[o];
              __syncwarp();
              if (lane == 0) { fs.sl_score[o] = nb.score; fs.sl_node[o] = nb.node; fs.sl_cnt[o] = nb.cnt; fs.sl_cat[o] = nb.cat; fs.sl_feas[o] = nf; }
              __syncwarp();
              since_sync += 1;
            }
            const int end_local = (int)F.rec[3].x, after = (int)F.rec[3].y;
            add_part(unpack_best(F.rec[2]));
            if (a_part) add_part(unpack_best(F.rec[4]));
            // lastProcessedNodeIndex moves past the to_find-th feasible node (predicate_helper.go:135-136)
            const int nxt = w.B * npc_ + end_local + 1;
            s_start = nxt >= N ? 0 : nxt;
            const int X = s_start / npc_;  // the CTA the next window starts in, and its feasible nodes from there on
            // (a winner that sits in CTA X at or after the new start adjusts s_tail when its publication is consumed)
            if (nxt < N && X == w.B) s_tail = after;
            else s_tail = fs.sl_feas[X];
            // ---- one step ahead: the next window only depends on where this one ended, not on which of its nodes wins -
            //      unless the winner's CTA lies inside it (its feasible count is about to change). The parts are scanned
            //      and published now, so that they are in flight during this step's bookkeeping; the next step takes them
            //      if it is a plain incremental step of the same group, and ignores them otherwise.
            SAMP_T(acc_ab);  // prof[13]: records folded, next start
            if (s_tail_valid && since_sync < RING_DEPTH / 2 - 8) {
              SampWin w2;
              window(w2);
              const int own = g.node >= 0 ? g.node / npc_ : -1;
              if (w2.total >= Kf && !w2.wrap && !(own >= 0 && in_window(w2, own))) {
                sp_w = w2; sp_pa = pc; sp_pb = pc + 1u;
                pc += 2; since_sync += 2;
                issue(w2, sp_pa, sp_pb);
                sp_valid = true;
                acc_n += 1;  // prof[9]: windows issued ahead
              }
            }
            SAMP_T(acc_bc);  // prof[14]: issuing the next window
          }
          g_best_score = g.score; g_best_node = g.node; g_best_cat = g.cat;
          g_best_owner = g.node >= 0 ? g.node / npc_ : -1;
          g_cnt = gc0; g_cnt1 = gc1;
          if (!FUT) g_cnt = gc0 + gc1;
          FPROF_MARK(3);
        } else
        if (pure && grp == cache_group) {
          // -------- incremental step: verdict cache, slot table and global best are already current --------
          if (since_sync >= RING_DEPTH / 2) {  // keep the publication ring from being overrun
            Best mine{F.cta_best_score, F.cta_best_node, (FUT && F.cta_best_cat == 1) ? F.cta_cnt1 : F.cta_cnt, FUT ? F.cta_best_cat : 0};
            __syncwarp();
            exchange_all_fast(p, mine, ag, fs);
            ag += 1; since_sync = 0;
          }
          n_incr += 1;
          FPROF_MARK(2);
        } else {
          // -------- full sweep --------
          Best mine{0.0, -1, 0, 0};
          int c0 = 0, c1 = 0;
          sweep_local(grp, rl, use_cache, mine, c0, c1);
          exchange_all_fast(p, mine, ag, fs);
          Best g = fold_slots<FUT>(fs, G, &g_best_owner);
          ag += 1; since_sync = 0; n_full += 1;
          cache_group = pure ? grp : -1;  // verdicts taken under an error cache are not reusable
          if (lane == 0) {
            F.cta_best_score = mine.score; F.cta_best_node = mine.node;
            if (FUT) { F.cta_cnt = c0; F.cta_cnt1 = c1; F.cta_best_cat = mine.cat; } else F.cta_cnt = mine.cnt;
          }
          g_best_score = g.score; g_best_node = g.node; g_best_cat = g.cat;
          if (!FUT) g_cnt = g.cnt;
          else {  // per-category totals over the slot table
            int t0 = 0, t1 = 0;
            for (int sl = lane; sl < G; sl += 32) { if (fs.sl_cat[sl] == 0) t0 += fs.sl_cnt[sl]; else t1 += fs.sl_cnt[sl]; }
            g_cnt = (int)__reduce_add_sync(0xffffffffu, (unsigned)t0);
            g_cnt1 = (int)__reduce_add_sync(0xffffffffu, (unsigned)t1);
          }
        }
        n_steps += 1;
        FPROF_MARK(3);
        if (PROF) t_c = clock64();

        if ((FUT ? g_cnt + g_cnt1 : g_cnt) == 0) {  // no feasible node, allocate.go:639-659
          __syncwarp();
          if (lane == 0) { if (out_cta) p.fit_errors[n_fit] = t; S.r_failed[rl] = 1; }
          n_fit += 1;
          __syncwarp();
          // job.NeedContinueAllocating, api/job_info.go:918-966
          bool cont;
          if (minav >= ntasks_total) {
            cont = false;
          } else if (minav < taskmintotal) {
            int left = 0;
            for (int r = 0; r < nroles; ++r)
              if (!S.r_failed[r]) left += S.r_pending[r];
            cont = ready + left >= minav;
          } else {
            cont = true;
            for (int r = 0; r < nroles; ++r) {
              if (!S.r_failed[r]) continue;
              const int mn = (S.r_flags[r] & VC_ROLE_IN_MIN_MAP) ? S.r_min[r] : 0;
              if (mn != 0 && S.r_occ[r] < mn) cont = false;
            }
          }
          if (cont) continue;
          break;
        }
        const int best = g_best_node;
        // gradient choice (allocate.go:750-776): idle candidates if there are any, else the future-idle ones -> pipeline
        const bool pipe = FUT && g_best_cat == 1;
        const int cnt_sel = pipe ? g_cnt1 : g_cnt;
        const double score = cnt_sel == 1 ? 0.0 : g_best_score;
        // ---- Statement.Allocate / Pipeline: node.AddTask on the owner CTA (api/node_info.go:435-484) ----
        if (best >= nbase && best < nbase + nmine) {
          const int i = best - nbase;
          // (the further placements of a run on this row happen before vclk moves: this stamp covers them)
          if (!SOFT && lane == 0) fs.mstamp[i] = F.vt_clock;
          if (lane < R) {
            if (pipe) {
              fs.pip[lane * cap + i] += req_l;
            } else {
              fs.idle[lane * cap + i] -= req_l;
              fs.used[lane * cap + i] += req_l;
            }
          }
          if (c.has_predicates) {  // predicates AllocateFunc, predicates.go:212-256
            if (lane == 16) fs.pod_count[i] += 1;
            if (lane >= 17 && lane < 17 + K) fs.kreq[(lane - 17) * cap + i] += S.trec.kreq[lane - 17];
            if (lane >= 24 && lane < 26) fs.knz[(lane - 24) * cap + i] += S.trec.knz[lane - 24];
          }
        }
        // every placement made while the verdict cache is valid is followed by exactly one publication of the
        // owner CTA's new best; the owner's evaluator warp starts on it now, overlapping the bookkeeping below
        pub_pending = pure && cache_group == grp;
        // ---- run length: how many placements in a row the control program would make on the winning node if it kept
        //      winning — the following tasks of this visit that share the group and the role, pass the queue's
        //      Allocatable gate, and come before ssn.JobReady turns true (the loop breaks there, allocate.go:676) ----
        int run_L = 1;
        bool vrun = false;  // the run's placements are one visit each (a Ready job gets one task per visit, allocate.go:676)
        if (pub_pending && fp.run_max > 1 && !pipe) {
          // placements (this one included) until ssn.JobReady turns true; <= 0: the job is Ready already
          int need = 0;
          if (f_gang_ready) {
            need = minav - pbe - ready;
            if (role_min_active) {  // CheckTaskReady: every role of the minimum map at its minimum (job_info.go:1024-1036)
              bool other_short = false;
              int need_rl = 0;
              for (int r = 0; r < nroles; ++r)
                if ((S.r_flags[r] & VC_ROLE_IN_MIN_MAP) && S.r_occ[r] < S.r_min[r]) {
                  if (r == rl) need_rl = S.r_min[r] - S.r_occ[r];
                  else other_short = true;  // placements of this role never make the job Ready
                }
              need = other_short ? RUN_MAX + 1 : max(need, need_rl);
            }
          }
          int lim = 0;
          if (need > 1) {
            lim = need;
          } else if (need <= 0 && visit_from_heap && !fp.share_on && q_mirror && !(f_over_prop && (qflags2 & 1u))) {
            // The visit ends with this placement, the statement commits and the job is pushed back with the key it was
            // popped with (Ready bit set, no drf share in ssn.JobOrderFn): it is the head of its queue again. The
            // queue is popped again when ssn.QueueOrderFn does not depend on the share or no other queue is active.
            // hdrf: the shares move with every placement, so only an otherwise empty heap pops the queue again
            bool again = p.hd_on ? hd_n == 0 : !f_qorder_prop;
            if (!again && !p.hd_on) {
              const int na = __popc(__ballot_sync(0xffffffffu, lane < Q && F.q_active[lane] != 0)) +
                             __popc(__ballot_sync(0xffffffffu, lane + 32 < Q && F.q_active[lane + 32] != 0));
              again = na <= 1;  // (the queue of this visit is marked inactive while it is being served or is the one)
            }
            if (again) { lim = RUN_MAX; vrun = true; }
          }
          if (lim > 1) {
            const bool same = mk.y == grp && mk.z - role_base == rl;  // lane l: task l+1 of the run
            const unsigned same_m = __ballot_sync(0xffffffffu, same);
            const int n_same = same_m == 0xffffffffu ? 32 : __ffs(~same_m) - 1;
            run_L = min(min(1 + n_same, lim), fp.run_max);
            if (f_alloc_prop && run_L > 1) {  // queueAllocatable for the placements after this one, per dimension
              int cdim = run_L;
              if (lane < R) {
                const int d = lane;
                const uint32_t rq_has = t_has & ~3u;
                const bool counted = d < 2 || ((rq_has & (1u << d)) && d != p.d.pods_dim);
                // after the first placement attr.allocated carries every requested dimension (proportion.go:475-497)
                if (counted && req_l > 0.0) {
                  double qa = qalloc_l + req_l;  // allocated as the gate of placement 1 sees it
                  const double de = (d < 2 || (qdes_has & (1u << d))) ? qdes_l : 0.0;
                  int cnt_ok = 1;
                  while (cnt_ok < run_L && !(qa + req_l > de)) { qa += req_l; cnt_ok += 1; }
                  cdim = cnt_ok;
                }
              }
              run_L = (int)__reduce_min_sync(0xffffffffu, (unsigned)cdim);
            }
          }
          if (run_L <= 1) vrun = false;
        }
        const int att0 = n_att;
        if (pub_pending) {
          pub_owner = g_best_owner; pub_node = best; pub_pc = pc; pc += 1;
          if (pub_owner == cta) {
            __syncwarp();
            if (lane == 0) {
              F.ev_i = best - nbase; F.ev_ring = (int)(pub_pc % RING_DEPTH); F.ev_tag = (pub_pc + 1u) & RUN_TAG_MASK;
              F.run_L = run_L; F.run_att0 = att0;
              if (FUT) F.ev_kind = pipe ? 1 : 0;
              S.cmd = run_L > 1 ? CMD_RUN : CMD_EVAL;
            }
            DBG_STAGE(0, (int)(pub_pc << 4) | (run_L > 1 ? 1 : 2));
            __syncthreads();  // B1 of CMD_EVAL
            DBG_STAGE(0, (int)(pub_pc << 4) | 3);
            if (PROF) t_post = clock64();
            if (PROF && !SAMP && t_join != 0) { acc_join_to_post += t_post - t_join; acc_ja += t_a - t_join; acc_ab += t_b - t_a; acc_bc += t_c - t_b; acc_cp += t_post - t_c; }
          }
        }
        // job.UpdateTaskStatus + event handlers: drf (drf.go:391-418), proportion (proportion.go:475-497)
        if (pipe) waiting += 1; else ready += 1;
        if (lane == 0) {
          S.r_pending[rl] -= 1;
          if (pipe) S.r_pip[rl] += 1; else S.r_occ[rl] += 1;
          ops[n_ops * 3 + 0] = t; ops[n_ops * 3 + 1] = best; ops[n_ops * 3 + 2] = pipe ? VC_OP_PIPELINE : VC_OP_ALLOCATE;
          ops_score[n_ops] = score;
        }
        n_ops += 1;
        n_att += 1;
        int extra = 0;  // further placements of a run on the same node (same group, same role), announced by its publication
        if (run_L > 1) {
          const int cnt_run = cnt_sel;  // candidates at every placement of the run (only the winner's row changes)
          resolve();
          extra = pub_m - 1;
          if (extra > 0) {
            if (lane < extra) {
              const int tj = mk.x;  // lane l: task l+1 of the run
              const int k = n_ops + lane;
              ops[k * 3 + 0] = tj; ops[k * 3 + 1] = best; ops[k * 3 + 2] = VC_OP_ALLOCATE;
              if (out_cta) {
                double sv = 0.0;
                if (cnt_run != 1) {  // the owner's entry for this attempt (usually there already: it was stored before the record)
                  uint4 v;
                  unsigned spins = 0;
                  const long long t0w = clock64();
                  do { v = mbox_load(fp.score_log + att0 + 1 + lane); PEER_WATCHDOG(spins, t0w); } while (v.z != (unsigned)(att0 + 2 + lane));
                  sv = __longlong_as_double((long long)((unsigned long long)v.x | ((unsigned long long)v.y << 32)));
                }
                ops_score[k] = sv;
              }
            }
            if (lane == 0) { S.r_pending[rl] -= extra; S.r_occ[rl] += extra; }
            ready += extra; n_ops += extra; n_att += extra; cursor += extra; n_steps += extra; n_incr += extra;
            if (vrun) vrun_extra = extra;
            // the record of the task after the run sits in lane `extra` (31 at most; a lane past the job's end holds -1s)
            meta.x = __shfl_sync(0xffffffffu, mk.x, extra); meta.y = __shfl_sync(0xffffffffu, mk.y, extra);
            meta.z = __shfl_sync(0xffffffffu, mk.z, extra); meta.w = __shfl_sync(0xffffffffu, mk.w, extra);
          }
        }
        if (c.has_drf) {
          for (int e = 0; e <= extra; ++e) jalloc_l += req_l;
          double sh = 0.0;
          if (lane < R && (lane < 2 || (p.total_has & (1u << lane))) && p.total[lane] >= VC_MIN_RESOURCE) sh = share_of(jalloc_l, p.total[lane]);
          for (int o = 16; o; o >>= 1) sh = fmax(sh, __shfl_xor_sync(0xffffffffu, sh, o));
          jshare = sh;
        }
        if (c.has_proportion && (qflags2 & 1u)) {
          if (lane < 2 || (lane < R && (t_has & (1u << lane))))
            for (int e = 0; e <= extra; ++e) qalloc_l += req_l;
          const uint32_t add = t_has & ~3u & ((1u << R) - 1u);
          if (add) { qalloc_has |= add; qflags2 &= ~2u; }
          double sh = 0.0;
          if (lane < R && (lane < 2 || (qdes_has & (1u << lane))) && qdes_l >= VC_MIN_RESOURCE) {
            const double al = (lane < 2 || (qalloc_has & (1u << lane))) ? qalloc_l : 0.0;
            sh = share_of(al, qdes_l);
          }
          for (int o = 16; o; o >>= 1) sh = fmax(sh, __shfl_xor_sync(0xffffffffu, sh, o));
          qshare = sh;
        }
        if (role_min_active) __syncwarp();
        if (job_ready_now()) break;  // ssn.SubJobReady, allocate.go:676-678
      }
      FPROF_MARK(4);
      // The publication of the visit's last placement is NOT awaited here: the statement bookkeeping and the next
      // queue / job pop below do not depend on it, so they overlap the evaluator; the next task's resolve() (or the
      // rollback just below, or the exit path) consumes it.

      // ---- statement outcome, allocate.go:681-693 and :330-337 ----
      __syncwarp();
      const bool jready = job_ready_now() && N != 0;
      bool stmt = jready;
      if (!stmt && N != 0) {  // ssn.JobPipelined needs the shared control block (rare path)
        if (lane == 0) { S.ready = ready; S.waiting = waiting; }
        __syncwarp();
        stmt = ctl_job_pipelined(c, S);
      }
      if (!stmt && n_ops > 0) {
        resolve();  // the evaluator must be idle and the slot table current before nodes are rolled back
        vt_stop();  // (the cache keeps the group's verdicts; a re-entry re-evaluates the rows rolled back)
        if (lane == 0) { S.cmd = CMD_DISCARD; S.n_ops = n_ops; }
        __syncthreads();  // B1
        discard_part();
        __syncthreads();  // B2
        for (int k = n_ops - 1; k >= 0; --k) {  // unallocate + DeallocateFunc handlers, reverse order
          const int ot = ops[k * 3 + 0];
          const int orl = p.t_role[ot] - role_base;
          const bool was_pipe = FUT && ops[k * 3 + 2] == VC_OP_PIPELINE;
          if (lane == 0) { S.r_pending[orl] += 1; if (was_pipe) S.r_pip[orl] -= 1; else S.r_occ[orl] -= 1; }
          if (was_pipe) waiting -= 1; else ready -= 1;
          const double orq = lane < R ? p.req[(size_t)lane * T + ot] : 0.0;
          if (c.has_drf) jalloc_l -= orq;
          if (c.has_proportion && (qflags2 & 1u)) {
            const uint32_t oh = p.req_has[ot];
            if (lane < 2) qalloc_l -= orq;
            else if (!(qflags2 & 2u) && lane < R && (oh & (1u << lane))) qalloc_l -= orq;
            if (!(qflags2 & 2u)) qalloc_has |= oh & ~3u & ((1u << R) - 1u);
          }
        }
        if (c.has_drf) {
          double sh = 0.0;
          if (lane < R && (lane < 2 || (p.total_has & (1u << lane))) && p.total[lane] >= VC_MIN_RESOURCE) sh = share_of(jalloc_l, p.total[lane]);
          for (int o = 16; o; o >>= 1) sh = fmax(sh, __shfl_xor_sync(0xffffffffu, sh, o));
          jshare = sh;
        }
        if (c.has_proportion && (qflags2 & 1u)) {
          double sh = 0.0;
          if (lane < R && (lane < 2 || (qdes_has & (1u << lane))) && qdes_l >= VC_MIN_RESOURCE) {
            const double al = (lane < 2 || (qalloc_has & (1u << lane))) ? qalloc_l : 0.0;
            sh = share_of(al, qdes_l);
          }
          for (int o = 16; o; o >>= 1) sh = fmax(sh, __shfl_xor_sync(0xffffffffu, sh, o));
          qshare = sh;
        }
        cache_group = -1;  // several nodes changed at once: drop the verdict cache
        __syncwarp();
      }
      // results (CTA 0): decisions copied lane-parallel
      if (out_cta && stmt) {
        for (int k = lane; k < n_ops; k += 32) {
          vc_decision dcs;
          dcs.task = ops[k * 3 + 0]; dcs.node = ops[k * 3 + 1]; dcs.kind = ops[k * 3 + 2];
          dcs.visit = n_vis + (vrun_extra ? k : 0); dcs.score = ops_score[k];
          p.decisions[n_dec + k] = dcs;
        }
      }
      if (out_cta && lane <= vrun_extra) {  // one record per visit; a folded run of visits carries one operation each
        vc_visit v;
        v.job = j;
        v.outcome = stmt ? (jready ? VC_VISIT_COMMIT : VC_VISIT_KEEP) : VC_VISIT_DISCARD;
        v.first_op = n_dec + lane;
        v.n_ops = vrun_extra ? 1 : (stmt ? n_ops : 0);
        p.visits[n_vis + lane] = v;
      }
      if (stmt) n_dec += n_ops;
      n_vis += 1 + vrun_extra;
      visit_id += vrun_extra;
      // jobs.Push(job) when committed and tasks remain (allocate.go:334-336)
      if (stmt && jready && cursor < task_end) {
        if (lane == 0) {
          HeapKey e;
          e.pre = jkey_pre; e.post = jkey_post; e.job = j; e.pad = 0;
          const bool rdy = ready + pbe >= minav;
          if (rdy && fp.ready_word == 1) e.pre |= 1ull << fp.ready_shift;
          if (rdy && fp.ready_word == 2) e.post |= 1ull << fp.ready_shift;
          e.share = fp.share_on ? (unsigned long long)__double_as_longlong(jshare) : 0ull;
          int i = q_hsize;
          while (i > 0) {
            int par = (i - 1) / 2;
            const HeapKey hp = h[par];
            if (!hk_less(e, hp)) break;
            h[i] = hp;
            i = par;
          }
          h[i] = e;
        }
        q_hsize += 1;
      }
      // ---- write the job / queue / role records back into the replica ----
      __syncwarp();
      // hdrf: drf.totalAllocated follows the visit's events (integer-valued: exact in any order)
      if (p.hd_on && lane < R) hd_tot_add(p.hd, lcta, lane, jalloc_l - jdyn[j].alloc[lane]);
      __syncwarp();
      if (lane == 0) {
        JobDyn *jd = &jdyn[j];
        jd->ready = ready; jd->waiting = waiting; jd->cursor = cursor - task_off; jd->share = jshare;
        QueueDyn *qd = &qdyn[q];
        qd->alloc_has = qalloc_has; qd->flags2 = qflags2; qd->active = 1;  // queues.Push(queue), allocate.go:346
        qd->scursor = q_scursor; qd->hsize = q_hsize; qd->share = qshare;
        if (q_mirror) { F.q_active[q] = 1; F.q_share[q] = qshare; }
      }
      if (lane < R) { jdyn[j].alloc[lane] = jalloc_l; qdyn[q].alloc[lane] = qalloc_l; }
      for (int r = lane; r < nroles; r += 32) {
        RoleDyn rd;
        rd.occ = S.r_occ[r]; rd.pip = S.r_pip[r]; rd.pending = S.r_pending[r]; rd.failed = S.r_failed[r];
        rdyn[role_base + r] = rd;
      }
      __syncwarp();
      if (p.hd_on) {  // queues.Push(queue) on the heap, after the tree caught up with the visit
        int nn = 0;
        if (lane == 0) nn = hd_push(p.hd, lcta, hd_n, j, q);
        hd_n = __shfl_sync(0xffffffffu, nn, 0);
      }
      FPROF_MARK(0);
    }
    if (pub_pending && pub_owner == cta) asm volatile("bar.sync 1, 64;" ::: "memory");  // pair the evaluator's last arrive
    if (lane == 0) {
      S.cmd = CMD_EXIT;
      S.n_dec = n_dec; S.n_vis = n_vis; S.n_fit = n_fit; S.n_steps = n_steps; S.n_full = n_full; S.n_incr = n_incr;
      S.last_idx = s_start;
      S.pick2 = n_owner_change;
      if (PROF) {
      atomicAdd((unsigned long long *)&p.prof[8], (unsigned long long)acc_post_to_joinstart);
      atomicAdd((unsigned long long *)&p.prof[9], (unsigned long long)acc_n);
      atomicAdd((unsigned long long *)&p.prof[10], (unsigned long long)acc_join_wait);
      atomicAdd((unsigned long long *)&p.prof[11], (unsigned long long)acc_join_to_post);
      atomicAdd((unsigned long long *)&p.prof[12], (unsigned long long)acc_ja);
      atomicAdd((unsigned long long *)&p.prof[13], (unsigned long long)acc_ab);
      atomicAdd((unsigned long long *)&p.prof[14], (unsigned long long)acc_bc);
      atomicAdd((unsigned long long *)&p.prof[15], (unsigned long long)acc_cp);
      if (out_cta) { p.counters[16] = F.vt_n[0]; p.counters[17] = F.vt_n[1]; }
      atomicAdd(&p.counters[18], vt_rows); atomicAdd(&p.counters[19], vt_fallback);
      }

    }
    __syncthreads();  // B1 of the exit command
  }

  // ---- epilogue: node state back to HBM, counters ----
  __syncthreads();
  for (int i = tid; i < nmine; i += blockDim.x) {
    const int n = nbase + i;
    for (int d = 0; d < R; ++d) {
      p.idle[(size_t)d * N + n] = fs.idle[d * cap + i];
      p.used[(size_t)d * N + n] = fs.used[d * cap + i];
      if (FUT) p.pip[(size_t)d * N + n] = fs.pip[d * cap + i];
    }
    for (int k = 0; k < K; ++k) p.kreq[(size_t)k * N + n] = fs.kreq[k * cap + i];
    for (int k = 0; k < 2; ++k) p.knz[(size_t)k * N + n] = fs.knz[k * cap + i];
    p.pod_count[n] = fs.pod_count[i];
  }
  if (cta == 0 && tid == 0) {
    p.counters[0] = S.n_dec;
    p.counters[1] = S.n_vis;
    p.counters[2] = S.n_fit;
    p.counters[3] = S.n_steps;
    if (SAMP) p.counters[4] = S.last_idx;
    p.counters[5] = S.n_full;
    p.counters[6] = S.n_incr;
    p.counters[7] = S.pick2;
    for (int k = 0; k < 8; ++k) p.prof[k] = S.prof[k];
  }
}
#undef VT
#undef VT_AT
#undef VT_GSTAMP

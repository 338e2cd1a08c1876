// vc_backfill.cuh — the backfill action (actions/backfill/backfill.go:58-116) as one persistent cooperative launch.
//
// The host has already fixed the visiting order (pickUpPendingTasks :118-199 evaluates its three order functions once,
// before the first placement), so the device loop is flat: for every BestEffort task in pick order
//   * every thread evaluates the plugin predicates of its node (ssn.PredicateForAllocateAction without allocate's
//     resource-fit wrapper, :66,83) and, when feasible, the node's util.PrioritizeNodes total;
//   * one mailbox all-gather (the commit kernel's `exchange`) gives every CTA the same arg-max
//     (util.SelectBestNodeAndScore, canonical tie-break) and the feasible-node count (one candidate: no scoring, :89-90);
//   * the owner thread applies Session.Allocate (framework/session.go:746-796): node.AddTask (Idle may go negative,
//     api/node_info.go:467-471) and the predicates plugin's AllocateFunc (pod count, k8s requested sums).
// The node axis is partitioned exactly as in k_commit (same CTA count, same shared-memory node slices, read from and
// written back to the working copies the allocate action left in HBM). A per-node verdict cache keyed by the task's
// (class, request) group makes a sweep re-evaluate only the node the previous placement touched.
// While consecutive tasks share their (class, request) group, only the CTA that received the previous placement can have
// a different local best: every CTA keeps the table of all CTAs' last records, the previous owner alone re-sweeps and
// publishes one record through a small ring, the others poll that one slot and fold the table (the full all-gather
// runs on a group switch and every 24 publications, which also bounds the ring).
// Bound: latency (one L2 round trip per task), like k_commit.
#pragma once
#include "vc_commit.cuh"

#define BF_REPL 8  // copies of a single-CTA publication (one 256-byte line each)

struct BackfillParams {
  int n;                  // tasks in pick order
  int B;                  // stride of the task arrays
  const int32_t *order;   // [n] index into the backfill task list
  const double *req;      // [R][B] Resreq (pods:1 only, but kept general)
  const double *kreq;     // [K][B]
  const double *knz;      // [2][B]
  const uint32_t *has;    // [B]
  const int32_t *klass;   // [B]
  const int32_t *group;   // [B] (class, request) group of the task
  int32_t *out_node;      // [n] chosen node per pick position, -1 = no feasible node
  double *out_score;      // [n] its util.PrioritizeNodes total (0.0 when it was the only candidate)
  const double *nta_static;  // [N] network-topology-aware entry of a pod WITHOUT a network topology whose request touches
                             // no weighted hypernode-binpack resource (every hypernode scores 0, a tier without a
                             // hypernode FullScore): state-independent; NULL when the plugin's map is empty
  int spec_depth;         // run-ahead depth: 32 when every quantity involved is integer-valued (row - m * request is then
                          // exactly what m successive placements leave), else 1
  int last_idx0;          // util.lastProcessedNodeIndex when the action starts (feasible-node sampling)
  int32_t *out_last_idx;  // [1] ... and when it ends
  long long *prof;        // [10] phase cycles of CTA 0 or NULL: sweep in gather steps, #gather steps, sweep as the republishing
                          // CTA, #such steps, mailbox all-gather, single-slot poll, fold + publish as republisher, apply + barriers
};

struct BfCtl {
  TaskRec trec2[3];  // ring of three: the record of task pos+2 is fetched while task pos waits in the mailbox, so that
  int group2[3];     // neither the sweep nor the run-ahead (which reads record pos+1) ever waits for a global load
  int cnt, best_node, max_soft;
  double best_score;
  unsigned seq;
  double w_score[32];
  int w_node[32], w_cnt[32], w_soft[32];
  // single-publisher steps: group the CTA table describes, CTA whose row changed in the previous step (-1 none),
  // publications since the last all-gather / so far
  int tb_group, prev_owner, since_sync;
  unsigned pc;
  // run-ahead: verdict of this CTA's best node for the NEXT task, assuming the current task lands on it
  // ... and for up to 32 further placements of the same group on it (lane m-1 evaluates the row after m pods):
  // entry spec_k is the next unused one
  int spec_node, spec_group, spec_pgroup, spec_k;
  int spec_flag[32];
  double spec_order[32];
  // feasible-node sampling (same scheme as k_commit<.,.,.,SAMP>)
  int last_idx, samp_proc, samp_total, samp_prefA, samp_prefB;
  unsigned seq2;
  int samp_w[4][8][2];
};

// A node's row as it will look once task `t` has been added to it (Session.Allocate + the predicates plugin's
// AllocateFunc): the same IEEE operations the owner thread applies, evaluated on the fly.
struct SpecNodeView {
  const SmemNodes &s;
  int i;
  const TaskRec &t;
  bool k8s;  // predicates plugin registered: k8s requested sums move too
  double m;  // pods added (1.0: bit-identical to one application for any input; > 1 only with integer-valued quantities)
  __device__ __forceinline__ double alloc(int d) const { return s.alloc[d * s.cap + i]; }
  __device__ __forceinline__ double idle(int d) const { return s.idle[d * s.cap + i] - m * t.req[d]; }
  __device__ __forceinline__ double used(int d) const { return s.used[d * s.cap + i] + m * t.req[d]; }
  __device__ __forceinline__ double rel(int) const { return 0.0; }
  __device__ __forceinline__ double pip(int) const { return 0.0; }
  __device__ __forceinline__ double kalloc(int k) const { return s.kalloc[k * s.cap + i]; }
  __device__ __forceinline__ double kreq(int k) const { return k8s ? s.kreq[k * s.cap + i] + m * t.kreq[k] : s.kreq[k * s.cap + i]; }
  __device__ __forceinline__ double knz(int k) const { return k8s ? s.knz[k * s.cap + i] + m * t.knz[k] : s.knz[k * s.cap + i]; }
};

// Warp arg-max of (score, node) with the canonical tie-break plus the candidate count, for the one-category record of
// the plain instance: four hardware reductions instead of the eight of local_warp_reduce (no soft-taint maximum, no
// topology pair, no sampling position). Every warp-wide collective adds its latency here, and three reductions sit on the
// per-task critical path.
__device__ __forceinline__ void simple_warp_reduce(Local &l) {
  constexpr unsigned FULLM = 0xffffffffu;
  const bool valid = l.node[0] >= 0;
  const unsigned long long key = valid ? score_key(l.score[0]) : 0ull;
  const unsigned hi = (unsigned)(key >> 32);
  const unsigned mhi = __reduce_max_sync(FULLM, hi);
  const unsigned lo = hi == mhi ? (unsigned)key : 0u;
  const unsigned mlo = __reduce_max_sync(FULLM, lo);
  const unsigned long long mkey = ((unsigned long long)mhi << 32) | mlo;
  const unsigned mnode = __reduce_min_sync(FULLM, (valid && key == mkey) ? (unsigned)l.node[0] : 0xffffffffu);
  if (mnode == 0xffffffffu) { l.node[0] = -1; l.score[0] = 0.0; }
  else { l.node[0] = (int)mnode; l.score[0] = score_of_key(mkey); }
  l.cnt[0] = (int)__reduce_add_sync(FULLM, (unsigned)l.cnt[0]);
}

// SOFT: the full (four-unit) mailbox record: needed when nodeorder's TaintToleration batch score is live (normalised
//       over the candidate set: two passes per task) and by SAMP
// SAMP: feasible-node sampling (util/predicate_helper.go:43-140 in its single-worker reading; a fresh PredicateHelper
//       per task, backfill.go:71, so there is no error cache): the candidates are the first `to_find` feasible nodes in
//       index order from lastProcessedNodeIndex, which then advances past the last node the scan looked at
template <bool SOFT, bool SAMP = false>
__global__ void __launch_bounds__(256, 1) k_backfill(K2Params p, BackfillParams b) {
  static_assert(!SAMP || SOFT, "the sampling variant rides on the full exchange");
  const DevConf &c = p.c;
  const int R = p.d.R, K = p.d.K, N = p.d.N;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int cta = blockIdx.x;
  const int nbase = p.d.node_begin + cta * p.npc;
  const int nmine = max(0, min(p.npc, p.d.node_end - nbase));
  const int cap = p.npc;

  unsigned char *sp = k2_smem;
  BfCtl &S = *reinterpret_cast<BfCtl *>(sp);
  sp += (sizeof(BfCtl) + 15) & ~(size_t)15;
  SmemNodes sn;
  sn.cap = cap;
  auto take = [&](int rows) { double *q = reinterpret_cast<double *>(sp); sp += (size_t)rows * cap * sizeof(double); return q; };
  sn.alloc = take(R); sn.idle = take(R); sn.used = take(R);
  sn.rel = nullptr; sn.pip = nullptr;  // FutureIdle plays no part: backfill has no resource-fit gradient
  sn.kalloc = take(K); sn.kreq = take(K); sn.knz = take(2);
  sn.nerr = nullptr;
  sn.max_tasks = reinterpret_cast<int32_t *>(sp); sp += (size_t)cap * 4;
  sn.pod_count = reinterpret_cast<int32_t *>(sp); sp += (size_t)cap * 4;
  sp = reinterpret_cast<unsigned char *>(((uintptr_t)sp + 7) & ~(uintptr_t)7);
  double *c_order = reinterpret_cast<double *>(sp); sp += (size_t)cap * 8;   // verdict cache: NodeOrderFn sum,
  int32_t *c_group = reinterpret_cast<int32_t *>(sp); sp += (size_t)cap * 4;  // the group it was computed for,
  uint8_t *c_flag = reinterpret_cast<uint8_t *>(sp); sp += (size_t)cap;       // bit0 feasible, bit1 has order score
  uint8_t *s_samp = reinterpret_cast<uint8_t *>(sp); sp += (size_t)cap;       // sampling: 1 = candidate
  sp = reinterpret_cast<unsigned char *>(((uintptr_t)sp + 7) & ~(uintptr_t)7);
  double *tb_score = reinterpret_cast<double *>(sp); sp += (size_t)p.n_cta * 8;  // last record of every CTA for tb_group
  int *tb_node = reinterpret_cast<int *>(sp); sp += (size_t)p.n_cta * 4;
  int *tb_cnt = reinterpret_cast<int *>(sp);

  for (int i = tid; i < nmine; i += blockDim.x) {
    const int n = nbase + i;
    for (int d = 0; d < R; ++d) {
      sn.alloc[d * cap + i] = p.alloc[(size_t)d * N + n];
      sn.idle[d * cap + i] = p.idle[(size_t)d * N + n];
      sn.used[d * cap + i] = p.used[(size_t)d * N + n];
    }
    for (int k = 0; k < K; ++k) {
      sn.kalloc[k * cap + i] = p.kalloc[(size_t)k * N + n];
      sn.kreq[k * cap + i] = p.kreq[(size_t)k * N + n];
    }
    for (int k = 0; k < 2; ++k) sn.knz[k * cap + i] = p.knz[(size_t)k * N + n];
    sn.max_tasks[i] = p.max_tasks[n];
    sn.pod_count[i] = p.pod_count[n];
  }
  for (int i = tid; i < cap; i += blockDim.x) c_group[i] = -1;
  if (tid == 0) { S.seq = 0; S.seq2 = 0; S.last_idx = b.last_idx0; S.spec_node = -1; S.tb_group = -1; S.prev_owner = -1; S.since_sync = 0; S.pc = 0; }
  __syncthreads();

  const bool two_pass = SOFT && c.soft_active;
  // stage the record of pick position `pos` into buffer pos & 1 (the last warp: it has the fewest nodes to sweep)
  auto stage = [&](int pos) {
    if (pos >= b.n || warp != nwarps - 1) return;
    const int t = b.order[pos];
    TaskRec &r = S.trec2[pos % 3];
    if (lane < R) r.req[lane] = b.req[(size_t)lane * b.B + t];
    if (lane < K) r.kreq[lane] = b.kreq[(size_t)lane * b.B + t];
    if (lane < 2) r.knz[lane] = b.knz[(size_t)lane * b.B + t];
    if (lane == 31) {
      r.has = b.has[t];
      r.klass = b.klass[t];
      S.group2[pos % 3] = b.group[t];
    }
  };
  stage(0);
  stage(1);
  long long pf[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0}, pf_last = clock64();
  const bool profiling = b.prof != nullptr && cta == 0 && tid == 0;
#define BF_MARK(k) do { if (profiling) { const long long now_ = clock64(); pf[k] += now_ - pf_last; pf_last = now_; } } while (0)
  for (int pos = 0; pos < b.n; ++pos) {
    __syncthreads();  // records `pos`, `pos + 1` staged; the owner thread is done with record pos - 1
    BF_MARK(7);
    const long long t_top = profiling ? clock64() : 0;
    const TaskRec &trec = S.trec2[pos % 3];
    const int group = S.group2[pos % 3];
    const uint32_t *cs_row = p.cstat + (size_t)trec.klass * N + nbase;
    int g_soft = 0;
    // cached or fresh (feasible, NodeOrderFn sum) of node i for the staged group
    auto verdict = [&](int i, uint32_t cs, bool *ok, bool *has_order, double *order) {
      if (c_group[i] == group) {
        *ok = (c_flag[i] & 1) != 0; *has_order = (c_flag[i] & 2) != 0; *order = c_order[i];
        return;
      }
      SmemNodeView nv{sn, i};
      *ok = (cs & CS_STATIC_OK) != 0;
      if (c.pred_predicates && sn.max_tasks[i] <= sn.pod_count[i]) *ok = false;  // predicates.go:662-671
      *has_order = false;
      *order = 0.0;
      if (*ok) *has_order = node_order(c, R, K, trec, nv, cs, order);
      c_group[i] = group; c_flag[i] = (uint8_t)((*ok ? 1 : 0) | (*has_order ? 2 : 0)); c_order[i] = *order;
    };
    const bool sampling = SAMP && c.to_find > 0;
    // single-publisher step? (uniform over the grid: it only depends on replicated state)
    const bool tracked = !SOFT && !SAMP;
    const bool full = !tracked || S.tb_group != group || S.since_sync >= 24;
    const bool sweeping = full || cta == S.prev_owner;
    if (SAMP && sampling) {
      const int start = S.last_idx, Kf = c.to_find;
      const int rows = (cap + (int)blockDim.x - 1) / (int)blockDim.x;
      const unsigned lt = (1u << lane) - 1u;
      for (int row = 0; row < rows; ++row) {
        const int i = row * blockDim.x + tid;
        int flag = 0;
        if (i < nmine) {
          bool ok, ho; double od;
          verdict(i, c_group[i] != group ? cs_row[i] : 0u, &ok, &ho, &od);
          flag = ok ? 1 : 2;
          s_samp[i] = (uint8_t)flag;
        }
        const bool inA = nbase + i >= start;
        const unsigned mA = __ballot_sync(0xffffffffu, flag == 1 && inA), mB = __ballot_sync(0xffffffffu, flag == 1 && !inA);
        if (lane == 0) { S.samp_w[row][warp][0] = __popc(mA); S.samp_w[row][warp][1] = __popc(mB); }
      }
      __syncthreads();
      if (warp == 0) {
        int a = 0, bb = 0;
        for (int e = lane; e < rows * nwarps; e += 32) { a += S.samp_w[e / nwarps][e % nwarps][0]; bb += S.samp_w[e / nwarps][e % nwarps][1]; }
        a = (int)__reduce_add_sync(0xffffffffu, (unsigned)a);
        bb = (int)__reduce_add_sync(0xffffffffu, (unsigned)bb);
        const unsigned seq2 = S.seq2 + 1;
        __syncwarp();
        const CountFold f = exchange_counts(p, a, bb, seq2);
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
        if (i >= nmine || flag != 1) continue;
        const int seg = inA ? 0 : 1;
        int before = (inA ? S.samp_prefA : S.samp_prefB) + __popc((inA ? mA : mB) & lt);
        for (int r2 = 0; r2 <= row; ++r2)
          for (int w2 = 0; w2 < (r2 < row ? nwarps : warp); ++w2) before += S.samp_w[r2][w2][seg];
        s_samp[i] = before < Kf ? 1 : 0;
        if (before == Kf - 1) S.samp_proc = (nbase + i - start + N) % N + 1;  // the scan stops here
      }
      __syncthreads();
    }
    for (int pass = 0; pass < (two_pass ? 2 : 1); ++pass) {
      Local mine;
      local_init(mine);
      for (int i = tid; sweeping && i < nmine; i += blockDim.x) {
        const uint32_t cs = (two_pass || c_group[i] != group) ? cs_row[i] : 0u;
        if (SAMP && sampling && s_samp[i] != 1) continue;  // outside the sampled candidate set
        bool ok, has_order;
        double order;
        verdict(i, cs, &ok, &has_order, &order);
        if (!ok) continue;
        const int soft = SOFT ? (int)((cs >> CS_SOFT_SHIFT) & 0xff) : 0;
        mine.cnt[0] += 1;
        mine.soft[0] = max(mine.soft[0], soft);
        if (two_pass && pass == 0) continue;
        const int n = nbase + i;
        // pods of a soft-mode topology job carry task.JobAllocatedHyperNode == "" here (only allocate.go:659 sets it):
        // batchNodeOrderFnForNetworkAwarePods returns no entries (:544-547)
        const double nta = (b.nta_static && !(trec.has & VC_HAS_TOPO_TASK)) ? b.nta_static[n] : 0.0;
        const double sc = total_score(c, has_order, order, soft, g_soft, nta);
        if (mine.node[0] < 0 || better(sc, n, mine.score[0], mine.node[0])) { mine.score[0] = sc; mine.node[0] = n; }
      }
      if (sweeping) {
        if (SOFT) local_warp_reduce<false>(mine); else simple_warp_reduce(mine);
        if (lane == 0) { S.w_score[warp] = mine.score[0]; S.w_node[warp] = mine.node[0]; S.w_cnt[warp] = mine.cnt[0]; S.w_soft[warp] = mine.soft[0]; }
      }
      if (profiling && sweeping) { pf[full ? 1 : 3] += 1; }
      BF_MARK(full ? 0 : (sweeping ? 2 : 7));
      __syncthreads();
      if (pass == 0) stage(pos + 2);  // into the buffer of pos - 1, while the mailbox is being waited on
      if (warp == 1 && !two_pass && !(SAMP && sampling)) {
        // run-ahead while warp 0 sits in the mailbox: if this CTA's best node wins, the next sweep would have to
        // re-evaluate exactly that node before anybody can publish - do it now, against the row as it will be
        Local l;
        local_init(l);
        bool go = true;
        if (sweeping) {
          if (lane < nwarps) { l.score[0] = S.w_score[lane]; l.node[0] = S.w_node[lane]; }
          if (SOFT) local_warp_reduce<false>(l); else simple_warp_reduce(l);
        } else {
          l.node[0] = tb_node[cta];  // unchanged since this CTA last published
          l.score[0] = tb_score[cta];
        }
        // The verdict depends on (node row, group of the pod added, group evaluated), not on the task index: once
        // computed for the CTA's best node it stays valid until that node changes, i.e. until this CTA wins - so a CTA
        // pays for it once, long before its turn, and the winner's next sweep is cache hits only.
        const int group_next = pos + 1 < b.n ? S.group2[(pos + 1) % 3] : -1;
        const int depth = b.spec_depth;
        go = group_next == group &&
             !(S.spec_node == l.node[0] && S.spec_pgroup == group && S.spec_group == group_next && S.spec_k < depth);
        if (go) {
          if (l.node[0] >= 0) {
            const int i = l.node[0] - nbase;
            const TaskRec &nt = S.trec2[(pos + 1) % 3];
            const uint32_t cs = p.cstat[(size_t)nt.klass * N + nbase + i];
            if (lane < depth) {
              SpecNodeView nv{sn, i, trec, c.has_predicates != 0, (double)(lane + 1)};
              bool ok = (cs & CS_STATIC_OK) != 0;
              if (c.pred_predicates && sn.max_tasks[i] <= sn.pod_count[i] + (c.has_predicates ? lane + 1 : 0)) ok = false;
              bool ho = false;
              double od = 0.0;
              if (ok) ho = node_order(c, R, K, nt, nv, cs, &od);
              S.spec_flag[lane] = (ok ? 1 : 0) | (ho ? 2 : 0);
              S.spec_order[lane] = od;
            }
            __syncwarp();
            if (lane == 0) { S.spec_group = group_next; S.spec_pgroup = group; S.spec_k = 0; S.spec_node = l.node[0]; }
          } else if (lane == 0) {
            S.spec_node = -1;
          }
        }
      }
      if (warp == 0) {
        Local l;
        local_init(l);
        if (sweeping) {
          if (lane < nwarps) { l.score[0] = S.w_score[lane]; l.node[0] = S.w_node[lane]; l.cnt[0] = S.w_cnt[lane]; l.soft[0] = S.w_soft[lane]; }
          if (SOFT) local_warp_reduce<false>(l); else simple_warp_reduce(l);
        }
        if (SAMP && sampling) l.proc = S.samp_proc;
        const unsigned seq = S.seq + 1;
        const unsigned pc = S.pc;
        const int prev_owner = S.prev_owner;
        __syncwarp();  // every lane has read S.seq / S.pc before lane 0 advances them
        Local g;
        if (full) {
          g = tracked ? exchange<SOFT>(p, l, seq, tb_score, tb_node, tb_cnt) : exchange<SOFT>(p, l, seq);
        } else {
          if (prev_owner >= 0) {  // one row changed since the table was current: its owner publishes, the others read
            // BF_REPL copies of the record in different lines: a single line polled by every CTA is a hot spot that
            // holds the publishing store back
            uint4 *slot = p.mbox2 + (size_t)(pc & 63u) * BF_REPL * MBOX_STRIDE;
            const unsigned tag = pc + 1;
            if (cta == prev_owner) {
              if (lane < BF_REPL) {
                const unsigned long long sb = (unsigned long long)__double_as_longlong(l.score[0]);
                mbox_store(slot + (size_t)lane * MBOX_STRIDE,
                           make_uint4((unsigned)sb, (unsigned)(sb >> 32), (unsigned)l.node[0], (tag << 2) | (unsigned)min(l.cnt[0], 2)));
              }
              if (lane == 0) { tb_score[cta] = l.score[0]; tb_node[cta] = l.node[0]; tb_cnt[cta] = min(l.cnt[0], 2); }
              if (profiling) pf[9] += clock64() - t_top;  // top barrier -> record on its way
            } else if (lane == 0) {
              uint4 v;
              const uint4 *mine_slot = slot + (size_t)(cta % BF_REPL) * MBOX_STRIDE;
              do { v = mbox_load(mine_slot); } while ((v.w >> 2) != (tag & 0x3fffffffu));
              if (profiling) pf[8] += clock64() - t_top;  // top barrier -> record seen
              tb_score[prev_owner] = __longlong_as_double((long long)((unsigned long long)v.x | ((unsigned long long)v.y << 32)));
              tb_node[prev_owner] = (int)v.z;
              tb_cnt[prev_owner] = (int)(v.w & 3u);
            }
            __syncwarp();
          }
          local_init(g);
          for (int k = lane; k < p.n_cta; k += 32) {
            Local o;
            local_init(o);
            o.score[0] = tb_score[k]; o.node[0] = tb_node[k]; o.cnt[0] = tb_cnt[k];
            local_fold(g, o);
          }
          simple_warp_reduce(g);
          g.cnt[0] = min(g.cnt[0], 2);
        }
        if (lane == 0) {
          if (full) S.seq = seq;
          if (tracked) {
            S.tb_group = group;
            if (full) S.since_sync = 0;
            else if (prev_owner >= 0) { S.since_sync += 1; S.pc = pc + 1; }
            S.prev_owner = g.cnt[0] > 0 ? (g.node[0] - p.d.node_begin) / p.npc : -1;
          }
          S.cnt = g.cnt[0]; S.best_node = g.node[0]; S.best_score = g.score[0]; S.max_soft = g.soft[0];
          if (SAMP && sampling && pass == (two_pass ? 1 : 0)) {  // lastProcessedNodeIndex = (start + processedNodes) % N
            const int processed = S.samp_total >= c.to_find ? g.proc : N;
            S.last_idx = (S.last_idx + processed) % N;
          }
        }
      }
      __syncthreads();
      BF_MARK(full ? 4 : (sweeping ? 6 : 5));
      g_soft = S.max_soft;
      if (S.cnt == 0) break;
    }
    const int cnt = S.cnt, best = S.best_node;
    const double score = cnt == 1 ? 0.0 : S.best_score;
    if (cta == 0 && tid == 0) {
      b.out_node[pos] = cnt == 0 ? -1 : best;
      b.out_score[pos] = cnt == 0 ? 0.0 : score;
    }
    if (cnt == 0) continue;  // job.NodesFitErrors[task.UID] = fitErrors, :84-87
    if (best >= nbase && best < nbase + nmine) {
      const int i = best - nbase;
      if ((i % blockDim.x) == tid) {
        if (nwarps > 1 && !two_pass && !(SAMP && sampling) && S.spec_node == best && S.spec_pgroup == group &&
            S.spec_k < b.spec_depth) {  // the run-ahead verdict of this row after one more pod of this group
          const int k = S.spec_k;
          c_group[i] = S.spec_group; c_flag[i] = (uint8_t)S.spec_flag[k]; c_order[i] = S.spec_order[k];
          S.spec_k = k + 1;
        } else {
          c_group[i] = -1;
          S.spec_node = -1;  // the row changes in a way the run-ahead did not assume
        }
        for (int d = 0; d < R; ++d) {
          sn.idle[d * cap + i] -= trec.req[d];
          sn.used[d * cap + i] += trec.req[d];
        }
        if (c.has_predicates) {  // predicates AllocateFunc, predicates.go:212-256
          sn.pod_count[i] += 1;
          for (int k = 0; k < K; ++k) sn.kreq[k * cap + i] += trec.kreq[k];
          for (int k = 0; k < 2; ++k) sn.knz[k * cap + i] += trec.knz[k];
        }
      }
    }
  }

  __syncthreads();
  for (int i = tid; i < nmine; i += blockDim.x) {
    const int n = nbase + i;
    for (int d = 0; d < R; ++d) {
      p.idle[(size_t)d * N + n] = sn.idle[d * cap + i];
      p.used[(size_t)d * N + n] = sn.used[d * cap + i];
    }
    for (int k = 0; k < K; ++k) p.kreq[(size_t)k * N + n] = sn.kreq[k * cap + i];
    for (int k = 0; k < 2; ++k) p.knz[(size_t)k * N + n] = sn.knz[k * cap + i];
    p.pod_count[n] = sn.pod_count[i];
  }
  if (cta == 0 && tid == 0) b.out_last_idx[0] = S.last_idx;
  if (profiling)
    for (int k = 0; k < 10; ++k) b.prof[k] = pf[k];
#undef BF_MARK
}

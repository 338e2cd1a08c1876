// vc_kernels.cuh — the CUDA kernels of libvcalloc.so (sm_90a).
//
//  k_class_static   K0  class x node static predicate / static score word (session open)
//  k_group_eval     K1a group x node dense evaluation on the opening snapshot
//  k_group_expand   K1b materialise the task x node mask + score matrix (HBM-write-bound)
//  k_commit         K2  persistent cooperative kernel: the exact sequential allocate loop
//
// See DESIGN.md for the data layout and the roofline of each kernel.
#pragma once
#include <cooperative_groups.h>

#include "vc_device.cuh"

namespace cg = cooperative_groups;

// =======================================================================================
// K0: class x node static word
// =======================================================================================
struct K0Params {
  DevDims d;
  DevConf c;
  const uint64_t *labels, *thard, *tsoft;  // [W][N]
  const uint32_t *nflags;
  const int32_t *zone;
  const uint8_t *zone_active;
  const uint64_t *c_sel, *c_aff, *c_tolh, *c_tols, *c_pref;
  const int32_t *c_naff, *c_npref, *c_prefw;
  const uint32_t *c_flags;
  uint32_t *cstat;  // [C][N]
};

__device__ __forceinline__ bool mask_subset(const uint64_t *need, const uint64_t *bits, int W, int N, int n) {
  bool ok = true;
  for (int w = 0; w < W; ++w) {
    uint64_t nd = need[w];
    if ((bits[(size_t)w * N + n] & nd) != nd) ok = false;
  }
  return ok;
}

// grid (ceil(N/256), C): one thread per (class, node); node words read coalesced, class rows broadcast.
__global__ void __launch_bounds__(256) k_class_static(K0Params p) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = blockIdx.y;
  const int N = p.d.N, Wl = p.d.Wl, Wt = p.d.Wt;
  if (n >= N) return;
  const uint32_t cf = p.c_flags[c];
  bool ok = true;
  // predicates plugin, static filters (plugins/predicates/predicates.go:673-693): NodeUnschedulable,
  // NodeAffinity (nodeSelector + required terms), TaintToleration (NoSchedule / NoExecute)
  bool pred_ok = true;
  if ((p.nflags[n] & VC_NODE_UNSCHEDULABLE) && !(cf & VC_CLASS_TOLERATES_UNSCHEDULABLE)) pred_ok = false;
  if (p.c.predicates_enable & VC_PRED_NODE_AFFINITY) {
    if (!mask_subset(p.c_sel + (size_t)c * Wl, p.labels, Wl, N, n)) pred_ok = false;
    int na = p.c_naff[c];
    if (na > 0) {
      bool any = false;
      for (int k = 0; k < na; ++k)
        if (mask_subset(p.c_aff + ((size_t)c * VC_MAX_TERMS + k) * Wl, p.labels, Wl, N, n)) any = true;
      if (!any) pred_ok = false;
    }
  }
  if (p.c.predicates_enable & VC_PRED_TAINT_TOLERATION) {
    for (int w = 0; w < Wt; ++w)
      if (p.thard[(size_t)w * N + n] & ~p.c_tolh[(size_t)c * Wt + w]) pred_ok = false;
  }
  // tdm predicateFn, plugins/tdm/tdm.go:146-171
  const int z = p.zone[n];
  bool tdm_ok = true;
  if (z >= 0) {
    if (!p.zone_active[z]) tdm_ok = false;
    else if (!(cf & VC_CLASS_REVOCABLE)) tdm_ok = false;
  }
  for (int i = 0; i < p.c.n_plugins; ++i) {
    if (!(p.c.enabled[i] & VC_EN_PREDICATE)) continue;
    if (p.c.plugin[i] == VC_PLUGIN_PREDICATES && !pred_ok) ok = false;
    if (p.c.plugin[i] == VC_PLUGIN_TDM && !tdm_ok) ok = false;
  }
  uint32_t word = ok ? CS_STATIC_OK : 0u;
  if (z >= 0) {  // tdm nodeOrderFn, tdm.go:174-195
    if (!p.zone_active[z]) word |= CS_TDM_ORDER_ERR;
    else if (cf & VC_CLASS_REVOCABLE) word |= CS_TDM_ORDER_MAX;
  }
  int soft = 0;
  for (int w = 0; w < Wt; ++w) soft += __popcll(p.tsoft[(size_t)w * N + n] & ~p.c_tols[(size_t)c * Wt + w]);
  if (soft > 255) soft = 255;
  word |= (uint32_t)soft << CS_SOFT_SHIFT;
  int naff = 0;
  for (int k = 0; k < p.c_npref[c]; ++k)
    if (mask_subset(p.c_pref + ((size_t)c * VC_MAX_TERMS + k) * Wl, p.labels, Wl, N, n))
      naff += p.c_prefw[(size_t)c * VC_MAX_TERMS + k];
  if (naff < 0) naff = 0;
  if (naff > 65535) naff = 65535;
  word |= (uint32_t)naff << CS_NAFF_SHIFT;
  p.cstat[(size_t)c * N + n] = word;
}

// =======================================================================================
// K1: dense pass on the opening snapshot
// =======================================================================================
struct GlobalNodeView {  // node columns straight from the SoA in HBM/L2
  const double *alloc_, *idle_, *used_, *rel_, *pip_, *kalloc_, *kreq_, *knz_;
  int N, n;
  __device__ __forceinline__ double alloc(int d) const { return alloc_[(size_t)d * N + n]; }
  __device__ __forceinline__ double idle(int d) const { return idle_[(size_t)d * N + n]; }
  __device__ __forceinline__ double used(int d) const { return used_[(size_t)d * N + n]; }
  __device__ __forceinline__ double rel(int d) const { return rel_[(size_t)d * N + n]; }
  __device__ __forceinline__ double pip(int d) const { return pip_[(size_t)d * N + n]; }
  __device__ __forceinline__ double kalloc(int k) const { return kalloc_[(size_t)k * N + n]; }
  __device__ __forceinline__ double kreq(int k) const { return kreq_[(size_t)k * N + n]; }
  __device__ __forceinline__ double knz(int k) const { return knz_[(size_t)k * N + n]; }
};

struct K1Params {
  DevDims d;
  DevConf c;
  int y_off;  // added to blockIdx.y: launches over more than 65535 groups / work items go out in slices
  const double *alloc, *idle, *used, *rel, *pip, *kalloc, *kreq, *knz;
  const int32_t *max_tasks, *pod_count;
  const uint32_t *cstat;
  // groups = distinct (class, request) records among the tasks
  int n_groups;
  const double *g_req;   // [R][G]
  const double *g_kreq;  // [K][G]
  const double *g_knz;   // [2][G]
  const uint32_t *g_has;
  const int32_t *g_class;
  // scratch [G][Nloc]
  double *g_order;       // order score (valid when cat != 2)
  uint8_t *g_cat;        // 0 idle-fit, 1 future-fit only, 2 infeasible; bit 7 = no order score (NodeOrderFn error)
  int32_t *g_stats;      // [G][4]: any0, any1, maxsoft0, maxsoft1 (atomics)
  unsigned long long *g_best;  // [G][2] packed (orderable score, ~node) per category -> atomicMax ... see below
  double *g_best_score;  // [G]
  int32_t *g_best_node;  // [G]
  // expansion
  int n_work;
  const int32_t *work_group, *work_begin, *work_end;  // task-list ranges per work item
  const int32_t *group_tasks;                         // task ids sorted by group
  uint32_t *mask_out;   // [T][2*mw] 32-bit halves of the uint64 mask rows
  double *score_out;    // [T][N]
  double *best_score;   // [T]
  int32_t *best_node;   // [T]
  int mw32;             // 32-bit words per mask row
  // network-topology-aware (hypernode binpacking of normal pods) on the opening snapshot
  int hn_H;
  const int32_t *hn_member;  // [L][N]
  const double *hn_alloc;    // [R][H]
  const double *hn_used;     // [R][H]
  double *hn_score;          // [G][H] getPodHyperNodeBinPackingScore(group, hypernode)
};

// K1h: grid (ceil(H/128), G). One thread per (group, hypernode).
__global__ void __launch_bounds__(128) k_hn_scores(K1Params p) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  const int g = blockIdx.y + p.y_off;
  if (h >= p.hn_H) return;
  TaskRec t;
  for (int d = 0; d < p.d.R; ++d) t.req[d] = p.g_req[(size_t)d * p.n_groups + g];
  t.has = p.g_has[g];
  const int H = p.hn_H;
  p.hn_score[(size_t)g * H + h] = hn_binpack_score(
      p.c, p.d.R, t, [&](int d) { return p.hn_used[(size_t)d * H + h]; }, [&](int d) { return p.hn_alloc[(size_t)d * H + h]; });
}

// K1a: grid (ceil(Nloc/256), G). One thread per (group, node): predicate, fit category, order score.
__global__ void __launch_bounds__(256) k_group_eval(K1Params p) {
  const int N = p.d.N;
  const int nloc = p.d.node_end - p.d.node_begin;
  const int li = blockIdx.x * blockDim.x + threadIdx.x;
  const int g = blockIdx.y + p.y_off;
  __shared__ TaskRec trec;
  if (threadIdx.x < p.d.R) trec.req[threadIdx.x] = p.g_req[(size_t)threadIdx.x * p.n_groups + g];
  if (threadIdx.x >= 32 && threadIdx.x < 32 + p.d.K) trec.kreq[threadIdx.x - 32] = p.g_kreq[(size_t)(threadIdx.x - 32) * p.n_groups + g];
  if (threadIdx.x >= 64 && threadIdx.x < 66) trec.knz[threadIdx.x - 64] = p.g_knz[(size_t)(threadIdx.x - 64) * p.n_groups + g];
  if (threadIdx.x == 96) { trec.has = p.g_has[g]; trec.klass = p.g_class[g]; }
  __syncthreads();
  int cat = 2, soft = 0;
  bool has_order = false;
  double order = 0.0;
  if (li < nloc) {
    const int n = p.d.node_begin + li;
    const uint32_t cs = p.cstat[(size_t)trec.klass * N + n];
    GlobalNodeView nv{p.alloc, p.idle, p.used, p.rel, p.pip, p.kalloc, p.kreq, p.knz, N, n};
    bool ok = (cs & CS_STATIC_OK) != 0;
    if (p.c.pred_predicates && p.max_tasks[n] <= p.pod_count[n]) ok = false;  // predicates.go:662-671
    int fc = fit_category(p.c, p.d.R, trec, nv);
    // allocate.predicate (allocate.go:816-824) requires the FutureIdle fit
    if (ok && fc != 2) {
      cat = fc;
      soft = (cs >> CS_SOFT_SHIFT) & 0xff;
      has_order = node_order(p.c, p.d.R, p.d.K, trec, nv, cs, &order);
    }
    p.g_order[(size_t)g * nloc + li] = order;
    p.g_cat[(size_t)g * nloc + li] = (uint8_t)(cat | (has_order ? 0 : 0x80));
  }
  // per-group reductions: does any idle-fit / future-fit node exist, max soft-taint count per category
  unsigned m0 = __ballot_sync(0xffffffffu, cat == 0), m1 = __ballot_sync(0xffffffffu, cat == 1);
  int s0 = cat == 0 ? soft : 0, s1 = cat == 1 ? soft : 0;
  for (int o = 16; o; o >>= 1) {
    s0 = max(s0, __shfl_xor_sync(0xffffffffu, s0, o));
    s1 = max(s1, __shfl_xor_sync(0xffffffffu, s1, o));
  }
  if ((threadIdx.x & 31) == 0) {
    if (m0) { atomicOr(&p.g_stats[g * 4 + 0], 1); if (s0) atomicMax(&p.g_stats[g * 4 + 2], s0); }
    if (m1) { atomicOr(&p.g_stats[g * 4 + 1], 1); if (s1) atomicMax(&p.g_stats[g * 4 + 3], s1); }
  }
}

// final score of (group g, local node li) given the group's chosen gradient; false -> not a candidate
__device__ __forceinline__ bool k1_final(const K1Params &p, int g, int li, int nloc, int chosen, int max_soft,
                                         int klassN_word_soft, double *score, bool *feasible) {
  uint8_t cw = p.g_cat[(size_t)g * nloc + li];
  int cat = cw & 3;
  *feasible = cat != 2;
  if (cat == 2 || cat != chosen) { *score = 0.0; return false; }
  double nta = 0.0;
  if (p.c.nta_on && !(p.g_has[g] & VC_HAS_TOPO_TASK)) {
    const int n = p.d.node_begin + li;
    nta = nta_node_score(p.c, [&](int l) {
      const int h = p.hn_member[(size_t)l * p.d.N + n];
      return h < 0 ? 1.0 : p.hn_score[(size_t)g * p.hn_H + h];
    });
  }
  *score = total_score(p.c, !(cw & 0x80), p.g_order[(size_t)g * nloc + li], klassN_word_soft, max_soft, nta);
  return true;
}

// K1a': per-group best (score, node) — grid (ceil(Nloc/256), G); block argmax then one atomic per block
// on a packed key is not possible for a 64-bit score + index, so blocks write partials and the last
// pass (k_group_best_final) folds them; Nloc/256 partials per group is tiny.
__global__ void __launch_bounds__(256) k_group_best_partial(K1Params p, double *part_score, int32_t *part_node) {
  const int N = p.d.N;
  const int nloc = p.d.node_end - p.d.node_begin;
  const int li = blockIdx.x * blockDim.x + threadIdx.x;
  const int g = blockIdx.y + p.y_off;
  const int chosen = p.g_stats[g * 4 + 0] ? 0 : (p.g_stats[g * 4 + 1] ? 1 : 2);
  const int max_soft = chosen == 0 ? p.g_stats[g * 4 + 2] : p.g_stats[g * 4 + 3];
  double bs = 0.0;
  int bn = -1;
  if (li < nloc && chosen != 2) {
    const int n = p.d.node_begin + li;
    int soft = (p.cstat[(size_t)p.g_class[g] * N + n] >> CS_SOFT_SHIFT) & 0xff;
    double sc;
    bool feas;
    if (k1_final(p, g, li, nloc, chosen, max_soft, soft, &sc, &feas)) { bs = sc; bn = n; }
  }
  for (int o = 16; o; o >>= 1) {
    double os = __shfl_xor_sync(0xffffffffu, bs, o);
    int on = __shfl_xor_sync(0xffffffffu, bn, o);
    if (on >= 0 && (bn < 0 || better(os, on, bs, bn))) { bs = os; bn = on; }
  }
  __shared__ double ws[8];
  __shared__ int wn[8];
  if ((threadIdx.x & 31) == 0) { ws[threadIdx.x >> 5] = bs; wn[threadIdx.x >> 5] = bn; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w)
      if (wn[w] >= 0 && (bn < 0 || better(ws[w], wn[w], bs, bn))) { bs = ws[w]; bn = wn[w]; }
    part_score[(size_t)g * gridDim.x + blockIdx.x] = bs;
    part_node[(size_t)g * gridDim.x + blockIdx.x] = bn;
  }
}
__global__ void k_group_best_final(K1Params p, const double *part_score, const int32_t *part_node, int nparts) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= p.n_groups) return;
  double bs = 0.0;
  int bn = -1;
  for (int i = 0; i < nparts; ++i) {
    int on = part_node[(size_t)g * nparts + i];
    double os = part_score[(size_t)g * nparts + i];
    if (on >= 0 && (bn < 0 || better(os, on, bs, bn))) { bs = os; bn = on; }
  }
  p.g_best_score[g] = bn >= 0 ? bs : 0.0;
  p.g_best_node[g] = bn;
}

// K1b: materialise. grid (ceil(Nloc/512), n_work); 256 threads, two adjacent nodes per thread so every
// warp store is one 512-byte coalesced, 16-byte-vectorised row segment; rows of the same group reuse the
// tile kept in registers. Streaming stores (st.global.cs): the matrix is written once and never re-read.
__global__ void __launch_bounds__(256) k_group_expand(K1Params p) {
  const int N = p.d.N;
  const int nloc = p.d.node_end - p.d.node_begin;
  const int w = blockIdx.y + p.y_off;
  const int g = p.work_group[w];
  const int chosen = p.g_stats[g * 4 + 0] ? 0 : (p.g_stats[g * 4 + 1] ? 1 : 2);
  const int max_soft = chosen == 0 ? p.g_stats[g * 4 + 2] : p.g_stats[g * 4 + 3];
  const int li0 = (blockIdx.x * blockDim.x + threadIdx.x) * 2;
  double s0 = 0.0, s1 = 0.0;
  bool f0 = false, f1 = false;
  const int klass = p.g_class[g];
  if (li0 < nloc) {
    int soft = (p.cstat[(size_t)klass * N + p.d.node_begin + li0] >> CS_SOFT_SHIFT) & 0xff;
    k1_final(p, g, li0, nloc, chosen, max_soft, soft, &s0, &f0);
  }
  if (li0 + 1 < nloc) {
    int soft = (p.cstat[(size_t)klass * N + p.d.node_begin + li0 + 1] >> CS_SOFT_SHIFT) & 0xff;
    k1_final(p, g, li0 + 1, nloc, chosen, max_soft, soft, &s1, &f1);
  }
  // mask bits of this warp: 64 nodes -> one uint64 word per row (two 32-bit halves)
  const unsigned b0 = __ballot_sync(0xffffffffu, f0), b1 = __ballot_sync(0xffffffffu, f1);
  // interleave: node li0 (even) and li0+1 (odd) -> bit positions 2*lane, 2*lane+1
  unsigned lo = 0, hi = 0;
  {
    const int lane = threadIdx.x & 31;
    // each lane builds one of the two 32-bit halves cooperatively: lanes 0..15 cover bits 0..31
    unsigned mylo = 0, myhi = 0;
    for (int l = 0; l < 16; ++l) {
      mylo |= ((b0 >> l) & 1u) << (2 * l);
      mylo |= ((b1 >> l) & 1u) << (2 * l + 1);
      myhi |= ((b0 >> (l + 16)) & 1u) << (2 * l);
      myhi |= ((b1 >> (l + 16)) & 1u) << (2 * l + 1);
    }
    lo = mylo; hi = myhi;
    (void)lane;
  }
  const int lane = threadIdx.x & 31;
  const int warp_li0 = (blockIdx.x * blockDim.x + (threadIdx.x & ~31)) * 2;  // first node of this warp
  const int gnode0 = p.d.node_begin + li0;
  const bool vec_ok = ((N & 1) == 0) && ((gnode0 & 1) == 0);
  const int tb = p.work_begin[w], te = p.work_end[w];
  for (int i = tb; i < te; ++i) {
    const int t = p.group_tasks[i];
    double *row = p.score_out + (size_t)t * N;
    if (li0 + 1 < nloc && vec_ok) {
      __stcs(reinterpret_cast<double2 *>(row + gnode0), make_double2(s0, s1));
    } else {
      if (li0 < nloc) __stcs(row + gnode0, s0);
      if (li0 + 1 < nloc) __stcs(row + gnode0 + 1, s1);
    }
    if (lane < 2 && warp_li0 < nloc) {
      const int word32 = (p.d.node_begin + warp_li0) / 32 + lane;
      if (word32 < p.mw32) {
        // a row's words are owned by exactly one warp when node_begin is a multiple of 64
        p.mask_out[(size_t)t * p.mw32 + word32] = lane == 0 ? lo : hi;
      }
    }
  }
}

// K1f: final score + feasibility word of every (group, node) of the shard — what every task row of the group holds.
// grid (ceil(Nloc/256), G).
__global__ void __launch_bounds__(256) k_group_final(K1Params p, double *g_final, uint32_t *g_maskw, int mwg) {
  const int N = p.d.N;
  const int nloc = p.d.node_end - p.d.node_begin;
  const int li = blockIdx.x * blockDim.x + threadIdx.x;
  const int g = blockIdx.y + p.y_off;
  const int chosen = p.g_stats[g * 4 + 0] ? 0 : (p.g_stats[g * 4 + 1] ? 1 : 2);
  const int max_soft = chosen == 0 ? p.g_stats[g * 4 + 2] : p.g_stats[g * 4 + 3];
  double sc = 0.0;
  bool feas = false;
  if (li < nloc) {
    const int soft = (p.cstat[(size_t)p.g_class[g] * N + p.d.node_begin + li] >> CS_SOFT_SHIFT) & 0xff;
    k1_final(p, g, li, nloc, chosen, max_soft, soft, &sc, &feas);
    g_final[(size_t)g * nloc + li] = sc;
  }
  const unsigned bits = __ballot_sync(0xffffffffu, feas);
  if ((threadIdx.x & 31) == 0 && (li >> 5) < mwg) g_maskw[(size_t)g * mwg + (li >> 5)] = bits;
}

// K1b (bulk variant): a CTA stages the (group, node-chunk) piece of the group's final row and mask words in shared
// memory and streams it to every task row of the work item with the bulk asynchronous copy engine (cp.async.bulk
// shared -> global; one elected thread issues one 16-byte-aligned store of the whole chunk per row, plus one for its
// mask bytes), so HBM sees long contiguous write bursts and no partial-line stores.
// grid (ceil(Nloc/chunk), n_work), 256 threads; chunk is a multiple of 128 nodes; dynamic smem = chunk*8.
// Needs an even N (16-byte row alignment of the score matrix). The mask rows go out through k_mask_expand_bulk.
__global__ void __launch_bounds__(256) k_group_expand_bulk(K1Params p, int chunk, const double *g_final, const uint32_t *g_maskw,
                                                          int mwg) {
  extern __shared__ __align__(128) unsigned char k1_smem[];
  double *tile = reinterpret_cast<double *>(k1_smem);
  const int N = p.d.N;
  const int nloc = p.d.node_end - p.d.node_begin;
  const int w = blockIdx.y + p.y_off;
  const int g = p.work_group[w];
  const int c0 = blockIdx.x * chunk;
  const int cn = min(chunk, nloc - c0);
  const int cn2 = cn & ~1;
  // stage: 16-byte loads of the group's final row, 4-byte loads of its mask words (zero padding past the row)
  const double2 *src2 = reinterpret_cast<const double2 *>(g_final + (size_t)g * nloc + c0);
  const bool al = (((size_t)g * nloc + c0) & 1) == 0;
  if (al) {
    for (int k = threadIdx.x; k < cn2 / 2; k += blockDim.x) reinterpret_cast<double2 *>(tile)[k] = __ldg(src2 + k);
    if ((cn & 1) && threadIdx.x == 0) tile[cn - 1] = g_final[(size_t)g * nloc + c0 + cn - 1];
  } else {
    for (int k = threadIdx.x; k < cn; k += blockDim.x) tile[k] = g_final[(size_t)g * nloc + c0 + k];
  }
  __syncthreads();
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy smem writes -> visible to the copy engine
  const int tb = p.work_begin[w], te = p.work_end[w];
  const int gnode0 = p.d.node_begin + c0;
  if (threadIdx.x == 0) {
    const uint32_t src = (uint32_t)__cvta_generic_to_shared(tile);
    const int bytes = cn2 * 8;
    for (int i = tb; i < te; ++i) {
      double *dst = p.score_out + (size_t)p.group_tasks[i] * N + gnode0;
      if (bytes > 0)
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
    }
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  } else if ((cn & 1) && threadIdx.x == 1) {
    for (int i = tb; i < te; ++i) p.score_out[(size_t)p.group_tasks[i] * N + gnode0 + cn - 1] = tile[cn - 1];
  }
  if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // smem must outlive the reads
}

// K1m: the feasibility-mask rows of a work item. The rows of one group are identical and mask rows have a 16-byte
// pitch, so the CTA replicates the group's row in shared memory and covers every run of consecutive task ids with
// ONE bulk store (tasks of a job are consecutive and share their group). grid n_work, 128 threads,
// dynamic smem = rows_per_item * pitch bytes.
__global__ void __launch_bounds__(128) k_mask_expand_bulk(K1Params p, const uint32_t *g_maskw, int mwg, int rows_cap) {
  extern __shared__ __align__(128) unsigned char k1m_smem[];
  uint32_t *rows = reinterpret_cast<uint32_t *>(k1m_smem);
  const int w = blockIdx.x;
  const int g = p.work_group[w];
  const int tb = p.work_begin[w], te = p.work_end[w];
  const int nr = min(te - tb, rows_cap);
  const int pitch = p.mw32;  // 32-bit words per row
  const int w0 = p.d.node_begin >> 5;
  for (int k = threadIdx.x; k < pitch; k += blockDim.x) {
    const int gw = k - w0;
    rows[k] = (gw >= 0 && gw < mwg) ? g_maskw[(size_t)g * mwg + gw] : 0u;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < (nr - 1) * pitch; k += blockDim.x) rows[pitch + k] = rows[k % pitch];
  __syncthreads();
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  if (threadIdx.x == 0) {
    const uint32_t src = (uint32_t)__cvta_generic_to_shared(rows);
    int i = tb;
    while (i < te) {
      const int t0 = p.group_tasks[i];
      int j = i + 1;
      while (j < te && j - i < nr && p.group_tasks[j] == t0 + (j - i)) ++j;
      unsigned char *dst = reinterpret_cast<unsigned char *>(p.mask_out) + (size_t)t0 * pitch * 4;
      const int bytes = (j - i) * pitch * 4;
      asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
      i = j;
    }
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
  }
}


// vc_snapshot_update_nodes: scatter the compact rows of the dirty nodes into the [dim][N] arrays of the uploaded session
struct NodeDeltaParams {
  int N, R, K, n;
  const int32_t *idx;   // [n] node index
  const double *vals;   // [(4 * R + 2 * K)][n]: idle, used, releasing, pipelined, k8s_requested, k8s_nonzero_requested
  const int32_t *pods;  // [n] pod_count
  double *idle, *used, *rel, *pip, *kreq, *knz;
  int32_t *pod_count;
};
__global__ void k_node_delta(NodeDeltaParams p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.n) return;
  const int n = p.idx[i];
  const size_t N = (size_t)p.N, m = (size_t)p.n;
  for (int d = 0; d < p.R; ++d) {
    p.idle[d * N + n] = p.vals[(size_t)d * m + i];
    p.used[d * N + n] = p.vals[(size_t)(p.R + d) * m + i];
    p.rel[d * N + n] = p.vals[(size_t)(2 * p.R + d) * m + i];
    p.pip[d * N + n] = p.vals[(size_t)(3 * p.R + d) * m + i];
  }
  for (int k = 0; k < p.K; ++k) p.kreq[k * N + n] = p.vals[(size_t)(4 * p.R + k) * m + i];
  for (int k = 0; k < 2; ++k) p.knz[k * N + n] = p.vals[(size_t)(4 * p.R + p.K + k) * m + i];
  p.pod_count[n] = p.pods[i];
}

// Micro-benchmark of the intra-GPU all-gather used by the commit kernels: G persistent CTAs, each posts one
// 16-byte self-tagged record per round and reads everybody's. Prints cycles per round for several layouts.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o exchange_bench exchange_bench.cu
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>

__device__ __forceinline__ void st_v4(uint4 *p, uint4 v) {
  asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 ld_v4(const uint4 *p) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint4 ld_relaxed_v4(const uint4 *p) {
  uint4 v;
  asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}

// mode 0: stride uint4 per slot (stride 16 = 256 B), one warp polls, up to 4-5 slots per lane
// mode 1: same with extra work_cycles of skew on odd CTAs
template <int STRIDE>
__global__ void k_allgather(uint4 *mbox, int rounds, long long *out, int jitter) {
  const int G = gridDim.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long t0 = clock64();
  unsigned acc = 0;
  for (int r = 1; r <= rounds; ++r) {
    if (jitter > 0) {  // per-CTA, per-round pseudo-random amount of "own work" before posting
      unsigned h = (blockIdx.x * 2654435761u) ^ (r * 40503u);
      h ^= h >> 13; h *= 0x5bd1e995u; h ^= h >> 15;
      long long until = clock64() + (long long)(h % (unsigned)jitter);
      while (clock64() < until) {}
    }
    if (warp == 0) {
      uint4 *base = mbox + (size_t)(r & 1) * G * STRIDE;
      if (lane == 0) st_v4(base + (size_t)blockIdx.x * STRIDE, make_uint4(blockIdx.x, acc, 7u, (unsigned)r));
      for (int s0 = 0; s0 < G; s0 += 128) {
        bool need[4];
        uint4 a[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) need[k] = s0 + k * 32 + lane < G;
        bool pending;
        do {
          pending = false;
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (need[k]) a[k] = ld_v4(base + (size_t)(s0 + k * 32 + lane) * STRIDE);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            if (!need[k]) continue;
            if (a[k].w != (unsigned)r) { pending = true; continue; }
            acc += a[k].x;
            need[k] = false;
          }
        } while (pending);
      }
      for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) { out[blockIdx.x * 2] = clock64() - t0; out[blockIdx.x * 2 + 1] = acc; }
}

// all-gather preceded, each round, by one ordinary global store into a large per-CTA region (models the undo-log /
// replica writes of the commit kernels): does a store that misses L2 delay the mailbox store behind it?
template <int STRIDE>
__global__ void k_allgather_dirty(uint4 *mbox, int rounds, long long *out, int *big, size_t big_stride, int same_thread) {
  const int G = gridDim.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long t0 = clock64();
  unsigned acc = 0;
  int *mine = big + (size_t)blockIdx.x * big_stride;
  for (int r = 1; r <= rounds; ++r) {
    if (!same_thread && threadIdx.x == 64) mine[((size_t)r * 32) % big_stride] = r;
    __syncthreads();
    if (warp == 0) {
      uint4 *base = mbox + (size_t)(r & 1) * G * STRIDE;
      if (lane == 0) {
        if (same_thread) mine[((size_t)r * 32) % big_stride] = r;
        st_v4(base + (size_t)blockIdx.x * STRIDE, make_uint4(blockIdx.x, acc, 7u, (unsigned)r));
      }
      for (int s0 = 0; s0 < G; s0 += 128) {
        bool need[4];
        uint4 a[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) need[k] = s0 + k * 32 + lane < G;
        bool pending;
        do {
          pending = false;
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (need[k]) a[k] = ld_v4(base + (size_t)(s0 + k * 32 + lane) * STRIDE);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            if (!need[k]) continue;
            if (a[k].w != (unsigned)r) { pending = true; continue; }
            acc += a[k].x;
            need[k] = false;
          }
        } while (pending);
      }
      for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) { out[blockIdx.x * 2] = clock64() - t0; out[blockIdx.x * 2 + 1] = acc; }
}

// hierarchical: every CTA posts; only CTA-group leaders... (placeholder for cluster variant)

// counter-based: each CTA posts its record then bumps ONE arrival counter per round (red.add); pollers spin on the
// counter only and then read all records once.
template <int STRIDE>
__global__ void k_counter(uint4 *mbox, unsigned *counters, int rounds, long long *out) {
  const int G = gridDim.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long t0 = clock64();
  unsigned acc = 0;
  for (int r = 1; r <= rounds; ++r) {
    if (warp == 0) {
      uint4 *base = mbox + (size_t)(r & 1) * G * STRIDE;
      if (lane == 0) {
        st_v4(base + (size_t)blockIdx.x * STRIDE, make_uint4(blockIdx.x, acc, 7u, (unsigned)r));
        __threadfence();
        atomicAdd(&counters[r & 3], 1u);
        unsigned target = (unsigned)G * (unsigned)((r + 3) / 4);
        while (*(volatile unsigned *)&counters[r & 3] < target) {}
      }
      __syncwarp();
      for (int s = lane; s < G; s += 32) acc += ld_v4(base + (size_t)s * STRIDE).x;
      for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) { out[blockIdx.x * 2] = clock64() - t0; out[blockIdx.x * 2 + 1] = acc; }
}

int main(int argc, char **argv) {
  int rounds = argc > 1 ? atoi(argv[1]) : 20000;
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  int G = prop.multiProcessorCount;
  if (argc > 2) G = atoi(argv[2]);
  uint4 *mbox;
  long long *out;
  unsigned *counters;
  cudaMalloc(&mbox, sizeof(uint4) * 64 * 2 * 1024);
  cudaMalloc(&out, 16 * 1024);
  cudaMalloc(&counters, 64);
  long long *h = (long long *)malloc(16 * 1024);
  auto run = [&](const char *name, const void *fn, void **args, int threads) {
    cudaMemset(mbox, 0, sizeof(uint4) * 64 * 2 * 1024);
    cudaMemset(counters, 0, 64);
    cudaError_t e = cudaLaunchCooperativeKernel(fn, dim3(G), dim3(threads), args, 0, 0);
    cudaDeviceSynchronize();
    if (e != cudaSuccess || cudaGetLastError() != cudaSuccess) { printf("%s: launch failed %s\n", name, cudaGetErrorString(e)); return; }
    cudaMemcpy(h, out, 16 * 1024, cudaMemcpyDeviceToHost);
    long long mx = 0;
    for (int i = 0; i < G; ++i) mx = h[2 * i] > mx ? h[2 * i] : mx;
    printf("%-40s G=%d threads=%d: %.0f cycles/round\n", name, G, threads, (double)mx / rounds);
  };
  int zero = 0;
  {
    void *args[] = {&mbox, &rounds, &out, &zero};
    run("allgather stride 256B", (const void *)k_allgather<16>, args, 128);
    run("allgather stride 256B (256 thr)", (const void *)k_allgather<16>, args, 256);
    run("allgather stride 16B", (const void *)k_allgather<1>, args, 128);
    run("allgather stride 128B", (const void *)k_allgather<8>, args, 128);
    run("allgather stride 32B", (const void *)k_allgather<2>, args, 128);
    for (int j : {1000, 3000, 10000}) {
      int jj = j;
      void *a2[] = {&mbox, &rounds, &out, &jj};
      char name[64];
      snprintf(name, sizeof name, "allgather 256B, own work U(0,%d)", j);
      run(name, (const void *)k_allgather<16>, a2, 128);
    }
  }
  {
    int *big;
    for (size_t mb : {1, 4}) {
      size_t big_stride = mb * 1024 * 1024 / 4;
      cudaMalloc(&big, big_stride * 4 * G);
      cudaMemset(big, 0, big_stride * 4 * G);
      for (int same = 0; same < 2; ++same) {
        void *args[] = {&mbox, &rounds, &out, &big, &big_stride, &same};
        char name[96];
        snprintf(name, sizeof name, "allgather 256B + dirty store %zu MB/CTA %s", mb, same ? "same thread" : "other warp");
        run(name, (const void *)k_allgather_dirty<16>, args, 128);
      }
      cudaFree(big);
    }
  }
  {
    void *args[] = {&mbox, &counters, &rounds, &out};
    run("counter + read-once stride 256B", (const void *)k_counter<16>, args, 128);
    run("counter + read-once stride 16B", (const void *)k_counter<1>, args, 128);
  }
  return 0;
}

// How fast can shared->global bulk copies write HBM?  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o bulk_store_bench bulk_store_bench.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
__global__ void k_bulk(double *out, size_t row_stride_elems, int rows, int chunk, int issuers) {
  extern __shared__ __align__(128) unsigned char sm[];
  double *tile = reinterpret_cast<double *>(sm);
  for (int i = threadIdx.x; i < chunk; i += blockDim.x) tile[i] = (double)i;
  __syncthreads();
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  const size_t base = (size_t)blockIdx.y * rows * row_stride_elems + (size_t)blockIdx.x * chunk;
  if ((threadIdx.x & 31) == 0 && (threadIdx.x >> 5) < issuers) {
    const int wi = threadIdx.x >> 5;
    const unsigned src = (unsigned)__cvta_generic_to_shared(tile);
    for (int r = wi; r < rows; r += issuers) {
      double *dst = out + base + (size_t)r * row_stride_elems;
      asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(chunk * 8) : "memory");
    }
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
  }
}
__global__ void k_plain(double2 *out, size_t n2) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n2; i += stride) __stcs(out + i, make_double2(1.0, 2.0));
}
int main() {
  const size_t N = 10000, T = 100000;
  double *out;
  cudaMalloc(&out, N * T * 8);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  auto time = [&](auto fn, const char *name) {
    fn(); cudaDeviceSynchronize();
    cudaEventRecord(e0);
    for (int i = 0; i < 5; ++i) fn();
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= 5;
    printf("%-60s %.3f ms  %.0f GB/s  (%s)\n", name, ms, N * T * 8 / ms / 1e6, cudaGetErrorString(cudaGetLastError()));
  };
  time([&] { cudaMemsetAsync(out, 0, N * T * 8); }, "cudaMemsetAsync");
  time([&] { k_plain<<<132 * 16, 256>>>((double2 *)out, N * T / 2); }, "plain st.cs double2, grid-stride");
  for (int issuers : {1, 4}) for (int chunk : {5000, 10000}) for (int rows : {64, 16}) {
    cudaFuncSetAttribute(k_bulk, cudaFuncAttributeMaxDynamicSharedMemorySize, chunk * 8);
    dim3 grid((unsigned)(N / chunk), (unsigned)(T / rows));
    char name[96];
    snprintf(name, sizeof name, "bulk: chunk %d, %d rows/CTA (stride N), %d issuing warps", chunk, rows, issuers);
    time([&] { k_bulk<<<grid, 256, chunk * 8>>>(out, N, rows, chunk, issuers); }, name);
  }
  return 0;
}

// layout.cu -- layout conversion between R's column-major n x m matrices (genes fastest; what
// .Call hands over, /root/reference/src/DESeq2.cpp:165-169,285-287) and the engine's gene-major
// rows (sample axis contiguous, row stride ld) that the warp-per-gene kernels read with 128-bit loads.
// Plain tiled shared-memory transposes: both global sides are fully coalesced.  Also the device queries the launchers
// share (SM count, persistent-grid size).
#include <algorithm>
#include <mutex>
#include <utility>
#include <vector>

#include "engine.h"
#include "nbmath.cuh"

namespace nb {
namespace {

template <typename T>
__global__ void __launch_bounds__(256) to_gene_major_kernel(const T* __restrict__ src, T* __restrict__ dst, int n,
                                                            int m, long long ld) {
  __shared__ T tile[32][33];
  const int i0 = blockIdx.x * 32, j0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  for (int jj = ty; jj < 32; jj += 8) {
    const int i = i0 + tx, j = j0 + jj;
    if (i < n && j < m) tile[jj][tx] = src[(size_t)i + (size_t)n * j];
  }
  __syncthreads();
  for (int ii = ty; ii < 32; ii += 8) {
    const int i = i0 + ii, j = j0 + tx;
    if (i < n && j < m) dst[(size_t)i * ld + j] = tile[tx][ii];
  }
}

__global__ void __launch_bounds__(256) to_col_major_kernel(const double* __restrict__ src, double* __restrict__ dst,
                                                           int n, int m, long long ld) {
  __shared__ double tile[32][33];
  const int i0 = blockIdx.x * 32, j0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int ii = ty; ii < 32; ii += 8) {
    const int i = i0 + ii, j = j0 + tx;
    if (i < n && j < m) tile[ii][tx] = src[(size_t)i * ld + j];
  }
  __syncthreads();
  for (int jj = ty; jj < 32; jj += 8) {
    const int i = i0 + tx, j = j0 + jj;
    if (i < n && j < m) dst[(size_t)i + (size_t)n * j] = tile[tx][jj];
  }
}

// Content hash of a gene-major matrix (hostrt.h::hash_elems computes the same value from the column-major host
// buffer): element (i, j) has canonical index i + n j.  out[0], out[1] must be zero on entry.
__global__ void __launch_bounds__(256) hash_gene_major_kernel(const void* __restrict__ src, int n, int m, long long ld,
                                                              int elem, unsigned long long* __restrict__ out) {
  const unsigned long long K1 = 0x9E3779B97F4A7C15ull, K2 = 0xD6E8FEB86659FD93ull;
  unsigned long long a = 0, b = 0;
  const long long total = (long long)n * ld;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const long long i = t / ld;
    const int j = (int)(t - i * ld);
    if (j >= m) continue;
    const unsigned long long v = (elem == 8) ? static_cast<const unsigned long long*>(src)[t]
                                             : (unsigned long long)static_cast<const unsigned int*>(src)[t];
    const unsigned long long e = (unsigned long long)i + (unsigned long long)n * (unsigned long long)j;
    const unsigned long long x1 = v ^ ((e + 1) * K1), x2 = v ^ ((e + 1) * K2);
    a += (unsigned long long)(unsigned int)x1 * (unsigned long long)(unsigned int)(x1 >> 32) + ((x1 << 32) | (x1 >> 32));
    b += (unsigned long long)(unsigned int)x2 * (unsigned long long)(unsigned int)(x2 >> 32) + ((x2 << 32) | (x2 >> 32));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(out, a);
    atomicAdd(out + 1, b);
  }
}

__global__ void special_test_kernel(const double* x, int n, double* lg, double* dg, double* tg) {
  init_log_table();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double a, b;
  lgamma_digamma_pos(x[i], a, b);
  lg[i] = a;
  dg[i] = b;
  tg[i] = trigamma_pos(x[i]);
}

}  // namespace

cudaError_t launch_to_gene_major(const void* src, void* dst, int n, int m, long long ld, int elem_size,
                                 cudaStream_t stream) {
  if (n == 0 || m == 0) return cudaSuccess;
  dim3 grid((n + 31) / 32, (m + 31) / 32), block(32, 8);
  if (elem_size == 4)
    to_gene_major_kernel<int32_t><<<grid, block, 0, stream>>>(static_cast<const int32_t*>(src),
                                                              static_cast<int32_t*>(dst), n, m, ld);
  else if (elem_size == 8)
    to_gene_major_kernel<double><<<grid, block, 0, stream>>>(static_cast<const double*>(src),
                                                             static_cast<double*>(dst), n, m, ld);
  else
    return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_to_col_major(const double* src, double* dst, int n, int m, long long ld, cudaStream_t stream) {
  if (n == 0 || m == 0) return cudaSuccess;
  dim3 grid((n + 31) / 32, (m + 31) / 32), block(32, 8);
  to_col_major_kernel<<<grid, block, 0, stream>>>(src, dst, n, m, ld);
  return cudaGetLastError();
}

cudaError_t launch_hash_gene_major(const void* src, int n, int m, long long ld, int elem_size,
                                   unsigned long long* out2, cudaStream_t stream) {
  cudaError_t e = cudaMemsetAsync(out2, 0, 2 * sizeof(unsigned long long), stream);
  if (e != cudaSuccess || n == 0 || m == 0) return e;
  const long long total = (long long)n * ld;
  long long blocks = (total + 255) / 256;
  const long long cap = (long long)device_sm_count() * 8;
  if (blocks > cap) blocks = cap;
  hash_gene_major_kernel<<<(unsigned)blocks, 256, 0, stream>>>(src, n, m, ld, elem_size, out2);
  return cudaGetLastError();
}

cudaError_t launch_special_test(const double* x, int n, double* lg, double* dg, double* tg, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  special_test_kernel<<<(n + 255) / 256, 256, 0, stream>>>(x, n, lg, dg, tg);
  return cudaGetLastError();
}

int device_sm_count() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;   // H100 SXM
  }
  return sms;
}

cudaError_t persistent_grid(const void* kernel, int threads, size_t smem, int genes_per_cta, int n, unsigned* grid) {
  struct Occupancy {
    const void* kernel;
    int threads;
    size_t smem;
    int ctas_per_sm;
  };
  static std::mutex mu;
  static std::vector<Occupancy> cache;
  static std::vector<std::pair<const void*, size_t>> smem_limit;   // the limit last set per kernel
  std::lock_guard<std::mutex> lk(mu);
  auto lim = std::find_if(smem_limit.begin(), smem_limit.end(), [&](const auto& l) { return l.first == kernel; });
  if (lim == smem_limit.end() || lim->second != smem) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    if (lim == smem_limit.end()) smem_limit.emplace_back(kernel, smem);
    else lim->second = smem;
  }
  auto hit = std::find_if(cache.begin(), cache.end(), [&](const Occupancy& o) {
    return o.kernel == kernel && o.threads == threads && o.smem == smem;
  });
  if (hit == cache.end()) {
    int c = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c, kernel, threads, smem);
    if (e != cudaSuccess) return e;
    if (c < 1) return cudaErrorLaunchOutOfResources;
    cache.push_back({kernel, threads, smem, c});
    hit = cache.end() - 1;
  }
  const long long want = ((long long)n + genes_per_cta - 1) / genes_per_cta;
  long long g = (long long)device_sm_count() * hit->ctas_per_sm;
  if (g > want) g = want;
  *grid = (unsigned)(g < 1 ? 1 : g);
  return cudaSuccess;
}

}  // namespace nb

// selftest_kernels.cu -- small kernels with known answers that pin the SIMT emulator's semantics
// (tests/test_simt_emu.py).  Written as ordinary CUDA (it also compiles with nvcc); TEST INFRASTRUCTURE ONLY.
#include <cuda_runtime.h>
#include <stdint.h>

__global__ void k_warp_collectives(double* out_sum, int* out_misc) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double v = (double)(threadIdx.x + 1);
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) out_sum[blockIdx.x * (blockDim.x >> 5) + warp] = v;
  int* m = out_misc + (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  m[0] = __shfl_sync(0xffffffffu, lane * 10, 5);               // broadcast of lane 5
  m[1] = __shfl_down_sync(0xffffffffu, lane, 3);               // lane + 3, own value past the end
  m[2] = __shfl_up_sync(0xffffffffu, lane, 2);                 // lane - 2, own value before the start
  m[3] = __shfl_xor_sync(0xffffffffu, lane, 1, 8);             // neighbour inside segments of 8
  m[4] = (int)__ballot_sync(0xffffffffu, lane % 3 == 0);
  m[5] = __any_sync(0xffffffffu, lane == 31) + 2 * __all_sync(0xffffffffu, lane < 31);
  m[6] = __shfl_sync(0xffffffffu, lane, 3, 4);                 // lane 3 of each segment of 4
  m[7] = __shfl_down_sync(0xffffffffu, lane, 1, 16);           // width 16: lane 15 keeps its own value
}

// cross-warp exchange through static and dynamic shared memory, ordered by __syncthreads
__global__ void k_cta_reverse(const int* in, int* out, int n) {
  __shared__ int stat[256];
  extern __shared__ __align__(16) double smem[];
  const int t = threadIdx.x, base = blockIdx.x * blockDim.x;
  stat[t] = (base + t < n) ? in[base + t] : -1;
  smem[t] = 0.5 * stat[t];
  __syncthreads();
  const int r = blockDim.x - 1 - t;
  if (base + t < n) out[base + t] = stat[r] + (int)(2.0 * smem[r]);
}

// persistent warps pulling items from an atomic queue; lane 0 fetches, the warp learns the index by shuffle
__global__ void k_queue(unsigned* counter, int n, int* owner_count, double* out) {
  const int lane = threadIdx.x & 31;
  for (;;) {
    unsigned q = 0;
    if (lane == 0) q = atomicAdd(counter, 1u);
    q = __shfl_sync(0xffffffffu, q, 0);
    if (q >= (unsigned)n) break;
    double v = (double)(q + 1) * (lane + 1);
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) { out[q] = v; atomicAdd(&owner_count[blockIdx.x], 1); }
  }
}

// A kernel with a real bug: lane l reads what lane l+1 wrote to shared memory with no __syncwarp in between.
// On the GPU this "works" whenever the warp happens to run converged; the emulator must NOT reproduce that luck.
__global__ void k_missing_syncwarp(int* out, int with_sync) {
  __shared__ int buf[32];
  const int lane = threadIdx.x & 31;
  buf[lane] = -1;
  __syncwarp();
  buf[lane] = lane;
  if (with_sync) __syncwarp();
  out[lane] = buf[(lane + 1) & 31];
}

// half of the warp never reaches a full-mask collective: undefined behaviour on the GPU, a reported deadlock here
__global__ void k_divergent_collective(int* out) {
  const int lane = threadIdx.x & 31;
  int v = lane;
  if (lane < 16) {
    for (;;) {            // these lanes wait for the others forever
      v = __shfl_xor_sync(0xffffffffu, v, 1);
      if (v < 0) break;
    }
  } else {
    __syncthreads();      // ... while the others sit in a different barrier
  }
  out[lane] = v;
}

// reading dynamic shared memory that was never written must yield the poison value (NaN), not a stale result
__global__ void k_uninitialised_smem(double* out) {
  extern __shared__ __align__(16) double smem[];
  out[threadIdx.x] = smem[threadIdx.x];
}

// touches the last double of its dynamic shared memory, so that a launch that runs is visible in `ran`
__global__ void k_smem_limit(int* ran, size_t doubles) {
  extern __shared__ __align__(16) double smem[];
  smem[doubles - 1] = 1.0;
  *ran = (int)smem[doubles - 1];
}

// the same, for the launches that never set the attribute (its limit stays the 48 KB default whatever ran before)
__global__ void k_smem_default(int* ran, size_t doubles) {
  extern __shared__ __align__(16) double smem[];
  smem[doubles - 1] = 1.0;
  *ran = (int)smem[doubles - 1];
}

extern "C" {
int st_warp_collectives(double* out_sum, int* out_misc, int blocks, int threads) {
  k_warp_collectives<<<blocks, threads, 0, 0>>>(out_sum, out_misc);
  return (int)cudaGetLastError();
}
int st_cta_reverse(const int* in, int* out, int n) {
  k_cta_reverse<<<(n + 255) / 256, 256, 256 * sizeof(double), 0>>>(in, out, n);
  return (int)cudaGetLastError();
}
int st_queue(unsigned* counter, int n, int* owner_count, double* out, int blocks, int threads) {
  k_queue<<<blocks, threads, 0, 0>>>(counter, n, owner_count, out);
  return (int)cudaGetLastError();
}
int st_missing_syncwarp(int* out, int with_sync) {
  k_missing_syncwarp<<<1, 32, 0, 0>>>(out, with_sync);
  return (int)cudaGetLastError();
}
int st_divergent_collective(int* out) {
  k_divergent_collective<<<1, 32, 0, 0>>>(out);
  return (int)cudaGetLastError();
}
// attr > 0: cudaFuncSetAttribute(MaxDynamicSharedMemorySize, attr) first (attr == 0: a kernel that never sets it);
// returns the first error
int st_smem_limit(int* ran, int bytes, int attr) {
  if (attr == 0) {
    k_smem_default<<<1, 32, (size_t)bytes, 0>>>(ran, (size_t)bytes / sizeof(double));
    return (int)cudaGetLastError();
  }
  {
    const cudaError_t e = cudaFuncSetAttribute(k_smem_limit, cudaFuncAttributeMaxDynamicSharedMemorySize, attr);
    if (e != cudaSuccess) return (int)e;
  }
  k_smem_limit<<<1, 32, (size_t)bytes, 0>>>(ran, (size_t)bytes / sizeof(double));
  return (int)cudaGetLastError();
}
int st_uninitialised_smem(double* out) {
  k_uninitialised_smem<<<1, 64, 64 * sizeof(double), 0>>>(out);
  return (int)cudaGetLastError();
}
}

/*
 * cuda_runtime.h (SIMT EMULATOR) -- TEST INFRASTRUCTURE ONLY.
 *
 * A stand-in for <cuda_runtime.h> that lets g++ compile the product's CUDA sources (deseq2_b200/csrc/*.cu, unmodified
 * apart from three mechanical rewrites done by tests/simt_emu/build_emu.py: the <<<...>>> launch syntax, the
 * `extern __shared__` declaration and one inline-PTX statement) into a host library that EXECUTES the kernels with
 * SIMT semantics on the CPU:
 *   - every CUDA thread of a CTA is a fiber (ucontext) on one OS thread; CTAs of a grid run one after the other;
 *   - a fiber runs until it reaches a warp collective (__shfl_*_sync, __syncwarp, votes) or __syncthreads, where it
 *     yields; the scheduler releases a barrier when every live lane named by the mask has arrived.  A lane that
 *     reads shared memory written by another lane without a barrier in between sees stale data here (lanes do
 *     NOT advance in lock step), and a collective that not all named lanes reach is reported as a deadlock: both
 *     are bugs on the GPU too, so the emulator doubles as a synchronisation checker;
 *   - "device memory" is host memory, streams are no-ops, launches are synchronous; fresh device and dynamic
 *     shared memory is poisoned with 0xFF bytes (NaNs) so reads of uninitialised memory surface in the results;
 *   - a launch whose DYNAMIC shared memory exceeds what sm_90 grants that kernel fails as on the GPU (see
 *     kDynSmemOptinMax below).  `__shared__` becomes `static`, so a kernel's STATIC shared memory is invisible here:
 *     the launch plans subtract it themselves (e.g. fit_generic.cu::plan_seg's 4 KB), and only a run on the GPU
 *     checks that the sum of both fits.
 * Purpose: the CPU test-suite (tests/test_emulated_kernels.py) runs the kernels' own source against the oracle
 * without a GPU.  Arithmetic is IEEE fp64 with FMA contraction like nvcc's default, but it is not bit-identical
 * to the GPU (MUFU.RCP64H seed, contraction choices), so the tests use the same tolerances as the -m gpu tests.
 *
 * The product never sees this file: it lives under tests/, is only on the include path of the emulator build,
 * and the library it produces (tests/simt_emu/_build/libb200nb_emu.so) is loaded by the tests alone.
 */
#ifndef SIMT_EMU_CUDA_RUNTIME_H
#define SIMT_EMU_CUDA_RUNTIME_H

#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <cmath>
#include <functional>

#define SIMT_EMU 1
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __shared__ static
#define __constant__ static
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))

/* ------------------------------------------------------------------ vector types */
struct uint3 { unsigned x, y, z; };
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {}
};
struct __attribute__((aligned(8))) int2 { int x, y; };
struct __attribute__((aligned(16))) int4 { int x, y, z, w; };
struct __attribute__((aligned(8))) uint2 { unsigned x, y; };
struct __attribute__((aligned(16))) uint4 { unsigned x, y, z, w; };
struct __attribute__((aligned(8))) float2 { float x, y; };
struct __attribute__((aligned(16))) float4 { float x, y, z, w; };
struct __attribute__((aligned(16))) double2 { double x, y; };
struct __attribute__((aligned(16))) double4 { double x, y, z, w; };
static inline int2 make_int2(int x, int y) { return int2{x, y}; }
static inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline double2 make_double2(double x, double y) { return double2{x, y}; }
static inline double4 make_double4(double x, double y, double z, double w) { return double4{x, y, z, w}; }

/* ------------------------------------------------------------------ built-in variables (set by the scheduler) */
extern uint3 threadIdx, blockIdx;
extern dim3 blockDim, gridDim;
static const int warpSize = 32;

/* ------------------------------------------------------------------ scheduler interface (emu.cpp) */
namespace simt_emu {
/* Per-block dynamic shared-memory limits of sm_90, enforced as the runtime does: a launch above the opt-in maximum,
 * or above 48 KB without a cudaFuncSetAttribute(MaxDynamicSharedMemorySize) for that kernel that allows it, fails
 * (cudaErrorInvalidValue from cudaGetLastError) and its kernel does not run. */
constexpr size_t kDynSmemDefault = 48 * 1024;
constexpr size_t kDynSmemOptinMax = 232448;
void launch(const void* kernel, dim3 grid, dim3 block, size_t dyn_smem_bytes, const std::function<void()>& body,
            const char* what = "", const char* where = "");
int set_max_dyn_smem(const void* kernel, int bytes);   /* cudaFuncSetAttribute(MaxDynamicSharedMemorySize) */
int last_error(bool reset);                             /* cudaGetLastError / cudaPeekAtLastError */
void* dyn_smem_ptr();
void barrier_warp(unsigned mask);
void barrier_cta();
uint64_t exchange(unsigned mask, uint64_t bits, int src_lane);   /* value held by src_lane (own if not named) */
unsigned ballot(unsigned mask, int pred);
int lane_id();
double rcp_approx_f64(double x);                                  /* rcp.approx.ftz.f64: ~20 good bits */
long long launches();
}  // namespace simt_emu

/* ------------------------------------------------------------------ warp collectives */
namespace simt_emu {
template <typename T>
inline T shfl_from(unsigned mask, T v, int src) {
  static_assert(sizeof(T) <= 8, "shuffle of at most 64 bits");
  uint64_t b = 0;
  memcpy(&b, &v, sizeof(T));
  b = exchange(mask, b, src);
  T r;
  memcpy(&r, &b, sizeof(T));
  return r;
}
}  // namespace simt_emu

template <typename T>
inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
  const int lane = simt_emu::lane_id(), base = lane & ~(width - 1);
  return simt_emu::shfl_from(mask, v, base | (src & (width - 1)));
}
template <typename T>
inline T __shfl_xor_sync(unsigned mask, T v, int lane_mask, int width = 32) {
  const int lane = simt_emu::lane_id(), base = lane & ~(width - 1);
  const int src = lane ^ lane_mask;
  return simt_emu::shfl_from(mask, v, (src >= base + width) ? lane : src);
}
template <typename T>
inline T __shfl_down_sync(unsigned mask, T v, unsigned delta, int width = 32) {
  const int lane = simt_emu::lane_id(), base = lane & ~(width - 1);
  const int src = lane + (int)delta;
  return simt_emu::shfl_from(mask, v, (src >= base + width) ? lane : src);
}
template <typename T>
inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int width = 32) {
  const int lane = simt_emu::lane_id(), base = lane & ~(width - 1);
  const int src = lane - (int)delta;
  return simt_emu::shfl_from(mask, v, (src < base) ? lane : src);
}
inline unsigned __ballot_sync(unsigned mask, int pred) { return simt_emu::ballot(mask, pred); }
inline int __any_sync(unsigned mask, int pred) { return simt_emu::ballot(mask, pred) != 0; }
inline int __all_sync(unsigned mask, int pred) { return simt_emu::ballot(mask, !pred) == 0; }
inline void __syncwarp(unsigned mask = 0xffffffffu) { simt_emu::barrier_warp(mask); }
inline void __syncthreads() { simt_emu::barrier_cta(); }
template <typename T>
inline T __ldcg(const T* p) { return *p; }
inline void __threadfence() {}
inline void __threadfence_block() {}

/* ------------------------------------------------------------------ memory / bit intrinsics */
template <typename T>
inline T __ldg(const T* p) { return *p; }
inline unsigned long long __umul64hi(unsigned long long a, unsigned long long b) {
  return (unsigned long long)(((unsigned __int128)a * b) >> 64);
}
inline int __double2hiint(double x) { uint64_t b; memcpy(&b, &x, 8); return (int)(b >> 32); }
inline int __double2loint(double x) { uint64_t b; memcpy(&b, &x, 8); return (int)(b & 0xffffffffu); }
inline double __hiloint2double(int hi, int lo) {
  const uint64_t b = ((uint64_t)(uint32_t)hi << 32) | (uint32_t)lo;
  double x;
  memcpy(&x, &b, 8);
  return x;
}
inline long long __double_as_longlong(double x) { long long b; memcpy(&b, &x, 8); return b; }
inline double __longlong_as_double(long long b) { double x; memcpy(&x, &b, 8); return x; }
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
inline int __ffs(int x) { return __builtin_ffs(x); }

/* one OS thread runs every fiber: plain read-modify-write is atomic with respect to the other CUDA threads */
template <typename T>
inline T atomicAdd(T* p, T v) { T o = *p; *p = o + v; return o; }
inline unsigned atomicAdd(unsigned* p, int v) { unsigned o = *p; *p = o + (unsigned)v; return o; }
template <typename T>
inline T atomicMax(T* p, T v) { T o = *p; if (v > o) *p = v; return o; }
template <typename T>
inline T atomicMin(T* p, T v) { T o = *p; if (v < o) *p = v; return o; }
template <typename T>
inline T atomicExch(T* p, T v) { T o = *p; *p = v; return o; }
template <typename T>
inline T atomicCAS(T* p, T cmp, T v) { T o = *p; if (o == cmp) *p = v; return o; }

/* ------------------------------------------------------------------ math (CUDA puts these in the global namespace) */
using std::isfinite;
using std::isinf;
using std::isnan;
inline double rsqrt(double x) { return 1.0 / sqrt(x); }
inline double rcp(double x) { return 1.0 / x; }
inline double __drcp_rn(double x) { return 1.0 / x; }
inline double __dsqrt_rn(double x) { return sqrt(x); }
inline double __dadd_rn(double a, double b) { volatile double r = a + b; return r; }
inline double __dmul_rn(double a, double b) { volatile double r = a * b; return r; }
inline double __fma_rn(double a, double b, double c) { return fma(a, b, c); }
inline double __int2double_rn(int x) { return (double)x; }
inline double __uint2double_rn(unsigned x) { return (double)x; }
inline double __ll2double_rn(long long x) { return (double)x; }
inline int __double2int_rn(double x) { return (int)nearbyint(x); }
inline int __double2int_rz(double x) { return (int)x; }
inline int __double2int_rd(double x) { return (int)floor(x); }
inline int __double2int_ru(double x) { return (int)ceil(x); }
inline int min(int a, int b) { return a < b ? a : b; }
inline int max(int a, int b) { return a > b ? a : b; }
inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
inline long long min(long long a, long long b) { return a < b ? a : b; }
inline long long max(long long a, long long b) { return a > b ? a : b; }
inline size_t min(size_t a, size_t b) { return a < b ? a : b; }
inline size_t max(size_t a, size_t b) { return a > b ? a : b; }
inline double min(double a, double b) { return fmin(a, b); }
inline double max(double a, double b) { return fmax(a, b); }

/* ------------------------------------------------------------------ runtime API (synchronous host stand-ins) */
typedef int cudaError_t;
enum {
  cudaSuccess = 0,
  cudaErrorInvalidValue = 1,
  cudaErrorMemoryAllocation = 2,
  cudaErrorLaunchOutOfResources = 701,
};
typedef struct simt_emu_stream* cudaStream_t;
typedef struct simt_emu_event* cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2,
                      cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16 };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaHostAllocDefault = 0 };

cudaError_t cudaMalloc(void** p, size_t bytes);
cudaError_t cudaFree(void* p);
cudaError_t cudaHostAlloc(void** p, size_t bytes, unsigned flags);
cudaError_t cudaFreeHost(void* p);
template <typename T>
inline cudaError_t cudaMalloc(T** p, size_t bytes) { return cudaMalloc(reinterpret_cast<void**>(p), bytes); }
template <typename T>
inline cudaError_t cudaHostAlloc(T** p, size_t bytes, unsigned flags) {
  return cudaHostAlloc(reinterpret_cast<void**>(p), bytes, flags);
}
inline cudaError_t cudaMemcpy2DAsync(void* d, size_t dpitch, const void* s, size_t spitch, size_t width, size_t height,
                                     cudaMemcpyKind, cudaStream_t = 0) {
  for (size_t r = 0; r < height; r++)
    memcpy(static_cast<char*>(d) + r * dpitch, static_cast<const char*>(s) + r * spitch, width);
  return cudaSuccess;
}
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = 0) {
  if (n) memmove(d, s, n);
  return cudaSuccess;
}
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) {
  if (n) memmove(d, s, n);
  return cudaSuccess;
}
inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = 0) {
  if (n) memset(d, v, n);
  return cudaSuccess;
}
inline cudaError_t cudaMemset(void* d, int v, size_t n) {
  if (n) memset(d, v, n);
  return cudaSuccess;
}
inline cudaError_t cudaGetLastError() { return simt_emu::last_error(true); }
inline cudaError_t cudaPeekAtLastError() { return simt_emu::last_error(false); }
inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "simt_emu error"; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = 0; return cudaSuccess; }
inline cudaError_t cudaStreamCreate(cudaStream_t* s) { *s = 0; return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = 0; return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = 0; return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = 0) { return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }   // the emulator executes in issue order
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.0f; return cudaSuccess; }
inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
inline cudaError_t cudaDeviceGetPCIBusId(char* s, int len, int) {   // no such device: the host pool then stays unbound
  if (len > 0) s[0] = 0;
  return cudaSuccess;
}
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
/* two "SMs", one resident CTA each: persistent kernels get a grid of 2, the second CTA finds the queue drained */
inline cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr, int) { *v = 2; return cudaSuccess; }
/* keyed by the kernel's address, as layout.cu::persistent_grid and the launch rewrite of build_emu.py both pass it */
template <typename K>
inline cudaError_t cudaFuncSetAttribute(K kernel, cudaFuncAttribute attr, int value) {
  if (attr != cudaFuncAttributeMaxDynamicSharedMemorySize) return cudaErrorInvalidValue;
  return simt_emu::set_max_dyn_smem(reinterpret_cast<const void*>(kernel), value);
}
template <typename K>
inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, K, int, size_t) { *n = 1; return cudaSuccess; }

#endif

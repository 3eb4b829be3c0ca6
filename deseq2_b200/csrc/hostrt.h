// hostrt.h -- host-side runtime of the HOST entry points (capi.cu): what sits between R's pageable column-major
// buffers and the device.  Nothing here touches CUDA except one PCI-bus-id query; it is plain C++17 + pthreads.
//
//   Pool        persistent worker threads (no OpenMP: an R process may carry its own OpenMP runtime, and torchrun exports
//               OMP_NUM_THREADS=1), bound as a group to the CPUs of the NUMA node the GPU hangs off
//               (/sys/bus/pci/devices/<bus id>/numa_node -> /sys/devices/system/node/nodeK/cpulist, intersected with the
//               process affinity): 8 ranks on a two-socket box otherwise stage through the wrong socket's memory.
//               Recreated after fork() (BiocParallel's multicore back-end forks R workers).
//   hash_elems  128-bit position-dependent content hash, commutative over elements, so the host (column-major, split
//               among threads) and the GPU (gene-major copy) compute the same value; it is what makes the device-side
//               input cache safe (capi.cu): a hit requires every element of the caller's buffer to hash to the value of
//               the resident copy -- not a pointer comparison (R copies the count matrix for each of the three calls of
//               one DESeq() run, and recycles addresses across runs).
#pragma once
#include <pthread.h>
#include <sched.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <unistd.h>
#if defined(__x86_64__) || defined(__i386__)
#include <immintrin.h>
#endif

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#ifndef MADV_POPULATE_WRITE
#define MADV_POPULATE_WRITE 23
#endif

namespace hostrt {

struct Hash128 {
  uint64_t a = 0, b = 0;
  bool operator==(const Hash128& o) const { return a == o.a && b == o.b; }
  void add(const Hash128& o) { a += o.a; b += o.b; }
};

// Content hash of `count` elements of `elem` (4 or 8) bytes whose canonical indices are first_index, first_index + 1, ...
// (the canonical index of entry (i, j) of an n x m matrix is i + n j, its position in R's column-major layout).
// Every element v (zero-extended to 64 bits) is xored with two keys derived from its index, and each keyed word
// x contributes lo32(x) * hi32(x) + swap32(x) to one of two 64-bit accumulators (the NH construction of UMAC / XXH3:
// one 32 x 32 -> 64 bit multiply per word, which SIMD units have -- the 64 x 64 -> 128 bit multiply of round 2's first
// hash ran at 3-4 GB/s per thread and was the critical path of every cache hit with eight ranks on one host).  The
// contributions are SUMMED, so the hash does not depend on the order or grouping in which the elements are visited: the
// host hashes the caller's column-major buffer split among threads, the GPU hashes its gene-major copy
// (layout.cu::hash_gene_major_kernel) -- same value iff same content (up to a 2^-64 accident; the keys are public,
// this is a cache key, not a MAC).
constexpr uint64_t kHashK1 = 0x9E3779B97F4A7C15ull, kHashK2 = 0xD6E8FEB86659FD93ull;
inline void hash_fold(uint64_t v, uint64_t index, uint64_t& a, uint64_t& b) {
  const uint64_t x1 = v ^ ((index + 1) * kHashK1), x2 = v ^ ((index + 1) * kHashK2);
  a += (x1 & 0xffffffffull) * (x1 >> 32) + ((x1 << 32) | (x1 >> 32));
  b += (x2 & 0xffffffffull) * (x2 >> 32) + ((x2 << 32) | (x2 >> 32));
}
inline Hash128 hash_elems_scalar(const unsigned char* s, size_t i, size_t count, int elem, uint64_t first_index, Hash128 h) {
  for (; i < count; i++) {
    uint64_t v;
    if (elem == 8) {
      memcpy(&v, s + 8 * i, 8);
    } else {
      uint32_t w;
      memcpy(&w, s + 4 * i, 4);
      v = w;
    }
    hash_fold(v, first_index + i, h.a, h.b);
  }
  return h;
}
#if (defined(__x86_64__) || defined(__i386__)) && defined(__GNUC__)
#define B200NB_HASH_AVX2 1
__attribute__((target("avx2"))) inline Hash128 hash_elems_avx2(const unsigned char* s, size_t count, int elem,
                                                                uint64_t first_index) {
  const uint64_t f = first_index + 1;
  __m256i k1 = _mm256_set_epi64x((long long)((f + 3) * kHashK1), (long long)((f + 2) * kHashK1),
                                 (long long)((f + 1) * kHashK1), (long long)(f * kHashK1));
  __m256i k2 = _mm256_set_epi64x((long long)((f + 3) * kHashK2), (long long)((f + 2) * kHashK2),
                                 (long long)((f + 1) * kHashK2), (long long)(f * kHashK2));
  const __m256i s1 = _mm256_set1_epi64x((long long)(4 * kHashK1)), s2 = _mm256_set1_epi64x((long long)(4 * kHashK2));
  __m256i a = _mm256_setzero_si256(), b = _mm256_setzero_si256();
  size_t i = 0;
  for (; i + 4 <= count; i += 4) {
    const __m256i v = (elem == 8) ? _mm256_loadu_si256(reinterpret_cast<const __m256i*>(s + 8 * i))
                                  : _mm256_cvtepu32_epi64(_mm_loadu_si128(reinterpret_cast<const __m128i*>(s + 4 * i)));
    const __m256i x1 = _mm256_xor_si256(v, k1), x2 = _mm256_xor_si256(v, k2);
    a = _mm256_add_epi64(a, _mm256_add_epi64(_mm256_mul_epu32(x1, _mm256_srli_epi64(x1, 32)), _mm256_shuffle_epi32(x1, 0xB1)));
    b = _mm256_add_epi64(b, _mm256_add_epi64(_mm256_mul_epu32(x2, _mm256_srli_epi64(x2, 32)), _mm256_shuffle_epi32(x2, 0xB1)));
    k1 = _mm256_add_epi64(k1, s1);
    k2 = _mm256_add_epi64(k2, s2);
  }
  uint64_t la[4], lb[4];
  _mm256_storeu_si256(reinterpret_cast<__m256i*>(la), a);
  _mm256_storeu_si256(reinterpret_cast<__m256i*>(lb), b);
  Hash128 h;
  h.a = la[0] + la[1] + la[2] + la[3];
  h.b = lb[0] + lb[1] + lb[2] + lb[3];
  return hash_elems_scalar(s, i, count, elem, first_index, h);
}
__attribute__((target("avx512f"))) inline Hash128 hash_elems_avx512(const unsigned char* s, size_t count, int elem,
                                                                    uint64_t first_index) {
  const uint64_t f = first_index + 1;
  uint64_t i1[8], i2[8];
  for (int l = 0; l < 8; l++) {
    i1[l] = (f + l) * kHashK1;
    i2[l] = (f + l) * kHashK2;
  }
  __m512i k1 = _mm512_loadu_si512(i1), k2 = _mm512_loadu_si512(i2);
  const __m512i s1 = _mm512_set1_epi64((long long)(8 * kHashK1)), s2 = _mm512_set1_epi64((long long)(8 * kHashK2));
  __m512i a = _mm512_setzero_si512(), b = _mm512_setzero_si512();
  size_t i = 0;
  for (; i + 8 <= count; i += 8) {
    const __m512i v = (elem == 8) ? _mm512_loadu_si512(s + 8 * i)
                                  : _mm512_cvtepu32_epi64(_mm256_loadu_si256(reinterpret_cast<const __m256i*>(s + 4 * i)));
    const __m512i x1 = _mm512_xor_si512(v, k1), x2 = _mm512_xor_si512(v, k2);
    a = _mm512_add_epi64(a, _mm512_add_epi64(_mm512_mul_epu32(x1, _mm512_srli_epi64(x1, 32)), _mm512_rol_epi64(x1, 32)));
    b = _mm512_add_epi64(b, _mm512_add_epi64(_mm512_mul_epu32(x2, _mm512_srli_epi64(x2, 32)), _mm512_rol_epi64(x2, 32)));
    k1 = _mm512_add_epi64(k1, s1);
    k2 = _mm512_add_epi64(k2, s2);
  }
  uint64_t la[8], lb[8];
  _mm512_storeu_si512(la, a);
  _mm512_storeu_si512(lb, b);
  Hash128 h;
  for (int l = 0; l < 8; l++) {
    h.a += la[l];
    h.b += lb[l];
  }
  return hash_elems_scalar(s, i, count, elem, first_index, h);
}
#endif
inline Hash128 hash_elems(const void* p, size_t count, int elem, uint64_t first_index) {
  const unsigned char* s = static_cast<const unsigned char*>(p);
#ifdef B200NB_HASH_AVX2
  static const int isa = __builtin_cpu_supports("avx512f") ? 2 : (__builtin_cpu_supports("avx2") ? 1 : 0);
  if (isa == 2) return hash_elems_avx512(s, count, elem, first_index);
  if (isa == 1) return hash_elems_avx2(s, count, elem, first_index);
#endif
  return hash_elems_scalar(s, 0, count, elem, first_index, Hash128());
}

inline int env_int(const char* name, int dflt, int lo, int hi) {
  const char* e = getenv(name);
  if (!e || !*e) return dflt;
  const int v = atoi(e);
  return v < lo ? lo : (v > hi ? hi : v);
}

// CPUs of NUMA node `node` that the process may run on; empty when unknown
inline std::vector<int> node_cpus(int node) {
  std::vector<int> out;
  if (node < 0) return out;
  char path[128];
  snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
  FILE* f = fopen(path, "r");
  if (!f) return out;
  char buf[4096];
  const bool ok = fgets(buf, sizeof(buf), f) != nullptr;
  fclose(f);
  if (!ok) return out;
  cpu_set_t allowed;
  CPU_ZERO(&allowed);
  if (sched_getaffinity(0, sizeof(allowed), &allowed) != 0) return out;
  for (char* tok = strtok(buf, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
    int lo = 0, hi = 0;
    if (sscanf(tok, "%d-%d", &lo, &hi) == 2) {
    } else if (sscanf(tok, "%d", &lo) == 1) {
      hi = lo;
    } else {
      continue;
    }
    for (int c = lo; c <= hi && c < CPU_SETSIZE; c++)
      if (CPU_ISSET(c, &allowed)) out.push_back(c);
  }
  return out;
}

inline int pci_numa_node(const char* pci_bus_id) {   // "0000:1b:00.0" (any case) -> node, or -1
  if (!pci_bus_id || !*pci_bus_id) return -1;
  std::string id(pci_bus_id);
  for (char& c : id) c = (char)tolower((unsigned char)c);
  const std::string path = "/sys/bus/pci/devices/" + id + "/numa_node";
  FILE* f = fopen(path.c_str(), "r");
  if (!f) return -1;
  int node = -1;
  if (fscanf(f, "%d", &node) != 1) node = -1;
  fclose(f);
  return node;
}

// CPUs the container may burn per scheduling period (cgroup v2 cpu.max, v1 cpu.cfs_quota_us / cfs_period_us), rounded
// up; 0 = no quota.  A process whose runnable (spinning!) threads exceed it is throttled as a whole for the rest of the
// 100 ms period, which leaves holes of tens of ms in the host timeline.
inline int cgroup_cpu_quota() {
  long long q = -1, per = 100000;
  if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
    char a[64] = "";
    if (fscanf(f, "%63s %lld", a, &per) >= 1 && strcmp(a, "max") != 0) q = atoll(a);
    fclose(f);
  } else if (FILE* g = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r")) {
    if (fscanf(g, "%lld", &q) != 1) q = -1;
    fclose(g);
    if (FILE* h = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r")) {
      if (fscanf(h, "%lld", &per) != 1) per = 100000;
      fclose(h);
    }
  }
  if (q <= 0 || per <= 0) return 0;
  return (int)((q + per - 1) / per);
}

inline int affinity_count() {
  cpu_set_t s;
  CPU_ZERO(&s);
  if (sched_getaffinity(0, sizeof(s), &s) != 0) return (int)sysconf(_SC_NPROCESSORS_ONLN);
  return CPU_COUNT(&s);
}

class Pool {
 public:
  // `cpus`: the CPU group the workers are bound to (empty = inherit the caller's affinity)
  Pool(int nthreads, const std::vector<int>& cpus) : nworkers_(nthreads > 1 ? nthreads - 1 : 0), pid_(getpid()), cpus_(cpus) {
    for (int w = 0; w < nworkers_; w++) th_.emplace_back([this, w] { worker(w + 1); });
  }
  ~Pool() {
    if (getpid() != pid_) {   // forked child: the threads do not exist here; do not join what was never cloned
      for (auto& t : th_) t.detach();
      return;
    }
    stop_.store(true, std::memory_order_release);
    gen_.fetch_add(1, std::memory_order_release);
    {
      std::lock_guard<std::mutex> lk(mu_);
      cv_.notify_all();
    }
    for (auto& t : th_) t.join();
  }
  int threads() const { return nworkers_ + 1; }
  pid_t pid() const { return pid_; }
  const std::vector<int>& cpus() const { return cpus_; }

  // f(task) for task in [0, ntasks), dynamically distributed over the workers and the caller; returns when all are done
  template <typename F>
  void parallel_for(size_t ntasks, F&& f) {
    if (ntasks == 0) return;
    if (nworkers_ == 0 || ntasks == 1) {
      for (size_t t = 0; t < ntasks; t++) f(t);
      return;
    }
    auto tramp = [](void* ctx, size_t t) { (*static_cast<typename std::remove_reference<F>::type*>(ctx))(t); };
    // publish the job, then bump the generation (release): a worker that observes the new generation (acquire) sees
    // the job.  Workers that are still spinning pick it up without any lock; sleepers are woken through the condvar.
    call_ = tramp;
    ctx_ = (void*)&f;
    ntasks_ = ntasks;
    next_.store(0, std::memory_order_relaxed);
    running_.store(nworkers_, std::memory_order_relaxed);
    gen_.fetch_add(1);                       // seq_cst: ordered against the sleepers_ read below (Dekker pattern with
    if (sleepers_.load() > 0) {              // the worker's "sleepers_++ ; re-read gen_" before it blocks)
      std::lock_guard<std::mutex> lk(mu_);
      cv_.notify_all();
    }
    for (size_t t; (t = next_.fetch_add(1, std::memory_order_relaxed)) < ntasks;) f(t);
    // wait for every worker to have left this generation (they may not touch `f` afterwards)
    for (long spin = 0; running_.load(std::memory_order_acquire) != 0; spin++) {
      if (spin > 2000) std::this_thread::yield();   // an oversubscribed host: let the straggler run
      else cpu_relax();
    }
  }

 private:
  static void cpu_relax() {
#if defined(__x86_64__) || defined(__i386__)
    __builtin_ia32_pause();
#endif
  }
  void bind_self() {
    if (cpus_.empty()) return;
    cpu_set_t s;
    CPU_ZERO(&s);
    for (int c : cpus_) CPU_SET(c, &s);
    pthread_setaffinity_np(pthread_self(), sizeof(s), &s);   // a group binding (the kernel balances inside the node)
  }
  void worker(int /*id*/) {
    bind_self();
    uint64_t seen = 0;
    for (;;) {
      // Wait for a new generation.  Host calls come in bursts (a staged upload is dozens of back-to-back parallel
      // regions, separated by event waits): poll for ~0.4 ms before going to sleep -- a condvar wake-up per region costs
      // more than the region itself (16 sleepers woken one after the other were measured to quadruple the upload time).
      uint64_t g = gen_.load(std::memory_order_acquire);
      if (g == seen) {
        const auto t0 = std::chrono::steady_clock::now();
        for (long spin = 0; g == seen; spin++) {
          cpu_relax();
          g = gen_.load(std::memory_order_acquire);
          if ((spin & 255) == 255) {
            if (std::chrono::steady_clock::now() - t0 > std::chrono::microseconds(kSpinMicros)) break;
            if (spin > 4096) std::this_thread::yield();   // still polling, but not hogging a CPU somebody may need
          }
        }
      }
      if (g == seen) {
        std::unique_lock<std::mutex> lk(mu_);
        sleepers_.fetch_add(1);
        cv_.wait(lk, [&] { return gen_.load() != seen; });
        sleepers_.fetch_sub(1);
        g = gen_.load(std::memory_order_acquire);
      }
      seen = g;
      if (stop_.load(std::memory_order_acquire)) return;
      void (*call)(void*, size_t) = call_;
      void* ctx = ctx_;
      const size_t nt = ntasks_;
      for (size_t t; (t = next_.fetch_add(1, std::memory_order_relaxed)) < nt;) call(ctx, t);
      running_.fetch_sub(1, std::memory_order_acq_rel);
    }
  }

  static constexpr long kSpinMicros = 400;
  int nworkers_;
  pid_t pid_;
  std::vector<int> cpus_;
  std::vector<std::thread> th_;
  std::mutex mu_;
  std::condition_variable cv_;
  std::atomic<uint64_t> gen_{0};
  std::atomic<size_t> next_{0};
  std::atomic<int> running_{0}, sleepers_{0};
  void (*call_)(void*, size_t) = nullptr;
  void* ctx_ = nullptr;
  size_t ntasks_ = 0;
  std::atomic<bool> stop_{false};
};

}  // namespace hostrt

// capi.cu -- the C ABI of libb200nb.so (declared in include/b200nb.h).
// Host entry points: R-layout pageable buffers -> (content-addressed device cache | pinned staging -> H2D -> device
// transpose to gene-major) -> kernels -> (transpose back) -> D2H through the pinned ring into the caller's result
// buffers.  Device entry points: enqueue only.  No CPU fallback anywhere.
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <math.h>
#include <stdlib.h>
#include <sys/mman.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <initializer_list>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#include "../../include/b200nb.h"
#include "engine.h"
#include "hostrt.h"

namespace {

thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};

int fail(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}

#define CU(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess) return fail("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

std::mutex g_call_mu;    // host entry points are serialised (one workspace / cache / pinned ring per process)
std::mutex g_arena_mu;   // guards the (re)allocation of the shared device arenas below

// ---------------------------------------------------------------- device workspace of the host entry points
// grow-only slots (one set per process; calls are serialised)
enum Slot {
  S_RAW, S_SMALL_IN, S_SMALL_OUT, S_NF, S_H, S_MUO, S_HC, S_SFI, S_RLOG, S_NSLOTS
};
constexpr int kMaxChunks = 8;
struct Workspace {
  void* p[S_NSLOTS] = {};
  size_t bytes[S_NSLOTS] = {};
  cudaStream_t stream = nullptr;     // uploads, layout conversion, downloads
  cudaStream_t compute = nullptr;    // kernels of the row-chunked path (overlap with the next chunk's upload)
  cudaEvent_t up_ev[kMaxChunks] = {}, layout_ev[kMaxChunks] = {}, done_ev = nullptr;
};
Workspace g_ws;

int ws_get(Slot s, size_t bytes, void** out) {
  if (bytes == 0) bytes = 16;
  if (g_ws.bytes[s] < bytes) {
    if (g_ws.p[s]) cudaFree(g_ws.p[s]);
    g_ws.p[s] = nullptr;
    g_ws.bytes[s] = 0;
    size_t want = bytes + bytes / 8;
    CU(cudaMalloc(&g_ws.p[s], want));
    g_ws.bytes[s] = want;
  }
  *out = g_ws.p[s];
  return 0;
}

int ws_stream(cudaStream_t* st) {
  if (!g_ws.stream) CU(cudaStreamCreateWithFlags(&g_ws.stream, cudaStreamNonBlocking));
  *st = g_ws.stream;
  return 0;
}
int ws_compute_stream(cudaStream_t* st) {
  if (!g_ws.compute) {
    CU(cudaStreamCreateWithFlags(&g_ws.compute, cudaStreamNonBlocking));
    for (auto& e : g_ws.up_ev) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    for (auto& e : g_ws.layout_ev) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&g_ws.done_ev, cudaEventDisableTiming));
  }
  *st = g_ws.compute;
  return 0;
}
// Row chunks of a call whose inputs have to be uploaded: the kernels of chunk c run (second stream) while chunk c + 1
// crosses PCIe.  B200NB_CHUNKS=1 disables; default: 4 chunks from 32768 genes, 2 from 16384.
int plan_chunks(int n) {
  const int forced = hostrt::env_int("B200NB_CHUNKS", 0, 0, kMaxChunks);   // read per call: tests toggle it
  if (forced) return n >= 2 * forced ? forced : 1;
  return n >= 32768 ? 4 : (n >= 16384 ? 2 : 1);
}

// ---------------------------------------------------------------- host worker pool (hostrt.h)
// B200NB_HOST_THREADS (default: see below); B200NB_NUMA_BIND=0
// keeps the workers on the caller's affinity mask instead of the GPU's node.
std::unique_ptr<hostrt::Pool> g_pool;
hostrt::Pool& pool() {
  if (!g_pool || g_pool->pid() != getpid()) {
    if (g_pool) (void)g_pool.release();   // forked child: the parent's threads are not ours to join
    std::vector<int> cpus;
    if (hostrt::env_int("B200NB_NUMA_BIND", 1, 0, 1)) {
      int dev = 0;
      char bus[64] = "";
      if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetPCIBusId(bus, sizeof(bus), dev) == cudaSuccess)
        cpus = hostrt::node_cpus(hostrt::pci_numa_node(bus));
    }
    // default: up to 16 threads, but no more than this process's share of the PHYSICAL cores it may use: the workers
    // spin between the parallel regions of one call, and 8 ranks x 16 spinning threads on a 2 x 32-core box would fight
    // each other (LOCAL_WORLD_SIZE is exported by torchrun; ranks spread over the NUMA nodes like their GPUs)
    const int avail = cpus.empty() ? hostrt::affinity_count() : (int)cpus.size();
    const int local_ranks = hostrt::env_int("LOCAL_WORLD_SIZE", 1, 1, 64);
    const int ranks_here = cpus.empty() ? local_ranks : (local_ranks + 1) / 2;
    int dflt = avail / 2 / (ranks_here > 0 ? ranks_here : 1);
    // ... and no more than the container's CPU quota leaves after the calling thread and the driver's helper threads
    // (the quota is shared by every rank of the container)
    const int quota = hostrt::cgroup_cpu_quota();
    if (quota > 0) {
      const int share = quota / local_ranks - 2;
      if (dflt > share) dflt = share;
    }
    if (dflt > 16) dflt = 16;
    if (dflt < 2) dflt = avail >= 2 ? 2 : 1;
    g_pool.reset(new hostrt::Pool(hostrt::env_int("B200NB_HOST_THREADS", dflt, 1, 128), cpus));
  }
  return *g_pool;
}

// traffic / cache statistics of the host entry points (b200nb_host_stats)
std::atomic<long long> g_h2d_bytes{0}, g_d2h_bytes{0}, g_cache_hits{0}, g_cache_misses{0}, g_cache_hit_bytes{0},
    g_hashed_bytes{0};

// ---------------------------------------------------------------- pinned staging ring
// R hands over ordinary (pageable) memory; cudaMemcpy from pageable memory is slow.  A ring of
// pinned buffers filled by the pool while the previous buffer is in flight reaches PCIe speed.
// Size of one ring buffer and of one pool task.  One rank per host: 8 MB buffers (fewest synchronisations).  Several
// ranks per host: the four buffers of every rank should stay resident in the shared last-level cache between the
// staging copy and the DMA that reads them -- so 4 MB from two local ranks, 2 MB from four.
// B200NB_STAGE_KB / B200NB_STAGE_BLOCK_KB override (read once, when the library loads).
static size_t default_stage_kb() {
  const int local_ranks = hostrt::env_int("LOCAL_WORLD_SIZE", 1, 1, 64);
  return local_ranks >= 4 ? 2048 : (local_ranks >= 2 ? 4096 : 8192);
}
const size_t kStageChunk = (size_t)hostrt::env_int("B200NB_STAGE_KB", (int)default_stage_kb(), 64, 262144) << 10;
constexpr int kStageRing = 4;
const size_t kBlock = (size_t)hostrt::env_int("B200NB_STAGE_BLOCK_KB", (int)(default_stage_kb() / 16), 16, 65536) << 10;   // unit of work of one pool task
struct Staging {
  void* buf[kStageRing] = {};
  cudaEvent_t ev[kStageRing] = {};
  void* small = nullptr;        // pinned scratch for the packed small vectors (grow-only)
  size_t small_bytes = 0;
  bool ready = false;
};
Staging g_stage;
int stage_init() {
  if (g_stage.ready) return 0;
  for (int i = 0; i < kStageRing; i++) {
    CU(cudaHostAlloc(&g_stage.buf[i], kStageChunk, cudaHostAllocDefault));
    CU(cudaEventCreateWithFlags(&g_stage.ev[i], cudaEventDisableTiming));
  }
  g_stage.ready = true;
  return 0;
}
int stage_small(size_t bytes, void** out) {
  if (g_stage.small_bytes < bytes) {
    if (g_stage.small) cudaFreeHost(g_stage.small);
    g_stage.small = nullptr;
    g_stage.small_bytes = 0;
    const size_t want = bytes + bytes / 4 + 4096;
    CU(cudaHostAlloc(&g_stage.small, want, cudaHostAllocDefault));
    g_stage.small_bytes = want;
  }
  *out = g_stage.small;
  return 0;
}

void par_memcpy(void* dst, const void* src, size_t bytes) {
  if (bytes < (1u << 20)) {
    memcpy(dst, src, bytes);
    return;
  }
  const size_t nb = (bytes + kBlock - 1) / kBlock;
  pool().parallel_for(nb, [&](size_t b) {
    const size_t lo = b * kBlock, hi = (lo + kBlock < bytes) ? lo + kBlock : bytes;
    memcpy(static_cast<char*>(dst) + lo, static_cast<const char*>(src) + lo, hi - lo);
  });
}

// content hash of a column-major host matrix (elements of `elem` bytes, canonical index = position), by the pool
hostrt::Hash128 par_hash(const void* src, size_t bytes, int elem) {
  const size_t nb = (bytes + kBlock - 1) / kBlock;
  std::vector<hostrt::Hash128> part(nb);
  pool().parallel_for(nb, [&](size_t b) {
    const size_t lo = b * kBlock, hi = (lo + kBlock < bytes) ? lo + kBlock : bytes;
    part[b] = hostrt::hash_elems(static_cast<const char*>(src) + lo, (hi - lo) / elem, elem, lo / elem);
  });
  hostrt::Hash128 h;
  for (const auto& q : part) h.add(q);
  g_hashed_bytes += (long long)bytes;
  return h;
}

// wall time the calling thread spent (a) copying into the pinned ring, (b) waiting for ring slots / DMA (HOST_TIMING)
std::atomic<long long> g_stage_copy_us{0}, g_stage_wait_us{0};
static inline long long now_us() {
  return std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// pageable host -> device through the pinned ring.  The ring position persists across transfers and a slot is only
// waited for when it is about to be refilled, so back-to-back uploads (y, then mu) keep the DMA engine busy; every host
// entry point ends with a stream synchronisation, which is what finally drains the ring.
int g_ring_pos = 0;
static int ring_next_slot() {
  const int b = g_ring_pos % kStageRing;
  g_ring_pos++;
  return b;
}
int h2d_staged(void* dst, const void* src, size_t bytes, cudaStream_t st) {
  if (bytes == 0) return 0;
  if (stage_init()) return 1;
  for (size_t off = 0; off < bytes;) {
    const int b = ring_next_slot();
    const size_t len = (bytes - off < kStageChunk) ? bytes - off : kStageChunk;
    const long long t0 = now_us();
    CU(cudaEventSynchronize(g_stage.ev[b]));   // returns at once for a slot that is not in flight
    const long long t1 = now_us();
    par_memcpy(g_stage.buf[b], static_cast<const char*>(src) + off, len);
    const long long t2 = now_us();
    g_stage_wait_us += t1 - t0;
    g_stage_copy_us += t2 - t1;
    CU(cudaMemcpyAsync(static_cast<char*>(dst) + off, g_stage.buf[b], len, cudaMemcpyHostToDevice, st));
    CU(cudaEventRecord(g_stage.ev[b], st));
    off += len;
  }
  g_h2d_bytes += (long long)bytes;
  return 0;
}

// Rows [g0, g0 + gc) of a column-major host matrix with n_total rows -> a contiguous column-major gc x m block on the
// device, staged in batches of whole column segments (one pool task per segment).
int h2d_rows(void* dst, const void* host, size_t n_total, size_t g0, size_t gc, int m, int elem, cudaStream_t st) {
  if (gc == n_total) return h2d_staged(dst, host, gc * m * elem, st);
  if (gc == 0) return 0;
  if (stage_init()) return 1;
  const size_t col = gc * elem;
  const char* src = static_cast<const char*>(host);
  if (col > kStageChunk) {   // a single column segment exceeds a ring buffer: column by column
    for (int j = 0; j < m; j++)
      if (h2d_staged(static_cast<char*>(dst) + (size_t)j * col, src + ((size_t)j * n_total + g0) * elem, col, st)) return 1;
    return 0;
  }
  const int cpc = (int)(kStageChunk / col);   // whole column segments per ring buffer (>= 1)
  for (int j = 0; j < m;) {
    const int b = ring_next_slot();
    const int nc = (m - j < cpc) ? m - j : cpc;
    const long long t0 = now_us();
    CU(cudaEventSynchronize(g_stage.ev[b]));
    const long long t1 = now_us();
    char* pin = static_cast<char*>(g_stage.buf[b]);
    pool().parallel_for((size_t)nc, [&](size_t c) {
      memcpy(pin + c * col, src + ((size_t)(j + (int)c) * n_total + g0) * elem, col);
    });
    const long long t2 = now_us();
    g_stage_wait_us += t1 - t0;
    g_stage_copy_us += t2 - t1;
    CU(cudaMemcpyAsync(static_cast<char*>(dst) + (size_t)j * col, pin, (size_t)nc * col, cudaMemcpyHostToDevice, st));
    CU(cudaEventRecord(g_stage.ev[b], st));
    j += nc;
  }
  g_h2d_bytes += (long long)(col * m);
  return 0;
}

// ---------------------------------------------------------------- pinned result memory (b200nb_host_alloc)
// A result matrix that the caller allocates with b200nb_host_alloc lives in page-locked memory: the device-to-host copy
// is then ONE DMA straight into it -- no staging ring, no scatter by host threads and, above all, no first-touch page
// faults (a freshly malloc'ed 40 MB hat-diagonal matrix costs milliseconds of faults, more than the kernels).
// Blocks are pooled: b200nb_host_free returns them for reuse; the pool keeps at most B200NB_PINNED_POOL_MB (default
// 1024) of idle blocks.  R can place the REALSXP itself there through allocVector3's custom allocator (r_shim/).
struct PinBlock {
  void* p;
  size_t cap;
  bool in_use;
};
std::vector<PinBlock> g_pin;
std::mutex g_pin_mu;
bool pinned_contains(const void* p, size_t bytes) {
  std::lock_guard<std::mutex> lk(g_pin_mu);
  const char* q = static_cast<const char*>(p);
  for (const auto& b : g_pin)
    if (b.in_use && q >= static_cast<const char*>(b.p) && q + bytes <= static_cast<const char*>(b.p) + b.cap) return true;
  return false;
}

// a page-locked destination (b200nb_host_alloc): enqueue ONE DMA and return true without waiting; false = not pinned
int d2h_async_if_pinned(void* dst, const void* src, size_t bytes, cudaStream_t st, bool* done) {
  *done = false;
  if (bytes == 0 || !pinned_contains(dst, bytes)) return 0;
  CU(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st));
  g_d2h_bytes += (long long)bytes;
  *done = true;
  return 0;
}

// device -> pageable host through the pinned ring; synchronous on return
int d2h_staged(void* dst, const void* src, size_t bytes, cudaStream_t st) {
  if (bytes == 0) return 0;
  if (pinned_contains(dst, bytes)) {   // the caller's buffer is page-locked (b200nb_host_alloc): one DMA, no staging
    CU(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    g_d2h_bytes += (long long)bytes;
    return 0;
  }
  if (stage_init()) return 1;
  const size_t nchunk = (bytes + kStageChunk - 1) / kStageChunk;
  auto issue = [&](size_t k) -> int {
    const int b = (int)(k % kStageRing);
    const size_t off = k * kStageChunk;
    const size_t len = (bytes - off < kStageChunk) ? bytes - off : kStageChunk;
    // (an upload of this call may still be reading the slot: same stream, so the copy below is ordered after it)
    CU(cudaMemcpyAsync(g_stage.buf[b], static_cast<const char*>(src) + off, len, cudaMemcpyDeviceToHost, st));
    CU(cudaEventRecord(g_stage.ev[b], st));
    return 0;
  };
  for (size_t k = 0; k < nchunk && k < (size_t)kStageRing - 1; k++)
    if (issue(k)) return 1;
  for (size_t k = 0; k < nchunk; k++) {
    if (k + kStageRing - 1 < nchunk && issue(k + kStageRing - 1)) return 1;
    const int b = (int)(k % kStageRing);
    const size_t off = k * kStageChunk;
    const size_t len = (bytes - off < kStageChunk) ? bytes - off : kStageChunk;
    CU(cudaEventSynchronize(g_stage.ev[b]));
    par_memcpy(static_cast<char*>(dst) + off, g_stage.buf[b], len);
  }
  g_d2h_bytes += (long long)bytes;
  return 0;
}

// ---------------------------------------------------------------- content-addressed device cache of input matrices
// One DESeq() run hands the SAME count matrix to fitDisp (MLE), fitDisp (MAP) and fitBeta, and the same fitted means to
// both fitDisp calls -- but as fresh R copies (objectNZ <- object[!allZero, ], R/core.R:706, 1016, 1405), so neither
// the pointer nor the SEXP identifies them.  Their CONTENT does: every large input matrix is hashed (128 bit, all
// bytes, by the pool -- a pure read at memory bandwidth, cheaper than staging it through pinned memory and PCIe), and
// a matrix whose (rows, columns, element size, hash) is already resident on the device in gene-major form is not
// uploaded again.  On a miss the hash is computed while the matrix is staged, so it costs no extra pass.  LRU, bounded
// by B200NB_CACHE_MB (default 8192; 0 disables the cache) and kCacheEntries.
constexpr int kCacheEntries = 8;
struct CacheEntry {
  bool valid = false;
  size_t n = 0;
  int m = 0, elem = 0;
  hostrt::Hash128 hash;    // of every element (valid when hash_known)
  bool hash_known = false; // false: the GPU is still computing it / it sits in the pinned slot g_hash_pin[index]
  uint64_t upload_call = 0; // host call (g_call_seq) that uploaded it
  hostrt::Hash128 fprint;  // of ~64 sampled 4 KB blocks: cheap pre-filter before a speculative hit (see Speculation)
  void* dev = nullptr;     // gene-major n x ld
  size_t cap = 0;          // bytes allocated at dev
  uint64_t last_use = 0;
};
CacheEntry g_cache[kCacheEntries];
uint64_t g_cache_clock = 0;
// the hash of a freshly uploaded matrix is computed ON THE DEVICE from its gene-major copy (layout.cu) and lands in a
// pinned slot with the stream synchronisation that ends the uploading call; the host never hashes what it uploads
unsigned long long* g_hash_dev = nullptr;   // kCacheEntries x 2 (device)
unsigned long long* g_hash_pin = nullptr;   // kCacheEntries x 2 (pinned host)
int hash_slots_init() {
  if (g_hash_dev) return 0;
  CU(cudaMalloc(&g_hash_dev, sizeof(unsigned long long) * 2 * kCacheEntries));
  CU(cudaHostAlloc(&g_hash_pin, sizeof(unsigned long long) * 2 * kCacheEntries, cudaHostAllocDefault));
  return 0;
}
// entry's hash, fetching it from the pinned slot the first time (every host call ends with a stream synchronisation,
// so the slot of an entry uploaded by an EARLIER call is final)
uint64_t g_call_seq = 0;   // incremented by every host entry point (under g_call_mu)
const hostrt::Hash128& entry_hash(CacheEntry& e) {
  if (!e.hash_known) {
    if (e.upload_call == g_call_seq && g_ws.stream) cudaStreamSynchronize(g_ws.stream);   // uploaded by THIS call
    const int k = (int)(&e - g_cache);
    e.hash.a = g_hash_pin[2 * k];
    e.hash.b = g_hash_pin[2 * k + 1];
    e.hash_known = true;
  }
  return e.hash;
}
size_t cache_limit_bytes() {
  static const size_t v = (size_t)hostrt::env_int("B200NB_CACHE_MB", 8192, 0, 1 << 20) << 20;
  return v;
}
void cache_clear(bool free_memory) {
  for (auto& e : g_cache) {
    e.valid = false;
    if (free_memory && e.dev) {
      cudaFree(e.dev);
      e.dev = nullptr;
      e.cap = 0;
    }
  }
}

long long ld_for(int m) { return ((long long)m + 3) & ~3LL; }

// ~64 evenly spaced 4 KB blocks (plus the last bytes): a few tens of microseconds on one thread
hostrt::Hash128 fingerprint(const void* host, size_t bytes) {
  const char* s = static_cast<const char*>(host);
  const size_t blk = 4096;
  if (bytes <= 80 * blk) return hostrt::hash_elems(s, bytes / 8, 8, 0);
  hostrt::Hash128 h;
  const size_t nblk = bytes / blk;
  for (int k = 0; k < 64; k++) {
    const size_t b = nblk * k / 64;
    h.add(hostrt::hash_elems(s + b * blk, blk / 8, 8, b * (blk / 8)));
  }
  h.add(hostrt::hash_elems(s + ((bytes - blk) & ~(size_t)7), blk / 8, 8, (bytes - blk) / 8));
  return h;
}

// Speculation: a call whose input looks like a resident matrix (same dimensions, same fingerprint) launches its kernels
// on the resident copy AT ONCE and checks the full content hash of the caller's buffer on the host while the GPU is
// busy; the results are only copied out after every such check has passed.  A failed check (the caller changed a few
// entries in place) costs one wasted launch: the call is redone with plain uploads.
struct Pending {
  CacheEntry* e;
  const void* host;
  size_t bytes;
  int elem;
};
struct CallInputs {
  bool speculate = true;
  std::vector<Pending> pending;
  std::vector<CacheEntry*> filling;   // cache entries this call is uploading into
  std::vector<void*> owned;   // uncached uploads of this call (freed when the call ends)
  bool validate() {           // true when every speculative hit was a real one
    bool ok = true;
    for (const auto& q : pending) {
      const hostrt::Hash128 h = par_hash(q.host, q.bytes, q.elem);
      if (h == entry_hash(*q.e)) {
        g_cache_hits++;
        g_cache_hit_bytes += (long long)q.bytes;
      } else {
        ok = false;
      }
    }
    pending.clear();
    return ok;
  }
  ~CallInputs() {
    for (void* p : owned) cudaFree(p);
  }
};

// One input matrix of a host call: where its gene-major device copy is (or will be).
struct MatIn {
  const void* host = nullptr;
  int n = 0, m = 0, elem = 0;
  void* dev = nullptr;          // gene-major n x ld
  bool resident = false;        // already on the device (verified or speculative hit): nothing to upload
  CacheEntry* fresh = nullptr;  // cache entry being filled by this call (nullptr: uncached allocation owned by the call)
  hostrt::Hash128 fp;
};

// Decide where the matrix comes from: a resident copy (speculatively, see Speculation) or a destination to upload into.
int mat_acquire(MatIn& M, CallInputs& ci) {
  const int n = M.n, m = M.m, elem = M.elem;
  const long long ld = ld_for(m);
  const size_t bytes = (size_t)n * m * elem, dbytes = (size_t)n * ld * elem + 64;
  const bool use_cache = cache_limit_bytes() >= dbytes;
  if (use_cache) {
    if (hash_slots_init()) return 1;
    M.fp = fingerprint(M.host, bytes);
    CacheEntry* cand = nullptr;
    for (auto& e : g_cache)
      if (e.valid && e.n == (size_t)n && e.m == m && e.elem == elem && e.fprint == M.fp &&
          (!cand || e.last_use > cand->last_use))
        cand = &e;
    if (cand && ci.speculate) {
      cand->last_use = ++g_cache_clock;
      ci.pending.push_back({cand, M.host, bytes, elem});
      M.dev = cand->dev;
      M.resident = true;
      return 0;
    }
    if (cand) {
      const hostrt::Hash128 h = par_hash(M.host, bytes, elem);
      for (auto& e : g_cache)
        if (e.valid && e.n == (size_t)n && e.m == m && e.elem == elem && entry_hash(e) == h) {
          e.last_use = ++g_cache_clock;
          g_cache_hits++;
          g_cache_hit_bytes += (long long)bytes;
          M.dev = e.dev;
          M.resident = true;
          return 0;
        }
    }
  }
  // miss: pick the destination (an invalid or the least recently used entry that no pending check of this call refers
  // to; evict while over the byte limit)
  if (use_cache) {
    g_cache_misses++;
    CacheEntry* dst = nullptr;
    auto in_use = [&](const CacheEntry* e) {
      for (const auto& q : ci.pending)
        if (q.e == e) return true;
      for (const CacheEntry* f : ci.filling)
        if (f == e) return true;
      return false;
    };
    for (auto& e : g_cache)
      if (!e.valid && !in_use(&e) && (!dst || e.cap >= dbytes)) dst = &e;
    if (!dst) {
      for (auto& e : g_cache)
        if (!in_use(&e) && (!dst || e.last_use < dst->last_use)) dst = &e;
    }
    if (!dst) return fail("device input cache: no free entry");
    dst->valid = false;
    size_t total = 0;
    for (const auto& e : g_cache) total += (&e == dst) ? 0 : e.cap;
    while (total + dbytes > cache_limit_bytes()) {
      CacheEntry* victim = nullptr;
      for (auto& e : g_cache)
        if (&e != dst && !in_use(&e) && e.cap > 0 && (!victim || e.last_use < victim->last_use)) victim = &e;
      if (!victim) break;
      total -= victim->cap;
      cudaFree(victim->dev);
      victim->dev = nullptr;
      victim->cap = 0;
      victim->valid = false;
    }
    if (dst->cap < dbytes) {
      if (dst->dev) cudaFree(dst->dev);
      dst->dev = nullptr;
      dst->cap = 0;
      CU(cudaMalloc(&dst->dev, dbytes + dbytes / 16));
      dst->cap = dbytes + dbytes / 16;
    }
    M.fresh = dst;
    M.dev = dst->dev;
    ci.filling.push_back(dst);
  } else {
    // cache disabled / matrix larger than the cache: its own allocation, freed when the call ends
    CU(cudaMalloc(&M.dev, dbytes));
    ci.owned.push_back(M.dev);
  }
  return 0;
}

// rows [g0, g0 + gc) of a non-resident matrix: (1) host -> device as a column-major gc x m block at `d_raw` (copy
// engine, stream `up`), (2) conversion to gene-major rows of the device copy (a kernel, stream `ks`).  The two halves
// are separate because in the row-chunked path they run on different streams: a persistent fit kernel occupies every
// SM, so a layout kernel queued on the UPLOAD stream would stall the next chunk's DMA behind the running compute.
int mat_h2d_rows(MatIn& M, size_t g0, size_t gc, void* d_raw, cudaStream_t up) {
  if (M.resident || gc == 0) return 0;
  return h2d_rows(d_raw, M.host, (size_t)M.n, g0, gc, M.m, M.elem, up);
}
int mat_layout_rows(MatIn& M, size_t g0, size_t gc, const void* d_raw, cudaStream_t ks) {
  if (M.resident || gc == 0) return 0;
  const long long ld = ld_for(M.m);
  CU(nb::launch_to_gene_major(d_raw, static_cast<char*>(M.dev) + g0 * (size_t)ld * M.elem, (int)gc, M.m, ld, M.elem, ks));
  g_launches++;
  return 0;
}

// after the last rows: the device computes the content hash of the complete copy and the entry becomes valid
int mat_finish(MatIn& M, cudaStream_t st) {
  if (M.resident || !M.fresh) return 0;
  CacheEntry* dst = M.fresh;
  const int k = (int)(dst - g_cache);
  CU(nb::launch_hash_gene_major(M.dev, M.n, M.m, ld_for(M.m), M.elem, g_hash_dev + 2 * k, st));
  CU(cudaMemcpyAsync(g_hash_pin + 2 * k, g_hash_dev + 2 * k, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  g_launches++;
  dst->valid = true;
  dst->n = (size_t)M.n;
  dst->m = M.m;
  dst->elem = M.elem;
  dst->hash_known = false;
  dst->upload_call = g_call_seq;
  dst->fprint = M.fp;
  dst->last_use = ++g_cache_clock;
  return 0;
}

// Packs small host vectors into one pinned buffer -> one H2D copy; add() returns the device address the piece will have.
struct SmallIn {
  std::vector<std::pair<const void*, size_t>> parts;
  size_t total = 0;
  size_t add(const void* p, size_t bytes) {
    const size_t off = total;
    parts.emplace_back(p, bytes);
    total += (bytes + 15) & ~(size_t)15;
    return off;
  }
  int upload(cudaStream_t st, char** dev_base) {
    void *pin, *dev;
    if (stage_small(total, &pin)) return 1;
    if (ws_get(S_SMALL_IN, total, &dev)) return 1;
    size_t off = 0;
    for (const auto& q : parts) {
      memcpy(static_cast<char*>(pin) + off, q.first, q.second);
      off += (q.second + 15) & ~(size_t)15;
    }
    CU(cudaMemcpyAsync(dev, pin, total, cudaMemcpyHostToDevice, st));
    CU(cudaStreamSynchronize(st));   // the pinned scratch is reused by the packed download of the same call
    g_h2d_bytes += (long long)total;
    *dev_base = static_cast<char*>(dev);
    return 0;
  }
};

// One D2H copy of a packed device region into pinned memory, then scattered to the caller's vectors.
struct SmallOut {
  struct Part { void* host; size_t off, bytes; };
  std::vector<Part> parts;
  size_t total = 0;
  size_t add(void* host, size_t bytes) {
    const size_t off = total;
    parts.push_back({host, off, bytes});
    total += (bytes + 15) & ~(size_t)15;
    return off;
  }
  int device(char** dev_base) {
    void* dev;
    if (ws_get(S_SMALL_OUT, total, &dev)) return 1;
    *dev_base = static_cast<char*>(dev);
    return 0;
  }
  // begin(): enqueue the device -> host copies behind the kernels (no wait).  The host entry points call it BEFORE they
  // verify a speculative cache hit, so the DMA overlaps the host-side hashing; if the verification fails the call is
  // repeated and the caller's buffers are simply written again (they are undefined until the call returns 0).
  bool all_pinned = false;
  void* pin = nullptr;
  int begin(const char* dev_base, cudaStream_t st) {
    all_pinned = true;   // the caller's vectors are page-locked (b200nb_host_alloc): DMA straight into them
    for (const auto& q : parts) all_pinned = all_pinned && (!q.host || pinned_contains(q.host, q.bytes));
    if (all_pinned) {
      for (const auto& q : parts)
        if (q.host) CU(cudaMemcpyAsync(q.host, dev_base + q.off, q.bytes, cudaMemcpyDeviceToHost, st));
      return 0;
    }
    if (stage_small(total, &pin)) return 1;
    CU(cudaMemcpyAsync(pin, dev_base, total, cudaMemcpyDeviceToHost, st));
    return 0;
  }
  int finish(cudaStream_t st) {
    CU(cudaStreamSynchronize(st));
    if (!all_pinned)
      for (const auto& q : parts)
        if (q.host) memcpy(q.host, static_cast<const char*>(pin) + q.off, q.bytes);
    g_d2h_bytes += (long long)total;
    return 0;
  }
  int download(const char* dev_base, cudaStream_t st) { return begin(dev_base, st) || finish(st); }
};

// device-side work-queue counters: a ring of slots, one per launch, so launches in flight on different
// streams never share a counter (a slot is reused only after kRing further launches).
constexpr int kRing = 1024;
unsigned int* g_counters = nullptr;
std::atomic<unsigned int> g_counter_next{0};
int next_counter(unsigned int** out) {
  std::lock_guard<std::mutex> lk(g_arena_mu);
  if (!g_counters) CU(cudaMalloc(&g_counters, sizeof(unsigned int) * kRing));
  *out = g_counters + (g_counter_next.fetch_add(1) % kRing);
  return 0;
}


// ONE device arena cut into a ring of equal slots, one slot per launch in flight (slot reuse after kSlots further
// launches; launches on one stream are ordered).  The arena is (re)allocated only when a call needs a larger slot than
// any before -- a per-slot cudaFree/cudaMalloc was measured to stall the pipeline by up to 80 ms whenever the gene
// count changed, and a lazily allocated ring stalled the first 8 steps of every run.
struct ArenaRing {
  static constexpr int kSlots = 16;
  void* arena = nullptr;
  size_t slot = 0;
  std::atomic<unsigned int> next{0};
  template <class T>
  int take(size_t bytes, T** out) {
    std::lock_guard<std::mutex> lk(g_arena_mu);
    bytes = (bytes + 255) & ~(size_t)255;
    if (slot < bytes) {
      if (arena) {
        CU(cudaDeviceSynchronize());
        CU(cudaFree(arena));
      }
      arena = nullptr;
      slot = 0;
      const size_t want = (bytes + bytes / 2 + 4095) & ~(size_t)4095;
      CU(cudaMalloc(&arena, want * kSlots));
      slot = want;
    }
    *out = reinterpret_cast<T*>(static_cast<char*>(arena) + (size_t)(next.fetch_add(1) % kSlots) * slot);
    return 0;
  }
};
ArenaRing g_scratch_ring;   // fit_disp launches: work queue + per-mode gene lists
ArenaRing g_design_ring;    // analysed designs of the general-p launches (prepare_design)

// ---------------------------------------------------------------- design analysis for the general-p kernels
// Distinct rows of the design matrix (what R/core.R:2450 modelMatrixGroups computes) and a row id per sample.
// <= 32 distinct rows: GROUPED (xg = G x ps); otherwise SAMPLEWISE (xg = all m rows, gid[j] = j).
bool use_generic(int p) {
  static const bool force = getenv("B200NB_FORCE_GENERIC") != nullptr;
  return force || p > nb::kMaxSmallP;
}

// Long rows on the small-p designs too: from m = 400 samples on the segmented general-p kernels (fit_generic_seg.cuh:
// one gene per warp, per-segment sums, 1024-entry factor table) beat the register-resident small-p kernels, whose
// per-sample X'WX accumulation and 256-entry table are sized for short rows (at m = 300 and below the small-p kernels
// win).  Only the device entry points take this route (it fetches the design matrix: one stream sync per call; see
// route_fit); the host entry points keep the small-p kernels, whose launches per row chunk overlap the uploads.
// B200NB_LONG_ROWS=<m> moves the threshold, 0 = off.
bool long_rows(int m, int use_weights) {
  if (use_weights) return false;
  int thr = 400;
  const char* e = getenv("B200NB_LONG_ROWS");
  if (e) thr = atoi(e);
  return thr > 0 && m >= thr;
}

struct DesignDev {
  const double* xg;
  const int* gid;
  int G, grouped;
  int saturated;       // G == p and the distinct rows form an invertible p x p matrix
  double sat_logdet;   // 2 log|det X_g|
  nb::SegLayout seg;   // sorted lane-chunk sample layout (grouped designs with m <= 65535), else seg.pos == nullptr
};
void apply_design(const DesignDev& dd, int use_weights, nb::DispArgs* a) {
  a->xg = dd.xg; a->gid = dd.gid; a->G = dd.G; a->grouped = dd.grouped;
  a->saturated = dd.saturated && !use_weights; a->sat_logdet = dd.sat_logdet;
  a->seg = dd.seg;
}
void apply_design(const DesignDev& dd, nb::BetaArgs* a) {
  a->xg = dd.xg; a->gid = dd.gid; a->G = dd.G; a->grouped = dd.grouped;
  a->seg = dd.seg;
}

// engine.h::SegLayout on the host: samples sorted by group (stable), dealt to the lanes in contiguous chunks
struct SegHost {
  std::vector<unsigned short> pos, inv, seg_end;
  std::vector<unsigned char> gfirst, glo, ghi;
  int kmax = 0;
};
void build_seg_layout(const std::vector<int>& gid, int m, int G, SegHost* h) {
  std::vector<int> order(m);
  {
    std::vector<int> start(G + 1, 0);
    for (int j = 0; j < m; j++) start[gid[j] + 1]++;
    for (int g = 0; g < G; g++) start[g + 1] += start[g];
    for (int j = 0; j < m; j++) order[start[gid[j]]++] = j;
  }
  const int q = m / 32, rem = m % 32;
  h->pos.assign(m, 0);
  h->inv.assign(m, 0);
  h->gfirst.assign(32, 0);
  h->glo.assign(G, 255);
  h->ghi.assign(G, 0);
  std::vector<std::vector<int>> ends(32);
  for (int l = 0; l < 32; l++) {
    const int n_l = q + (l < rem ? 1 : 0);
    const int s0 = l * q + (l < rem ? l : rem);
    for (int i = 0; i < n_l; i++) {
      const int j = order[s0 + i], g = gid[j];
      h->pos[j] = (unsigned short)(i * 32 + l);
      h->inv[i * 32 + l] = (unsigned short)j;
      if (i == 0) h->gfirst[l] = (unsigned char)g;
      if (l < h->glo[g]) h->glo[g] = (unsigned char)l;
      if (l > h->ghi[g]) h->ghi[g] = (unsigned char)l;
      if (i + 1 == n_l || gid[order[s0 + i + 1]] != g) ends[l].push_back(i + 1);
    }
  }
  h->kmax = 1;
  for (int l = 0; l < 32; l++) h->kmax = std::max(h->kmax, (int)ends[l].size());
  h->seg_end.assign((size_t)h->kmax * 32, 0xffff);
  for (int l = 0; l < 32; l++)
    for (size_t r = 0; r < ends[l].size(); r++) h->seg_end[r * 32 + l] = (unsigned short)ends[l][r];
}
// x_host: m x p column-major.  Uploads xg / gid on `st`.
int prepare_design(const double* x_host, int m, int p, cudaStream_t st, DesignDev* out) {
  const int ps = p | 1;
  std::vector<int> gid(m), rep;
  for (int j = 0; j < m; j++) {
    int found = -1;
    for (size_t g = 0; g < rep.size() && found < 0; g++) {
      bool same = true;
      for (int k = 0; k < p && same; k++) same = (x_host[j + (size_t)m * k] == x_host[rep[g] + (size_t)m * k]);
      if (same) found = (int)g;
    }
    if (found < 0) {
      if (rep.size() > 32) break;   // too many distinct rows: samplewise
      found = (int)rep.size();
      rep.push_back(j);
    }
    gid[j] = found;
  }
  const bool grouped = rep.size() <= 32;
  const int rows = grouped ? (int)rep.size() : m;
  std::vector<double> xg((size_t)rows * ps, 0.0);
  for (int r = 0; r < rows; r++) {
    const int j = grouped ? rep[r] : r;
    for (int k = 0; k < p; k++) xg[(size_t)r * ps + k] = x_host[j + (size_t)m * k];
  }
  if (!grouped)
    for (int j = 0; j < m; j++) gid[j] = j;
  // one packed upload: [xg | gid | segment layout (pos, inv, seg_end, gfirst, glo, ghi)]
  const size_t xbytes = xg.size() * sizeof(double), gbytes = (size_t)m * sizeof(int);
  const bool with_seg = grouped && m <= 65535;
  SegHost sh;
  if (with_seg) build_seg_layout(gid, m, (int)rep.size(), &sh);
  auto up16 = [](size_t v) { return (v + 15) & ~(size_t)15; };
  const size_t o_gid = up16(xbytes), o_pos = up16(o_gid + gbytes);
  const size_t o_inv = up16(o_pos + sh.pos.size() * 2), o_end = up16(o_inv + sh.inv.size() * 2);
  const size_t o_gf = up16(o_end + sh.seg_end.size() * 2), o_lo = up16(o_gf + sh.gfirst.size());
  const size_t o_hi = up16(o_lo + sh.glo.size()), need = up16(o_hi + sh.ghi.size());
  std::vector<char> pack(need, 0);
  memcpy(pack.data(), xg.data(), xbytes);
  memcpy(pack.data() + o_gid, gid.data(), gbytes);
  if (with_seg) {
    memcpy(pack.data() + o_pos, sh.pos.data(), sh.pos.size() * 2);
    memcpy(pack.data() + o_inv, sh.inv.data(), sh.inv.size() * 2);
    memcpy(pack.data() + o_end, sh.seg_end.data(), sh.seg_end.size() * 2);
    memcpy(pack.data() + o_gf, sh.gfirst.data(), sh.gfirst.size());
    memcpy(pack.data() + o_lo, sh.glo.data(), sh.glo.size());
    memcpy(pack.data() + o_hi, sh.ghi.data(), sh.ghi.size());
  }
  char* base = nullptr;
  if (g_design_ring.take(need, &base)) return 1;
  // pageable H2D copies are staged before cudaMemcpyAsync returns, so the vector may die at scope exit
  CU(cudaMemcpyAsync(base, pack.data(), need, cudaMemcpyHostToDevice, st));
  CU(cudaStreamSynchronize(st));
  out->xg = reinterpret_cast<const double*>(base);
  out->gid = reinterpret_cast<const int*>(base + o_gid);
  out->seg = nb::SegLayout{};
  if (with_seg) {
    out->seg.pos = reinterpret_cast<const unsigned short*>(base + o_pos);
    out->seg.inv = reinterpret_cast<const unsigned short*>(base + o_inv);
    out->seg.seg_end = reinterpret_cast<const unsigned short*>(base + o_end);
    out->seg.gfirst = reinterpret_cast<const unsigned char*>(base + o_gf);
    out->seg.glo = reinterpret_cast<const unsigned char*>(base + o_lo);
    out->seg.ghi = reinterpret_cast<const unsigned char*>(base + o_hi);
    out->seg.kmax = sh.kmax;
  }
  out->G = grouped ? (int)rep.size() : m;
  out->grouped = grouped ? 1 : 0;
  out->saturated = 0;
  out->sat_logdet = 0.0;
  if (grouped && (int)rep.size() == p) {
    // log|det| of the p x p matrix of distinct rows (partial-pivot LU)
    std::vector<double> a((size_t)p * p);
    for (int r = 0; r < p; r++)
      for (int k = 0; k < p; k++) a[(size_t)r * p + k] = xg[(size_t)r * ps + k];
    double logdet = 0.0;
    bool ok = true;
    for (int c = 0; c < p && ok; c++) {
      int pr = c;
      for (int r = c + 1; r < p; r++)
        if (fabs(a[(size_t)r * p + c]) > fabs(a[(size_t)pr * p + c])) pr = r;
      if (fabs(a[(size_t)pr * p + c]) < 1e-12) { ok = false; break; }
      if (pr != c)
        for (int k = 0; k < p; k++) { double t = a[(size_t)c * p + k]; a[(size_t)c * p + k] = a[(size_t)pr * p + k]; a[(size_t)pr * p + k] = t; }
      logdet += log(fabs(a[(size_t)c * p + c]));
      for (int r = c + 1; r < p; r++) {
        const double f = a[(size_t)r * p + c] / a[(size_t)c * p + c];
        for (int k = c; k < p; k++) a[(size_t)r * p + k] -= f * a[(size_t)c * p + k];
      }
    }
    if (ok) {
      out->saturated = 1;
      out->sat_logdet = 2.0 * logdet;
    }
  }
  return 0;
}

// design matrix given as a DEVICE pointer (the *_dev entry points): fetch it (m*p doubles) and analyse.
// This synchronises `st`; it only happens on the general-p path.
int prepare_design_from_device(const double* x_dev, int m, int p, cudaStream_t st, DesignDev* out) {
  std::vector<double> xh((size_t)m * p);
  CU(cudaMemcpyAsync(xh.data(), x_dev, xh.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return prepare_design(xh.data(), m, p, st, out);
}

// Which launcher fits a fitDisp, fitDispGrid or fitBeta call with n > 0 genes.  The general-p kernels (generic, with
// the analysed design in dd) take p > kMaxSmallP and rows the small-p kernels cannot hold; with allow_long_rows,
// fitDisp and fitBeta also send long unweighted rows there when the design gets a segment layout.  Everything else
// runs on the small-p kernels.  launches: the kernels the chosen launcher starts (b200nb_kernel_launches).
enum FitKind { FIT_DISP, FIT_DISP_GRID, FIT_BETA };
struct FitRoute {
  bool generic = false;
  DesignDev dd;
  int launches = 0;
};
int route_fit(FitKind kind, const double* x_dev, int m, int p, int use_weights, int nf_is_vector, bool allow_long_rows,
              cudaStream_t st, FitRoute* r) {
  const bool fits = kind == FIT_BETA ? nb::fit_beta_smallp_fits(m, p, use_weights, nf_is_vector)
                                     : nb::fit_disp_smallp_fits(m, p, use_weights);
  r->generic = use_generic(p) || !fits;
  if (r->generic || (kind != FIT_DISP_GRID && allow_long_rows && long_rows(m, use_weights))) {
    if (prepare_design_from_device(x_dev, m, p, st, &r->dd)) return 1;
    r->generic = r->generic || r->dd.seg.pos != nullptr;
  }
  // small-p fitDisp: classify [+ bucket sort] + both design variants of the line search; fitDispGrid: one kernel;
  // fitBeta: both design variants
  r->launches = r->generic ? 1 : kind == FIT_DISP ? nb::fit_disp_smallp_launches(m) : kind == FIT_DISP_GRID ? 1 : 2;
  return 0;
}

// The library keeps per-process device state (work-queue arenas, workspace, pinned staging): one process drives one
// GPU, as in the one-process-per-GPU deployment the engine is built for.  A second device in the same process is
// refused loudly instead of silently using buffers that live on the first one.
int g_bound_device = -1;
int check_device() {
  int dev = -1;
  CU(cudaGetDevice(&dev));
  if (g_bound_device < 0) g_bound_device = dev;
  if (dev != g_bound_device)
    return fail("libb200nb is bound to CUDA device %d in this process (current device is %d): use one process per GPU",
                g_bound_device, dev);
  return 0;
}

// Argument checks of the entry points: each returns 0, or 1 with the reason in g_err.  They touch no device, so a bad
// argument is refused before any CUDA call; every entry point calls check_device() itself before its first launch.
int check_dims(int n, int m, int p) {
  if (n < 0 || m < 1 || p < 1) return fail("bad dimensions n=%d m=%d p=%d", n, m, p);
  if (p > nb::kMaxP) return fail("p=%d not supported (max %d design columns)", p, nb::kMaxP);
  return 0;
}

// y_type is a known code (anything else would be read as int32), and y is given when there are rows to read
int check_y(const char* what, const void* y, int y_type, long long n) {
  if (y_type != B200NB_Y_INT32 && y_type != B200NB_Y_F64) return fail("%s: bad y_type %d", what, y_type);
  if (n > 0 && !y) return fail("%s: y == NULL", what);
  return 0;
}

// the row stride `name` of a gene-major matrix: >= m, and a multiple of 4 where the kernels read rows with 16-byte
// vector loads (aligned)
int check_ld(const char* what, const char* name, long long ld, int m, bool aligned) {
  if (ld < m || (aligned && (ld & 3)))
    return fail("%s: %s=%lld must be >= m=%d%s", what, name, ld, m, aligned ? " and a multiple of 4" : "");
  return 0;
}

int check_factors(const char* what, const double* size_factors, const double* nf) {
  if ((size_factors == nullptr) == (nf == nullptr)) return fail("%s: give exactly one of size_factors and nf", what);
  return 0;
}

// the pointers a call with n > 0 rows of work reads or writes
int check_ptrs(const char* what, long long n, std::initializer_list<const void*> ptrs) {
  for (const void* q : ptrs)
    if (n > 0 && !q) return fail("%s: null pointer argument", what);
  return 0;
}

bool finite_pos(double v) { return v > 0.0 && v < HUGE_VAL; }

// B200NB_HOST_TIMING=1: the host entry points print where their wall time goes (hashing + upload incl. layout
// conversion / kernels / download) to stderr; it adds a stream synchronisation between the phases, so it is a
// diagnosis aid, not something to leave on while measuring.
bool host_timing() {
  static const bool on = hostrt::env_int("B200NB_HOST_TIMING", 0, 0, 1) != 0;
  return on;
}
struct PhaseClock {
  std::chrono::steady_clock::time_point t0;
  double ms[3] = {0.0, 0.0, 0.0};
  int phase = 0;
  bool on;
  cudaStream_t st;
  long long h2d0, d2h0, hit0, hashed0, copy0, wait0;
  explicit PhaseClock(cudaStream_t s) : on(host_timing()), st(s) {
    if (on) {
      t0 = std::chrono::steady_clock::now();
      h2d0 = g_h2d_bytes; d2h0 = g_d2h_bytes; hit0 = g_cache_hit_bytes; hashed0 = g_hashed_bytes;
      copy0 = g_stage_copy_us; wait0 = g_stage_wait_us;
    }
  }
  void next() {   // close the current phase
    if (!on || phase > 2) return;
    cudaStreamSynchronize(st);
    const auto t1 = std::chrono::steady_clock::now();
    ms[phase++] = std::chrono::duration<double, std::milli>(t1 - t0).count();
    t0 = t1;
  }
  void report(const char* what, int n) {   // closes the last phase
    next();
    if (on)
      fprintf(stderr, "b200nb timing %s %d genes: hash+upload %.3f ms, kernels %.3f ms, download %.3f ms | H2D %.1f MB, "
                      "D2H %.1f MB, hashed %.1f MB, served from the device cache %.1f MB; upload staging: %.3f ms copying "
                      "into the pinned ring, %.3f ms waiting for ring slots\n", what, n, ms[0], ms[1], ms[2],
              (g_h2d_bytes - h2d0) / 1e6, (g_d2h_bytes - d2h0) / 1e6, (g_hashed_bytes - hashed0) / 1e6,
              (g_cache_hit_bytes - hit0) / 1e6, (g_stage_copy_us - copy0) / 1e3, (g_stage_wait_us - wait0) / 1e3);
  }
};

// The input matrices of a host call: acquires them (mat_acquire), fills the device copies of those that are not
// resident and runs launch_rows(g0, gc, stream) on rows [g0, g0 + gc) of them -- in one piece, or, when a matrix has
// to be uploaded, in `chunks` row chunks whose layout conversion and kernels run on the compute stream while the next
// chunk crosses PCIe.  Then the device hashes the fresh copies (mat_finish).
template <class F>
int upload_and_launch(const std::vector<MatIn*>& mats, CallInputs& ci, int n, int chunks, cudaStream_t st,
                      PhaseClock& clk, F&& launch_rows) {
  bool any_miss = false;
  for (MatIn* M : mats) {
    if (mat_acquire(*M, ci)) return 1;
    any_miss = any_miss || !M->resident;
  }
  const int C = any_miss ? chunks : 1;
  if (C == 1) {
    for (MatIn* M : mats) {
      void* d_raw;
      if (M->resident) continue;
      if (ws_get(S_RAW, (size_t)n * M->m * M->elem, &d_raw) || mat_h2d_rows(*M, 0, n, d_raw, st) ||
          mat_layout_rows(*M, 0, n, d_raw, st))
        return 1;
    }
    clk.next();
    if (launch_rows((size_t)0, n, st)) return 1;
  } else {
    cudaStream_t ks;
    if (ws_compute_stream(&ks)) return 1;
    const size_t gc = (((size_t)n + C - 1) / C + 63) & ~(size_t)63;
    // two sets of raw (column-major) chunk buffers: chunk c + 1 crosses PCIe into one while chunk c is converted
    // from the other
    std::vector<size_t> roff;
    size_t rset = 0;
    for (MatIn* M : mats) {
      roff.push_back(rset);
      rset += (gc * M->m * M->elem + 255) & ~(size_t)255;
    }
    void* rawbase;
    if (ws_get(S_RAW, 2 * rset, &rawbase)) return 1;
    int c = 0;
    for (size_t g0 = 0; g0 < (size_t)n; g0 += gc, c++) {
      const size_t cnt = (g0 + gc <= (size_t)n) ? gc : (size_t)n - g0;
      char* raw = static_cast<char*>(rawbase) + (size_t)(c & 1) * rset;
      if (c >= 2) CU(cudaStreamWaitEvent(st, g_ws.layout_ev[c - 2], 0));   // this buffer set has been consumed
      for (size_t i = 0; i < mats.size(); i++)
        if (mat_h2d_rows(*mats[i], g0, cnt, raw + roff[i], st)) return 1;
      CU(cudaEventRecord(g_ws.up_ev[c], st));
      CU(cudaStreamWaitEvent(ks, g_ws.up_ev[c], 0));
      for (size_t i = 0; i < mats.size(); i++)
        if (mat_layout_rows(*mats[i], g0, cnt, raw + roff[i], ks)) return 1;
      CU(cudaEventRecord(g_ws.layout_ev[c], ks));
      if (launch_rows(g0, (int)cnt, ks)) return 1;
    }
    CU(cudaEventRecord(g_ws.done_ev, ks));
    CU(cudaStreamWaitEvent(st, g_ws.done_ev, 0));   // hashing and the download below follow the last kernel
    clk.next();
  }
  for (MatIn* M : mats)
    if (mat_finish(*M, st)) return 1;
  return 0;
}

bool speculation_on() {
  static const bool on = hostrt::env_int("B200NB_SPECULATE", 1, 0, 1) != 0;
  return on;
}

// The protocol of the host entry points.  Calls are serialised and numbered (g_call_seq).  Each runs at most twice:
// attempt 0 may launch on resident copies of its input matrices before their content has been verified
// (CallInputs::validate, overlapped with the kernels); if a verification fails the attempt returns kRetry, its launch
// is discarded and attempt 1 repeats the call with verified inputs only.  B200NB_SPECULATE=0 skips attempt 0's mode.
constexpr int kRetry = 2;
template <class F>
int host_call(const char* name, int n, F&& attempt) {
  std::lock_guard<std::mutex> lk(g_call_mu);
  g_call_seq++;
  cudaStream_t st;
  if (ws_stream(&st)) return 1;
  for (int k = 0; k < 2; k++) {
    PhaseClock clk(st);
    CallInputs ci;
    ci.speculate = (k == 0) && speculation_on();
    const int rc = attempt(ci, clk, st);
    if (rc == 0) clk.report(name, n);
    if (rc != kRetry) return rc;
    CU(cudaStreamSynchronize(st));
  }
  return fail("%s: input verification failed twice", name);
}

}  // namespace

extern "C" {

const char* b200nb_last_error(void) { return g_err; }
const char* b200nb_version(void) { return "b200nb 0.2 (sm_90a)"; }
long long b200nb_kernel_launches(void) { return g_launches.load(); }

int b200nb_device_count(void) {
  int c = 0;
  if (cudaGetDeviceCount(&c) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return c;
}

void* b200nb_host_alloc(size_t bytes) {
  if (bytes == 0) bytes = 16;
  std::lock_guard<std::mutex> lk(g_pin_mu);
  PinBlock* best = nullptr;
  for (auto& b : g_pin)
    if (!b.in_use && b.cap >= bytes && b.cap <= 2 * bytes + (1u << 20) && (!best || b.cap < best->cap)) best = &b;
  if (best) {
    best->in_use = true;
    return best->p;
  }
  const size_t cap = (bytes + ((size_t)2 << 20) - 1) & ~(((size_t)2 << 20) - 1);
  void* p = nullptr;
  if (cudaHostAlloc(&p, cap, cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;   // the caller falls back to ordinary memory
  }
  g_pin.push_back({p, cap, true});
  return p;
}

void b200nb_host_free(void* p) {
  if (!p) return;
  std::lock_guard<std::mutex> lk(g_pin_mu);
  size_t idle = 0;
  for (auto& b : g_pin) {
    if (b.p == p) b.in_use = false;
    if (!b.in_use) idle += b.cap;
  }
  const size_t limit = (size_t)hostrt::env_int("B200NB_PINNED_POOL_MB", 1024, 0, 1 << 20) << 20;
  for (size_t i = g_pin.size(); i-- > 0 && idle > limit;)
    if (!g_pin[i].in_use) {
      idle -= g_pin[i].cap;
      cudaFreeHost(g_pin[i].p);
      g_pin.erase(g_pin.begin() + (long)i);
    }
}

void b200nb_cache_clear(void) {
  std::lock_guard<std::mutex> lk(g_call_mu);
  cache_clear(false);
}

int b200nb_test_hash(const void* p, long long count, int elem, long long first_index, unsigned long long* out2) {
  if ((elem != 4 && elem != 8) || count < 0) return fail("b200nb_test_hash: bad arguments");
  const unsigned char* s = static_cast<const unsigned char*>(p);
  const hostrt::Hash128 ref = hostrt::hash_elems_scalar(s, 0, (size_t)count, elem, (uint64_t)first_index, hostrt::Hash128());
  int variants = 1;
  bool ok = hostrt::hash_elems(s, (size_t)count, elem, (uint64_t)first_index) == ref;   // the dispatched one
#ifdef B200NB_HASH_AVX2
  if (__builtin_cpu_supports("avx2")) {
    variants++;
    ok = ok && hostrt::hash_elems_avx2(s, (size_t)count, elem, (uint64_t)first_index) == ref;
  }
  if (__builtin_cpu_supports("avx512f")) {
    variants++;
    ok = ok && hostrt::hash_elems_avx512(s, (size_t)count, elem, (uint64_t)first_index) == ref;
  }
#endif
  out2[0] = ref.a;
  out2[1] = ref.b;
  return ok ? variants : -1;
}

int b200nb_host_stats(long long* out, int n) {
  const long long v[6] = {g_h2d_bytes.load(), g_d2h_bytes.load(), g_cache_hits.load(), g_cache_misses.load(),
                          g_cache_hit_bytes.load(), g_hashed_bytes.load()};
  for (int i = 0; i < n && i < 6; i++) out[i] = v[i];
  return 6;
}

void b200nb_release_workspace(void) {
  std::lock_guard<std::mutex> lk(g_call_mu);
  cache_clear(true);
  for (int s = 0; s < S_NSLOTS; s++) {
    if (g_ws.p[s]) cudaFree(g_ws.p[s]);
    g_ws.p[s] = nullptr;
    g_ws.bytes[s] = 0;
  }
  if (g_stage.ready) {
    for (int i = 0; i < kStageRing; i++) {
      cudaFreeHost(g_stage.buf[i]);
      cudaEventDestroy(g_stage.ev[i]);
      g_stage.buf[i] = nullptr;
    }
    g_stage.ready = false;
  }
  if (g_stage.small) cudaFreeHost(g_stage.small);
  g_stage.small = nullptr;
  g_stage.small_bytes = 0;
}

/* ------------------------------------------------------------------ device entry points */

// fitDisp or fitDispGrid (a.grid) on the kernels route_fit picks; allow_long_rows: see route_fit
static int launch_disp(nb::DispArgs& a, bool allow_long_rows, cudaStream_t st) {
  if (a.n == 0) return 0;
  FitRoute r;
  if (check_device() || g_scratch_ring.take(nb::disp_scratch_bytes(a.n), &a.scratch) ||
      route_fit(a.grid ? FIT_DISP_GRID : FIT_DISP, a.x, a.m, a.p, a.use_weights, 0, allow_long_rows, st, &r))
    return 1;
  if (r.generic) apply_design(r.dd, a.use_weights, &a);
  CU(r.generic ? nb::launch_fit_disp_generic(a, st) : nb::launch_fit_disp(a, st));
  g_launches += r.launches;
  return 0;
}

// b200nb_fit_disp_dev and b200nb_fit_beta_dev after their argument checks
static int fit_disp_dev(const void* y, int y_type, const double* x, const double* mu_hat, const double* log_alpha,
                        const double* log_alpha_prior_mean, double log_alpha_prior_sigmasq, double min_log_alpha,
                        double kappa_0, double tol, int maxit, int use_prior, const double* weights,
                        int use_weights, double weight_threshold, int use_cr, int n, int m, int p, long long ld,
                        double* out_log_alpha, int32_t* out_iter, int32_t* out_iter_accept,
                        double* out_last_change, double* out_initial_lp, double* out_initial_dlp,
                        double* out_last_lp, double* out_last_dlp, double* out_last_d2lp, cudaStream_t st,
                        bool allow_long_rows) {
  nb::DispArgs a{};
  a.y = y; a.y_is_f64 = (y_type == B200NB_Y_F64); a.mu = mu_hat; a.w = use_weights ? weights : nullptr; a.x = x;
  a.log_alpha_in = log_alpha; a.prior_mean = log_alpha_prior_mean;
  a.prior_sigmasq = log_alpha_prior_sigmasq; a.min_log_alpha = min_log_alpha; a.kappa_0 = kappa_0; a.tol = tol;
  a.maxit = maxit; a.use_prior = use_prior; a.use_weights = use_weights; a.use_cr = use_cr;
  a.weight_threshold = weight_threshold; a.n = n; a.m = m; a.p = p; a.ld = ld;
  a.log_alpha = out_log_alpha; a.iter = out_iter; a.iter_accept = out_iter_accept; a.last_change = out_last_change;
  a.initial_lp = out_initial_lp; a.initial_dlp = out_initial_dlp; a.last_lp = out_last_lp; a.last_dlp = out_last_dlp;
  a.last_d2lp = out_last_d2lp; a.grid = nullptr; a.grid_n = 0;
  return launch_disp(a, allow_long_rows, st);
}

static int fit_beta_dev(const void* y, int y_type, const double* x, const double* nf, int nf_is_vector,
                        const double* alpha_hat, const double* contrast, const double* beta_mat,
                        const double* lambda, const double* weights, int use_weights, double tol, int maxit,
                        int use_qr, double minmu, int n, int m, int p, long long ld, double* out_beta_mat,
                        double* out_beta_var_mat, double* out_iter, double* out_hat_diagonals,
                        double* out_contrast_num, double* out_contrast_denom, double* out_deviance, double* out_mu,
                        cudaStream_t st, bool allow_long_rows) {
  unsigned int* ctr;
  if ((n > 0 && check_device()) || next_counter(&ctr)) return 1;
  nb::BetaArgs a{};
  a.y = y; a.y_is_f64 = (y_type == B200NB_Y_F64); a.nf = nf; a.nf_is_vector = nf_is_vector;
  a.w = use_weights ? weights : nullptr; a.x = x; a.alpha_hat = alpha_hat; a.contrast = contrast; a.beta_in = beta_mat;
  a.lambda = lambda; a.use_weights = use_weights; a.tol = tol; a.maxit = maxit; a.use_qr = use_qr; a.minmu = minmu;
  a.n = n; a.m = m; a.p = p; a.ld = ld; a.beta_out = out_beta_mat; a.beta_var = out_beta_var_mat; a.iter = out_iter;
  a.hat_diag = out_hat_diagonals; a.mu_out = out_mu; a.contrast_num = out_contrast_num;
  a.contrast_denom = out_contrast_denom; a.deviance = out_deviance; a.counter = ctr;
  if (n == 0) return 0;
  FitRoute r;
  if (route_fit(FIT_BETA, x, m, p, use_weights, nf_is_vector, allow_long_rows, st, &r)) return 1;
  if (r.generic) apply_design(r.dd, &a);
  CU(r.generic ? nb::launch_fit_beta_generic(a, st) : nb::launch_fit_beta(a, st));
  g_launches += r.launches;
  return 0;
}

int b200nb_fit_disp_dev(const void* y, int y_type, const double* x, const double* mu_hat, const double* log_alpha,
                        const double* log_alpha_prior_mean, double log_alpha_prior_sigmasq, double min_log_alpha,
                        double kappa_0, double tol, int maxit, int use_prior, const double* weights,
                        int use_weights, double weight_threshold, int use_cr, int n, int m, int p, long long ld,
                        double* out_log_alpha, int32_t* out_iter, int32_t* out_iter_accept,
                        double* out_last_change, double* out_initial_lp, double* out_initial_dlp,
                        double* out_last_lp, double* out_last_dlp, double* out_last_d2lp, void* stream) {
  if (check_dims(n, m, p) || check_y("fit_disp", y, y_type, n) || check_ld("fit_disp", "ld", ld, m, true)) return 1;
  if (use_weights && !weights) return fail("use_weights set but weights == NULL");
  if (check_ptrs("fit_disp", n, {x, mu_hat, log_alpha, log_alpha_prior_mean, out_log_alpha, out_iter, out_iter_accept,
                                 out_last_change, out_initial_lp, out_initial_dlp, out_last_lp, out_last_dlp,
                                 out_last_d2lp}))
    return 1;
  return fit_disp_dev(y, y_type, x, mu_hat, log_alpha, log_alpha_prior_mean, log_alpha_prior_sigmasq, min_log_alpha,
                      kappa_0, tol, maxit, use_prior, weights, use_weights, weight_threshold, use_cr, n, m, p, ld,
                      out_log_alpha, out_iter, out_iter_accept, out_last_change, out_initial_lp, out_initial_dlp,
                      out_last_lp, out_last_dlp, out_last_d2lp, (cudaStream_t)stream, true);
}

int b200nb_fit_disp_grid_dev(const void* y, int y_type, const double* x, const double* mu_hat,
                             const double* disp_grid, int disp_grid_n, const double* log_alpha_prior_mean,
                             double log_alpha_prior_sigmasq, int use_prior, const double* weights, int use_weights,
                             double weight_threshold, int use_cr, int n, int m, int p, long long ld,
                             double* out_log_alpha, void* stream) {
  if (check_dims(n, m, p) || check_y("fit_disp_grid", y, y_type, n) || check_ld("fit_disp_grid", "ld", ld, m, true) ||
      check_ptrs("fit_disp_grid", n, {x, mu_hat, disp_grid, log_alpha_prior_mean, out_log_alpha}))
    return 1;
  if (disp_grid_n < 2) return fail("disp_grid needs at least 2 points");
  if (use_weights && !weights) return fail("use_weights set but weights == NULL");
  nb::DispArgs a{};
  a.y = y; a.y_is_f64 = (y_type == B200NB_Y_F64); a.mu = mu_hat; a.w = use_weights ? weights : nullptr; a.x = x;
  a.log_alpha_in = nullptr; a.prior_mean = log_alpha_prior_mean; a.prior_sigmasq = log_alpha_prior_sigmasq;
  a.use_prior = use_prior; a.use_weights = use_weights; a.use_cr = use_cr; a.weight_threshold = weight_threshold;
  a.n = n; a.m = m; a.p = p; a.ld = ld; a.log_alpha = out_log_alpha; a.grid = disp_grid; a.grid_n = disp_grid_n;
  return launch_disp(a, false, (cudaStream_t)stream);
}

int b200nb_fit_beta_dev(const void* y, int y_type, const double* x, const double* nf, int nf_is_vector,
                        const double* alpha_hat, const double* contrast, const double* beta_mat,
                        const double* lambda, const double* weights, int use_weights, double tol, int maxit,
                        int use_qr, double minmu, int n, int m, int p, long long ld, double* out_beta_mat,
                        double* out_beta_var_mat, double* out_iter, double* out_hat_diagonals,
                        double* out_contrast_num, double* out_contrast_denom, double* out_deviance, double* out_mu,
                        void* stream) {
  if (check_dims(n, m, p) || check_y("fit_beta", y, y_type, n) || check_ld("fit_beta", "ld", ld, m, true)) return 1;
  if (use_weights && !weights) return fail("use_weights set but weights == NULL");
  if (maxit < 0) return fail("maxit must be >= 0");
  if (check_ptrs("fit_beta", n, {x, nf, alpha_hat, contrast, beta_mat, lambda, out_beta_mat, out_beta_var_mat, out_iter,
                                 out_contrast_num, out_contrast_denom, out_deviance}))
    return 1;
  return fit_beta_dev(y, y_type, x, nf, nf_is_vector, alpha_hat, contrast, beta_mat, lambda, weights, use_weights, tol,
                      maxit, use_qr, minmu, n, m, p, ld, out_beta_mat, out_beta_var_mat, out_iter, out_hat_diagonals,
                      out_contrast_num, out_contrast_denom, out_deviance, out_mu, (cudaStream_t)stream, true);
}

int b200nb_nb_loglik_dev(const void* y, int y_type, const double* x, const double* nf, int nf_is_vector,
                         const double* alpha_hat, const double* beta_mat, const double* weights, int use_weights,
                         double minmu, int n, int m, int p, long long ld, double* out_loglik, double* out_mu,
                         void* stream) {
  if (check_dims(n, m, p) || check_y("nb_loglik", y, y_type, n) || check_ld("nb_loglik", "ld", ld, m, true)) return 1;
  if (use_weights && !weights) return fail("use_weights set but weights == NULL");
  if (!out_loglik) return fail("out_loglik == NULL");
  if (check_ptrs("nb_loglik", n, {x, nf, alpha_hat, beta_mat}) || (n > 0 && check_device())) return 1;
  nb::LogLikArgs a{};
  a.y = y; a.y_is_f64 = (y_type == B200NB_Y_F64); a.x = x; a.nf = nf; a.nf_is_vector = nf_is_vector;
  a.alpha = alpha_hat; a.beta = beta_mat; a.w = use_weights ? weights : nullptr; a.n = n; a.m = m; a.p = p; a.ld = ld;
  a.minmu = minmu > 0.0 ? minmu : 0.0; a.loglik = out_loglik; a.mu_out = out_mu;
  CU(nb::launch_nb_loglik(a, (cudaStream_t)stream));
  if (n > 0) g_launches++;
  return 0;
}

int b200nb_beta_optim_dev(const void* y, int y_type, const double* x, const double* nf, int nf_is_vector,
                          const double* alpha_hat, const double* lambda, const double* beta_start,
                          const double* weights, int use_weights, int maxit, int n, int m, int p, long long ld,
                          double* out_beta_mat, int32_t* out_converged, int32_t* out_iter, void* stream) {
  if (check_dims(n, m, p) || check_y("beta_optim", y, y_type, n) || check_ld("beta_optim", "ld", ld, m, true)) return 1;
  if (use_weights && !weights) return fail("use_weights set but weights == NULL");
  if (maxit < 1) return fail("maxit must be >= 1");
  if (check_ptrs("beta_optim", n, {x, nf, alpha_hat, lambda, beta_start, out_beta_mat, out_converged, out_iter}) ||
      (n > 0 && check_device()))
    return 1;
  nb::OptimArgs a{};
  a.y = y; a.y_is_f64 = (y_type == B200NB_Y_F64); a.x = x; a.nf = nf; a.nf_is_vector = nf_is_vector;
  a.alpha = alpha_hat; a.lambda = lambda; a.beta_in = beta_start; a.w = use_weights ? weights : nullptr;
  a.bound = 30.0 * 0.693147180559945309417232121458; a.maxit = maxit; a.n = n; a.m = m; a.p = p; a.ld = ld;
  a.beta_out = out_beta_mat; a.converged = out_converged; a.iter = out_iter;
  CU(nb::launch_beta_optim(a, (cudaStream_t)stream));
  if (n > 0) g_launches++;
  return 0;
}

int b200nb_to_gene_major_dev(const void* src, void* dst, int n, int m, long long ld, int elem_size, void* stream) {
  if (elem_size != 4 && elem_size != 8) return fail("to_gene_major: elem_size=%d must be 4 or 8", elem_size);
  if (check_ld("to_gene_major", "ld", ld, m, false) || check_ptrs("to_gene_major", n, {src, dst})) return 1;
  if (n > 0 && check_device()) return 1;
  CU(nb::launch_to_gene_major(src, dst, n, m, ld, elem_size, (cudaStream_t)stream));
  g_launches++;
  return 0;
}

int b200nb_to_col_major_dev(const double* src, double* dst, int n, int m, long long ld, void* stream) {
  if (check_ld("to_col_major", "ld", ld, m, false) || check_ptrs("to_col_major", n, {src, dst})) return 1;
  if (n > 0 && check_device()) return 1;
  CU(nb::launch_to_col_major(src, dst, n, m, ld, (cudaStream_t)stream));
  g_launches++;
  return 0;
}

// the checks and arguments the three prep variants share; exactly one of size_factors and nf is read
static int prep_args(const char* what, nb::PrepArgs& a, const void* y, int y_type, const double* x, const double* proj,
                     const double* size_factors, const double* nf, double xim, double min_disp, double max_disp,
                     double minmu, int n, int m, int p, long long ld, double* base_mean, double* base_var,
                     int32_t* all_zero, double* alpha0, double* mu_lin, double* beta0) {
  if (check_dims(n, m, p) || check_y(what, y, y_type, n) || check_ld(what, "ld", ld, m, true)) return 1;
  if (m <= p) return fail("prep needs m > p (m=%d, p=%d)", m, p);
  if (check_ptrs(what, n, {x, proj, size_factors ? size_factors : nf, base_mean, base_var, all_zero, alpha0}) ||
      (n > 0 && check_device()))
    return 1;
  a = nb::PrepArgs{};
  a.y = y; a.y_is_f64 = (y_type == B200NB_Y_F64); a.x = x; a.proj = proj; a.size_factors = size_factors; a.nf = nf;
  a.xim = xim; a.min_disp = min_disp; a.max_disp = max_disp; a.minmu = minmu; a.n = n; a.m = m; a.p = p; a.ld = ld;
  a.base_mean = base_mean; a.base_var = base_var; a.all_zero = all_zero; a.alpha0 = alpha0; a.mu_lin = mu_lin;
  a.beta0 = beta0;
  a.gid = nullptr; a.xg = nullptr; a.G = 0;
  return 0;
}

static int prep_launch(nb::PrepArgs& a, void* stream) {
  const char* pg = getenv("B200NB_PREP_GROUPED");   // "0": always the streaming kernel (A/B switch, read per call)
  if (a.n > 0 && (long long)a.m * a.p >= 1024 && !(pg && pg[0] == '0')) {
    // long rows: a design with few distinct rows is handled per group (this fetches the m x p design: one stream sync)
    DesignDev dd;
    if (prepare_design_from_device(a.x, a.m, a.p, (cudaStream_t)stream, &dd)) return 1;
    if (dd.grouped) { a.gid = dd.gid; a.xg = dd.xg; a.G = dd.G; }
  }
  CU(nb::launch_prep(a, (cudaStream_t)stream));
  if (a.n > 0) g_launches++;
  return 0;
}

int b200nb_prep_dev(const void* y, int y_type, const double* x, const double* proj, const double* size_factors,
                    double xim, double min_disp, double max_disp, double minmu, int n, int m, int p, long long ld,
                    double* base_mean, double* base_var, int32_t* all_zero, double* alpha0, double* mu_lin,
                    double* beta0, void* stream) {
  nb::PrepArgs a;
  if (prep_args("prep", a, y, y_type, x, proj, size_factors, nullptr, xim, min_disp, max_disp, minmu, n, m, p, ld,
                base_mean, base_var, all_zero, alpha0, mu_lin, beta0))
    return 1;
  return prep_launch(a, stream);
}

int b200nb_prep_weighted_dev(const void* y, int y_type, const double* x, const double* proj,
                             const double* size_factors, double xim, double min_disp, double max_disp, double minmu,
                             int n, int m, int p, long long ld, double* base_mean, double* base_var,
                             int32_t* all_zero, double* alpha0, double* mu_lin, double* beta0, const double* weights,
                             double weight_threshold, double* out_weights_norm, int32_t* out_weights_fail,
                             int32_t* out_status, void* stream) {
  nb::PrepArgs a;
  if (prep_args("prep_weighted", a, y, y_type, x, proj, size_factors, nullptr, xim, min_disp, max_disp, minmu, n, m, p,
                ld, base_mean, base_var, all_zero, alpha0, mu_lin, beta0))
    return 1;
  if (p > 32) return fail("weighted prep supports p <= 32 (p=%d)", p);
  if (check_ptrs("prep_weighted", n, {weights, out_weights_norm, out_weights_fail, out_status})) return 1;
  if (!(weight_threshold >= 0.0)) return fail("weight_threshold must be >= 0");
  a.weights = weights; a.weight_threshold = weight_threshold; a.weights_norm = out_weights_norm;
  a.weights_fail = out_weights_fail; a.status = out_status;
  if (n > 0) CU(cudaMemsetAsync(out_status, 0, sizeof(int32_t), (cudaStream_t)stream));
  return prep_launch(a, stream);
}

int b200nb_prep_nf_dev(const void* y, int y_type, const double* x, const double* proj, const double* nf, double xim,
                       double min_disp, double max_disp, double minmu, int n, int m, int p, long long ld,
                       double* base_mean, double* base_var, int32_t* all_zero, double* alpha0, double* mu_lin,
                       double* beta0, void* stream) {
  nb::PrepArgs a;
  if (prep_args("prep_nf", a, y, y_type, x, proj, nullptr, nf, xim, min_disp, max_disp, minmu, n, m, p, ld, base_mean,
                base_var, all_zero, alpha0, mu_lin, beta0))
    return 1;
  return prep_launch(a, stream);
}

int b200nb_trend_fit_dev(const double* means, const double* disps, int n, double min_disp, double* out4,
                         void* stream) {
  if (n < 1) return fail("trend fit needs at least one gene");
  if (check_ptrs("trend_fit", n, {means, disps, out4}) || check_device()) return 1;
  CU(nb::launch_trend_fit(means, disps, n, min_disp, out4, (cudaStream_t)stream));
  g_launches++;
  return 0;
}

// b200nb_cooks_dev and b200nb_cooks_nf_dev: exactly one of size_factors and nf is read
static int cooks_common(const char* what, const void* y, int y_type, const double* mu, const double* hat,
                        const double* size_factors, const double* nf, const int32_t* cell_ptr,
                        const int32_t* cell_samples, int ncell, int n, int m, int p, long long ld, double* cooks,
                        double* max_cooks, double* robust_disp, void* stream) {
  if (check_dims(n, m, p) || check_y(what, y, y_type, n) || check_ld(what, "ld", ld, m, true)) return 1;
  if (ncell < 1 || ncell > m) return fail("bad number of design cells %d", ncell);
  if (check_ptrs(what, n, {mu, hat, size_factors ? size_factors : nf, cell_ptr, cell_samples, max_cooks, robust_disp}))
    return 1;
  if (n > 0 && check_device()) return 1;
  nb::CooksArgs a{};
  a.y = y; a.y_is_f64 = (y_type == B200NB_Y_F64); a.mu = mu; a.hat = hat; a.size_factors = size_factors;
  a.cell_ptr = cell_ptr; a.cell_samples = cell_samples; a.ncell = ncell; a.n = n; a.m = m; a.p = p; a.ld = ld;
  a.cooks = cooks; a.max_cooks = max_cooks; a.robust_disp = robust_disp; a.nf = nf;
  a.max_cell = 0;
  if (n > 0 && m > 256) {
    // long rows: the size of the largest cell decides how much per-warp scratch the trimmed means need (one small
    // device-to-host copy and a stream sync; short rows need none of it)
    std::vector<int32_t> cp((size_t)ncell + 1);
    CU(cudaMemcpyAsync(cp.data(), cell_ptr, cp.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    CU(cudaStreamSynchronize((cudaStream_t)stream));
    for (int c = 0; c < ncell; c++) a.max_cell = std::max(a.max_cell, (int)(cp[c + 1] - cp[c]));
  }
  CU(nb::launch_cooks(a, (cudaStream_t)stream));
  if (n > 0) g_launches++;
  return 0;
}

int b200nb_cooks_dev(const void* y, int y_type, const double* mu, const double* hat, const double* size_factors,
                     const int32_t* cell_ptr, const int32_t* cell_samples, int ncell, int n, int m, int p,
                     long long ld, double* cooks, double* max_cooks, double* robust_disp, void* stream) {
  return cooks_common("cooks", y, y_type, mu, hat, size_factors, nullptr, cell_ptr, cell_samples, ncell, n, m, p, ld,
                      cooks, max_cooks, robust_disp, stream);
}

int b200nb_cooks_nf_dev(const void* y, int y_type, const double* mu, const double* hat, const double* nf,
                        const int32_t* cell_ptr, const int32_t* cell_samples, int ncell, int n, int m, int p,
                        long long ld, double* cooks, double* max_cooks, double* robust_disp, void* stream) {
  return cooks_common("cooks_nf", y, y_type, mu, hat, nullptr, nf, cell_ptr, cell_samples, ncell, n, m, p, ld, cooks,
                      max_cooks, robust_disp, stream);
}

int b200nb_beta_prior_quantile_dev(const double* beta_log2, int n, int p, const double* base_mean,
                                   const double* disp_fit, const int32_t* col_a, const int32_t* col_b, int k,
                                   double prob, double* out_q, void* stream) {
  if (n < 1 || p < 1 || k < 0) return fail("bad dimensions n=%d p=%d k=%d", n, p, k);
  if (!(prob > 0.0 && prob < 1.0)) return fail("prob=%g must lie in (0, 1)", prob);
  if (k == 0) return 0;
  if (check_ptrs("beta_prior_quantile", k, {beta_log2, base_mean, disp_fit, col_a, col_b, out_q}) || check_device())
    return 1;
  // the column list is tiny (k <= a few hundred): fetch it once to check every index (one stream sync)
  std::vector<int32_t> ca((size_t)k), cb((size_t)k);
  CU(cudaMemcpyAsync(ca.data(), col_a, k * sizeof(int32_t), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  CU(cudaMemcpyAsync(cb.data(), col_b, k * sizeof(int32_t), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  CU(cudaStreamSynchronize((cudaStream_t)stream));
  for (int c = 0; c < k; c++) {
    if (ca[c] < 0 || ca[c] >= p) return fail("column %d: a=%d must lie in [0, %d)", c, ca[c], p);
    if (cb[c] < -1 || cb[c] >= p) return fail("column %d: b=%d must lie in [-1, %d)", c, cb[c], p);
  }
  nb::BetaPriorQArgs a{};
  a.beta = beta_log2; a.n = n; a.base_mean = base_mean; a.disp_fit = disp_fit; a.col_a = col_a; a.col_b = col_b;
  a.k = k; a.prob = prob; a.out_q = out_q;
  CU(nb::launch_beta_prior_quantile(a, (cudaStream_t)stream));
  g_launches++;
  return 0;
}

static int size_factors_common(const char* what, const void* y, int y_type, const double* divisor, int poscounts,
                               int n, int m, long long ld, double* loggeomeans, double* scratch_gm,
                               double* scratch_cm, double* size_factors, int32_t* n_finite, void* stream) {
  if (n < 1) return fail("size factors need at least one gene");
  if (check_dims(n, m, 1) || check_y(what, y, y_type, n) || check_ld(what, "ld", ld, m, true) ||
      check_ptrs(what, n, {loggeomeans, scratch_gm, scratch_cm, size_factors, n_finite}) || check_device())
    return 1;
  nb::SizeFactorArgs a{};
  a.y = y; a.y_is_f64 = (y_type == B200NB_Y_F64); a.poscounts = poscounts ? 1 : 0; a.n = n; a.m = m; a.ld = ld;
  a.loggeomeans = loggeomeans; a.ratios = scratch_gm; a.ratios_colmajor = scratch_cm; a.size_factors = size_factors;
  a.n_finite = n_finite; a.divisor = divisor;
  CU(nb::launch_size_factors(a, (cudaStream_t)stream));
  g_launches += 3;
  return 0;
}

int b200nb_size_factors_dev(const void* y, int y_type, int poscounts, int n, int m, long long ld,
                            double* loggeomeans, double* scratch_gm, double* scratch_cm, double* size_factors,
                            int32_t* n_finite, void* stream) {
  return size_factors_common("size_factors", y, y_type, nullptr, poscounts, n, m, ld, loggeomeans, scratch_gm,
                             scratch_cm, size_factors, n_finite, stream);
}

int b200nb_size_factors_norm_dev(const void* y, int y_type, const double* divisor, int poscounts, int n, int m,
                                 long long ld, double* loggeomeans, double* scratch_gm, double* scratch_cm,
                                 double* size_factors, int32_t* n_finite, void* stream) {
  if (divisor == nullptr) return fail("size_factors_norm needs the divisor matrix");
  return size_factors_common("size_factors_norm", y, y_type, divisor, poscounts, n, m, ld, loggeomeans, scratch_gm,
                             scratch_cm, size_factors, n_finite, stream);
}

// The objective tiles of b200nb_sf_iterate_objective_dev: the grow-only workspace slot S_SFI (taken under g_call_mu,
// which also serialises it against the host entry points).  128 MB of gene log-likelihoods per tile by default: one
// tile up to 50 000 genes x 335 objective columns.
constexpr size_t kSfiTileBytes = (size_t)128 << 20;

int b200nb_sf_iterate_objective_dev(const void* y, int y_type, const double* q, const double* alpha,
                                    const double* par, double h, double Q, int n, int m, long long ld,
                                    int max_tile_cols, double* out, void* stream) {
  if (n < 1 || m < 1) return fail("sf_iterate_objective: bad dimensions n=%d m=%d (both must be >= 1)", n, m);
  if (check_ld("sf_iterate_objective", "ld", ld, m, true) || check_y("sf_iterate_objective", y, y_type, n)) return 1;
  if (!finite_pos(h)) return fail("sf_iterate_objective: h=%g must be finite and > 0", h);
  if (!(Q >= 0.0 && Q < 1.0)) return fail("sf_iterate_objective: Q=%g must lie in [0, 1)", Q);
  if (max_tile_cols < 0) return fail("sf_iterate_objective: max_tile_cols=%d must be >= 0", max_tile_cols);
  if (check_ptrs("sf_iterate_objective", n, {q, alpha, par, out}) || check_device()) return 1;
  const int cols = 2 * m + 1;
  long long tile = (long long)(kSfiTileBytes / ((size_t)n * sizeof(double)));
  if (max_tile_cols > 0 && tile > max_tile_cols) tile = max_tile_cols;
  tile = std::max(1LL, std::min(tile, (long long)cols));
  std::lock_guard<std::mutex> lk(g_call_mu);
  void* ws = nullptr;
  if (ws_get(S_SFI, ((size_t)3 + (size_t)tile) * (size_t)n * sizeof(double), &ws)) return 1;
  nb::SfIterateArgs a{};
  a.y = y; a.y_is_f64 = (y_type == B200NB_Y_F64); a.q = q; a.alpha = alpha; a.par = par; a.h = h; a.Q = Q;
  a.n = n; a.m = m; a.ld = ld; a.tile = (int)tile;
  a.abc = static_cast<double*>(ws);
  a.ll = a.abc + (size_t)3 * n;
  a.out = out;
  CU(nb::launch_sf_iterate_objective(a, (cudaStream_t)stream));
  g_launches += 2 * ((cols + tile - 1) / tile);
  return 0;
}

int b200nb_transform_dev(const void* y, int y_type, const double* size_factors, const double* nf, int n, int m,
                         long long ld, int mode, double c0, double c1, double* out, long long ld_out, void* stream) {
  if (n < 0 || m < 0) return fail("transform: bad dimensions n=%d m=%d (both must be >= 0)", n, m);
  if (check_ld("transform", "ld", ld, m, false) || check_ld("transform", "ld_out", ld_out, m, false) ||
      check_factors("transform", size_factors, nf) || check_y("transform", y, y_type, n))
    return 1;
  if (!y || !out) return fail("transform: null pointer argument");
  nb::TransformArgs a{};
  a.mode = mode;
  a.ln2 = log(2.0);
  switch (mode) {
    case B200NB_TRANSFORM_VST_PARAMETRIC:
      if (!finite_pos(c0) || !finite_pos(c1))
        return fail("transform: asymptDisp=%g and extraPois=%g must be finite and > 0", c0, c1);
      a.c0 = c0; a.c1 = 1.0 + c1; a.c2 = 2.0 * c0; a.c3 = 4.0 * c0;
      break;
    case B200NB_TRANSFORM_VST_MEAN:
      if (!finite_pos(c0)) return fail("transform: alpha=%g must be finite and > 0", c0);
      a.c0 = c0; a.c1 = log(c0); a.c2 = log(4.0);
      break;
    case B200NB_TRANSFORM_LOG2:
      if (!(c0 >= 0.0 && c0 < HUGE_VAL)) return fail("transform: pc=%g must be finite and >= 0", c0);
      a.c0 = c0;
      break;
    default:
      return fail("transform: bad mode %d", mode);
  }
  if (n == 0 || m == 0) return 0;
  if (check_device()) return 1;
  a.y = y; a.y_is_f64 = (y_type == B200NB_Y_F64); a.size_factors = size_factors; a.nf = nf;
  a.n = n; a.m = m; a.ld = ld; a.ld_out = ld_out; a.out = out;
  CU(nb::launch_transform(a, (cudaStream_t)stream));
  g_launches++;
  return 0;
}

// qnorm(1 - 0.05 / 2): the normal quantile rlog's weighted upper quantile is matched to (R/core.R:2416-2419)
constexpr double kRlogSdScale = 1.959963984540054;

int b200nb_rlog_fit_dev(const void* y, int y_type, const double* size_factors, const double* nf,
                        const double* intercept, const double* disp_fit, int n, int m, long long ld,
                        double beta_prior_var, double tol, int maxit, double minmu, double* out, long long ld_out,
                        double* out_intercept, double* out_iter, void* stream) {
  if (n < 0 || m < 1) return fail("rlog_fit: bad dimensions n=%d m=%d (n >= 0, m >= 1)", n, m);
  if (check_ld("rlog_fit", "ld", ld, m, false) || check_ld("rlog_fit", "ld_out", ld_out, m, false) ||
      check_factors("rlog_fit", size_factors, nf) || check_y("rlog_fit", y, y_type, n))
    return 1;
  if (!finite_pos(beta_prior_var)) return fail("rlog_fit: betaPriorVar=%g must be finite and > 0", beta_prior_var);
  if (!finite_pos(tol)) return fail("rlog_fit: tol=%g must be finite and > 0", tol);
  if (!finite_pos(minmu)) return fail("rlog_fit: minmu=%g must be finite and > 0", minmu);
  if (maxit < 1) return fail("rlog_fit: maxit=%d must be >= 1", maxit);
  if (!y || !disp_fit || !out || !out_iter || (!intercept && !out_intercept))
    return fail("rlog_fit: null pointer argument");
  if (n == 0) return 0;
  if (check_device()) return 1;
  const double ln2 = log(2.0);
  nb::RlogFitArgs a{};
  a.y = y; a.y_is_f64 = (y_type == B200NB_Y_F64); a.size_factors = size_factors; a.nf = nf; a.intercept = intercept;
  a.disp_fit = disp_fit;
  // fitNbinomGLMs' lambda / log(2)^2 (R/fitNbinomGLMs.R:160) of rlogData's lambda = 1 / betaPriorVar, 1e-6 (:243-247)
  a.lambda = (1.0 / beta_prior_var) / (ln2 * ln2);
  a.lambda0 = 1e-6 / (ln2 * ln2);
  a.tol = tol; a.maxit = maxit; a.minmu = minmu; a.log_minmu = log(minmu); a.ln2 = ln2;
  a.n = n; a.m = m; a.ld = ld; a.ld_out = ld_out; a.out = out; a.out_intercept = intercept ? nullptr : out_intercept;
  a.iter = out_iter;
  CU(nb::launch_rlog_fit(a, (cudaStream_t)stream));
  g_launches++;
  return 0;
}

// The per-CTA partials of b200nb_rlog_prior_var_dev: the grow-only workspace slot S_RLOG (taken under g_call_mu, as
// S_SFI; a few hundred KB)
int b200nb_rlog_prior_var_dev(const void* y, int y_type, const double* size_factors, const double* nf,
                              const double* base_mean, const double* disp_fit, int n, int m, long long ld,
                              double* out_var, void* stream) {
  if (n < 1 || m < 1) return fail("rlog_prior_var: bad dimensions n=%d m=%d (both must be >= 1)", n, m);
  if (check_ld("rlog_prior_var", "ld", ld, m, false) || check_factors("rlog_prior_var", size_factors, nf)) return 1;
  if (check_ptrs("rlog_prior_var", n, {base_mean, disp_fit, out_var}) || check_y("rlog_prior_var", y, y_type, n) ||
      check_device())
    return 1;
  std::lock_guard<std::mutex> lk(g_call_mu);
  void* ws = nullptr;
  if (ws_get(S_RLOG, nb::rlog_prior_scratch_bytes(n, m), &ws)) return 1;
  nb::RlogPriorArgs a{};
  a.y = y; a.y_is_f64 = (y_type == B200NB_Y_F64); a.size_factors = size_factors; a.nf = nf; a.base_mean = base_mean;
  a.disp_fit = disp_fit; a.n = n; a.m = m; a.ld = ld; a.prob = 0.95; a.sd_scale = kRlogSdScale;
  a.st = static_cast<nb::RlogPriorState*>(ws);
  a.out_var = out_var;
  CU(nb::launch_rlog_prior_var(a, (cudaStream_t)stream));
  g_launches += 2 * (1 + 16);
  return 0;
}

static bool padj_method_ok(int method) { return method >= B200NB_PADJ_BH && method <= B200NB_PADJ_NONE; }

int b200nb_results_gene_dev(const void* y, int y_type, int n, int m, long long ld, const double* lfc, const double* se,
                            const double* stat, const double* pvalue, int negate, const int32_t* zero_mask, int lrt,
                            int alt, double lfc_threshold, const double* max_cooks, double cooks_cutoff,
                            const int32_t* keep, const int32_t* replace, const double* base_mean, double* out_lfc,
                            double* out_se, double* out_stat, double* out_pvalue, void* stream) {
  if (n < 0 || m < 1) return fail("results_gene: bad dimensions n=%d m=%d (n >= 0, m >= 1)", n, m);
  if (check_ld("results_gene", "ld", ld, m, false)) return 1;
  if (alt < B200NB_ALT_NONE || alt > B200NB_ALT_LESS) return fail("results_gene: unknown altHypothesis code %d", alt);
  if (!(lfc_threshold >= 0.0 && lfc_threshold < HUGE_VAL))
    return fail("results_gene: lfcThreshold=%g must be finite and >= 0", lfc_threshold);
  if (!lfc || !se || !stat || !pvalue || !out_lfc || !out_se || !out_stat || !out_pvalue || (zero_mask && !y) ||
      (replace && !base_mean))
    return fail("results_gene: null pointer argument");
  if (zero_mask && check_y("results_gene", y, y_type, n)) return 1;
  if (n == 0) return 0;
  if (check_device()) return 1;
  nb::ResultsGeneArgs a{};
  a.y = y; a.y_is_f64 = (y_type == B200NB_Y_F64); a.n = n; a.m = m; a.ld = ld;
  a.lfc = lfc; a.se = se; a.stat = stat; a.pvalue = pvalue; a.negate = negate != 0; a.lrt = lrt != 0; a.alt = alt;
  a.zero_mask = zero_mask; a.lfc_threshold = lfc_threshold; a.cooks_cutoff = cooks_cutoff; a.max_cooks = max_cooks;
  a.keep = keep; a.replace = replace; a.base_mean = base_mean;
  a.out_lfc = out_lfc; a.out_se = out_se; a.out_stat = out_stat; a.out_pvalue = out_pvalue;
  CU(nb::launch_results_gene(a, (cudaStream_t)stream));
  g_launches++;
  return 0;
}

int b200nb_results_heuristic_dev(const void* y, int y_type, const int64_t* rows, int k, int m, long long ld,
                                 const double* cooks, long long ld_cooks, int32_t* keep, void* stream) {
  if (k < 0 || m < 1) return fail("results_heuristic: bad dimensions k=%d m=%d (k >= 0, m >= 1)", k, m);
  if (check_ld("results_heuristic", "ld", ld, m, false) ||
      check_ld("results_heuristic", "ld_cooks", ld_cooks, m, false) || check_y("results_heuristic", y, y_type, k))
    return 1;
  if (!y || !rows || !cooks || !keep) return fail("results_heuristic: null pointer argument");
  if (k == 0) return 0;
  if (check_device()) return 1;
  nb::ResultsHeuristicArgs a{};
  a.y = y; a.y_is_f64 = (y_type == B200NB_Y_F64); a.rows = rows; a.k = k; a.m = m; a.ld = ld; a.ld_cooks = ld_cooks;
  a.cooks = cooks; a.keep = keep;
  CU(nb::launch_results_heuristic(a, (cudaStream_t)stream));
  g_launches++;
  return 0;
}

// one CTA per probability: the grid's x dimension bound kept well inside every launch limit
constexpr int kMaxTheta = 65535;

int b200nb_filter_cutoffs_dev(const double* filter, int n, const double* theta, int n_theta, double* out,
                              void* stream) {
  if (n < 1) return fail("filter_cutoffs: n=%d must be >= 1", n);
  if (n_theta < 1 || n_theta > kMaxTheta) return fail("filter_cutoffs: n_theta=%d must be in [1, %d]", n_theta, kMaxTheta);
  if (check_ptrs("filter_cutoffs", n, {filter, theta, out}) || check_device()) return 1;
  nb::FilterCutoffArgs a{};
  a.filter = filter; a.n = n; a.theta = theta; a.out = out;
  CU(nb::launch_filter_cutoffs(a, n_theta, (cudaStream_t)stream));
  g_launches++;
  return 0;
}

int b200nb_filter_numrej_dev(const double* p_sorted, const double* filter_sorted, int n, const double* cutoffs,
                             int n_theta, int method, double alpha, int32_t* out_numrej, void* stream) {
  if (n < 1) return fail("filter_numrej: n=%d must be >= 1", n);
  if (n_theta < 1 || n_theta > kMaxTheta) return fail("filter_numrej: n_theta=%d must be in [1, %d]", n_theta, kMaxTheta);
  if (!padj_method_ok(method)) return fail("filter_numrej: unknown p.adjust method code %d", method);
  if (!(alpha > 0.0 && alpha < 1.0)) return fail("filter_numrej: alpha=%g must be in (0, 1)", alpha);
  if (check_ptrs("filter_numrej", n, {p_sorted, filter_sorted, cutoffs, out_numrej}) || check_device()) return 1;
  nb::PadjArgs a{};
  a.p_sorted = p_sorted; a.filter_sorted = filter_sorted; a.n = n; a.cutoffs = cutoffs; a.method = method;
  a.alpha = alpha; a.out_numrej = out_numrej;
  CU(nb::launch_filter_numrej(a, n_theta, (cudaStream_t)stream));
  g_launches++;
  return 0;
}

int b200nb_padj_dev(const double* p_sorted, const double* filter_sorted, const int64_t* order, int n,
                    const double* cutoffs, int j, int method, double* out, void* stream) {
  if (n < 1) return fail("padj: n=%d must be >= 1", n);
  if (j < 0) return fail("padj: j=%d must be >= 0", j);
  if (!padj_method_ok(method)) return fail("padj: unknown p.adjust method code %d", method);
  if (check_ptrs("padj", n, {p_sorted, filter_sorted, order, out}) || check_device()) return 1;
  nb::PadjArgs a{};
  a.p_sorted = p_sorted; a.filter_sorted = filter_sorted; a.order = order; a.n = n; a.cutoffs = cutoffs; a.j = j;
  a.method = method; a.out = out;
  CU(nb::launch_padj(a, (cudaStream_t)stream));
  g_launches++;
  return 0;
}

/* ------------------------------------------------------------------ host entry points */
/* Each runs through host_call (the speculation protocol) and upload_and_launch (its input matrices). */

int b200nb_fit_disp(const void* y, int y_type, const double* x, const double* mu_hat, const double* log_alpha,
                    const double* log_alpha_prior_mean, double log_alpha_prior_sigmasq, double min_log_alpha,
                    double kappa_0, double tol, int maxit, int use_prior, const double* weights, int use_weights,
                    double weight_threshold, int use_cr, int n, int m, int p,
                    double* out_log_alpha, int32_t* out_iter, int32_t* out_iter_accept, double* out_last_change,
                    double* out_initial_lp, double* out_initial_dlp, double* out_last_lp, double* out_last_dlp,
                    double* out_last_d2lp) {
  if (check_dims(n, m, p) || check_y("fitDisp", y, y_type, n)) return 1;
  if (n == 0) return 0;
  if (use_weights && !weights) return fail("use_weights set but weights == NULL");
  if (check_ptrs("fitDisp", n, {x, mu_hat, log_alpha, log_alpha_prior_mean}) || check_device()) return 1;
  const int ye = (y_type == B200NB_Y_F64) ? 8 : 4;
  const long long ld = ld_for(m);
  return host_call("fitDisp", n, [&](CallInputs& ci, PhaseClock& clk, cudaStream_t st) -> int {
    MatIn My{y, n, m, ye}, Mmu{mu_hat, n, m, 8}, Mw{weights, n, m, 8};
    std::vector<MatIn*> mats{&My, &Mmu};
    if (use_weights) mats.push_back(&Mw);
    SmallIn in;
    const size_t o_x = in.add(x, sizeof(double) * m * p), o_la = in.add(log_alpha, sizeof(double) * n),
                 o_pm = in.add(log_alpha_prior_mean, sizeof(double) * n);
    char* din;
    if (in.upload(st, &din)) return 1;
    SmallOut out;
    double* hd[7] = {out_log_alpha, out_last_change, out_initial_lp, out_initial_dlp, out_last_lp, out_last_dlp,
                     out_last_d2lp};
    size_t od[7];
    for (int k = 0; k < 7; k++) od[k] = out.add(hd[k], sizeof(double) * n);
    const size_t oi = out.add(out_iter, sizeof(int32_t) * n), oia = out.add(out_iter_accept, sizeof(int32_t) * n);
    char* dout;
    if (out.device(&dout)) return 1;
    auto D = [&](size_t off) { return reinterpret_cast<double*>(dout + off); };
    // kernels on rows [g0, g0 + gc) of the device copies
    auto launch_rows = [&](size_t g0, int gc, cudaStream_t ks) -> int {
      const char* yb = static_cast<const char*>(My.dev) + g0 * (size_t)ld * ye;
      const double* mub = static_cast<const double*>(Mmu.dev) + g0 * (size_t)ld;
      const double* wb = use_weights ? static_cast<const double*>(Mw.dev) + g0 * (size_t)ld : nullptr;
      return fit_disp_dev(yb, y_type, reinterpret_cast<const double*>(din + o_x), mub,
                          reinterpret_cast<const double*>(din + o_la) + g0,
                          reinterpret_cast<const double*>(din + o_pm) + g0, log_alpha_prior_sigmasq, min_log_alpha,
                          kappa_0, tol, maxit, use_prior, wb, use_weights, weight_threshold, use_cr, gc, m, p, ld,
                          D(od[0]) + g0, reinterpret_cast<int32_t*>(dout + oi) + g0,
                          reinterpret_cast<int32_t*>(dout + oia) + g0, D(od[1]) + g0, D(od[2]) + g0, D(od[3]) + g0,
                          D(od[4]) + g0, D(od[5]) + g0, D(od[6]) + g0, ks, false);
    };
    if (upload_and_launch(mats, ci, n, use_generic(p) ? 1 : plan_chunks(n), st, clk, launch_rows)) return 1;
    if (out.begin(dout, st)) return 1;     // the result DMA queues behind the kernels ...
    const bool verified = ci.validate();   // ... while the host hashes the inputs of a speculative hit
    clk.next();
    if (!verified) return kRetry;
    return out.finish(st);
  });
}

int b200nb_fit_disp_grid(const void* y, int y_type, const double* x, const double* mu_hat, const double* disp_grid,
                         int disp_grid_n, const double* log_alpha_prior_mean, double log_alpha_prior_sigmasq,
                         int use_prior, const double* weights, int use_weights, double weight_threshold, int use_cr,
                         int n, int m, int p, double* out_log_alpha) {
  if (check_dims(n, m, p) || check_y("fitDispGrid", y, y_type, n)) return 1;
  if (n == 0) return 0;
  if (use_weights && !weights) return fail("use_weights set but weights == NULL");
  if (disp_grid_n < 2) return fail("disp_grid needs at least 2 points");
  if (check_ptrs("fitDispGrid", n, {x, mu_hat, disp_grid, log_alpha_prior_mean}) || check_device()) return 1;
  const int ye = (y_type == B200NB_Y_F64) ? 8 : 4;
  const long long ld = ld_for(m);
  return host_call("fitDispGrid", n, [&](CallInputs& ci, PhaseClock& clk, cudaStream_t st) -> int {
    MatIn My{y, n, m, ye}, Mmu{mu_hat, n, m, 8}, Mw{weights, n, m, 8};
    std::vector<MatIn*> mats{&My, &Mmu};
    if (use_weights) mats.push_back(&Mw);
    SmallIn in;
    const size_t o_x = in.add(x, sizeof(double) * m * p), o_grid = in.add(disp_grid, sizeof(double) * disp_grid_n),
                 o_pm = in.add(log_alpha_prior_mean, sizeof(double) * n);
    char* din;
    if (in.upload(st, &din)) return 1;
    SmallOut out;
    const size_t o_la = out.add(out_log_alpha, sizeof(double) * n);
    char* dout;
    if (out.device(&dout)) return 1;
    auto launch_all = [&](size_t, int, cudaStream_t ks) -> int {   // one piece: every row
      return b200nb_fit_disp_grid_dev(My.dev, y_type, reinterpret_cast<const double*>(din + o_x),
                                      (const double*)Mmu.dev, reinterpret_cast<const double*>(din + o_grid),
                                      disp_grid_n, reinterpret_cast<const double*>(din + o_pm),
                                      log_alpha_prior_sigmasq, use_prior, (const double*)Mw.dev, use_weights,
                                      weight_threshold, use_cr, n, m, p, ld, reinterpret_cast<double*>(dout + o_la), ks);
    };
    if (upload_and_launch(mats, ci, n, 1, st, clk, launch_all)) return 1;
    if (out.begin(dout, st)) return 1;
    const bool verified = ci.validate();
    clk.next();
    if (!verified) return kRetry;
    return out.finish(st);
  });
}

// R always hands fitBeta an n x m matrix of normalisation factors, which for the usual size-factor analysis is the same
// row n times (R/core.R:2221-2228).  One parallel read of the matrix tells (it stops at the first differing entry); if
// so, only the m factors cross PCIe and the kernel takes its size-factor-vector path (log nf once per CTA instead of
// once per gene and sample).  Same values in, same results out; any NaN or differing entry keeps the matrix path.
// B200NB_SF_DETECT=0 switches the check off.
static bool rows_identical(const double* a, size_t n, int m) {
  std::atomic<int> differs{0};
  pool().parallel_for((size_t)m, [&](size_t j) {
    if (differs.load(std::memory_order_relaxed)) return;
    const double* c = a + j * n;
    const double v = c[0];
    bool same = (v == v);
    for (size_t i0 = 0; i0 < n && same; i0 += 4096) {
      const size_t i1 = (i0 + 4096 < n) ? i0 + 4096 : n;
      int bad = 0;
      for (size_t i = i0; i < i1; i++) bad |= (c[i] != v);
      same = !bad;
    }
    if (!same) differs.store(1, std::memory_order_relaxed);
  });
  return differs.load() == 0;
}
// first and last row equal: the cheap necessary condition that decides whether the full scan is worth speculating on
static bool rows_maybe_identical(const double* a, size_t n, int m) {
  for (int j = 0; j < m; j++) {
    const double v = a[(size_t)j * n];
    if (!(v == v) || a[(size_t)j * n + n - 1] != v || a[(size_t)j * n + n / 2] != v) return false;
  }
  return true;
}

int b200nb_fit_beta(const void* y, int y_type, const double* x, const double* nf, const double* alpha_hat,
                    const double* contrast, const double* beta_mat, const double* lambda, const double* weights,
                    int use_weights, double tol, int maxit, int use_qr, double minmu, int n, int m, int p,
                    double* out_beta_mat, double* out_beta_var_mat, double* out_iter, double* out_hat_diagonals,
                    double* out_contrast_num, double* out_contrast_denom, double* out_deviance, double* out_mu) {
  if (check_dims(n, m, p) || check_y("fitBeta", y, y_type, n)) return 1;
  if (n == 0) return 0;
  if (use_weights && !weights) return fail("use_weights set but weights == NULL");
  if (check_ptrs("fitBeta", n, {x, nf, alpha_hat, contrast, beta_mat, lambda}) || check_device()) return 1;
  if (maxit < 0) return fail("maxit must be >= 0");
  const int ye = (y_type == B200NB_Y_F64) ? 8 : 4;
  const long long ld = ld_for(m);
  const bool sf_detect = hostrt::env_int("B200NB_SF_DETECT", 1, 0, 1) != 0;
  return host_call("fitBeta", n, [&](CallInputs& ci, PhaseClock& clk, cudaStream_t st) -> int {
    // normalisation factors: a replicated size-factor vector?  With speculation the full scan of the matrix is
    // deferred until the kernels are running (the three probed rows decide what to launch with)
    std::vector<double> sfv;
    bool sf_unverified = false;
    if (sf_detect && rows_maybe_identical(nf, (size_t)n, m)) {
      sf_unverified = ci.speculate;
      if (ci.speculate || rows_identical(nf, (size_t)n, m)) {
        sfv.resize(m);
        for (int j = 0; j < m; j++) sfv[j] = nf[(size_t)j * n];
        if (!ci.speculate) g_hashed_bytes += (long long)sizeof(double) * n * m;   // scanned before the launch
      }
    }
    MatIn My{y, n, m, ye}, Mnf{nf, n, m, 8}, Mw{weights, n, m, 8};
    std::vector<MatIn*> mats{&My};
    if (sfv.empty()) mats.push_back(&Mnf);
    if (use_weights) mats.push_back(&Mw);
    SmallIn in;
    const size_t o_x = in.add(x, sizeof(double) * m * p), o_alpha = in.add(alpha_hat, sizeof(double) * n),
                 o_c = in.add(contrast, sizeof(double) * p), o_lam = in.add(lambda, sizeof(double) * p),
                 o_b = in.add(beta_mat, sizeof(double) * n * p),
                 o_sf = sfv.empty() ? 0 : in.add(sfv.data(), sizeof(double) * m);
    char* din;
    if (in.upload(st, &din)) return 1;
    SmallOut out;
    const size_t o_bo = out.add(out_beta_mat, sizeof(double) * n * p),
                 o_bv = out.add(out_beta_var_mat, sizeof(double) * n * p), o_it = out.add(out_iter, sizeof(double) * n),
                 o_cn = out.add(out_contrast_num, sizeof(double) * n),
                 o_cd = out.add(out_contrast_denom, sizeof(double) * n),
                 o_dev = out.add(out_deviance, sizeof(double) * n);
    char* dout;
    if (out.device(&dout)) return 1;
    void *d_h = nullptr, *d_mu = nullptr, *d_hc = nullptr;
    if (out_hat_diagonals && ws_get(S_H, sizeof(double) * n * ld, &d_h)) return 1;
    if (out_mu && ws_get(S_MUO, sizeof(double) * n * ld, &d_mu)) return 1;
    if ((out_hat_diagonals || out_mu) && ws_get(S_HC, sizeof(double) * n * m, &d_hc)) return 1;
    auto Din = [&](size_t off) { return reinterpret_cast<const double*>(din + off); };
    auto Dout = [&](size_t off) { return reinterpret_cast<double*>(dout + off); };
    auto launch_all = [&](size_t, int, cudaStream_t ks) -> int {   // one piece: every row
      return fit_beta_dev(My.dev, y_type, Din(o_x), sfv.empty() ? (const double*)Mnf.dev : Din(o_sf),
                          sfv.empty() ? 0 : 1, Din(o_alpha), Din(o_c), Din(o_b), Din(o_lam), (const double*)Mw.dev,
                          use_weights, tol, maxit, use_qr, minmu, n, m, p, ld, Dout(o_bo), Dout(o_bv), Dout(o_it),
                          (double*)d_h, Dout(o_cn), Dout(o_cd), Dout(o_dev), (double*)d_mu, ks, false);
    };
    if (upload_and_launch(mats, ci, n, 1, st, clk, launch_all)) return 1;
    if (out_hat_diagonals && b200nb_to_col_major_dev((const double*)d_h, (double*)d_hc, n, m, ld, st)) return 1;
    // Results in page-locked memory (b200nb_host_alloc) leave by DMA right behind the kernels, overlapping the host-side
    // verification below; a failed verification repeats the call and overwrites them.
    bool h_sent = false, mu_sent = false;
    if (out_hat_diagonals && d2h_async_if_pinned(out_hat_diagonals, d_hc, sizeof(double) * (size_t)n * m, st, &h_sent)) return 1;
    if (out_mu && (!out_hat_diagonals || h_sent) && pinned_contains(out_mu, sizeof(double) * (size_t)n * m)) {
      if (b200nb_to_col_major_dev((const double*)d_mu, (double*)d_hc, n, m, ld, st)) return 1;   // stream-ordered after H's DMA
      if (d2h_async_if_pinned(out_mu, d_hc, sizeof(double) * (size_t)n * m, st, &mu_sent)) return 1;
    }
    const bool small_early = (!out_hat_diagonals || h_sent) && (!out_mu || mu_sent);
    if (small_early && out.begin(dout, st)) return 1;
    bool verified = ci.validate();   // host-side hashing / scanning while the kernels run
    if (sf_unverified) {
      const bool same = rows_identical(nf, (size_t)n, m);
      g_hashed_bytes += (long long)sizeof(double) * n * m;
      verified = verified && same;
    }
    clk.next();
    if (!verified) return kRetry;
    if (out_hat_diagonals && !h_sent) {
      if (d2h_staged(out_hat_diagonals, d_hc, sizeof(double) * (size_t)n * m, st)) return 1;
    }
    if (out_mu && !mu_sent) {
      if (b200nb_to_col_major_dev((const double*)d_mu, (double*)d_hc, n, m, ld, st)) return 1;
      if (d2h_staged(out_mu, d_hc, sizeof(double) * (size_t)n * m, st)) return 1;
    }
    if (!small_early && out.begin(dout, st)) return 1;
    return out.finish(st);
  });
}

int b200nb_test_special(const double* x, int n, double* out_lgamma, double* out_digamma, double* out_trigamma) {
  if (n <= 0) return 0;
  return host_call("special", n, [&](CallInputs&, PhaseClock&, cudaStream_t st) -> int {
    SmallIn in;
    const size_t o_x = in.add(x, sizeof(double) * n);
    char* din;
    if (in.upload(st, &din)) return 1;
    SmallOut out;
    const size_t o_l = out.add(out_lgamma, sizeof(double) * n), o_d = out.add(out_digamma, sizeof(double) * n),
                 o_t = out.add(out_trigamma, sizeof(double) * n);
    char* dout;
    if (out.device(&dout)) return 1;
    CU(nb::launch_special_test(reinterpret_cast<const double*>(din + o_x), n, reinterpret_cast<double*>(dout + o_l),
                               reinterpret_cast<double*>(dout + o_d), reinterpret_cast<double*>(dout + o_t), st));
    g_launches++;
    return out.download(dout, st);
  });
}

}  // extern "C"

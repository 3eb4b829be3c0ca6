// emu.cpp -- fiber scheduler of the SIMT emulator (see cuda_runtime.h in this directory).  TEST INFRASTRUCTURE ONLY.
#include <stdio.h>
#include <sys/mman.h>
#if !defined(__x86_64__) || defined(SIMT_EMU_USE_UCONTEXT)
#include <ucontext.h>
#endif

#include <algorithm>
#include <mutex>
#include <string>
#include <vector>

#include "cuda_runtime.h"

uint3 threadIdx, blockIdx;
dim3 blockDim, gridDim;

namespace simt_emu {
namespace {

enum State { RUNNABLE, WAIT_WARP, WAIT_CTA, DONE };
constexpr size_t kStack = 512 * 1024;

#if defined(__x86_64__) && !defined(SIMT_EMU_USE_UCONTEXT)
// Minimal System V x86-64 context switch (callee-saved registers + MXCSR + x87 control word).  glibc's swapcontext
// makes a sigprocmask system call per switch, which dominated the run time of the emulated tests.
extern "C" void simt_emu_switch(void** save_sp, void* load_sp);
asm(R"(
.text
.globl simt_emu_switch
.type simt_emu_switch,@function
simt_emu_switch:
    pushq %rbp
    pushq %rbx
    pushq %r12
    pushq %r13
    pushq %r14
    pushq %r15
    subq $8, %rsp
    stmxcsr (%rsp)
    fnstcw 4(%rsp)
    movq %rsp, (%rdi)
    movq %rsi, %rsp
    ldmxcsr (%rsp)
    fldcw 4(%rsp)
    addq $8, %rsp
    popq %r15
    popq %r14
    popq %r13
    popq %r12
    popq %rbx
    popq %rbp
    ret
.size simt_emu_switch,.-simt_emu_switch
.section .note.GNU-stack,"",@progbits
.text
)");
struct Context { void* sp; };
#else
struct Context { ucontext_t uc; };
#endif

struct Fiber {
  Context ctx;
  State state;
  unsigned wait_mask;
  unsigned parity;  // number of exchanges done: selects the exchange slot
  long long ncoll;  // warp collectives (shuffles, votes, __syncwarp) this thread executed
  uint3 tid;
};

std::vector<Fiber> fibers;
std::vector<char*> stacks;
Context sched_ctx;
int cur = -1;
const std::function<void()>* body = nullptr;
uint64_t (*xchg)[2][32] = nullptr;  // [warp][slot][lane]
unsigned (*xtag)[2][32] = nullptr;  // which exchange (per-lane count) the slot was written for
std::vector<uint64_t> xchg_store;
std::vector<unsigned> xtag_store;
void* dyn_smem = nullptr;
size_t dyn_smem_cap = 0;
long long n_launches = 0;
long long max_coll = 0;   // the most warp collectives any thread of the running launch executed

char* stack_for(size_t i) {
  while (stacks.size() <= i) {
    void* p = mmap(nullptr, kStack, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (p == MAP_FAILED) { perror("simt_emu: mmap"); abort(); }
    mprotect(p, 4096, PROT_NONE);  // guard page at the low end
    stacks.push_back(static_cast<char*>(p));
  }
  return stacks[i];
}

#if defined(__x86_64__) && !defined(SIMT_EMU_USE_UCONTEXT)
void switch_to(Context& from, Context& to) { simt_emu_switch(&from.sp, to.sp); }

void trampoline() {
  (*body)();
  fibers[cur].state = DONE;
  switch_to(fibers[cur].ctx, sched_ctx);
  abort();  // a finished fiber is never resumed
}

void make_fiber(Context& c, char* stack_lo, size_t size) {
  uintptr_t top = (reinterpret_cast<uintptr_t>(stack_lo) + size) & ~uintptr_t(15);
  void** p = reinterpret_cast<void**>(top);
  p[-1] = nullptr;                                   // return address of trampoline (never used)
  p[-2] = reinterpret_cast<void*>(&trampoline);      // popped by `ret`; rsp % 16 == 8 at entry as the ABI wants
  for (int k = 3; k <= 8; k++) p[-k] = nullptr;      // rbp rbx r12 r13 r14 r15
  uint32_t* csr = reinterpret_cast<uint32_t*>(&p[-9]);
  csr[0] = 0x1F80;                                   // MXCSR default
  csr[1] = 0x037F;                                   // x87 control word default
  c.sp = &p[-9];
}
#else
void switch_to(Context& from, Context& to) { swapcontext(&from.uc, &to.uc); }

void trampoline() {
  (*body)();
  fibers[cur].state = DONE;
  // returning follows uc_link back to the scheduler
}

void make_fiber(Context& c, char* stack_lo, size_t size) {
  getcontext(&c.uc);
  c.uc.uc_stack.ss_sp = stack_lo;
  c.uc.uc_stack.ss_size = size;
  c.uc.uc_link = &sched_ctx.uc;
  makecontext(&c.uc, trampoline, 0);
}
#endif

void yield_to_scheduler() {
  const int me = cur;
  switch_to(fibers[me].ctx, sched_ctx);
}

[[noreturn]] void die(const char* what) {
  fprintf(stderr, "simt_emu: %s (block %u,%u,%u)\n", what, blockIdx.x, blockIdx.y, blockIdx.z);
  for (size_t i = 0; i < fibers.size(); i++)
    if (fibers[i].state != DONE && fibers[i].state != RUNNABLE)
      fprintf(stderr, "  thread %zu: %s mask %08x\n", i, fibers[i].state == WAIT_WARP ? "warp collective" : "__syncthreads",
              fibers[i].wait_mask);
  abort();
}

// Release a warp-level barrier if every live lane named by the mask of the first waiting lane waits with that mask.
bool try_release_warp(int w, int nthreads) {
  const int lo = w * 32, hi = (lo + 32 < nthreads) ? lo + 32 : nthreads;
  int first = -1;
  for (int i = lo; i < hi; i++)
    if (fibers[i].state == WAIT_WARP) { first = i; break; }
  if (first < 0) return false;
  const unsigned mask = fibers[first].wait_mask;
  for (int i = lo; i < hi; i++) {
    if (!((mask >> (i - lo)) & 1u) || fibers[i].state == DONE) continue;
    if (fibers[i].state != WAIT_WARP || fibers[i].wait_mask != mask) return false;
  }
  for (int i = lo; i < hi; i++)
    if (((mask >> (i - lo)) & 1u) && fibers[i].state == WAIT_WARP) fibers[i].state = RUNNABLE;
  return true;
}

// Order in which the runnable lanes of a warp (and the warps of a CTA) get the CPU between barriers.  The hardware
// gives no ordering guarantee between lanes that are not separated by a barrier, so a kernel must give the same
// result under every order: SIMT_EMU_ORDER=reverse runs lanes and warps from the top down, SIMT_EMU_ORDER=random[:seed]
// reshuffles them at every scheduling round (xorshift; deterministic for a given seed).  A shared-memory hand-off
// that only works because lane i happens to run before lane j shows up as a wrong result under one of them.
enum Order { FORWARD, REVERSE, RANDOM };
Order sched_order() {
  static Order o = [] {
    const char* e = getenv("SIMT_EMU_ORDER");
    if (!e) return FORWARD;
    if (!strncmp(e, "reverse", 7)) return REVERSE;
    if (!strncmp(e, "random", 6)) return RANDOM;
    return FORWARD;
  }();
  return o;
}
uint64_t rng_state = [] {
  const char* e = getenv("SIMT_EMU_ORDER");
  const char* c = e ? strchr(e, ':') : nullptr;
  return c ? strtoull(c + 1, nullptr, 10) * 2654435761ull + 88172645463325252ull : 88172645463325252ull;
}();
inline uint64_t rng_next() {
  rng_state ^= rng_state << 13;
  rng_state ^= rng_state >> 7;
  rng_state ^= rng_state << 17;
  return rng_state;
}
void make_order(int* idx, int n) {
  for (int i = 0; i < n; i++) idx[i] = i;
  const Order o = sched_order();
  if (o == REVERSE) {
    for (int i = 0; i < n; i++) idx[i] = n - 1 - i;
  } else if (o == RANDOM) {
    for (int i = n - 1; i > 0; i--) {
      const int j = (int)(rng_next() % (uint64_t)(i + 1));
      const int t = idx[i]; idx[i] = idx[j]; idx[j] = t;
    }
  }
}

void run_cta(int nthreads) {
  const int nwarps = (nthreads + 31) / 32;
  int worder[32], lorder[32];
  for (;;) {
    bool progress = false, all_done = true;
    make_order(worder, nwarps);
    for (int wi = 0; wi < nwarps; wi++) {
      const int w = worder[wi];
      const int lo = w * 32, hi = (lo + 32 < nthreads) ? lo + 32 : nthreads;
      make_order(lorder, hi - lo);
      for (int li = 0; li < hi - lo; li++) {
        const int i = lo + lorder[li];
        if (fibers[i].state != RUNNABLE) continue;
        cur = i;
        threadIdx = fibers[i].tid;
        switch_to(sched_ctx, fibers[i].ctx);
        progress = true;
      }
      while (try_release_warp(w, nthreads)) progress = true;
    }
    bool any_cta_wait = false, all_live_wait = true;
    for (int i = 0; i < nthreads; i++) {
      if (fibers[i].state == DONE) continue;
      all_done = false;
      if (fibers[i].state == WAIT_CTA) any_cta_wait = true;
      else all_live_wait = false;
    }
    if (all_done) return;
    if (any_cta_wait && all_live_wait) {
      for (int i = 0; i < nthreads; i++)
        if (fibers[i].state == WAIT_CTA) fibers[i].state = RUNNABLE;
      progress = true;
    }
    if (!progress) die("deadlock: a barrier or warp collective is not reached by every thread it names");
  }
}

}  // namespace

int lane_id() { return (int)((threadIdx.x + threadIdx.y * blockDim.x + threadIdx.z * blockDim.x * blockDim.y) & 31u); }
void* dyn_smem_ptr() { return dyn_smem; }
long long launches() { return n_launches; }

void barrier_warp(unsigned mask) {
  if (cur < 0) die("warp collective outside a kernel");
  if (!((mask >> lane_id()) & 1u)) die("a thread executes a *_sync collective whose mask does not name it");
  if (++fibers[cur].ncoll > max_coll) max_coll = fibers[cur].ncoll;
  fibers[cur].state = WAIT_WARP;
  fibers[cur].wait_mask = mask;
  yield_to_scheduler();
}

void barrier_cta() {
  if (cur < 0) die("__syncthreads outside a kernel");
  fibers[cur].state = WAIT_CTA;
  fibers[cur].wait_mask = 0;
  yield_to_scheduler();
}

uint64_t exchange(unsigned mask, uint64_t bits, int src_lane) {
  const int me = cur, w = me >> 5, lane = me & 31;
  const unsigned seq = ++fibers[me].parity, slot = seq & 1u;
  xchg[w][slot][lane] = bits;
  xtag[w][slot][lane] = seq;
  barrier_warp(mask);
  // a lane can run at most one exchange ahead of the slowest lane of its collective, so two slots suffice; a
  // source lane that did not take part in this exchange (not named, or exited earlier) yields the caller's own value
  if (src_lane < 0 || src_lane > 31 || !((mask >> src_lane) & 1u)) return bits;
  if (xtag[w][slot][src_lane] != seq) return bits;
  return xchg[w][slot][src_lane];
}

unsigned ballot(unsigned mask, int pred) {
  const int me = cur, w = me >> 5, lane = me & 31;
  const unsigned seq = ++fibers[me].parity, slot = seq & 1u;
  xchg[w][slot][lane] = pred ? 1u : 0u;
  xtag[w][slot][lane] = seq;
  barrier_warp(mask);
  unsigned r = 0;
  for (int l = 0; l < 32; l++)
    if (((mask >> l) & 1u) && xtag[w][slot][l] == seq && xchg[w][slot][l]) r |= 1u << l;
  return r;
}

double rcp_approx_f64(double x) {
  // MUFU.RCP64H produces the high word of 1/x (about 20 good mantissa bits) and a zero low word
  double r = 1.0 / x;
  uint64_t b;
  memcpy(&b, &r, 8);
  b &= 0xffffffff00000000ull;
  memcpy(&r, &b, 8);
  return r;
}

// the runtime's per-host-thread last error, and the dynamic shared-memory limit set per kernel
thread_local int t_last_error = 0;
std::mutex smem_attr_mu;
std::vector<std::pair<const void*, size_t>> smem_attr;

int last_error(bool reset) {
  const int e = t_last_error;
  if (reset) t_last_error = 0;
  return e;
}

int set_max_dyn_smem(const void* kernel, int bytes) {
  if (bytes < 0 || (size_t)bytes > kDynSmemOptinMax) return cudaErrorInvalidValue;
  std::lock_guard<std::mutex> lk(smem_attr_mu);
  for (auto& a : smem_attr)
    if (a.first == kernel) { a.second = (size_t)bytes; return cudaSuccess; }
  smem_attr.emplace_back(kernel, (size_t)bytes);
  return cudaSuccess;
}

size_t max_dyn_smem(const void* kernel) {
  std::lock_guard<std::mutex> lk(smem_attr_mu);
  for (const auto& a : smem_attr)
    if (a.first == kernel) return a.second;
  return kDynSmemDefault;
}

// one line per launch, "<kernel expression> | <launching function> | <threads> | <dynamic shared bytes> | <collectives>",
// where <collectives> is the most warp collectives (shuffles, votes, __syncwarp) any thread of the launch executed (0
// for a refused launch): tests read it to see which kernel a launch plan chose, and whether a kernel did any work
// after its entry test (simt_emu_launch_log)
std::mutex log_mu;
std::string launch_log;

void log_launch(const char* what, const char* where, dim3 block, size_t dyn_smem_bytes, long long collectives) {
  std::lock_guard<std::mutex> lk(log_mu);
  char tail[96];
  snprintf(tail, sizeof tail, " | %u | %zu | %lld\n", block.x * block.y * block.z, dyn_smem_bytes, collectives);
  if (launch_log.size() > (1u << 22)) launch_log.clear();   // nobody reads it: keep it bounded
  launch_log += std::string(what) + " | " + where + tail;
}

void launch(const void* kernel, dim3 grid, dim3 block, size_t dyn_smem_bytes, const std::function<void()>& kernel_body,
            const char* what, const char* where) {
  if (dyn_smem_bytes > max_dyn_smem(kernel)) {   // refused before it runs, as the runtime refuses it
    log_launch(what, where, block, dyn_smem_bytes, 0);
    fprintf(stderr, "simt_emu: launch refused: %zu bytes of dynamic shared memory, the kernel may use %zu\n",
            dyn_smem_bytes, max_dyn_smem(kernel));
    t_last_error = cudaErrorInvalidValue;
    return;
  }
  // one grid at a time: host threads that launch concurrently (the chunk workers of capi.cu) are serialised here
  static std::mutex launch_mu;
  std::lock_guard<std::mutex> lk(launch_mu);
  if (cur >= 0) die("nested launch");
  const int nthreads = (int)(block.x * block.y * block.z);
  if (nthreads <= 0 || nthreads > 1024) die("bad block size");
  n_launches++;
  max_coll = 0;
  if (dyn_smem_bytes + 64 > dyn_smem_cap) {
    free(dyn_smem);
    dyn_smem_cap = dyn_smem_bytes + 64;
    if (posix_memalign(&dyn_smem, 128, dyn_smem_cap)) die("out of memory");
  }
  const int nwarps = (nthreads + 31) / 32;
  xchg_store.assign((size_t)nwarps * 64, 0);
  xchg = reinterpret_cast<uint64_t(*)[2][32]>(xchg_store.data());
  xtag_store.assign((size_t)nwarps * 64, 0);
  xtag = reinterpret_cast<unsigned(*)[2][32]>(xtag_store.data());
  fibers.resize(nthreads);
  body = &kernel_body;
  blockDim = block;
  gridDim = grid;
  for (unsigned bz = 0; bz < grid.z; bz++)
    for (unsigned by = 0; by < grid.y; by++)
      for (unsigned bx = 0; bx < grid.x; bx++) {
        blockIdx = uint3{bx, by, bz};
        memset(dyn_smem, 0xFF, dyn_smem_cap);  // uninitialised shared memory reads as NaN
        std::fill(xtag_store.begin(), xtag_store.end(), 0u);
        for (int i = 0; i < nthreads; i++) {
          Fiber& f = fibers[i];
          make_fiber(f.ctx, stack_for(i) + 4096, kStack - 4096);
          f.state = RUNNABLE;
          f.wait_mask = 0;
          f.parity = 0;
          f.ncoll = 0;
          f.tid = uint3{(unsigned)i % block.x, ((unsigned)i / block.x) % block.y, (unsigned)i / (block.x * block.y)};
        }
        run_cta(nthreads);
      }
  cur = -1;
  body = nullptr;
  log_launch(what, where, block, dyn_smem_bytes, max_coll);
}

}  // namespace simt_emu

// "device" allocations: host memory, poisoned so that reads of never-written device memory show up as NaNs
cudaError_t cudaMalloc(void** p, size_t bytes) {
  void* q = nullptr;
  if (posix_memalign(&q, 256, bytes ? bytes : 256)) return cudaErrorMemoryAllocation;
  memset(q, 0xFF, bytes);
  *p = q;
  return cudaSuccess;
}
cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
cudaError_t cudaHostAlloc(void** p, size_t bytes, unsigned) {
  void* q = nullptr;
  if (posix_memalign(&q, 256, bytes ? bytes : 256)) return cudaErrorMemoryAllocation;
  *p = q;
  return cudaSuccess;
}
cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }

extern "C" long long simt_emu_launches() { return simt_emu::launches(); }
// returns the launch log's length; with a buffer, copies the log into it (NUL-terminated, truncated to len) and clears it
extern "C" long long simt_emu_launch_log(char* buf, long long len) {
  std::lock_guard<std::mutex> lk(simt_emu::log_mu);
  const long long n = (long long)simt_emu::launch_log.size();
  if (buf && len > 0) {
    const long long k = n < len - 1 ? n : len - 1;
    memcpy(buf, simt_emu::launch_log.data(), (size_t)k);
    buf[k] = 0;
    simt_emu::launch_log.clear();
  }
  return n;
}

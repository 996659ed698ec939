// simt.cpp (TEST INFRASTRUCTURE) -- fiber scheduler and runtime-API stubs behind
// tests/native/emul/cuda_runtime.h.  See that header for the execution model.
#include <cuda_runtime.h>
#include <stdio.h>
#include <sys/mman.h>

#include <dlfcn.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

// MS_TSAN (tools/emul_tsan.sh): kernels + engine are compiled with -fsanitize=thread, this file is
// not.  Every emulated thread is a TSan fiber; the scheduler's context switches carry no
// synchronisation, __syncthreads() and warp collectives are release/acquire pairs, a kernel launch
// is ordered after the host code before it and before the host code after it, and CTAs of a launch
// are chained (their __shared__ statics are the same host memory).  What TSan then reports is two
// threads of ONE CTA touching the same shared / global location with no barrier in between.
#ifdef MS_TSAN
extern "C" {
void* __tsan_get_current_fiber(void);
void* __tsan_create_fiber(unsigned flags);
void __tsan_destroy_fiber(void* fiber);
void __tsan_switch_to_fiber(void* fiber, unsigned flags);
void __tsan_acquire(void* addr);
void __tsan_release(void* addr);
}
#define TSAN(x) x
#else
#define TSAN(x)
#endif

namespace simt {

thread_local Tls tls;

// ------------------------------------------------------------------ context switch (x86-64 SysV)
extern "C" void simt_switch(void** save_sp, void* load_sp);
asm(R"(
.text
.globl simt_switch
.type simt_switch,@function
simt_switch:
  pushq %rbp
  pushq %rbx
  pushq %r12
  pushq %r13
  pushq %r14
  pushq %r15
  movq %rsp, (%rdi)
  movq %rsi, %rsp
  popq %r15
  popq %r14
  popq %r13
  popq %r12
  popq %rbx
  popq %rbp
  ret
.size simt_switch,.-simt_switch
)");

constexpr size_t kStack = 128 << 10;
constexpr unsigned kMaxThreads = 1024;

struct Warp {
  unsigned live = 0;       // lanes that have not exited
  unsigned count = 0;      // lanes waiting in the current collective
  unsigned gen = 0;
  int op = 0, arg0 = 0;
  bool arrived[32];
  uint64_t in[32];
  int arg[32];
  uint64_t out[2][32];
};

struct Sched {
  char* stacks = nullptr;            // kMaxThreads * kStack
  void* sp[kMaxThreads];
  bool done[kMaxThreads];
  void* main_sp = nullptr;
  unsigned nt = 0, live = 0, cur = 0;
  unsigned bar_count = 0, bar_gen = 0;
  int bar_or[2] = {0, 0};
  Warp warps[kMaxThreads / 32];
  const std::function<void()>* body = nullptr;
  unsigned char* smem = nullptr;
  uint64_t progress = 0;
  void* fib[kMaxThreads];            // MS_TSAN: TSan fiber of each emulated thread
  void* main_fib = nullptr;
  char sync_bar, sync_launch_begin, sync_launch_end, sync_cta_chain;   // MS_TSAN: addresses to release / acquire on
  char sync_warp[kMaxThreads / 32];
  unsigned bar_calls[kMaxThreads];   // MS_TSAN self-test
};
static thread_local Sched* g_s = nullptr;          // the scheduler of the launch that runs now
static thread_local Sched* g_top = nullptr;        // top-level launches
static thread_local Sched* g_nested = nullptr;     // MS_EMUL_STREAMS: work run while a top-level CTA is parked

static Sched* new_sched() {
  Sched* s = new Sched();
  s->stacks = (char*)mmap(nullptr, (size_t)kMaxThreads * kStack, PROT_READ | PROT_WRITE,
                          MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
  if (s->stacks == (char*)MAP_FAILED) { fprintf(stderr, "simt: mmap failed\n"); abort(); }
  if (posix_memalign((void**)&s->smem, 128, 256 << 10)) abort();
  return s;
}

static Sched* sched() {
  if (!g_s) g_s = g_top = new_sched();
  return g_s;
}

static void maybe_interleave();   // MS_EMUL_STREAMS, below
thread_local bool in_cta_pool = false;   // MS_EMUL_CTAS, below

[[noreturn]] static void die(const char* what) {
  fprintf(stderr, "simt emulator: %s (block %u thread %u)\n", what, tls.bid.x, tls.tid.x);
  abort();
}

static void yield_to_scheduler() {
  Sched* s = g_s;
  const unsigned me = s->cur;
  TSAN(__tsan_switch_to_fiber(s->main_fib, 1);)
  simt_switch(&s->sp[me], s->main_sp);
  tls.tid.x = me;   // resumed
}

static void release_barrier(Sched* s) {
  s->bar_count = 0;
  s->bar_or[(s->bar_gen + 1) & 1] = 0;
  s->bar_gen++;
  s->progress++;
}

static void finish_collective(Warp& w);

static void fiber_main() {
  Sched* s = g_s;
  TSAN(__tsan_acquire(&s->sync_launch_begin); __tsan_acquire(&s->sync_cta_chain);)
  (*s->body)();
  TSAN(__tsan_release(&s->sync_launch_end); __tsan_release(&s->sync_cta_chain);)
  const unsigned me = s->cur;
  s->done[me] = true;
  s->live--;
  s->progress++;
  Warp& w = s->warps[me >> 5];
  w.live--;
  // an exiting thread may complete what the others are waiting for
  if (s->bar_count && s->bar_count == s->live) release_barrier(s);
  if (w.count && w.count == w.live) finish_collective(w);
  void* dummy;
  TSAN(__tsan_switch_to_fiber(s->main_fib, 1);)
  simt_switch(&dummy, s->main_sp);
  die("resumed a finished thread");
}

static int barrier(int pred, bool plain);
void sync_threads() { (void)barrier(0, true); }
int sync_threads_or(int pred) { return barrier(pred, false); }

static int barrier(int pred, bool plain) {
  if (in_cta_pool && g_s->bar_count == 0) cta_switch(SW_BARRIER);   // the CTA's first thread to arrive
  maybe_interleave();
  Sched* s = g_s;
#ifdef MS_TSAN
  // self-test of the race check: MS_TSAN_SKIP_BARRIER=k turns every k-th barrier of every CTA into
  // a no-op (the same one for all its threads), which TSan must then report
  static const unsigned skip = getenv("MS_TSAN_SKIP_BARRIER") ? (unsigned)atoi(getenv("MS_TSAN_SKIP_BARRIER")) : 0;
  if (skip && plain && (++s->bar_calls[s->cur] % skip) == 0) return 0;
#endif
  const unsigned gen = s->bar_gen;
  if (pred) s->bar_or[gen & 1] = 1;
  s->bar_count++;
  s->progress++;
  TSAN(__tsan_release(&s->sync_bar);)
  if (s->bar_count == s->live) release_barrier(s);
  while (s->bar_gen == gen) yield_to_scheduler();
  TSAN(__tsan_acquire(&s->sync_bar);)
  return s->bar_or[gen & 1];
}

static void finish_collective(Warp& w) {
  uint64_t* out = w.out[w.gen & 1];
  uint64_t any = 0, ballot = 0;
  for (int l = 0; l < 32; l++)
    if (w.arrived[l] && w.in[l]) { any = 1; ballot |= 1ull << l; }
  for (int l = 0; l < 32; l++) {
    if (!w.arrived[l]) continue;
    switch (w.op) {
      case OP_SHFL_UP: out[l] = (l >= w.arg0 && w.arrived[l - w.arg0]) ? w.in[l - w.arg0] : w.in[l]; break;
      case OP_SHFL_XOR: out[l] = w.arrived[l ^ w.arg0] ? w.in[l ^ w.arg0] : w.in[l]; break;
      case OP_SHFL_IDX: { const int src = w.arg[l] & 31; out[l] = w.arrived[src] ? w.in[src] : w.in[l]; break; }
      case OP_MATCH_ANY: {
        uint64_t m = 0;
        for (int q = 0; q < 32; q++) if (w.arrived[q] && w.in[q] == w.in[l]) m |= 1ull << q;
        out[l] = m;
        break;
      }
      case OP_ANY: out[l] = any; break;
      case OP_BALLOT: out[l] = ballot; break;
      default: die("unknown warp collective");
    }
  }
  for (int l = 0; l < 32; l++) w.arrived[l] = false;
  w.count = 0;
  w.op = 0;
  w.gen++;
  g_s->progress++;
}

uint64_t warp_op(int op, unsigned mask, uint64_t v, int arg) {
  Sched* s = g_s;
  const unsigned me = s->cur, lane = me & 31;
  Warp& w = s->warps[me >> 5];
  if (!((mask >> lane) & 1u)) die("warp collective called by a lane outside its mask");
  if (w.count == 0) {
    w.op = op;
    w.arg0 = arg;
  } else if (w.op != op || (op != OP_SHFL_IDX && w.arg0 != arg)) {
    die("divergent warp collective: lanes of one warp reached different __*_sync calls");
  }
  const unsigned gen = w.gen;
  w.arrived[lane] = true;
  w.in[lane] = v;
  w.arg[lane] = arg;
  w.count++;
  s->progress++;
  TSAN(__tsan_release(&s->sync_warp[me >> 5]);)
  if (w.count == w.live) finish_collective(w);
  while (w.gen == gen) yield_to_scheduler();
  TSAN(__tsan_acquire(&s->sync_warp[me >> 5]);)
  return w.out[gen & 1][lane];
}

void relax() {
  // a spin-wait (k_barrier polling a peer's flag): let the other host threads (shards) run AND
  // the other fibers of this CTA, which on a GPU would be running concurrently
  std::this_thread::yield();
  if (in_cta_pool) cta_switch(SW_SPIN);   // ... and the other resident CTAs of this launch
  if (g_s && g_s->body) {
    g_s->progress++;
    yield_to_scheduler();
  }
}

unsigned char* dyn_smem() { return sched()->smem; }

static void run_cta(Sched* s, unsigned nt) {
  s->nt = nt;
  s->live = nt;
  s->bar_count = 0;
  s->bar_or[0] = s->bar_or[1] = 0;
  const unsigned nw = (nt + 31) / 32;
  for (unsigned w = 0; w < nw; w++) {
    Warp& W = s->warps[w];
    W.live = (w + 1) * 32 <= nt ? 32 : nt - w * 32;
    W.count = 0;
    W.op = 0;
    for (int l = 0; l < 32; l++) W.arrived[l] = false;
  }
  for (unsigned t = 0; t < nt; t++) {
    s->done[t] = false;
    s->bar_calls[t] = 0;
    uintptr_t top = (uintptr_t)(s->stacks + (size_t)(t + 1) * kStack) & ~(uintptr_t)15;
    void** p = (void**)top;
    p[-1] = nullptr;                  // return address slot of fiber_main (never used)
    p[-2] = (void*)&fiber_main;       // popped by simt_switch's ret
    for (int r = 3; r <= 8; r++) p[-r] = nullptr;   // rbp rbx r12-r15
    s->sp[t] = (void*)(p - 8);
    TSAN(s->fib[t] = __tsan_create_fiber(0);)
  }
  TSAN(s->main_fib = __tsan_get_current_fiber();)
  // MS_EMUL_ORDER: 0 = threads resume in index order (default), 1 = reverse, 2 = a different
  // pseudo-random order every sweep.  Results must not depend on it: a missing barrier usually does.
  static const int order_mode = getenv("MS_EMUL_ORDER") ? atoi(getenv("MS_EMUL_ORDER")) : 0;
  static thread_local uint32_t lcg = 12345u;
  while (s->live) {
    const uint64_t before = s->progress;
    uint32_t mul = 1, add = 0;
    if (order_mode == 2) {            // t -> (t * odd + add) mod 2^k is a permutation of [0, 2^k)
      lcg = lcg * 1664525u + 1013904223u;
      mul = (lcg >> 8) | 1u;
      add = lcg >> 20;
    }
    unsigned span = 1;
    while (span < nt) span <<= 1;
    for (unsigned u = 0; u < span; u++) {
      unsigned t = u;
      if (order_mode == 1) t = span - 1 - u;
      else if (order_mode == 2) t = (u * mul + add) & (span - 1);
      if (t >= nt) continue;
      if (s->done[t]) continue;
      s->cur = t;
      tls.tid.x = t;
      TSAN(__tsan_switch_to_fiber(s->fib[t], 1);)
      simt_switch(&s->main_sp, s->sp[t]);
    }
    if (s->live && s->progress == before) die("deadlock: no thread of the CTA can make progress");
  }
  TSAN(for (unsigned t = 0; t < nt; t++) __tsan_destroy_fiber(s->fib[t]);)
}

// MS_EMUL_PROFILE=1: wall time per (grid, block) launch shape, printed at exit
struct ProfRow { unsigned grid, block; uint64_t n; double sec; };
static ProfRow g_prof[64];
static int g_nprof = 0;
static void prof_dump() {
  for (int i = 0; i < g_nprof; i++)
    fprintf(stderr, "simt profile: grid %5u block %4u launches %8llu total %.3f s (%.1f us each)\n", g_prof[i].grid,
            g_prof[i].block, (unsigned long long)g_prof[i].n, g_prof[i].sec, 1e6 * g_prof[i].sec / (double)g_prof[i].n);
}
static void launch_impl(unsigned grid, unsigned block, size_t dyn, const std::function<void()>& body);
void launch(unsigned grid, unsigned block, size_t dyn, const std::function<void()>& body) {
  static const bool profile = getenv("MS_EMUL_PROFILE") != nullptr;
  if (!profile) { launch_impl(grid, block, dyn, body); return; }
  const auto t0 = std::chrono::steady_clock::now();
  launch_impl(grid, block, dyn, body);
  const double dt = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  int i = 0;
  while (i < g_nprof && !(g_prof[i].grid == grid && g_prof[i].block == block)) i++;
  if (i == g_nprof) {
    if (g_nprof == 64) return;
    if (g_nprof == 0) atexit(prof_dump);
    g_prof[g_nprof++] = ProfRow{grid, block, 0, 0.0};
  }
  g_prof[i].n++;
  g_prof[i].sec += dt;
}
static bool ctas_launch(unsigned grid, unsigned block, size_t dyn, const std::function<void()>& body);
static void launch_impl(unsigned grid, unsigned block, size_t dyn, const std::function<void()>& body) {
  if (block == 0 || block > kMaxThreads) die("bad block size");
  if (dyn > (256u << 10)) die("dynamic shared memory too large");
  if (in_cta_pool) die("nested kernel launch");
  if (ctas_launch(grid, block, dyn, body)) return;
  Sched* s = sched();
  if (s->body) die("nested kernel launch");
  s->body = &body;
  tls.bdim = dim3{block, 1, 1};
  tls.gdim = dim3{grid, 1, 1};
  tls.tid = uint3{0, 0, 0};
  static const int order_mode = getenv("MS_EMUL_ORDER") ? atoi(getenv("MS_EMUL_ORDER")) : 0;
  TSAN(__tsan_release(&s->sync_launch_begin);)
  for (unsigned bb = 0; bb < grid; bb++) {
    const unsigned b = order_mode ? grid - 1 - bb : bb;     // CTAs must not depend on launch order either
    tls.bid = uint3{b, 0, 0};
    memset(s->smem, 0xCD, dyn);
    run_cta(s, block);
  }
  TSAN(__tsan_acquire(&s->sync_launch_end);)
  s->body = nullptr;
}

}  // namespace simt

// ------------------------------------------------------------------ MS_EMUL_STREAMS: asynchronous streams
// A stream is a FIFO of operations owned by the host thread that enqueued them; event k of a stream is
// complete once `done` has reached its position.  Nothing runs out of stream order, nothing runs before a
// cudaStreamWaitEvent dependency is met; apart from that the seeded choices below decide what runs when.
struct simt_stream;
struct simt_event {
  std::chrono::steady_clock::time_point t;
  simt_stream* s = nullptr;   // the stream and position of the last record (nullptr: complete)
  uint64_t seq = 0;
};
struct simt_op {
  enum Kind { LAUNCH, WORK, RECORD, WAIT } kind;
  std::function<void()> fn;   // LAUNCH: the kernel body; WORK: a copy or memset
  const void* kern = nullptr;
  unsigned grid = 0, block = 0;
  size_t dyn = 0;
  simt_event* ev = nullptr;   // RECORD
  simt_stream* dep = nullptr; // WAIT: (stream, position) of the awaited record, fixed when enqueued
  uint64_t dep_seq = 0;
};
struct simt_stream {
  std::deque<simt_op> q;
  uint64_t enq = 0, done = 0;
  std::thread::id owner;
};

namespace simt {

static std::mutex g_reg_mu;                        // the stream registry and the interleave counters
static std::vector<simt_stream*> g_streams;
static std::map<std::pair<const void*, const void*>, uint64_t> g_pairs;   // (parked kernel, kernel run meanwhile)
static std::atomic<int64_t> g_seed{-2};            // -2: not read yet, -1: synchronous streams
static std::atomic<uint64_t> g_seed_gen{0};
static thread_local uint64_t t_rng = 0, t_rng_gen = ~0ull;
static thread_local simt_stream* t_run_stream = nullptr;   // stream of the top-level launch running now
static thread_local const void* t_run_kern = nullptr;
static thread_local bool t_nested = false;
static thread_local const void* t_kern = nullptr;          // the kernel launch() is about to run (MS_EMUL_CTAS counters)
static std::thread::id host_thread();                      // MS_EMUL_CTAS: the thread that launched, seen from a worker

static bool streams_async() {
  int64_t v = g_seed.load();
  if (v == -2) {
    const char* e = getenv("MS_EMUL_STREAMS");
    int64_t want = (e && *e) ? (int64_t)strtoull(e, nullptr, 0) : -1;
    g_seed.compare_exchange_strong(v, want);
    v = g_seed.load();
  }
#ifdef MS_TSAN
  return false;      // the TSan fiber bookkeeping assumes one launch at a time
#else
  return v >= 0;
#endif
}

static uint64_t rng() {                            // splitmix64 of the seed, per host thread
  if (t_rng_gen != g_seed_gen.load()) { t_rng = (uint64_t)g_seed.load(); t_rng_gen = g_seed_gen.load(); }
  uint64_t z = (t_rng += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

static bool dep_met(const simt_op& op) { return op.dep == nullptr || op.dep->done >= op.dep_seq; }

static void exec_head(simt_stream* st);
static void run_until(simt_stream* st, uint64_t seq);

static void run_launch(simt_stream* st, const simt_op& op) {
  simt_stream* const ps = t_run_stream;
  const void* const pk = t_run_kern;
  if (!t_nested) { t_run_stream = st; t_run_kern = op.kern; }
  t_kern = op.kern;
  launch(op.grid, op.block, op.dyn, op.fn);
  t_run_stream = ps; t_run_kern = pk;
}

static void exec_head(simt_stream* st) {
  simt_op op = std::move(st->q.front());
  st->q.pop_front();
  switch (op.kind) {
    case simt_op::LAUNCH: run_launch(st, op); break;
    case simt_op::WORK: op.fn(); break;
    case simt_op::RECORD: op.ev->t = std::chrono::steady_clock::now(); break;
    case simt_op::WAIT:
      if (!dep_met(op)) {
        if (t_nested) die("MS_EMUL_STREAMS: nested work waits on an event");
        run_until(op.dep, op.dep_seq);
      }
      break;
  }
  st->done++;
}

// streams of this host thread (other than `except`) whose next operation may run now, skipping launches of
// `not_kern` (its __shared__ statics are in use by the parked CTA)
static simt_stream* pick_ready(simt_stream* except, const void* not_kern) {
  std::vector<simt_stream*> ready;
  {
    std::lock_guard<std::mutex> g(g_reg_mu);
    const std::thread::id me = host_thread();
    for (simt_stream* st : g_streams) {
      if (st == except || st->owner != me || st->q.empty()) continue;
      const simt_op& h = st->q.front();
      if (h.kind == simt_op::WAIT && !dep_met(h)) continue;
      if (h.kind == simt_op::LAUNCH && not_kern && h.kern == not_kern) continue;
      ready.push_back(st);
    }
  }
  return ready.empty() ? nullptr : ready[rng() % ready.size()];
}

static void run_until(simt_stream* st, uint64_t seq) {
  while (st->done < seq) {
    if (st->q.empty()) die("MS_EMUL_STREAMS: waiting for work that was never enqueued");
    const simt_op& h = st->q.front();
    if (h.kind == simt_op::WAIT && !dep_met(h)) { run_until(h.dep, h.dep_seq); continue; }
    if (!t_nested && (rng() & 1)) {            // the GPU may as well have started another stream's work first
      if (simt_stream* o = pick_ready(st, nullptr)) { exec_head(o); continue; }
    }
    exec_head(st);
  }
}

static void drain_all() {
  if (!streams_async()) return;
  if (t_nested) die("MS_EMUL_STREAMS: host synchronisation inside a kernel");
  for (;;) {
    simt_stream* pending = nullptr;
    {
      std::lock_guard<std::mutex> g(g_reg_mu);
      const std::thread::id me = std::this_thread::get_id();
      for (simt_stream* st : g_streams)
        if (st->owner == me && !st->q.empty()) { pending = st; break; }
    }
    if (!pending) return;
    run_until(pending, pending->enq);
  }
}

static void push(simt_stream* st, simt_op op) {
  st->owner = std::this_thread::get_id();
  st->q.push_back(std::move(op));
  st->enq++;
}

// at a __syncthreads() of a top-level kernel: maybe run one ready operation of another stream to completion
static void maybe_interleave() {
  if (t_nested || !t_run_stream || g_s != g_top || !streams_async()) return;
  if (rng() % 8) return;
  simt_stream* o = pick_ready(t_run_stream, t_run_kern);
  if (!o) return;
  if (o->q.front().kind == simt_op::LAUNCH) {
    std::lock_guard<std::mutex> g(g_reg_mu);
    g_pairs[{t_run_kern, o->q.front().kern}]++;
  }
  if (!g_nested) g_nested = new_sched();
  const Tls saved = tls;
  const bool pooled = in_cta_pool;
  g_s = g_nested;
  t_nested = true;
  in_cta_pool = false;       // MS_EMUL_CTAS: the nested work runs to completion before any other CTA resumes
  exec_head(o);
  in_cta_pool = pooled;
  t_nested = false;
  g_s = g_top;
  tls = saved;
}

void enqueue_launch(cudaStream_t st, const void* kern, unsigned grid, unsigned block, size_t dyn,
                    std::function<void()> body) {
  if (!st || !streams_async() || t_nested) {   // nested work launches nothing, so this is host code
    drain_all();
    t_kern = kern;
    launch(grid, block, dyn, body);
    return;
  }
  simt_op op{simt_op::LAUNCH};
  op.fn = std::move(body);
  op.kern = kern; op.grid = grid; op.block = block; op.dyn = dyn;
  push(st, std::move(op));
}

// ------------------------------------------------------------------ MS_EMUL_CTAS: CTAs of a launch concurrently
// A launch of two or more CTAs runs on a pool of worker host threads that belongs to the launching host thread
// (a shard has its own): one resident CTA per worker, 2 x MS_EMUL_SMS workers (a persistent k_round grid is SMs x
// one CTA, so it is fully resident), and a worker whose CTA finishes takes the next block index.  Each worker has
// its own fiber scheduler and, through thread_local, its own __shared__ statics.  A baton lets exactly one thread
// of the pool (or the launcher) run at a time, so a run is a function of the seed: at each switch point a seeded
// choice may park the whole running CTA and hand the baton to another resident one.  A spin-wait always offers it.
struct CtaPool {
  std::mutex mu;
  std::condition_variable cv;
  int turn = -1;                  // who holds the baton: a worker, or -1 = the launching thread
  bool quit = false;
  std::vector<std::thread> threads;
  std::vector<int> block;         // per worker: the block index of its CTA, -1 = none
  std::vector<int> hold;          // per worker: passes it stays parked for
  std::thread::id owner;
  // the launch in progress
  const std::function<void()>* body = nullptr;
  unsigned grid = 0, nthreads = 0, next = 0;
  size_t dyn = 0;
  simt_stream* run_stream = nullptr;
  const void* run_kern = nullptr;
  uint64_t passes = 0;            // baton passes from a CTA that had started and not finished
  uint64_t rng = 0, rng_gen = ~0ull;
  ~CtaPool() {
    { std::lock_guard<std::mutex> g(mu); quit = true; }
    cv.notify_all();
    for (auto& t : threads) t.join();
  }
};
static std::atomic<int64_t> g_cta_seed{-2};       // -2: not read yet, -1: off
static std::atomic<uint64_t> g_cta_gen{0};
static std::mutex g_cta_mu;                        // the counters below
static std::map<const void*, std::pair<uint64_t, uint64_t>> g_cta_counts;   // kernel -> (overlapped launches, passes)
static thread_local std::unique_ptr<CtaPool> t_own_pool;   // on a launching thread
static thread_local CtaPool* t_pool = nullptr;             // on a worker: its pool
static thread_local int t_worker = -1;

static std::thread::id host_thread() { return t_pool ? t_pool->owner : std::this_thread::get_id(); }

static bool ctas_on() {
  int64_t v = g_cta_seed.load();
  if (v == -2) {
    const char* e = getenv("MS_EMUL_CTAS");
    int64_t want = (e && *e) ? (int64_t)strtoll(e, nullptr, 0) : -1;
    if (want < -1) want = -1;
    g_cta_seed.compare_exchange_strong(v, want);
    v = g_cta_seed.load();
  }
#ifdef MS_TSAN
  return false;      // the TSan build keeps CTAs sequential (their __shared__ statics are chained on purpose)
#else
  return v >= 0;
#endif
}

static uint64_t cta_rng(CtaPool* P) {
  if (P->rng_gen != g_cta_gen.load()) { P->rng = (uint64_t)g_cta_seed.load() * 0x2545F4914F6CDD1Dull; P->rng_gen = g_cta_gen.load(); }
  uint64_t z = (P->rng += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// hands the baton to `to` and waits until it comes back (under the pool's lock: the hand-over orders memory)
static void hand_over(CtaPool* P, int to, int me) {
  std::unique_lock<std::mutex> lk(P->mu);
  P->turn = to;
  P->cv.notify_all();
  P->cv.wait(lk, [&] { return P->turn == me; });
}

void cta_switch(int why) {
  CtaPool* P = t_pool;
  const int me = t_worker;
  bool any = false;
  for (int w = 0; w < (int)P->block.size() && !any; w++) any = w != me && P->block[w] >= 0;
  if (!any) return;
  const uint64_t r = cta_rng(P);
  // how often each switch point passes: a CTA start one time in two, the CTA's first arrival at a barrier one in
  // four, an atomic or fence one in eight, a spin-wait always
  static const unsigned mask[] = {1, 3, 7, 7, 0};
  if (r & mask[why]) return;
  // A CTA parked here stays parked for the next 512-1535 switches one time in eight, and for 32-95 of them one time
  // in eight: an SM busy elsewhere, which is what lets a bounded poll such as wheel_block's give up on its publisher.
  // Held CTAs are passed over; a spin-wait that finds nobody else counts down their holds instead (so an unbounded
  // wait still reaches them), any other switch point takes a held CTA when nobody else is left.
  for (int& h : P->hold)
    if (h > 0) h--;
  if (why != SW_SPIN) {
    if (((r >> 40) & 7) == 1) P->hold[me] = 512 + (int)((r >> 45) & 1023);
    else if (((r >> 40) & 7) == 0) P->hold[me] = 32 + (int)((r >> 45) & 63);
  }
  int cand[256], n = 0;
  for (int pass = 0; pass < (why == SW_SPIN ? 1 : 2) && n == 0; pass++)
    for (int w = 0; w < (int)P->block.size(); w++)
      if (w != me && P->block[w] >= 0 && (pass || P->hold[w] == 0)) cand[n++] = w;
  if (!n) return;
  if (why != SW_START) P->passes++;
  hand_over(P, cand[(r >> 16) % (uint64_t)n], me);
}

static void free_sched(Sched* s) {
  if (!s) return;
  munmap(s->stacks, (size_t)kMaxThreads * kStack);
  free(s->smem);
  delete s;
}

static void cta_worker(CtaPool* P, int me) {
  t_pool = P;
  t_worker = me;
  g_s = g_top = new_sched();
  std::unique_lock<std::mutex> lk(P->mu);
  for (;;) {
    P->cv.wait(lk, [&] { return P->turn == me || P->quit; });
    if (P->quit) break;
    lk.unlock();
    t_run_stream = P->run_stream;            // MS_EMUL_STREAMS at a __syncthreads() of this launch
    t_run_kern = P->run_kern;
    while (P->block[me] >= 0) {
      tls.bdim = dim3{P->nthreads, 1, 1};
      tls.gdim = dim3{P->grid, 1, 1};
      tls.bid = uint3{(unsigned)P->block[me], 0, 0};
      tls.tid = uint3{0, 0, 0};
      in_cta_pool = true;
      cta_switch(SW_START);                  // a CTA may start late
      g_s->body = P->body;
      memset(g_s->smem, 0xCD, P->dyn);
      run_cta(g_s, P->nthreads);
      g_s->body = nullptr;
      in_cta_pool = false;
      P->block[me] = P->next < P->grid ? (int)P->next++ : -1;
    }
    t_run_stream = nullptr;
    t_run_kern = nullptr;
    lk.lock();
    int to = -1;                             // another resident CTA, else the launch is over
    for (int w = 0; w < (int)P->block.size() && to < 0; w++)
      if (P->block[w] >= 0) to = w;
    P->turn = to;
    P->cv.notify_all();
  }
  free_sched(g_top);
  free_sched(g_nested);
  g_s = g_top = g_nested = nullptr;
}

static bool ctas_launch(unsigned grid, unsigned block, size_t dyn, const std::function<void()>& body) {
  if (grid < 2 || t_nested || !ctas_on()) return false;
  const char* e = getenv("MS_EMUL_SMS");
  const int sms = e ? atoi(e) : 1;
  const unsigned resident = (unsigned)std::min(std::max(2 * sms, 2), 256);
  if (!t_own_pool) { t_own_pool.reset(new CtaPool()); t_own_pool->owner = std::this_thread::get_id(); }
  CtaPool* P = t_own_pool.get();
  while (P->threads.size() < resident) {
    P->block.push_back(-1);
    P->hold.push_back(0);
    P->threads.emplace_back(cta_worker, P, (int)P->threads.size());
  }
  P->body = &body;
  P->grid = grid;
  P->nthreads = block;
  P->dyn = dyn;
  P->run_stream = t_run_stream;
  P->run_kern = t_run_kern;
  P->passes = 0;
  const unsigned first = std::min(grid, resident);
  for (unsigned w = 0; w < P->block.size(); w++) { P->block[w] = w < first ? (int)w : -1; P->hold[w] = 0; }
  P->next = first;
  {
    std::unique_lock<std::mutex> lk(P->mu);
    P->turn = (int)(cta_rng(P) % first);
    P->cv.notify_all();
    P->cv.wait(lk, [&] { return P->turn == -1; });
  }
  std::lock_guard<std::mutex> g(g_cta_mu);
  auto& c = g_cta_counts[t_kern];
  c.first += P->passes ? 1 : 0;
  c.second += P->passes;
  return true;
}

}  // namespace simt

// test hooks (tests/test_cta_interleave.py): switch the CTA mode at run time (-1: off), and per kernel (symbol
// substring) the launches in which two CTAs overlapped and the baton passes from a CTA in mid-flight
extern "C" void simt_ctas(long long seed) {
  simt::g_cta_seed.store(seed < 0 ? -1 : seed);
  simt::g_cta_gen++;
}
extern "C" void simt_cta_counts(const char* kern, unsigned long long* overlapped, unsigned long long* passes) {
  std::lock_guard<std::mutex> g(simt::g_cta_mu);
  *overlapped = *passes = 0;
  for (const auto& kv : simt::g_cta_counts) {
    Dl_info a{};
    if (!dladdr(kv.first, &a) || !a.dli_sname || !strstr(a.dli_sname, kern)) continue;
    *overlapped += kv.second.first;
    *passes += kv.second.second;
  }
}
extern "C" void simt_cta_counts_reset() {
  std::lock_guard<std::mutex> g(simt::g_cta_mu);
  simt::g_cta_counts.clear();
}

// test hooks (tests/test_stream_overlap.py): switch the stream mode at run time, and count the kernels that
// ran while a top-level CTA was parked, by (parked kernel, kernel) symbol substrings
extern "C" void simt_streams(long long seed) {
  simt::drain_all();
  simt::g_seed.store(seed < 0 ? -1 : seed);
  simt::g_seed_gen++;
}
extern "C" unsigned long long simt_interleaved(const char* parked, const char* ran) {
  std::lock_guard<std::mutex> g(simt::g_reg_mu);
  unsigned long long n = 0;
  for (const auto& kv : simt::g_pairs) {
    Dl_info a{}, b{};
    if (!dladdr(kv.first.first, &a) || !dladdr(kv.first.second, &b) || !a.dli_sname || !b.dli_sname) continue;
    if (strstr(a.dli_sname, parked) && strstr(b.dli_sname, ran)) n += kv.second;
  }
  return n;
}
extern "C" void simt_interleaved_reset() {
  std::lock_guard<std::mutex> g(simt::g_reg_mu);
  simt::g_pairs.clear();
}

long long clock64() {
  return (long long)std::chrono::duration_cast<std::chrono::nanoseconds>(
             std::chrono::steady_clock::now().time_since_epoch()).count();
}

// -------------------------------------------------------------------- runtime API stubs
using simt::drain_all;
using simt::streams_async;

static simt_op work_op(std::function<void()> fn) {
  simt_op op{simt_op::WORK};
  op.fn = std::move(fn);
  return op;
}

const char* cudaGetErrorString(cudaError_t e) {
  switch (e) {
    case cudaSuccess: return "no error";
    case cudaErrorMemoryAllocation: return "out of memory";
    case cudaErrorNotSupported: return "operation not supported (emulation)";
    default: return "invalid value";
  }
}
cudaError_t cudaGetLastError() { return cudaSuccess; }
cudaError_t cudaSetDevice(int) { return cudaSuccess; }
cudaError_t cudaGetDeviceCount(int* n) { *n = 8; return cudaSuccess; }
cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) {
  memset(p, 0, sizeof(*p));
  strcpy(p->name, "simt-emulator");
  const char* e = getenv("MS_EMUL_SMS");
  p->multiProcessorCount = e ? atoi(e) : 1;
  p->sharedMemPerBlockOptin = 227 << 10;
  p->totalGlobalMem = (size_t)8 << 30;
  p->major = 9;
  return cudaSuccess;
}
cudaError_t cudaMalloc(void** p, size_t bytes) {
  void* q = nullptr;
  if (posix_memalign(&q, 256, bytes ? bytes : 1)) return cudaErrorMemoryAllocation;
  memset(q, 0xCD, bytes);   // device memory is not zeroed for you
  *p = q;
  return cudaSuccess;
}
cudaError_t cudaFree(void* p) { drain_all(); free(p); return cudaSuccess; }
cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { drain_all(); memmove(d, s, n); return cudaSuccess; }
cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind k, cudaStream_t st) {
  if (!st || !streams_async()) { drain_all(); memmove(d, s, n); return cudaSuccess; }
  if (k == cudaMemcpyHostToDevice) {          // the source is taken when the copy is enqueued (it may be on the stack)
    auto src = std::make_shared<std::vector<unsigned char>>((const unsigned char*)s, (const unsigned char*)s + n);
    simt::push(st, work_op([=]() { memmove(d, src->data(), n); }));
  } else {
    simt::push(st, work_op([=]() { memmove(d, s, n); }));
  }
  return cudaSuccess;
}
cudaError_t cudaMemset(void* d, int v, size_t n) { drain_all(); memset(d, v, n); return cudaSuccess; }
cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t st) {
  if (!st || !streams_async()) { drain_all(); memset(d, v, n); return cudaSuccess; }
  simt::push(st, work_op([=]() { memset(d, v, n); }));
  return cudaSuccess;
}
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) {
  *s = new simt_stream();
  std::lock_guard<std::mutex> g(simt::g_reg_mu);
  simt::g_streams.push_back(*s);
  return cudaSuccess;
}
cudaError_t cudaStreamDestroy(cudaStream_t s) {
  if (streams_async()) simt::run_until(s, s->enq);
  std::lock_guard<std::mutex> g(simt::g_reg_mu);
  simt::g_streams.erase(std::find(simt::g_streams.begin(), simt::g_streams.end(), s));
  // the object stays: an event may still name it (as complete: done == enq)
  return cudaSuccess;
}
cudaError_t cudaStreamSynchronize(cudaStream_t s) {
  if (!streams_async()) return cudaSuccess;
  if (!s) drain_all();
  else simt::run_until(s, s->enq);
  return cudaSuccess;
}
cudaError_t cudaStreamWaitEvent(cudaStream_t s, cudaEvent_t e, unsigned) {
  if (!streams_async() || !e->s) return cudaSuccess;
  if (!s) { simt::run_until(e->s, e->seq); return cudaSuccess; }
  simt_op op{simt_op::WAIT};
  op.dep = e->s; op.dep_seq = e->seq;
  simt::push(s, std::move(op));
  return cudaSuccess;
}
cudaError_t cudaStreamIsCapturing(cudaStream_t, cudaStreamCaptureStatus* st) { *st = cudaStreamCaptureStatusNone; return cudaSuccess; }
cudaError_t cudaStreamBeginCapture(cudaStream_t, cudaStreamCaptureMode) { return cudaErrorNotSupported; }
cudaError_t cudaStreamEndCapture(cudaStream_t, cudaGraph_t* g) { *g = nullptr; return cudaErrorNotSupported; }
cudaError_t cudaGraphInstantiate(cudaGraphExec_t* e, cudaGraph_t, unsigned long long) { *e = nullptr; return cudaErrorNotSupported; }
cudaError_t cudaGraphLaunch(cudaGraphExec_t, cudaStream_t) { return cudaErrorNotSupported; }
cudaError_t cudaGraphDestroy(cudaGraph_t) { return cudaSuccess; }
cudaError_t cudaGraphExecDestroy(cudaGraphExec_t) { return cudaSuccess; }
cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = new simt_event(); return cudaSuccess; }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = new simt_event(); return cudaSuccess; }
cudaError_t cudaEventDestroy(cudaEvent_t e) { drain_all(); delete e; return cudaSuccess; }
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t s) {
  if (!s || !streams_async()) {
    drain_all();
    e->t = std::chrono::steady_clock::now();
    e->s = nullptr;
    return cudaSuccess;
  }
  simt_op op{simt_op::RECORD};
  op.ev = e;
  simt::push(s, std::move(op));
  e->s = s;
  e->seq = s->enq;
  return cudaSuccess;
}
cudaError_t cudaEventSynchronize(cudaEvent_t e) {
  if (streams_async() && e->s) simt::run_until(e->s, e->seq);
  return cudaSuccess;
}
cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) {
  *ms = std::chrono::duration<float, std::milli>(b->t - a->t).count();
  return cudaSuccess;
}
cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t* h, void* p) {
  memset(h, 0, sizeof(*h));
  memcpy(h->reserved, &p, sizeof(p));
  return cudaSuccess;
}
cudaError_t cudaIpcOpenMemHandle(void** p, cudaIpcMemHandle_t h, unsigned) {
  memcpy(p, h.reserved, sizeof(*p));
  return cudaSuccess;
}
cudaError_t cudaIpcCloseMemHandle(void*) { return cudaSuccess; }

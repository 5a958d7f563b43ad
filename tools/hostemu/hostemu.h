// One-fiber-per-thread executor for the kernel templates of kornia_b200/csrc (see README.md in this directory).
// A CTA is a set of ucontext fibers scheduled round-robin on one OS thread:
//   __syncthreads()        parks the fiber until every live fiber of the CTA has arrived;
//   tma::mbar_wait()       polls and yields;
//   tma::load_3d()         copies the box (zero fill outside the tensor) and completes bytes on the mbarrier -- at once in
//                          EAGER mode, or only when no fiber can make progress in LAZY mode.  EAGER exposes a load that
//                          lands on data still being read, LAZY exposes a read that does not wait for its load.
// The emulator checks what the hardware would trap or hang on: 16-byte aligned innermost coordinate (traps,
// tools/tma_probe.cu), 128-byte aligned destination, byte counts that match expect_tx, deadlocks.
// No warp-level primitives: kernels that need lock-step lanes (shuffles, votes, elect) cannot run here.
#pragma once
#include <ucontext.h>

#include <deque>
#include <functional>
#include <map>
#include <vector>

#include "../../kornia_b200/csrc/warp_tma.cuh"  // kb200::tma::EmuMap / EmuBar (tma_emu.inl)

uint3 threadIdx, blockIdx;
dim3 blockDim, gridDim;

namespace emu {

struct PendingReduce;
struct Fiber {
  ucontext_t ctx;
  std::vector<char> stack;
  bool done = false, at_barrier = false, spinning = false, at_wsync = false;
  unsigned wgen = 0;  // warp collectives completed by this lane
  unsigned lin = 0;   // linear thread index
  uint3 tid;
  std::vector<struct PendingReduce> reduces;  // bulk async-groups are per thread
};
struct PendingReduce {
  kb200::tma::EmuMap map;
  uint32_t src;
  int c[3];
};
struct WarpState {
  unsigned long long slot[2][32];
};
struct PendingTma {
  void* dst;
  kb200::tma::EmuMap map;
  uint64_t* bar;
  int c[3];
};

static ucontext_t sched_ctx;
static Fiber* cur = nullptr;
static std::function<void()> body;
static bool lazy_tma = false;
static std::deque<PendingTma> pending;
static std::map<uint64_t*, long long> bar_tx;
static long long n_tma = 0, n_barriers = 0, n_wsync = 0, n_reduce = 0;
static std::vector<WarpState> warps;
static char* smem_base = nullptr;   // the CTA's shared array (set_smem) for 32-bit shared addresses
static size_t smem_size = 0;
static void set_smem(void* base, size_t size) {
  smem_base = static_cast<char*>(base);
  smem_size = size;
}

static void fail(const char* what) {
  fprintf(stderr, "hostemu: %s (block %u, thread %u)\n", what, blockIdx.x, cur ? cur->tid.x : 0u);
  abort();
}

static void complete(const PendingTma& t) {
  const auto& m = t.map;
  float* dst = static_cast<float*>(t.dst);
  for (uint32_t z = 0; z < m.box[2]; ++z)
    for (uint32_t y = 0; y < m.box[1]; ++y)
      for (uint32_t x = 0; x < m.box[0]; ++x) {
        const long long gx = (long long)t.c[0] + x, gy = (long long)t.c[1] + y, gz = (long long)t.c[2] + z;
        float v = 0.f;
        if (gx >= 0 && gy >= 0 && gz >= 0 && gx < (long long)m.dims[0] && gy < (long long)m.dims[1] && gz < (long long)m.dims[2])
          v = *reinterpret_cast<const float*>(reinterpret_cast<const char*>(m.base) + gz * m.strides[1] + gy * m.strides[0] + gx * 4);
        dst[((size_t)z * m.box[1] + y) * m.box[0] + x] = v;
      }
  bar_tx[t.bar] -= (long long)m.box[0] * m.box[1] * m.box[2] * 4;
  if (bar_tx[t.bar] < 0) fail("a TMA load delivered more bytes than the mbarrier expected");
  kb200::tma::emu_bar_try_complete(t.bar);
  ++n_tma;
}

static void yield() { swapcontext(&cur->ctx, &sched_ctx); }

static void trampoline() {
  body();
  cur->done = true;
  swapcontext(&cur->ctx, &sched_ctx);
}

// Run one CTA of `block` threads; blockIdx / gridDim are set by the caller.
static void run_cta(dim3 block, const std::function<void()>& fn) {
  const unsigned n = block.x * block.y * block.z;
  static std::vector<Fiber> fibers;
  if (fibers.size() < n) fibers.resize(n);
  body = fn;
  blockDim = block;
  warps.assign((n + 31) / 32, WarpState{});
  pending.clear();
  bar_tx.clear();
  for (unsigned i = 0; i < n; ++i) {
    Fiber& f = fibers[i];
    if (f.stack.empty()) f.stack.resize(512 * 1024);
    f.done = f.at_barrier = f.spinning = f.at_wsync = false;
    f.wgen = 0;
    f.lin = i;
    f.reduces.clear();
    f.tid = make_uint3(i % block.x, (i / block.x) % block.y, i / (block.x * block.y));
    getcontext(&f.ctx);
    f.ctx.uc_stack.ss_sp = f.stack.data();
    f.ctx.uc_stack.ss_size = f.stack.size();
    f.ctx.uc_link = nullptr;
    makecontext(&f.ctx, trampoline, 0);
  }
  for (;;) {
    unsigned live = 0, parked = 0, stuck = 0;
    bool finished = false;  // a thread that ran to its end in this pass may have arrived on a barrier others spin on
    for (unsigned i = 0; i < n; ++i) {
      Fiber& f = fibers[i];
      if (f.done) continue;
      ++live;
      if (f.at_barrier || f.at_wsync) {
        ++parked;
        continue;
      }
      cur = &f;
      threadIdx = f.tid;
      f.spinning = false;
      swapcontext(&sched_ctx, &f.ctx);
      if (f.done) {
        finished = true;
        continue;
      }
      if (f.at_barrier) ++parked;  // arrived during this pass
      else if (f.spinning) ++stuck;
    }
    if (live == 0) break;
    // warp rendezvous: release every warp whose live lanes have all arrived
    bool released = false;
    for (unsigned w = 0; w * 32 < n; ++w) {
      unsigned wl = 0, wa = 0;
      for (unsigned i = w * 32; i < std::min(n, w * 32 + 32); ++i) {
        if (fibers[i].done) continue;
        ++wl;
        if (fibers[i].at_wsync) ++wa;
      }
      if (wl && wa == wl) {
        for (unsigned i = w * 32; i < std::min(n, w * 32 + 32); ++i) fibers[i].at_wsync = false;
        released = true;
        ++n_wsync;
      }
    }
    // recount after the pass
    live = parked = 0;
    unsigned spinning = 0, wparked = 0;
    for (unsigned i = 0; i < n; ++i) {
      if (fibers[i].done) continue;
      ++live;
      if (fibers[i].at_barrier) ++parked;
      else if (fibers[i].at_wsync) ++wparked;
      else if (fibers[i].spinning) ++spinning;
    }
    if (live == 0) break;
    if (released || finished) continue;
    if (parked == live) {  // barrier complete
      for (unsigned i = 0; i < n; ++i) fibers[i].at_barrier = false;
      ++n_barriers;
    } else if (parked + wparked + spinning == live) {  // nobody can move: the outstanding loads land now (LAZY), else it is a hang
      if (pending.empty()) fail("deadlock: every thread waits on a barrier or an mbarrier and no load is in flight");
      complete(pending.front());
      pending.pop_front();
    }
  }
  if (!pending.empty()) fail("the CTA exited with TMA loads in flight");
  for (unsigned i = 0; i < n; ++i)
    if (!fibers[i].reduces.empty()) fail("a thread exited with TMA reduce-adds it never waited for");
  for (auto& kv : bar_tx)
    if (kv.second != 0) fail("the CTA exited with an mbarrier still expecting bytes");
  cur = nullptr;
}

template <typename F>
static void launch(unsigned grid, dim3 block, const F& fn) {
  gridDim = dim3(grid, 1, 1);
  for (unsigned b = 0; b < grid; ++b) {
    blockIdx = make_uint3(b, 0, 0);
    run_cta(block, fn);
  }
}
template <typename F>
static void launch3(dim3 grid, dim3 block, const F& fn) {
  gridDim = grid;
  for (unsigned z = 0; z < grid.z; ++z)
    for (unsigned y = 0; y < grid.y; ++y)
      for (unsigned x = 0; x < grid.x; ++x) {
        blockIdx = make_uint3(x, y, z);
        run_cta(block, fn);
      }
}

static CUtensorMap make_map(const float* base, int W, int H, int planes, int bw, int bh, int bc) {
  CUtensorMap m;
  memset(&m, 0, sizeof(m));
  kb200::tma::EmuMap e{base, {(uint64_t)W, (uint64_t)H, (uint64_t)planes}, {(uint64_t)W * 4, (uint64_t)H * W * 4}, {(uint32_t)bw, (uint32_t)bh, (uint32_t)bc}};
  static_assert(sizeof(e) <= sizeof(m), "descriptor fits the opaque bytes");
  if ((W * 4) % 16 != 0 || ((size_t)base & 15) != 0 || (bw * 4) % 16 != 0 || bw > 256 || bh > 256 || bc > 256) {
    fprintf(stderr, "hostemu: cuTensorMapEncodeTiled would reject this map\n");
    abort();
  }
  memcpy(&m, &e, sizeof(e));
  return m;
}

}  // namespace emu

void __syncthreads() {
  emu::cur->at_barrier = true;
  emu::yield();
}
int emu_lane() { return (int)(emu::cur->lin & 31u); }
unsigned long long emu_warp_exchange(unsigned long long mine, int src_lane) {
  emu::Fiber* f = emu::cur;
  emu::WarpState& w = emu::warps[f->lin >> 5];
  const unsigned par = f->wgen & 1u;
  w.slot[par][f->lin & 31u] = mine;
  f->at_wsync = true;
  emu::yield();
  ++f->wgen;
  return w.slot[par][src_lane & 31];
}
void __syncwarp(unsigned) { emu_warp_exchange(0ull, 0); }
unsigned __ballot_sync(unsigned, int pred) {
  // every lane needs every deposit: exchange once, then read all slots of that generation
  emu::Fiber* f = emu::cur;
  emu::WarpState& w = emu::warps[f->lin >> 5];
  const unsigned par = f->wgen & 1u;
  emu_warp_exchange(pred ? 1ull : 0ull, 0);
  unsigned bits = 0;
  const unsigned base = (f->lin >> 5) * 32, n = blockDim.x * blockDim.y * blockDim.z;
  for (unsigned l = 0; l < 32 && base + l < n; ++l)
    if (w.slot[par][l]) bits |= 1u << l;
  return bits;
}
int __any_sync(unsigned m, int pred) { return __ballot_sync(m, pred) != 0u; }
int __all_sync(unsigned m, int pred) {
  const unsigned base = (emu::cur->lin >> 5) * 32, n = blockDim.x * blockDim.y * blockDim.z;
  const unsigned lanes = std::min(32u, n - base);
  return __ballot_sync(m, pred) == (lanes == 32 ? 0xffffffffu : ((1u << lanes) - 1));
}
#include <cfenv>
float __fadd_rd(float a, float b) {
  const int old = fegetround();
  fesetround(FE_DOWNWARD);
  volatile float va = a, vb = b;
  volatile float r = va + vb;
  fesetround(old);
  return r;
}
int atomicAdd(int* p, int v) {
  const int old = *p;
  *p = old + v;
  return old;
}
float atomicAdd(float* p, float v) {
  const float old = *p;
  *p = old + v;
  return old;
}
double atomicAdd(double* p, double v) {
  const double old = *p;
  *p = old + v;
  return old;
}
int atomicMax(int* p, int v) {
  const int old = *p;
  *p = std::max(old, v);
  return old;
}
namespace kb200 {
namespace tma {
void emu_spin() {
  emu::cur->spinning = true;
  emu::yield();
}
long long& emu_bar_tx(uint64_t* bar) { return emu::bar_tx[bar]; }
long long& emu_lds_count() {
  static long long n = 0;
  return n;
}
uint32_t emu_smem_addr(const void* p) {
  const char* c = static_cast<const char*>(p);
  if (!emu::smem_base || c < emu::smem_base || c >= emu::smem_base + emu::smem_size) emu::fail("smem_u32 of a pointer outside the CTA's shared array");
  return (uint32_t)(c - emu::smem_base) + 0x10000u;
}
float* emu_smem_ptr(uint32_t addr) {
  const uint32_t off = addr - 0x10000u;
  if (off >= emu::smem_size || (off & 3u)) emu::fail("ld/st.shared outside the CTA's shared array (or misaligned)");
  return reinterpret_cast<float*>(emu::smem_base + off);
}
static void emu_reduce_complete(const emu::PendingReduce& r) {
  const auto& m = r.map;
  if (r.c[0] < 0 || r.c[1] < 0 || r.c[2] < 0) emu::fail("TMA reduce with a negative coordinate (traps: tools/tma_reduce_probe.cu)");
  if (((long long)r.c[0] * 4) % 16 != 0) emu::fail("TMA reduce: innermost coordinate not 16-byte aligned");
  const float* src = emu_smem_ptr(r.src);
  if (((size_t)src & 127) != 0) emu::fail("TMA reduce: shared-memory source not 128-byte aligned");
  for (uint32_t z = 0; z < m.box[2]; ++z)
    for (uint32_t y = 0; y < m.box[1]; ++y)
      for (uint32_t x = 0; x < m.box[0]; ++x) {
        const long long gx = (long long)r.c[0] + x, gy = (long long)r.c[1] + y, gz = (long long)r.c[2] + z;
        if (gx >= (long long)m.dims[0] || gy >= (long long)m.dims[1] || gz >= (long long)m.dims[2]) continue;  // clipped
        float* g = reinterpret_cast<float*>(reinterpret_cast<char*>(const_cast<float*>(m.base)) + gz * m.strides[1] + gy * m.strides[0] + gx * 4);
        *g += src[((size_t)z * m.box[1] + y) * m.box[0] + x];
      }
  ++emu::n_reduce;
}
void emu_reduce_add_issue(const EmuMap* map, uint32_t src_smem, int c0, int c1, int c2) {
  emu::PendingReduce r{*map, src_smem, {c0, c1, c2}};
  if (emu::lazy_tma) emu::cur->reduces.push_back(r);  // reads the strip as late as the kernel allows: at its wait_group
  else emu_reduce_complete(r);
}
void emu_bulk_wait(bool) {
  for (const auto& r : emu::cur->reduces) emu_reduce_complete(r);
  emu::cur->reduces.clear();
}
void emu_tma_issue(void* dst, const EmuMap* map, uint64_t* bar, int c0, int c1, int c2) {
  if (((long long)c0 * 4) % 16 != 0) emu::fail("TMA: innermost coordinate not 16-byte aligned (traps)");
  if (((size_t)dst & 127) != 0) emu::fail("TMA: shared-memory destination not 128-byte aligned");
  emu::PendingTma t{dst, *map, bar, {c0, c1, c2}};
  if (emu::lazy_tma) emu::pending.push_back(t);
  else emu::complete(t);
}
}  // namespace tma
}  // namespace kb200

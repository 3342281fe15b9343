// h2d.cu -- packed, pipelined ingest of pageable host Arrow buffers (see h2d.hpp).
//
// Replaces, for the GPU path, what arrow::ffi + a plain cudaMemcpy per buffer would do at the boundary the Rust shim
// crosses per RecordBatch (SURVEY.md section 8b): Arrow's fixed widths are an in-memory format, not a wire format.
#include <climits>
#include "h2d.hpp"
#include "kernels.hpp"

#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <array>
#include <cstdlib>
#include <cstring>

namespace sg {

namespace {

constexpr int64_t MAX_PIECE_ROWS = 256 * 1024;
constexpr size_t SLOT_BYTES = (size_t)MAX_PIECE_ROWS * 16;     // 4 MiB: one piece of the widest column
// rows per piece: SAILGPU_PACK_PIECE_ROWS (a multiple of 1024, at most 256 Ki).  Every piece costs three driver calls (copy, expand
// kernel, event) that serialise across the packer threads, so small pieces spend a large share of the import there;
// the one-pass packer no longer needs the piece to stay in L2 for a second loop
static int64_t piece_rows() {      // read per batch: A/B measurements in one process
  const char* e = getenv("SAILGPU_PACK_PIECE_ROWS");
  const int64_t r = e && *e ? atoll(e) : MAX_PIECE_ROWS;
  return std::max<int64_t>(1024, std::min<int64_t>(MAX_PIECE_ROWS, r / 1024 * 1024));
}

enum Enc : int { ENC_RAW = 0, ENC_INT = 1, ENC_VIEW = 2 };

// ---- device side: packed piece -> Arrow layout ---------------------------------------------------
__global__ void unpack_int_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int64_t n, int w_in, int out_width, long long base) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    unsigned long long d;
    switch (w_in) {
      case 1: d = src[i]; break;
      case 2: d = reinterpret_cast<const uint16_t*>(src)[i]; break;
      case 4: d = reinterpret_cast<const uint32_t*>(src)[i]; break;
      default: d = reinterpret_cast<const unsigned long long*>(src)[i];
    }
    const long long v = (long long)((unsigned long long)base + d);
    if (out_width == 16) { ulonglong2 w; w.x = (unsigned long long)v; w.y = (unsigned long long)(v >> 63); reinterpret_cast<ulonglong2*>(dst)[i] = w; }
    else if (out_width == 8) reinterpret_cast<long long*>(dst)[i] = v;
    else reinterpret_cast<int*>(dst)[i] = (int)v;
  }
}
// packed row: [length byte][L bytes]  ->  16-byte inline view {len:u32, bytes[12]}
__global__ void unpack_view_kernel(const uint8_t* __restrict__ src, ulonglong2* __restrict__ dst, int64_t n, int L) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint8_t* p = src + i * (1 + L);
    const unsigned len = p[0];
    unsigned long long lo = len, hi = 0;
    for (int k = 0; k < L; ++k) {
      const unsigned long long b = k < (int)len ? p[1 + k] : 0;      // bytes past the string stay zero (Arrow requires zero padding)
      if (k < 4) lo |= b << (32 + 8 * k); else hi |= b << (8 * (k - 4));
    }
    ulonglong2 v; v.x = lo; v.y = hi;
    dst[i] = v;
  }
}

// ---- host side: piece -> staging slot (loops in h2d_pack.cpp: AVX-512 / AVX2 / baseline clones) -------
struct Packed { int enc; size_t bytes; long long base; int w; };
}  // namespace
extern "C" {
void sg_scan_dec128(const int64_t* p, int64_t n, int64_t* mn, int64_t* mx, uint64_t* bad);
void sg_scan_i64(const int64_t* p, int64_t n, int64_t* mn, int64_t* mx);
void sg_scan_i32(const int32_t* p, int64_t n, int32_t* mn, int32_t* mx);
uint32_t sg_scan_view_maxlen(const uint32_t* p, int64_t n);
void sg_pack_i64(uint8_t* out, const int64_t* vals, int64_t stride, int64_t n, int64_t base, int w);
void sg_pack_i32(uint8_t* out, const int32_t* vals, int64_t n, int32_t base, int w);
void sg_pack_views(uint8_t* out, const uint8_t* views, int64_t n, uint32_t L);
void sg_packchk_dec128(uint8_t* out, const int64_t* p, int64_t n, int64_t base, int w, int64_t* mn, int64_t* mx, uint64_t* bad);
void sg_packchk_i64(uint8_t* out, const int64_t* p, int64_t n, int64_t base, int w, int64_t* mn, int64_t* mx);
void sg_packchk_i32(uint8_t* out, const int32_t* p, int64_t n, int32_t base, int w, int32_t* mn, int32_t* mx);
uint32_t sg_packchk_views(uint8_t* out, const uint8_t* views, int64_t n, uint32_t L);
}
namespace {

static inline int width_for(unsigned long long range) { return range < (1ull << 8) ? 1 : range < (1ull << 16) ? 2 : range < (1ull << 32) ? 4 : 8; }

// A guess of the piece's value range from 64 strided samples (prefetched together: one DRAM round trip).  The window of the
// guessed width is centred on the sampled range and must be at least twice as wide, so that values the sample missed still fit.
constexpr int N_SAMPLES = 64;
struct Guess { bool ok; long long base; int w; };
template <class T>
static Guess guess_range(const T* p, int64_t n, int64_t stride, int max_w) {
  const int64_t step = std::max<int64_t>(1, n / N_SAMPLES);
  for (int64_t i = 0; i < n; i += step) __builtin_prefetch(p + i * stride);
  long long mn = LLONG_MAX, mx = LLONG_MIN;
  for (int64_t i = 0; i < n; i += step) { const long long v = (long long)p[i * stride]; mn = v < mn ? v : mn; mx = v > mx ? v : mx; }
  const unsigned long long range = (unsigned long long)mx - (unsigned long long)mn;
  if (range >= (1ull << 31)) return {false, 0, 0};
  int w = 1;
  while (w <= 4 && (2 * range + 2) > (w == 4 ? (1ull << 32) : (1ull << (8 * w)))) w *= 2;
  if (w > max_w) return {false, 0, 0};
  const unsigned long long window = w == 4 ? (1ull << 32) : (1ull << (8 * w));
  const long long slack = (long long)((window - 1 - range) / 2);
  if (mn < LLONG_MIN + slack) return {false, 0, 0};
  return {true, mn - slack, w};
}
static inline bool fits(long long mn, long long mx, long long base, int w) {
  if (mn < base) return false;
  const unsigned long long top = (unsigned long long)mx - (unsigned long long)base;
  return w >= 8 || top < (w == 4 ? (1ull << 32) : (1ull << (8 * w)));
}

static Packed pack_piece(const HostStager::Item& it, uint8_t* out, bool narrow) {
  const int64_t n = it.n;
  if (narrow && n > 0 && it.kind == HostCol::Dec128) {
    const int64_t* p = reinterpret_cast<const int64_t*>(it.src);
    int64_t mn, mx; uint64_t bad = 0;
    const Guess g = guess_range(p, n, 2, 4);
    if (g.ok) {
      sg_packchk_dec128(out, p, n, g.base, g.w, &mn, &mx, &bad);
      if (!bad && fits(mn, mx, g.base, g.w)) return {ENC_INT, (size_t)n * g.w, g.base, g.w};
    } else sg_scan_dec128(p, n, &mn, &mx, &bad);
    if (!bad) {
      const int w = width_for((unsigned long long)mx - (unsigned long long)mn);
      sg_pack_i64(out, p, 2, n, mn, w);
      return {ENC_INT, (size_t)n * w, mn, w};
    }
  } else if (narrow && n > 0 && it.kind == HostCol::Int64) {
    const int64_t* p = reinterpret_cast<const int64_t*>(it.src);
    int64_t mn, mx;
    const Guess g = guess_range(p, n, 1, 4);
    if (g.ok) {
      sg_packchk_i64(out, p, n, g.base, g.w, &mn, &mx);
      if (fits(mn, mx, g.base, g.w)) return {ENC_INT, (size_t)n * g.w, g.base, g.w};
    } else sg_scan_i64(p, n, &mn, &mx);
    const int w = width_for((unsigned long long)mx - (unsigned long long)mn);
    if (w < 8) { sg_pack_i64(out, p, 1, n, mn, w); return {ENC_INT, (size_t)n * w, mn, w}; }
  } else if (narrow && n > 0 && it.kind == HostCol::Int32) {
    const int32_t* p = reinterpret_cast<const int32_t*>(it.src);
    int32_t mn, mx;
    const Guess g = guess_range(p, n, 1, 2);
    if (g.ok && g.base >= INT32_MIN) {
      sg_packchk_i32(out, p, n, (int32_t)g.base, g.w, &mn, &mx);
      if (fits(mn, mx, g.base, g.w)) return {ENC_INT, (size_t)n * g.w, g.base, g.w};
    } else sg_scan_i32(p, n, &mn, &mx);
    const int w = width_for((unsigned long long)((long long)mx - (long long)mn));
    if (w < 4) { sg_pack_i32(out, p, n, mn, w); return {ENC_INT, (size_t)n * w, (long long)mn, w}; }
  } else if (narrow && n > 0 && it.kind == HostCol::View16) {
    const uint32_t* lens = reinterpret_cast<const uint32_t*>(it.src);
    uint32_t L = 13;
    const int64_t step = std::max<int64_t>(1, n / N_SAMPLES);
    for (int64_t i = 0; i < n; i += step) __builtin_prefetch(lens + 4 * i);
    uint32_t Ls = 0;
    for (int64_t i = 0; i < n; i += step) Ls = std::max(Ls, lens[4 * i]);
    if (Ls <= 12) {
      L = sg_packchk_views(out, it.src, n, Ls);
      if (L <= Ls) return {ENC_VIEW, (size_t)(1 + Ls) * (size_t)n, 0, (int)Ls};
    }
    if (L > 12) L = sg_scan_view_maxlen(lens, n);      // (a rejected guess left the true maximum in L)
    if (L <= 12) { sg_pack_views(out, it.src, n, L); return {ENC_VIEW, (size_t)(1 + L) * (size_t)n, 0, (int)L}; }
  }
  const size_t bytes = (size_t)n * (size_t)it.width;
  memcpy(out, it.src, bytes);
  return {ENC_RAW, bytes, 0, 0};
}

}  // namespace

// ---- the pool -----------------------------------------------------------------------------------
struct PackPool {
  struct Slot { uint8_t* host = nullptr; uint8_t* dev = nullptr; cudaEvent_t free_ev = nullptr; bool used = false; };
  struct Worker { std::thread th; std::array<Slot, 2> slots; cudaStream_t stream = nullptr; cudaEvent_t done_ev = nullptr; int turn = 0; bool touched = false; };
  Ctx* ctx = nullptr;
  bool narrow = true;
  std::vector<Worker> workers;
  Worker inline_w;                 // small batches are staged by the calling thread itself (no wake-ups)
  std::mutex mu;
  std::condition_variable cv_work, cv_done;
  const std::vector<HostStager::Item>* work = nullptr;
  std::atomic<size_t> next{0};
  size_t total = 0, finished_workers = 0;
  uint64_t epoch = 0;
  bool stop = false;
  std::string error;
  // NUMA (SAILGPU_PACK_NUMA=0 turns it off): the packers run on the CPUs of the node the producer's pages live on.  A reader on
  // the other socket gets only part of the local bandwidth.  In a small probe process the scheduler happens to keep the
  // threads near the data and binding is neutral, but in bench.py -- host tables first touched by the main thread, packers
  // created later -- binding is what keeps the packers next to their data.
  cpu_set_t allowed;                         // the process's affinity when the pool was created
  std::vector<cpu_set_t> node_cpus;          // allowed CPUs of every NUMA node (empty sets: unknown)
  std::atomic<int> want_node{-1};

  void read_topology() {
    CPU_ZERO(&allowed);
    if (sched_getaffinity(0, sizeof(allowed), &allowed) != 0) return;
    for (int node = 0; node < 64; ++node) {
      char path[96];
      snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
      FILE* f = fopen(path, "r");
      if (!f) break;
      cpu_set_t set; CPU_ZERO(&set);
      int a = 0, b = 0;
      for (;;) {
        if (fscanf(f, "%d", &a) != 1) break;
        b = a;
        int ch = fgetc(f);
        if (ch == '-') { if (fscanf(f, "%d", &b) != 1) break; ch = fgetc(f); }
        for (int c = a; c <= b && c < CPU_SETSIZE; ++c) if (CPU_ISSET(c, &allowed)) CPU_SET(c, &set);
        if (ch != ',') break;
      }
      fclose(f);
      node_cpus.push_back(set);
    }
  }
  // node of the page `p` lives on (move_pages with a null target only queries), -1 when the kernel does not tell
  static int node_of(const void* p) {
    void* page = reinterpret_cast<void*>(reinterpret_cast<uintptr_t>(p) & ~(uintptr_t)4095);
    int status = -1;
    if (syscall(SYS_move_pages, 0, 1ul, &page, nullptr, &status, 0) != 0) return -1;
    return status;
  }
  void bind_self(int node, int* current) {
    if (node == *current || node < 0 || node >= (int)node_cpus.size() || CPU_COUNT(&node_cpus[(size_t)node]) == 0) return;
    if (sched_setaffinity(0, sizeof(cpu_set_t), &node_cpus[(size_t)node]) == 0) *current = node;
  }

  void process(Worker& w, const HostStager::Item& it) {
    Slot& s = w.slots[(size_t)(w.turn++ & 1)];
    if (s.used && cudaEventSynchronize(s.free_ev) != cudaSuccess) throw std::runtime_error("staging slot event");
    const Packed pk = pack_piece(it, s.host, narrow);
    cudaError_t e;
    if (pk.enc == ENC_RAW) {
      e = cudaMemcpyAsync(it.dst, s.host, pk.bytes, cudaMemcpyHostToDevice, w.stream);
    } else {
      e = cudaMemcpyAsync(s.dev, s.host, pk.bytes, cudaMemcpyHostToDevice, w.stream);
      if (e == cudaSuccess) {
        const int grid = (int)std::min<int64_t>((it.n + 255) / 256, grid_cap(4));
        if (pk.enc == ENC_INT) unpack_int_kernel<<<grid, 256, 0, w.stream>>>(s.dev, it.dst, it.n, pk.w, it.width, pk.base);
        else unpack_view_kernel<<<grid, 256, 0, w.stream>>>(s.dev, reinterpret_cast<ulonglong2*>(it.dst), it.n, pk.w);
        e = cudaGetLastError();
      }
    }
    if (e == cudaSuccess) e = cudaEventRecord(s.free_ev, w.stream);
    if (e != cudaSuccess) throw std::runtime_error(std::string("host staging: ") + cudaGetErrorString(e));
    s.used = true;
    w.touched = true;
    ctx->h2d_bytes += pk.bytes;
  }

  void run(size_t wi) {
    cudaSetDevice(ctx->device);
    Worker& w = workers[wi];
    uint64_t seen = 0;
    int my_node = -1;
    for (;;) {
      {
        std::unique_lock<std::mutex> lk(mu);
        cv_work.wait(lk, [&] { return stop || epoch != seen; });
        if (stop) return;
        seen = epoch;
      }
      bind_self(want_node.load(), &my_node);
      std::string err;
      for (;;) {
        const size_t i = next.fetch_add(1);
        if (i >= total) break;
        try { process(w, (*work)[i]); } catch (const std::exception& e) { err = e.what(); }
      }
      if (w.touched) cudaEventRecord(w.done_ev, w.stream);
      std::lock_guard<std::mutex> lk(mu);
      if (!err.empty() && error.empty()) error = err;
      if (++finished_workers == workers.size()) cv_done.notify_all();
    }
  }
};

static PackPool* pool_of(Ctx* ctx) {
  if (ctx->pack_pool) return ctx->pack_pool;
  auto* p = new PackPool();
  p->ctx = ctx;
  // packer threads: the CPUs this process may use (affinity mask, cgroup quota), shared by the ranks of the node, at most 32
  const char* nt = getenv("SAILGPU_PACK_THREADS");
  int avail = (int)std::thread::hardware_concurrency();
  { cpu_set_t set; if (sched_getaffinity(0, sizeof(set), &set) == 0) avail = std::min(avail > 0 ? avail : 1 << 20, (int)CPU_COUNT(&set)); }
  if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
    long long quota = 0, period = 0;
    if (fscanf(f, "%lld %lld", &quota, &period) == 2 && quota > 0 && period > 0) avail = std::min<long long>(avail, (quota + period - 1) / period);
    fclose(f);
  }
  const char* lw = getenv("LOCAL_WORLD_SIZE");
  const int ranks = std::max(1, lw && *lw ? atoi(lw) : ctx->world);
  const int n = std::max(1, nt && *nt ? atoi(nt) : std::min(32, std::max(2, avail / ranks)));
  const char* nw = getenv("SAILGPU_H2D_PACK");
  p->narrow = !(nw && *nw && atoi(nw) == 0);
  p->workers.resize((size_t)n);
  { const char* e = getenv("SAILGPU_PACK_NUMA"); if (!(e && *e && atoi(e) == 0)) p->read_topology(); }
  auto init_worker = [](PackPool::Worker& w) {
    SG_CUDA(cudaStreamCreateWithFlags(&w.stream, cudaStreamNonBlocking));
    SG_CUDA(cudaEventCreateWithFlags(&w.done_ev, cudaEventDisableTiming));
    for (auto& s : w.slots) {
      SG_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&s.host), SLOT_BYTES, cudaHostAllocDefault));
      SG_CUDA(cudaMalloc(reinterpret_cast<void**>(&s.dev), SLOT_BYTES));
      SG_CUDA(cudaEventCreateWithFlags(&s.free_ev, cudaEventDisableTiming));
    }
  };
  for (auto& w : p->workers) init_worker(w);
  init_worker(p->inline_w);
  for (size_t i = 0; i < p->workers.size(); ++i) p->workers[i].th = std::thread([p, i] { p->run(i); });
  ctx->pack_pool = p;
  return p;
}

void destroy_pack_pool(Ctx* ctx) {
  PackPool* p = ctx->pack_pool;
  if (!p) return;
  { std::lock_guard<std::mutex> lk(p->mu); p->stop = true; }
  p->cv_work.notify_all();
  for (auto& w : p->workers) if (w.th.joinable()) w.th.join();
  std::vector<PackPool::Worker*> all;
  for (auto& w : p->workers) all.push_back(&w);
  all.push_back(&p->inline_w);
  for (PackPool::Worker* wp : all) {
    PackPool::Worker& w = *wp;
    for (auto& s : w.slots) { if (s.host) cudaFreeHost(s.host); if (s.dev) cudaFree(s.dev); if (s.free_ev) cudaEventDestroy(s.free_ev); }
    if (w.done_ev) cudaEventDestroy(w.done_ev);
    if (w.stream) cudaStreamDestroy(w.stream);
  }
  delete p;
  ctx->pack_pool = nullptr;
}

void HostStager::add(HostCol kind, void* dst, const void* src, int64_t n, int width) {
  if (n <= 0) return;
  const int64_t piece = kind == HostCol::Raw ? (int64_t)SLOT_BYTES / std::max(1, width) : piece_rows();
  for (int64_t o = 0; o < n; o += piece) {
    const int64_t k = std::min(piece, n - o);
    items.push_back({kind, static_cast<uint8_t*>(dst) + o * width, static_cast<const uint8_t*>(src) + o * width, k, width});
  }
}

void HostStager::flush() {
  if (items.empty()) return;
  PackPool* p = pool_of(ctx);
  { const char* nw = getenv("SAILGPU_H2D_PACK"); p->narrow = !(nw && *nw && atoi(nw) == 0); }      // read per batch (A/B measurements, fallback)
  // the destination buffers were allocated (stream-ordered) on the compute stream: the copy streams must not start before that
  cudaEvent_t alloc_ev;
  SG_CUDA(cudaEventCreateWithFlags(&alloc_ev, cudaEventDisableTiming));
  SG_CUDA(cudaEventRecord(alloc_ev, ctx->stream));
  size_t payload = 0;
  for (auto& it : items) payload += (size_t)it.n * (size_t)it.width;
  if (payload <= (1u << 20)) {      // a small batch: stage it on this thread
    PackPool::Worker& w = p->inline_w;
    SG_CUDA(cudaStreamWaitEvent(w.stream, alloc_ev, 0));
    SG_CUDA(cudaEventDestroy(alloc_ev));
    std::string err;
    try { for (auto& it : items) p->process(w, it); } catch (const std::exception& e) { err = e.what(); }
    items.clear();
    SG_CHECK(err.empty(), SAILGPU_ERR_CUDA, err);
    SG_CUDA(cudaEventRecord(w.done_ev, w.stream));
    SG_CUDA(cudaStreamWaitEvent(ctx->stream, w.done_ev, 0));
    return;
  }
  for (auto& w : p->workers) SG_CUDA(cudaStreamWaitEvent(w.stream, alloc_ev, 0));
  SG_CUDA(cudaEventDestroy(alloc_ev));
  if (p->node_cpus.size() > 1) {      // run the packers next to the batch: the node of its largest column's first page
    const HostStager::Item* big = &items[0];
    for (auto& it : items) if ((size_t)it.n * (size_t)it.width > (size_t)big->n * (size_t)big->width) big = &it;
    p->want_node.store(PackPool::node_of(big->src));
  }
  {
    std::lock_guard<std::mutex> lk(p->mu);
    p->work = &items;
    p->total = items.size();
    p->next.store(0);
    p->finished_workers = 0;
    p->error.clear();
    for (auto& w : p->workers) w.touched = false;
    p->epoch++;
  }
  p->cv_work.notify_all();
  {
    std::unique_lock<std::mutex> lk(p->mu);
    p->cv_done.wait(lk, [&] { return p->finished_workers == p->workers.size(); });
    p->work = nullptr;
  }
  items.clear();
  SG_CHECK(p->error.empty(), SAILGPU_ERR_CUDA, p->error);
  for (auto& w : p->workers)
    if (w.touched) SG_CUDA(cudaStreamWaitEvent(ctx->stream, w.done_ev, 0));
}

}  // namespace sg

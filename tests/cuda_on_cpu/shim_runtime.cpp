// TEST INFRASTRUCTURE ONLY -- runtime of the "CUDA on CPU" shim (see common.cuh in this directory).
#include "common.cuh"

#include <sys/mman.h>

thread_local ShimBlock g_blk;
thread_local uint64_t g_smem_hi = 0;
thread_local std::deque<std::function<void()>> g_async;
int g_async_mode = 0;
thread_local void* g_static_self = nullptr;
thread_local std::unordered_map<const void*, ShimMbar> g_mbar;
thread_local uint8_t* g_dyn_smem = nullptr;
thread_local size_t g_dyn_bytes = 0;
thread_local bool g_whole_grid_next = false;
thread_local ShimCluster* g_cluster = nullptr;
thread_local int g_cluster_rank = 0;
thread_local ShimIdx g_tid, g_bid;
ShimIdx g_bdim, g_gdim;

void shim_set_dyn_smem(size_t bytes) {
  static thread_local std::vector<uint8_t> buf;
  buf.assign(bytes + 4096, 0xCD);                          // poisoned: a kernel must not rely on zeroed shared memory
  // 1024-aligned in EVERY CTA: on the GPU all CTAs see the same shared-memory window, so a kernel's own alignment arithmetic gives the
  // same offset everywhere -- distributed-shared-memory addressing relies on that
  g_dyn_smem = (uint8_t*)(((uintptr_t)buf.data() + 1023) & ~(uintptr_t)1023);
  g_dyn_bytes = bytes;
}

// ---- fibers: swap the callee-saved registers and the stack pointer (System V x86-64)
extern "C" void shim_switch(void** save_sp, void* load_sp);
asm(R"(
.text
.globl shim_switch
.type shim_switch,@function
shim_switch:
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
.size shim_switch,.-shim_switch
)");

namespace {
struct Fiber { void* sp; ShimIdx tid; bool done; };
constexpr size_t kStack = 256 << 10;
thread_local std::vector<Fiber> g_fibers;
thread_local void* g_sched_sp = nullptr;
thread_local int g_cur = -1;
thread_local const std::function<void()>* g_body = nullptr;

void fiber_main() {
  (*g_body)();
  // a thread that has returned no longer takes part in barriers (CUDA semantics): release anybody it would have kept waiting
  --g_blk.alive;
  if (g_blk.arrived > 0 && g_blk.arrived >= g_blk.alive) { g_blk.arrived = 0; ++g_blk.gen; }
  ShimBlock::Warp& w = g_blk.warp[g_cur >> 5];
  --w.alive;
  if (w.arrived > 0 && w.arrived >= w.alive) { w.arrived = 0; ++w.gen; }
  g_fibers[g_cur].done = true;
  shim_switch(&g_fibers[g_cur].sp, g_sched_sp);
  abort();                                                 // a finished fiber is never resumed
}
}  // namespace

void shim_yield() {
  Fiber& f = g_fibers[g_cur];
  f.tid = g_tid;
  shim_switch(&f.sp, g_sched_sp);
}

void shim_run_block(const std::function<void()>& body, dim3 block) {
  const int n = (int)(block.x * block.y * block.z);
  static thread_local char* arena = nullptr;
  static thread_local size_t arena_fibers = 0;
  if ((size_t)n > arena_fibers) {
    if (arena) munmap(arena, arena_fibers * kStack);
    arena = (char*)mmap(nullptr, (size_t)n * kStack, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (arena == MAP_FAILED) { perror("shim: mmap of the fiber stacks"); abort(); }
    arena_fibers = (size_t)n;
  }
  g_blk.alive = n;
  g_blk.arrived = 0;
  for (int i = 0; i < 16; ++i) g_blk.named_arrived[i] = 0;
  for (int w = 0; w < 64; ++w) {
    const int lanes = n - w * 32;
    g_blk.warp[w].alive = lanes <= 0 ? 0 : (lanes > 32 ? 32 : lanes);
    g_blk.warp[w].arrived = 0;
  }
  g_body = &body;
  g_fibers.assign((size_t)n, Fiber{});
  for (int i = 0; i < n; ++i) {
    Fiber& f = g_fibers[i];
    f.tid = {(unsigned)(i % (int)block.x), (unsigned)((i / (int)block.x) % (int)block.y), (unsigned)(i / (int)(block.x * block.y))};
    f.done = false;
    uintptr_t top = ((uintptr_t)arena + (size_t)(i + 1) * kStack) & ~(uintptr_t)15;
    void** sp = (void**)top;
    *--sp = nullptr;                                       // the "return address" fiber_main would see (never used)
    *--sp = (void*)&fiber_main;                            // popped by the `ret` of the first switch into this fiber
    for (int r = 0; r < 6; ++r) *--sp = nullptr;           // rbp rbx r12 r13 r14 r15
    f.sp = sp;
  }
  // CTS_SHIM_ORDER = reverse | random: the order in which the fibers of a block get the CPU.  A kernel that is correct only for one
  // interleaving (a missing __syncthreads / __syncwarp, an assumed warp-synchronous step) gives different results under another one.
  static const char* order_env = getenv("CTS_SHIM_ORDER");
  const int order = !order_env ? 0 : (order_env[0] == 'r' && order_env[1] == 'e' ? 1 : (order_env[0] == 'r' ? 2 : 0));
  static thread_local uint64_t rng = 0x9E3779B97F4A7C15ull;
  std::vector<int> perm((size_t)n);
  for (int i = 0; i < n; ++i) perm[(size_t)i] = order == 1 ? n - 1 - i : i;
  int left = n;
  while (left > 0) {
    if (order == 2)
      for (int i = n - 1; i > 0; --i) {
        rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17;
        std::swap(perm[(size_t)i], perm[(size_t)(rng % (uint64_t)(i + 1))]);
      }
    for (int j = 0; j < n; ++j) {
      const int i = perm[(size_t)j];
      Fiber& f = g_fibers[(size_t)i];
      if (f.done) continue;
      g_cur = i;
      g_tid = f.tid;
      shim_switch(&g_sched_sp, f.sp);
      if (f.done) --left;
    }
  }
  shim_async_all();                                        // whatever is still outstanding completes before the CTA retires
  g_cur = -1;
}

// kernels whose CTAs wait for each other WITHOUT being a cluster (the low-latency all-reduce with several sub-slices per token): the
// test asks for the whole grid to run concurrently, one OS thread per CTA
static int g_concurrent_grid = 0;
extern "C" void shim_concurrent_grid(int on) { g_concurrent_grid = on; }

// grid = clusters one after the other; the CTAs of a cluster concurrently (one OS thread each; a cluster of 1 runs in the caller)
void shim_launch(const std::function<void()>& body, dim3 grid, dim3 block, size_t smem, dim3 cl) {
  { const char* e = getenv("CTS_SHIM_ASYNC"); g_async_mode = e && e[0] == '1'; }
  g_gdim = {grid.x, grid.y, grid.z};
  g_bdim = {block.x, block.y, block.z};
  const int csize = (int)(cl.x * cl.y * cl.z);
  if (g_concurrent_grid && csize == 1 && grid.x * grid.y * grid.z <= 64) {
    std::vector<std::thread> th;
    for (unsigned z = 0; z < grid.z; ++z)
      for (unsigned y = 0; y < grid.y; ++y)
        for (unsigned x = 0; x < grid.x; ++x)
          th.emplace_back([&, x, y, z] {
            g_bid = {x, y, z};
            g_cluster = nullptr;
            g_cluster_rank = 0;
            shim_set_dyn_smem(smem);
            shim_run_block(body, block);
          });
    for (auto& t : th) t.join();
    return;
  }
  for (unsigned z = 0; z < grid.z; z += cl.z)
    for (unsigned y = 0; y < grid.y; y += cl.y)
      for (unsigned x = 0; x < grid.x; x += cl.x) {
        if (csize == 1) {
          g_bid = {x, y, z};
          g_cluster = nullptr;
          g_cluster_rank = 0;
          shim_set_dyn_smem(smem);
          shim_run_block(body, block);
          continue;
        }
        ShimCluster cluster;
        cluster.size = csize;
        pthread_barrier_init(&cluster.bar, nullptr, (unsigned)csize);
        pthread_barrier_t ready;                           // every CTA publishes its shared-memory base before any of them runs
        pthread_barrier_init(&ready, nullptr, (unsigned)csize);
        std::vector<std::thread> th;
        for (int r = 0; r < csize; ++r)
          th.emplace_back([&, r] {
            const unsigned rx = (unsigned)r % cl.x, ry = ((unsigned)r / cl.x) % cl.y, rz = (unsigned)r / (cl.x * cl.y);
            g_bid = {x + rx, y + ry, z + rz};
            g_cluster = &cluster;
            g_cluster_rank = r;
            shim_set_dyn_smem(smem);
            cluster.dyn_base[r] = g_dyn_smem;
            pthread_barrier_wait(&ready);
            shim_run_block(body, block);
          });
        for (auto& t : th) t.join();
        pthread_barrier_destroy(&cluster.bar);
        pthread_barrier_destroy(&ready);
      }
}

int cts_set_error(cts_ctx* ctx, int code, const char* fmt, ...) {
  if (ctx) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(ctx->err, sizeof(ctx->err), fmt, ap);
    va_end(ap);
  }
  return code;
}

extern "C" int cts_version(void) { return 100; }
extern "C" const char* cts_arch(void) { return "host-shim"; }
extern "C" int cts_ctx_create(int device, cts_ctx** out) {
  cts_ctx* c = new cts_ctx();
  c->device = device;
  c->sm_count = 148;
  c->decode_stages = 96;
  c->l2_prefetch_mb = 0;
  c->no_persistent_gemm = 0;
  c->norm_cluster = 8;
  c->no_next_prefetch = 0;
  c->next_prefetch_mb = 0;
  c->no_ts_fused = 0;
  c->scratch = calloc(1, 4096);
  c->max_smem_optin = 232448;
  c->err[0] = 0;
  *out = c;
  return CTS_OK;
}
extern "C" void cts_ctx_destroy(cts_ctx* ctx) { delete ctx; }
extern "C" const char* cts_last_error(const cts_ctx* ctx) { return ctx ? ctx->err : "null ctx"; }

// ---- cudaMalloc / cudaIpc* over POSIX shared memory
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>
#include <map>
#include <string>
namespace {
struct ShmBlock { std::string name; size_t bytes; bool owner; };
std::map<void*, ShmBlock> g_shm;
}
int cudaMalloc(void** p, size_t bytes) {
  static int counter = 0;
  char name[64];
  snprintf(name, sizeof(name), "/cts_shim_%d_%d", (int)getpid(), counter++);
  const int fd = shm_open(name, O_CREAT | O_EXCL | O_RDWR, 0600);
  if (fd < 0 || ftruncate(fd, (off_t)bytes) != 0) return 2;
  void* q = mmap(nullptr, bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  if (q == MAP_FAILED) return 2;
  g_shm[q] = ShmBlock{name, bytes, true};
  *p = q;
  return 0;
}
int cudaFree(void* p) {
  auto it = g_shm.find(p);
  if (it == g_shm.end()) return 1;
  munmap(p, it->second.bytes);
  if (it->second.owner) shm_unlink(it->second.name.c_str());
  g_shm.erase(it);
  return 0;
}
int cudaIpcGetMemHandle(cudaIpcMemHandle_t* h, void* p) {
  auto it = g_shm.find(p);
  if (it == g_shm.end()) return 1;
  memset(h->reserved, 0, 64);
  snprintf(h->reserved, 48, "%s", it->second.name.c_str());
  const unsigned long long n = it->second.bytes;
  memcpy(h->reserved + 48, &n, 8);
  return 0;
}
int cudaIpcOpenMemHandle(void** p, cudaIpcMemHandle_t h, unsigned) {
  unsigned long long n = 0;
  memcpy(&n, h.reserved + 48, 8);
  const int fd = shm_open(h.reserved, O_RDWR, 0600);
  if (fd < 0) return 2;
  void* q = mmap(nullptr, (size_t)n, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  if (q == MAP_FAILED) return 2;
  g_shm[q] = ShmBlock{h.reserved, (size_t)n, false};
  *p = q;
  return 0;
}
int cudaIpcCloseMemHandle(void* p) { return cudaFree(p); }

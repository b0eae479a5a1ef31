// lc_ctx.cc — context lifecycle, HBM arena, scratch buffers, error state.
#include <execinfo.h>
#include <signal.h>
#include <unistd.h>

#include <cstdlib>

#include "host_common.h"

std::atomic<uint64_t> g_validated_gen{1};  // see lc_lane::tok_* (host_common.h)

namespace lc {

// Debugging aid (LC_DEBUG_SEGV=1): print the native stack of a crashing thread before dying.
static void segv_handler(int sig) {
  void* bt[96];
  const int n = backtrace(bt, 96);
  const char msg[] = "\n[liblc_gpu] fatal signal, native backtrace:\n";
  ssize_t w = write(2, msg, sizeof(msg) - 1);
  (void)w;
  backtrace_symbols_fd(bt, n, 2);
  signal(sig, SIG_DFL);
  raise(sig);
}

static void maybe_install_segv_handler() {
  static bool done = false;
  if (done) return;
  done = true;
  const char* e = std::getenv("LC_DEBUG_SEGV");
  if (!e || e[0] != '1') return;
  static char alt[1 << 16];
  stack_t ss;
  ss.ss_sp = alt;
  ss.ss_size = sizeof(alt);
  ss.ss_flags = 0;
  sigaltstack(&ss, nullptr);
  struct sigaction sa;
  std::memset(&sa, 0, sizeof(sa));
  sa.sa_handler = segv_handler;
  sa.sa_flags = SA_ONSTACK;
  sigaction(SIGSEGV, &sa, nullptr);
  sigaction(SIGBUS, &sa, nullptr);
  sigaction(SIGABRT, &sa, nullptr);
}

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }

// ---- arena -------------------------------------------------------------------------------------
DeviceArena::~DeviceArena() {
  for (auto& s : slabs_)
    if (s.base) cudaFree(s.base);
}

uint8_t* DeviceArena::alloc(uint64_t bytes, uint32_t* slab_out) {
  bytes = round_up(bytes ? bytes : 1, 128);
  hit_limit_ = false;
  // 1. first fit among the holes left by released entries
  for (uint32_t i = 0; i < slabs_.size(); ++i) {
    Slab& s = slabs_[i];
    if (!s.base) continue;
    for (auto it = s.holes.begin(); it != s.holes.end(); ++it) {
      if (it->second < bytes) continue;
      const uint64_t off = it->first, rest = it->second - bytes;
      s.holes.erase(it);
      if (rest) s.holes.emplace(off + bytes, rest);
      s.live += bytes;
      used_ += bytes;
      *slab_out = i;
      return s.base + off;
    }
  }
  // 2. bump inside an existing slab
  for (uint32_t i = 0; i < slabs_.size(); ++i) {
    Slab& s = slabs_[i];
    if (!s.base) continue;
    if (s.bump + bytes <= s.size) {
      uint8_t* p = s.base + s.bump;
      s.bump += bytes;
      s.live += bytes;
      used_ += bytes;
      *slab_out = i;
      return p;
    }
  }
  // 3. a new slab, as long as the reservation stays within the limit
  Slab s;
  s.size = bytes > kSlabBytes ? bytes : kSlabBytes;
  if (limit_ && reserved_ + s.size > limit_) {
    if (reserved_ + bytes > limit_) {  // the reservation is what the budget bounds
      hit_limit_ = true;
      return nullptr;
    }
    s.size = limit_ - reserved_;                       // the last slab takes what is left of it
  }
  if (cudaMalloc(reinterpret_cast<void**>(&s.base), s.size) != cudaSuccess) {
    cudaGetLastError();
    // retry with an exact-size slab before giving up
    s.size = bytes;
    if (cudaMalloc(reinterpret_cast<void**>(&s.base), s.size) != cudaSuccess) {
      cudaGetLastError();
      return nullptr;
    }
  }
  reserved_ += s.size;
  s.bump = bytes;
  s.live = bytes;
  used_ += bytes;
  // reuse a vacated slot if any
  for (uint32_t i = 0; i < slabs_.size(); ++i) {
    if (!slabs_[i].base) {
      slabs_[i] = s;
      *slab_out = i;
      return s.base;
    }
  }
  slabs_.push_back(s);
  *slab_out = static_cast<uint32_t>(slabs_.size() - 1);
  return s.base;
}

void DeviceArena::free(uint32_t slab, uint8_t* p, uint64_t bytes) {
  bytes = round_up(bytes ? bytes : 1, 128);
  if (slab >= slabs_.size() || !p) return;
  Slab& s = slabs_[slab];
  if (!s.base || p < s.base || p + bytes > s.base + s.size) return;
  s.live -= bytes;
  used_ -= bytes;
  if (s.live == 0) {
    if (s.size != kSlabBytes) {  // odd-sized slab: give it back
      cudaFree(s.base);
      reserved_ -= s.size;
      s = Slab();
    } else {
      s.bump = 0;
      s.holes.clear();
    }
    return;
  }
  uint64_t off = static_cast<uint64_t>(p - s.base), len = bytes;
  // coalesce with the neighbours
  auto next = s.holes.lower_bound(off);
  if (next != s.holes.begin()) {
    auto prev = std::prev(next);
    if (prev->first + prev->second == off) {
      off = prev->first;
      len += prev->second;
      s.holes.erase(prev);
    }
  }
  if (next != s.holes.end() && off + len == next->first) {
    len += next->second;
    s.holes.erase(next);
  }
  if (off + len == s.bump) s.bump = off;  // the top of the slab: roll the bump pointer back
  else s.holes.emplace(off, len);
}

void DeviceArena::reset() {
  for (auto& s : slabs_) {
    s.bump = 0;
    s.live = 0;
    s.holes.clear();
  }
  used_ = 0;
}

// ---- scratch -----------------------------------------------------------------------------------
Scratch::~Scratch() {
  if (d) cudaFree(d);
  if (h) cudaFreeHost(h);
}

int Scratch::reserve(uint64_t d_bytes, uint64_t h_bytes) {
  d_bytes += 4096;
  h_bytes += 4096;
  if (d_bytes > d_cap) {
    uint64_t cap = d_cap ? d_cap : (8ull << 20);
    while (cap < d_bytes) cap *= 2;
    if (d) cudaFree(d);
    d = nullptr;
    d_cap = 0;
    if (cudaMalloc(reinterpret_cast<void**>(&d), cap) != cudaSuccess) {
      cudaGetLastError();
      if (cudaMalloc(reinterpret_cast<void**>(&d), d_bytes) != cudaSuccess) {
        cudaGetLastError();
        set_error("scratch: cudaMalloc of %llu bytes failed", (unsigned long long)d_bytes);
        return LC_ERR_OOM;
      }
      cap = d_bytes;
    }
    d_cap = cap;
  }
  if (h_bytes > h_cap) {
    uint64_t cap = h_cap ? h_cap : (4ull << 20);
    while (cap < h_bytes) cap *= 2;
    if (h) cudaFreeHost(h);
    h = nullptr;
    h_cap = 0;
    if (cudaHostAlloc(reinterpret_cast<void**>(&h), cap, cudaHostAllocDefault) != cudaSuccess) {
      cudaGetLastError();
      set_error("scratch: cudaHostAlloc of %llu bytes failed", (unsigned long long)cap);
      return LC_ERR_OOM;
    }
    h_cap = cap;
  }
  d_off = 0;
  h_off = 0;
  return LC_OK;
}

// ---- lanes -------------------------------------------------------------------------------------
namespace {
thread_local lc_lane* g_cur_lane = nullptr;        // set by the entry point (lane_enter) for the duration of a call
thread_local bool g_arena_hit_limit = false;
struct LaneKey {
  uint64_t uid;
  lc_lane* lane;
};
thread_local std::vector<LaneKey> g_my_lanes;      // this thread's lane in every context it has called into
std::atomic<uint64_t> g_ctx_uid{1};
}  // namespace

uint64_t next_ctx_uid() { return g_ctx_uid.fetch_add(1); }

// The calling thread's lane of `ctx`, created on first use (its own non-blocking stream). Returns nullptr on CUDA failure.
lc_lane* lane_of_thread(lc_ctx* ctx) {
  for (const LaneKey& k : g_my_lanes)
    if (k.uid == ctx->uid) return k.lane;
  auto lane = std::make_unique<lc_lane>();
  if (cudaStreamCreateWithFlags(&lane->own_stream, cudaStreamNonBlocking) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  lane->stream = lane->own_stream;
  lc_lane* raw = lane.get();
  {
    std::lock_guard<std::mutex> g(ctx->mu);
    ctx->lanes.push_back(std::move(lane));
  }
  g_my_lanes.push_back({ctx->uid, raw});
  return raw;
}

lc_lane* lane_enter(lc_ctx* ctx) {
  lc_lane* prev = g_cur_lane;
  g_cur_lane = lane_of_thread(ctx);
  if (!g_cur_lane) {  // no stream to be had for this thread: share the context's first lane rather than fail the call
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!ctx->lanes.empty()) g_cur_lane = ctx->lanes[0].get();
  }
  return prev;
}
void lane_leave(lc_lane* prev) { g_cur_lane = prev; }
void lane_set_current(lc_lane* l) { g_cur_lane = l; }

// Entries published by one thread are read by others on their own streams: wait for this lane's work before an entry
// becomes visible, and for EVERY lane's work before an entry's HBM range is handed back to the arena.
void sync_all_lanes(lc_ctx* ctx) {
  std::vector<cudaStream_t> streams;
  {
    std::lock_guard<std::mutex> g(ctx->mu);
    for (auto& l : ctx->lanes) streams.push_back(l->stream);
  }
  for (cudaStream_t st : streams) cudaStreamSynchronize(st);
}

void release_entry(lc_ctx* ctx, Entry* e) {
  if (!e) return;
  if (e->refcount.fetch_sub(1) > 1) return;
  if (e->d_blob) {
    bool many;
    {
      std::lock_guard<std::mutex> g(ctx->mu);
      many = ctx->lanes.size() > 1;
    }
    if (many) sync_all_lanes(ctx);  // another thread's scan may still be reading the blob on its stream
    ctx->arena_free(e->slab, e->d_blob, e->blob_bytes);
  }
  ctx->epoch++;
  e->magic = 0;
  ctx->n_entries--;
  delete e;
}

}  // namespace lc

using namespace lc;

lc_lane* lc_ctx::L() const { return g_cur_lane; }

uint8_t* lc_ctx::arena_alloc(uint64_t bytes, uint32_t* slab_out) {
  std::lock_guard<std::mutex> g(mu);
  g_arena_hit_limit = false;
  if (budget && arena.bytes_used() + round_up(bytes ? bytes : 1, 128) > budget) {  // the budget is checked with the allocation
    g_arena_hit_limit = true;
    return nullptr;
  }
  uint8_t* p = arena.alloc(bytes, slab_out);
  if (!p) g_arena_hit_limit = arena.at_limit();
  return p;
}
void lc_ctx::arena_free(uint32_t slab, uint8_t* p, uint64_t bytes) {
  std::lock_guard<std::mutex> g(mu);
  arena.free(slab, p, bytes);
}
uint64_t lc_ctx::arena_used() {
  std::lock_guard<std::mutex> g(mu);
  return arena.bytes_used();
}
bool lc_ctx::arena_at_limit() const { return g_arena_hit_limit; }
std::shared_ptr<FsstCodec> lc_ctx::codec_of(uint64_t scope) {
  std::shared_ptr<CodecSlot> slot;
  {
    std::lock_guard<std::mutex> g(mu);
    auto it = codecs.find(scope);
    if (it == codecs.end()) return nullptr;
    slot = it->second;
  }
  std::lock_guard<std::mutex> g(slot->mu);  // a table being trained right now: wait for it
  return slot->codec;
}
std::shared_ptr<lc_ctx::CodecSlot> lc_ctx::codec_slot(uint64_t scope) {
  std::lock_guard<std::mutex> g(mu);
  auto& slot = codecs[scope];
  if (!slot) slot = std::make_shared<CodecSlot>();
  return slot;
}

extern "C" {

const char* lc_last_error(void) { return get_error(); }
const char* lc_version(void) { return "liquid_cache_b200 0.1 (sm_90a)"; }

int lc_ctx_create(int device_id, uint64_t hbm_budget_bytes, lc_ctx** out) {
  if (!out) {
    set_error("lc_ctx_create: out is NULL");
    return LC_ERR_INVALID;
  }
  maybe_install_segv_handler();
  int n_dev = 0;
  cudaError_t e = cudaGetDeviceCount(&n_dev);
  if (e != cudaSuccess || n_dev == 0) {
    cudaGetLastError();
    set_error("no CUDA device visible (%s); this library has no CPU fallback",
              e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
    return LC_ERR_NO_DEVICE;
  }
  if (device_id < 0 || device_id >= n_dev) {
    set_error("device %d out of range (%d devices)", device_id, n_dev);
    return LC_ERR_INVALID;
  }
  LC_CUDA_OK(cudaSetDevice(device_id));
  cudaDeviceProp prop;
  LC_CUDA_OK(cudaGetDeviceProperties(&prop, device_id));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("device %d is sm_%d%d; this library ships sm_90a code only", device_id, prop.major, prop.minor);
    return LC_ERR_NO_DEVICE;
  }
  lc_ctx* ctx = new lc_ctx();
  ctx->device = device_id;
  ctx->budget = hbm_budget_bytes;
  ctx->uid = next_ctx_uid();
  ctx->arena.set_limit(hbm_budget_bytes ? round_up(hbm_budget_bytes, 2ull << 20) : 0);
  if (!lane_of_thread(ctx)) {  // the creating thread's lane: the context's first stream
    set_error("cudaStreamCreate failed: %s", cudaGetErrorString(cudaGetLastError()));
    delete ctx;
    return LC_ERR_CUDA;
  }
  // keep stream-ordered allocations cached in the pool across synchronisations (the default threshold of 0
  // hands the memory back to the driver at every sync, which costs milliseconds per call)
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device_id) == cudaSuccess) {
    uint64_t keep = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  }
  cudaGetLastError();
  *out = ctx;
  return LC_OK;
}

void lc_ctx_destroy(lc_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  sync_all_lanes(ctx);
  lc_lane* prev = lane_enter(ctx);
  std::vector<Entry*> held;
  {
    std::lock_guard<std::mutex> g(ctx->mu);
    for (auto& kv : ctx->cache)
      if (Entry* e = entry_of(kv.second)) held.push_back(e);
    ctx->cache.clear();
  }
  for (Entry* e : held) release_entry(ctx, e);
  for (auto& kv : ctx->codecs) {
    auto& c = kv.second->codec;
    if (!c) continue;
    if (c->d_dec) cudaFree(c->d_dec);
    if (c->d_enc) cudaFree(c->d_enc);
    c->d_dec = nullptr;
    c->d_enc = nullptr;
  }
  for (auto& lp : ctx->lanes) {
    lc_lane* l = lp.get();
    lane_set_current(l);
    drop_ref_cache(ctx);
    if (l->d_needle) cudaFree(l->d_needle);
    if (l->sel_stage) cudaFreeHost(l->sel_stage);
    if (l->d_pairs) cudaFree(l->d_pairs);
    if (l->copy_stream) cudaStreamDestroy(l->copy_stream);
    for (cudaEvent_t& e : l->ev_chunk)
      if (e) cudaEventDestroy(e);
    if (l->ev_a) cudaEventDestroy(l->ev_a);
    if (l->ev_b) cudaEventDestroy(l->ev_b);
    if (l->own_stream) cudaStreamDestroy(l->own_stream);
  }
  if (ctx->d_prof) cudaFree(ctx->d_prof);
  lane_leave(prev);
  delete ctx;  // threads that called into this context keep a stale (uid-keyed, never matched again) lane pointer
}

int lc_ctx_set_stream(lc_ctx* ctx, void* cuda_stream) {  // the calling thread's lane
  if (!ctx) return LC_ERR_INVALID;
  lc_lane* l = lane_of_thread(ctx);
  if (!l) return LC_ERR_CUDA;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(l->stream);
  l->stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : l->own_stream;
  return LC_OK;
}

int lc_ctx_synchronize(lc_ctx* ctx) {  // the calling thread's work
  if (!ctx) return LC_ERR_INVALID;
  lc_lane* l = lane_of_thread(ctx);
  if (!l) return LC_ERR_CUDA;
  cudaSetDevice(ctx->device);
  LC_CUDA_OK(cudaStreamSynchronize(l->stream));
  return LC_OK;
}

int lc_ctx_profile_counters(lc_ctx* ctx, int enable, uint64_t out[16]) {
  if (!ctx) return LC_ERR_INVALID;
  lc_lane* prev = lane_enter(ctx);
  struct Leave {
    lc_lane* p;
    ~Leave() { lane_leave(p); }
  } leave{prev};
  if (!ctx->L()) return LC_ERR_CUDA;
  cudaSetDevice(ctx->device);
  if (!ctx->d_prof) {
    if (cudaMalloc(reinterpret_cast<void**>(&ctx->d_prof), 128) != cudaSuccess) {
      cudaGetLastError();
      set_error("cudaMalloc for profile counters failed");
      return LC_ERR_OOM;
    }
    LC_CUDA_OK(cudaMemsetAsync(ctx->d_prof, 0, 128, ctx->L()->stream));
  }
  LC_CUDA_OK(cudaStreamSynchronize(ctx->L()->stream));
  if (out) {
    unsigned long long tmp[16] = {0};
    LC_CUDA_OK(cudaMemcpy(tmp, ctx->d_prof, 128, cudaMemcpyDeviceToHost));
    for (int i = 0; i < 16; ++i) out[i] = tmp[i];
  }
  if (enable && !ctx->prof_on) LC_CUDA_OK(cudaMemset(ctx->d_prof, 0, 128));
  ctx->prof_on = enable != 0;
  return LC_OK;
}

int lc_ctx_kernel_timing(lc_ctx* ctx, int enable) {  // the calling thread's lane
  if (!ctx) return LC_ERR_INVALID;
  lc_lane* prev = lane_enter(ctx);
  struct Leave {
    lc_lane* p;
    ~Leave() { lane_leave(p); }
  } leave{prev};
  if (!ctx->L()) return LC_ERR_CUDA;
  cudaSetDevice(ctx->device);
  if (enable && !ctx->L()->ev_a) {
    LC_CUDA_OK(cudaEventCreate(&ctx->L()->ev_a));
    LC_CUDA_OK(cudaEventCreate(&ctx->L()->ev_b));
  }
  ctx->L()->timing_on = enable != 0;
  ctx->L()->timing_valid = false;
  return LC_OK;
}

float lc_ctx_last_kernel_ms(lc_ctx* ctx) {
  if (!ctx) return -1.0f;
  lc_lane* prev = lane_enter(ctx);
  struct Leave {
    lc_lane* p;
    ~Leave() { lane_leave(p); }
  } leave{prev};
  if (!ctx->L() || !ctx->L()->timing_valid) return -1.0f;
  cudaSetDevice(ctx->device);
  if (cudaEventSynchronize(ctx->L()->ev_b) != cudaSuccess) return -1.0f;
  float ms = -1.0f;
  if (cudaEventElapsedTime(&ms, ctx->L()->ev_a, ctx->L()->ev_b) != cudaSuccess) return -1.0f;
  return ms;
}

int lc_ctx_stats(lc_ctx* ctx, lc_stats* out) {
  if (!ctx || !out) return LC_ERR_INVALID;
  out->entries = ctx->n_entries;
  out->hbm_bytes_used = ctx->arena_used();
  std::lock_guard<std::mutex> g(ctx->mu);
  out->hbm_bytes_budget = ctx->budget;
  out->kernel_launches = ctx->kernel_launches;
  out->h2d_bytes = ctx->h2d_bytes;
  out->d2h_bytes = ctx->d2h_bytes;
  out->hbm_bytes_reserved = ctx->arena.bytes_reserved();
  return LC_OK;
}

}  // extern "C"

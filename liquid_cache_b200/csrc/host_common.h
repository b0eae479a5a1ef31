// host_common.h — host-side state behind the C ABI: context, HBM arena, scratch, entries.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/lc_gpu.h"
#include "entry_layout.h"
#include "squeeze_plan.h"
#include "fixed_math.cuh"
#include "kernels.h"

namespace lc {

// ---- errors ------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
const char* get_error();

#define LC_CUDA_OK(expr)                                                                       \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      ::lc::set_error("CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__, __LINE__, \
                      cudaGetErrorString(_e));                                                 \
      return LC_ERR_CUDA;                                                                      \
    }                                                                                          \
  } while (0)

#define LC_TRY(expr)            \
  do {                          \
    int _rc = (expr);           \
    if (_rc != LC_OK) return _rc; \
  } while (0)

inline uint64_t round_up(uint64_t x, uint64_t a) { return (x + a - 1) / a * a; }

// ---- HBM arena ---------------------------------------------------------------------------------
// Entries are immutable blobs; the arena hands out 128-byte aligned ranges from large cudaMalloc'd
// slabs: bump pointer per slab, freed ranges kept as coalesced holes and reused first-fit (a range freed at the top of
// a slab rolls the bump pointer back), so insert / replace / remove churn recycles HBM instead of growing the
// reservation. `limit` caps the RESERVATION (what cudaMalloc has handed out), which is what with_max_memory_bytes bounds.
class DeviceArena {
 public:
  ~DeviceArena();
  // returns nullptr on cudaMalloc failure, or when a new slab would take the reservation past `limit` (0 = no limit)
  uint8_t* alloc(uint64_t bytes, uint32_t* slab_out);
  void free(uint32_t slab, uint8_t* p, uint64_t bytes);
  void set_limit(uint64_t limit) { limit_ = limit; }
  bool at_limit() const { return hit_limit_; }  // did the last failed alloc() stop at the limit (rather than at cudaMalloc)?
  void reset();
  uint64_t bytes_used() const { return used_; }
  uint64_t bytes_reserved() const { return reserved_; }

 private:
  struct Slab {
    uint8_t* base = nullptr;
    uint64_t size = 0, bump = 0, live = 0;
    std::map<uint64_t, uint64_t> holes;  // offset -> bytes, below `bump`, coalesced
  };
  uint64_t limit_ = 0;
  bool hit_limit_ = false;
  static constexpr uint64_t kSlabBytes = 256ull << 20;
  std::vector<Slab> slabs_;
  uint64_t used_ = 0, reserved_ = 0;
};

// Growable device + pinned-host scratch, bump-allocated inside one API call.
struct Scratch {
  uint8_t* d = nullptr;
  uint64_t d_cap = 0, d_off = 0;
  uint8_t* h = nullptr;  // pinned
  uint64_t h_cap = 0, h_off = 0;
  ~Scratch();
  void reset() { d_off = 0; h_off = 0; }
  // Both return nullptr on allocation failure. Growing invalidates earlier pointers, so callers
  // reserve() the total first.
  int reserve(uint64_t d_bytes, uint64_t h_bytes);
  uint8_t* dev(uint64_t bytes) {
    uint64_t o = round_up(d_off, 256);
    if (o + bytes > d_cap) return nullptr;
    d_off = o + bytes;
    return d + o;
  }
  uint8_t* host(uint64_t bytes) {
    uint64_t o = round_up(h_off, 64);
    if (o + bytes > h_cap) return nullptr;
    h_off = o + bytes;
    return h + o;
  }
};

// ---- FSST symbol table (host copy + device copies), one per compressor scope --------------------
struct FsstCodec {
  FsstTable dec;                       // decode view (symbols + lengths)
  std::unique_ptr<FsstEncTable> enc;   // encode lookup
  FsstTable* d_dec = nullptr;          // device copies (cudaMalloc'd, tiny)
  FsstEncTable* d_enc = nullptr;
};
// fsst_host.cc
void fsst_train(const uint8_t* const* strs, const uint32_t* lens, size_t n, FsstCodec* out);
void fsst_from_symbols(const uint64_t* vals, const uint8_t* lens, size_t n, FsstCodec* out);
size_t fsst_compress_host(const FsstCodec& c, const uint8_t* in, size_t len, uint8_t* out);
size_t fsst_decompress_host(const FsstTable& t, const uint8_t* in, size_t len, uint8_t* out, size_t cap);

// ---- entries -----------------------------------------------------------------------------------
constexpr uint32_t kEntryMagic = 0x4C43454Eu;

struct Entry {
  uint32_t magic = kEntryMagic;
  int32_t liquid_type = 0;  // lc_liquid_type
  uint8_t* d_blob = nullptr;
  uint32_t blob_bytes = 0;
  uint32_t slab = 0;
  uint32_t n = 0;
  std::atomic<uint32_t> refcount{1};
  uint32_t dec_width = 0;    // decimals: bytes per Arrow value (16 = Decimal128, 32 = Decimal256)
  std::string arrow_format;  // original arrow type as C format string (dictionary: "S" + value fmt in dict_format)
  std::string dict_value_format;
  IntHeader ih;   // host copies of the blob header
  StrHeader sh;
  std::vector<uint8_t> shared_prefix;  // byte-view: host copy (predicate planning)
  std::shared_ptr<FsstCodec> codec;    // byte-view
  // squeezed integers (LiquidPrimitiveClampedArray / LiquidPrimitiveQuantizedArray): the blob holds half-width codes,
  // the full LQDA image sits behind the caller's read function
  int32_t squeeze_kind = 0;            // 0 = a full entry, 1 clamp, 2 quantize, 3 date component (SqueezedDate32Array)
  uint64_t bucket_width = 0;           // quantize
  uint32_t date_field = 0;             // date component: 0 year, 1 month, 2 day, 3 day of week
  std::string orig_format;             // date component: the column's own arrow type (the blob itself reads as Date32)
  lc_backing_read backing_read = nullptr;
  void* backing_user = nullptr;
  uint64_t backing_len = 0;            // disk_range = 0..backing_len
  uint32_t fixed_width = 0;            // LiquidFixedLenByteArray (decimals outside u64): bytes per value, else 0
};

// int_encode's answer for a decimal array with values outside u64: the caller stores it as LiquidFixedLenByteArray
// (str_encode over the 16 / 32-byte values) under the column chunk's compressor scope
constexpr int LC_INTERNAL_FIXED_LEN = 1000;
// order-preserving form of fixed-width decimals: fixed_math.cuh (host + device)

// integer-shaped blobs (IntHeader + FastLanes chunks): integers, ALP floats, u64 decimals
inline bool is_int_blob(int32_t liquid_type) {
  return liquid_type == LC_LIQUID_INTEGER || liquid_type == LC_LIQUID_FLOAT || liquid_type == LC_LIQUID_DECIMAL;
}

inline Entry* entry_of(lc_handle h) {
  Entry* e = reinterpret_cast<Entry*>(static_cast<uintptr_t>(h));
  return (e && e->magic == kEntryMagic) ? e : nullptr;
}

}  // namespace lc

// Everything one call mutates besides the shared cache state: stream, scratch, staging buffers, the per-list device caches.
// One per CALLING THREAD (created on the thread's first call into a context, owned by the context), so calls from
// different threads never share mutable state and need no lock while they run — the reference's `Arc<LiquidCache>` is hit by
// every DataFusion partition task at once (cache/core.rs:52-63, index.rs:12-60). The first lane carries the context's own
// stream (or the caller's, lc_ctx_set_stream applies to the calling thread's lane).
// Key of a cached list of handles / entry pointers. Four independent lanes so that a 12 k-element list hashes in a few
// microseconds (a single multiply chain is latency-bound: ~20 us per call, paid by every filter of a scan).
inline uint64_t hash_words(const uint64_t* p, uint64_t n) {
  uint64_t a = 0x9E3779B97F4A7C15ull ^ n, b = 0xC2B2AE3D27D4EB4Full, c = 0x165667B19E3779F9ull, d = 0x27D4EB2F165667C5ull;
  uint64_t i = 0;
  for (; i + 4 <= n; i += 4) {
    a = (a ^ p[i]) * 0xff51afd7ed558ccdull;
    b = (b ^ p[i + 1]) * 0xc4ceb9fe1a85ec53ull;
    c = (c ^ p[i + 2]) * 0x9fb21c651e98df25ull;
    d = (d ^ p[i + 3]) * 0xd6e8feb86659fd93ull;
  }
  for (; i < n; ++i) a = (a ^ p[i]) * 0xff51afd7ed558ccdull;
  uint64_t x = a ^ (b >> 17) ^ (c << 23) ^ (d >> 31) ^ (b << 41);
  x ^= x >> 32;
  return x;
}

extern std::atomic<uint64_t> g_validated_gen;  // lc_ctx.cc

struct lc_lane {
  cudaStream_t own_stream = nullptr;
  cudaStream_t stream = nullptr;
  lc::Scratch scratch;
  uint8_t* d_needle = nullptr;   // small device buffer for predicate needles (lc_scan_filter)
  std::string needle_in_buffer;  // ... what it holds, and the stream the upload was ordered on
  cudaStream_t needle_stream = nullptr;
  double onepass_bytes_per_row = 96.0;  // decoded bytes per row of the last sparse string read (sizes the speculative download)
  cudaStream_t copy_stream = nullptr;  // results of chunk c travel to the host while chunk c+1 is computed
  cudaEvent_t ev_chunk[4] = {nullptr, nullptr, nullptr, nullptr};
  void* ref_cache = nullptr;     // scan_host.cc: device-side entry lists cached per handle list
  // handle arrays already validated (hash of the array -> entries) for the batched calls: a repeated call over the same
  // column costs a hash of the array instead of one pointer chase per handle; any release bumps `epoch` and voids them
  // Entry lists handed out by the validation caches (lc_abi.cc) are immutable while they live. `tok_*` names the one the
  // current call was given and the value of g_validated_gen at that moment; `fast_*` remembers the hash scan_host.cc
  // computed for exactly that (pointer, n, generation) — so the SAME list on the NEXT call finds its device-side list
  // without hashing and comparing 12 k pointers again. Any creation or destruction of a validated list anywhere bumps
  // the generation, which voids both.
  const void* tok_ptr = nullptr;
  uint64_t tok_n = 0, tok_gen = 0;
  const void* fast_ptr = nullptr;
  uint64_t fast_n = 0, fast_gen = 0, fast_key = 0, fast_epoch = 0;
  struct ValidatedHandles {
    uint64_t key = 0, n = 0, epoch = 0;
    std::vector<lc_handle> handles;  // the list itself: the key only pre-filters, the match is exact
    std::vector<lc::Entry*> es;
  };
  std::vector<ValidatedHandles> validated;
  uint8_t* d_pairs = nullptr;    // device buffer for sparse selection uploads ({word index, word} pairs)
  uint64_t d_pairs_cap = 0;
  uint8_t* sel_stage = nullptr;  // pinned staging of the caller's selection bitmaps (batched calls)
  uint64_t sel_stage_cap = 0;
  bool timing_on = false;        // lc_ctx_kernel_timing
  bool timing_valid = false;
  cudaEvent_t ev_a = nullptr, ev_b = nullptr;
  bool squeeze_internal = false; // squeeze_host.cc is driving the batch functions (they refuse squeezed entries otherwise)
};

struct lc_ctx {
  int device = 0;
  uint64_t budget = 0;
  uint64_t uid = 0;              // process-unique: keys the calling threads' lane lookup
  // SHARED state. `mu` is held only around the short operations on it (arena alloc / free, cache map, codec map, lane list)
  // — never across a kernel launch or a synchronisation.
  std::mutex mu;
  lc::DeviceArena arena;
  std::unordered_map<uint64_t, lc_handle> cache;                               // entry_id -> handle
  struct CodecSlot {             // one per compressor scope: trained once, by whoever gets there first
    std::mutex mu;
    std::shared_ptr<lc::FsstCodec> codec;
  };
  std::unordered_map<uint64_t, std::shared_ptr<CodecSlot>> codecs;             // compressor scope -> table
  std::vector<std::unique_ptr<lc_lane>> lanes;
  std::atomic<uint64_t> n_entries{0};
  std::atomic<uint64_t> kernel_launches{0}, h2d_bytes{0}, d2h_bytes{0};
  std::atomic<uint64_t> epoch{0};           // bumped whenever an entry is released (invalidates cached entry lists)
  std::atomic<uint64_t> squeeze_reads{0}, squeeze_saved{0};  // backing reads / calls answered from the half-width codes
  unsigned long long* d_prof = nullptr;  // profile counters (lc_ctx_profile_counters; measurement aid, shared)
  bool prof_on = false;

  // the calling thread's lane (set by the entry point's Guard for the duration of the call)
  lc_lane* L() const;
  // arena under the lock; the budget is checked inside, with the allocation
  uint8_t* arena_alloc(uint64_t bytes, uint32_t* slab_out);
  void arena_free(uint32_t slab, uint8_t* p, uint64_t bytes);
  uint64_t arena_used();
  bool arena_at_limit() const;   // did the calling thread's last failed arena_alloc stop at the budget?
  // codec of a compressor scope, or null; and the slot to train under
  std::shared_ptr<lc::FsstCodec> codec_of(uint64_t scope);
  std::shared_ptr<CodecSlot> codec_slot(uint64_t scope);
};

namespace lc {

// An arena range that goes back to the arena unless an Entry took it over (early returns after a CUDA error).
struct ArenaBlock {
  lc_ctx* ctx;
  uint8_t* p = nullptr;
  uint32_t slab = 0;
  uint64_t bytes = 0;
  ArenaBlock(lc_ctx* c, uint64_t b) : ctx(c), bytes(b) { p = c->arena_alloc(b, &slab); }
  ~ArenaBlock() {
    if (p) ctx->arena_free(slab, p, bytes);
  }
  uint8_t* release() {  // ownership moves to an Entry
    uint8_t* r = p;
    p = nullptr;
    return r;
  }
  ArenaBlock(const ArenaBlock&) = delete;
  ArenaBlock& operator=(const ArenaBlock&) = delete;
};

// ---- Arrow C data helpers (arrow_io.cc) ---------------------------------------------------------
struct HostBuf {  // 64-byte aligned host allocation
  uint8_t* p = nullptr;
  uint64_t bytes = 0;
};
uint8_t* host_alloc(uint64_t bytes, bool force_pinned = false);  // force_pinned: a page-locked block even below 1 MiB
void host_free(uint8_t* p);

// A host_alloc block that goes back to host_free unless release() handed it to export_array (early returns, CUDA errors).
struct HostBlock {
  uint8_t* p = nullptr;
  uint64_t bytes = 0;  // what the Arrow buffer holds; the allocation may be larger
  HostBlock() = default;
  HostBlock(uint64_t alloc_bytes, uint64_t b, bool force_pinned = false) : p(host_alloc(alloc_bytes, force_pinned)), bytes(b) {}
  ~HostBlock() { host_free(p); }
  HostBlock(HostBlock&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; }
  HostBlock& operator=(HostBlock&& o) noexcept {
    if (this != &o) {
      host_free(p);
      p = o.p;
      bytes = o.bytes;
      o.p = nullptr;
    }
    return *this;
  }
  HostBuf release() {  // ownership moves into an exported array
    HostBuf r{p, bytes};
    p = nullptr;
    return r;
  }
};

// Parsed view of an input array (borrowed pointers).
struct ArrowIn {
  enum Kind { K_INT, K_BYTES, K_VIEW, K_DICT, K_FLOAT, K_DECIMAL } kind;
  uint8_t phys = 0, tbits = 0;
  uint32_t dec_width = 0;  // K_DECIMAL: 16 / 32 bytes per value
  bool is_signed = false;
  uint8_t byte_type = 0;  // ByteType of the ORIGINAL array type
  int64_t length = 0, offset = 0, null_count = 0;
  const uint8_t* validity = nullptr;  // bitmap with bit offset `offset`
  const void* values = nullptr;       // ints: native values (not yet offset); bytes: int32 offsets
  const uint8_t* data = nullptr;      // bytes: value bytes
  const void* const* view_buffers = nullptr;  // views: variadic data buffers
  int64_t n_view_buffers = 0;
  // dictionary (keys must be uint16)
  const uint16_t* dict_keys = nullptr;
  int64_t dict_len = 0, dict_offset = 0;
  const int32_t* dict_offsets = nullptr;
  const uint8_t* dict_data = nullptr;
  const uint8_t* dict_validity = nullptr;
  std::string format, dict_value_format;
};
int parse_arrow_input(const ArrowSchema* schema, const ArrowArray* array, ArrowIn* out);
inline bool bit_get(const uint8_t* bits, int64_t i) { return (bits[i >> 3] >> (i & 7)) & 1; }
// copy `n` bits starting at bit `off` of src into dst (bit offset 0), zero padding to `dst_bytes`
void copy_bits(const uint8_t* src, int64_t off, int64_t n, uint8_t* dst, uint64_t dst_bytes);
uint64_t popcount_bits(const uint8_t* bits, uint64_t n);

// Build caller-owned Arrow C structs around malloc'd buffers (released by the release callbacks).
void export_schema(const std::string& format, const std::string& dict_value_format, ArrowSchema* out);
// buffers: ownership moves into the array. dictionary may be null.
void export_array(int64_t length, int64_t null_count, std::vector<HostBuf> buffers, ArrowArray* dictionary,
                  ArrowArray* out);

// ---- per-type host orchestration ----------------------------------------------------------------
// int_host.cc
int int_encode(lc_ctx* ctx, const ArrowIn& in, Entry** out);
int int_encode_many(lc_ctx* ctx, const std::vector<ArrowIn>& ins, std::vector<Entry*>* out);  // K_INT batches only
// ipc_host.cc: LQDA (the reference's serialized form) of integer-shaped entries
int entry_to_bytes(lc_ctx* ctx, const Entry* e, uint8_t* out, uint64_t cap, uint64_t* out_bytes);
int entry_from_bytes(lc_ctx* ctx, const uint8_t* bytes, uint64_t len, const std::shared_ptr<FsstCodec>& codec, Entry** out);
int symbol_table_to_bytes(const FsstCodec& c, uint8_t* out, uint64_t cap, uint64_t* out_bytes);
int symbol_table_from_bytes(const uint8_t* bytes, uint64_t len, FsstCodec* out);
int register_codec(lc_ctx* ctx, uint64_t scope, const std::shared_ptr<FsstCodec>& codec);  // str_host.cc: device copies + ctx->codecs
// str_host.cc
int str_encode(lc_ctx* ctx, const ArrowIn& in, int32_t hint, uint64_t scope, Entry** out);
int str_encode_many(lc_ctx* ctx, const std::vector<ArrowIn>& ins, int32_t hint, const uint64_t* scopes, std::vector<Entry*>* out);

// scan_host.cc: batched operations over homogeneous entry lists (all int or all byte-view)
struct PredOut {
  uint8_t* values;            // host
  uint8_t* validity;          // host or null
  const uint64_t* byte_offsets;
  uint64_t* len;
  uint64_t* null_count;
  uint64_t* true_count;       // optional: set bits of each mask (nulls count as false)
};
int eval_predicate_batch(lc_ctx* ctx, Entry* const* entries, uint64_t n, const lc_predicate* pred,
                         const uint8_t* const* sel_bits, const PredOut& out);
// Selections that already live in HBM (the scan pipeline): word-aligned per entry.
struct DevSel {
  const uint32_t* d_base;      // selection words of all batches, back to back
  const uint64_t* word_off;    // per entry, in u32 words
  const uint32_t* k;           // per entry popcount (host copy)
  bool all_rows;               // no filter applied yet: every row selected
};
// Where a get() leaves its result.
struct DeviceOut {             // caller-owned device buffers (lc_scan_read_device)
  void* d_values;
  uint64_t values_cap;
  void* d_offsets;
  void* d_validity;
  uint64_t* out_rows;
  uint64_t* out_value_bytes;
  uint64_t* out_null_count;
};
int to_arrow_batch(lc_ctx* ctx, Entry* const* entries, uint64_t n, const uint8_t* const* sel_bits,
                   const DevSel* dev_sel, ArrowSchema* out_schema, ArrowArray* out_array,
                   const DeviceOut* dev_out = nullptr);

// squeeze_host.cc
int squeezed_eval_predicate_many(lc_ctx* ctx, Entry* const* entries, uint64_t n, const lc_predicate* pred,
                                 const uint8_t* const* sel_bits, const PredOut& out);
int squeeze_doubt(const Entry* e, const lc_predicate* pred, lc_predicate* probe);
int squeeze_hydrate(lc_ctx* ctx, const Entry* sq, Entry** full);
int squeeze_entry(lc_ctx* ctx, Entry* full, int32_t policy, int32_t hint, lc_backing_read read, void* user, uint8_t* bytes_out,
                  uint64_t cap, uint64_t* out_bytes, Entry** out);
int squeezed_eval_predicate(lc_ctx* ctx, Entry* sq, const lc_predicate* pred, const uint8_t* sel_bits, const PredOut& out);
int squeezed_to_arrow(lc_ctx* ctx, Entry* sq, const uint8_t* sel_bits, ArrowSchema* out_schema, ArrowArray* out_array);
int squeezed_component_array(lc_ctx* ctx, Entry* sq, int32_t lossy, ArrowSchema* out_schema, ArrowArray* out_array);

// Device-planned reads of a scan (scan_host.cc scan_read_fused): sizes of the previous read of the same scan (they size the
// capacities and the speculative download of the next one) and the buffers kept between calls.
constexpr int LC_INTERNAL_FALLBACK = 1001;
struct FusedRead {
  bool have_spec = false;
  uint64_t spec_rows = 0, spec_bytes = 0, spec_ulen = 0;
  uint8_t* d_buf = nullptr;
  uint64_t d_cap = 0;
  uint8_t* a_buf = nullptr;      // scratch of the asynchronous form (scan_read_async)
  uint64_t a_cap = 0;
  ScanPlanHdr* h_hdr = nullptr;  // pinned
};
struct FusedDeviceOut {  // lc_scan_read_borrowed: the concatenated result left in the scan's own device buffer
  void* d_values = nullptr;
  void* d_offsets = nullptr;  // byte views: int32[rows + 1] (the closing offset included); integers: nullptr
  uint64_t rows = 0, value_bytes = 0;
};
int scan_read_fused(lc_ctx* ctx, FusedRead* fr, Entry* const* entries, uint64_t n, const uint32_t* d_sel, const uint64_t* d_word_off,
                    const uint32_t* d_counts2, uint64_t total_rows_in, ArrowSchema* out_schema, ArrowArray* out_array,
                    FusedDeviceOut* dev_out = nullptr);
int scan_read_async(lc_ctx* ctx, FusedRead* fr, Entry* const* entries, uint64_t n, const uint32_t* d_sel, const uint64_t* d_word_off,
                    const uint32_t* d_counts2, void* d_values, uint64_t values_cap, void* d_offsets, uint64_t rows_cap, void* d_header);
void fused_read_learn(FusedRead* fr, const ArrowArray* arr, int64_t value_bytes, uint64_t ulen_words);
void fused_read_free(FusedRead* fr);

int refine_batch(lc_ctx* ctx, Entry* const* entries, uint64_t n, const lc_predicate* pred, uint32_t* d_sel_base,
                 const uint64_t* d_word_off, bool all_rows, uint32_t* d_counts);
void drop_ref_cache(lc_ctx* ctx);


void release_entry(lc_ctx* ctx, Entry* e);
// lanes (lc_ctx.cc)
lc_lane* lane_of_thread(lc_ctx* ctx);
lc_lane* lane_enter(lc_ctx* ctx);     // makes the calling thread's lane current; returns the previous current lane
void lane_leave(lc_lane* prev);
void lane_set_current(lc_lane* l);
void sync_all_lanes(lc_ctx* ctx);

}  // namespace lc

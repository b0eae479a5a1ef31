// lc_abi.cc — extern "C" entry points declared in include/lc_gpu.h.
#include <algorithm>
#include <cstddef>
#include <cstring>

#include "host_common.h"

using namespace lc;

namespace {

// An entry point's frame: the calling thread's lane becomes current (stream, scratch, staging buffers — nothing another
// thread touches), the device is selected. NO context-wide lock is held while the call runs: shared state (arena, entry map,
// codec map) is locked inside the few operations that touch it.
struct Guard {
  lc_ctx* ctx;
  lc_lane* prev;
  explicit Guard(lc_ctx* c) : ctx(c), prev(lane_enter(c)) {
    cudaSetDevice(c->device);
    if (c->L()) c->L()->scratch.reset();
  }
  ~Guard() { lane_leave(prev); }
  Guard(const Guard&) = delete;
  Guard& operator=(const Guard&) = delete;
};
#define LC_LANE_OK(ctx)                                           \
  do {                                                            \
    if (!(ctx)->L()) {                                            \
      set_error("could not create a CUDA stream for this thread"); \
      return LC_ERR_CUDA;                                         \
    }                                                             \
  } while (0)

// Make freshly encoded entries visible under their ids: their kernels have finished (other threads read them on their own
// streams), the map is updated under the lock, whatever they replace is released outside it.
int publish_entries(lc_ctx* ctx, const uint64_t* ids, Entry* const* es, uint64_t n) {
  const cudaError_t ce = cudaStreamSynchronize(ctx->L()->stream);
  std::vector<Entry*> old;
  {
    std::lock_guard<std::mutex> g(ctx->mu);
    for (uint64_t i = 0; i < n; ++i) {
      auto it = ctx->cache.find(ids[i]);
      if (it != ctx->cache.end()) old.push_back(entry_of(it->second));  // overwrite (index insert replaces)
      ctx->cache[ids[i]] = static_cast<lc_handle>(reinterpret_cast<uintptr_t>(es[i]));
    }
  }
  for (Entry* e : old) release_entry(ctx, e);
  if (ce != cudaSuccess) {
    set_error("CUDA error while finishing an insert: %s", cudaGetErrorString(ce));
    return LC_ERR_CUDA;
  }
  return LC_OK;
}

int encode_locked(lc_ctx* ctx, const ArrowSchema* schema, const ArrowArray* array, int32_t hint, uint64_t scope,
                  Entry** out) {
  ArrowIn in;
  LC_TRY(parse_arrow_input(schema, array, &in));
  if (in.kind == ArrowIn::K_INT || in.kind == ArrowIn::K_FLOAT || in.kind == ArrowIn::K_DECIMAL) {
    const int rc = int_encode(ctx, in, out);
    if (rc != LC_INTERNAL_FIXED_LEN) return rc;
    // LiquidFixedLenByteArray::from_decimal_array (fix_len_byte_array.rs:274-323): u16 dictionary over the 16 / 32-byte
    // values, FSST-compressed under the column chunk's compressor (with_fsst_compressor_or_train, transcode.rs:118-131)
    in.byte_type = in.dec_width == 16 ? BT_DECIMAL128 : BT_DECIMAL256;
    ctx->L()->scratch.reset();
    return str_encode(ctx, in, LC_HINT_NONE, scope, out);
  }
  return str_encode(ctx, in, hint, scope, out);
}

}  // namespace

struct lc_scan {
  lc_ctx* ctx = nullptr;
  uint64_t n = 0;
  std::vector<uint32_t> rows;
  std::vector<uint64_t> word_off;
  uint64_t total_words = 0;
  uint32_t* d_sel = nullptr;
  uint32_t* d_counts = nullptr;
  uint64_t* d_word_off = nullptr;
  // squeezed entries only (scan_filter_squeezed), allocated on first use: probe copy / snapshot of the selection, probe counts
  uint32_t* d_probe = nullptr;
  uint32_t* d_save = nullptr;
  uint32_t* d_pcounts = nullptr;
  // lc_scan_filter_or only, allocated on first use: the term buffer T and the accumulator A (selection-sized), counts the
  // term launches write (nobody reads them) and the batch row counts k_sel_or masks the tails with
  uint32_t* d_term = nullptr;
  uint32_t* d_acc = nullptr;
  uint32_t* d_tcounts = nullptr;
  uint32_t* d_rows = nullptr;
  bool all_rows = true;       // no filter applied yet
  bool counts_on_device = false;
  bool counts_cached = false;
  std::vector<uint32_t> counts;
  // handle lists already validated against this scan (hash of the handle array -> entries), so that repeated
  // filters over the same columns cost a hash of the array instead of 12k pointer chases
  struct Validated {
    uint64_t key = 0, epoch = 0;
    bool any_squeezed = false;
    std::vector<lc_handle> handles;  // the list itself: the key only pre-filters, the match is exact
    std::vector<Entry*> es;
  };
  std::vector<Validated> validated;
  FusedRead fused;  // device-planned reads: what the previous read of this scan looked like
  // A scan is driven by one thread at a time (its device state is ordered by that thread's stream); if another thread
  // continues it, the previous thread's stream is drained first.
  std::mutex mu;
  lc_lane* last_lane = nullptr;
};

struct ScanGuard {
  std::unique_lock<std::mutex> lk;
  Guard g;
  explicit ScanGuard(lc_scan* sc) : lk(sc->mu), g(sc->ctx) {
    lc_lane* cur = sc->ctx->L();
    if (sc->last_lane && sc->last_lane != cur) cudaStreamSynchronize(sc->last_lane->stream);
    sc->last_lane = cur;
  }
};

static_assert(sizeof(lc_handle) == sizeof(uint64_t), "handle lists hash as 64-bit words");
static uint64_t hash_handles(const lc_handle* h, uint64_t n) { return hash_words(reinterpret_cast<const uint64_t*>(h), n); }

// Batched calls outside a scan: same idea, cached on the context (call with the context lock held).
static int entries_cached(lc_ctx* ctx, const lc_handle* handles, uint64_t n, Entry* const** out) {
  if (n < 64) {  // short lists (the single-entry calls) are validated in place and never evict a big cached list
    static thread_local std::vector<Entry*> small;
    small.resize(n);
    for (uint64_t i = 0; i < n; ++i) {
      small[i] = entry_of(handles[i]);
      if (!small[i]) {
        set_error("invalid handle at position %llu", (unsigned long long)i);
        return LC_ERR_INVALID;
      }
    }
    *out = small.data();
    return LC_OK;
  }
  const uint64_t key = hash_handles(handles, n);
  auto token = [&](const void* p) {  // the list this call works on, for scan_host.cc's lookup of its device-side twin
    ctx->L()->tok_ptr = p;
    ctx->L()->tok_n = n;
    ctx->L()->tok_gen = g_validated_gen.load(std::memory_order_acquire);
  };
  for (auto& v : ctx->L()->validated) {
    if (v.key == key && v.n == n && v.epoch == ctx->epoch && std::memcmp(v.handles.data(), handles, n * sizeof(lc_handle)) == 0) {
      *out = v.es.data();
      token(*out);
      return LC_OK;
    }
  }
  lc_lane::ValidatedHandles v;
  v.key = key;
  v.n = n;
  v.epoch = ctx->epoch;
  v.handles.assign(handles, handles + n);
  v.es.resize(n);
  for (uint64_t i = 0; i < n; ++i) {
    v.es[i] = entry_of(handles[i]);
    if (!v.es[i]) {
      set_error("invalid handle at position %llu", (unsigned long long)i);
      return LC_ERR_INVALID;
    }
  }
  g_validated_gen.fetch_add(1, std::memory_order_acq_rel);  // a list is born (and maybe one dropped): older tokens are void
  if (ctx->L()->validated.size() >= 8) ctx->L()->validated.erase(ctx->L()->validated.begin());
  ctx->L()->validated.push_back(std::move(v));
  *out = ctx->L()->validated.back().es.data();
  token(*out);
  return LC_OK;
}

static int scan_entries_cached(lc_scan* scan, const lc_handle* handles, Entry* const** out, bool* any_squeezed = nullptr) {
  const uint64_t key = hash_handles(handles, scan->n);
  auto token = [&](const void* p) {
    lc_lane* L = scan->ctx->L();
    L->tok_ptr = p;
    L->tok_n = scan->n;
    L->tok_gen = g_validated_gen.load(std::memory_order_acquire);
  };
  for (auto& v : scan->validated) {
    if (v.key == key && v.epoch == scan->ctx->epoch && std::memcmp(v.handles.data(), handles, scan->n * sizeof(lc_handle)) == 0) {
      *out = v.es.data();
      if (any_squeezed) *any_squeezed = v.any_squeezed;
      token(*out);
      return LC_OK;
    }
  }
  lc_scan::Validated v;
  v.key = key;
  v.epoch = scan->ctx->epoch;
  v.handles.assign(handles, handles + scan->n);
  v.es.resize(scan->n);
  for (uint64_t i = 0; i < scan->n; ++i) {
    v.es[i] = entry_of(handles[i]);
    if (!v.es[i] || v.es[i]->n != scan->rows[i]) {
      set_error("scan: handle %llu invalid or row count differs from the scan's", (unsigned long long)i);
      return LC_ERR_INVALID;
    }
  }
  for (uint64_t i = 0; i < scan->n && !v.any_squeezed; ++i) v.any_squeezed = v.es[i]->squeeze_kind != 0;  // squeezing bumps the epoch
  if (any_squeezed) *any_squeezed = v.any_squeezed;
  g_validated_gen.fetch_add(1, std::memory_order_acq_rel);
  if (scan->validated.size() >= 8) scan->validated.erase(scan->validated.begin());
  scan->validated.push_back(std::move(v));
  *out = scan->validated.back().es.data();
  token(*out);
  return LC_OK;
}

extern "C" {

int lc_encode(lc_ctx* ctx, const struct ArrowSchema* schema, const struct ArrowArray* array, int32_t hint,
              uint64_t compressor_scope, lc_handle* out) {
  if (!ctx || !out) {
    set_error("lc_encode: NULL argument");
    return LC_ERR_INVALID;
  }
  Guard g(ctx);
  Entry* e = nullptr;
  LC_TRY(encode_locked(ctx, schema, array, hint, compressor_scope, &e));
  *out = static_cast<lc_handle>(reinterpret_cast<uintptr_t>(e));
  return LC_OK;
}

void lc_release(lc_ctx* ctx, lc_handle h) {
  if (!ctx) return;
  Guard g(ctx);
  release_entry(ctx, entry_of(h));
}

// The three getters dereference the handle under the context lock, like every other call: a handle being released on
// another thread is either still whole or already refused by entry_of's magic check.
uint64_t lc_len(lc_ctx* ctx, lc_handle h) {
  std::unique_lock<std::mutex> g;
  if (ctx) g = std::unique_lock<std::mutex>(ctx->mu);
  Entry* e = entry_of(h);
  return e ? e->n : 0;
}

uint64_t lc_memory_size(lc_ctx* ctx, lc_handle h) {
  std::unique_lock<std::mutex> g;
  if (ctx) g = std::unique_lock<std::mutex>(ctx->mu);
  Entry* e = entry_of(h);
  return e ? e->blob_bytes : 0;
}

int32_t lc_data_type(lc_ctx* ctx, lc_handle h) {
  std::unique_lock<std::mutex> g;
  if (ctx) g = std::unique_lock<std::mutex>(ctx->mu);
  Entry* e = entry_of(h);
  if (e && e->fixed_width) return LC_LIQUID_FIXED_LEN_BYTE_ARRAY;  // a byte-view blob inside, LiquidFixedLenByteArray outside
  return e ? e->liquid_type : 0;
}

int lc_entry_image(lc_ctx* ctx, lc_handle h, uint8_t* out, uint64_t cap, uint64_t* out_bytes) {
  Entry* e = entry_of(h);
  if (!ctx || !e || !out_bytes) {
    set_error("lc_entry_image: bad argument");
    return LC_ERR_INVALID;
  }
  *out_bytes = e->blob_bytes;
  if (!out) return LC_OK;
  if (cap < e->blob_bytes) {
    set_error("lc_entry_image: buffer of %llu bytes, entry has %u", (unsigned long long)cap, e->blob_bytes);
    return LC_ERR_INVALID;
  }
  Guard g(ctx);
  LC_CUDA_OK(cudaMemcpyAsync(out, e->d_blob, e->blob_bytes, cudaMemcpyDeviceToHost, ctx->L()->stream));
  LC_CUDA_OK(cudaStreamSynchronize(ctx->L()->stream));
  ctx->d2h_bytes += e->blob_bytes;
  return LC_OK;
}

int lc_entry_fsst_table(lc_ctx* ctx, lc_handle h, uint8_t* out, uint64_t cap, uint64_t* out_bytes) {
  Entry* e = entry_of(h);
  if (!ctx || !e || !out_bytes || e->liquid_type != LC_LIQUID_BYTE_VIEW || !e->codec) {
    set_error("lc_entry_fsst_table: not a byte-view entry");
    return LC_ERR_INVALID;
  }
  *out_bytes = sizeof(FsstTable);
  if (!out) return LC_OK;
  if (cap < sizeof(FsstTable)) {
    set_error("lc_entry_fsst_table: buffer too small");
    return LC_ERR_INVALID;
  }
  Guard g(ctx);
  // read it back from the device copy the kernels use, not from the host copy it was uploaded from
  LC_CUDA_OK(cudaMemcpyAsync(out, e->codec->d_dec, sizeof(FsstTable), cudaMemcpyDeviceToHost, ctx->L()->stream));
  LC_CUDA_OK(cudaStreamSynchronize(ctx->L()->stream));
  return LC_OK;
}

int lc_to_bytes(lc_ctx* ctx, lc_handle h, uint8_t* out, uint64_t cap, uint64_t* out_bytes) {
  Entry* e = entry_of(h);
  if (!ctx || !e || !out_bytes) {
    set_error("lc_to_bytes: bad argument");
    return LC_ERR_INVALID;
  }
  if (e->squeeze_kind) {
    set_error("lc_to_bytes: a squeezed entry has no serialized form (its full image is the backing)");
    return LC_ERR_UNSUPPORTED_TYPE;
  }
  if (e->fixed_width) {
    set_error("lc_to_bytes: the LQDA form of LiquidFixedLenByteArray (fix_len_byte_array.rs:116-270) is not built");
    return LC_ERR_UNSUPPORTED_TYPE;
  }
  Guard g(ctx);
  return entry_to_bytes(ctx, e, out, cap, out_bytes);
}

int lc_from_bytes(lc_ctx* ctx, const uint8_t* bytes, uint64_t len, lc_handle* out) {
  if (!ctx || !bytes || !out) {
    set_error("lc_from_bytes: NULL argument");
    return LC_ERR_INVALID;
  }
  Guard g(ctx);
  Entry* e = nullptr;
  LC_TRY(entry_from_bytes(ctx, bytes, len, nullptr, &e));
  *out = static_cast<lc_handle>(reinterpret_cast<uintptr_t>(e));
  return LC_OK;
}

int lc_from_bytes_scoped(lc_ctx* ctx, const uint8_t* bytes, uint64_t len, uint64_t compressor_scope, lc_handle* out) {
  if (!ctx || !bytes || !out) {
    set_error("lc_from_bytes_scoped: NULL argument");
    return LC_ERR_INVALID;
  }
  Guard g(ctx);
  LC_LANE_OK(ctx);
  Entry* e = nullptr;
  LC_TRY(entry_from_bytes(ctx, bytes, len, ctx->codec_of(compressor_scope), &e));
  *out = static_cast<lc_handle>(reinterpret_cast<uintptr_t>(e));
  return LC_OK;
}

int lc_ctx_save_symbol_table(lc_ctx* ctx, uint64_t compressor_scope, uint8_t* out, uint64_t cap, uint64_t* out_bytes) {
  if (!ctx || !out_bytes) return LC_ERR_INVALID;
  Guard g(ctx);
  std::shared_ptr<FsstCodec> codec = ctx->codec_of(compressor_scope);
  if (!codec) {
    set_error("no symbol table for scope %llu", (unsigned long long)compressor_scope);
    return LC_ERR_NOT_FOUND;
  }
  return symbol_table_to_bytes(*codec, out, cap, out_bytes);
}

int lc_ctx_load_symbol_table(lc_ctx* ctx, uint64_t compressor_scope, const uint8_t* bytes, uint64_t len) {
  if (!ctx || !bytes) return LC_ERR_INVALID;
  Guard g(ctx);
  LC_LANE_OK(ctx);
  if (ctx->codec_of(compressor_scope)) {
    set_error("scope %llu already has a symbol table", (unsigned long long)compressor_scope);
    return LC_ERR_INVALID;
  }
  auto codec = std::make_shared<FsstCodec>();
  LC_TRY(symbol_table_from_bytes(bytes, len, codec.get()));
  return register_codec(ctx, compressor_scope, codec);
}

int lc_arrow_format(lc_ctx*, lc_handle h, char* buf, size_t buf_len) {
  Entry* e = entry_of(h);
  if (!e || !buf || buf_len == 0) return LC_ERR_INVALID;
  std::string f = e->orig_format.empty() ? e->arrow_format : e->orig_format;  // a date-component entry reports its column's type
  if (!e->dict_value_format.empty()) f += ":" + e->dict_value_format;  // "S:u" = Dictionary<UInt16, Utf8>
  if (f.size() + 1 > buf_len) return LC_ERR_INVALID;
  std::memcpy(buf, f.c_str(), f.size() + 1);
  return LC_OK;
}

uint64_t lc_mask_bytes(uint64_t n_rows) { return round_up((n_rows + 7) / 8, 16); }

int lc_to_arrow_many(lc_ctx* ctx, const lc_handle* handles, uint64_t n, const uint8_t* const* sel_bits,
                     struct ArrowSchema* out_schema, struct ArrowArray* out_array) {
  if (!ctx || !handles || !out_schema || !out_array || n == 0) {
    set_error("lc_to_arrow_many: bad argument");
    return LC_ERR_INVALID;
  }
  Guard g(ctx);
  Entry* const* es = nullptr;
  LC_TRY(entries_cached(ctx, handles, n, &es));
  return to_arrow_batch(ctx, es, n, sel_bits, nullptr, out_schema, out_array);
}

int lc_to_arrow(lc_ctx* ctx, lc_handle h, const uint8_t* sel_bits, uint64_t sel_len, struct ArrowSchema* out_schema,
                struct ArrowArray* out_array) {
  Entry* e = entry_of(h);
  if (!e) {
    set_error("invalid handle");
    return LC_ERR_INVALID;
  }
  if (sel_bits && sel_len != e->n) {
    set_error("selection has %llu bits, entry has %u rows", (unsigned long long)sel_len, e->n);
    return LC_ERR_INVALID;
  }
  if (e->squeeze_kind) {
    if (!ctx || !out_schema || !out_array) {
      set_error("lc_to_arrow: bad argument");
      return LC_ERR_INVALID;
    }
    Guard g(ctx);
    return squeezed_to_arrow(ctx, e, sel_bits, out_schema, out_array);
  }
  const uint8_t* sels[1] = {sel_bits};
  return lc_to_arrow_many(ctx, &h, 1, sel_bits ? sels : nullptr, out_schema, out_array);
}

int lc_squeeze(lc_ctx* ctx, lc_handle h, int32_t policy, int32_t hint, lc_backing_read read, void* user, uint8_t* bytes_out,
               uint64_t cap, uint64_t* out_bytes, lc_handle* out_squeezed) {
  Entry* e = entry_of(h);
  if (!ctx || !e || !out_bytes || !out_squeezed) {
    set_error("lc_squeeze: bad argument");
    return LC_ERR_INVALID;
  }
  Guard g(ctx);
  Entry* sq = nullptr;
  *out_squeezed = 0;
  LC_TRY(squeeze_entry(ctx, e, policy, hint, read, user, bytes_out, cap, out_bytes, &sq));
  *out_squeezed = static_cast<lc_handle>(reinterpret_cast<uintptr_t>(sq));
  return LC_OK;
}

int lc_squeezed_component(lc_ctx* ctx, lc_handle h, int32_t lossy, struct ArrowSchema* out_schema, struct ArrowArray* out_array) {
  Entry* e = entry_of(h);
  if (!ctx || !e || !out_schema || !out_array) {
    set_error("lc_squeezed_component: bad argument");
    return LC_ERR_INVALID;
  }
  Guard g(ctx);
  return squeezed_component_array(ctx, e, lossy, out_schema, out_array);
}

int lc_squeezed_info(lc_ctx* ctx, lc_handle h, uint64_t out[6]) {
  Entry* e = entry_of(h);
  if (!ctx || !e || !out) {
    set_error("lc_squeezed_info: bad argument");
    return LC_ERR_INVALID;
  }
  Guard g(ctx);
  out[0] = static_cast<uint64_t>(e->squeeze_kind);
  out[1] = e->liquid_type == LC_LIQUID_INTEGER ? e->ih.bit_width : 0;
  out[2] = e->squeeze_kind == 3 ? e->date_field : e->bucket_width;
  out[3] = e->backing_len;
  out[4] = ctx->squeeze_reads;
  out[5] = ctx->squeeze_saved;
  return LC_OK;
}

// IN lists are planned on full entries only: a squeezed entry's codes would need a probe per list value.
static int refuse_in_list_on_squeezed(const lc_predicate* pred) {
  if (pred->op != LC_OP_IN && pred->op != LC_OP_NOT_IN) return LC_OK;
  set_error("IN lists do not run on squeezed entries");
  return LC_ERR_UNSUPPORTED_EXPR;
}

int lc_eval_predicate_many(lc_ctx* ctx, const lc_handle* handles, uint64_t n, const lc_predicate* pred,
                           const uint8_t* const* sel_bits, uint8_t* out_values, uint8_t* out_validity,
                           const uint64_t* out_byte_offsets, uint64_t* out_len, uint64_t* out_null_count,
                           uint64_t* out_true_count) {
  if (!ctx || !handles || !pred || !out_values) {
    set_error("lc_eval_predicate_many: NULL argument");
    return LC_ERR_INVALID;
  }
  if (n > 1 && !out_byte_offsets) {
    set_error("lc_eval_predicate_many: out_byte_offsets required for n > 1");
    return LC_ERR_INVALID;
  }
  Guard g(ctx);
  Entry* const* es = nullptr;
  LC_TRY(entries_cached(ctx, handles, n, &es));
  PredOut po{out_values, out_validity, out_byte_offsets, out_len, out_null_count, out_true_count};
  bool any_squeezed = false;
  for (uint64_t i = 0; i < n && !any_squeezed; ++i) any_squeezed = es[i]->squeeze_kind != 0;
  if (any_squeezed) LC_TRY(refuse_in_list_on_squeezed(pred));
  if (any_squeezed) return squeezed_eval_predicate_many(ctx, es, n, pred, sel_bits, po);  // probes + backing reads where needed
  return eval_predicate_batch(ctx, es, n, pred, sel_bits, po);
}

int lc_eval_predicate(lc_ctx* ctx, lc_handle h, const lc_predicate* pred, const uint8_t* sel_bits, uint64_t sel_len,
                      uint8_t* out_values, uint8_t* out_validity, uint64_t* out_len, uint64_t* out_null_count) {
  Entry* e = entry_of(h);
  if (!e) {
    set_error("invalid handle");
    return LC_ERR_INVALID;
  }
  if (sel_bits && sel_len != e->n) {
    set_error("selection has %llu bits, entry has %u rows", (unsigned long long)sel_len, e->n);
    return LC_ERR_INVALID;
  }
  const uint8_t* sels[1] = {sel_bits};
  const uint64_t off0 = 0;
  if (e->squeeze_kind) {
    if (!ctx || !pred || !out_values) {
      set_error("lc_eval_predicate: NULL argument");
      return LC_ERR_INVALID;
    }
    LC_TRY(refuse_in_list_on_squeezed(pred));
    Guard g(ctx);
    PredOut po{out_values, out_validity, &off0, out_len, out_null_count, nullptr};
    return squeezed_eval_predicate(ctx, e, pred, sel_bits, po);
  }
  return lc_eval_predicate_many(ctx, &h, 1, pred, sel_bits ? sels : nullptr, out_values, out_validity, &off0, out_len,
                                out_null_count, nullptr);
}

int lc_and_then(lc_ctx* ctx, const uint8_t* left_bits, uint64_t left_len, const uint8_t* right_bits, uint64_t right_len,
                uint8_t* out_bits) {
  if (!ctx || !left_bits || !out_bits || (!right_bits && right_len)) {
    set_error("lc_and_then: NULL argument");
    return LC_ERR_INVALID;
  }
  if (left_len > 0xffffffffull) {
    set_error("lc_and_then: selection too long");
    return LC_ERR_INVALID;
  }
  const uint64_t ones = popcount_bits(left_bits, left_len);
  if (ones != right_len) {
    // debug_assert_eq!(left.count_set_bits(), right.len())  (datafusion/src/utils.rs:63-67)
    set_error("lc_and_then: right has %llu bits but left has %llu set bits", (unsigned long long)right_len,
              (unsigned long long)ones);
    return LC_ERR_INVALID;
  }
  if (left_len == right_len) {  // utils.rs:69-72
    std::memcpy(out_bits, right_bits, (right_len + 7) / 8);
    return LC_OK;
  }
  Guard g(ctx);
  const uint64_t lw = round_up((left_len + 31) / 32, 4) * 4, rw = round_up((right_len + 31) / 32, 4) * 4 + 16;
  Scratch& sc = ctx->L()->scratch;
  LC_TRY(sc.reserve(2 * lw + rw + 1024, 2 * lw + rw + 1024));
  uint8_t* h_l = sc.host(lw);
  uint8_t* h_r = sc.host(rw);
  uint8_t* h_o = sc.host(lw);
  uint8_t* d_l = sc.dev(lw);
  uint8_t* d_r = sc.dev(rw);
  uint8_t* d_o = sc.dev(lw);
  if (!h_l || !h_r || !h_o || !d_l || !d_r || !d_o) return LC_ERR_OOM;
  copy_bits(left_bits, 0, static_cast<int64_t>(left_len), h_l, lw);
  copy_bits(right_bits, 0, static_cast<int64_t>(right_len), h_r, rw);
  cudaStream_t s = ctx->L()->stream;
  LC_CUDA_OK(cudaMemcpyAsync(d_l, h_l, lw, cudaMemcpyHostToDevice, s));
  LC_CUDA_OK(cudaMemcpyAsync(d_r, h_r, rw, cudaMemcpyHostToDevice, s));
  LC_CUDA_OK(launch_and_then(reinterpret_cast<const uint32_t*>(d_l), static_cast<uint32_t>(left_len),
                             reinterpret_cast<const uint32_t*>(d_r), reinterpret_cast<uint32_t*>(d_o), s));
  LC_CUDA_OK(cudaMemcpyAsync(h_o, d_o, lw, cudaMemcpyDeviceToHost, s));
  LC_CUDA_OK(cudaStreamSynchronize(s));
  ctx->kernel_launches++;
  ctx->h2d_bytes += lw + rw;
  ctx->d2h_bytes += lw;
  std::memcpy(out_bits, h_o, (left_len + 7) / 8);
  return LC_OK;
}

/* ---------------------------------------------------- LiquidCache-level calls ---- */

int lc_cache_insert(lc_ctx* ctx, uint64_t entry_id, const struct ArrowSchema* schema, const struct ArrowArray* array,
                    int32_t hint) {
  if (!ctx) return LC_ERR_INVALID;
  Guard g(ctx);
  Entry* e = nullptr;
  // FSST table scope = (file, row group, column): entry id with the batch bits cleared (cache/id.rs:15-22)
  const uint64_t scope = entry_id & ~0xFFFFull;
  LC_TRY(encode_locked(ctx, schema, array, hint, scope, &e));
  return publish_entries(ctx, &entry_id, &e, 1);
}

int lc_cache_insert_many(lc_ctx* ctx, const uint64_t* entry_ids, uint64_t n, const struct ArrowSchema* const* schemas,
                         const struct ArrowArray* const* arrays, int32_t hint) {
  if (!ctx || (n && (!entry_ids || !schemas || !arrays))) {
    set_error("lc_cache_insert_many: NULL argument");
    return LC_ERR_INVALID;
  }
  if (n == 0) return LC_OK;
  Guard g(ctx);
  std::vector<ArrowIn> ins(n);
  bool all_int = true;
  for (uint64_t i = 0; i < n; ++i) {
    LC_TRY(parse_arrow_input(schemas[i], arrays[i], &ins[i]));
    all_int = all_int && ins[i].kind == ArrowIn::K_INT;
  }
  bool all_bytes = true;
  for (uint64_t i = 0; i < n; ++i)
    all_bytes = all_bytes && (ins[i].kind == ArrowIn::K_BYTES || ins[i].kind == ArrowIn::K_VIEW || ins[i].kind == ArrowIn::K_DICT);
  std::vector<Entry*> es;
  if (all_int) {
    // integer-like batches: one pass over the whole list (int_host.cc int_encode_many)
    LC_TRY(int_encode_many(ctx, ins, &es));
  } else if (all_bytes) {
    // byte-view batches: the five encode stages once over the whole list (str_host.cc str_encode_many)
    std::vector<uint64_t> scopes(n);
    for (uint64_t i = 0; i < n; ++i) scopes[i] = entry_ids[i] & ~0xFFFFull;
    LC_TRY(str_encode_many(ctx, ins, hint, scopes.data(), &es));
  } else {
    // floats, decimals, mixed lists: batch by batch; all or nothing like the batched passes
    for (uint64_t i = 0; i < n; ++i) {
      Entry* e = nullptr;
      ctx->L()->scratch.reset();
      const int rc = encode_locked(ctx, schemas[i], arrays[i], hint, entry_ids[i] & ~0xFFFFull, &e);
      if (rc != LC_OK) {
        for (Entry* made : es) release_entry(ctx, made);
        return rc;
      }
      es.push_back(e);
    }
  }
  return publish_entries(ctx, entry_ids, es.data(), n);
}

int lc_cache_is_cached(lc_ctx* ctx, uint64_t entry_id) {
  if (!ctx) return 0;
  std::lock_guard<std::mutex> g(ctx->mu);
  return ctx->cache.count(entry_id) ? 1 : 0;
}

int lc_cache_remove(lc_ctx* ctx, uint64_t entry_id) {
  if (!ctx) return LC_ERR_INVALID;
  Guard g(ctx);
  Entry* e = nullptr;
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    auto it = ctx->cache.find(entry_id);
    if (it == ctx->cache.end()) return LC_ERR_NOT_FOUND;
    e = entry_of(it->second);
    ctx->cache.erase(it);
  }
  release_entry(ctx, e);
  return LC_OK;
}

int lc_cache_reset(lc_ctx* ctx) {
  if (!ctx) return LC_ERR_INVALID;
  Guard g(ctx);
  LC_LANE_OK(ctx);
  cudaStreamSynchronize(ctx->L()->stream);
  std::vector<Entry*> held;
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    for (auto& kv : ctx->cache) held.push_back(entry_of(kv.second));
    ctx->cache.clear();
  }
  for (Entry* e : held) release_entry(ctx, e);
  return LC_OK;
}

int lc_cache_handles(lc_ctx* ctx, const uint64_t* entry_ids, uint64_t n, lc_handle* out) {
  if (!ctx || !entry_ids || !out) return LC_ERR_INVALID;
  std::lock_guard<std::mutex> g(ctx->mu);
  for (uint64_t i = 0; i < n; ++i) {
    auto it = ctx->cache.find(entry_ids[i]);
    if (it == ctx->cache.end()) {
      set_error("entry %llu not cached", (unsigned long long)entry_ids[i]);
      return LC_ERR_NOT_FOUND;
    }
    out[i] = it->second;
  }
  return LC_OK;
}

int lc_cache_retain(lc_ctx* ctx, uint64_t entry_id, lc_handle* out) {
  if (!ctx || !out) return LC_ERR_INVALID;
  std::lock_guard<std::mutex> g(ctx->mu);
  auto it = ctx->cache.find(entry_id);
  if (it == ctx->cache.end()) {
    set_error("entry %llu not cached", (unsigned long long)entry_id);
    return LC_ERR_NOT_FOUND;
  }
  Entry* e = entry_of(it->second);
  if (!e) return LC_ERR_INVALID;
  e->refcount++;
  *out = it->second;
  return LC_OK;
}

int lc_cache_get(lc_ctx* ctx, uint64_t entry_id, const uint8_t* sel_bits, uint64_t sel_len,
                 struct ArrowSchema* out_schema, struct ArrowArray* out_array) {
  lc_handle h;
  LC_TRY(lc_cache_retain(ctx, entry_id, &h));  // the entry cannot go away under the call (another thread may replace the id)
  const int rc = lc_to_arrow(ctx, h, sel_bits, sel_len, out_schema, out_array);
  lc_release(ctx, h);
  return rc;
}

int lc_cache_eval_predicate(lc_ctx* ctx, uint64_t entry_id, const lc_predicate* pred, const uint8_t* sel_bits,
                            uint64_t sel_len, uint8_t* out_values, uint8_t* out_validity, uint64_t* out_len,
                            uint64_t* out_null_count) {
  lc_handle h;
  LC_TRY(lc_cache_retain(ctx, entry_id, &h));
  const int rc = lc_eval_predicate(ctx, h, pred, sel_bits, sel_len, out_values, out_validity, out_len, out_null_count);
  lc_release(ctx, h);
  return rc;
}

/* --------------------------------------------- device-resident scan pipeline ---- */

int lc_scan_begin(lc_ctx* ctx, uint64_t n_batches, const uint64_t* rows_per_batch, lc_scan** out) {
  if (!ctx || !rows_per_batch || !out || n_batches == 0) {
    set_error("lc_scan_begin: bad argument");
    return LC_ERR_INVALID;
  }
  Guard g(ctx);
  lc_scan* sc = new lc_scan();
  sc->ctx = ctx;
  sc->n = n_batches;
  sc->rows.resize(n_batches);
  sc->word_off.resize(n_batches);
  uint64_t w = 0;
  for (uint64_t i = 0; i < n_batches; ++i) {
    if (rows_per_batch[i] > 0x7fffffffull) {
      delete sc;
      set_error("batch too large");
      return LC_ERR_INVALID;
    }
    sc->rows[i] = static_cast<uint32_t>(rows_per_batch[i]);
    sc->word_off[i] = w;
    w += round_up((rows_per_batch[i] + 31) / 32, 4);
  }
  sc->total_words = w;
  if (cudaMalloc(reinterpret_cast<void**>(&sc->d_sel), (w + 4) * 4) != cudaSuccess ||
      cudaMalloc(reinterpret_cast<void**>(&sc->d_counts), n_batches * 8 + 16) != cudaSuccess ||
      cudaMalloc(reinterpret_cast<void**>(&sc->d_word_off), n_batches * 8 + 16) != cudaSuccess) {
    cudaGetLastError();
    if (sc->d_sel) cudaFree(sc->d_sel);
    if (sc->d_counts) cudaFree(sc->d_counts);
    delete sc;
    set_error("lc_scan_begin: cudaMalloc failed");
    return LC_ERR_OOM;
  }
  if (cudaMemcpyAsync(sc->d_word_off, sc->word_off.data(), n_batches * 8, cudaMemcpyHostToDevice, ctx->L()->stream) != cudaSuccess ||
      cudaStreamSynchronize(ctx->L()->stream) != cudaSuccess) {
    set_error("lc_scan_begin: upload failed: %s", cudaGetErrorString(cudaGetLastError()));
    cudaFree(sc->d_sel);
    cudaFree(sc->d_counts);
    cudaFree(sc->d_word_off);
    delete sc;
    return LC_ERR_CUDA;
  }
  *out = sc;
  return LC_OK;
}

int lc_scan_reset(lc_scan* scan) {
  if (!scan) return LC_ERR_INVALID;
  ScanGuard g(scan);
  scan->all_rows = true;
  scan->counts_on_device = false;
  scan->counts_cached = false;
  return LC_OK;
}

int lc_scan_set_selection(lc_scan* scan, uint64_t batch, const uint8_t* sel_bits, uint64_t sel_len) {
  if (!scan || batch >= scan->n || !sel_bits || sel_len != scan->rows[batch]) {
    set_error("lc_scan_set_selection: bad argument");
    return LC_ERR_INVALID;
  }
  lc_ctx* ctx = scan->ctx;
  ScanGuard g(scan);
  cudaStream_t s = ctx->L()->stream;
  if (scan->all_rows) {
    LC_CUDA_OK(cudaMemsetAsync(scan->d_sel, 0xFF, scan->total_words * 4, s));
    scan->all_rows = false;
  }
  const uint64_t words = round_up((sel_len + 31) / 32, 4);
  LC_TRY(ctx->L()->scratch.reserve(0, words * 4 + 256));
  uint8_t* hb = ctx->L()->scratch.host(words * 4);
  if (!hb) return LC_ERR_OOM;
  copy_bits(sel_bits, 0, static_cast<int64_t>(sel_len), hb, words * 4);
  LC_CUDA_OK(cudaMemcpyAsync(scan->d_sel + scan->word_off[batch], hb, words * 4, cudaMemcpyHostToDevice, s));
  LC_CUDA_OK(cudaStreamSynchronize(s));
  ctx->h2d_bytes += words * 4;
  scan->counts_on_device = false;
  scan->counts_cached = false;
  return LC_OK;
}

// lc_scan_filter over a list with squeezed (clamp / quantize) entries: selection &= valid & cmp stays one pass over the
// whole list — the kernel's planner compares codes the way each header asks for — around two cheap extras:
//   before  a probe pass per squeeze form in doubt, on a COPY of the selection, tells which entries have a selected row the
//           codes cannot decide (hybrid_primitive_array.rs: Err(NeedsBacking));
//   after   only those entries get their selection words back, read their LQDA image through the caller's function,
//           and are refined again as full entries.
// `d_target` is the selection refined in place (all_rows: it starts as every row and is written, not read), `d_counts`
// the stride-2 survivor counts: the running selection and its counts for lc_scan_filter, a work buffer for
// lc_scan_filter_or's terms.
static int scan_filter_squeezed(lc_scan* scan, Entry* const* es, const lc_predicate* pred, uint32_t* d_target, bool all_rows,
                                uint32_t* d_counts) {
  lc_ctx* ctx = scan->ctx;
  const uint64_t n = scan->n;
  struct Internal {  // the batch functions refuse squeezed entries unless squeeze code drives them
    lc_ctx* c;
    bool prev;
    explicit Internal(lc_ctx* x) : c(x), prev(x->L()->squeeze_internal) { x->L()->squeeze_internal = true; }
    ~Internal() { c->L()->squeeze_internal = prev; }
  } internal(ctx);
  if (pred->op < LC_OP_EQ || pred->op > LC_OP_GE) {
    set_error("operator %d is not supported on integer columns", pred->op);
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  std::vector<uint8_t> doubt(n, 0);
  lc_predicate probes[3] = {};
  uint64_t n_doubt[4] = {0, 0, 0, 0};
  for (uint64_t i = 0; i < n; ++i) {
    if (es[i]->squeeze_kind == 3) {
      set_error("lc_scan_filter: entry %llu is a date-component entry; those answer through lc_eval_predicate", (unsigned long long)i);
      return LC_ERR_INVALID;
    }
    lc_predicate probe{};
    const int d = squeeze_doubt(es[i], pred, &probe);
    doubt[i] = static_cast<uint8_t>(d);
    n_doubt[d]++;
    if (d == 1 || d == 2) probes[d] = probe;
  }
  std::vector<uint8_t> backing(n, 0);
  for (uint64_t i = 0; i < n; ++i) backing[i] = doubt[i] == 3;
  const bool any_doubt = n_doubt[1] || n_doubt[2] || n_doubt[3];
  cudaStream_t s = ctx->L()->stream;
  // work areas kept with the scan: a copy of the selection for the probes, one to restore from, probe counts
  const uint64_t sel_bytes = scan->total_words * 4 + 64;
  if (any_doubt && !scan->d_probe) {
    if (cudaMalloc(reinterpret_cast<void**>(&scan->d_probe), sel_bytes) != cudaSuccess ||
        cudaMalloc(reinterpret_cast<void**>(&scan->d_save), sel_bytes) != cudaSuccess ||
        cudaMalloc(reinterpret_cast<void**>(&scan->d_pcounts), n * 8 + 16) != cudaSuccess) {
      cudaGetLastError();
      set_error("lc_scan_filter: cudaMalloc for the probe selection failed");
      return LC_ERR_OOM;  // lc_scan_end frees whatever was allocated
    }
  }
  uint32_t* d_probe = scan->d_probe;
  uint32_t* d_save = scan->d_save;
  uint32_t* d_pcounts = scan->d_pcounts;
  if (any_doubt && !all_rows)
    LC_CUDA_OK(cudaMemcpyAsync(d_save, d_target, scan->total_words * 4, cudaMemcpyDeviceToDevice, s));
  std::vector<uint32_t> pc(n * 2);
  for (int form = 1; form <= 2; ++form) {
    if (!n_doubt[form]) continue;
    if (!all_rows) LC_CUDA_OK(cudaMemcpyAsync(d_probe, d_target, scan->total_words * 4, cudaMemcpyDeviceToDevice, s));
    ctx->L()->scratch.reset();
    LC_TRY(refine_batch(ctx, es, n, &probes[form], d_probe, scan->d_word_off, all_rows, d_pcounts));
    LC_CUDA_OK(cudaMemcpyAsync(pc.data(), d_pcounts, n * 8, cudaMemcpyDeviceToHost, s));
    LC_CUDA_OK(cudaStreamSynchronize(s));
    ctx->d2h_bytes += n * 8;
    for (uint64_t i = 0; i < n; ++i)
      if (doubt[i] == form && pc[2 * i]) backing[i] = 1;
  }
  // ---- the predicate over the whole list ----
  ctx->L()->scratch.reset();
  LC_TRY(refine_batch(ctx, es, n, pred, d_target, scan->d_word_off, all_rows, d_counts));
  // ---- entries the codes could not decide ----
  for (uint64_t i = 0; i < n; ++i) {
    if (es[i]->squeeze_kind && !backing[i]) ctx->squeeze_saved++;
    if (!backing[i]) continue;
    const uint64_t words = (static_cast<uint64_t>(scan->rows[i]) + 31) / 32;
    if (!all_rows)
      LC_CUDA_OK(cudaMemcpyAsync(d_target + scan->word_off[i], d_save + scan->word_off[i], words * 4, cudaMemcpyDeviceToDevice, s));
    Entry* full = nullptr;
    LC_TRY(squeeze_hydrate(ctx, es[i], &full));
    Entry* one[1] = {full};
    ctx->L()->scratch.reset();
    const int rc = refine_batch(ctx, one, 1, pred, d_target, scan->d_word_off + i, all_rows, d_counts + 2 * i);
    release_entry(ctx, full);
    LC_TRY(rc);
  }
  return LC_OK;
}

int lc_scan_filter(lc_scan* scan, const lc_handle* handles, const lc_predicate* pred) {
  if (!scan || !handles || !pred) {
    set_error("lc_scan_filter: NULL argument");
    return LC_ERR_INVALID;
  }
  lc_ctx* ctx = scan->ctx;
  ScanGuard g(scan);
  Entry* const* es = nullptr;
  bool any_squeezed = false;
  LC_TRY(scan_entries_cached(scan, handles, &es, &any_squeezed));
  if (any_squeezed) LC_TRY(refuse_in_list_on_squeezed(pred));
  if (any_squeezed) LC_TRY(scan_filter_squeezed(scan, es, pred, scan->d_sel, scan->all_rows, scan->d_counts));
  else LC_TRY(refine_batch(ctx, es, scan->n, pred, scan->d_sel, scan->d_word_off, scan->all_rows, scan->d_counts));
  scan->all_rows = false;
  scan->counts_on_device = true;
  scan->counts_cached = false;
  return LC_OK;
}

// selection := selection & OR_d AND_{t in d} (valid_t & pred_t). Every term is refined exactly as lc_scan_filter would
// refine it, but into the term buffer T, which starts each disjunct as the part of the selection no earlier disjunct has
// accepted (S & ~A); k_sel_or then folds T into the accumulator A, or, after the last disjunct, writes S and its counts.
// S is written by that last launch only, so a term refused anywhere in the list leaves the selection and counts as they were.
int lc_scan_filter_or(lc_scan* scan, uint64_t n_terms, const lc_handle* const* handles, const lc_predicate* preds,
                      const uint32_t* group) {
  if (!scan || !handles || !preds || n_terms == 0) {
    set_error("lc_scan_filter_or: NULL argument or no terms");
    return LC_ERR_INVALID;
  }
  for (uint64_t t = 0; t < n_terms; ++t) {
    if (!handles[t]) {
      set_error("lc_scan_filter_or: term %llu has no handle list", (unsigned long long)t);
      return LC_ERR_INVALID;
    }
    if (group && (t == 0 ? group[0] != 0u : (group[t] != group[t - 1] && group[t] != group[t - 1] + 1u))) {
      set_error("lc_scan_filter_or: group must start at 0 and step by 0 or 1 (term %llu)", (unsigned long long)t);
      return LC_ERR_INVALID;
    }
  }
  lc_ctx* ctx = scan->ctx;
  ScanGuard g(scan);
  // every handle list is checked against the scan before anything runs
  for (uint64_t t = 0; t < n_terms; ++t) {
    Entry* const* es = nullptr;
    LC_TRY(scan_entries_cached(scan, handles[t], &es));
  }
  cudaStream_t s = ctx->L()->stream;
  const uint64_t n = scan->n;
  const uint64_t sel_bytes = scan->total_words * 4 + 64;
  if (!scan->d_rows) {  // set last, once everything else is in place (a failed first call leaves the rest for the next)
    auto alloc = [](uint32_t** p, uint64_t bytes) { return *p || cudaMalloc(reinterpret_cast<void**>(p), bytes) == cudaSuccess; };
    uint32_t* d_rows = nullptr;
    if (!alloc(&scan->d_term, sel_bytes) || !alloc(&scan->d_acc, sel_bytes) || !alloc(&scan->d_tcounts, n * 8 + 16) ||
        !alloc(&d_rows, n * 4 + 16)) {
      cudaGetLastError();
      set_error("lc_scan_filter_or: cudaMalloc for the work selections failed");
      return LC_ERR_OOM;  // lc_scan_end frees whatever was allocated
    }
    // pageable source that lives as long as the scan
    if (cudaMemcpyAsync(d_rows, scan->rows.data(), n * 4, cudaMemcpyHostToDevice, s) != cudaSuccess) {
      set_error("lc_scan_filter_or: upload of the row counts failed: %s", cudaGetErrorString(cudaGetLastError()));
      cudaFree(d_rows);
      return LC_ERR_CUDA;
    }
    scan->d_rows = d_rows;
    ctx->h2d_bytes += n * 4;
  }
  const uint32_t n_groups = (group ? group[n_terms - 1] : static_cast<uint32_t>(n_terms - 1)) + 1u;
  uint64_t t = 0;
  for (uint32_t d = 0; d < n_groups; ++d) {
    // T := S & ~A was left by the previous merge; the first disjunct starts from S itself
    bool t_all = false;
    if (d == 0) {
      if (scan->all_rows) t_all = true;
      else LC_CUDA_OK(cudaMemcpyAsync(scan->d_term, scan->d_sel, scan->total_words * 4, cudaMemcpyDeviceToDevice, s));
    }
    for (; t < n_terms && (group ? group[t] : t) == d; ++t) {
      Entry* const* es = nullptr;
      bool any_squeezed = false;
      LC_TRY(scan_entries_cached(scan, handles[t], &es, &any_squeezed));
      ctx->L()->scratch.reset();  // float terms decode into the lane scratch
      if (any_squeezed) {
        LC_TRY(refuse_in_list_on_squeezed(&preds[t]));
        LC_TRY(scan_filter_squeezed(scan, es, &preds[t], scan->d_term, t_all, scan->d_tcounts));
      } else {
        LC_TRY(refine_batch(ctx, es, n, &preds[t], scan->d_term, scan->d_word_off, t_all, scan->d_tcounts));
      }
      t_all = false;
    }
    LC_CUDA_OK(launch_sel_or(scan->d_sel, scan->all_rows, scan->d_term, scan->d_acc, scan->d_word_off, scan->d_rows,
                             static_cast<uint32_t>(n), d == 0, d + 1 == n_groups, scan->d_counts, s));
    ctx->kernel_launches++;
  }
  scan->all_rows = false;
  scan->counts_on_device = true;
  scan->counts_cached = false;
  return LC_OK;
}

int lc_scan_selection_layout(lc_scan* scan, uint64_t* word_offsets, uint64_t* total_words) {
  if (!scan) return LC_ERR_INVALID;
  if (word_offsets)
    for (uint64_t i = 0; i < scan->n; ++i) word_offsets[i] = scan->word_off[i];
  if (total_words) *total_words = scan->total_words;
  return LC_OK;
}

int lc_scan_store_selections(lc_scan* scan, uint32_t* out_words, uint64_t n_words) {
  if (!scan || !out_words || n_words < scan->total_words) {
    set_error("lc_scan_store_selections: need room for %llu words", (unsigned long long)(scan ? scan->total_words : 0));
    return LC_ERR_INVALID;
  }
  lc_ctx* ctx = scan->ctx;
  ScanGuard g(scan);
  if (scan->all_rows) {
    for (uint64_t i = 0; i < scan->n; ++i) {
      const uint64_t words = (scan->rows[i] + 31) / 32, padded = round_up(words, 4);
      uint32_t* w = out_words + scan->word_off[i];
      for (uint64_t k = 0; k < padded; ++k) w[k] = k < words ? 0xffffffffu : 0u;
      if (scan->rows[i] & 31) w[words - 1] = (1u << (scan->rows[i] & 31)) - 1u;
    }
    return LC_OK;
  }
  LC_CUDA_OK(cudaMemcpyAsync(out_words, scan->d_sel, scan->total_words * 4, cudaMemcpyDeviceToHost, ctx->L()->stream));
  LC_CUDA_OK(cudaStreamSynchronize(ctx->L()->stream));
  ctx->d2h_bytes += scan->total_words * 4;
  for (uint64_t i = 0; i < scan->n; ++i)  // rows past the batch's length carry no meaning
    if (scan->rows[i] & 31) out_words[scan->word_off[i] + (scan->rows[i] + 31) / 32 - 1] &= (1u << (scan->rows[i] & 31)) - 1u;
  return LC_OK;
}

int lc_scan_load_selections(lc_scan* scan, const uint32_t* words, uint64_t n_words) {
  if (!scan || !words || n_words < scan->total_words) {
    set_error("lc_scan_load_selections: need %llu words", (unsigned long long)(scan ? scan->total_words : 0));
    return LC_ERR_INVALID;
  }
  lc_ctx* ctx = scan->ctx;
  ScanGuard g(scan);
  LC_CUDA_OK(cudaMemcpyAsync(scan->d_sel, words, scan->total_words * 4, cudaMemcpyHostToDevice, ctx->L()->stream));
  LC_CUDA_OK(cudaStreamSynchronize(ctx->L()->stream));  // `words` is the caller's memory
  ctx->h2d_bytes += scan->total_words * 4;
  scan->all_rows = false;
  scan->counts_on_device = false;
  scan->counts_cached = false;
  return LC_OK;
}

static int scan_fetch_counts(lc_scan* scan) {
  if (scan->counts_cached) return LC_OK;
  lc_ctx* ctx = scan->ctx;
  scan->counts.assign(scan->n, 0);
  if (scan->all_rows) {
    for (uint64_t i = 0; i < scan->n; ++i) scan->counts[i] = scan->rows[i];
  } else if (scan->counts_on_device) {
    std::vector<uint32_t> tmp(scan->n * 2);
    LC_CUDA_OK(cudaMemcpyAsync(tmp.data(), scan->d_counts, scan->n * 8, cudaMemcpyDeviceToHost, ctx->L()->stream));
    LC_CUDA_OK(cudaStreamSynchronize(ctx->L()->stream));
    ctx->d2h_bytes += scan->n * 8;
    for (uint64_t i = 0; i < scan->n; ++i) scan->counts[i] = tmp[2 * i];
  } else {
    // selections were seeded from the host and not filtered yet: count them from a copy
    std::vector<uint32_t> words(scan->total_words);
    LC_CUDA_OK(cudaMemcpyAsync(words.data(), scan->d_sel, scan->total_words * 4, cudaMemcpyDeviceToHost, ctx->L()->stream));
    LC_CUDA_OK(cudaStreamSynchronize(ctx->L()->stream));
    ctx->d2h_bytes += scan->total_words * 4;
    for (uint64_t i = 0; i < scan->n; ++i)
      scan->counts[i] = static_cast<uint32_t>(
          popcount_bits(reinterpret_cast<const uint8_t*>(words.data() + scan->word_off[i]), scan->rows[i]));
  }
  scan->counts_cached = true;
  return LC_OK;
}

int lc_scan_counts(lc_scan* scan, uint64_t* out_counts, uint64_t* out_total) {
  if (!scan) return LC_ERR_INVALID;
  ScanGuard g(scan);
  LC_TRY(scan_fetch_counts(scan));
  uint64_t tot = 0;
  for (uint64_t i = 0; i < scan->n; ++i) {
    if (out_counts) out_counts[i] = scan->counts[i];
    tot += scan->counts[i];
  }
  if (out_total) *out_total = tot;
  return LC_OK;
}

int lc_scan_selection(lc_scan* scan, uint64_t batch, uint8_t* out_bits) {
  if (!scan || batch >= scan->n || !out_bits) return LC_ERR_INVALID;
  lc_ctx* ctx = scan->ctx;
  ScanGuard g(scan);
  const uint32_t rows = scan->rows[batch];
  const uint64_t nbytes = (rows + 7) / 8;
  if (scan->all_rows) {
    std::memset(out_bits, 0xFF, nbytes);
  } else {
    const uint64_t words = (rows + 31) / 32;
    std::vector<uint32_t> tmp(words + 1);
    LC_CUDA_OK(cudaMemcpyAsync(tmp.data(), scan->d_sel + scan->word_off[batch], words * 4, cudaMemcpyDeviceToHost,
                               ctx->L()->stream));
    LC_CUDA_OK(cudaStreamSynchronize(ctx->L()->stream));
    ctx->d2h_bytes += words * 4;
    std::memcpy(out_bits, tmp.data(), nbytes);
  }
  if (rows & 7) out_bits[nbytes - 1] &= static_cast<uint8_t>((1u << (rows & 7)) - 1u);
  return LC_OK;
}

// Only batches with surviving rows are read, as LiquidCacheReader::read_from_cache does
// (liquid_cache_reader.rs:346-349 returns early when the selection is empty).
static void scan_nonempty(lc_scan* scan, const std::vector<Entry*>& es, std::vector<Entry*>* es2,
                          std::vector<uint64_t>* woff2, std::vector<uint32_t>* k2) {
  for (uint64_t i = 0; i < scan->n; ++i) {
    if (scan->counts[i] == 0) continue;
    es2->push_back(es[i]);
    woff2->push_back(scan->word_off[i]);
    k2->push_back(scan->counts[i]);
  }
  if (es2->empty()) {  // keep one batch so the (empty) result still carries the column's type
    es2->push_back(es[0]);
    woff2->push_back(scan->word_off[0]);
    k2->push_back(scan->counts[0]);
  }
}

int lc_scan_read(lc_scan* scan, const lc_handle* handles, struct ArrowSchema* out_schema,
                 struct ArrowArray* out_array) {
  if (!scan || !handles || !out_schema || !out_array) return LC_ERR_INVALID;
  lc_ctx* ctx = scan->ctx;
  ScanGuard g(scan);
  // the handle list of a column is validated once per scan (hash of the array), not once per read: 12 k pointer chases
  // per call were ~0.05-0.1 ms of every get of the bench step
  Entry* const* esp = nullptr;
  LC_TRY(scan_entries_cached(scan, handles, &esp));
  // After a filter the counts are on the device: read with device-side bookkeeping and one synchronisation
  // (scan_read_fused), sized by the previous read of this scan; the first read, and shapes that path does not cover, are
  // planned on the host below.
  if (scan->counts_on_device && !scan->all_rows) {
    uint64_t total_in = 0;
    for (uint32_t r : scan->rows) total_in += r;
    const int rc = scan_read_fused(ctx, &scan->fused, esp, scan->n, scan->d_sel, scan->d_word_off, scan->d_counts, total_in,
                                   out_schema, out_array);
    if (rc != LC_INTERNAL_FALLBACK) return rc;
  }
  const std::vector<Entry*> es(esp, esp + scan->n);
  LC_TRY(scan_fetch_counts(scan));
  ctx->L()->scratch.reset();
  std::vector<Entry*> es2;
  std::vector<uint64_t> woff2;
  std::vector<uint32_t> k2;
  scan_nonempty(scan, es, &es2, &woff2, &k2);
  DevSel ds{scan->d_sel, woff2.data(), k2.data(), scan->all_rows};
  LC_TRY(to_arrow_batch(ctx, es2.data(), es2.size(), nullptr, &ds, out_schema, out_array));
  // teach the next read of this scan its sizes: rows, value bytes (byte views: the data buffer), dictionary scratch
  int64_t value_bytes = 0;
  uint64_t ulen = 0;
  if (out_array->n_buffers == 3 && out_array->buffers[1]) {
    const int32_t* off = static_cast<const int32_t*>(out_array->buffers[1]);
    value_bytes = off[out_array->length] - off[0];
    for (Entry* e : es2) ulen += (e->sh.n_unique + 3u) & ~3u;
  }
  fused_read_learn(&scan->fused, out_array, value_bytes, ulen);
  return LC_OK;
}

int lc_scan_read_device(lc_scan* scan, const lc_handle* handles, void* d_values, uint64_t values_cap, void* d_offsets,
                        void* d_validity, uint64_t* out_rows, uint64_t* out_value_bytes, uint64_t* out_null_count) {
  if (!scan || !handles) return LC_ERR_INVALID;
  lc_ctx* ctx = scan->ctx;
  ScanGuard g(scan);
  Entry* const* esp = nullptr;
  LC_TRY(scan_entries_cached(scan, handles, &esp));
  LC_TRY(scan_fetch_counts(scan));
  ctx->L()->scratch.reset();
  DevSel ds{scan->d_sel, scan->word_off.data(), scan->counts.data(), scan->all_rows};
  DeviceOut dout{d_values, values_cap, d_offsets, d_validity, out_rows, out_value_bytes, out_null_count};
  return to_arrow_batch(ctx, esp, scan->n, nullptr, &ds, nullptr, nullptr, &dout);
}

int lc_scan_read_borrowed(lc_scan* scan, const lc_handle* handles, void** d_values, void** d_offsets, uint64_t* out_rows,
                          uint64_t* out_value_bytes) {
  if (!scan || !handles || !d_values || !d_offsets || !out_rows || !out_value_bytes) return LC_ERR_INVALID;
  lc_ctx* ctx = scan->ctx;
  ScanGuard g(scan);
  Entry* const* esp = nullptr;
  LC_TRY(scan_entries_cached(scan, handles, &esp));
  if (!scan->counts_on_device || scan->all_rows) {
    set_error("lc_scan_read_borrowed: no filter has run on this scan yet");
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  uint64_t total_in = 0;
  for (uint32_t r : scan->rows) total_in += r;
  FusedDeviceOut out;
  const int rc = scan_read_fused(ctx, &scan->fused, esp, scan->n, scan->d_sel, scan->d_word_off, scan->d_counts, total_in, nullptr,
                                 nullptr, &out);
  if (rc == LC_INTERNAL_FALLBACK) {
    set_error("lc_scan_read_borrowed: this read is not planned on the device (first read of the scan, nulls, or capacities outgrown)");
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  LC_TRY(rc);
  *d_values = out.d_values;
  *d_offsets = out.d_offsets;
  *out_rows = out.rows;
  *out_value_bytes = out.value_bytes;
  return LC_OK;
}

static_assert(sizeof(lc_read_header) == sizeof(ScanPlanHdr) && offsetof(lc_read_header, rows) == offsetof(ScanPlanHdr, rows) &&
                  offsetof(lc_read_header, value_bytes) == offsetof(ScanPlanHdr, bytes) &&
                  offsetof(lc_read_header, overflow) == offsetof(ScanPlanHdr, overflow),
              "lc_read_header is the plan header the kernels write");

int lc_scan_read_async(lc_scan* scan, const lc_handle* handles, void* d_values, uint64_t values_cap, void* d_offsets,
                       uint64_t rows_cap, void* d_header) {
  if (!scan || !handles || !d_values || !d_header) return LC_ERR_INVALID;
  lc_ctx* ctx = scan->ctx;
  ScanGuard g(scan);
  Entry* const* esp = nullptr;
  LC_TRY(scan_entries_cached(scan, handles, &esp));
  if (!scan->counts_on_device || scan->all_rows) {
    set_error("lc_scan_read_async: no filter has run on this scan yet");
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  const int rc = scan_read_async(ctx, &scan->fused, esp, scan->n, scan->d_sel, scan->d_word_off, scan->d_counts, d_values, values_cap,
                                 d_offsets, rows_cap, d_header);
  if (rc == LC_INTERNAL_FALLBACK) {
    set_error("lc_scan_read_async: this column is not read by the device-planned path (nulls, views, dictionaries, floats, decimals)");
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  return rc;
}

void lc_scan_end(lc_scan* scan) {
  if (!scan) return;
  {
    ScanGuard g(scan);
    cudaStreamSynchronize(scan->ctx->L()->stream);
    if (scan->d_sel) cudaFree(scan->d_sel);
    if (scan->d_probe) cudaFree(scan->d_probe);
    if (scan->d_save) cudaFree(scan->d_save);
    if (scan->d_pcounts) cudaFree(scan->d_pcounts);
    if (scan->d_term) cudaFree(scan->d_term);
    if (scan->d_acc) cudaFree(scan->d_acc);
    if (scan->d_tcounts) cudaFree(scan->d_tcounts);
    if (scan->d_rows) cudaFree(scan->d_rows);
    if (scan->d_counts) cudaFree(scan->d_counts);
    if (scan->d_word_off) cudaFree(scan->d_word_off);
    fused_read_free(&scan->fused);
  }
  g_validated_gen.fetch_add(1, std::memory_order_acq_rel);  // the scan's validated lists go with it
  delete scan;
}

}  // extern "C"

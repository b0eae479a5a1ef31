// squeeze_host.cc — squeezed integer entries: half-width codes in HBM, the full LQDA image behind the caller's read
// function (host memory or disk, the caller's choice).
// Reference: LiquidPrimitiveArray::squeeze (/root/reference/src/core/src/liquid_array/primitive_array.rs:389-499),
// LiquidPrimitiveClampedArray / LiquidPrimitiveQuantizedArray (liquid_array/hybrid_primitive_array.rs:72-790),
// LiquidSqueezedArray (liquid_array/mod.rs:209-263), SqueezeIoHandler (mod.rs:282-…).
//
// A squeezed entry is an ordinary integer blob (IntHeader + FastLanes chunks) whose packed words are the codes at
// bit_width / 2 and whose reference is the full entry's: decoding it gives `reference + code`. Both policies then reduce
// to the integer scan kernels that exist already:
//   Clamp     code = min(offset, sentinel). `reference + code` IS the value below the sentinel, and a sentinel row stands
//             for "some value >= reference + sentinel": when the literal sits below that bound (the reference's
//             resolves_on_sentinel) the plain comparison of `reference + code` with the literal gives exactly the constants
//             of hybrid_primitive_array.rs:232-240; otherwise a selected sentinel row makes the call read the backing.
//   Quantize  code = offset / bucket_width. b < q / b > q decide, b == q decides only at a bucket edge (:566-598): the same
//             operator against `reference + q` is the answer whenever no selected row sits in bucket q.
// "Is there a selected, valid row with code c" is one more run of the scan kernel (`= reference + c`, true count).
// When the codes cannot decide, the image is read back through the caller's function, becomes a temporary full entry
// (entry_from_bytes) and the call runs on that — what hydrate_full_arrow + arrow's kernels do in the reference.
#include <vector>

#include "host_common.h"
#include "squeeze_plan.h"

namespace lc {

namespace {

struct SqueezeScope {  // lets the batch functions accept a squeezed entry while this file drives them
  lc_ctx* ctx;
  bool prev;
  explicit SqueezeScope(lc_ctx* c) : ctx(c), prev(c->L()->squeeze_internal) { c->L()->squeeze_internal = true; }
  ~SqueezeScope() { ctx->L()->squeeze_internal = prev; }
};

SqueezeFacts facts_of(const Entry* e) { return SqueezeFacts{e->ih, e->squeeze_kind, e->bucket_width}; }
__int128 reference_of(const Entry* e) { const SqueezeFacts f = facts_of(e); return reference_of(&f); }
bool literal_of(const Entry* e, const lc_predicate* pred, __int128* k) { const SqueezeFacts f = facts_of(e); return literal_of(&f, pred, k); }
lc_predicate int_predicate(const Entry* e, int32_t op, __int128 lit) { const SqueezeFacts f = facts_of(e); return int_predicate(&f, op, lit); }
Doubt doubt_of(const Entry* e, int32_t op, __int128 k) { const SqueezeFacts f = facts_of(e); return doubt_of(&f, op, k); }

// selected, valid rows of `sq` whose decoded value equals `value`
int count_equal(lc_ctx* ctx, Entry* sq, __int128 value, const uint8_t* sel_bits, uint64_t* count) {
  const lc_predicate p = int_predicate(sq, LC_OP_EQ, value);
  std::vector<uint8_t> vals(round_up((static_cast<uint64_t>(sq->n) + 7) / 8, 16) + 16);
  uint64_t len = 0, nulls = 0, trues = 0;
  const uint64_t off0 = 0;
  PredOut po{vals.data(), nullptr, &off0, &len, &nulls, &trues};
  const uint8_t* sels[1] = {sel_bits};
  Entry* list[1] = {sq};
  ctx->L()->scratch.reset();
  LC_TRY(eval_predicate_batch(ctx, list, 1, &p, sel_bits ? sels : nullptr, po));
  *count = trues;
  return LC_OK;
}

// hydrate_full_arrow (hybrid_primitive_array.rs:116-127): the backing bytes as a temporary full entry
int hydrate(lc_ctx* ctx, const Entry* sq, Entry** full) {
  std::vector<uint8_t> image(sq->backing_len);
  ctx->squeeze_reads++;
  const int rc = sq->backing_read ? sq->backing_read(sq->backing_user, 0, sq->backing_len, image.data()) : -1;
  if (rc != 0) {
    set_error("squeezed entry: reading %llu backing bytes failed (%d)", (unsigned long long)sq->backing_len, rc);
    return LC_ERR_INVALID;
  }
  ctx->L()->scratch.reset();
  LC_TRY(entry_from_bytes(ctx, image.data(), image.size(), nullptr, full));
  const std::string& want_format = sq->orig_format.empty() ? sq->arrow_format : sq->orig_format;
  if ((*full)->n != sq->n || (*full)->liquid_type != LC_LIQUID_INTEGER || (*full)->arrow_format != want_format) {
    release_entry(ctx, *full);
    *full = nullptr;
    set_error("squeezed entry: the backing bytes are not the image this entry was squeezed from");
    return LC_ERR_INVALID;
  }
  return LC_OK;
}

}  // namespace

namespace {

long long ticks_per_day_of(const std::string& format) {  // 0 for Date32
  if (format.rfind("tss", 0) == 0) return 86400ll;
  if (format.rfind("tsm", 0) == 0) return 86400000ll;
  if (format.rfind("tsu", 0) == 0) return 86400000000ll;
  if (format.rfind("tsn", 0) == 0) return 86400000000000ll;
  return 0;
}

struct ArenaWork {  // a work area borrowed from the arena, handed back on every way out
  lc_ctx* ctx;
  uint8_t* p = nullptr;
  uint32_t slab = 0;
  uint64_t bytes = 0;
  ArenaWork(lc_ctx* c, uint64_t b) : ctx(c), bytes(b) { p = c->arena_alloc(b, &slab); }
  ~ArenaWork() {
    if (p) ctx->arena_free(slab, p, bytes);
  }
  ArenaWork(const ArenaWork&) = delete;
  ArenaWork& operator=(const ArenaWork&) = delete;
};

// SqueezedDate32Array::from_liquid_date32 / from_liquid_timestamp (squeezed_date32_array.rs:63-223): decode, one component
// per row, its min / max over the valid rows, offsets from the min packed as a 32-bit column. The blob is an ordinary
// Int32-shaped entry (reference = smallest component), so decoding it gives to_component_date32.
int squeeze_date_entry(lc_ctx* ctx, Entry* full, uint32_t field, lc_backing_read read, void* user, uint64_t image_len, Entry** out) {
  const IntHeader& fh = full->ih;
  const uint32_t n = full->n, tb = fh.tbits / 8;
  cudaStream_t s = ctx->L()->stream;
  ArenaWork vals(ctx, round_up(static_cast<uint64_t>(n) * tb, 256) + 256), comp(ctx, round_up(static_cast<uint64_t>(n) * 4, 256) + 256);
  if (!vals.p || !comp.p) {
    set_error(ctx->arena_at_limit() ? "cache full: the HBM reservation has reached the budget for the squeeze work areas" : "HBM arena: cudaMalloc failed for the squeeze work areas");
    return ctx->arena_at_limit() ? LC_ERR_CACHE_FULL : LC_ERR_OOM;
  }
  if (n) {
    uint64_t rows = 0, vbytes = 0, nulls = 0;
    DeviceOut dout{vals.p, static_cast<uint64_t>(n) * tb, nullptr, nullptr, &rows, &vbytes, &nulls};
    Entry* list[1] = {full};
    ctx->L()->scratch.reset();
    LC_TRY(to_arrow_batch(ctx, list, 1, nullptr, nullptr, nullptr, nullptr, &dout));
  }
  ctx->L()->scratch.reset();
  Scratch& sc = ctx->L()->scratch;
  LC_TRY(sc.reserve(2048, 2048));
  IntMinMaxWork* h_mm = reinterpret_cast<IntMinMaxWork*>(sc.host(256));
  IntPackWork* h_pw = reinterpret_cast<IntPackWork*>(sc.host(256));
  uint64_t* h_mmout = reinterpret_cast<uint64_t*>(sc.host(256));
  uint8_t* d_mm = sc.dev(256);
  uint8_t* d_pw = sc.dev(256);
  uint8_t* d_mmout = sc.dev(256);
  if (!h_mm || !h_pw || !h_mmout || !d_mm || !d_pw || !d_mmout) {
    set_error("lc_squeeze: scratch exhausted");
    return LC_ERR_OOM;
  }
  const uint32_t* d_valid = fh.has_nulls ? reinterpret_cast<const uint32_t*>(full->d_blob + fh.validity_off) : nullptr;
  LC_CUDA_OK(launch_date_component(vals.p, n, fh.tbits, field, ticks_per_day_of(full->arrow_format), reinterpret_cast<int32_t*>(comp.p), s));
  ctx->kernel_launches++;
  h_mm->values = comp.p;
  h_mm->validity = d_valid;
  h_mm->out = reinterpret_cast<uint64_t*>(d_mmout);
  h_mm->n = n;
  h_mm->phys = PT_I32;
  h_mmout[0] = h_mmout[1] = h_mmout[2] = 0;
  if (n) {
    LC_CUDA_OK(cudaMemcpyAsync(d_mm, h_mm, sizeof(IntMinMaxWork), cudaMemcpyHostToDevice, s));
    LC_CUDA_OK(launch_int_minmax(reinterpret_cast<const IntMinMaxWork*>(d_mm), 1, s));
    ctx->kernel_launches++;
    LC_CUDA_OK(cudaMemcpyAsync(h_mmout, d_mmout, 32, cudaMemcpyDeviceToHost, s));
    LC_CUDA_OK(cudaStreamSynchronize(s));
  }
  const int64_t mn = static_cast<int64_t>(h_mmout[0]), mx = static_cast<int64_t>(h_mmout[1]);
  const uint64_t n_valid = h_mmout[2];

  IntHeader h;
  std::memset(&h, 0, sizeof(h));
  h.magic = kMagicInt;
  h.phys = PT_I32;
  h.tbits = 32;
  h.n = n;
  h.n_chunks = (n + 1023) / 1024;
  h.is_signed = 1;
  h.has_nulls = fh.has_nulls;
  h.null_count = fh.null_count;
  if (n_valid == 0) {  // BitPackedArray::new_null_array, reference_value 0 (:78-90, :116-124)
    h.bit_width = 0;
    h.reference = 0;
    h.has_nulls = n > 0;
    h.null_count = n;
  } else {
    const uint64_t span = static_cast<uint64_t>(mx - mn);
    h.bit_width = static_cast<uint8_t>(span == 0 ? 1u : 64u - static_cast<uint32_t>(__builtin_clzll(span)));
    h.reference = static_cast<uint64_t>(mn) & 0xffffffffull;
  }
  const uint64_t valid_bytes = h.has_nulls ? round_up((static_cast<uint64_t>(n) + 7) / 8, 16) : 0;
  h.validity_off = h.has_nulls ? 64 : 0;
  h.packed_off = static_cast<uint32_t>(64 + valid_bytes);
  const uint64_t blob_bytes = round_up(h.packed_off + static_cast<uint64_t>(h.n_chunks) * 128ull * h.bit_width, 16);
  h.blob_bytes = static_cast<uint32_t>(blob_bytes);
  if (ctx->budget && ctx->arena_used() + blob_bytes > ctx->budget) {
    set_error("cache full: %llu + %llu > budget %llu", (unsigned long long)ctx->arena_used(), (unsigned long long)blob_bytes,
              (unsigned long long)ctx->budget);
    return LC_ERR_CACHE_FULL;
  }
  uint32_t slab = 0;
  uint8_t* d_blob = ctx->arena_alloc(blob_bytes, &slab);
  if (!d_blob) {
    set_error(ctx->arena_at_limit() ? "cache full: the HBM reservation has reached the budget for %llu bytes" : "HBM arena: cudaMalloc failed for %llu bytes", (unsigned long long)blob_bytes);
    return ctx->arena_at_limit() ? LC_ERR_CACHE_FULL : LC_ERR_OOM;
  }
  std::memset(h_pw, 0, sizeof(*h_pw));
  h_pw->values = comp.p;
  h_pw->validity = d_valid;  // an entirely null column: every validity bit of the full entry is clear already
  h_pw->blob = d_blob;
  h_pw->pack_null_slots = 0;
  h_pw->hdr = h;
  cudaError_t ce = cudaMemcpyAsync(d_pw, h_pw, sizeof(IntPackWork), cudaMemcpyHostToDevice, s);
  if (ce == cudaSuccess) ce = launch_int_pack(reinterpret_cast<const IntPackWork*>(d_pw), 1, s);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);
  if (ce != cudaSuccess) {
    ctx->arena_free(slab, d_blob, blob_bytes);
    set_error("CUDA error in lc_squeeze: %s", cudaGetErrorString(ce));
    return LC_ERR_CUDA;
  }
  ctx->kernel_launches++;
  Entry* e = new Entry();
  e->liquid_type = LC_LIQUID_INTEGER;
  e->d_blob = d_blob;
  e->blob_bytes = h.blob_bytes;
  e->slab = slab;
  e->n = n;
  e->arrow_format = "tdD";  // what the blob decodes to: the component values typed Date32 (to_component_date32)
  e->orig_format = full->arrow_format;
  e->ih = h;
  e->squeeze_kind = 3;
  ctx->epoch++;  // cached entry lists remember whether they hold squeezed entries
  e->date_field = field;
  e->backing_read = read;
  e->backing_user = user;
  e->backing_len = image_len;
  ctx->n_entries++;
  *out = e;
  return LC_OK;
}

}  // namespace

int squeeze_entry(lc_ctx* ctx, Entry* full, int32_t policy, int32_t hint, lc_backing_read read, void* user, uint8_t* bytes_out,
                  uint64_t cap, uint64_t* out_bytes, Entry** out) {
  *out = nullptr;
  *out_bytes = 0;
  const bool is_date = full->arrow_format == "tdD" || full->arrow_format.rfind("ts", 0) == 0;
  if (is_date && full->liquid_type == LC_LIQUID_INTEGER && full->squeeze_kind == 0) {
    // Date32 / Timestamp: only a hint that names a date field squeezes (primitive_array.rs:399-411)
    if (hint < LC_HINT_EXTRACT_YEAR || hint > LC_HINT_EXTRACT_DAY_OF_WEEK) return LC_OK;
    uint64_t image_len = 0;
    LC_TRY(entry_to_bytes(ctx, full, nullptr, 0, &image_len));
    *out_bytes = image_len;
    if (!bytes_out) return LC_OK;  // size query
    if (cap < image_len || !read) {
      set_error("lc_squeeze: needs a buffer of %llu bytes and a read function", (unsigned long long)image_len);
      return LC_ERR_INVALID;
    }
    ctx->L()->scratch.reset();
    LC_TRY(entry_to_bytes(ctx, full, bytes_out, cap, &image_len));
    return squeeze_date_entry(ctx, full, static_cast<uint32_t>(hint - LC_HINT_EXTRACT_YEAR), read, user, image_len, out);
  }
  if (policy != LC_SQUEEZE_CLAMP && policy != LC_SQUEEZE_QUANTIZE) {
    set_error("lc_squeeze: unknown policy %d", policy);
    return LC_ERR_INVALID;
  }
  // None in the reference: no hint (:394); no bit width (all null) or fewer than 8 bits (:414-417). Floats, decimals and
  // byte views have squeezed forms of their own in the reference; none of them is built here.
  if (full->liquid_type != LC_LIQUID_INTEGER || full->squeeze_kind != 0 || hint == LC_HINT_NONE || is_date) return LC_OK;
  const IntHeader& fh = full->ih;
  if (fh.bit_width < 8) return LC_OK;

  uint64_t image_len = 0;
  LC_TRY(entry_to_bytes(ctx, full, nullptr, 0, &image_len));
  *out_bytes = image_len;
  if (!bytes_out) return LC_OK;  // size query
  if (cap < image_len) {
    set_error("lc_squeeze: buffer of %llu bytes, the full image needs %llu", (unsigned long long)cap, (unsigned long long)image_len);
    return LC_ERR_INVALID;
  }
  if (!read) {
    set_error("lc_squeeze: a squeezed entry needs a read function for its backing bytes");
    return LC_ERR_INVALID;
  }
  ctx->L()->scratch.reset();
  LC_TRY(entry_to_bytes(ctx, full, bytes_out, cap, &image_len));  // full bytes (original format) are what goes to disk (:396)

  const uint32_t n = full->n, tb = fh.tbits / 8;
  const uint32_t new_bw = fh.bit_width / 2;  // >= 4
  const uint64_t tmask = fh.tbits == 64 ? ~0ull : ((1ull << fh.tbits) - 1ull);
  cudaStream_t s = ctx->L()->stream;

  // ---- the full entry's values, decoded into a work area of their own (k_int_scan<DECODE>) ----
  const uint64_t work_bytes = round_up(static_cast<uint64_t>(n) * tb, 256) + 256;
  uint32_t wslab = 0;
  uint8_t* d_vals = ctx->arena_alloc(work_bytes, &wslab);
  if (!d_vals) {
    set_error(ctx->arena_at_limit() ? "cache full: the HBM reservation has reached the budget for %llu bytes" : "HBM arena: cudaMalloc failed for %llu bytes", (unsigned long long)work_bytes);
    return ctx->arena_at_limit() ? LC_ERR_CACHE_FULL : LC_ERR_OOM;
  }
  struct Work {  // returned to the arena on every way out
    lc_ctx* ctx;
    uint32_t slab;
    uint8_t* p;
    uint64_t bytes;
    ~Work() { ctx->arena_free(slab, p, bytes); }
  } work{ctx, wslab, d_vals, work_bytes};
  {
    uint64_t rows = 0, vbytes = 0, nulls = 0;
    DeviceOut dout{d_vals, static_cast<uint64_t>(n) * tb, nullptr, nullptr, &rows, &vbytes, &nulls};
    Entry* list[1] = {full};
    ctx->L()->scratch.reset();
    LC_TRY(to_arrow_batch(ctx, list, 1, nullptr, nullptr, nullptr, nullptr, &dout));
  }
  ctx->L()->scratch.reset();
  Scratch& sc = ctx->L()->scratch;
  LC_TRY(sc.reserve(2048, 2048));
  IntMinMaxWork* h_mm = reinterpret_cast<IntMinMaxWork*>(sc.host(256));
  IntPackWork* h_pw = reinterpret_cast<IntPackWork*>(sc.host(256));
  uint64_t* h_mmout = reinterpret_cast<uint64_t*>(sc.host(256));
  uint8_t* d_mm = sc.dev(256);
  uint8_t* d_pw = sc.dev(256);
  uint8_t* d_mmout = sc.dev(256);
  if (!h_mm || !h_pw || !h_mmout || !d_mm || !d_pw || !d_mmout) {
    set_error("lc_squeeze: scratch exhausted");
    return LC_ERR_OOM;
  }
  const uint32_t* d_valid = fh.has_nulls ? reinterpret_cast<const uint32_t*>(full->d_blob + fh.validity_off) : nullptr;

  uint64_t limit = (1ull << new_bw) - 1ull;  // the sentinel, or the last bucket
  uint64_t bucket_width = 0;
  if (policy == LC_SQUEEZE_QUANTIZE) {
    // max offset -> bucket width = ceil((max_offset + 1) / bucket_count), at least 1 (:457-470). Null slots hold offset 0
    // in an entry built here, so the maximum over the valid rows is the maximum over all of them.
    h_mm->values = d_vals;
    h_mm->validity = d_valid;
    h_mm->out = reinterpret_cast<uint64_t*>(d_mmout);
    h_mm->n = n;
    h_mm->phys = fh.phys;
    LC_CUDA_OK(cudaMemcpyAsync(d_mm, h_mm, sizeof(IntMinMaxWork), cudaMemcpyHostToDevice, s));
    LC_CUDA_OK(launch_int_minmax(reinterpret_cast<const IntMinMaxWork*>(d_mm), 1, s));
    ctx->kernel_launches++;
    LC_CUDA_OK(cudaMemcpyAsync(h_mmout, d_mmout, 32, cudaMemcpyDeviceToHost, s));
    LC_CUDA_OK(cudaStreamSynchronize(s));
    const uint64_t max_off = (h_mmout[1] - fh.reference) & tmask;
    const uint64_t range = max_off == ~0ull ? ~0ull : max_off + 1;  // saturating_add(1)
    const uint64_t buckets = 1ull << new_bw;
    bucket_width = range / buckets + (range % buckets ? 1 : 0);
    if (bucket_width == 0) bucket_width = 1;
  }
  LC_CUDA_OK(launch_squeeze_map(d_vals, n, fh.tbits, fh.reference, policy == LC_SQUEEZE_QUANTIZE, limit, bucket_width, s));
  ctx->kernel_launches++;

  // ---- the squeezed blob: same header and validity, packed at half the width ----
  IntHeader h = fh;
  h.bit_width = static_cast<uint8_t>(new_bw);
  h.squeeze_kind = static_cast<uint8_t>(policy + 1);  // the scan kernel's planner compares codes accordingly (k_int.cu)
  set_int_bucket_width(&h, bucket_width);
  const uint64_t packed_bytes = static_cast<uint64_t>(h.n_chunks) * 128ull * new_bw;
  const uint64_t blob_bytes = round_up(h.packed_off + packed_bytes, 16);
  h.blob_bytes = static_cast<uint32_t>(blob_bytes);
  if (ctx->budget && ctx->arena_used() + blob_bytes > ctx->budget) {
    set_error("cache full: %llu + %llu > budget %llu", (unsigned long long)ctx->arena_used(), (unsigned long long)blob_bytes,
              (unsigned long long)ctx->budget);
    return LC_ERR_CACHE_FULL;
  }
  uint32_t slab = 0;
  uint8_t* d_blob = ctx->arena_alloc(blob_bytes, &slab);
  if (!d_blob) {
    set_error(ctx->arena_at_limit() ? "cache full: the HBM reservation has reached the budget for %llu bytes" : "HBM arena: cudaMalloc failed for %llu bytes", (unsigned long long)blob_bytes);
    return ctx->arena_at_limit() ? LC_ERR_CACHE_FULL : LC_ERR_OOM;
  }
  std::memset(h_pw, 0, sizeof(*h_pw));
  h_pw->values = d_vals;
  h_pw->validity = d_valid;
  h_pw->blob = d_blob;
  h_pw->pack_null_slots = 0;
  h_pw->hdr = h;
  cudaError_t ce = cudaMemcpyAsync(d_pw, h_pw, sizeof(IntPackWork), cudaMemcpyHostToDevice, s);
  if (ce == cudaSuccess) ce = launch_int_pack(reinterpret_cast<const IntPackWork*>(d_pw), 1, s);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);
  if (ce != cudaSuccess) {
    ctx->arena_free(slab, d_blob, blob_bytes);
    set_error("CUDA error in lc_squeeze: %s", cudaGetErrorString(ce));
    return LC_ERR_CUDA;
  }
  ctx->kernel_launches++;

  Entry* e = new Entry();
  e->liquid_type = LC_LIQUID_INTEGER;
  e->d_blob = d_blob;
  e->blob_bytes = h.blob_bytes;
  e->slab = slab;
  e->n = n;
  e->arrow_format = full->arrow_format;
  e->ih = h;
  e->squeeze_kind = policy + 1;
  ctx->epoch++;  // cached entry lists remember whether they hold squeezed entries
  e->bucket_width = bucket_width;
  e->backing_read = read;
  e->backing_user = user;
  e->backing_len = image_len;
  ctx->n_entries++;
  *out = e;
  return LC_OK;
}

namespace {

// What the half-width codes can say about `col <op> k` (try_eval_predicate_inner of either array). The predicate itself
// runs on the squeezed entry unchanged — k_int_scan's planner compares `reference + code` (Clamp) or bucket indices
// (Quantize, from the header's squeeze_kind / bucket width). What is decided here is whether the codes MAY not decide, and
// which probe finds the rows that make them fail:
//   Clamp     resolves_on_sentinel (hybrid_primitive_array.rs:196-219) false -> rows at the sentinel (kLitSentinelPublic)
//   Quantize  on_equal_bucket (:599-631) unknown -> rows in the literal's bucket: `= k`, which the planner turns into b == q
// selected, valid rows of `sq` that the probe finds
int count_probe(lc_ctx* ctx, Entry* sq, const lc_predicate& probe, const uint8_t* sel_bits, uint64_t* count) {
  std::vector<uint8_t> vals(round_up((static_cast<uint64_t>(sq->n) + 7) / 8, 16) + 16);
  uint64_t len = 0, nulls = 0, trues = 0;
  const uint64_t off0 = 0;
  PredOut po{vals.data(), nullptr, &off0, &len, &nulls, &trues};
  const uint8_t* sels[1] = {sel_bits};
  Entry* list[1] = {sq};
  ctx->L()->scratch.reset();
  LC_TRY(eval_predicate_batch(ctx, list, 1, &probe, sel_bits ? sels : nullptr, po));
  *count = trues;
  return LC_OK;
}

}  // namespace

int squeezed_eval_predicate(lc_ctx* ctx, Entry* sq, const lc_predicate* pred, const uint8_t* sel_bits, const PredOut& out) {
  SqueezeScope scope(ctx);
  const uint8_t* sels[1] = {sel_bits};
  if (sq->squeeze_kind == 3) {
    // SqueezedDate32Array::try_eval_predicate (:478-485): filter (which reads the backing unless nothing is selected),
    // then the predicate on the filtered rows
    if (sel_bits && popcount_bits(sel_bits, sq->n) == 0) {
      if (out.len) out.len[0] = 0;
      if (out.null_count) out.null_count[0] = 0;
      if (out.true_count) out.true_count[0] = 0;
      return LC_OK;
    }
    Entry* full = nullptr;
    LC_TRY(hydrate(ctx, sq, &full));
    Entry* list1[1] = {full};
    ctx->L()->scratch.reset();
    const int rc = eval_predicate_batch(ctx, list1, 1, pred, sel_bits ? sels : nullptr, out);
    release_entry(ctx, full);
    return rc;
  }
  if (pred->op < LC_OP_EQ || pred->op > LC_OP_GE) {
    set_error("operator %d is not supported on integer columns", pred->op);
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  __int128 k = 0;
  bool from_codes = false;  // a literal outside the column's type (Ok(None)) goes the long way round
  if (literal_of(sq, pred, &k)) {
    from_codes = true;
    const Doubt d = doubt_of(sq, pred->op, k);
    if (d.possible) {
      uint64_t hits = 0;
      LC_TRY(count_probe(ctx, sq, d.probe, sel_bits, &hits));
      if (hits) from_codes = false;  // Err(NeedsBacking)
    }
  }
  Entry* list[1] = {sq};
  if (from_codes) {
    ctx->squeeze_saved++;  // io.trace_io_saved()
    ctx->L()->scratch.reset();
    return eval_predicate_batch(ctx, list, 1, pred, sel_bits ? sels : nullptr, out);
  }
  Entry* full = nullptr;
  LC_TRY(hydrate(ctx, sq, &full));
  list[0] = full;
  ctx->L()->scratch.reset();
  const int rc = eval_predicate_batch(ctx, list, 1, pred, sel_bits ? sels : nullptr, out);
  release_entry(ctx, full);
  return rc;
}

// For the scan pipeline (lc_abi.cc lc_scan_filter): what the codes of ONE entry can say about the predicate.
//   returns 0: they decide (or the entry is a full one); 1 / 2: they decide unless the clamp / quantize probe finds a
//   selected row (*probe is that probe); 3: the backing is needed whatever the rows (literal outside the column's type)
int squeeze_doubt(const Entry* e, const lc_predicate* pred, lc_predicate* probe) {
  if (!e->squeeze_kind) return 0;
  __int128 k = 0;
  if (!literal_of(e, pred, &k)) return 3;
  const Doubt d = doubt_of(e, pred->op, k);
  if (!d.possible) return 0;
  *probe = d.probe;
  return e->squeeze_kind;
}

int squeeze_hydrate(lc_ctx* ctx, const Entry* sq, Entry** full) { return hydrate(ctx, sq, full); }

// The same over a LIST of entries — any mix of full and squeezed (clamp / quantize) integer entries of one column — in a
// few launches for the whole list: one probe pass per squeeze form that has entries in doubt, one pass of the predicate
// itself, then only the entries whose probe found a row go back to their backing bytes one by one.
int squeezed_eval_predicate_many(lc_ctx* ctx, Entry* const* entries, uint64_t n, const lc_predicate* pred,
                                 const uint8_t* const* sel_bits, const PredOut& out_in) {
  SqueezeScope scope(ctx);
  if (pred->op < LC_OP_EQ || pred->op > LC_OP_GE) {
    set_error("operator %d is not supported on integer columns", pred->op);
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  const uint64_t zero_off = 0;
  PredOut out = out_in;
  if (!out.byte_offsets) {
    if (n > 1) {
      set_error("eval_predicate_many: out_byte_offsets required for n > 1");
      return LC_ERR_INVALID;
    }
    out.byte_offsets = &zero_off;
  }
  std::vector<uint8_t> doubt(n, 0), backing(n, 0);  // doubt: 1 clamp probe, 2 quantize probe
  lc_predicate probes[3] = {};
  uint64_t n_doubt[3] = {0, 0, 0};
  for (uint64_t i = 0; i < n; ++i) {
    Entry* e = entries[i];
    if (e->squeeze_kind == 3 || (e->squeeze_kind && e->liquid_type != LC_LIQUID_INTEGER)) {
      set_error("eval_predicate_many: entry %llu is a date-component entry; those answer through lc_eval_predicate", (unsigned long long)i);
      return LC_ERR_INVALID;
    }
    if (!e->squeeze_kind) continue;
    __int128 k = 0;
    if (!literal_of(e, pred, &k)) {
      backing[i] = 1;
      continue;
    }
    const Doubt d = doubt_of(e, pred->op, k);
    if (!d.possible) continue;
    doubt[i] = static_cast<uint8_t>(e->squeeze_kind);
    probes[e->squeeze_kind] = d.probe;  // the same for every entry of that form: the sentinel probe / `= k`
    n_doubt[e->squeeze_kind]++;
  }
  // `= k` over quantized entries is its own probe: the predicate pass below tells which entries have a row in bucket q
  const bool self_probe = pred->op == LC_OP_EQ && n_doubt[2] && !n_doubt[1];
  std::vector<uint64_t> own_trues;
  if (self_probe && !out.true_count) {
    own_trues.assign(n, 0);
    out.true_count = own_trues.data();
  }
  // ---- probe passes: true counts per entry; masks land in a scratch area laid out like the caller's ----
  if ((n_doubt[1] || n_doubt[2]) && !self_probe) {
    uint64_t span = 0;
    for (uint64_t i = 0; i < n; ++i) span = std::max<uint64_t>(span, out.byte_offsets[i] + round_up((static_cast<uint64_t>(entries[i]->n) + 7) / 8, 16));
    std::vector<uint8_t> tmp(span + 64);
    std::vector<uint64_t> len(n), nulls(n), trues(n);
    for (int form = 1; form <= 2; ++form) {
      if (!n_doubt[form]) continue;
      PredOut po{tmp.data(), nullptr, out.byte_offsets, len.data(), nulls.data(), trues.data()};
      ctx->L()->scratch.reset();
      LC_TRY(eval_predicate_batch(ctx, entries, n, &probes[form], sel_bits, po));
      for (uint64_t i = 0; i < n; ++i)
        if (doubt[i] == form && trues[i]) backing[i] = 1;  // Err(NeedsBacking)
    }
  }
  // ---- the predicate over the whole list ----
  ctx->L()->scratch.reset();
  LC_TRY(eval_predicate_batch(ctx, entries, n, pred, sel_bits, out));
  if (self_probe)
    for (uint64_t i = 0; i < n; ++i)
      if (doubt[i] == 2 && out.true_count[i]) backing[i] = 1;  // Err(NeedsBacking)
  // ---- entries the codes could not decide: their slots are overwritten with the full entry's answer ----
  for (uint64_t i = 0; i < n; ++i) {
    if (entries[i]->squeeze_kind && !backing[i]) ctx->squeeze_saved++;
    if (!backing[i]) continue;
    Entry* full = nullptr;
    LC_TRY(hydrate(ctx, entries[i], &full));
    Entry* list[1] = {full};
    const uint8_t* sels[1] = {sel_bits ? sel_bits[i] : nullptr};
    PredOut po{out.values, out.validity, out.byte_offsets + i, out.len ? out.len + i : nullptr, out.null_count ? out.null_count + i : nullptr,
               out.true_count ? out.true_count + i : nullptr};
    ctx->L()->scratch.reset();
    const int rc = eval_predicate_batch(ctx, list, 1, pred, sels[0] ? sels : nullptr, po);
    release_entry(ctx, full);
    LC_TRY(rc);
  }
  return LC_OK;
}

int squeezed_to_arrow(lc_ctx* ctx, Entry* sq, const uint8_t* sel_bits, ArrowSchema* out_schema, ArrowArray* out_array) {
  SqueezeScope scope(ctx);
  const uint8_t* sels[1] = {sel_bits};
  Entry* list[1] = {sq};
  bool from_codes = false;
  if (sq->squeeze_kind == 3 && sel_bits && popcount_bits(sel_bits, sq->n) == 0) {
    // new_empty_array(original type) without a read (:465-468)
    export_schema(sq->orig_format, "", out_schema);
    std::vector<HostBuf> bufs(2);
    bufs[1] = HostBuf{host_alloc(8), 0};  // a zero-length values buffer that is still a buffer
    export_array(0, 0, std::move(bufs), nullptr, out_array);
    return LC_OK;
  }
  if (sq->squeeze_kind == LC_SQUEEZE_CLAMP + 1) {
    // to_arrow_known_only (:129-157) / filter (:324-335): below the sentinel `reference + code` is the value itself
    if (sel_bits && popcount_bits(sel_bits, sq->n) == 0) {
      from_codes = true;  // new_empty_array
    } else {
      const __int128 sent_abs = reference_of(sq) + ((static_cast<__int128>(1) << sq->ih.bit_width) - 1);
      uint64_t hits = 0;
      LC_TRY(count_equal(ctx, sq, sent_abs, sel_bits, &hits));
      from_codes = hits == 0;
    }
  }
  if (from_codes) {
    ctx->L()->scratch.reset();
    return to_arrow_batch(ctx, list, 1, sel_bits ? sels : nullptr, nullptr, out_schema, out_array);
  }
  Entry* full = nullptr;  // Quantize always (:684-686), Clamp when a selected row sits at the sentinel
  LC_TRY(hydrate(ctx, sq, &full));
  list[0] = full;
  ctx->L()->scratch.reset();
  const int rc = to_arrow_batch(ctx, list, 1, sel_bits ? sels : nullptr, nullptr, out_schema, out_array);
  release_entry(ctx, full);
  return rc;
}

// SqueezedDate32Array::to_component_array (:276-282, lossy) / to_component_date32 (:286-294): no backing read
int squeezed_component_array(lc_ctx* ctx, Entry* sq, int32_t lossy, ArrowSchema* out_schema, ArrowArray* out_array) {
  SqueezeScope scope(ctx);
  if (sq->squeeze_kind != 3) {
    set_error("lc_squeezed_component: not a date-component entry");
    return LC_ERR_INVALID;
  }
  Entry* list[1] = {sq};
  ctx->L()->scratch.reset();
  if (!lossy) return to_arrow_batch(ctx, list, 1, nullptr, nullptr, out_schema, out_array);
  const uint32_t n = sq->n;
  const long long ticks = ticks_per_day_of(sq->orig_format);
  const uint32_t out_tb = ticks ? 8 : 4;
  const uint64_t vwords = (static_cast<uint64_t>(n) + 31) / 32;
  ArenaWork comp(ctx, round_up(static_cast<uint64_t>(n) * 4, 256) + 256), res(ctx, round_up(static_cast<uint64_t>(n) * out_tb, 256) + 256),
      val(ctx, round_up(vwords * 4, 256) + 256);
  if (!comp.p || !res.p || !val.p) {
    set_error(ctx->arena_at_limit() ? "cache full: the HBM reservation has reached the budget for the component work areas" : "HBM arena: cudaMalloc failed for the component work areas");
    return ctx->arena_at_limit() ? LC_ERR_CACHE_FULL : LC_ERR_OOM;
  }
  cudaStream_t s = ctx->L()->stream;
  uint64_t rows = 0, vbytes = 0, nulls = 0;
  if (n) {
    DeviceOut dout{comp.p, static_cast<uint64_t>(n) * 4, nullptr, val.p, &rows, &vbytes, &nulls};
    LC_TRY(to_arrow_batch(ctx, list, 1, nullptr, nullptr, nullptr, nullptr, &dout));  // k_int_scan<DECODE> (+ validity)
  }
  LC_CUDA_OK(launch_date_lossy(reinterpret_cast<const int32_t*>(comp.p), nulls ? reinterpret_cast<const uint32_t*>(val.p) : nullptr, n,
                               sq->date_field, ticks, res.p, s));
  ctx->kernel_launches++;
  HostBlock values(static_cast<uint64_t>(n) * out_tb, static_cast<uint64_t>(n) * out_tb);
  HostBlock validity;
  if (nulls) {
    const uint64_t bitmap_bytes = (static_cast<uint64_t>(n) + 7) / 8;
    validity = HostBlock(round_up(bitmap_bytes, 4), bitmap_bytes);
  }
  if ((n && !values.p) || (nulls && !validity.p)) {
    set_error("host allocation failed");
    return LC_ERR_OOM;
  }
  if (n) LC_CUDA_OK(cudaMemcpyAsync(values.p, res.p, static_cast<uint64_t>(n) * out_tb, cudaMemcpyDeviceToHost, s));
  if (nulls) LC_CUDA_OK(cudaMemcpyAsync(validity.p, val.p, round_up(validity.bytes, 4), cudaMemcpyDeviceToHost, s));
  LC_CUDA_OK(cudaStreamSynchronize(s));
  ctx->d2h_bytes += values.bytes + validity.bytes;
  export_schema(sq->orig_format, "", out_schema);
  std::vector<HostBuf> bufs{validity.release(), values.release()};
  export_array(static_cast<int64_t>(n), static_cast<int64_t>(nulls), std::move(bufs), nullptr, out_array);
  return LC_OK;
}

}  // namespace lc

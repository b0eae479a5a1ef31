// liquid_cache.hpp — header-only C++ mirror of the reference's cache front door over the C ABI.
//
// Same names and argument meaning as the Rust API it stands in for
//   LiquidCacheBuilder            /root/reference/src/core/src/cache/builders.rs:32-158
//   LiquidCache::{insert,get,eval_predicate,is_cached,reset}   src/core/src/cache/core.rs:122-277
//   Insert / Get / EvaluatePredicate builders                  builders.rs:162-356
// The reference's builders are IntoFuture; here `.run()` / `.read()` stand for `.await`. Return conventions follow the
// reference: Get/EvaluatePredicate::read return false (Option::None) when the entry is absent; insert throws CacheFull
// (Result<(), CacheFull>); unsupported dtypes throw UnsupportedType so the caller keeps the Arrow array.
// Arrays cross as Arrow C Data Interface structs, exactly as in include/lc_gpu.h. No compute happens in this header.
#pragma once
#include <cstdint>
#include <stdexcept>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/lc_gpu.h"

namespace liquid_cache {

struct CacheFull : std::runtime_error { using std::runtime_error::runtime_error; };
struct UnsupportedType : std::runtime_error { using std::runtime_error::runtime_error; };
struct UnsupportedExpr : std::runtime_error { using std::runtime_error::runtime_error; };
struct GpuError : std::runtime_error { using std::runtime_error::runtime_error; };

inline void check(int rc) {
  if (rc == LC_OK) return;
  const std::string msg = lc_last_error();
  switch (rc) {
    case LC_ERR_CACHE_FULL: throw CacheFull(msg);
    case LC_ERR_UNSUPPORTED_TYPE: throw UnsupportedType(msg);
    case LC_ERR_UNSUPPORTED_EXPR: throw UnsupportedExpr(msg);
    default: throw GpuError(msg);
  }
}

using EntryID = uint64_t;
// ParquetArrayID packing (src/datafusion/src/cache/id.rs:15-22)
inline EntryID parquet_array_id(uint64_t file, uint64_t rg, uint64_t col, uint64_t batch) {
  return (file << 48) | (rg << 32) | (col << 16) | batch;
}

// A selection: Arrow BooleanBuffer bytes at bit offset 0.
struct BooleanBuffer {
  const uint8_t* bits = nullptr;
  uint64_t len = 0;
};

// A validated predicate (LiquidExpr, src/core/src/cache/liquid_expr.rs:33-44) already lowered to (op, literal).
struct LiquidExpr {
  lc_predicate pred{};
  std::string bytes;  // owns the literal for byte-like columns, and the encoded values of an IN list
  // the native form with the literal pointer taken from THIS object's bytes (copies and moves of a LiquidExpr stay valid)
  const lc_predicate* native() {
    if (pred.op == LC_OP_IN || pred.op == LC_OP_NOT_IN) {
      pred.lit_bytes = reinterpret_cast<const uint8_t*>(bytes.data());  // lit_len stays the number of values
    } else if (pred.lit_kind == LC_LIT_BYTES) {
      pred.lit_bytes = reinterpret_cast<const uint8_t*>(bytes.data());
      pred.lit_len = bytes.size();
    }
    return &pred;
  }
  static LiquidExpr compare_i64(lc_op op, int64_t v) {
    LiquidExpr e;
    e.pred.op = op;
    e.pred.lit_kind = LC_LIT_I64;
    e.pred.lit_i64 = v;
    return e;
  }
  static LiquidExpr compare_u64(lc_op op, uint64_t v) {
    LiquidExpr e;
    e.pred.op = op;
    e.pred.lit_kind = LC_LIT_U64;
    e.pred.lit_u64 = v;
    return e;
  }
  // Float32 / Float64 column: ScalarValue::Float32(v) is widened exactly (float_array.rs columns; arrow-ord total order)
  static LiquidExpr compare_f64(lc_op op, double v) {
    LiquidExpr e;
    e.pred.op = op;
    e.pred.lit_kind = LC_LIT_F64;
    std::memcpy(&e.pred.lit_u64, &v, 8);
    return e;
  }
  // Decimal128/256 column: unscaled value at the column's scale, two's complement halves (decimal_array.rs columns)
  static LiquidExpr compare_decimal(lc_op op, uint64_t low, int64_t high) {
    LiquidExpr e;
    e.pred.op = op;
    e.pred.lit_kind = LC_LIT_I128;
    e.pred.lit_u64 = low;
    e.pred.lit_i64 = high;
    return e;
  }
  static LiquidExpr compare_bytes(lc_op op, std::string v) {
    LiquidExpr e;
    e.bytes = std::move(v);
    e.pred.op = op;
    e.pred.lit_kind = LC_LIT_BYTES;
    e.pred.lit_bytes = reinterpret_cast<const uint8_t*>(e.bytes.data());
    e.pred.lit_len = e.bytes.size();
    return e;
  }
  static LiquidExpr like(std::string pattern, bool negated = false) {
    return compare_bytes(negated ? LC_OP_NOT_LIKE : LC_OP_LIKE, std::move(pattern));
  }
  // `col [NOT] IN (values)` (InListExpr; the reference's LiquidExpr does not admit it): integer / date / timestamp columns
  static LiquidExpr in_list_i64(const std::vector<int64_t>& values, bool negated = false) {
    return in_list_words(LC_LIT_I64, values.data(), values.size(), negated);
  }
  static LiquidExpr in_list_u64(const std::vector<uint64_t>& values, bool negated = false) {
    return in_list_words(LC_LIT_U64, values.data(), values.size(), negated);
  }
  // byte-like columns: the values in Arrow's Utf8 layout, int32 offsets[n + 1] then the bytes
  static LiquidExpr in_list_bytes(const std::vector<std::string>& values, bool negated = false) {
    LiquidExpr e;
    e.pred.op = negated ? LC_OP_NOT_IN : LC_OP_IN;
    e.pred.lit_kind = LC_LIT_BYTES;
    e.pred.lit_len = values.size();
    int32_t off = 0;
    e.bytes.append(reinterpret_cast<const char*>(&off), 4);
    for (const std::string& v : values) {
      off += static_cast<int32_t>(v.size());
      e.bytes.append(reinterpret_cast<const char*>(&off), 4);
    }
    for (const std::string& v : values) e.bytes += v;
    e.native();
    return e;
  }

 private:
  static LiquidExpr in_list_words(int32_t kind, const void* words, size_t n, bool negated) {
    LiquidExpr e;
    e.pred.op = negated ? LC_OP_NOT_IN : LC_OP_IN;
    e.pred.lit_kind = kind;
    e.pred.lit_len = n;
    e.bytes.assign(static_cast<const char*>(words), n * 8);  // little-endian hosts: the words as they are in memory
    e.native();
    return e;
  }
};

struct BooleanArray {
  std::vector<uint8_t> values, validity;
  uint64_t len = 0, null_count = 0;
};

class LiquidCache;

class Insert {
 public:
  Insert(LiquidCache* c, EntryID id, const ArrowSchema* s, const ArrowArray* a) : c_(c), id_(id), s_(s), a_(a) {}
  Insert& with_skip_gc() { return *this; }
  Insert& with_squeeze_hint(lc_hint h) { hint_ = h; return *this; }
  void run();
 private:
  LiquidCache* c_; EntryID id_; const ArrowSchema* s_; const ArrowArray* a_; lc_hint hint_ = LC_HINT_NONE;
};

class Get {
 public:
  Get(LiquidCache* c, EntryID id) : c_(c), id_(id) {}
  Get& with_selection(const BooleanBuffer& sel) { sel_ = sel; return *this; }
  // false = entry absent (Option::None); otherwise out_schema/out_array own the result
  bool read(ArrowSchema* out_schema, ArrowArray* out_array);
 private:
  LiquidCache* c_; EntryID id_; BooleanBuffer sel_;
};

class EvaluatePredicate {
 public:
  EvaluatePredicate(LiquidCache* c, EntryID id, const LiquidExpr& e) : c_(c), id_(id), e_(e) {}
  EvaluatePredicate& with_selection(const BooleanBuffer& sel) { sel_ = sel; return *this; }
  bool read(BooleanArray* out);
 private:
  LiquidCache* c_; EntryID id_; LiquidExpr e_; BooleanBuffer sel_;
};

class LiquidCache {
 public:
  LiquidCache(int device, uint64_t max_memory_bytes, size_t batch_size) : batch_size_(batch_size) {
    check(lc_ctx_create(device, max_memory_bytes, &ctx_));
  }
  ~LiquidCache() { lc_ctx_destroy(ctx_); }
  LiquidCache(const LiquidCache&) = delete;
  LiquidCache& operator=(const LiquidCache&) = delete;

  Insert insert(EntryID id, const ArrowSchema* schema, const ArrowArray* array) { return Insert(this, id, schema, array); }
  Get get(EntryID id) { return Get(this, id); }
  EvaluatePredicate eval_predicate(EntryID id, const LiquidExpr& expr) { return EvaluatePredicate(this, id, expr); }
  bool is_cached(EntryID id) const { return lc_cache_is_cached(ctx_, id) != 0; }
  void reset() { check(lc_cache_reset(ctx_)); }
  size_t batch_size() const { return batch_size_; }
  lc_stats stats() const { lc_stats s{}; check(lc_ctx_stats(ctx_, &s)); return s; }
  lc_ctx* raw() const { return ctx_; }
 private:
  lc_ctx* ctx_ = nullptr;
  size_t batch_size_;
};

class LiquidCacheBuilder {
 public:
  LiquidCacheBuilder& with_batch_size(size_t n) { batch_size_ = n; return *this; }
  LiquidCacheBuilder& with_max_memory_bytes(uint64_t n) { max_memory_ = n; return *this; }
  LiquidCacheBuilder& with_device(int d) { device_ = d; return *this; }
  // cache / hydration / squeeze policies, disk store: CPU-tier knobs of the reference, no effect on an HBM cache
  LiquidCache* build() { return new LiquidCache(device_, max_memory_, batch_size_); }
 private:
  size_t batch_size_ = 8192; uint64_t max_memory_ = 0; int device_ = 0;
};

inline void Insert::run() { check(lc_cache_insert(c_->raw(), id_, s_, a_, hint_)); }

inline bool Get::read(ArrowSchema* out_schema, ArrowArray* out_array) {
  if (!c_->is_cached(id_)) return false;
  check(lc_cache_get(c_->raw(), id_, sel_.bits, sel_.len, out_schema, out_array));
  return true;
}

inline bool EvaluatePredicate::read(BooleanArray* out) {
  if (!c_->is_cached(id_)) return false;
  lc_handle h;
  check(lc_cache_handles(c_->raw(), &id_, 1, &h));
  const uint64_t nb = lc_mask_bytes(lc_len(c_->raw(), h));
  out->values.assign(nb, 0);
  out->validity.assign(nb, 0);
  check(lc_cache_eval_predicate(c_->raw(), id_, e_.native(), sel_.bits, sel_.len, out->values.data(), out->validity.data(),
                                &out->len, &out->null_count));
  return true;
}

}  // namespace liquid_cache

/*
 * lc_gpu.h — C ABI of the H100-native liquid-cache hot path.
 *
 * This is the drop-in boundary for ONE path of XiangpengHao/liquid-cache: the
 * insert() transcode Arrow -> liquid, and get() / with_selection() /
 * eval_predicate() on liquid columns, with the liquid columns resident in HBM
 * and every array-sized loop running as a hand-written sm_90a CUDA kernel.
 *
 * The reference has no FFI seam; its seam is the Rust trait
 *   trait LiquidArray            src/core/src/liquid_array/mod.rs:82-146
 * and the cache front door
 *   LiquidCache::{insert,get,eval_predicate}   src/core/src/cache/core.rs:122-142
 *   Insert / Get / EvaluatePredicate builders  src/core/src/cache/builders.rs:162-356
 * Each entry point below names the reference item it stands in for. The Rust
 * side binding (a `GpuLiquidArray: LiquidArray` adapter) is in INTEGRATION.md.
 *
 * Conventions
 *   - plain C, no C++/torch types; arrays cross as Arrow C Data Interface
 *     structs (borrowed on input, caller-owned on output via `release`).
 *   - every function returns LC_OK (0) or a negative lc_status; nothing
 *     throws or aborts. lc_last_error() gives a thread-local message.
 *   - selections are Arrow BooleanBuffer bytes (LSB-first), bit offset 0,
 *     `sel_len` bits long, NULL meaning "all rows".
 *   - there is NO CPU fallback behind these calls: without a CUDA device
 *     lc_ctx_create() fails with LC_ERR_NO_DEVICE; shapes the kernels do not
 *     cover return LC_ERR_UNSUPPORTED_* so the caller can take the reference's
 *     own fallback (byte_view_array/mod.rs:360-361, transcode.rs:155-159).
 *   - one lc_ctx per process per GPU (one process per GPU); entry points are
 *     thread-safe (serialised on the context).
 */
#ifndef LC_GPU_H
#define LC_GPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- Arrow C Data Interface (https://arrow.apache.org/docs/format/CDataInterface.html) ---- */
#ifndef ARROW_C_DATA_INTERFACE
#define ARROW_C_DATA_INTERFACE
#define ARROW_FLAG_DICTIONARY_ORDERED 1
#define ARROW_FLAG_NULLABLE 2
#define ARROW_FLAG_MAP_KEYS_SORTED 4
struct ArrowSchema {
  const char* format;
  const char* name;
  const char* metadata;
  int64_t flags;
  int64_t n_children;
  struct ArrowSchema** children;
  struct ArrowSchema* dictionary;
  void (*release)(struct ArrowSchema*);
  void* private_data;
};
struct ArrowArray {
  int64_t length;
  int64_t null_count;
  int64_t offset;
  int64_t n_buffers;
  int64_t n_children;
  const void** buffers;
  struct ArrowArray** children;
  struct ArrowArray* dictionary;
  void (*release)(struct ArrowArray*);
  void* private_data;
};
#endif

typedef struct lc_ctx lc_ctx;   /* one per process; owns the device, stream, HBM arena      */
typedef uint64_t lc_handle;     /* device-resident liquid column (an `Arc<dyn LiquidArray>`) */

typedef enum lc_status {
  LC_OK = 0,
  LC_ERR_INVALID = -1,           /* bad argument (length mismatch, NULL pointer ...)            */
  LC_ERR_UNSUPPORTED_TYPE = -2,  /* mirrors transcode's Err(array): caller keeps the Arrow array */
  LC_ERR_UNSUPPORTED_EXPR = -3,  /* mirrors try_eval_predicate -> None / LiquidExpr::try_new None */
  LC_ERR_CACHE_FULL = -4,        /* mirrors cache/mod.rs CacheFull                              */
  LC_ERR_NOT_FOUND = -5,         /* entry absent (reference returns Option::None)               */
  LC_ERR_CUDA = -6,
  LC_ERR_OOM = -7,
  LC_ERR_NO_DEVICE = -8
} lc_status;

/* Predicate operator. Reference: ByteViewOperator (byte_view_array/operator.rs:45-52,66-82) and the
 * Operator whitelist of LiquidExpr (cache/liquid_expr.rs:85-127). */
typedef enum lc_op {
  LC_OP_EQ = 0,
  LC_OP_NE = 1,
  LC_OP_LT = 2,
  LC_OP_LE = 3,
  LC_OP_GT = 4,
  LC_OP_GE = 5,
  LC_OP_LIKE = 6,        /* LikeExpr / LikeMatch; literal is the SQL pattern WITH its % signs */
  LC_OP_NOT_LIKE = 7,    /* negated LikeExpr / NotLikeMatch                                    */
  LC_OP_CONST_TRUE = 8,  /* Literal(Boolean(true))  on a byte-like column (helpers.rs:72-78)   */
  LC_OP_CONST_FALSE = 9,
  /* `col [NOT] IN (v1, ..., vn)`: DataFusion's InListExpr over a list without nulls. The reference's LiquidExpr does
   * not admit it (the caller decodes and lets DataFusion evaluate); this library evaluates it on the device.
   *   lit_len   number of list values (0 = empty list: false for IN, true for NOT IN on every valid row)
   *   lit_kind  LC_LIT_I64 / LC_LIT_U64: lit_bytes holds lit_len little-endian 8-byte integers (no alignment needed);
   *             LC_LIT_BYTES: Arrow's Utf8 layout in one buffer, int32 offsets[lit_len + 1] (offsets[0] == 0,
   *             non-decreasing) followed by offsets[lit_len] value bytes (LC_ERR_INVALID when malformed)
   * Null rows give null (value bit 0, validity bit 0); lc_scan_filter turns them into false, as for every conjunct.
   * Duplicates do not matter. Accepted on integer / date / timestamp and byte-view entries; float, decimal, squeezed
   * entries and lists over the caps below return LC_ERR_UNSUPPORTED_EXPR and write nothing. */
  LC_OP_IN = 10,
  LC_OP_NOT_IN = 11
} lc_op;

/* Largest IN list evaluated on the device: values per list, and value bytes of an LC_LIT_BYTES list. */
#define LC_IN_LIST_MAX_VALUES 256
#define LC_IN_LIST_MAX_BYTES 16384

/* CacheExpression hint (cache/expressions.rs:38-53) — only SUBSTRING_SEARCH changes the encoding
 * (it turns on the per-unique 32-bit fingerprints, transcode.rs:165). */
typedef enum lc_hint {
  LC_HINT_NONE = 0, LC_HINT_PREDICATE = 1, LC_HINT_SUBSTRING_SEARCH = 2,
  /* CacheExpression::ExtractDate32 { field } (expressions.rs:40-44, Date32Field): only lc_squeeze looks at these */
  LC_HINT_EXTRACT_YEAR = 3, LC_HINT_EXTRACT_MONTH = 4, LC_HINT_EXTRACT_DAY = 5, LC_HINT_EXTRACT_DAY_OF_WEEK = 6
} lc_hint;

typedef enum lc_literal_kind {
  LC_LIT_I64 = 0,
  LC_LIT_U64 = 1,
  LC_LIT_BYTES = 2,
  LC_LIT_I128 = 3, /* Decimal128/256 literal, unscaled, SAME scale as the column (DataFusion coerces it):
                      lit_u64 = low 64 bits, lit_i64 = high 64 bits (two's complement). A Decimal256 literal that needs more
                      than 128 bits travels as LC_LIT_BYTES: the 32 little-endian bytes of the unscaled integer */
  LC_LIT_F64 = 4   /* Float32/Float64 literal: lit_u64 = IEEE bits of the value as f64 (a Float32 literal is
                      widened exactly by the caller and narrowed back here) */
} lc_literal_kind;

/* `col <op> literal` after DataFusion's coercion (the reference receives the same thing inside a
 * PhysicalExpr; src/core/src/liquid_array/mod.rs:265-280, operator.rs:134-176). */
typedef struct lc_predicate {
  int32_t op;            /* lc_op */
  int32_t lit_kind;      /* lc_literal_kind */
  int64_t lit_i64;       /* LC_LIT_I64: signed ints, Date32/64, Timestamp; LC_LIT_I128: high half */
  uint64_t lit_u64;      /* LC_LIT_U64: unsigned ints; LC_LIT_I128: low half; LC_LIT_F64: f64 bits */
  const uint8_t* lit_bytes; /* LC_LIT_BYTES: Utf8/Binary literal or LIKE pattern */
  uint64_t lit_len;
} lc_predicate;

/* Liquid logical type, numbering of LiquidDataType (liquid_array/mod.rs:52-65). */
typedef enum lc_liquid_type {
  LC_LIQUID_INTEGER = 1,
  LC_LIQUID_FLOAT = 2,     /* LiquidFloatArray: ALP (float_array.rs) */
  LC_LIQUID_FIXED_LEN_BYTE_ARRAY = 3, /* LiquidFixedLenByteArray: Decimal128/256 with values outside u64, u16 dictionary +
                              FSST over the 16 / 32-byte values (fix_len_byte_array.rs). The values are kept in
                              order-preserving byte form, so `col <op> LC_LIT_I128` runs on the dictionary like a byte-view
                              comparison (the reference decodes, filters and compares: LiquidArray default) */
  LC_LIQUID_BYTE_VIEW = 4,
  LC_LIQUID_DECIMAL = 6    /* LiquidDecimalArray: Decimal128/256 whose values fit u64 (decimal_array.rs) */
} lc_liquid_type;

typedef struct lc_stats {
  uint64_t entries;            /* CacheStats.total_entries   (cache/core.rs:68-119) */
  uint64_t hbm_bytes_used;     /* CacheStats.memory_usage_bytes, counted in HBM     */
  uint64_t hbm_bytes_budget;   /* LiquidCacheBuilder::with_max_memory_bytes         */
  uint64_t kernel_launches;    /* our CUDA kernels launched since ctx creation       */
  uint64_t h2d_bytes;
  uint64_t d2h_bytes;
  uint64_t hbm_bytes_reserved; /* what the arena holds from cudaMalloc (live entries + reusable holes): the figure the budget bounds */
} lc_stats;

/* ------------------------------------------------------------------ context ---- */

/* LiquidCacheBuilder::new().with_max_memory_bytes(b).build()  (cache/builders.rs:50-157).
 * device_id: CUDA ordinal. hbm_budget_bytes: 0 = no limit. */
int lc_ctx_create(int device_id, uint64_t hbm_budget_bytes, lc_ctx** out);
void lc_ctx_destroy(lc_ctx* ctx);
/* Run everything on an externally owned cudaStream_t (e.g. torch's current stream) instead of the
 * context's own stream. NULL restores the context stream. */
int lc_ctx_set_stream(lc_ctx* ctx, void* cuda_stream);
int lc_ctx_synchronize(lc_ctx* ctx);
int lc_ctx_stats(lc_ctx* ctx, lc_stats* out);
/* Measurement aid (off by default): while enabled, the byte-view predicate kernel adds, per launch,
 *   out[0] += dictionary entries looked at, out[1] += candidates whose FSST codes were walked,
 *   out[2] += compressed bytes of those candidates
 *   out[4..11] += SM cycles one CTA of the string predicate kernel spent per phase (staging wait, plan, symbol
 *                 tables, candidate gate, code walk, row-section wait, rows, total), summed over CTAs
 * so a benchmark can state the ALGORITHMIC bytes of a scan exactly. Costs a few atomics; never enable it in
 * a timed region. */
int lc_ctx_profile_counters(lc_ctx* ctx, int enable, uint64_t out[16]);
/* Measurement aid: while enabled, every predicate launch (lc_scan_filter / lc_eval_predicate*) is bracketed by a
 * pair of CUDA events recorded on the launching stream immediately around the kernel launch.
 * lc_ctx_last_kernel_ms waits for the most recent one and returns its duration (negative if none). */
int lc_ctx_kernel_timing(lc_ctx* ctx, int enable);
float lc_ctx_last_kernel_ms(lc_ctx* ctx);
const char* lc_last_error(void);
const char* lc_version(void);

/* --------------------------------------------------- LiquidArray-level calls ---- */

/* transcode_liquid_inner_with_hint (cache/transcode.rs:46-290): Arrow -> liquid, into HBM.
 *   ints/dates/timestamps -> LiquidPrimitiveArray::from_arrow_array (primitive_array.rs:159-206)
 *   Float32/Float64 -> LiquidFloatArray::from_arrow_array (ALP; float_array.rs:266-269, 609-751)
 *   Decimal128/256 whose valid values all fit u64 -> LiquidDecimalArray (decimal_array.rs:127-178); other
 *     decimals (the reference's FSST LiquidFixedLenByteArray) are declined
 *   Utf8/Binary/Utf8View/BinaryView/Dictionary<UInt16,_> -> LiquidByteViewArray (conversions.rs:260-373)
 * compressor_scope identifies the FSST symbol table to train-or-reuse
 * (with_fsst_compressor_or_train, transcode.rs:16-33; one table per (file,row-group,column)).
 * Anything else returns LC_ERR_UNSUPPORTED_TYPE and the caller keeps the Arrow array. */
int lc_encode(lc_ctx* ctx, const struct ArrowSchema* schema, const struct ArrowArray* array,
              int32_t hint, uint64_t compressor_scope, lc_handle* out);
void lc_release(lc_ctx* ctx, lc_handle h);

uint64_t lc_len(lc_ctx* ctx, lc_handle h);           /* LiquidArray::len                      */
uint64_t lc_memory_size(lc_ctx* ctx, lc_handle h);   /* LiquidArray::get_array_memory_size    */
int32_t lc_data_type(lc_ctx* ctx, lc_handle h);      /* LiquidArray::data_type -> lc_liquid_type */
/* The entry's HBM image (layout: liquid_cache_b200/csrc/entry_layout.h) copied to host memory, and the FSST symbol
 * table its byte-view sections are coded against (2320-byte lc::FsstTable; LC_ERR_INVALID for integer entries).
 * The closest reference call is LiquidArray::to_bytes (liquid_array/mod.rs:116-121); the image is this library's own
 * format, not LQDA (SURVEY section 8f-2). Pass out == NULL to query the size. Used by the insert-parity tests. */
int lc_entry_image(lc_ctx* ctx, lc_handle h, uint8_t* out, uint64_t cap, uint64_t* out_bytes);
int lc_entry_fsst_table(lc_ctx* ctx, lc_handle h, uint8_t* out, uint64_t cap, uint64_t* out_bytes);
/* LiquidArray::original_arrow_data_type, as an Arrow C format string copied into buf. */
int lc_arrow_format(lc_ctx* ctx, lc_handle h, char* buf, size_t buf_len);
/* LiquidArray::to_bytes (liquid_array/mod.rs:116-121): the entry in the reference's serialized form, LQDA
 * (liquid_array/ipc.rs:158-250; primitive_array.rs:603-654, float_array.rs:393-520, decimal_array.rs:180-218,
 * raw/bit_pack_array.rs:181-252), for Integer / Float / Decimal entries — what the reference writes when it spills an
 * entry to disk; byte-view entries in the layout of byte_view_array/serialization.rs:87-220. out == NULL asks for the size. */
int lc_to_bytes(lc_ctx* ctx, lc_handle h, uint8_t* out, uint64_t cap, uint64_t* out_bytes);
/* ipc::read_from_bytes (liquid_array/ipc.rs:252-283) for the same three logical types: an LQDA image becomes an
 * HBM-resident entry (the Arrow type follows from the physical type id / the decimal header). The image is checked
 * (section bounds, bit width, patch indices) and refused with LC_ERR_INVALID instead of panicking. */
int lc_from_bytes(lc_ctx* ctx, const uint8_t* bytes, uint64_t len, lc_handle* out);
/* Byte-view images (byte_view_array/serialization.rs:87-325) need the symbol table of their column chunk, which the
 * reference passes in LiquidIPCContext (ipc.rs:238-249): the table registered under `compressor_scope` is used. */
int lc_from_bytes_scoped(lc_ctx* ctx, const uint8_t* bytes, uint64_t len, uint64_t compressor_scope, lc_handle* out);
/* save_symbol_table / load_symbol_table (raw/fsst_buffer.rs:854-932): count u8, symbol lengths, symbols as u64 LE.
 * load registers the table under a scope that has none yet. */
int lc_ctx_save_symbol_table(lc_ctx* ctx, uint64_t compressor_scope, uint8_t* out, uint64_t cap, uint64_t* out_bytes);
int lc_ctx_load_symbol_table(lc_ctx* ctx, uint64_t compressor_scope, const uint8_t* bytes, uint64_t len);

/* ---- squeezed integer entries --------------------------------------------------------------------------------------
 * LiquidArray::squeeze (liquid_array/mod.rs, primitive_array.rs:389-499): when HBM is the scarce tier an integer entry is
 * replaced by its half-width codes (LiquidPrimitiveClampedArray / LiquidPrimitiveQuantizedArray,
 * hybrid_primitive_array.rs) while the full LQDA image moves behind the caller's SqueezeIoHandler (mod.rs:282-…): host
 * memory or disk. lc_to_arrow / lc_eval_predicate on the squeezed handle answer from the codes when those decide and read
 * the image back (one `read` call for the whole range, like hydrate_full_arrow) when they cannot; the result is always
 * the full entry's. lc_eval_predicate_many takes any mix of full and squeezed (clamp / quantize) entries of one column: a
 * probe pass per squeeze form finds the entries whose codes cannot decide, one pass evaluates the predicate over the whole
 * list, and only those entries are read back and re-evaluated. lc_scan_filter does the same on the device-resident selection
 * (probes run on a copy of it). lc_to_arrow_many and lc_scan_read* take full entries only: rows are read from a squeezed
 * column through lc_to_arrow, entry by entry. */
typedef int (*lc_backing_read)(void* user, uint64_t offset, uint64_t len, uint8_t* dst); /* 0 = ok; SqueezeIoHandler::read */
typedef enum lc_squeeze_policy { LC_SQUEEZE_CLAMP = 0, LC_SQUEEZE_QUANTIZE = 1 } lc_squeeze_policy; /* IntegerSqueezePolicy */
/* Returns the pair of LiquidArray::squeeze: the full bytes (written to bytes_out, *out_bytes long) and the squeezed entry.
 * *out_squeezed == 0 and *out_bytes == 0 is the reference's None: no hint, a Date32 / Timestamp column under a hint
 * that names no date field, an all-null column or one narrower than 8 bits, or a logical type other than Integer. bytes_out == NULL asks for the size only. `h` stays valid; the caller releases it once the bytes
 * are stored (the reference swaps the cache entry). `read` is called under the context lock, on the calling thread. */
int lc_squeeze(lc_ctx* ctx, lc_handle h, int32_t policy, int32_t hint, lc_backing_read read, void* user, uint8_t* bytes_out,
               uint64_t cap, uint64_t* out_bytes, lc_handle* out_squeezed);
/* out[0] = 0 for a full entry, 1 clamp, 2 quantize, 3 date component; out[1] = bit width of the codes; out[2] = bucket
 * width (quantize) or the date field (0 year, 1 month, 2 day, 3 day of week); out[3] = length of the backing image;
 * out[4], out[5] = backing reads / calls answered from the codes, context-wide. */
int lc_squeezed_info(lc_ctx* ctx, lc_handle h, uint64_t out[6]);
/* Date32 / Timestamp columns squeeze — only under an LC_HINT_EXTRACT_* hint — to the one date component the hint names
 * (SqueezedDate32Array, liquid_array/squeezed_date32_array.rs:44-223; `policy` is ignored). lc_to_arrow and
 * lc_eval_predicate on such a handle always read the backing (:430-486). What the codes give without a read:
 *   lossy != 0  SqueezedDate32Array::to_component_array (:276-282): an array of the column's own type whose date has the
 *               stored component (Year -> y-01-01, Month -> 1970-m-01, Day -> 1970-01-d, DayOfWeek -> 1970-01-04 + dow;
 *               timestamps at midnight), so the query's date_part over it gives the component back
 *   lossy == 0  to_component_date32 (:286-294): the component values themselves, typed Date32 */
int lc_squeezed_component(lc_ctx* ctx, lc_handle h, int32_t lossy, struct ArrowSchema* out_schema, struct ArrowArray* out_array);

/* LiquidArray::to_arrow_array (sel_bits == NULL) / LiquidArray::filter(&BooleanBuffer)
 * (primitive_array.rs:350-374, byte_view_array/mod.rs:266-290,421-424). The result has the
 * ORIGINAL arrow type, length popcount(sel), host buffers owned through `release`. */
int lc_to_arrow(lc_ctx* ctx, lc_handle h, const uint8_t* sel_bits, uint64_t sel_len,
                struct ArrowSchema* out_schema, struct ArrowArray* out_array);

/* LiquidArray::try_eval_predicate(&LiquidExpr, &BooleanBuffer) (liquid_array/mod.rs:123-130):
 * apply the selection, then evaluate; output is a BooleanArray of length popcount(sel):
 *   out_values   ceil(out_len/8) bytes, LSB-first   (caller buffer of >= ceil(len/8) bytes)
 *   out_validity same size; may be NULL if the caller does not want it
 *   *out_null_count  nulls among the selected rows (0 => validity is all ones)
 * Value bits under a null are written as 0 (the reference leaves them unspecified). */
int lc_eval_predicate(lc_ctx* ctx, lc_handle h, const lc_predicate* pred, const uint8_t* sel_bits,
                      uint64_t sel_len, uint8_t* out_values, uint8_t* out_validity, uint64_t* out_len,
                      uint64_t* out_null_count);

/* Batched forms — same semantics per element, ONE launch sequence for all entries. This is how a
 * scan over a row group (or a whole column) should call in: 8192-row entries are too small to
 * amortise a launch each.
 *   sel_bits[i]   NULL = all rows of entry i (sel_bits itself may be NULL = all rows everywhere)
 *   out_values    caller buffer; entry i's mask starts at byte out_byte_offsets[i] (the caller
 *                 reserves lc_mask_bytes(len_i) = ceil(len_i/8) rounded up to 16 bytes per entry)
 *   out_validity  same layout, may be NULL
 *   out_len[i], out_null_count[i] as above
 *   out_true_count[i]  (may be NULL) set bits of mask i with nulls counted as false — what the caller's
 *                 `count_set_bits()` early-exit (liquid_cache_reader.rs:308-311) would compute
 * When the offsets are ascending and 4-byte aligned the call may write anywhere inside
 * [out_byte_offsets[0], out_byte_offsets[n-1] + lc_mask_bytes(len_{n-1})): the result moves in one copy
 * (straight from the device if the buffers are page-locked). */
uint64_t lc_mask_bytes(uint64_t n_rows);
int lc_eval_predicate_many(lc_ctx* ctx, const lc_handle* handles, uint64_t n, const lc_predicate* pred,
                           const uint8_t* const* sel_bits, uint8_t* out_values, uint8_t* out_validity,
                           const uint64_t* out_byte_offsets, uint64_t* out_len, uint64_t* out_null_count,
                           uint64_t* out_true_count);

/* Batched get-with-selection: the filtered arrays of all entries CONCATENATED into one Arrow array
 * (in `handles` order) — what LiquidCacheReader::read_from_cache + concat produce for one column
 * (src/datafusion/src/reader/runtime/liquid_cache_reader.rs:342-391). All handles must share the
 * original arrow type. */
int lc_to_arrow_many(lc_ctx* ctx, const lc_handle* handles, uint64_t n, const uint8_t* const* sel_bits,
                     struct ArrowSchema* out_schema, struct ArrowArray* out_array);

/* boolean_buffer_and_then(left, right) (src/datafusion/src/utils.rs:62-236, the BMI2 PDEP routine):
 * out bit p = left[p] & right[rank_left(p)]; right has popcount(left) bits. out has left_len bits. */
int lc_and_then(lc_ctx* ctx, const uint8_t* left_bits, uint64_t left_len, const uint8_t* right_bits,
                uint64_t right_len, uint8_t* out_bits);

/* ---------------------------------------------------- LiquidCache-level calls ---- */

/* LiquidCache::insert(entry_id, array) (cache/core.rs:122-128, builders.rs:193-204). Transcodes
 * eagerly into HBM. LC_ERR_UNSUPPORTED_TYPE: caller keeps the array (reference keeps MemoryArrow).
 * LC_ERR_CACHE_FULL mirrors Result<(), CacheFull>. entry_id packs file<<48|rg<<32|col<<16|batch
 * (src/datafusion/src/cache/id.rs:15-22); the FSST table scope is entry_id with batch cleared. */
int lc_cache_insert(lc_ctx* ctx, uint64_t entry_id, const struct ArrowSchema* schema,
                    const struct ArrowArray* array, int32_t hint);
/* The same insert for a LIST of batches (e.g. every batch of a row group, one or several columns): entry_ids[i] gets
 * arrays[i]. Integer / date / timestamp batches are transcoded in one pass (one upload, two kernels over the whole
 * list, two synchronisations per call instead of per batch); other types are transcoded batch by batch. All or
 * nothing: on an error no entry of the list is inserted. The reference inserts batch by batch from
 * LiquidCacheReader (cache/core.rs:122-128); this is the batched form of that loop. */
int lc_cache_insert_many(lc_ctx* ctx, const uint64_t* entry_ids, uint64_t n, const struct ArrowSchema* const* schemas,
                         const struct ArrowArray* const* arrays, int32_t hint);
int lc_cache_is_cached(lc_ctx* ctx, uint64_t entry_id);                       /* core.rs is_cached */
int lc_cache_remove(lc_ctx* ctx, uint64_t entry_id);
int lc_cache_reset(lc_ctx* ctx);                                              /* core.rs reset     */
/* Resolve entry ids to handles (borrowed; valid until remove/reset). LC_ERR_NOT_FOUND if any absent. */
int lc_cache_handles(lc_ctx* ctx, const uint64_t* entry_ids, uint64_t n, lc_handle* out);
/* cache.get(&id).with_selection(&sel)        (builders.rs:218-276, core.rs:595-634) */
/* Arc<dyn LiquidArray> out of the cache (`LiquidCache::try_read_liquid`, cache/core.rs:243-252): the entry's handle with
 * ONE MORE reference, resolved under the cache lock. The handle stays valid — and keeps answering for the entry as it was
 * when retained — after the id is re-inserted, removed or the cache is reset; give it back with lc_release.
 * (lc_cache_handles returns BORROWED handles for the duration of a scan over entries the caller keeps cached.) */
int lc_cache_retain(lc_ctx* ctx, uint64_t entry_id, lc_handle* out);
int lc_cache_get(lc_ctx* ctx, uint64_t entry_id, const uint8_t* sel_bits, uint64_t sel_len,
                 struct ArrowSchema* out_schema, struct ArrowArray* out_array);
/* cache.eval_predicate(&id, &expr).with_selection(&sel)   (builders.rs:314-356, core.rs:862-930) */
int lc_cache_eval_predicate(lc_ctx* ctx, uint64_t entry_id, const lc_predicate* pred,
                            const uint8_t* sel_bits, uint64_t sel_len, uint8_t* out_values,
                            uint8_t* out_validity, uint64_t* out_len, uint64_t* out_null_count);

/* --------------------------------------------- device-resident scan pipeline ---- */
/* The per-batch loop of LiquidCacheReader::build_predicate_filter + read_from_cache
 * (liquid_cache_reader.rs:297-391) for MANY batches at once, with the running selection kept in
 * HBM between conjuncts: predicate -> nulls-to-false -> boolean_buffer_and_then all stay on device.
 *
 *   lc_scan_begin(n_batches, rows[i])            running selection := all rows
 *   lc_scan_filter(scan, handles[i], pred)       selection := and_then(selection, eval(handles[i]))
 *   lc_scan_filter_or(scan, terms, ...)          selection &= OR of AND groups of such predicates
 *   lc_scan_counts(scan, counts[i])              popcount(selection_i)  (one D2H of n u32)
 *   lc_scan_selection(scan, i, bits)             copy selection of batch i to host
 *   lc_scan_read(scan, handles[i], out)          concatenated get().with_selection(selection_i)
 */
typedef struct lc_scan lc_scan;
int lc_scan_begin(lc_ctx* ctx, uint64_t n_batches, const uint64_t* rows_per_batch, lc_scan** out);
/* running selection := all rows again (reuse one scan object for the next query over the same batches) */
int lc_scan_reset(lc_scan* scan);
/* Optional: seed the running selection of batch i from host bits (RowSelection of the reader). */
int lc_scan_set_selection(lc_scan* scan, uint64_t batch, const uint8_t* sel_bits, uint64_t sel_len);
/* The running selection of ALL batches in one copy each way, for conjuncts the caller evaluates itself (the reference's
 * fallback for shapes LiquidExpr::try_new does not admit, e.g. IN lists: src/datafusion/src/cache/column.rs:143-151).
 * Layout: batch i's bits start at 32-bit word word_offsets[i] (LSB first; padding bits are ignored on load and zero on
 * store); lc_scan_selection_layout reports the offsets (n_batches values) and the total word count. */
int lc_scan_selection_layout(lc_scan* scan, uint64_t* word_offsets, uint64_t* total_words);
int lc_scan_store_selections(lc_scan* scan, uint32_t* out_words, uint64_t n_words);
int lc_scan_load_selections(lc_scan* scan, const uint32_t* words, uint64_t n_words);
int lc_scan_filter(lc_scan* scan, const lc_handle* handles, const lc_predicate* pred);
/* A disjunction over columns as ONE conjunct of the scan: CachedRowGroup::evaluate_selection_with_predicate's
 * multi-column OR (src/datafusion/src/cache/mod.rs:111-150: every leaf evaluated under the same selection, the masks
 * joined with or_kleene), generalised to an OR of AND groups:
 *   selection := selection AND OR_d ( AND_{t in d} (valid_t AND preds[t]) )
 *   handles[t]  n_batches handles of term t's column, in the scan's batch order (several terms may name one column)
 *   preds[t]    anything lc_scan_filter accepts on that column
 *   group[t]    disjunct of term t: non-decreasing, starting at 0, without gaps; NULL = every term its own disjunct
 * A null term is false, which is exact: a DNF row is TRUE under Kleene logic exactly when some disjunct has every term
 * TRUE, and the reader turns null into false. Bad arguments (n_terms == 0, NULL pointers, a malformed group, handles whose
 * row counts differ from the scan's) return LC_ERR_INVALID; a term lc_scan_filter would refuse returns its refusal
 * (LC_ERR_UNSUPPORTED_EXPR). Either way the running selection and its counts are left as they were. Cost: the kernels of
 * every term as lc_scan_filter would launch them, plus one merge kernel per disjunct; nothing crosses PCIe that
 * lc_scan_filter would not move for the same terms. */
int lc_scan_filter_or(lc_scan* scan, uint64_t n_terms, const lc_handle* const* handles, const lc_predicate* preds,
                      const uint32_t* group);
int lc_scan_counts(lc_scan* scan, uint64_t* out_counts, uint64_t* out_total);
int lc_scan_selection(lc_scan* scan, uint64_t batch, uint8_t* out_bits);
int lc_scan_read(lc_scan* scan, const lc_handle* handles, struct ArrowSchema* out_schema,
                 struct ArrowArray* out_array);
/* Same as lc_scan_read but leaves the concatenated result in device memory the CALLER owns (e.g. a
 * torch tensor) so it can be handed to NCCL without touching the host:
 *   fixed-width: values -> d_values (out_rows * width bytes), validity bytes -> d_validity
 *   byte-view:   offsets(int32, out_rows+1) -> d_offsets, bytes -> d_values, validity -> d_validity
 * Call first with all pointers NULL to get the sizes. */
int lc_scan_read_device(lc_scan* scan, const lc_handle* handles, void* d_values, uint64_t values_cap,
                        void* d_offsets, void* d_validity, uint64_t* out_rows, uint64_t* out_value_bytes,
                        uint64_t* out_null_count);
/* lc_scan_read for a consumer ON THE DEVICE (the NCCL gather of the filtered batches to rank 0, SURVEY §8e): the
 * concatenated result of the column stays in the scan's own device buffer — *d_values (value bytes; integers: native
 * values), *d_offsets (byte views: int32[rows + 1]; integers: NULL) — valid until the next read on this scan. Planned on
 * the device like lc_scan_read (one synchronisation, a 64-byte header is all that crosses PCIe). Returns
 * LC_ERR_UNSUPPORTED_EXPR when this read cannot be planned on the device (the first read of a scan, nulls, other types,
 * a result that outgrew the capacities): use lc_scan_read_device then. */
int lc_scan_read_borrowed(lc_scan* scan, const lc_handle* handles, void** d_values, void** d_offsets, uint64_t* out_rows,
                          uint64_t* out_value_bytes);
/* lc_scan_read for a consumer on the device, WITHOUT any host synchronisation: the concatenated result is written into
 * caller-owned device buffers of the stated capacities — d_values (value bytes; integers: native values), d_offsets (byte
 * views: int32[rows + 1], closing offset included; integers: may be NULL) — and a 64-byte lc_read_header into d_header
 * (device memory). Everything is enqueued on the calling thread's stream and the call returns; the caller reads the header
 * after its own synchronisation. overflow != 0 means a capacity was short and NOTHING was written besides the header
 * (rows is still valid: retry with larger buffers). Returns LC_ERR_UNSUPPORTED_EXPR for shapes this path does not plan on
 * the device (nulls, views, dictionaries, floats, decimals). */
typedef struct lc_read_header {
  uint32_t batches_with_rows;
  uint32_t overflow;       /* 0 ok, 1 rows over rows_cap (or internal scratch), 2 bytes over values_cap / 2 GiB */
  uint64_t rows, value_bytes, nulls;
  uint64_t reserved[4];
} lc_read_header;
int lc_scan_read_async(lc_scan* scan, const lc_handle* handles, void* d_values, uint64_t values_cap, void* d_offsets,
                       uint64_t rows_cap, void* d_header);
void lc_scan_end(lc_scan* scan);

#ifdef __cplusplus
}
#endif
#endif /* LC_GPU_H */

// kernels.h — work-item structs and launchers of the sm_90a kernels (host-visible side).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "entry_layout.h"

namespace lc {

// Shared-memory budget of the scan kernels: a fixed control area + the staged entry blob.
constexpr uint32_t kScanFixedSmem = 4608;
constexpr uint32_t kStageCap = 100 * 1024;  // entries larger than this are read straight from global
// Grid of the grid-stride element-wise kernels: 8 resident 256-thread CTAs on each of an H100 SXM's 132 SMs.
constexpr uint32_t kGridStrideCap = 132u * 8u;

enum ScanMode : int32_t {
  MODE_DECODE = 0,  // to_arrow_array / filter: values (+validity) of the selected rows
  MODE_PRED = 1,    // try_eval_predicate: compact mask (+validity) over the selected rows
  MODE_REFINE = 2,  // device pipeline: selection := selection & valid & cmp, full length, in place
};

// One entry of a batched scan: where its blob lives and how much of it to stage. Built once per handle list
// and cached on the device; everything else a scan kernel needs is planned ON THE DEVICE from the blob header.
struct alignas(16) EntryRef {
  const uint8_t* blob;
  uint32_t blob_bytes;
  uint32_t head_bytes;   // byte-view: header .. keys (everything but the compressed values); ints: = blob_bytes
  uint32_t sp_end;       // byte-view: end of header + shared prefix
  uint32_t pk_off;       // byte-view: start of the prefix keys (= end of fingerprints + residuals)
  uint32_t rows_off;     // byte-view: start of validity/keys
  uint32_t rows;
};
static_assert(sizeof(EntryRef) == 32, "EntryRef must be 32 bytes");

constexpr uint64_t kNoSel = ~0ull;  // sel_off value meaning "every row of this entry is selected"

// Per-launch addressing of selections and outputs. Offsets are per entry so outputs can be dense.
struct ScanIo {
  const EntryRef* refs;
  const uint32_t* sel_base;   // selection words of all entries; nullptr = all rows everywhere
  const uint64_t* sel_off;    // per entry: word offset into sel_base, or kNoSel
  void* out_base;             // DECODE: native values; PRED: mask words; REFINE: selection words (may alias sel_base)
  const uint64_t* out_off;    // per entry: DECODE element offset; PRED/REFINE word offset
  uint32_t* valid_base;       // DECODE/PRED: validity words of the output (nullptr = not wanted)
  const uint64_t* valid_off;  // per entry word offset
  uint32_t* counts;           // per entry `counts_stride` u32: [0]=k (REFINE: survivors), [1]=nulls among selected, [2]=bytes
  uint32_t counts_stride;
  uint32_t pad;
  const uint32_t* abort_flag; // device-planned reads: non-zero = a capacity is short, the kernel must not write (nullptr = none)
};

// `col <op> literal` on an integer column, as it crossed the C ABI; lowered to the packed domain per entry
// on the device (u = v - reference against a threshold, or a constant when the literal is outside the window).
struct IntPredDesc {
  int32_t op;        // lc_op EQ..GE, or IN / NOT_IN (the values are then in an IntInList)
  int32_t lit_kind;  // LC_LIT_I64 / LC_LIT_U64 / kLitAboveAll
  int64_t lit_i;
  uint64_t lit_u;
};
// The values of `col [NOT] IN (list)` on an integer column: 64-bit patterns of the column's own domain, sorted in the
// column's order (signed or unsigned) and without duplicates. Device memory (the host build of int_plan.cuh: host memory).
struct IntInList {
  const uint64_t* v;
  uint32_t n;
  uint32_t pad;
};
constexpr int32_t kOpIn = 10, kOpNotIn = 11;  // lc_op LC_OP_IN / LC_OP_NOT_IN
constexpr uint32_t kInListMaxValues = 256;     // LC_IN_LIST_MAX_VALUES
constexpr uint32_t kInListMaxBytes = 16384;    // LC_IN_LIST_MAX_BYTES
// device buffer of one IN list: 8-byte integers, or int32 offsets[n + 1] + value bytes (+ padding)
constexpr uint32_t kInListBlobCap = 4u * (kInListMaxValues + 1u) + kInListMaxBytes + 64u;
constexpr int32_t kLitAboveAll = 7;  // decimal literal beyond u64: larger than every value of the column
constexpr int32_t kLitSentinel = 8;  // squeezed (clamp) entries: "code == all ones of the entry's width", whatever the op says

struct alignas(16) IntMinMaxWork {  // 32 bytes
  const void* values;         // native T[n] in device scratch
  const uint32_t* validity;   // bit-offset-0 validity words or nullptr
  uint64_t* out;              // [0]=min, [1]=max (sign- or zero-extended), [2]=valid count
  uint32_t n;
  uint32_t phys;              // PhysType
};

struct alignas(16) IntPackWork {  // 96 bytes
  const void* values;
  const uint32_t* validity;
  uint8_t* blob;
  uint64_t pack_null_slots;  // != 0: null slots are packed like any other value (ALP floats: the reference encodes
                             // whatever the Arrow buffer holds there, float_array.rs:633-640); 0: they are zeroed
  IntHeader hdr;
};
static_assert(sizeof(IntPackWork) == 96, "IntPackWork must be 96 bytes");

// `in` is read for IN / NOT_IN predicates only.
cudaError_t launch_int_scan(int mode, uint32_t n_entries, const ScanIo& io, const IntPredDesc& pred,
                            uint32_t max_blob_bytes, cudaStream_t s, const IntInList& in = IntInList{});
// Full-length integer predicates (REFINE, PRED over all rows) on lists whose entries all have fields of at most 32 bits:
// register-resident FastLanes unpack, one warp per chunk (k_int_bits.cu). `io.counts`, if set, must be zeroed on the
// stream before the launch; max_rows = rows of the longest entry of the list.
cudaError_t launch_int_bits(int mode, uint32_t n_entries, const ScanIo& io, const IntPredDesc& pred, uint32_t max_rows,
                            cudaStream_t s, const IntInList& in = IntInList{});

cudaError_t launch_int_minmax(const IntMinMaxWork* d_works, uint32_t n_works, cudaStream_t s);
cudaError_t launch_int_pack(const IntPackWork* d_works, uint32_t n_works, cudaStream_t s);

// ---- ALP floats and u64 decimals (k_num.cu) -----------------------------------------------------
// Both ride on the integer blob: a float entry packs its ALP-encoded signed integers (+ a patch list), a decimal
// entry packs the low 64 bits of values known to fit u64. k_int_scan<DECODE> produces the integers of the selected
// rows; the kernels below turn them into the column's own type or compare them.
struct AlpEncResult {        // read back by the host to size the entry blob (one small D2H)
  uint32_t e, f;             // chosen Exponents
  uint32_t n_patches;
  uint32_t first_ok;         // first row that is not a patch (0xFFFFFFFF if every row is one)
  long long min, max;        // of the encoded integers after patched slots took the fill value
  uint32_t pad[2];
};
struct AlpEncIo {
  const void* values;        // native floats, n of them (null slots hold whatever the Arrow buffer held)
  const uint32_t* validity;  // bit-offset-0 words or nullptr; only the sampling of get_best_exponents looks at it
  uint32_t n;
  uint32_t is_f64;
  uint32_t sample_step;      // 0: n <= 1024, the whole array is the sample; else n / 1024 (float_array.rs:719-727)
  uint32_t sample_cnt;       // sampled slots before nulls are dropped
  unsigned long long* sizes; // one per (e, f) pair, in the reference's loop order
  AlpEncResult* res;
  void* enc;                 // n encoded integers (i32 / i64)
  uint32_t* exc_words;       // ceil(n/32) words: bit = row needs a patch
  uint32_t* patch_idx;       // up to n
  void* patch_val;           // up to n native floats
};
cudaError_t launch_alp_encode(const AlpEncIo& io, cudaStream_t s);  // search + encode + patch list; res valid after the stream drains

// After k_int_scan<DECODE> over float entries: integers -> floats in place, then the patches of the selected rows.
// Uses io.refs / sel_base / sel_off / out_base / out_off (element offsets) / counts[0] = rows written per entry.
cudaError_t launch_alp_finish(uint32_t n_entries, const ScanIo& io, uint32_t tbits, cudaStream_t s);

// Float comparison over decoded values (arrow-ord total order), one CTA per entry.
struct FloatCmpIo {
  const EntryRef* refs;
  const void* vals_base;        // decoded floats
  const uint64_t* vals_off;     // per entry element offset
  const uint32_t* vals_counts;  // counts of the decode launch: [e * vals_stride] = values of entry e (PRED only)
  uint32_t vals_stride;
  uint32_t refine;              // 0: PRED (compact mask over the selected rows); 1: REFINE (values cover all rows)
  const uint32_t* and_base;     // PRED: compact validity words of the decode launch (nullptr = none)
  const uint64_t* and_off;
  const uint32_t* sel_base;     // REFINE: running selection, ANDed in (nullptr = all rows)
  const uint64_t* sel_off;
  uint32_t* out_base;           // mask words (PRED) / selection words (REFINE; may alias sel_base)
  const uint64_t* out_off;      // per entry word offset
  uint32_t* counts;             // PRED: [2] = set bits; REFINE: [0] = survivors, [1] = 0
  uint32_t counts_stride;
  int32_t op;                   // lc_op EQ..GE
  long long lit_key;            // total-order key of the literal in the column's float type
};
cudaError_t launch_float_cmp(uint32_t n_entries, const FloatCmpIo& io, uint32_t tbits, cudaStream_t s);

// Decimal128/256 <-> u64. narrow: out[i] = low 64 bits (0 for nulls); *flag |= 1 if a valid value is outside u64.
cudaError_t launch_dec_narrow(const void* d_in, const uint32_t* d_validity, uint32_t n, uint32_t width_bytes,
                              unsigned long long* d_out, uint32_t* d_flag, cudaStream_t s);
cudaError_t launch_dec_widen(const unsigned long long* d_in, uint64_t n, uint32_t width_bytes, void* d_out, cudaStream_t s);

// LQDA patch indices: u32 in the entry, u64 in the file; narrow raises *flag when an index is >= limit.
// squeeze: decoded values -> reference + (clamped offset | bucket index), in place (quantize: limit = bucket_count - 1,
// else limit = sentinel)
cudaError_t launch_squeeze_map(void* d_vals, uint32_t n, uint32_t tbits, unsigned long long ref, uint32_t quantize,
                               unsigned long long limit, unsigned long long bucket_width, cudaStream_t s);
// date-component squeeze: decoded Date32 days (in_bits 32) or Timestamp ticks (in_bits 64, ticks_per_day of the unit) ->
// int32 component per row (field 0 year, 1 month, 2 day, 3 day of week); and back to a date / timestamp with that component
cudaError_t launch_date_component(const void* d_in, uint32_t n, uint32_t in_bits, uint32_t field, long long ticks_per_day,
                                  int32_t* d_out, cudaStream_t s);
cudaError_t launch_date_lossy(const int32_t* d_comp, const uint32_t* d_valid, uint32_t n, uint32_t field, long long ticks_per_day,
                              void* d_out, cudaStream_t s);
cudaError_t launch_widen_u32(const uint32_t* d_in, uint32_t n, unsigned long long* d_out, cudaStream_t s);
cudaError_t launch_narrow_u64(const unsigned long long* d_in, uint32_t n, unsigned long long limit, uint32_t* d_out, uint32_t* d_flag,
                              cudaStream_t s);

// ---- byte-view (string) path -------------------------------------------------------------------
enum StrPredKind : int32_t {
  SP_CONST = 0,     // every unique gets `const_result`
  SP_EQ_SHORT = 1,  // needle suffix <= 7 bytes: decided on PrefixKey alone (comparisons.rs:33-49)
  SP_EQ_LONG = 2,   // length + prefix7 gates, then full compare of the decoded value (comparisons.rs:51-79)
  SP_ORD = 3,       // prefix7 compare, ties decoded and compared in full (comparisons.rs:114-151,351-405)
  SP_ORD_EMPTY = 4, // needle suffix empty: decided on PrefixKey.len (comparisons.rs:371-381)
  SP_LIKE = 5,      // fingerprint gate + substring match on the encoded bytes (comparisons.rs:159-183,600-651)
  SP_IN = 6,        // IN list: every needle planned like SP_EQ_*, looked up by PrefixKey, long ties compared in full
};

constexpr uint32_t kMaxNeedle = 1024;  // needle bytes staged into shared memory

// Predicate on a byte-view column as it crossed the C ABI. The per-entry case analysis (shared prefix vs needle,
// prefix-key shortcut, candidates) happens on the device, from the entry's own header.
struct alignas(16) StrPredDesc {
  int32_t op;            // lc_op (EQ..GE, LIKE, NOT_LIKE)
  uint32_t needle_len;   // full needle (for LIKE: the inner pattern without the % signs)
  uint32_t needle_fp;    // fingerprint of the LIKE needle (fingerprint.rs:19-26)
  uint32_t n_planes;     // distinct trigram bits of the LIKE needle (0 below three bytes): the filter planes the gate ANDs
  unsigned long long needle_bloom[4];  // the same bits as a 256-bit set (entry_layout.h trigram_bit)
  uint8_t planes[32];    // ... and as a list, ascending (needles on the streaming path have at most 29 trigrams)
  const uint8_t* needle; // device: needle bytes padded to 4, then needle_len x u16 KMP failure links
  unsigned long long* prof;  // optional device counters {uniques, candidates, candidate bytes}; nullptr = off
  // streaming LIKE kernel (k_str_like): the needle's Shift-And step table of every FSST symbol table the list uses
  // (512 x 16 bytes each, built per launch by k_like_steps) and each entry's index into them; nullptr = not prepared
  const void* like_steps;
  const uint32_t* entry_table;
  // IN / NOT_IN: `needle` points at the list (int32 offsets[list_n + 1], then the value bytes; sorted, no duplicates)
  // and needle_len is 0 (nothing is staged by the single-needle code)
  uint32_t list_n;
  uint32_t pad_list;
};
// One step table per distinct FSST symbol table of the list: d_tables[t] -> d_steps + t * 512 entries of 16 bytes.
cudaError_t launch_like_steps(const uint64_t* d_tables, uint32_t n_tables, const StrPredDesc& pred, void* d_steps, cudaStream_t s);

cudaError_t launch_str_scan(int mode, uint32_t n_entries, const ScanIo& io, const StrPredDesc& pred,
                            uint32_t max_head_bytes, uint32_t max_unique, uint32_t max_meta_bytes, cudaStream_t s);

// Device-side bookkeeping of a get over a device-resident selection (k_scan_plan.cu): totals the host reads back with
// the result, and the refusal flag the decode kernels honour when a capacity chosen before the counts were known is short.
struct alignas(16) ScanPlanHdr {  // 64 bytes
  uint32_t n_hit;      // entries with surviving rows
  uint32_t overflow;   // 0 ok, 1 rows / dictionary scratch over capacity, 2 bytes over capacity (or past int32 offsets)
  uint64_t rows, bytes, nulls, ulen_words, vwords;
  uint64_t pad;
};
static_assert(sizeof(ScanPlanHdr) == 64, "ScanPlanHdr must be 64 bytes");
cudaError_t launch_scan_plan_rows(const uint32_t* d_counts2, const uint32_t* d_n_unique, uint32_t n, uint64_t cap_rows, uint64_t cap_ulen,
                                  uint64_t* d_row_base, uint64_t* d_vword_off, uint64_t* d_ulen_off, ScanPlanHdr* d_hdr, cudaStream_t s);
cudaError_t launch_scan_plan_bytes(const uint32_t* d_counts4, uint32_t n, uint64_t cap_bytes, uint64_t* d_byte_base,
                                   int32_t* d_out_offsets, ScanPlanHdr* d_hdr, cudaStream_t s);

// get()/filter() for byte-view entries: pass 1 (selected keys, decoded lengths, local offsets), host prefix
// sums over the per-entry counts, pass 2 (decode, one warp per selected row).
struct StrGatherIo {
  ScanIo io;                 // refs / selections / validity out / counts ([0]=k,[1]=nulls,[2]=decoded bytes)
  uint32_t* row_off_base;    // scratch: per entry k+1 local offsets at row_off_base[row_base[i] + i]
  uint32_t* row_key_base;    // scratch: per entry k dictionary keys at row_key_base[row_base[i]]  (0xFFFFFFFF = null)
  uint32_t* ulen_base;       // scratch: decoded length per unique at ulen_base[ulen_off[i]]
  const uint64_t* row_base;  // per entry: rows selected before it (pass 1: an upper bound layout; pass 2: exact)
  const uint64_t* ulen_off;  // per entry
  // device-planned reads (k_scan_plan.cu): rows that survived per entry (stride 2; entries with none are skipped) and the
  // plan header whose overflow flag makes every CTA return at once. Both nullptr on the host-planned path.
  const uint32_t* k_hint;
  const ScanPlanHdr* plan;
  uint32_t sparse_max;       // device-planned reads: entries with 1..sparse_max survivors take k_str_lengths_sparse (0 = none do)
  uint32_t pad_sparse;
  // pass 2 only
  // entries of which at least as many rows are selected as the dictionary has values: the dictionary is decoded ONCE into
  // dict_scratch + dict_base[e] and the rows copy from there (the reference's to_dict_arrow + cast, byte_view_array/
  // helpers.rs:14-64); dict_base[e] == ~0 (or dict_scratch == nullptr): every selected row decodes its own value
  const uint64_t* dict_base;
  uint8_t* dict_scratch;
  const uint64_t* byte_base; // per entry: decoded bytes before it
  int32_t* out_offsets;      // concatenated offsets (rows + 1)
  uint8_t* out_bytes;        // concatenated values
};

cudaError_t launch_str_lengths(uint32_t n_entries, const StrGatherIo& g, uint32_t max_head_bytes, cudaStream_t s);
cudaError_t launch_str_decode(uint32_t n_entries, const StrGatherIo& g, cudaStream_t s);
// pass 1 for entries with a handful of survivors (device-planned reads of lists without nulls): one warp per entry, straight
// from global memory — no staging of the entry's head for one or two rows
cudaError_t launch_str_lengths_sparse(uint32_t n_entries, const StrGatherIo& g, cudaStream_t s);
// the whole device-planned read of a selective scan as ONE kernel (chained scan across its CTAs; k_str.cu): uses g.io.refs /
// sel_base / sel_off, g.k_hint, g.out_offsets, g.out_bytes; writes *d_hdr (rows, bytes, overflow); d_status is
// (ceil(n_entries / 8) + 1) x 8 bytes of scratch
cudaError_t launch_str_read_onepass(uint32_t n_entries, const StrGatherIo& g, uint64_t cap_rows, uint64_t cap_bytes, ScanPlanHdr* d_hdr,
                                    unsigned long long* d_status, cudaStream_t s);

// ---- FSST compression at insert ----------------------------------------------------------------
struct alignas(16) FsstEncTable {
  // Greedy longest-match lookup used by the compress kernel. Built on the host at training time.
  //   long symbols (3..8 bytes): open-addressed hash on the first 3 bytes, one symbol per slot
  //   short symbols: 65536-entry table indexed by the next two bytes -> code | len<<8 (len 1 or 2),
  //                  or 0xFFFF... escape marker
  uint64_t hash_sym[2048];
  uint16_t hash_meta[2048];   // code | len<<8 ; 0 = empty slot
  uint16_t short_code[65536]; // code | len<<8 ; len==0 => escape the byte
  uint16_t one_byte[256];     // code | 1<<8 of the 1-byte symbol for this byte, 0 = none (last-byte fallback)
};

// ---- byte-view insert on the device (k_str_encode.cu) -------------------------------------------------
// Rows arrive as (offset, length) pairs into one uploaded byte pool plus an optional validity bitmap.
struct StrEncResult {      // read back by the host to size the entry blob (one small D2H)
  uint32_t n_unique;
  uint32_t shared_prefix_len;
  uint32_t null_count;
  uint32_t max_value_len;
  uint32_t offset_bytes;   // CompactOffsets residual width 1/2/4
  uint32_t comp_bytes;
  int32_t slope, intercept;
  unsigned long long uncompressed_bytes;
  uint32_t error;          // 1 = more than 65536 distinct values, 2 = compressed dictionary over 4 GiB
  uint32_t pad;
};

struct StrEncIo {
  const uint8_t* pool;
  const uint32_t* row_off;
  const uint32_t* row_len;
  const uint32_t* valid;     // n bits, nullptr = no nulls
  uint32_t n;
  uint32_t table_mask;       // dictionary hash table capacity - 1 (power of two >= 2n)
  uint32_t* row_slot;        // n: hash slot of the row's value; later the unique id of leader rows
  uint32_t* table;           // capacity: smallest row index holding the slot's value (0xFFFFFFFF = empty)
  uint32_t* leader;          // n: first row with the same value (0xFFFFFFFF for null rows)
  uint16_t* keys;            // n (null rows hold 0)
  uint32_t* uniq_row;        // U: row of the unique's first occurrence, in first-occurrence order
  uint32_t* clen;            // U compressed lengths
  uint32_t* offsets;         // U + 1
  unsigned long long* pkeys; // U PrefixKeys
  uint32_t* fps;             // U fingerprints (nullptr = not requested)
  unsigned long long* blooms;// U x kBloomWords trigram filters, built together with the fingerprints
  uint8_t* comp;             // compressed values, back to back
  uint8_t* resid;            // (U + 1) * offset_bytes
  const FsstEncTable* enc;
  StrEncResult* res;
};
// Enqueues the whole pipeline (dictionary -> keys -> compress -> offsets fit); `res` is valid once the stream drains.
cudaError_t launch_str_encode(const StrEncIo& io, cudaStream_t s);
// The same five stages over a list of batches (one work item per batch in device memory); see k_str_encode.cu.
cudaError_t launch_str_encode_many(const StrEncIo* d_ios, uint32_t n_batches, uint32_t max_n, uint32_t* d_tables,
                                   size_t table_words, cudaStream_t s);

// Laying out the entry blobs of a batched insert: one work item per batch, up to 9 sections copied from the encode
// pipeline's work areas into the blob (dst offsets 16-byte aligned), the gap behind each section zero-filled up to the
// next one, the 128-byte header written from the work item. One launch instead of ten async calls per batch.
struct alignas(16) StrAsmSeg {
  const uint8_t* src;
  uint32_t dst_off;
  uint32_t bytes;
};
struct alignas(16) StrAsmWork {
  uint8_t* blob;
  uint32_t blob_bytes;
  uint32_t n_segs;
  StrHeader hdr;
  StrAsmSeg segs[9];  // ascending dst_off
};
cudaError_t launch_str_assemble(const StrAsmWork* d_works, uint32_t n_batches, cudaStream_t s);
// single-batch insert: the trigram rows of the work area (n_unique read from d_res) -> the blob's plane-major section
cudaError_t launch_bloom_planes(const unsigned long long* d_rows, const StrEncResult* d_res, uint32_t* d_planes, cudaStream_t s);

// ---- bit utilities -----------------------------------------------------------------------------
// boolean_buffer_and_then: out[p] = left[p] & right[rank_left(p)]  (datafusion/src/utils.rs:62-236)
cudaError_t launch_gather_nonzero(const uint32_t* d_words, uint64_t n_words, unsigned long long* d_pairs, uint64_t budget,
                                  unsigned long long* d_counter, cudaStream_t s);
cudaError_t launch_scatter_words(const unsigned long long* d_pairs, uint64_t n, uint32_t* d_base, cudaStream_t s);
cudaError_t launch_concat_validity(const uint32_t* d_valid_base, const uint64_t* d_valid_off, const uint64_t* d_row_base,
                                   const uint32_t* d_counts, uint32_t counts_stride, uint32_t n_entries, uint64_t rows,
                                   uint32_t* d_out, cudaStream_t s);
cudaError_t launch_build_views(const int32_t* d_offsets, uint32_t total_bytes, const uint8_t* d_data, const uint32_t* d_validity,
                               uint64_t rows, void* d_views, cudaStream_t s);
// LiquidFixedLenByteArray results: decoded (offsets, bytes) -> values at a fixed stride of `width` bytes, null slots zero
// LiquidFixedLenByteArray insert: n little-endian values of `width` bytes at the start of the pool -> order-preserving form
cudaError_t launch_fixed_to_ordered(uint8_t* d_pool, uint32_t n, uint32_t width, cudaStream_t s);
cudaError_t launch_fixed_from_var(const int32_t* d_offsets, uint32_t total_bytes, const uint8_t* d_data, const uint32_t* d_validity,
                                  uint64_t rows, uint32_t width, void* d_out, cudaStream_t s);
cudaError_t launch_and_then(const uint32_t* d_left, uint32_t left_bits, const uint32_t* d_right, uint32_t* d_out,
                            cudaStream_t s);
// lc_scan_filter_or, end of one disjunct over the scan's selection layout (batch i: word_off[i], rows[i] bits, padded to 4
// words). Not last: acc := (first ? term : acc | term), term := sel & ~acc. Last: sel := (first ? term : acc | term),
// counts[2i] = its popcount, counts[2i + 1] = 0. sel_all: the running selection is every row (sel is only written when
// last). Tail bits and padding come out zero.
cudaError_t launch_sel_or(uint32_t* d_sel, bool sel_all, uint32_t* d_term, uint32_t* d_acc, const uint64_t* d_word_off,
                          const uint32_t* d_rows, uint32_t n, bool first, bool last, uint32_t* d_counts, cudaStream_t s);

}  // namespace lc

// entry_layout.h — HBM layout of a liquid column ("entry blob"), shared by host and device code.
//
// One entry = ONE contiguous, 128-byte aligned allocation in the HBM arena: a fixed header
// followed by 16-byte aligned sections. A scan kernel gets {blob pointer, blob bytes} per entry
// and can stage the whole entry into shared memory with a single TMA bulk copy
// (cp.async.bulk), header included, without a dependent pointer chase.
//
// Integer entries restate LiquidPrimitiveArray<T> + BitPackedArray<U>
//   (src/core/src/liquid_array/primitive_array.rs:122-127, raw/bit_pack_array.rs:11-20):
//   reference value, bit width, validity bitmap, FastLanes-order packed 1024-value chunks.
// Byte-view entries restate LiquidByteViewArray<FsstArray>
//   (src/core/src/liquid_array/byte_view_array/mod.rs:76-89, raw/fsst_buffer.rs:160-383):
//   u16 dictionary keys, 8-byte PrefixKeys, optional u32 fingerprints, CompactOffsets
//   (slope/intercept + 1/2/4-byte residuals), shared prefix, FSST-compressed unique values.
#pragma once
#include <stdint.h>

namespace lc {

constexpr uint32_t kMagicInt = 0x3149514Cu;  // "LQI1"
constexpr uint32_t kMagicStr = 0x3153514Cu;  // "LQS1"
constexpr uint32_t kChunkRows = 1024;        // FastLanes block (bit_pack_array.rs:76-78)
constexpr uint32_t kTileRows = 8192;         // rows one CTA pass covers (= reference batch size)

// Physical type ids follow the reference's IPC numbering (liquid_array/ipc.rs:26-47).
enum PhysType : uint8_t {
  PT_I8 = 0, PT_I16 = 1, PT_I32 = 2, PT_I64 = 3,
  PT_U8 = 4, PT_U16 = 5, PT_U32 = 6, PT_U64 = 7,
  PT_F32 = 8, PT_F64 = 9,
  PT_DATE32 = 10, PT_DATE64 = 11,
  PT_TS_S = 12, PT_TS_MS = 13, PT_TS_US = 14, PT_TS_NS = 15,
};

// ArrowByteType numbering (byte_view_array/mod.rs:113-122).
enum ByteType : uint8_t {
  BT_UTF8 = 0, BT_UTF8_VIEW = 1, BT_DICT16_BINARY = 2, BT_DICT16_UTF8 = 3, BT_BINARY = 4, BT_BINARY_VIEW = 5,
  // not ArrowByteType: LiquidFixedLenByteArray (fix_len_byte_array.rs:26-36), every value 16 / 32 bytes
  BT_DECIMAL128 = 6, BT_DECIMAL256 = 7,
};

struct alignas(16) IntHeader {   // 64 bytes
  uint32_t magic;
  uint8_t phys;        // PhysType
  uint8_t tbits;       // 8/16/32/64: width of the native (and unsigned twin) type
  uint8_t bit_width;   // W in 1..tbits; 0 = entire array null (bit_pack_array.rs:18)
  uint8_t has_nulls;
  uint32_t n;          // rows
  uint32_t n_chunks;   // ceil(n/1024)
  uint64_t reference;  // reference_value (= min over valid rows), raw bits zero-extended
  uint32_t validity_off;  // byte offset of the validity bitmap (0 if !has_nulls)
  uint32_t packed_off;    // byte offset of chunk 0; chunk c at packed_off + c*128*W
  uint32_t blob_bytes;    // total bytes incl. header, multiple of 16
  uint32_t null_count;
  uint32_t is_signed;     // ordering of the logical type
  // ALP floats only (LiquidFloatArray, liquid_array/float_array.rs:230-239): the packed words hold the ALP-encoded
  // signed integers minus `reference`; rows the (e, f) pair cannot represent exactly are patched after decoding.
  uint32_t alp_ef;        // Exponents: e | f << 8
  uint32_t n_patches;
  uint32_t patch_idx_off; // n_patches x u32 row indices, ascending (behind the packed chunks)
  uint32_t patch_val_off; // n_patches x native float
  // squeezed integer entries only (LiquidPrimitiveClampedArray / LiquidPrimitiveQuantizedArray, hybrid_primitive_array.rs):
  // the packed words are half-width CODES — min(offset, sentinel) under Clamp, offset / bucket_width under Quantize. The
  // predicate planner of k_int_scan reads these to compare in the right domain; a quantized entry keeps its bucket width
  // in the two patch offset words above (an integer entry has no patches).
  uint8_t squeeze_kind;   // 0 = a full entry, 1 clamp, 2 quantize
  uint8_t pad8[3];
};
#ifdef __CUDACC__
#define LC_HD __host__ __device__
#define LC_HOST_DEVICE __host__ __device__
#else
#define LC_HD
#define LC_HOST_DEVICE
#endif
LC_HD inline unsigned long long int_bucket_width(const IntHeader& h) {
  return static_cast<unsigned long long>(h.patch_idx_off) | (static_cast<unsigned long long>(h.patch_val_off) << 32);
}
inline void set_int_bucket_width(IntHeader* h, unsigned long long bw) {
  h->patch_idx_off = static_cast<uint32_t>(bw);
  h->patch_val_off = static_cast<uint32_t>(bw >> 32);
}
static_assert(sizeof(IntHeader) == 64, "IntHeader must be 64 bytes");

struct alignas(16) StrHeader {   // 128 bytes
  uint32_t magic;
  uint8_t arrow_type;   // ByteType
  uint8_t has_nulls;
  uint8_t has_fp;       // fingerprints present (hint SubstringSearch)
  uint8_t offset_bytes; // CompactOffsets residual width 1/2/4 (fsst_buffer.rs:311-358)
  uint32_t n;           // rows
  uint32_t n_unique;    // dictionary size U (<= 65536)
  int32_t slope;        // CompactOffsets header (fsst_buffer.rs:267-296)
  int32_t intercept;
  uint32_t shared_prefix_len;
  // sections, in blob order: header | shared prefix | fingerprints | residuals | prefix keys |
  //                          validity | keys | compressed values   (each 16-byte aligned).
  // A LIKE scan stages [header .. residuals] + [validity, keys]; every other predicate stages
  // [header, shared prefix] + [prefix keys] + [validity, keys].
  uint32_t validity_off;      // n bits (0 if !has_nulls)
  uint32_t keys_off;          // n x u16 (null rows hold key 0)
  uint32_t prefix_keys_off;   // U x 8 B {prefix7[7], len}
  uint32_t fp_off;            // U x u32 (0 if !has_fp)
  uint32_t resid_off;         // (U+1) x offset_bytes
  uint32_t shared_prefix_off; // shared_prefix_len bytes
  uint32_t fsst_off;          // compressed unique values, back to back
  uint32_t fsst_bytes;
  uint32_t blob_bytes;
  uint32_t null_count;
  uint32_t max_value_len;     // longest decoded unique value (sizing hint)
  uint64_t uncompressed_bytes;// sum of decoded unique value lengths (RawFsstBuffer.uncompressed_bytes)
  uint64_t table_ptr;         // device pointer to this column-chunk's FsstTable
  uint32_t head_bytes;        // bytes from blob start to the end of the keys (what the scan kernels stage)
  uint32_t sp_end;            // end of the shared prefix section (= fp_off if has_fp else resid_off)
  uint32_t rows_off;          // start of the per-row sections (validity if has_nulls, else keys)
  uint32_t bloom_off;         // trigram filter, 256 bit PLANES of ceil(U/32) words each (bloom_plane_words), between the keys and the compressed values (0 = none)
  uint32_t pad[6];
};
static_assert(sizeof(StrHeader) == 128, "StrHeader must be 128 bytes");

// Private substring pre-filter, built beside the reference's 32-bucket byte fingerprints whenever those are requested
// (SubstringSearch hint): a 256-bit set per dictionary value with bit trigram_bit(b[i], b[i+1], b[i+2]) for every three
// adjacent bytes. A value can only contain a needle if it has all of the needle's trigram bits, so values failing the test
// are skipped WITHOUT walking their codes; values passing it are still matched exactly. Measured on the bench URL column
// (profiles/filter_rates.py): for '%google%' the reference gate passes ~40 % of the dictionary, gate + a 64-bit bigram
// set 5.9 %, gate + this set 0.05 % (true matches 0.017 %). Results are identical by construction; NOT LIKE keeps the
// reference rule "invert only if the reference gate let something through". Needles shorter than three bytes have no
// trigram: their mask is empty and only the reference gate applies.
// Stored plane-major ("bit-sliced"): plane t is a bitmap over the dictionary, bit i = value i has trigram bit t. A needle
// with k distinct trigram bits is tested against the WHOLE dictionary by AND-ing k planes — k * ceil(U/32) coalesced words
// per entry (0.9 KB for '%google%' over 1 752 values) instead of one 32-byte sector per value (56 KB), and the result is
// already the candidate bitmap. Same bits, same false-positive rate, same size (32 U bytes, padded per plane to a word).
constexpr uint32_t kBloomWords = 4;     // x u64 per dictionary value while a set is being BUILT (row-major work area of the insert)
constexpr uint32_t kBloomPlanes = 64u * kBloomWords;
LC_HOST_DEVICE inline uint32_t bloom_plane_words(uint32_t n_unique) { return (n_unique + 31u) >> 5; }
LC_HOST_DEVICE inline unsigned long long bloom_section_bytes(uint32_t n_unique) {
  return 4ull * kBloomPlanes * bloom_plane_words(n_unique);  // a multiple of 1024
}
LC_HOST_DEVICE inline uint32_t trigram_bit(uint32_t a, uint32_t b, uint32_t c) {
  return (((a << 16) | (b << 8) | c) * 0x9E3779B1u) >> 24;  // 0..255
}

// FSST symbol table as the decode kernels see it (fsst-rs Decompressor: <=255 symbols of 1..8 bytes,
// code 255 = escape; raw/fsst_buffer.rs:854-883 is the reference's save format of the same content).
struct alignas(16) FsstTable {
  uint64_t symbols[256];  // little-endian packed symbol bytes; entry 255 unused
  uint8_t lens[256];      // symbol length 1..8; lens[255] = 0
  uint32_t n_symbols;
  uint32_t pad[3];
};
static_assert(sizeof(FsstTable) == 2048 + 256 + 16, "FsstTable layout");

// Unsigned-domain predicate on packed integers: u = v - reference, compared against thr.
enum UCmp : int32_t { UC_FALSE = 0, UC_TRUE = 1, UC_EQ = 2, UC_NE = 3, UC_LT = 4, UC_LE = 5, UC_GT = 6, UC_GE = 7 };

}  // namespace lc

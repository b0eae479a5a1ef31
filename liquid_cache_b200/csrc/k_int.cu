// k_int.cu — frame-of-reference + FastLanes bit-packed integers on sm_90a.
//
// Reference semantics restated (all under /root/reference/src/core/src/liquid_array/):
//   encode  LiquidPrimitiveArray::from_arrow_array   primitive_array.rs:159-206
//           get_bit_width                            ../utils/mod.rs:24-32
//           BitPackedArray::from_primitive           raw/bit_pack_array.rs:71-124
//   decode  BitPackedArray::to_primitive             raw/bit_pack_array.rs:127-169
//           LiquidPrimitiveArray::to_arrow_array     primitive_array.rs:350-368
//   filter / try_eval_predicate                      primitive_array.rs:370-379
//
// Design (H100): one CTA per entry (an 8192-row batch). The CTA pulls the whole entry blob
// (header + validity + packed chunks) into shared memory with ONE TMA bulk copy, then every lane
// decodes "its" row straight out of the FastLanes layout (two shared loads + a funnel shift), so
// rows come out in logical order and selection -> write-offset compaction is a warp ballot plus a
// prefix sum over 32-bit selection words. The comparison runs in the packed domain
// (u = v - reference against a host-precomputed threshold), never materialising the column.
// Purely HBM-bound integer work: no tensor cores.
#include <type_traits>

#include "device_utils.cuh"
#include "kernels.h"
#include "int_plan.cuh"
#include "wspec_math.cuh"
#include "scan_rows.cuh"

namespace lc {

// ------------------------------------------------------------------------------------------------
// FastLanes unified transposed order (crate fastlanes 0.5.0, BitPacking::unchecked_{pack,unpack}):
// a 1024-value block of a T-bit type has LANES = 1024/T lanes; logical index of (row r, lane l) is
//   (r % 8) * 128 + FL_ORDER[r / 8] * 16 + l,  FL_ORDER = {0,4,2,6,1,5,3,7} = 3-bit reversal
// lane l's W-bit fields are concatenated over rows into T-bit words, word k stored at
// packed[LANES * k + l]. Inverting the index map gives a direct random-access decode.
// ------------------------------------------------------------------------------------------------
template <typename U>
struct FL {
  static constexpr uint32_t T = sizeof(U) * 8;
  static constexpr uint32_t LANES = 1024 / T;
  static constexpr uint32_t LOG_O = (T == 64) ? 3 : (T == 32) ? 2 : (T == 16) ? 1 : 0;
};

// Storage-order walk of one 1024-row chunk by one warp: 32 steps, step j touches exactly ONE packed word per
// lane (two when the W-bit field straddles a word) and covers the 32 consecutive logical rows of word order(j):
//   T = 32: step j = packed row r = j, lane = FastLanes lane          -> logical word 4(r%8) + bitrev2(r/8)
//   T = 64: 16 lanes only, so the two half-warps take rows r and r+32 (FL_ORDER[o+4] = FL_ORDER[o]+1 makes the
//           two halves adjacent): j = 8o + s, r = 8(o + 4*half) + s   -> the same word formula
//   T = 16: 64 lanes, two steps per row (lanes 0-31 / 32-63)          -> 4(r%8) + 2(r/8) + half
//   T =  8: 128 lanes, four steps per row                             -> word j
// Compared with decoding "row i" by inverting the index map this needs ~5x fewer instructions per row.
template <typename U>
struct FLOrder {
  __device__ __forceinline__ uint32_t operator()(uint32_t j) const {
    constexpr uint32_t T = sizeof(U) * 8;
    if (T >= 32) return (j & 7u) * 4u + (__brev(j >> 3) >> 30);
    if (T == 16) {
      const uint32_t r = j >> 1;
      return (r & 7u) * 4u + (r >> 3) * 2u + (j & 1u);
    }
    return j;
  }
};

// One packed value for (step j, lane): rows, lanes and the W-bit field position as in the table above.
// The lane's bit stream is read as 32-bit words and the field is cut out with one funnel shift; 64-bit
// columns whose frame-of-reference range fits 32 bits (EventTime, dates, most ids) never touch 64-bit ALU ops.
template <uint32_t T>
__device__ __forceinline__ void fl_row_lane(uint32_t j, uint32_t lane, uint32_t* r, uint32_t* L) {
  if (T == 64) {
    *r = ((j >> 3) + 4u * (lane >> 4)) * 8u + (j & 7u);
    *L = lane & 15u;
  } else if (T == 32) {
    *r = j;
    *L = lane;
  } else if (T == 16) {
    *r = j >> 1;
    *L = (j & 1u) * 32u + lane;
  } else {
    *r = j >> 2;
    *L = (j & 3u) * 32u + lane;
  }
}

// T = 64, W <= 32: value as u32
__device__ __forceinline__ uint32_t fl_step64_lo(const uint32_t* __restrict__ c32, uint32_t j, uint32_t lane, uint32_t W,
                                                 uint32_t mask) {
  uint32_t r, L;
  fl_row_lane<64>(j, lane, &r, &L);
  const uint32_t b = r * W, w = b >> 5, sh = b & 31u;
  // 32-bit word w of lane L lives in 64-bit lane word w/2 (16 lanes interleaved), half w%2
  const uint32_t i0 = ((w >> 1) * 16u + L) * 2u + (w & 1u);
  const uint32_t lo = c32[i0];
  uint32_t hi = 0;
  if (sh + W > 32u) {
    const uint32_t w1 = w + 1u;
    hi = c32[((w1 >> 1) * 16u + L) * 2u + (w1 & 1u)];
  }
  return __funnelshift_r(lo, hi, sh) & mask;
}

// T = 64, W > 32: value as u64 from up to three 32-bit words
__device__ __forceinline__ uint64_t fl_step64_hi(const uint32_t* __restrict__ c32, uint32_t j, uint32_t lane, uint32_t W) {
  uint32_t r, L;
  fl_row_lane<64>(j, lane, &r, &L);
  const uint32_t b = r * W, w = b >> 5, sh = b & 31u;
  auto word = [&](uint32_t x) -> uint32_t { return c32[((x >> 1) * 16u + L) * 2u + (x & 1u)]; };
  const uint32_t w0 = word(w), w1 = word(w + 1u);
  const uint32_t w2 = (sh + W > 64u) ? word(w + 2u) : 0u;
  const uint64_t v = (static_cast<uint64_t>(__funnelshift_r(w1, w2, sh)) << 32) | __funnelshift_r(w0, w1, sh);
  return W < 64u ? (v & ((1ull << W) - 1ull)) : v;
}

// T = 32
__device__ __forceinline__ uint32_t fl_step32(const uint32_t* __restrict__ c32, uint32_t j, uint32_t lane, uint32_t W,
                                              uint32_t mask) {
  const uint32_t b = j * W, k = b >> 5, sh = b & 31u;
  const uint32_t lo = c32[32u * k + lane];
  const uint32_t hi = (sh + W > 32u) ? c32[32u * (k + 1u) + lane] : 0u;
  return __funnelshift_r(lo, hi, sh) & mask;
}

// T = 16 / 8: fields never exceed 16 bits, two narrow loads
template <typename U>
__device__ __forceinline__ uint32_t fl_step_small(const U* __restrict__ chunk, uint32_t j, uint32_t lane, uint32_t W,
                                                  uint32_t mask) {
  constexpr uint32_t T = FL<U>::T, LANES = FL<U>::LANES;
  uint32_t r, L;
  fl_row_lane<T>(j, lane, &r, &L);
  const uint32_t b = r * W, k = b / T, sh = b % T;
  uint32_t v = chunk[LANES * k + L];
  if (sh + W > T) v |= static_cast<uint32_t>(chunk[LANES * (k + 1u) + L]) << (T & 31u);
  return (v >> sh) & mask;
}

// Everything a CTA needs for its entry, resolved from ScanIo.
struct EntryIo {
  const uint32_t* sel;
  void* out;
  uint32_t* out_valid;
  uint32_t* counts;
};

__device__ __forceinline__ EntryIo resolve_io(const ScanIo& io, uint32_t e, uint32_t elem_bytes) {
  EntryIo r;
  r.sel = nullptr;
  if (io.sel_base) {
    const uint64_t so = io.sel_off[e];
    if (so != kNoSel) r.sel = io.sel_base + so;
  }
  r.out = io.out_base ? static_cast<uint8_t*>(io.out_base) + io.out_off[e] * elem_bytes : nullptr;
  r.out_valid = io.valid_base ? io.valid_base + io.valid_off[e] : nullptr;
  r.counts = io.counts ? io.counts + static_cast<size_t>(e) * io.counts_stride : nullptr;
  return r;
}

// The three per-entry offsets of ScanIo, fetched one iteration ahead by threads 0..2 of a persistent CTA so the
// dependent global loads are off the entry's critical path.
__device__ __forceinline__ uint64_t load_io_word(const ScanIo& io, uint32_t e, uint32_t t) {
  if (t == 0) return io.sel_base ? io.sel_off[e] : kNoSel;
  if (t == 1) return io.out_base ? io.out_off[e] : 0ull;
  return io.valid_base ? io.valid_off[e] : 0ull;
}
__device__ __forceinline__ uint64_t load_ref_word(const ScanIo& io, uint32_t e, uint32_t t) {
  return t == 0 ? reinterpret_cast<uint64_t>(io.refs[e].blob) : static_cast<uint64_t>(io.refs[e].blob_bytes);
}
__device__ __forceinline__ EntryIo resolve_io_slot(const ScanIo& io, const uint64_t* slot, uint32_t e, uint32_t elem_bytes) {
  EntryIo r;
  const uint64_t so = slot[0];
  r.sel = (io.sel_base && so != kNoSel) ? io.sel_base + so : nullptr;
  r.out = io.out_base ? static_cast<uint8_t*>(io.out_base) + slot[1] * elem_bytes : nullptr;
  r.out_valid = io.valid_base ? io.valid_base + slot[2] : nullptr;
  r.counts = io.counts ? io.counts + static_cast<size_t>(e) * io.counts_stride : nullptr;
  return r;
}

// ---- the common case without compaction ------------------------------------------------------------
// REFINE (selection &= valid & cmp) and PRED over all rows produce FULL-LENGTH bit words, so no rank / prefix
// sum is needed. Per entry the CTA first writes a 64-row STEP TABLE into shared memory: for storage-order step j
// (and half-warp, for 64-bit lanes) the byte offsets of the one/two/three 32-bit words holding the W-bit field,
// the funnel shift, and where the step's mask word lands. A warp then takes a 1024-row chunk and runs
//   LDS.128 step | 2x LDS field words | SHF | LOP | IADD | ISETP | VOTE | STS (lane 0)
// per 32 rows (~12 instructions; the general path is ~90, the per-step recomputation ~50), and finishes the chunk
// with ONE coalesced pass over its 32 mask words: AND with validity / selection, store, popcount.
// Requires the entry blob staged in shared memory (`chunk0` is a shared-memory pointer).
struct FastStep {
  uint32_t off0, off1, sh, pad;  // byte offsets from the lane's base; funnel shift
};

template <typename U>
__device__ __forceinline__ void build_fast_steps(ScanSmem* sm, uint32_t W) {
  constexpr uint32_t T = FL<U>::T;
  FastStep* tab = reinterpret_cast<FastStep*>(sm->sel);  // 64 x 16 B (the compaction tables are unused here)
  uint32_t* off2 = sm->off;                              // third word, W > 32 only
  if (threadIdx.x < 64u) {
    const uint32_t j = threadIdx.x & 31u, hw = threadIdx.x >> 5;
    FastStep st;
    st.pad = 0;
    uint32_t o2 = 0;
    if (T >= 32) {
      uint32_t r, L;
      fl_row_lane<T>(j, hw * 16u, &r, &L);
      const uint32_t b = r * W, w = b >> 5;
      st.sh = b & 31u;
      const uint32_t nw = (st.sh + W + 31u) >> 5;
      // 32-bit word x of a lane: T=64 -> 64-bit lane word x/2 (16 lanes interleaved), half x%2; T=32 -> row x of 32 lanes
      auto byte_off = [](uint32_t x) -> uint32_t { return T == 64 ? (x >> 1) * 128u + (x & 1u) * 4u : x * 128u; };
      st.off0 = byte_off(w);
      st.off1 = nw > 1u ? byte_off(w + 1u) : st.off0;
      o2 = nw > 2u ? byte_off(w + 2u) : st.off1;
    } else {
      st.off0 = st.off1 = st.sh = 0;
    }
    tab[threadIdx.x] = st;
    off2[threadIdx.x] = o2;
  }
}

template <typename U, int MODE, typename C>
__device__ __forceinline__ void int_bits_fast(const EntryIo& w, const IntHeader* h, const uint8_t* packed,
                                              const uint32_t* valid, const URange<C>& g, ScanSmem* sm, uint32_t& tab_key,
                                              uint32_t* fast_cnt) {
  constexpr uint32_t T = FL<U>::T;
  const uint32_t n = h->n, W = h->bit_width;
  const uint32_t n_words = (n + 31u) >> 5, n_chunks = (n + 1023u) >> 10;
  const uint32_t chunk_bytes = 128u * W;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  uint32_t* out_bits = reinterpret_cast<uint32_t*>(w.out);
  uint32_t* out_valid = (MODE == MODE_PRED && valid) ? w.out_valid : nullptr;
  const uint32_t* sel = w.sel;
  const uint32_t tail = n & 31u;
  // the step table only depends on (T, W): neighbouring entries of a column nearly always share it, and then
  // neither the table nor its barrier is needed again
  const uint32_t key = (T << 8) | W;
  if (tab_key != key) {
    build_fast_steps<U>(sm, W);
    __syncthreads();
    tab_key = key;
  }
  const FastStep* tab = reinterpret_cast<const FastStep*>(sm->sel) + (T == 64 ? (lane >> 4) * 32u : 0u);
  const uint32_t* off2 = sm->off + (T == 64 ? (lane >> 4) * 32u : 0u);
  const uint32_t ordl = FLOrder<U>()(lane);  // lane j keeps the mask word of step j = logical word order(j)
  const uint32_t lane_off = T == 64 ? (lane & 15u) * 8u : lane * 4u;
  const uint32_t mask32 = W >= 32u ? 0xffffffffu : ((1u << W) - 1u);
  const uint64_t mask64 = W >= 64u ? ~0ull : ((1ull << W) - 1ull);
  const uint32_t negmask = g.neg ? kFullMask : 0u;
  uint32_t survivors = 0;
  for (uint32_t c = warp; c < n_chunks; c += 8u) {
    const uint8_t* chunk = packed + c * chunk_bytes;
    const uint32_t lbase = smem_u32(chunk) + lane_off;  // 32-bit shared address: LDS, no 64-bit pointer math
    const uint32_t wi = c * 32u + ordl;  // a permutation inside one 128-byte line: still one coalesced access
    uint32_t sw = kFullMask;  // issued before the step loop: the global load overlaps the 32 steps
    if (sel && wi < n_words) sw = sel[wi];
    uint32_t mine = 0;
    for (uint32_t j0 = 0; j0 < 32; j0 += 8) {
      const uint32_t lrel = lane - j0;
#pragma unroll
      for (uint32_t k = 0; k < 8; ++k) {
        const uint32_t j = j0 + k;
        const FastStep st = tab[j];
        bool hit;
        if (T >= 32) {
          const uint32_t w0 = lds_u32(lbase + st.off0);
          const uint32_t w1 = lds_u32(lbase + st.off1);
          if (sizeof(C) == 8) {
            const uint32_t w2 = lds_u32(lbase + off2[j]);
            const uint64_t u =
                ((static_cast<uint64_t>(__funnelshift_r(w1, w2, st.sh)) << 32) | __funnelshift_r(w0, w1, st.sh)) & mask64;
            hit = (static_cast<C>(u - g.lo)) <= g.span;
          } else {
            const uint32_t u = __funnelshift_r(w0, w1, st.sh) & mask32;
            hit = (static_cast<C>(u - g.lo)) <= g.span;
          }
        } else {
          const uint32_t u = fl_step_small<U>(reinterpret_cast<const U*>(chunk), j, lane, W, mask32);
          hit = (static_cast<C>(u - g.lo)) <= g.span;
        }
        const uint32_t cw = __ballot_sync(kFullMask, hit);
        if (lrel == k) mine = cw;  // no shared-memory store in the loop: the steps of a group can overlap
      }
    }
    if (wi < n_words) {
      uint32_t cw = mine ^ negmask;  // negated ranges flip once per word
      uint32_t vw = valid ? valid[wi] : kFullMask;
      if (wi == n_words - 1u && tail) vw &= (1u << tail) - 1u;  // rows past n in the padded last chunk
      const uint32_t vo = vw;
      cw &= vw & sw;
      out_bits[wi] = cw;
      if (out_valid) out_valid[wi] = vo;
      survivors += __popc(cw);
    }
  }
  if (w.counts) {
    // the survivor count is flushed by thread 0 at the top of the CTA's NEXT round (after the round's closing barrier),
    // so no barrier is spent on it here
    survivors = warp_sum(survivors);
    if (lane == 0 && survivors) atomicAdd(fast_cnt, survivors);
    if (MODE == MODE_PRED && threadIdx.x == 0) {
      w.counts[0] = n;
      w.counts[1] = h->null_count;
    }
  }
}

// ---- width-specialised variant of int_bits_fast -------------------------------------------------------------------
// With the bit width a template parameter the 32 storage-order steps unroll into straight-line code whose word offsets,
// funnel shifts and masks are immediates: no step table in shared memory, no LDS.128 of a table row, no address IADDs,
// and the second field word is only loaded by the steps whose field actually straddles a word. Per 32 rows that is
// ~7.5 instructions (W = 17: 2 LDS on 16 of 32 steps, 1 on the rest) where the table version issues 11-12.
// Geometry (see FLOrder / fl_row_lane): T = 32: step j = packed row j, word k = j*W/32 of lane `lane` at byte 128*k + 4*lane.
// T = 64: 16 lanes of 64-bit words; half-warp h takes row r + 32, i.e. the same shift and 32-bit word index x + W. 32-bit
// word x of lane L sits at byte (x/2)*128 + (x%2)*4 + 8*L, so moving by W words is a constant byte distance when W is even
// and one of two constants (by the parity of x) when W is odd: two per-lane bases cover both.
template <typename U, int MODE, uint32_t W>
__device__ __forceinline__ void int_bits_fast_w(const EntryIo& w, const IntHeader* h, const uint8_t* packed,
                                                const uint32_t* valid, const URange<uint32_t>& g, uint32_t* fast_cnt) {
  constexpr uint32_t T = FL<U>::T;
  static_assert(T == 32 || T == 64, "width-specialised path: 32- and 64-bit columns");
  static_assert(W >= 1 && W <= 32, "width-specialised path: fields of at most 32 bits");
  const uint32_t n = h->n;
  const uint32_t n_words = (n + 31u) >> 5, n_chunks = (n + 1023u) >> 10;
  constexpr uint32_t chunk_bytes = 128u * W;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  uint32_t* out_bits = reinterpret_cast<uint32_t*>(w.out);
  uint32_t* out_valid = (MODE == MODE_PRED && valid) ? w.out_valid : nullptr;
  const uint32_t* sel = w.sel;
  const uint32_t tail = n & 31u;
  const uint32_t ordl = wspec_out_word(lane);  // = FLOrder<U>()(lane) for T >= 32
  const uint32_t negmask = g.neg ? kFullMask : 0u;
  uint32_t survivors = 0;
  for (uint32_t c = warp; c < n_chunks; c += 8u) {
    const uint8_t* chunk = packed + c * chunk_bytes;
    const WspecBases<T, W> bs = wspec_bases<T, W>(smem_u32(chunk), lane);  // wspec_math.cuh: checked on the CPU for every (T, W)
    const uint32_t wi = c * 32u + ordl;
    uint32_t sw = kFullMask;
    if (sel && wi < n_words) sw = sel[wi];
    uint32_t mine = 0;
#pragma unroll
    for (uint32_t j = 0; j < 32; ++j) {
      const uint32_t u = wspec_value<T, W>(bs, j, [](uint32_t a) { return lds_u32(a); });
      const bool hit = (u - g.lo) <= g.span;
      const uint32_t cw = __ballot_sync(kFullMask, hit);
      if (lane == j) mine = cw;
    }
    if (wi < n_words) {
      uint32_t cw = mine ^ negmask;
      uint32_t vw = valid ? valid[wi] : kFullMask;
      if (wi == n_words - 1u && tail) vw &= (1u << tail) - 1u;
      const uint32_t vo = vw;
      cw &= vw & sw;
      out_bits[wi] = cw;
      if (out_valid) out_valid[wi] = vo;
      survivors += __popc(cw);
    }
  }
  if (w.counts) {
    survivors = warp_sum(survivors);
    if (lane == 0 && survivors) atomicAdd(fast_cnt, survivors);
    if (MODE == MODE_PRED && threadIdx.x == 0) {
      w.counts[0] = n;
      w.counts[1] = h->null_count;
    }
  }
}

template <typename U, int MODE>
__device__ __forceinline__ void int_bits_fast_w_dispatch(uint32_t W, const EntryIo& w, const IntHeader* h, const uint8_t* packed,
                                                         const uint32_t* valid, const URange<uint32_t>& g, uint32_t* fast_cnt) {
  switch (W) {
#define LC_W(k) case k: int_bits_fast_w<U, MODE, k>(w, h, packed, valid, g, fast_cnt); break;
    LC_W(1) LC_W(2) LC_W(3) LC_W(4) LC_W(5) LC_W(6) LC_W(7) LC_W(8) LC_W(9) LC_W(10) LC_W(11) LC_W(12) LC_W(13) LC_W(14) LC_W(15) LC_W(16)
    LC_W(17) LC_W(18) LC_W(19) LC_W(20) LC_W(21) LC_W(22) LC_W(23) LC_W(24) LC_W(25) LC_W(26) LC_W(27) LC_W(28) LC_W(29) LC_W(30) LC_W(31)
    default: int_bits_fast_w<U, MODE, 32>(w, h, packed, valid, g, fast_cnt); break;
#undef LC_W
  }
}

template <typename U, int MODE, bool SET>
__device__ __forceinline__ bool int_scan_entry(const EntryIo& w, const IntPredDesc& pred, const IntInList& in, const uint8_t* base,
                                               bool staged, ScanSmem* sm, uint32_t& tab_key, uint32_t* fast_cnt) {
  constexpr uint32_t T = FL<U>::T;
  const IntHeader* h = reinterpret_cast<const IntHeader*>(base);
  const uint32_t W = h->bit_width;
  const U ref = static_cast<U>(h->reference);
  int32_t kind = UC_TRUE;
  uint64_t thr64 = 0;
  if (MODE != MODE_DECODE && !SET) plan_int_pred(h, pred, &kind, &thr64);
  const uint8_t* packed = base + h->packed_off;
  const uint32_t* valid = h->has_nulls ? reinterpret_cast<const uint32_t*>(base + h->validity_off) : nullptr;
  const uint32_t chunk_bytes = 128u * W;
  U* out_vals = reinterpret_cast<U*>(w.out);
  uint32_t* out_bits = reinterpret_cast<uint32_t*>(w.out);
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t n = h->n, nulls = h->null_count;

  if (W == 0) {  // entirely null (bit_pack_array.rs:18): nothing packed; masks are all false, values never read
    auto cmp = [&](uint32_t, uint32_t, uint32_t) -> bool { return false; };
    auto emit = [&](uint32_t, uint32_t dst, uint32_t, uint32_t) { out_vals[dst] = ref; };
    tab_key = 0;
    scan_entry_rows<MODE>(w.sel, n, valid, nulls, out_bits, w.out_valid, w.counts, sm, cmp, emit);
    return false;
  }
  if constexpr (SET) {
    // IN lists on the general row loop, every shape (k_int_bits is their fast path): plan_int_in per entry; a set test
    // looks the packed value up among the slice's offsets in global memory
    tab_key = 0;
    URange<uint64_t> g;
    uint32_t a = 0, b = 0;
    const bool set = plan_int_in<uint64_t>(h, pred.op, in, &g, &a, &b);
    const uint64_t ref64 = window_ref(h);
    const uint32_t mask = W >= 32u ? 0xffffffffu : ((1u << W) - 1u);
    auto val = [&](uint32_t c, uint32_t j) -> uint64_t {
      const uint8_t* chunk = packed + static_cast<size_t>(c) * chunk_bytes;
      if (T == 64 && W > 32u) return fl_step64_hi(reinterpret_cast<const uint32_t*>(chunk), j, lane, W);
      if (T == 64) return fl_step64_lo(reinterpret_cast<const uint32_t*>(chunk), j, lane, W, mask);
      if (T == 32) return fl_step32(reinterpret_cast<const uint32_t*>(chunk), j, lane, W, mask);
      return fl_step_small<U>(reinterpret_cast<const U*>(chunk), j, lane, W, mask);
    };
    auto cmp = [&](uint32_t, uint32_t c, uint32_t j) -> bool {
      const uint64_t u = val(c, j);
      const bool hit = set ? in_sorted<uint64_t>(u, b - a, [&](uint32_t i) { return in.v[a + i] - ref64; }) : (u - g.lo) <= g.span;
      return hit != g.neg;
    };
    auto emit = [&](uint32_t, uint32_t, uint32_t, uint32_t) {};
    scan_entry_rows<MODE>(w.sel, n, valid, nulls, out_bits, w.out_valid, w.counts, sm, cmp, emit, FLOrder<U>());
    return false;
  }
  // full-length bit outputs from a staged entry: no compaction needed
  const bool fast = staged && ((MODE == MODE_REFINE) || (MODE == MODE_PRED && w.sel == nullptr));
  if (fast && MODE != MODE_DECODE) {
    if (T == 64 && W > 32u) {
      int_bits_fast<U, MODE, uint64_t>(w, h, packed, valid, make_range<uint64_t>(kind, thr64), sm, tab_key, fast_cnt);
    } else {
      if constexpr (T >= 32) {
        // 32- and 64-bit columns with fields of at most 32 bits: straight-line code per width (no step table)
        int_bits_fast_w_dispatch<U, (MODE == MODE_DECODE ? MODE_PRED : MODE)>(W, w, h, packed, valid, make_range<uint32_t>(kind, thr64),
                                                                              fast_cnt);
      } else {
        int_bits_fast<U, MODE, uint32_t>(w, h, packed, valid, make_range<uint32_t>(kind, thr64), sm, tab_key, fast_cnt);
      }
    }
    return w.counts != nullptr;  // count deferred
  }
  tab_key = 0;  // the general path reuses the table's shared memory
  if (T == 64 && W > 32u) {
    const URange<uint64_t> g = make_range<uint64_t>(kind, thr64);
    auto val = [&](uint32_t c, uint32_t j) -> uint64_t {
      return fl_step64_hi(reinterpret_cast<const uint32_t*>(packed + static_cast<size_t>(c) * chunk_bytes), j, lane, W);
    };
    auto cmp = [&](uint32_t, uint32_t c, uint32_t j) -> bool { return ((val(c, j) - g.lo) <= g.span) != g.neg; };
    auto emit = [&](uint32_t, uint32_t dst, uint32_t c, uint32_t j) { out_vals[dst] = static_cast<U>(val(c, j) + ref); };
    scan_entry_rows<MODE>(w.sel, n, valid, nulls, out_bits, w.out_valid, w.counts, sm, cmp, emit, FLOrder<U>());
    return false;
  }
  // everything else fits 32 bits in the packed domain
  const uint32_t mask = W >= 32u ? 0xffffffffu : ((1u << W) - 1u);
  const URange<uint32_t> g = make_range<uint32_t>(kind, thr64);
  auto val = [&](uint32_t c, uint32_t j) -> uint32_t {
    const uint8_t* chunk = packed + static_cast<size_t>(c) * chunk_bytes;
    if (T == 64) return fl_step64_lo(reinterpret_cast<const uint32_t*>(chunk), j, lane, W, mask);
    if (T == 32) return fl_step32(reinterpret_cast<const uint32_t*>(chunk), j, lane, W, mask);
    return fl_step_small<U>(reinterpret_cast<const U*>(chunk), j, lane, W, mask);
  };
  auto cmp = [&](uint32_t, uint32_t c, uint32_t j) -> bool { return ((val(c, j) - g.lo) <= g.span) != g.neg; };
  auto emit = [&](uint32_t, uint32_t dst, uint32_t c, uint32_t j) {
    out_vals[dst] = static_cast<U>(static_cast<U>(val(c, j)) + ref);
  };
  scan_entry_rows<MODE>(w.sel, n, valid, nulls, out_bits, w.out_valid, w.counts, sm, cmp, emit, FLOrder<U>());
  return false;
}

// Persistent CTAs: each CTA walks entries blockIdx.x, +gridDim.x, ... with a two-deep TMA pipeline — while the
// warps work on the entry staged in one shared-memory buffer, thread 0 has already issued the bulk copy of the
// CTA's next entry into the other buffer (its own mbarrier, phase = use count parity). Entry fetch latency is
// hidden behind compute instead of being paid once per 8192 rows.
template <int MODE, bool SET>
__global__ void __launch_bounds__(256, 4) k_int_scan(ScanIo io, IntPredDesc pred, uint32_t n_entries, uint32_t stage_bytes, IntInList in) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  ScanSmem* sm = reinterpret_cast<ScanSmem*>(smem_raw);
  uint8_t* stage0 = smem_raw + kScanFixedSmem;

  if (io.abort_flag && *io.abort_flag) return;  // device-planned read whose capacities were short (k_scan_plan.cu)
  const uint32_t G = gridDim.x;
  const bool staged = stage_bytes != 0;  // the host sizes the stage for the largest entry of the launch, or passes 0
  if (threadIdx.x == 0) {
    sm->fcnt[0] = 0;
    sm->fcnt[1] = 0;
    mbar_init(&sm->bar[0], 1);
    mbar_init(&sm->bar[1], 1);
    fence_mbar_init();
    if (staged && blockIdx.x < n_entries) {
      const EntryRef r0 = io.refs[blockIdx.x];
      mbar_expect_tx(&sm->bar[0], r0.blob_bytes);
      tma_bulk_g2s(stage0, r0.blob, r0.blob_bytes, &sm->bar[0]);
    }
  }
  if (threadIdx.x < 3u && blockIdx.x < n_entries) sm->io_slot[0][threadIdx.x] = load_io_word(io, blockIdx.x, threadIdx.x);
  if (threadIdx.x - 3u < 2u && blockIdx.x + G < n_entries) sm->ref_slot[threadIdx.x - 3u] = load_ref_word(io, blockIdx.x + G, threadIdx.x - 3u);
  __syncthreads();
  uint32_t it = 0;
  uint32_t tab_key = 0;   // (T, W) the step table in shared memory was built for; 0 = none
  bool pending = false;   // the previous entry left its survivor count in fcnt[buf ^ 1]
  auto flush_count = [&](uint32_t e_prev, uint32_t slot) {  // thread 0, after the round's closing barrier
    uint32_t* c = io.counts + static_cast<size_t>(e_prev) * io.counts_stride;
    const uint32_t v = sm->fcnt[slot];
    sm->fcnt[slot] = 0;
    if (MODE == MODE_REFINE) {
      c[0] = v;
      c[1] = 0;
    } else {
      c[2] = v;
    }
  };
  for (uint32_t e = blockIdx.x; e < n_entries; e += G, ++it) {
    const uint32_t buf = it & 1u;
    const bool more = e + G < n_entries;
    if (pending && threadIdx.x == 0) flush_count(e - G, buf ^ 1u);
    scan_smem_init(sm);
    if (threadIdx.x == 0 && staged && more) {  // prefetch this CTA's next entry into the other buffer
      const uint32_t nbytes = static_cast<uint32_t>(sm->ref_slot[1]);
      mbar_expect_tx(&sm->bar[buf ^ 1u], nbytes);
      tma_bulk_g2s(stage0 + (buf ^ 1u) * stage_bytes, reinterpret_cast<const void*>(sm->ref_slot[0]), nbytes,
                   &sm->bar[buf ^ 1u]);
    }
    // threads 0..2: io offsets of the next entry; threads 3..4: blob / size of the one after. Both are consumed at
    // the bottom of the iteration, so the global loads have the whole entry to complete.
    uint64_t nx_io = 0;  // consumed at the bottom of the iteration: the load has the whole entry to complete
    if (threadIdx.x < 3u && more) nx_io = load_io_word(io, e + G, threadIdx.x);
    if (threadIdx.x - 3u < 2u && e + 2u * G < n_entries) nx_io = load_ref_word(io, e + 2u * G, threadIdx.x - 3u);
    __syncthreads();
    const uint8_t* base;
    if (staged) {
      mbar_wait(&sm->bar[buf], (it >> 1) & 1u);
      base = stage0 + buf * stage_bytes;
    } else {
      base = io.refs[e].blob;
    }
    const IntHeader* h = reinterpret_cast<const IntHeader*>(base);
    const EntryIo w = resolve_io_slot(io, sm->io_slot[buf], e, MODE == MODE_DECODE ? h->tbits / 8u : 4u);
    switch (h->tbits) {
      case 8: pending = int_scan_entry<uint8_t, MODE, SET>(w, pred, in, base, staged, sm, tab_key, &sm->fcnt[buf]); break;
      case 16: pending = int_scan_entry<uint16_t, MODE, SET>(w, pred, in, base, staged, sm, tab_key, &sm->fcnt[buf]); break;
      case 32: pending = int_scan_entry<uint32_t, MODE, SET>(w, pred, in, base, staged, sm, tab_key, &sm->fcnt[buf]); break;
      default: pending = int_scan_entry<uint64_t, MODE, SET>(w, pred, in, base, staged, sm, tab_key, &sm->fcnt[buf]); break;
    }
    if (threadIdx.x < 3u) sm->io_slot[buf ^ 1u][threadIdx.x] = nx_io;
    else if (threadIdx.x < 5u) sm->ref_slot[threadIdx.x - 3u] = nx_io;
    __syncthreads();  // everyone is done with stage[buf] and the control area before the next round reuses them
  }
  if (pending && threadIdx.x == 0 && it > 0) flush_count(blockIdx.x + (it - 1u) * G, (it - 1u) & 1u);
}

cudaError_t launch_int_scan(int mode, uint32_t n_entries, const ScanIo& io, const IntPredDesc& pred,
                            uint32_t max_blob_bytes, cudaStream_t s, const IntInList& in) {
  if (n_entries == 0) return cudaSuccess;
  const uint32_t stage = max_blob_bytes <= kStageCap ? ((max_blob_bytes + 127u) & ~127u) : 0u;
  // Two stage buffers (prefetch of the CTA's next entry) only while >= 3 CTAs still fit on an SM; wide columns
  // (W = 64: 64 KB per entry) are better off with one buffer per CTA and more CTAs in flight.
  const bool pipelined = stage != 0 && 3u * (kScanFixedSmem + 2u * stage + 1024u) <= 227u * 1024u;
  const uint32_t smem = kScanFixedSmem + (pipelined ? 2u : 1u) * stage;
  static bool attr_set = false;
  static int n_sm = 132;
  if (!attr_set) {
    cudaError_t e;
    for (auto k : {k_int_scan<MODE_DECODE, false>, k_int_scan<MODE_PRED, false>, k_int_scan<MODE_REFINE, false>,
                   k_int_scan<MODE_PRED, true>, k_int_scan<MODE_REFINE, true>}) {
      e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kScanFixedSmem + 2 * kStageCap);
      if (e != cudaSuccess) return e;
    }
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    attr_set = true;
  }
  // pipelined: persistent grid, as many CTAs as fit at once (4 per SM by registers); else one CTA per entry
  uint32_t grid = n_entries;
  if (pipelined) {
    uint32_t per_sm = 4;
    while (per_sm > 1 && per_sm * (smem + 1024u) > 227u * 1024u) --per_sm;
    grid = static_cast<uint32_t>(n_sm) * per_sm;
    if (grid > n_entries) grid = n_entries;
  }
  const bool set = mode != MODE_DECODE && (pred.op == kOpIn || pred.op == kOpNotIn);
  switch (mode) {
    case MODE_DECODE: k_int_scan<MODE_DECODE, false><<<grid, 256, smem, s>>>(io, pred, n_entries, stage, in); break;
    case MODE_PRED:
      if (set) k_int_scan<MODE_PRED, true><<<grid, 256, smem, s>>>(io, pred, n_entries, stage, in);
      else k_int_scan<MODE_PRED, false><<<grid, 256, smem, s>>>(io, pred, n_entries, stage, in);
      break;
    default:
      if (set) k_int_scan<MODE_REFINE, true><<<grid, 256, smem, s>>>(io, pred, n_entries, stage, in);
      else k_int_scan<MODE_REFINE, false><<<grid, 256, smem, s>>>(io, pred, n_entries, stage, in);
      break;
  }
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// encode pass 1: min / max over valid rows (arrow aggregate min/max, primitive_array.rs:160,171)
// ------------------------------------------------------------------------------------------------
template <typename N, bool SIGNED>
__device__ __forceinline__ void minmax_entry(const IntMinMaxWork& w, uint64_t* s_red) {
  const N* v = reinterpret_cast<const N*>(w.values);
  using Wide = typename std::conditional<SIGNED, long long, unsigned long long>::type;
  Wide mn = SIGNED ? static_cast<Wide>(0x7fffffffffffffffLL) : static_cast<Wide>(~0ULL);
  Wide mx = SIGNED ? static_cast<Wide>(0x8000000000000000ULL) : static_cast<Wide>(0);
  uint32_t cnt = 0;
  for (uint32_t i = threadIdx.x; i < w.n; i += blockDim.x) {
    const bool ok = w.validity ? ((w.validity[i >> 5] >> (i & 31u)) & 1u) : true;
    if (ok) {
      const Wide x = static_cast<Wide>(v[i]);
      mn = x < mn ? x : mn;
      mx = x > mx ? x : mx;
      ++cnt;
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const Wide omn = static_cast<Wide>(__shfl_xor_sync(kFullMask, static_cast<unsigned long long>(mn), d));
    const Wide omx = static_cast<Wide>(__shfl_xor_sync(kFullMask, static_cast<unsigned long long>(mx), d));
    mn = omn < mn ? omn : mn;
    mx = omx > mx ? omx : mx;
    cnt += __shfl_xor_sync(kFullMask, cnt, d);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    s_red[warp * 3 + 0] = static_cast<uint64_t>(mn);
    s_red[warp * 3 + 1] = static_cast<uint64_t>(mx);
    s_red[warp * 3 + 2] = cnt;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint64_t total = 0;
    for (uint32_t i = 0; i < blockDim.x / 32; ++i) {
      const Wide omn = static_cast<Wide>(s_red[i * 3 + 0]);
      const Wide omx = static_cast<Wide>(s_red[i * 3 + 1]);
      mn = omn < mn ? omn : mn;
      mx = omx > mx ? omx : mx;
      total += s_red[i * 3 + 2];
    }
    w.out[0] = static_cast<uint64_t>(mn);
    w.out[1] = static_cast<uint64_t>(mx);
    w.out[2] = total;
  }
}

__global__ void __launch_bounds__(256) k_int_minmax(const IntMinMaxWork* __restrict__ works) {
  __shared__ uint64_t s_red[8 * 3];
  const IntMinMaxWork w = works[blockIdx.x];
  switch (w.phys) {
    case PT_I8: minmax_entry<int8_t, true>(w, s_red); break;
    case PT_I16: minmax_entry<int16_t, true>(w, s_red); break;
    case PT_I32: case PT_DATE32: minmax_entry<int32_t, true>(w, s_red); break;
    case PT_U8: minmax_entry<uint8_t, false>(w, s_red); break;
    case PT_U16: minmax_entry<uint16_t, false>(w, s_red); break;
    case PT_U32: minmax_entry<uint32_t, false>(w, s_red); break;
    case PT_U64: minmax_entry<uint64_t, false>(w, s_red); break;
    default: minmax_entry<int64_t, true>(w, s_red); break;  // I64, DATE64, TS_*
  }
}

cudaError_t launch_int_minmax(const IntMinMaxWork* d_works, uint32_t n_works, cudaStream_t s) {
  if (n_works == 0) return cudaSuccess;
  k_int_minmax<<<n_works, 256, 0, s>>>(d_works);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// encode pass 2: (v - reference) -> FastLanes pack, fused; one thread per OUTPUT word, gathering the
// rows whose W-bit fields overlap it (coalesced reads across lanes, no atomics). Null slots are
// zeroed (the reference leaves whatever the Arrow buffer held; Arrow equality ignores them).
// ------------------------------------------------------------------------------------------------
template <typename U>
__device__ __forceinline__ void pack_entry(const IntPackWork& w) {
  constexpr uint32_t T = FL<U>::T, LANES = FL<U>::LANES;
  const IntHeader& h = w.hdr;
  const uint32_t W = h.bit_width, n = h.n;
  if (W == 0) return;
  const U* in = reinterpret_cast<const U*>(w.values);
  U* out = reinterpret_cast<U*>(w.blob + h.packed_off);
  const U ref = static_cast<U>(h.reference);
  const U mask = (W < T) ? static_cast<U>((static_cast<U>(1) << W) - static_cast<U>(1)) : static_cast<U>(~static_cast<U>(0));
  const uint32_t chunk_words = 1024u * W / T;
  const uint32_t total = h.n_chunks * chunk_words;
  for (uint32_t g = threadIdx.x; g < total; g += blockDim.x) {
    const uint32_t c = g / chunk_words, within = g % chunk_words;
    const uint32_t k = within / LANES, l = within % LANES;
    const uint32_t bit0 = k * T;
    const uint32_t r0 = bit0 / W;
    uint32_t r1 = (bit0 + T - 1u) / W;
    if (r1 > T - 1u) r1 = T - 1u;
    U word = 0;
    for (uint32_t r = r0; r <= r1; ++r) {
      const uint32_t idx = c * 1024u + (r & 7u) * 128u + (__brev(r >> 3) >> 29) * 16u + l;
      U val = 0;
      if (idx < n) {
        const bool ok = (w.validity && !w.pack_null_slots) ? ((w.validity[idx >> 5] >> (idx & 31u)) & 1u) : true;
        if (ok) val = static_cast<U>(static_cast<U>(in[idx] - ref) & mask);
      }
      const uint32_t b = r * W;
      if (b >= bit0) word = static_cast<U>(word | static_cast<U>(val << (b - bit0)));
      else word = static_cast<U>(word | static_cast<U>(val >> (bit0 - b)));
    }
    out[g] = word;
  }
}

__global__ void __launch_bounds__(256) k_int_pack(const IntPackWork* __restrict__ works) {
  const IntPackWork& w = works[blockIdx.x];
  const IntHeader& h = w.hdr;
  // header + validity
  if (threadIdx.x < sizeof(IntHeader) / 4) {
    reinterpret_cast<uint32_t*>(w.blob)[threadIdx.x] = reinterpret_cast<const uint32_t*>(&h)[threadIdx.x];
  }
  if (h.has_nulls) {
    uint32_t* dst = reinterpret_cast<uint32_t*>(w.blob + h.validity_off);
    const uint32_t n_words = (h.n + 31u) >> 5;
    const uint32_t padded = (h.packed_off - h.validity_off) / 4;
    for (uint32_t i = threadIdx.x; i < padded; i += blockDim.x) {
      uint32_t v = 0;
      if (i < n_words) {
        v = w.validity[i];
        if (i == n_words - 1u && (h.n & 31u)) v &= (1u << (h.n & 31u)) - 1u;
      }
      dst[i] = v;
    }
  }
  switch (h.tbits) {
    case 8: pack_entry<uint8_t>(w); break;
    case 16: pack_entry<uint16_t>(w); break;
    case 32: pack_entry<uint32_t>(w); break;
    default: pack_entry<uint64_t>(w); break;
  }
}

cudaError_t launch_int_pack(const IntPackWork* d_works, uint32_t n_works, cudaStream_t s) {
  if (n_works == 0) return cudaSuccess;
  k_int_pack<<<n_works, 256, 0, s>>>(d_works);
  return cudaGetLastError();
}

}  // namespace lc

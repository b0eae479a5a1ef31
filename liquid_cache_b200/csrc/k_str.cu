// k_str.cu — byte-view (dictionary + FSST) columns on sm_90a: predicates and get-with-selection.
//
// Reference semantics restated (all under /root/reference/src/core/src/liquid_array/byte_view_array/):
//   try_eval_predicate            mod.rs:357-362, helpers.rs:44-92
//   compare_equals / not_equals   comparisons.rs:21-90
//   compare_with_inner (+prefix)  comparisons.rs:114-151, 351-405, 469-501
//   compare_like_substring        comparisons.rs:159-183, 600-651; fingerprint.rs:19-36
//   dictionary -> rows            comparisons.rs:325-347
//   filter / to_arrow_array       mod.rs:266-290, 421-424; helpers.rs:14-64; ../raw/fsst_buffer.rs:88-119, 642-663
//
// Design (H100): one CTA per entry. Two TMA bulk copies are issued up front: (A) header + dictionary
// metadata (shared prefix, 8-byte prefix keys, fingerprints, offset residuals), (B) validity + u16
// keys. Phase 1 evaluates the predicate ONCE PER DICTIONARY ENTRY on the encoded form (prefix keys /
// fingerprints first, FSST codes walked only for the candidates that survive) into a bitmap in shared
// memory while copy B is still in flight; phase 2 broadcasts the bitmap through the keys with the
// same ballot + prefix-sum selection machinery the integer path uses (scan_rows.cuh).
#include <cstdlib>

#include "../../include/lc_gpu.h"
#include "device_utils.cuh"
#include "kernels.h"
#include "like_math.cuh"
#include "scan_rows.cuh"

namespace lc {

struct StrView {
  const StrHeader* h;
  const uint8_t* sp;
  const uint64_t* pk;
  const uint32_t* fp;
  const uint32_t* planes;  // trigram filter planes (entry_layout.h), always in global memory
  const uint8_t* resid;
  const uint32_t* valid;
  const uint16_t* keys;
  const uint8_t* fsst;  // always in global memory
};

// head: where the header + sections up to head_bytes live (shared or global); blob: global blob.
__device__ __forceinline__ StrView make_view(const uint8_t* head, const uint8_t* blob) {
  StrView v;
  v.h = reinterpret_cast<const StrHeader*>(head);
  v.sp = head + v.h->shared_prefix_off;
  v.pk = reinterpret_cast<const uint64_t*>(head + v.h->prefix_keys_off);
  v.fp = v.h->has_fp ? reinterpret_cast<const uint32_t*>(head + v.h->fp_off) : nullptr;
  v.resid = head + v.h->resid_off;
  v.valid = v.h->has_nulls ? reinterpret_cast<const uint32_t*>(head + v.h->validity_off) : nullptr;
  v.keys = reinterpret_cast<const uint16_t*>(head + v.h->keys_off);
  v.fsst = blob + v.h->fsst_off;
  v.planes = v.h->bloom_off ? reinterpret_cast<const uint32_t*>(blob + v.h->bloom_off) : nullptr;
  return v;
}

// CompactOffsets::get_offset (raw/fsst_buffer.rs:365-368)
__device__ __forceinline__ uint32_t dict_offset(const StrView& v, uint32_t i) {
  int32_t r;
  const uint32_t ob = v.h->offset_bytes;
  if (ob == 1) r = reinterpret_cast<const int8_t*>(v.resid)[i];
  else if (ob == 2) r = reinterpret_cast<const int16_t*>(v.resid)[i];
  else r = reinterpret_cast<const int32_t*>(v.resid)[i];
  return static_cast<uint32_t>(v.h->slope * static_cast<int32_t>(i) + v.h->intercept + r);
}

// Sequential reader over a compressed value: one aligned 8-byte global load per 8 codes, bytes peeled off
// with constant shifts.
struct CodeStream {
  const uint8_t* base;
  uint32_t p, end;
  uint64_t cur;
  __device__ __forceinline__ void init(const uint8_t* fsst, uint32_t start, uint32_t end_) {
    base = fsst;
    p = start;
    end = end_;
    cur = 0;
    if (p < end) cur = *reinterpret_cast<const uint64_t*>(base + (p & ~7u)) >> ((p & 7u) * 8u);
  }
  __device__ __forceinline__ uint32_t next() {
    const uint32_t b = static_cast<uint32_t>(cur) & 0xffu;
    cur >>= 8;
    ++p;
    if ((p & 7u) == 0 && p < end) cur = *reinterpret_cast<const uint64_t*>(base + p);
    return b;
  }
};

// Walk the decoded bytes of one value (thread-serial); f(byte) returns false to stop early.
template <typename F>
__device__ __forceinline__ void decode_visit(const uint8_t* fsst, uint32_t start, uint32_t end,
                                             const uint64_t* s_sym, const uint8_t* s_len, F&& f) {
  CodeStream cs;
  cs.init(fsst, start, end);
  while (cs.p < cs.end) {
    const uint32_t code = cs.next();
    if (code == 255u) {
      if (cs.p >= cs.end) break;
      if (!f(cs.next())) return;
    } else {
      uint64_t sym = s_sym[code];
      const uint32_t l = s_len[code];
      for (uint32_t t = 0; t < l; ++t) {
        if (!f(static_cast<uint32_t>(sym & 0xffu))) return;
        sym >>= 8;
      }
    }
  }
}

__device__ __forceinline__ uint32_t decoded_length(const uint8_t* fsst, uint32_t start, uint32_t end,
                                                   const uint8_t* s_len) {
  CodeStream cs;
  cs.init(fsst, start, end);
  uint32_t n = 0;
  while (cs.p < cs.end) {
    const uint32_t code = cs.next();
    if (code == 255u) {
      if (cs.p >= cs.end) break;
      cs.next();
      ++n;
    } else {
      n += s_len[code];
    }
  }
  return n;
}

// byte-wise lexicographic compare of the decoded value against the needle: -1 / 0 / +1
__device__ __forceinline__ int full_compare(const StrView& v, uint32_t i, const uint64_t* s_sym,
                                            const uint8_t* s_len, const uint8_t* nd, uint32_t m) {
  const uint32_t start = dict_offset(v, i), end = dict_offset(v, i + 1u);
  uint32_t pos = 0;
  int ord = 0;
  decode_visit(v.fsst, start, end, s_sym, s_len, [&](uint32_t b) -> bool {
    if (pos >= m) {
      ord = 1;  // value is longer than the needle and equal so far
      return false;
    }
    const uint32_t nb = nd[pos];
    if (b != nb) {
      ord = b < nb ? -1 : 1;
      return false;
    }
    ++pos;
    return true;
  });
  if (ord == 0 && pos < m) ord = -1;  // value is a proper prefix of the needle
  return ord;
}

// substring test with the needle's KMP failure links (exact, any needle length <= kMaxNeedle)
__device__ __forceinline__ bool contains_needle(const StrView& v, uint32_t i, const uint64_t* s_sym,
                                                const uint8_t* s_len, const uint8_t* nd, const uint16_t* fail,
                                                uint32_t m) {
  const uint32_t start = dict_offset(v, i), end = dict_offset(v, i + 1u);
  uint32_t q = 0;
  bool found = false;
  decode_visit(v.fsst, start, end, s_sym, s_len, [&](uint32_t b) -> bool {
    while (q > 0 && nd[q] != b) q = fail[q - 1u];
    if (nd[q] == b) ++q;
    if (q == m) {
      found = true;
      return false;
    }
    return true;
  });
  return found;
}

__device__ __forceinline__ uint64_t bswap64(uint64_t x) {
  const uint32_t lo = static_cast<uint32_t>(x), hi = static_cast<uint32_t>(x >> 32);
  return (static_cast<uint64_t>(__byte_perm(lo, 0, 0x0123)) << 32) | __byte_perm(hi, 0, 0x0123);
}

__device__ __forceinline__ void load_fsst_table(const FsstTable* t, uint64_t* s_sym, uint8_t* s_len) {
  const uint64_t* gs = t->symbols;
  for (uint32_t i = threadIdx.x; i < 256u; i += blockDim.x) s_sym[i] = gs[i];
  const uint32_t* gl = reinterpret_cast<const uint32_t*>(t->lens);
  uint32_t* sl = reinterpret_cast<uint32_t*>(s_len);
  for (uint32_t i = threadIdx.x; i < 64u; i += blockDim.x) sl[i] = gl[i];
}

// ------------------------------------------------------------------------------------------------
// predicate kernel
// ------------------------------------------------------------------------------------------------
struct EntryIo {
  const uint32_t* sel;
  void* out;
  uint32_t* out_valid;
  uint32_t* counts;
};

__device__ __forceinline__ EntryIo resolve_io(const ScanIo& io, uint32_t e) {
  EntryIo r;
  r.sel = nullptr;
  if (io.sel_base) {
    const uint64_t so = io.sel_off[e];
    if (so != kNoSel) r.sel = io.sel_base + so;
  }
  r.out = io.out_base ? static_cast<uint8_t*>(io.out_base) + io.out_off[e] * 4u : nullptr;
  r.out_valid = io.valid_base ? io.valid_base + io.valid_off[e] : nullptr;
  r.counts = io.counts ? io.counts + static_cast<size_t>(e) * io.counts_stride : nullptr;
  return r;
}

// Per-entry plan, decided on the device from the entry's own shared prefix (thread 0, then broadcast).
// Restates the case analysis of comparisons.rs:21-82 (equality), :351-405 + :469-501 (ordering), :159-183 (LIKE).
struct StrPlan {
  int32_t kind;
  uint32_t flags;       // bit0 const result, bit1 negate, bit2 LIKE without fingerprints (plain semantics)
  uint32_t cmp_len;
  uint32_t pad;
  uint64_t key_expect;
};

// The PrefixKey (prefix7 + length, 255 = "255 or more") a dictionary value equal to the needle nd[0..m) has in an entry
// whose shared prefix is sp[0..spl) (comparisons.rs:33-49). False when the needle does not start with the shared prefix:
// then no value of the entry can equal it.
__device__ __forceinline__ bool eq_prefix_key(const uint8_t* nd, uint32_t m, const uint8_t* sp, uint32_t spl, uint64_t* key) {
  bool has_prefix = m >= spl;
  for (uint32_t i = 0; has_prefix && i < spl; ++i) has_prefix = nd[i] == sp[i];
  if (!has_prefix) return false;
  const uint32_t L = m - spl;
  uint64_t k = 0;
  for (uint32_t b = 0; b < (L < 7u ? L : 7u); ++b) k |= static_cast<uint64_t>(nd[spl + b]) << (8u * b);
  k |= static_cast<uint64_t>(L >= 255u ? 255u : L) << 56;
  *key = k;
  return true;
}

__device__ __forceinline__ void plan_str_pred(const StrView& v, const StrPredDesc& pred, const uint8_t* nd,
                                              StrPlan* out) {
  const int op = pred.op;
  const uint32_t m = pred.needle_len, spl = v.h->shared_prefix_len;
  StrPlan p;
  p.kind = SP_CONST;
  p.flags = 0;
  p.cmp_len = 0;
  p.pad = 0;
  p.key_expect = 0;
  if (op == LC_OP_CONST_TRUE || op == LC_OP_CONST_FALSE) {
    p.flags = (op == LC_OP_CONST_TRUE) ? 1u : 0u;
  } else if (op == LC_OP_EQ || op == LC_OP_NE) {
    const bool neg = (op == LC_OP_NE);
    uint64_t k = 0;
    if (!eq_prefix_key(nd, m, v.sp, spl, &k)) {
      p.flags = neg ? 1u : 0u;  // no value can equal the needle
    } else {
      p.key_expect = k;
      p.kind = (m - spl <= 7u) ? SP_EQ_SHORT : SP_EQ_LONG;
      p.flags = neg ? 2u : 0u;
    }
  } else if (op >= LC_OP_LT && op <= LC_OP_GE) {
    const bool less_op = (op == LC_OP_LT || op == LC_OP_LE);
    const uint32_t c_len = m < spl ? m : spl;
    int c = 0;
    for (uint32_t i = 0; c == 0 && i < c_len; ++i) c = static_cast<int>(v.sp[i]) - static_cast<int>(nd[i]);
    if (c != 0 || m < spl) {
      // compare_with_shared_prefix: decided for the whole dictionary; a needle shorter than the shared
      // prefix is smaller than every value
      const bool res = (c < 0) ? less_op : !less_op;
      p.flags = res ? 1u : 0u;
    } else {
      const uint32_t L7 = (m - spl) < 7u ? (m - spl) : 7u;
      if (L7 == 0) {
        p.kind = SP_ORD_EMPTY;
      } else {
        uint64_t k = 0;
        for (uint32_t b = 0; b < L7; ++b) k |= static_cast<uint64_t>(nd[spl + b]) << (8u * (7u - b));
        p.kind = SP_ORD;
        p.key_expect = k;
        p.cmp_len = L7;
      }
    }
  } else if (op == LC_OP_IN || op == LC_OP_NOT_IN) {  // the needles are planned by all threads (in_list_table)
    p.kind = SP_IN;
    p.flags = op == LC_OP_NOT_IN ? 2u : 0u;
  } else {  // LIKE / NOT LIKE
    p.kind = SP_LIKE;
    p.flags = (op == LC_OP_NOT_LIKE ? 2u : 0u) | (v.h->has_fp ? 0u : 4u);
  }
  *out = p;
}

// ---- substring match directly on FSST codes --------------------------------------------------------
// Shift-And over the needle (m <= 31): state bit j <=> needle[0..j] matches the text ending here; one text
// byte b maps S -> ((S << 1) | 1) & M[b]. That map is linear over OR, so the effect of a whole symbol
// (1..8 bytes) collapses into three masks computed once per CTA from the column chunk's symbol table:
//     S' = ((S << L) & A) | B        and   "the needle completed inside this symbol"  <=>  (S & H) | hit0
// One FSST code then costs one 16-byte shared-memory load and ~6 ALU ops, instead of ~8 bytes x (load,
// compare, branch). Values are never decompressed: this IS the predicate evaluated on the encoded bytes.
// Bit 31 of the state is a constant 1 (needles are <= 31 bytes on this path, B always re-sets it), so "completed
// at the symbol's first bytes regardless of the state" (hit0) is just bit 31 of H and the hit test is one AND.
constexpr uint32_t kLikeWarps = 8;     // warps of the CTA that may walk the candidate queue
constexpr uint32_t kCandPerWarp = 32;  // ... one more warp for every 32 candidates (measured: 96 and 192 are slower)

__device__ __forceinline__ void build_sym_steps(const uint64_t* s_sym, const uint8_t* s_len, const uint8_t* nd,
                                                uint32_t m, uint32_t* s_M, SymStep* s_step) {
  // M[b]: bit j set iff needle[j] == b
  for (uint32_t b = threadIdx.x; b < 256u; b += blockDim.x) {
    uint32_t bits = 0;
    for (uint32_t j = 0; j < m; ++j) bits |= (nd[j] == b ? 1u : 0u) << j;
    s_M[b] = bits;
  }
  __syncthreads();
  // entries 0..254: FSST codes; 255: the escape marker (identity, the next byte is a literal);
  // entries 256..511: a literal byte b (what follows an escape) = a one-byte symbol
  for (uint32_t c = threadIdx.x; c < 512u; c += blockDim.x) {
    const uint64_t sym = c < 256u ? s_sym[c] : static_cast<uint64_t>(c - 256u);
    const uint32_t L = c < 255u ? s_len[c] : (c == 255u ? 0u : 1u);
    s_step[c] = like_sym_step(sym, L, s_M, m);
  }
}

// Lanes pull candidates from a shared queue and each walks its value's codes, eight codes (one aligned 8-byte
// word of the compressed value) per trip. A value is a chain of dependent 8-byte loads, so the walk keeps FOUR words
// per lane in flight: ring register w[R] holds the word of the current trip and is re-requested (word + 4) as soon
// as it has been consumed. Every busy lane advances exactly one word per trip, which makes the ring position
// warp-uniform: the loop body is instantiated for R = 0..3 and the ring is plain registers with static names — no
// moves that would wait on a load in flight. (With one word of lookahead a handful of candidates per entry took as
// long as hundreds: every trip paid a full L2/DRAM latency.) The steps are branch-free (an escape just switches the
// table half used for the following byte) and refills are warp-synchronous — when at least a quarter of the lanes
// are out of work they all take new candidates in one converged pass and go on with the trip.
struct LikeLane {
  uint32_t S, hit, cur_i, pending, p, end;
  uint64_t w[4];
};

template <int R, typename View>
__device__ __forceinline__ bool like_trip(const View& v, const uint16_t* s_cand, uint32_t ncand, uint32_t* queue,
                                          const SymStep* s_step, uint32_t* s_dict, LikeLane& st, bool& exhausted) {
  const int lane = threadIdx.x & 31;
  const uint8_t* base = v.fsst;
  bool idle = (st.p >= st.end) || (st.hit != 0);
  uint32_t idle_mask = __ballot_sync(kFullMask, idle);
  if (idle_mask == kFullMask || (!exhausted && __popc(idle_mask) >= 8)) {
    if (st.hit) {
      atomicOr(&s_dict[st.cur_i >> 5], 1u << (st.cur_i & 31u));
      st.hit = 0;
      st.p = st.end;
    }
    if (exhausted) return false;  // only reached with every lane idle: done
    uint32_t qb = 0;
    if (lane == 0) qb = atomicAdd(queue, static_cast<uint32_t>(__popc(idle_mask)));
    qb = __shfl_sync(kFullMask, qb, 0);
    const uint32_t idx = qb + __popc(idle_mask & lanemask_lt());
    if (idle && idx < ncand) {
      st.cur_i = s_cand[idx];
      st.p = dict_offset(v, st.cur_i);
      st.end = dict_offset(v, st.cur_i + 1u);
      st.S = kStateOne;
      st.pending = 0;
      if (st.p < st.end) {  // request the first four words; the first one is consumed by THIS trip from w[R]
        const uint32_t w0 = st.p & ~7u;
        st.w[R] = *reinterpret_cast<const uint64_t*>(base + w0);
        st.w[(R + 1) & 3] = (w0 + 8u < st.end) ? *reinterpret_cast<const uint64_t*>(base + w0 + 8u) : 0ull;
        st.w[(R + 2) & 3] = (w0 + 16u < st.end) ? *reinterpret_cast<const uint64_t*>(base + w0 + 16u) : 0ull;
        st.w[(R + 3) & 3] = (w0 + 24u < st.end) ? *reinterpret_cast<const uint64_t*>(base + w0 + 24u) : 0ull;
      }
    }
    exhausted = (qb + __popc(idle_mask)) >= ncand;
    idle = (st.p >= st.end);
  }
  // one compressed word: up to eight table steps on w[R], then re-request the word four ahead into w[R]
  const uint32_t word_end = (st.p & ~7u) + 8u;
  const uint32_t lim = word_end < st.end ? word_end : st.end;
  const uint32_t cnt = idle ? 0u : lim - st.p;  // bytes to consume; they sit at byte positions (p & 7) ..
  const uint64_t cur = st.w[R] >> ((st.p & 7u) * 8u);
  if (!idle && word_end + 24u < st.end) st.w[R] = *reinterpret_cast<const uint64_t*>(base + word_end + 24u);
  const uint32_t lo = static_cast<uint32_t>(cur), hi = static_cast<uint32_t>(cur >> 32);
  // any 0xFF byte (escape marker) among the bytes we are about to consume?  (SWAR zero-byte test on ~word)
  const uint32_t nlo = ~lo, nhi = ~hi;
  const uint32_t zlo = (nlo - 0x01010101u) & ~nlo & 0x80808080u, zhi = (nhi - 0x01010101u) & ~nhi & 0x80808080u;
  // bytes beyond cnt may belong to the next value: only the first cnt bytes count
  const uint64_t keep = cnt >= 8u ? ~0ull : ((1ull << (8u * cnt)) - 1ull);
  const uint32_t klo = static_cast<uint32_t>(keep), khi = static_cast<uint32_t>(keep >> 32);
  const bool has_esc = (st.pending != 0u) || (((zlo & klo) | (zhi & khi)) != 0u);
  uint32_t S = st.S, hit = st.hit;
  if (__any_sync(kFullMask, has_esc && cnt != 0u)) {
    // general path: an escape switches the table half used for the following byte
    uint32_t pending = st.pending;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (static_cast<uint32_t>(k) < cnt) {
        const uint32_t b = ((k < 4 ? lo : hi) >> (8 * (k & 3))) & 0xffu;
        const SymStep e = s_step[b + (pending << 8)];
        hit |= S & e.H;
        S = ((S << e.L) & e.A) | e.B;
        pending = (pending == 0u && b == 255u) ? 1u : 0u;
      }
    }
    st.pending = pending;
  } else {
    // fast path (no escape in any lane's word): plain table steps. (Tried and dropped: an 8-word bitmap of the codes
    // that cannot touch the match state, to skip their 16-byte rows — fewer bank conflicts, but the extra lookup
    // cost more than it saved.)
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (static_cast<uint32_t>(k) < cnt) {
        const uint32_t b = ((k < 4 ? lo : hi) >> (8 * (k & 3))) & 0xffu;
        const SymStep e = s_step[b];
        hit |= S & e.H;
        S = ((S << e.L) & e.A) | e.B;
      }
    }
  }
  st.S = S;
  st.hit = hit;
  st.p += cnt;
  return true;
}

template <typename View>
__device__ __forceinline__ void like_candidates(const View& v, const uint16_t* s_cand, uint32_t ncand,
                                                uint32_t* queue, const SymStep* s_step, uint32_t* s_dict) {
  LikeLane st;
  st.S = 0;
  st.hit = 0;
  st.cur_i = 0;
  st.pending = 0;
  st.p = 0;
  st.end = 0;
  st.w[0] = st.w[1] = st.w[2] = st.w[3] = 0;
  bool exhausted = false;  // warp-uniform: the queue has nothing left
  for (;;) {
    if (!like_trip<0>(v, s_cand, ncand, queue, s_step, s_dict, st, exhausted)) break;
    if (!like_trip<1>(v, s_cand, ncand, queue, s_step, s_dict, st, exhausted)) break;
    if (!like_trip<2>(v, s_cand, ncand, queue, s_step, s_dict, st, exhausted)) break;
    if (!like_trip<3>(v, s_cand, ncand, queue, s_step, s_dict, st, exhausted)) break;
  }
}

// A FEW candidates per entry (what the trigram filter leaves of a selective needle): the 32-lane queue above would walk one
// value on one lane, a chain of ~50 dependent table steps, with 31 lanes idle. A step is S' = ((S << L) & A) | B with the hit
// test (S & H) != 0 (bit 31 of S is a constant 1, bit 31 of H means "hits whatever the state"), and two steps in a row are
// again one step of the same form:
//     L = L1 + L2,  A = (A1 << L2) & A2,  B = ((B1 << L2) & A2) | B2,  H = H1 | ((A1 & H2) >> L1) | (B1 & H2 ? bit 31 : 0)
// so the warp takes 32 codes of the value at once, one per lane (escape markers and the literal behind them are told apart
// as in warp_decode), combines the 32 steps in order with five shuffle rounds and applies the result to the running state.
template <typename View>
__device__ __forceinline__ void like_candidates_warp(const View& v, const uint16_t* s_cand, uint32_t ncand, const SymStep* steps,
                                                     uint32_t* s_dict) {
  const uint32_t lane = threadIdx.x & 31u;
  for (uint32_t c = 0; c < ncand; ++c) {
    const uint32_t i = s_cand[c];
    const uint32_t start = dict_offset(v, i), end = dict_offset(v, i + 1u);
    const uint8_t* code = v.fsst + start;
    const uint32_t clen = end - start;
    uint32_t S = kStateOne, carry_lit = 0;
    bool hit = false;
    for (uint32_t base = 0; base < clen && !hit; base += 32u) {
      const uint32_t idx = base + lane;
      const bool in = idx < clen;
      const uint32_t b = in ? code[idx] : 0u;
      const uint32_t F = __ballot_sync(kFullMask, in && b == 255u);
      const uint32_t Fp = carry_lit ? (F & ~1u) : F;
      const uint32_t zeros = ~Fp & lanemask_lt();
      const uint32_t run = zeros ? (lane - 1u - (31u - __clz(zeros))) : lane;
      const bool lit = (lane == 0u) ? (carry_lit != 0u) : ((run & 1u) != 0u);
      const bool esc = in && (b == 255u) && !lit;
      SymStep st = step_identity();  // lanes past the end and escape markers
      if (in && !esc) st = steps[b + (lit ? 256u : 0u)];
#pragma unroll
      for (uint32_t d = 1; d < 32u; d <<= 1) {
        SymStep o;
        o.L = __shfl_down_sync(kFullMask, st.L, d);
        o.A = __shfl_down_sync(kFullMask, st.A, d);
        o.B = __shfl_down_sync(kFullMask, st.B, d);
        o.H = __shfl_down_sync(kFullMask, st.H, d);
        if ((lane & (2u * d - 1u)) == 0u) st = step_then(st, o);
      }
      const uint32_t Lc = __shfl_sync(kFullMask, st.L, 0), Ac = __shfl_sync(kFullMask, st.A, 0);
      const uint32_t Bc = __shfl_sync(kFullMask, st.B, 0), Hc = __shfl_sync(kFullMask, st.H, 0);
      hit = (S & Hc) != 0u;
      S = (shl_sat(S, Lc) & Ac) | Bc | kStateOne;
      carry_lit = __shfl_sync(kFullMask, esc ? 1u : 0u, 31);
    }
    if (hit && lane == 0u) s_dict[i >> 5] |= 1u << (i & 31u);
    __syncwarp();
  }
}

// ---- IN lists ---------------------------------------------------------------------------------------
// Per entry, every needle of the list (pred.needle: int32 offsets[list_n + 1], then the bytes; read from global memory) is
// planned as `=` plans it: does it start with the shared prefix, and which PrefixKey would an equal value have. Thread t
// plans needle t; the (key, needle) pairs are then sorted by key in shared memory (bitonic, kInListMaxValues = 256 slots,
// needles without the prefix and empty slots at the end), so that a dictionary value finds the needles with its own key by
// one binary search. A key whose length byte is <= 7 belongs to a short needle, and an equal key IS an equal value; a
// longer key only makes the value a candidate, decided by full_compare against each long needle with that key.
constexpr uint32_t kInTableBytes = kInListMaxValues * 8u + kInListMaxValues * 2u;
static_assert(kInListMaxValues == 256u, "one needle per thread of the 256-thread CTA");

__device__ __forceinline__ const int32_t* in_offsets(const StrPredDesc& pred) { return reinterpret_cast<const int32_t*>(pred.needle); }
__device__ __forceinline__ const uint8_t* in_bytes(const StrPredDesc& pred) { return pred.needle + 4u * (pred.list_n + 1u); }

// returns the number of needles that have the prefix (the sorted prefix of the table)
__device__ __forceinline__ uint32_t in_list_table(const StrView& v, const StrPredDesc& pred, uint64_t* s_key, uint16_t* s_tag) {
  const uint32_t t = threadIdx.x;
  uint64_t key = ~0ull;
  uint32_t tag = 0xffffu;  // empty slot
  if (t < pred.list_n) {
    const int32_t* off = in_offsets(pred);
    const uint32_t o = static_cast<uint32_t>(off[t]), len = static_cast<uint32_t>(off[t + 1u]) - o;
    if (eq_prefix_key(in_bytes(pred) + o, len, v.sp, v.h->shared_prefix_len, &key)) {
      tag = t;
    } else {
      key = ~0ull;
      tag = 0x8000u | t;
    }
  }
  s_key[t] = key;
  s_tag[t] = static_cast<uint16_t>(tag);
  const uint32_t n_valid = static_cast<uint32_t>(__syncthreads_count(tag < 0x8000u));
  for (uint32_t k = 2; k <= kInListMaxValues; k <<= 1) {
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
      const uint32_t l = t ^ j;
      if (l > t) {
        const uint64_t ka = s_key[t], kb = s_key[l];
        const uint16_t ta = s_tag[t], tb = s_tag[l];
        const bool gt = ka > kb || (ka == kb && ta > tb);
        if (gt == ((t & k) == 0)) {
          s_key[t] = kb;
          s_key[l] = ka;
          s_tag[t] = tb;
          s_tag[l] = ta;
        }
      }
      __syncthreads();
    }
  }
  return n_valid;
}

__device__ __forceinline__ uint32_t in_lower_bound(const uint64_t* s_key, uint32_t n, uint64_t key) {
  uint32_t lo = 0, len = n;
  while (len > 0) {
    const uint32_t half = len >> 1;
    if (s_key[lo + half] < key) {
      lo += half + 1u;
      len -= half + 1u;
    } else {
      len = half;
    }
  }
  return lo;
}

// The body of the predicate kernel, instantiated per address space of the staged sections so that the
// compiler emits LDS / LDG instead of generic loads. IN: the instantiation for IN lists (SP_IN; s_nd holds the table).
template <int MODE, bool IN>
__device__ __forceinline__ void str_scan_body(const StrView& v, const EntryIo& w, const StrPredDesc& pred,
                                              ScanSmem* sm, uint64_t* s_sym, uint8_t* s_len, StrPlan* s_plan,
                                              const uint8_t* s_nd, const uint16_t* s_fail, uint32_t* s_dict,
                                              uint16_t* s_cand, uint32_t* s_M, SymStep* s_step, uint32_t dict_words,
                                              uint64_t* bar_rows, uint32_t bar_parity, uint64_t& table_cache,
                                              long long t_start) {
  const uint32_t m = pred.needle_len;
  // measurement aid (pred.prof): thread 0 stamps the phase boundaries with the SM clock
  long long t_prev = t_start;
  auto stamp = [&](int slot) {
#ifdef LC_PHASE_PROF  // build with -DLC_PHASE_PROF for the per-phase cycle split (reported by bench.py)
    if (pred.prof && threadIdx.x == 0) {
      const long long t = clock64();
      atomicAdd(&pred.prof[4 + slot], static_cast<unsigned long long>(t - t_prev));
      t_prev = t;
    }
#endif
  };
  stamp(0);  // staging wait
  if (threadIdx.x == 0) plan_str_pred(v, pred, s_nd, s_plan);
  __syncthreads();
  stamp(1);  // plan
  const StrPlan plan = *s_plan;
  const uint32_t U = v.h->n_unique;
  const int lane = threadIdx.x & 31;
  const int32_t kind = plan.kind;
  const bool neg = (plan.flags & 2u) != 0;
  const bool needs_table = (kind == SP_EQ_LONG || kind == SP_ORD || kind == SP_LIKE || kind == SP_IN);
  uint64_t* s_in_key = reinterpret_cast<uint64_t*>(const_cast<uint8_t*>(s_nd));
  uint16_t* s_in_tag = reinterpret_cast<uint16_t*>(s_in_key + kInListMaxValues);
  uint32_t in_valid = 0;
  if constexpr (IN) in_valid = in_list_table(v, pred, s_in_key, s_in_tag);  // ends with a barrier
  const bool fast_like = (kind == SP_LIKE) && m <= 31u;
  if (needs_table && v.h->table_ptr != table_cache) {
    // symbol table + step table of this column chunk; a CTA walks consecutive entries, which usually share it
    load_fsst_table(reinterpret_cast<const FsstTable*>(v.h->table_ptr), s_sym, s_len);
    __syncthreads();
    if (fast_like) build_sym_steps(s_sym, s_len, s_nd, m, s_M, s_step);
    table_cache = v.h->table_ptr;
  }
  stamp(2);  // symbol tables (includes no barrier after build_sym_steps: its consumers sync later)

  // ---------------- phase 1: one decision per dictionary entry ----------------
  if (kind == SP_CONST) {
    const uint32_t fill = (plan.flags & 1u) ? kFullMask : 0u;
    for (uint32_t i = threadIdx.x; i < dict_words; i += 256u) s_dict[i] = fill;
  } else if (fast_like) {
    // LIKE candidates: the reference gate (byte-class fingerprints, comparisons.rs:600-615), then the private trigram
    // filter on its survivors. Each thread owns the uniques i0 + lane of its warp's stripes; their gate inputs
    // (fingerprint from the staged head, trigram filter from global memory) are loaded up front, four stripes at a
    // time, so the global loads overlap instead of each one stalling a ballot round. One ballot per stripe appends
    // the survivors to the queue. (An earlier version also ordered the queue by length class — worth 3 % with ~700
    // candidates per entry, nothing with the handful the trigram filter leaves, at the price of a second pass.)
    uint32_t* cand_cnt = sm->warp_tot;  // [0] queue length (unused scratch in this phase)
    const uint32_t pw = bloom_plane_words(U);
    if (threadIdx.x == 0) cand_cnt[0] = 0;
    __syncthreads();
    for (uint32_t g0 = (threadIdx.x & ~31u); g0 < U; g0 += 1024u) {
      // four stripes in flight: fingerprint (staged head) + the stripe's word of each of the needle's filter planes (lane t
      // fetches plane t's word; their AND over the warp is the stripe's candidate word)
      uint32_t fpv[4], pwd[4];
#pragma unroll
      for (uint32_t t = 0; t < 4; ++t) {
        const uint32_t i0 = g0 + t * 256u;
        const uint32_t i = i0 + lane;
        fpv[t] = (i < U && v.fp) ? v.fp[i] : 0u;
        pwd[t] = kFullMask;
        if (i0 < U && v.planes && static_cast<uint32_t>(lane) < pred.n_planes)
          pwd[t] = __ldg(v.planes + static_cast<size_t>(pred.planes[lane]) * pw + (i0 >> 5));
      }
#pragma unroll
      for (uint32_t t = 0; t < 4; ++t) {
        const uint32_t i0 = g0 + t * 256u;
        if (i0 >= U) break;  // warp-uniform
        const uint32_t i = i0 + lane;
        const bool ref_ok = (i < U) && (v.fp ? ((fpv[t] & pred.needle_fp) == pred.needle_fp) : true);
        const uint32_t cwd = __reduce_and_sync(kFullMask, pwd[t]);  // every lane takes part (not behind ref_ok)
        const bool cand = ref_ok && ((cwd >> lane) & 1u);
        const uint32_t rw = __ballot_sync(kFullMask, ref_ok);
        const uint32_t cw = __ballot_sync(kFullMask, cand);
        uint32_t base = 0;
        if (lane == 0) {
          s_dict[i0 >> 5] = 0;
          if (rw) atomicAdd(&sm->misc[0], __popc(rw));
          if (cw) base = atomicAdd(&cand_cnt[0], __popc(cw));
        }
        if (cw) {
          base = __shfl_sync(kFullMask, base, 0);
          if (cand) s_cand[base + __popc(cw & lanemask_lt())] = static_cast<uint16_t>(i);
        }
      }
    }
    __syncthreads();
    const uint32_t ncand = cand_cnt[0];
    if (pred.prof) {  // measurement aid, never on in a timed run
      unsigned long long bytes = 0;
      for (uint32_t c = threadIdx.x; c < ncand; c += 256u)
        bytes += dict_offset(v, s_cand[c] + 1u) - dict_offset(v, s_cand[c]);
      if (bytes) atomicAdd(&pred.prof[2], bytes);
      if (threadIdx.x == 0) {
        atomicAdd(&pred.prof[0], static_cast<unsigned long long>(U));
        atomicAdd(&pred.prof[1], static_cast<unsigned long long>(ncand));
      }
    }
    // An entry has only a few hundred candidates: spread over all 256 lanes each lane would get 2-3 values and the
    // pass would last as long as its LONGEST value (a value's codes are inherently sequential) with most lanes idle.
    // Half of the warps walk the queue; the others wait at the barrier and cost no issue slots, which the SM's other
    // resident CTAs use.
    stamp(3);  // candidate gate
    // Warps beyond the number of candidates / 32 would find the queue empty: they skip the walk and wait at the
    // barrier. (Giving each lane several values — fewer walking warps — was measured and is slower: the walk is a
    // latency chain per lane, not an issue-slot problem.)
    const uint32_t walk_warps = ncand >= kCandPerWarp * kLikeWarps ? kLikeWarps : (ncand + kCandPerWarp - 1u) / kCandPerWarp;
    if ((threadIdx.x >> 5) < walk_warps) like_candidates(v, s_cand, ncand, &sm->misc[1], s_step, s_dict);
    if (neg) {
      // NOT LIKE inverts every dictionary result — but, as in the reference, only inside
      // apply_like_match_on_candidates, i.e. only when the fingerprint gate let something through
      // (comparisons.rs:166-180, 644-648). Without fingerprints (flags bit2) it is a plain negation.
      __syncthreads();
      const bool invert = (plan.flags & 4u) ? true : (sm->misc[0] != 0);  // misc[0]: passes of the REFERENCE gate
      if (invert)
        for (uint32_t i = threadIdx.x; i < dict_words; i += 256u) s_dict[i] = ~s_dict[i];
    }
  } else {
    const uint32_t op = static_cast<uint32_t>(pred.op);
    for (uint32_t i0 = (threadIdx.x & ~31u); i0 < U; i0 += 256u) {
      const uint32_t i = i0 + lane;
      const bool act = i < U;
      bool res = false, cand = false;
      if (kind == SP_LIKE) {
        cand = v.fp ? ((v.fp[act ? i : 0] & pred.needle_fp) == pred.needle_fp) : true;
      } else {
        const uint64_t key = act ? v.pk[i] : 0ull;
        if (kind == SP_EQ_SHORT) {
          res = (key == plan.key_expect) != neg;
        } else if (kind == SP_EQ_LONG) {
          cand = (key == plan.key_expect);
          res = neg;
        } else if (IN && kind == SP_IN) {
          const uint32_t t = in_lower_bound(s_in_key, in_valid, key);
          const bool hit = t < in_valid && s_in_key[t] == key;
          if ((key >> 56) <= 7u) {
            res = hit != neg;  // short needle: the key decides
          } else {
            cand = hit;
            res = neg;
          }
        } else if (kind == SP_ORD) {
          const uint64_t mask = ~0ull << (8u * (8u - plan.cmp_len));
          const uint64_t a = bswap64(key) & mask;
          if (a < plan.key_expect) res = (op == LC_OP_LT || op == LC_OP_LE);
          else if (a > plan.key_expect) res = (op == LC_OP_GT || op == LC_OP_GE);
          else cand = true;
        } else {  // SP_ORD_EMPTY
          const bool empty = (key >> 56) == 0;
          res = (op == LC_OP_LT) ? false : (op == LC_OP_LE) ? empty : (op == LC_OP_GT) ? !empty : true;
        }
      }
      res = res && act;
      cand = cand && act;
      const uint32_t rw = __ballot_sync(kFullMask, res);
      const uint32_t cw = __ballot_sync(kFullMask, cand);
      if (lane == 0) s_dict[i0 >> 5] = rw;
      if (cw) {
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(&sm->misc[0], __popc(cw));
        base = __shfl_sync(kFullMask, base, 0);
        if (cand) s_cand[base + __popc(cw & lanemask_lt())] = static_cast<uint16_t>(i);
      }
    }
    __syncthreads();
    const uint32_t ncand = sm->misc[0];
    if (pred.prof) {  // measurement aid, never on in a timed run
      unsigned long long bytes = 0;
      for (uint32_t c = threadIdx.x; c < ncand; c += 256u)
        bytes += dict_offset(v, s_cand[c] + 1u) - dict_offset(v, s_cand[c]);
      if (bytes) atomicAdd(&pred.prof[2], bytes);
      if (threadIdx.x == 0) {
        atomicAdd(&pred.prof[0], static_cast<unsigned long long>(U));
        atomicAdd(&pred.prof[1], static_cast<unsigned long long>(ncand));
      }
    }
    // candidates: walk the FSST codes of the value
    if (fast_like) {
      like_candidates(v, s_cand, ncand, &sm->misc[1], s_step, s_dict);
    } else {
      for (uint32_t c = threadIdx.x; c < ncand; c += 256u) {
        const uint32_t i = s_cand[c];
        bool res;
        if (kind == SP_LIKE) {
          res = contains_needle(v, i, s_sym, s_len, s_nd, s_fail, m);
        } else if (IN && kind == SP_IN) {
          const uint64_t key = v.pk[i];
          const int32_t* off = in_offsets(pred);
          bool eq = false;
          for (uint32_t t = in_lower_bound(s_in_key, in_valid, key); !eq && t < in_valid && s_in_key[t] == key; ++t) {
            const uint32_t j = s_in_tag[t], o = static_cast<uint32_t>(off[j]);
            eq = full_compare(v, i, s_sym, s_len, in_bytes(pred) + o, static_cast<uint32_t>(off[j + 1u]) - o) == 0;
          }
          res = eq != neg;
        } else {
          const int ord = full_compare(v, i, s_sym, s_len, s_nd, m);
          if (kind == SP_EQ_LONG) res = (ord == 0) != neg;
          else res = (op == LC_OP_LT) ? ord < 0 : (op == LC_OP_LE) ? ord <= 0 : (op == LC_OP_GT) ? ord > 0 : ord >= 0;
        }
        if ((kind == SP_EQ_LONG || (IN && kind == SP_IN)) && neg) {
          if (!res) atomicAnd(&s_dict[i >> 5], ~(1u << (i & 31u)));
        } else if (res) {
          atomicOr(&s_dict[i >> 5], 1u << (i & 31u));
        }
      }
    }
    if (kind == SP_LIKE && neg) {
      // NOT LIKE inverts every dictionary result — but, as in the reference, only inside
      // apply_like_match_on_candidates, i.e. only when the fingerprint gate let something through
      // (comparisons.rs:166-180, 644-648). Without fingerprints (flags bit2) it is a plain negation.
      __syncthreads();
      const bool invert = (plan.flags & 4u) ? true : (ncand != 0);
      if (invert)
        for (uint32_t i = threadIdx.x; i < dict_words; i += 256u) s_dict[i] = ~s_dict[i];
    }
  }
  __syncthreads();
  stamp(4);  // code walk (or the non-LIKE phase 1)
  if (bar_rows) mbar_wait(bar_rows, bar_parity);
  stamp(5);  // row sections

  // ---------------- phase 2: dictionary results -> rows ----------------
  const uint16_t* keys = v.keys;
  if (MODE == MODE_REFINE || (MODE == MODE_PRED && w.sel == nullptr)) {
    // Full-length outputs need no compaction: a warp takes a 1024-row chunk, 32 steps of key -> result bit -> ballot
    // with lane j keeping the word of step j, then ONE coalesced pass over the chunk's 32 mask words (AND validity /
    // selection, store, popcount). ~9 instructions per 32 rows instead of ~32 on the general path.
    const uint32_t n = v.h->n, n_words = (n + 31u) >> 5, n_chunks = (n + 1023u) >> 10, tail = n & 31u;
    const uint32_t warp = threadIdx.x >> 5;
    uint32_t* out_bits = reinterpret_cast<uint32_t*>(w.out);
    uint32_t* out_valid = (MODE == MODE_PRED && v.valid) ? w.out_valid : nullptr;
    uint32_t survivors = 0;
    for (uint32_t c = warp; c < n_chunks; c += 8u) {
      const uint32_t wi = c * 32u + lane;
      uint32_t sw = kFullMask;  // issued before the steps: the global load overlaps them
      if (w.sel && wi < n_words) sw = w.sel[wi];
      uint32_t mine = 0;
      const uint32_t row0 = c * 1024u + lane;
      const bool full = (c + 1u) * 1024u <= n;
#pragma unroll 8
      for (uint32_t j = 0; j < 32; ++j) {
        const uint32_t row = row0 + j * 32u;
        const uint32_t k = (full || row < n) ? keys[row] : 0u;
        const uint32_t cw = __ballot_sync(kFullMask, (s_dict[k >> 5] >> (k & 31u)) & 1u);
        if (static_cast<uint32_t>(lane) == j) mine = cw;
      }
      if (wi < n_words) {
        uint32_t vw = v.valid ? v.valid[wi] : kFullMask;
        if (wi == n_words - 1u && tail) vw &= (1u << tail) - 1u;
        const uint32_t cw = mine & vw & sw;
        out_bits[wi] = cw;
        if (out_valid) out_valid[wi] = vw;
        survivors += __popc(cw);
      }
    }
    if (w.counts) {
      survivors = warp_sum(survivors);
      if (lane == 0 && survivors) atomicAdd(&sm->counts[0], survivors);
      __syncthreads();
      if (threadIdx.x == 0) {
        if (MODE == MODE_REFINE) {
          w.counts[0] = sm->counts[0];
          w.counts[1] = 0;
        } else {
          w.counts[0] = n;
          w.counts[1] = v.h->null_count;
          w.counts[2] = sm->counts[0];
        }
      }
    }
    stamp(6);
#ifdef LC_PHASE_PROF
    if (pred.prof && threadIdx.x == 0) atomicAdd(&pred.prof[11], static_cast<unsigned long long>(clock64() - t_start));
#endif
    return;
  }
  auto cmp = [&](uint32_t row, uint32_t, uint32_t) -> bool {
    const uint32_t k = keys[row];
    return (s_dict[k >> 5] >> (k & 31u)) & 1u;
  };
  auto emit = [&](uint32_t, uint32_t, uint32_t, uint32_t) {};
  scan_entry_rows<MODE>(w.sel, v.h->n, v.valid, v.h->null_count, reinterpret_cast<uint32_t*>(w.out), w.out_valid,
                        w.counts, sm, cmp, emit);
  stamp(6);  // rows
#ifdef LC_PHASE_PROF
  if (pred.prof && threadIdx.x == 0) atomicAdd(&pred.prof[11], static_cast<unsigned long long>(clock64() - t_start));
#endif
  (void)t_prev;
}

// Shared-memory map of the predicate kernel (after the fixed ScanSmem area):
//   symbols 2048 | lengths 256 | plan 32 | M[256] 1024 | SymStep[512] 8192 | needle | KMP links | dictionary
//   result bits | candidate list | staged entry head
constexpr uint32_t kStrScanTables = 2048u + 256u + 32u + 1024u + 8192u;

template <int MODE, bool IN>
__global__ void __launch_bounds__(256, 4)
k_str_scan(ScanIo io, StrPredDesc pred, uint32_t stage_cap, uint32_t dict_words, uint32_t n_entries, uint32_t per_cta) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  ScanSmem* sm = reinterpret_cast<ScanSmem*>(smem_raw);
  uint64_t* s_sym = reinterpret_cast<uint64_t*>(smem_raw + kScanFixedSmem);
  uint8_t* s_len = reinterpret_cast<uint8_t*>(s_sym + 256);
  StrPlan* s_plan = reinterpret_cast<StrPlan*>(s_len + 256);
  uint32_t* s_M = reinterpret_cast<uint32_t*>(s_len + 256 + 32);
  SymStep* s_step = reinterpret_cast<SymStep*>(s_M + 256);
  uint8_t* s_nd = reinterpret_cast<uint8_t*>(s_step + 512);
  const uint32_t m = pred.needle_len;
  const uint32_t nd_bytes = IN ? kInTableBytes : ((m + 15u) & ~15u);  // IN lists: the needle table in place of the needle
  uint16_t* s_fail = reinterpret_cast<uint16_t*>(s_nd + nd_bytes);
  uint32_t* s_dict = reinterpret_cast<uint32_t*>(s_nd + nd_bytes + ((2u * m + 15u) & ~15u));
  uint16_t* s_cand = reinterpret_cast<uint16_t*>(s_dict + dict_words);
  uint8_t* stage = reinterpret_cast<uint8_t*>(s_cand) + (((dict_words * 64u) + 127u) & ~127u);
  stage = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(stage) + 127u) & ~static_cast<uintptr_t>(127u));

  const bool is_like = (pred.op == LC_OP_LIKE || pred.op == LC_OP_NOT_LIKE);
  if (threadIdx.x == 0) {
    mbar_init(&sm->bar[0], 1);
    mbar_init(&sm->bar[1], 1);
    fence_mbar_init();
  }
  // needle + KMP links (shared by all entries of the launch)
  for (uint32_t i = threadIdx.x; i < m; i += 256u) {
    s_nd[i] = pred.needle[i];
    s_fail[i] = reinterpret_cast<const uint16_t*>(pred.needle + ((m + 3u) & ~3u))[i];
  }
  // A CTA takes `per_cta` CONSECUTIVE entries: neighbours in a scan are batches of the same column chunk, so the
  // FSST symbol table and the needle's step table are built once and reused (table_cache).
  uint64_t table_cache = 0;
  uint32_t n_staged = 0;  // uses of the two mbarriers so far -> wait parity
  const uint32_t e_end = (blockIdx.x + 1u) * per_cta < n_entries ? (blockIdx.x + 1u) * per_cta : n_entries;
  for (uint32_t e = blockIdx.x * per_cta; e < e_end; ++e) {
#ifdef LC_PHASE_PROF
    const long long t_start = pred.prof ? clock64() : 0;
#else
    const long long t_start = 0;
#endif
    const EntryRef ref = io.refs[e];
    const EntryIo w = resolve_io(io, e);
    const bool staged = (is_like ? ref.head_bytes - (ref.rows_off - ref.pk_off) : ref.head_bytes) <= stage_cap;
    scan_smem_init(sm);
    if (threadIdx.x == 0 && staged) {
      // (A) what phase 1 needs: LIKE -> header, shared prefix, fingerprints, offset residuals (no prefix keys);
      //     everything else -> header, shared prefix and the prefix keys (residuals stay in global memory,
      //     only the few prefix ties ever look at them)
      if (is_like) {
        mbar_expect_tx(&sm->bar[0], ref.pk_off);
        tma_bulk_g2s(stage, ref.blob, ref.pk_off, &sm->bar[0]);
      } else {
        const uint32_t pk_bytes = ref.rows_off - ref.pk_off;
        mbar_expect_tx(&sm->bar[0], ref.sp_end + pk_bytes);
        tma_bulk_g2s(stage, ref.blob, ref.sp_end, &sm->bar[0]);
        if (pk_bytes) tma_bulk_g2s(stage + ref.pk_off, ref.blob + ref.pk_off, pk_bytes, &sm->bar[0]);
      }
      // (B) what phase 2 needs, in flight while phase 1 computes: validity + keys. For LIKE they are packed right
      //     behind the metadata (the prefix keys are not staged, so their slot is not reserved either).
      const uint32_t rest = ref.head_bytes - ref.rows_off;
      mbar_expect_tx(&sm->bar[1], rest);
      tma_bulk_g2s(stage + (is_like ? ref.pk_off : ref.rows_off), ref.blob + ref.rows_off, rest, &sm->bar[1]);
    }
    for (uint32_t i = threadIdx.x; i < dict_words; i += 256u) s_dict[i] = 0;
    __syncthreads();
    if (staged) {
      const uint32_t parity = n_staged & 1u;
      ++n_staged;
      mbar_wait(&sm->bar[0], parity);
      StrView v = make_view(stage, ref.blob);
      if (is_like) {
        v.pk = reinterpret_cast<const uint64_t*>(ref.blob + v.h->prefix_keys_off);  // not staged, not used
        const uint32_t shift = ref.rows_off - ref.pk_off;                             // rows section moved down
        v.keys = reinterpret_cast<const uint16_t*>(reinterpret_cast<const uint8_t*>(v.keys) - shift);
        if (v.valid) v.valid = reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(v.valid) - shift);
      } else {
        v.resid = ref.blob + v.h->resid_off;
        v.fp = nullptr;
      }
      str_scan_body<MODE, IN>(v, w, pred, sm, s_sym, s_len, s_plan, s_nd, s_fail, s_dict, s_cand, s_M, s_step, dict_words,
                          &sm->bar[1], parity, table_cache, t_start);
    } else {
      const StrView v = make_view(ref.blob, ref.blob);
      str_scan_body<MODE, IN>(v, w, pred, sm, s_sym, s_len, s_plan, s_nd, s_fail, s_dict, s_cand, s_M, s_step, dict_words,
                          nullptr, 0, table_cache, t_start);
    }
    __syncthreads();  // the staged sections and the control area are reused by the next entry
  }
}

// ------------------------------------------------------------------------------------------------
// LIKE / NOT LIKE '%needle%' (needle <= 31 bytes) with full-length outputs: the streaming form of the scan.
//
// What an entry costs is decided by what its DICTIONARY says, not by its rows:
//   gate     fingerprint -> trigram filter (loaded only by lanes the fingerprint let through, one 32-byte sector each)
//            -> the few survivors are matched exactly on their FSST codes (Shift-And over the decoded bytes)
//   result   no dictionary value matched  => every row is false: the mask words are written as zeros and the u16 keys
//            are NEVER READ (the common case of a selective predicate);
//            NOT LIKE with no match       => every valid selected row is true: validity AND selection, keys not read;
//            otherwise                    => dictionary bits are broadcast through the keys (coalesced reads)
// Results are the reference's (comparisons.rs:159-183, 325-347, 600-651) bit for bit: a row's answer is its dictionary
// value's answer, and both shortcuts are that rule applied to a dictionary whose answers are all equal.
//
// One WARP per entry, no block-wide phase: an entry is a chain of short dependent steps (header -> gate loads -> a
// handful of code walks -> 1 KB of output), and a CTA that takes them together waits at every barrier for its slowest
// lane. Independent warps keep 8 x as many entries in flight per SM and a walking lane stalls only its own warp.
// The CTA's warps take neighbouring entries (one column chunk = one FSST symbol table, read through L1), each
// warp prefetches the next entry's header word and the blob pointer of the one after (registers), fingerprints and
// trigram sets stream from global memory with coalesced / sector-sized loads, four stripes of 32 values in flight.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kLikeCandCap = 512;  // per-warp candidate list (u16); a full list is walked and reused
constexpr uint32_t kWarpWalkMax = 12;   // up to this many candidates are walked by the whole warp, one value at a time

static_assert(offsetof(StrHeader, shared_prefix_len) == 24 && offsetof(StrHeader, prefix_keys_off) == 36, "header words");
static_assert(offsetof(StrHeader, n) == 8 && offsetof(StrHeader, n_unique) == 12 && offsetof(StrHeader, slope) == 16 &&
                  offsetof(StrHeader, intercept) == 20 && offsetof(StrHeader, validity_off) == 28 &&
                  offsetof(StrHeader, keys_off) == 32 && offsetof(StrHeader, fp_off) == 40 && offsetof(StrHeader, resid_off) == 44 &&
                  offsetof(StrHeader, fsst_off) == 52 && offsetof(StrHeader, null_count) == 64 &&
                  offsetof(StrHeader, table_ptr) == 80 && offsetof(StrHeader, bloom_off) == 100,
              "k_str_like reads the header by word offset");

// The needle's Shift-And step table for each FSST symbol table of the list, written to global memory once per launch:
// the walk of a candidate then costs one 16-byte (L1-resident) load and ~6 ALU ops per FSST code instead of ~25
// instructions per decoded byte.
__global__ void __launch_bounds__(256) k_like_steps(const uint64_t* __restrict__ tables, StrPredDesc pred, SymStep* __restrict__ out) {
  __shared__ uint64_t s_sym[256];
  __shared__ __align__(16) uint8_t s_len[256];
  __shared__ uint32_t s_M[256];
  __shared__ SymStep s_step[512];
  __shared__ uint8_t s_nd[32];
  if (threadIdx.x < pred.needle_len) s_nd[threadIdx.x] = pred.needle[threadIdx.x];
  load_fsst_table(reinterpret_cast<const FsstTable*>(tables[blockIdx.x]), s_sym, s_len);
  __syncthreads();
  build_sym_steps(s_sym, s_len, s_nd, pred.needle_len, s_M, s_step);
  __syncthreads();
  SymStep* dst = out + static_cast<size_t>(blockIdx.x) * 512u;
  for (uint32_t c = threadIdx.x; c < 512u; c += 256u) dst[c] = s_step[c];
}

cudaError_t launch_like_steps(const uint64_t* d_tables, uint32_t n_tables, const StrPredDesc& pred, void* d_steps, cudaStream_t s) {
  if (n_tables == 0) return cudaSuccess;
  k_like_steps<<<n_tables, 256, 0, s>>>(d_tables, pred, static_cast<SymStep*>(d_steps));
  return cudaGetLastError();
}

// AUX = the launch also counts (NOT LIKE's inversion rule needs the passes of the reference gate; the untimed measurement
// launch feeds the profile counters). The plain LIKE launch carries none of that state through the gate loop.
template <int MODE, int OCC, bool AUX>
__global__ void __launch_bounds__(256, OCC)
k_str_like(ScanIo io, StrPredDesc pred_in, uint32_t dict_words, uint32_t n_entries, uint32_t per_cta) {
  StrPredDesc pred = pred_in;
  if (!AUX) pred.prof = nullptr;
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  // per warp: walk queue head (4 words) | dictionary answer bits | candidate list
  uint32_t* s_queue = reinterpret_cast<uint32_t*>(smem_raw) + warp * (4u + dict_words + kLikeCandCap / 2u);
  uint32_t* s_dict = s_queue + 4;
  uint16_t* s_cand = reinterpret_cast<uint16_t*>(s_dict + dict_words);
  const bool neg = AUX && pred.op == LC_OP_NOT_LIKE;
  const SymStep* steps_all = static_cast<const SymStep*>(pred.like_steps);
  for (uint32_t i = lane; i < dict_words; i += 32u) s_dict[i] = 0;
  if (lane == 0) s_queue[0] = 0;
  __syncwarp();
  // the needle's filter planes, one per lane (broadcast by shuffle where the gate walks them)
  const uint32_t n_planes = pred.n_planes;
  const uint32_t my_plane = lane < n_planes ? pred_in.planes[lane] : 0u;
  const uint32_t e0 = blockIdx.x * per_cta;
  const uint32_t e_end = e0 + per_cta < n_entries ? e0 + per_cta : n_entries;
  uint32_t e = e0 + warp;
  if (e >= e_end) return;
  // software pipeline: header word of the next entry, blob pointer of the one after
  const uint8_t* blob0 = io.refs[e].blob;
  uint32_t hw0 = __ldg(reinterpret_cast<const uint32_t*>(blob0) + lane);
  const uint8_t* blob1 = (e + 8u < e_end) ? io.refs[e + 8u].blob : nullptr;
  for (; e < e_end; e += 8u) {
    uint32_t hw1 = hw0;
    if (e + 8u < e_end) hw1 = __ldg(reinterpret_cast<const uint32_t*>(blob1) + lane);
    const uint8_t* blob2 = (e + 16u < e_end) ? io.refs[e + 16u].blob : nullptr;
    const uint8_t* blob = blob0;
    // Header words are pulled out of hw0 (one register, lane i = word i) where they are needed rather than all up front:
    // the gate loop is where registers are scarce.
    const uint32_t hw_lo = __shfl_sync(kFullMask, hw0, 1);  // arrow_type | has_nulls << 8 | has_fp << 16 | offset_bytes << 24
    const uint32_t U = __shfl_sync(kFullMask, hw0, 3);
    const bool has_fp = (hw_lo >> 16) & 0xffu;
    const uint32_t bloom_off = __shfl_sync(kFullMask, hw0, 25);
    const uint32_t* fp = has_fp ? reinterpret_cast<const uint32_t*>(blob + __shfl_sync(kFullMask, hw0, 10)) : nullptr;

    // ---- gate + walk ----
    uint32_t ncand = 0, n_ref = 0, walked = 0;
    unsigned long long walked_bytes = 0;
    bool walked_any = false;
    auto walk = [&]() {  // match the listed candidates exactly on their FSST codes (Shift-And, one table step per code)
      __syncwarp();
      StrView v{};  // what the walk needs: header (slope / intercept / residual width), residuals, compressed values
      v.h = reinterpret_cast<const StrHeader*>(blob);
      v.resid = blob + __shfl_sync(kFullMask, hw0, 11);
      v.fsst = blob + __shfl_sync(kFullMask, hw0, 13);
      const SymStep* steps = steps_all + static_cast<size_t>(pred.entry_table[e]) * 512u;
      if (ncand <= kWarpWalkMax) like_candidates_warp(v, s_cand, ncand, steps, s_dict);  // a handful: the warp takes each value together
      else like_candidates(v, s_cand, ncand, s_queue, steps, s_dict);
      __syncwarp();
      if (lane == 0) s_queue[0] = 0;
      walked += ncand;
      walked_any = true;
      ncand = 0;
      __syncwarp();
    };
    // The candidate bitmap of the dictionary, 32 values per word, lane l holding words l, l + 32, ...
    //   with the private filter: the AND of the needle's planes (entry_layout.h) — n_planes coalesced words per lane, all
    //     requested before the first AND; fingerprints are not read at all (a value that fails them cannot match, and the
    //     walk is exact, so the answer is the reference's with or without them);
    //   without it (needles below three bytes, entries loaded from LQDA): the reference gate, one ballot per 32 values.
    const uint32_t n_cw = (U + 31u) >> 5;
    const uint32_t* planes = bloom_off ? reinterpret_cast<const uint32_t*>(blob + bloom_off) : nullptr;
    const bool by_planes = planes != nullptr && n_planes != 0u;
    auto push = [&](uint32_t bits, uint32_t idx0) {  // set bits -> candidate list; at most 16 per lane, so a walked list has room
      const uint32_t cnt = __popc(bits);
      const uint32_t incl = warp_incl_scan(cnt, lane);
      const uint32_t total = __shfl_sync(kFullMask, incl, 31);
      if (total == 0u) return;
      if (ncand + total > kLikeCandCap) walk();
      uint32_t pos = ncand + incl - cnt;
      while (bits) {
        const uint32_t b = __ffs(bits) - 1u;
        bits &= bits - 1u;
        s_cand[pos++] = static_cast<uint16_t>(idx0 + b);
      }
      ncand += total;
      __syncwarp();
    };
    auto emit = [&](uint32_t acc, uint32_t w) {
      if (__any_sync(kFullMask, acc != 0u)) {
        push(acc & 0xffffu, w * 32u);
        push(acc >> 16, w * 32u + 16u);
      }
    };
    if (by_planes) {
      for (uint32_t w0 = 0; w0 < n_cw; w0 += 64u) {
        const uint32_t wa = w0 + lane, wb = w0 + 32u + lane;
        const bool in_a = wa < n_cw, in_b = wb < n_cw;
        uint32_t a = in_a ? kFullMask : 0u, b = in_b ? kFullMask : 0u;
#pragma unroll 4
        for (uint32_t t = 0; t < n_planes; ++t) {
          const uint32_t* pl = planes + static_cast<size_t>(__shfl_sync(kFullMask, my_plane, t)) * n_cw;
          if (in_a) a &= __ldg(pl + wa);
          if (in_b) b &= __ldg(pl + wb);
        }
        emit(a, wa);
        if (w0 + 32u < n_cw) emit(b, wb);
      }
      if ((neg || pred.prof) && fp) {  // NOT LIKE's inversion rule / the counters want the passes of the reference gate
        for (uint32_t i = lane; i < U; i += 32u) n_ref += ((__ldg(fp + i) & pred.needle_fp) == pred.needle_fp) ? 1u : 0u;
        n_ref = warp_sum(n_ref);
      }
    } else {
      for (uint32_t w0 = 0; w0 < n_cw; w0 += 32u) {
        uint32_t acc = 0;
#pragma unroll 4
        for (uint32_t j = 0; j < 32u; ++j) {
          const uint32_t i = (w0 + j) * 32u + lane;
          if (i - lane >= U) break;  // warp-uniform
          const bool ok = (i < U) && (!fp || ((__ldg(fp + (i < U ? i : 0u)) & pred.needle_fp) == pred.needle_fp));
          const uint32_t bw = __ballot_sync(kFullMask, ok);
          if (lane == j) acc = bw;
          if (neg || pred.prof) n_ref += (lane == 0u) ? __popc(bw) : 0u;
        }
        emit(acc, w0 + lane);
      }
      if (neg || pred.prof) n_ref = __shfl_sync(kFullMask, n_ref, 0);
    }
    if (pred.prof) {  // measurement aid, never on in a timed run
      unsigned long long bytes = 0;
      StrView v{};
      v.h = reinterpret_cast<const StrHeader*>(blob);
      v.resid = blob + __shfl_sync(kFullMask, hw0, 11);
      for (uint32_t c = lane; c < ncand; c += 32u) bytes += dict_offset(v, s_cand[c] + 1u) - dict_offset(v, s_cand[c]);
      for (int d = 16; d > 0; d >>= 1) bytes += __shfl_xor_sync(kFullMask, bytes, d);
      walked_bytes = bytes;
    }
    if (ncand) walk();
    bool any = false;
    uint32_t n_match = 0;  // dictionary values that matched (the walk set their bits)
    if (walked_any) {
      for (uint32_t i = lane; i < n_cw; i += 32u) n_match += __popc(s_dict[i]);
      n_match = warp_sum(n_match);
      any = n_match != 0u;
    }
    if (pred.prof && lane == 0) {
      atomicAdd(&pred.prof[0], static_cast<unsigned long long>(U));
      atomicAdd(&pred.prof[1], static_cast<unsigned long long>(walked));
      atomicAdd(&pred.prof[2], walked_bytes);
      atomicAdd(&pred.prof[12], static_cast<unsigned long long>(n_ref));
      // what the reference's data for this predicate is besides the keys: header, fingerprints, all offset residuals
      atomicAdd(&pred.prof[13], static_cast<unsigned long long>(128u + (has_fp ? 4u * U : 0u) + (hw_lo >> 24) * (U + 1u)));
      // ... and what THIS gate read: the needle's planes, or the fingerprints where an entry has no filter
      atomicAdd(&pred.prof[14], static_cast<unsigned long long>(by_planes ? 4u * n_planes * n_cw : (has_fp ? 4u * U : 0u)));
      if (any) atomicAdd(&pred.prof[3], 1ull);
    }
    // NOT LIKE inverts every dictionary answer — but, as in the reference, only inside apply_like_match_on_candidates,
    // i.e. only when the fingerprint gate let something through (comparisons.rs:166-180, 644-648). Without
    // fingerprints it is a plain negation.
    const bool invert = neg && (!has_fp || n_ref != 0u);

    // per-entry io and the header words of the output phase
    const uint64_t so = io.sel_base ? io.sel_off[e] : kNoSel;
    const uint64_t oo = io.out_off[e];
    const uint64_t vo = (MODE == MODE_PRED && io.valid_base) ? io.valid_off[e] : 0ull;
    const uint32_t n = __shfl_sync(kFullMask, hw0, 2);
    const uint32_t validity_off = __shfl_sync(kFullMask, hw0, 7), keys_off = __shfl_sync(kFullMask, hw0, 8);
    const uint32_t null_count = __shfl_sync(kFullMask, hw0, 16);
    const bool has_nulls = (hw_lo >> 8) & 0xffu;
    const uint32_t* sel = (io.sel_base && so != kNoSel) ? io.sel_base + so : nullptr;
    uint32_t* out_bits = reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(io.out_base) + oo * 4u);
    const uint32_t* valid = has_nulls ? reinterpret_cast<const uint32_t*>(blob + validity_off) : nullptr;
    uint32_t* out_valid = (MODE == MODE_PRED && valid && io.valid_base) ? io.valid_base + vo : nullptr;
    const uint32_t n_words = (n + 31u) >> 5, tail = n & 31u;
    uint32_t survivors = 0;
    if (!any) {
      // every dictionary value has the same answer: the rows need no keys
      const bool all_true = invert;
      for (uint32_t wi = lane; wi < n_words; wi += 32u) {
        uint32_t vw = kFullMask;
        if (all_true || out_valid) {
          vw = valid ? __ldg(valid + wi) : kFullMask;
          if (wi == n_words - 1u && tail) vw &= (1u << tail) - 1u;
        }
        uint32_t cw = 0;
        if (all_true) cw = vw & (sel ? sel[wi] : kFullMask);
        out_bits[wi] = cw;
        if (out_valid) out_valid[wi] = vw;
        survivors += __popc(cw);
      }
    } else {
      const uint32_t flip = invert ? kFullMask : 0u;
      const uint16_t* keys = reinterpret_cast<const uint16_t*>(blob + keys_off);
      const uint32_t n_chunks = (n + 1023u) >> 10;
      if (n_match <= 4u) {
        // The usual case of a selective needle — one or two dictionary values matched: their ids sit in registers (both
        // halves of a word, so a 32-bit word of two keys is tested with a handful of logic ops) and the keys come as
        // 16-byte loads, eight rows per lane and load. Lane l's eight answers of load j are a byte of the mask word of rows
        // [256 j + 32 (l / 4), + 32); two shuffles assemble the word in the four lanes of the group, and the lane with
        // l % 4 == j keeps it — so a chunk of 1024 rows costs 4 loads and 8 shuffles per lane instead of 32 loads, 32
        // shared-memory lookups and 32 ballots.
        uint32_t mid[4] = {0u, 0u, 0u, 0u};
        {
          uint32_t got = 0;
          for (uint32_t i0 = 0; i0 < n_cw; i0 += 32u) {
            const uint32_t i = i0 + lane;
            uint32_t bits = i < n_cw ? s_dict[i] : 0u;
            uint32_t have;
            while ((have = __ballot_sync(kFullMask, bits != 0u)) != 0u) {
              const uint32_t leader = __ffs(have) - 1u;
              const uint32_t id = __shfl_sync(kFullMask, i * 32u + (bits ? __ffs(bits) - 1u : 0u), leader);
              if (lane == leader) bits &= bits - 1u;
              if (got == 0u) mid[0] = mid[1] = mid[2] = mid[3] = id * 0x10001u;  // unused slots repeat the first id
              else if (got == 1u) mid[1] = id * 0x10001u;
              else if (got == 2u) mid[2] = id * 0x10001u;
              else mid[3] = id * 0x10001u;
              ++got;
            }
          }
        }
        auto pair_eq = [&](uint32_t x) -> uint32_t {  // bit 0 / bit 1: the low / high key of the word is a matched id
          uint32_t e = 0;
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            if (t == 0 || static_cast<uint32_t>(t) < n_match) {
              const uint32_t r = x ^ mid[t];  // a zero half = equal
              e |= ~(r | ((r & 0x7fff7fffu) + 0x7fff7fffu)) & 0x80008000u;
            }
          }
          return ((e >> 15) & 1u) | ((e >> 30) & 2u);
        };
        const uint32_t grp = lane & 3u;
        uint4 q[4], qn[4];
        auto load_keys = [&](uint32_t c, uint4 (&dst)[4]) {
#pragma unroll
          for (uint32_t j = 0; j < 4; ++j) {
            const uint32_t row0 = c * 1024u + j * 256u + lane * 8u;
            // a load that starts inside the rows may run into the section's padding (16-byte aligned), never past it
            dst[j] = row0 < n ? __ldg(reinterpret_cast<const uint4*>(keys + row0)) : make_uint4(0u, 0u, 0u, 0u);
          }
        };
        load_keys(0u, qn);
        for (uint32_t c = 0; c < n_chunks; ++c) {
          const uint32_t wi = c * 32u + grp * 8u + (lane >> 2);  // the mask word this lane ends up with
          uint32_t sw = kFullMask, vw = kFullMask;
          if (wi < n_words) {
            if (sel) sw = sel[wi];
            if (valid) vw = __ldg(valid + wi);
          }
          // this chunk's keys were requested while the previous one was being tested; the next chunk's go out now
#pragma unroll
          for (uint32_t j = 0; j < 4; ++j) q[j] = qn[j];
          if (c + 1u < n_chunks) load_keys(c + 1u, qn);
          uint32_t mine = 0;
#pragma unroll
          for (uint32_t j = 0; j < 4; ++j) {
            uint32_t x = (pair_eq(q[j].x) | (pair_eq(q[j].y) << 2) | (pair_eq(q[j].z) << 4) | (pair_eq(q[j].w) << 6)) << (8u * grp);
            x |= __shfl_xor_sync(kFullMask, x, 1);
            x |= __shfl_xor_sync(kFullMask, x, 2);
            if (grp == j) mine = x;
          }
          if (wi < n_words) {
            if (wi == n_words - 1u && tail) vw &= (1u << tail) - 1u;
            const uint32_t cw = (mine ^ flip) & vw & sw;
            out_bits[wi] = cw;
            if (out_valid) out_valid[wi] = vw;
            survivors += __popc(cw);
          }
        }
      } else
      for (uint32_t c = 0; c < n_chunks; ++c) {
        const uint32_t wi = c * 32u + lane;
        uint32_t sw = kFullMask, vw = kFullMask;
        if (wi < n_words) {
          if (sel) sw = sel[wi];
          if (valid) vw = __ldg(valid + wi);
        }
        uint32_t mine = 0;
        const uint32_t row0 = c * 1024u + lane;
        const bool full = (c + 1u) * 1024u <= n;
        // the chunk's 1024 keys are requested up front (32 coalesced 64-byte loads in flight per warp), then looked up
        uint32_t kk[32];
#pragma unroll
        for (uint32_t j = 0; j < 32; ++j) {
          const uint32_t row = row0 + j * 32u;
          kk[j] = (full || row < n) ? __ldg(keys + row) : 0u;
        }
#pragma unroll
        for (uint32_t j = 0; j < 32; ++j) {
          const uint32_t k = kk[j];
          const uint32_t cw = __ballot_sync(kFullMask, (s_dict[k >> 5] >> (k & 31u)) & 1u);
          if (lane == j) mine = cw;
        }
        if (wi < n_words) {
          if (wi == n_words - 1u && tail) vw &= (1u << tail) - 1u;
          const uint32_t cw = (mine ^ flip) & vw & sw;
          out_bits[wi] = cw;
          if (out_valid) out_valid[wi] = vw;
          survivors += __popc(cw);
        }
      }
      __syncwarp();
      for (uint32_t i = lane; i < ((U + 31u) >> 5); i += 32u) s_dict[i] = 0;  // the bits this entry set
      __syncwarp();
    }
    if (io.counts) {
      survivors = warp_sum(survivors);
      if (lane == 0) {
        uint32_t* cnt = io.counts + static_cast<size_t>(e) * io.counts_stride;
        if (MODE == MODE_REFINE) {
          cnt[0] = survivors;
          cnt[1] = 0;
        } else {
          cnt[0] = n;
          cnt[1] = null_count;
          cnt[2] = survivors;
        }
      }
    }
    hw0 = hw1;
    blob0 = blob1;
    blob1 = blob2;
  }
}

static uint32_t str_like_smem(uint32_t dict_words) { return 8u * (16u + dict_words * 4u + kLikeCandCap * 2u); }

static uint32_t str_scan_smem(uint32_t needle_len, uint32_t dict_words, uint32_t stage, bool in_list) {
  const uint32_t nd = in_list ? kInTableBytes : (needle_len + 15u) & ~15u;
  const uint32_t fl = (2u * needle_len + 15u) & ~15u;
  return kScanFixedSmem + kStrScanTables + nd + fl + dict_words * 4u + (((dict_words * 64u) + 127u) & ~127u) + 128u +
         stage;
}

cudaError_t launch_str_scan(int mode, uint32_t n_entries, const ScanIo& io, const StrPredDesc& pred,
                            uint32_t max_head_bytes, uint32_t max_unique, uint32_t max_meta_bytes, cudaStream_t s) {
  if (n_entries == 0) return cudaSuccess;
  const uint32_t dict_words = ((max_unique + 31u) / 32u + 3u) & ~3u;
  constexpr uint32_t kMaxSmem = 227u * 1024u;
  static int n_sm = 0;
  if (!n_sm) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  }
  // the streaming LIKE kernel: substring needles the Shift-And walk covers, full-length outputs, heads that leave room for
  // at least two CTAs per SM with both stage buffers
  const bool like_op = pred.op == LC_OP_LIKE || pred.op == LC_OP_NOT_LIKE;
  const bool full_len = mode == MODE_REFINE || (mode == MODE_PRED && io.sel_base == nullptr);
  if (like_op && full_len && pred.needle_len >= 1u && pred.needle_len <= 31u && max_meta_bytes != 0u && pred.like_steps) {
    const uint32_t smem = str_like_smem(dict_words);
    if (smem <= 100u * 1024u) {
      // register budget: 4 CTAs per SM (64 registers) by default; LC_LIKE_OCC=3 selects the 80-register build (experiments)
      static const int occ_pref = [] {
        const char* e = std::getenv("LC_LIKE_OCC");
        return (e && e[0] == '3') ? 3 : 4;
      }();
      const bool aux = pred.op == LC_OP_NOT_LIKE || pred.prof != nullptr;
      auto kern3 = [&](int md, bool ax) -> void (*)(ScanIo, StrPredDesc, uint32_t, uint32_t, uint32_t) {
        if (occ_pref == 3) {
          if (ax) return md == MODE_PRED ? k_str_like<MODE_PRED, 3, true> : k_str_like<MODE_REFINE, 3, true>;
          return md == MODE_PRED ? k_str_like<MODE_PRED, 3, false> : k_str_like<MODE_REFINE, 3, false>;
        }
        if (ax) return md == MODE_PRED ? k_str_like<MODE_PRED, 4, true> : k_str_like<MODE_REFINE, 4, true>;
        return md == MODE_PRED ? k_str_like<MODE_PRED, 4, false> : k_str_like<MODE_REFINE, 4, false>;
      };
      auto kern = [&](int md) { return kern3(md, aux); };
      static bool like_attr = false;
      if (!like_attr) {
        for (int md : {static_cast<int>(MODE_PRED), static_cast<int>(MODE_REFINE)})
          for (bool ax : {false, true}) {
            cudaError_t e = cudaFuncSetAttribute(kern3(md, ax), cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
            if (e != cudaSuccess) return e;
          }
        like_attr = true;
      }
      int occ = 0;
      cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern(mode), 256, smem);
      if (e != cudaSuccess) return e;
      if (occ < 1) occ = 1;
      // A CTA's 8 warps share a run of neighbouring entries (same symbol table -> same step table in L1). Runs are short —
      // about four waves of CTAs — so that the hardware's CTA scheduler evens out entries that cost more (walks, rows).
      const uint32_t resident = static_cast<uint32_t>(n_sm * occ);
      static const uint32_t waves = [] {  // LC_LIKE_WAVES: CTA waves the list is cut into (experiments; default 4)
        const char* e = std::getenv("LC_LIKE_WAVES");
        const int v = e ? std::atoi(e) : 4;
        return static_cast<uint32_t>(v < 1 ? 1 : (v > 16 ? 16 : v));
      }();
      uint32_t per_cta = (n_entries + waves * resident - 1u) / (waves * resident);
      per_cta = (per_cta + 7u) & ~7u;  // whole rounds of the CTA's 8 warps
      const uint32_t grid = (n_entries + per_cta - 1u) / per_cta;
      kern(mode)<<<grid, 256, smem, s>>>(io, pred, dict_words, n_entries, per_cta);
      return cudaGetLastError();
    }
  }
  uint32_t stage = (max_head_bytes + 127u) & ~127u;
  const bool in_list = pred.op == LC_OP_IN || pred.op == LC_OP_NOT_IN;
  if (str_scan_smem(pred.needle_len, dict_words, stage, in_list) > 110u * 1024u) stage = 0;  // keep >= 2 CTAs per SM
  const uint32_t smem = str_scan_smem(pred.needle_len, dict_words, stage, in_list);
  if (smem > kMaxSmem) return cudaErrorInvalidValue;
  static bool attr_set = false;
  if (!attr_set) {
    for (auto k : {k_str_scan<MODE_PRED, false>, k_str_scan<MODE_REFINE, false>, k_str_scan<MODE_PRED, true>,
                   k_str_scan<MODE_REFINE, true>}) {
      cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
      if (e != cudaSuccess) return e;
    }
    attr_set = true;
  }
  // consecutive entries per CTA (table reuse), as long as the grid still covers the GPU several times over
  uint32_t per_cta = n_entries / (148u * 4u * 3u);
  per_cta = per_cta < 1u ? 1u : (per_cta > 4u ? 4u : per_cta);
  const uint32_t grid = (n_entries + per_cta - 1u) / per_cta;
  auto kern = in_list ? (mode == MODE_PRED ? k_str_scan<MODE_PRED, true> : k_str_scan<MODE_REFINE, true>)
                      : (mode == MODE_PRED ? k_str_scan<MODE_PRED, false> : k_str_scan<MODE_REFINE, false>);
  kern<<<grid, 256, smem, s>>>(io, pred, stage, dict_words, n_entries, per_cta);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// get / filter, pass 1: selected keys, decoded lengths, local offsets
// ------------------------------------------------------------------------------------------------
// One entry: selected keys, decoded lengths, local offsets. `phase` is the parity of the staging barrier (flipped by every
// staged entry of the CTA), `table_cache` the symbol table already in shared memory.
__device__ __forceinline__ void str_lengths_entry(const StrGatherIo& g, uint32_t e, uint32_t stage_cap, ScanSmem* sm, uint64_t* s_sym,
                                                  uint8_t* s_len, uint8_t* stage, uint32_t& phase, uint64_t& table_cache) {
  const EntryRef ref = g.io.refs[e];
  const EntryIo w = resolve_io(g.io, e);
  const bool staged = ref.head_bytes <= stage_cap;
  scan_smem_init(sm);
  if (threadIdx.x == 0 && staged) {
    mbar_expect_tx(&sm->bar[0], ref.head_bytes);
    tma_bulk_g2s(stage, ref.blob, ref.head_bytes, &sm->bar[0]);
  }
  __syncthreads();
  const uint8_t* head = ref.blob;
  if (staged) {
    mbar_wait(&sm->bar[0], phase);
    phase ^= 1u;
    head = stage;
  }
  const StrView v = make_view(head, ref.blob);
  if (v.h->table_ptr != table_cache) {
    load_fsst_table(reinterpret_cast<const FsstTable*>(v.h->table_ptr), s_sym, s_len);
    table_cache = v.h->table_ptr;
  }
  const uint32_t U = v.h->n_unique, spl = v.h->shared_prefix_len, n = v.h->n;
  uint32_t* row_off = g.row_off_base + g.row_base[e] + e;
  uint32_t* row_key = g.row_key_base + g.row_base[e];
  uint32_t* ulen = g.ulen_base + g.ulen_off[e];
  // how many rows are selected decides whether every unique's length is worth computing up front
  uint32_t k_sel = n;
  if (w.sel) {
    uint32_t c = 0;
    const uint32_t n_words = (n + 31u) >> 5, tail = n & 31u;
    for (uint32_t i = threadIdx.x; i < n_words; i += 256u) {
      uint32_t sw = w.sel[i];
      if (i == n_words - 1u && tail) sw &= (1u << tail) - 1u;
      c += __popc(sw);
    }
    c = warp_sum(c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&sm->misc[1], c);
    __syncthreads();
    k_sel = sm->misc[1];
  } else {
    __syncthreads();
  }
  const bool precomp = static_cast<uint64_t>(k_sel) * 4ull >= U;
  if (precomp) {
    // decoded length of every unique: PrefixKey.len when < 255, else walk the codes
    for (uint32_t i = threadIdx.x; i < U; i += 256u) {
      const uint32_t l = static_cast<uint32_t>(v.pk[i] >> 56);
      uint32_t len = spl + l;
      const uint32_t start = dict_offset(v, i), end = dict_offset(v, i + 1u);
      if (start == end) len = 0;  // empty value (fsst_buffer.rs:100-113)
      else if (l == 255u) len = decoded_length(v.fsst, start, end, s_len);
      ulen[i] = len;
    }
    __syncthreads();
  }
  const uint16_t* keys = v.keys;
  const uint32_t* valid = v.valid;
  auto cmp = [&](uint32_t, uint32_t, uint32_t) -> bool { return false; };
  auto emit = [&](uint32_t row, uint32_t dst, uint32_t, uint32_t) {
    const bool ok = valid ? ((valid[row >> 5] >> (row & 31u)) & 1u) : true;
    uint32_t len = 0, key = 0xFFFFFFFFu;
    if (ok) {
      key = keys[row];
      if (precomp) {
        len = ulen[key];
      } else {
        const uint32_t l = static_cast<uint32_t>(v.pk[key] >> 56);
        const uint32_t start = dict_offset(v, key), end = dict_offset(v, key + 1u);
        if (start == end) len = 0;
        else if (l == 255u) len = decoded_length(v.fsst, start, end, s_len);
        else len = spl + l;
      }
    }
    row_off[dst] = len;
    row_key[dst] = key;
  };
  scan_entry_rows<MODE_DECODE>(w.sel, n, valid, v.h->null_count, nullptr, w.out_valid, w.counts, sm, cmp, emit);
  __syncthreads();
  // exclusive scan of the selected rows' lengths -> local offsets (in place), total bytes
  const uint32_t k = w.counts[0];
  uint32_t carry = 0;
  for (uint32_t base = 0; base < k; base += 256u) {
    const uint32_t j = base + threadIdx.x;
    const uint32_t len = j < k ? row_off[j] : 0u;
    uint32_t tot;
    const uint32_t excl = block_excl_scan_256(len, sm->warp_tot, &tot);
    if (j < k) row_off[j] = carry + excl;
    carry += tot;
  }
  if (threadIdx.x == 0) {
    row_off[k] = carry;
    w.counts[2] = carry;
  }
}

// Host-planned gets launch one CTA per entry (per_cta = 1, no k_hint). Device-planned reads do not know on the host which
// entries have rows, so a CTA takes a RANGE of entries, looks at their survivor counts in one coalesced round and leaves
// at once when none of them is its business — the common case of a selective scan, where every batch with survivors has a
// handful and belongs to k_str_lengths_sparse (12 207 one-entry CTAs that only exit are not free).
__global__ void __launch_bounds__(256) k_str_lengths(StrGatherIo g, uint32_t stage_cap, uint32_t n_entries, uint32_t per_cta) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  ScanSmem* sm = reinterpret_cast<ScanSmem*>(smem_raw);
  uint64_t* s_sym = reinterpret_cast<uint64_t*>(smem_raw + kScanFixedSmem);
  uint8_t* s_len = reinterpret_cast<uint8_t*>(s_sym + 256);
  uint8_t* stage = s_len + 256;

  const uint32_t e_lo = blockIdx.x * per_cta, e_hi = min(n_entries, e_lo + per_cta);
  if (g.k_hint) {
    bool mine = false;
    for (uint32_t e = e_lo + threadIdx.x; e < e_hi; e += 256u) mine |= g.k_hint[2u * e] > g.sparse_max;
    if (!__syncthreads_or(mine) || g.plan->overflow) return;
  }
  if (threadIdx.x == 0) {
    mbar_init(&sm->bar[0], 1);
    fence_mbar_init();
  }
  __syncthreads();
  uint32_t phase = 0;
  uint64_t table_cache = 0;
  for (uint32_t e = e_lo; e < e_hi; ++e) {
    if (g.k_hint && g.k_hint[2u * e] <= g.sparse_max) continue;  // nothing selected, or k_str_lengths_sparse's
    str_lengths_entry(g, e, stage_cap, sm, s_sym, s_len, stage, phase, table_cache);
    __syncthreads();  // shared state (counters, staged head) is reused by the next entry
  }
}

// A selective scan leaves one or two rows in most of the batches it leaves any in (the bench column: 3 971 rows in 3 400 of
// 12 207 batches). Staging 30 KB of entry head and synchronising a CTA for that is all overhead, so such entries get ONE WARP each, reading only what the rows need: the selection words, the key,
// its PrefixKey (length byte) and its two offsets. Lists without nulls only (the device-planned read's precondition).
__global__ void __launch_bounds__(256) k_str_lengths_sparse(StrGatherIo g, uint32_t n_entries) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t e = blockIdx.x * 8u + (threadIdx.x >> 5);
  if (e >= n_entries) return;
  const uint32_t k = g.k_hint[2u * e];
  if (k == 0u || k > g.sparse_max || g.plan->overflow) return;
  const uint8_t* blob = g.io.refs[e].blob;
  const uint32_t hw = __ldg(reinterpret_cast<const uint32_t*>(blob) + lane);
  const uint32_t n = __shfl_sync(kFullMask, hw, 2), spl = __shfl_sync(kFullMask, hw, 6);
  const uint32_t keys_off = __shfl_sync(kFullMask, hw, 8), pk_off = __shfl_sync(kFullMask, hw, 9);
  const uint32_t resid_off = __shfl_sync(kFullMask, hw, 11), fsst_off = __shfl_sync(kFullMask, hw, 13);
  const uint64_t table_ptr = static_cast<uint64_t>(__shfl_sync(kFullMask, hw, 20)) | (static_cast<uint64_t>(__shfl_sync(kFullMask, hw, 21)) << 32);
  StrView v{};
  v.h = reinterpret_cast<const StrHeader*>(blob);
  v.resid = blob + resid_off;
  v.fsst = blob + fsst_off;
  const uint16_t* keys = reinterpret_cast<const uint16_t*>(blob + keys_off);
  const uint64_t* pk = reinterpret_cast<const uint64_t*>(blob + pk_off);
  const uint8_t* s_len = reinterpret_cast<const FsstTable*>(table_ptr)->lens;
  const uint32_t* sel = g.io.sel_base + g.io.sel_off[e];
  const uint64_t rb = g.row_base[e];
  uint32_t* row_off = g.row_off_base + rb + e;
  uint32_t* row_key = g.row_key_base + rb;
  // lane L owns the selection words [L * per, (L + 1) * per): set bits in order = rows in order
  const uint32_t n_words = (n + 31u) >> 5, per = (n_words + 31u) / 32u, tail = n & 31u;
  uint32_t cnt = 0;
  for (uint32_t q = 0; q < per; ++q) {
    const uint32_t wi = lane * per + q;
    if (wi >= n_words) break;
    uint32_t sw = sel[wi];
    if (wi == n_words - 1u && tail) sw &= (1u << tail) - 1u;
    cnt += __popc(sw);
  }
  uint32_t dst = warp_incl_scan(cnt, static_cast<int>(lane)) - cnt;
  if (cnt) {
    for (uint32_t q = 0; q < per; ++q) {
      const uint32_t wi = lane * per + q;
      if (wi >= n_words) break;
      uint32_t sw = sel[wi];
      if (wi == n_words - 1u && tail) sw &= (1u << tail) - 1u;
      while (sw) {
        const uint32_t b = __ffs(sw) - 1u;
        sw &= sw - 1u;
        const uint32_t key = keys[wi * 32u + b];
        const uint32_t l = static_cast<uint32_t>(pk[key] >> 56);
        const uint32_t start = dict_offset(v, key), end = dict_offset(v, key + 1u);
        uint32_t len = spl + l;
        if (start == end) len = 0;  // empty value (fsst_buffer.rs:100-113)
        else if (l == 255u) len = decoded_length(v.fsst, start, end, s_len);
        row_off[dst] = len;
        row_key[dst] = key;
        ++dst;
      }
    }
  }
  __syncwarp();
  // exclusive scan of the k lengths (k <= sparse_max, a few warp rounds), total bytes
  uint32_t carry = 0;
  for (uint32_t base = 0; base < k; base += 32u) {
    const uint32_t j = base + lane;
    const uint32_t len = j < k ? row_off[j] : 0u;
    const uint32_t incl = warp_incl_scan(len, static_cast<int>(lane));
    if (j < k) row_off[j] = carry + incl - len;
    carry += __shfl_sync(kFullMask, incl, 31);
  }
  if (lane == 0) {
    row_off[k] = carry;
    uint32_t* cnt4 = g.io.counts + static_cast<size_t>(e) * g.io.counts_stride;
    cnt4[0] = k;
    cnt4[1] = 0;
    cnt4[2] = carry;
  }
}

cudaError_t launch_str_lengths_sparse(uint32_t n_entries, const StrGatherIo& g, cudaStream_t s) {
  if (n_entries == 0 || g.sparse_max == 0) return cudaSuccess;
  k_str_lengths_sparse<<<(n_entries + 7u) / 8u, 256, 0, s>>>(g, n_entries);
  return cudaGetLastError();
}

cudaError_t launch_str_lengths(uint32_t n_entries, const StrGatherIo& g, uint32_t max_head_bytes, cudaStream_t s) {
  if (n_entries == 0) return cudaSuccess;
  uint32_t stage = (max_head_bytes + 127u) & ~127u;
  if (stage > kStageCap) stage = 0;
  const uint32_t smem = kScanFixedSmem + 2048u + 256u + stage;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(k_str_lengths, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kScanFixedSmem + 2304u + kStageCap);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  const uint32_t per_cta = g.k_hint ? (n_entries + 2367u) / 2368u : 1u;  // device-planned reads: entry ranges (see the kernel)
  k_str_lengths<<<(n_entries + per_cta - 1u) / per_cta, 256, smem, s>>>(g, stage, n_entries, per_cta);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// get / filter, pass 2: one warp per selected row, one lane per FSST code
// ------------------------------------------------------------------------------------------------
// fsst-rs Decompressor::decompress_into restated for a warp: lane p looks at compressed byte p of a
// 32-byte window; a byte is an escaped literal iff it is preceded by an odd run of unconsumed 0xFF
// bytes (ballot + clz), otherwise it is an escape marker (0xFF) or a code whose symbol length comes
// from the table; an exclusive scan of the produced lengths gives each lane its output position.
__device__ __forceinline__ uint32_t warp_decode(const uint8_t* __restrict__ c, uint32_t clen,
                                                uint8_t* __restrict__ out, const uint64_t* s_sym,
                                                const uint8_t* s_len, int lane) {
  uint32_t produced = 0;
  uint32_t carry_lit = 0;
  for (uint32_t base = 0; base < clen; base += 32u) {
    const uint32_t idx = base + lane;
    const bool in = idx < clen;
    const uint32_t b = in ? c[idx] : 0u;
    const uint32_t F = __ballot_sync(kFullMask, in && b == 255u);
    const uint32_t Fp = carry_lit ? (F & ~1u) : F;
    const uint32_t zeros = ~Fp & lanemask_lt();
    const uint32_t run = zeros ? (lane - 1u - (31u - __clz(zeros))) : static_cast<uint32_t>(lane);
    const bool lit = (lane == 0) ? (carry_lit != 0) : ((run & 1u) != 0);
    const bool esc = in && (b == 255u) && !lit;
    const uint32_t l = !in ? 0u : lit ? 1u : esc ? 0u : s_len[b];
    const uint32_t incl = warp_incl_scan(l, lane);
    if (l) {
      uint64_t val = lit ? static_cast<uint64_t>(b) : s_sym[b];
      uint8_t* o = out + produced + incl - l;
      for (uint32_t t = 0; t < l; ++t) {
        o[t] = static_cast<uint8_t>(val);
        val >>= 8;
      }
    }
    produced += __shfl_sync(kFullMask, incl, 31);
    carry_lit = __shfl_sync(kFullMask, esc ? 1u : 0u, 31);
  }
  return produced;
}

__device__ __forceinline__ void str_decode_entry(const StrGatherIo& g, uint32_t e, uint64_t* s_sym, uint8_t* s_len, uint32_t* s_wtot,
                                                 uint64_t& table_cache) {
  const uint32_t k = g.io.counts[static_cast<size_t>(e) * g.io.counts_stride];
  const EntryRef ref = g.io.refs[e];
  const StrView v = make_view(ref.blob, ref.blob);
  if (v.h->table_ptr != table_cache) {
    load_fsst_table(reinterpret_cast<const FsstTable*>(v.h->table_ptr), s_sym, s_len);
    table_cache = v.h->table_ptr;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint64_t rb = g.row_base[e];
  const uint32_t* row_off = g.row_off_base + rb + e;
  const uint32_t* row_key = g.row_key_base + rb;
  const uint32_t byte_base = static_cast<uint32_t>(g.byte_base[e]);
  int32_t* out_offsets = g.out_offsets + rb;
  // final offsets of this entry's slice (the closing offset of the whole array is written by the host)
  for (uint32_t j = threadIdx.x; j < k; j += 256u) out_offsets[j] = static_cast<int32_t>(byte_base + row_off[j]);
  if (g.dict_scratch && g.dict_base[e] != ~0ull) {
    // Dense get: decode every dictionary value once (the FSST work: ~35 codes per URL), then the rows are plain copies out
    // of the decoded dictionary — 8192 rows over ~1 750 values means 4-5 x less decoding than a decode per row.
    const uint32_t U = v.h->n_unique;
    uint32_t* ulen = g.ulen_base + g.ulen_off[e];  // pass 1 left every value's decoded length here: lengths -> offsets, in place
    uint32_t total = 0;
    for (uint32_t base = 0; base < U; base += 256u) {
      const uint32_t i = base + threadIdx.x;
      const uint32_t len = i < U ? ulen[i] : 0u;
      uint32_t tile;
      const uint32_t excl = block_excl_scan_256(len, s_wtot, &tile);
      if (i < U) ulen[i] = total + excl;
      total += tile;
    }
    __syncthreads();
    uint8_t* dict = g.dict_scratch + g.dict_base[e];
    for (uint32_t u = warp; u < U; u += 8u) {
      const uint32_t start = dict_offset(v, u), end = dict_offset(v, u + 1u);
      if (start != end) warp_decode(v.fsst + start, end - start, dict + ulen[u], s_sym, s_len, lane);
    }
    __syncthreads();
    for (uint32_t j = warp; j < k; j += 8u) {
      const uint32_t key = row_key[j];
      if (key == 0xFFFFFFFFu) continue;
      const uint32_t o0 = ulen[key], o1 = key + 1u < U ? ulen[key + 1u] : total;
      const uint8_t* src = dict + o0;
      uint8_t* dst = g.out_bytes + byte_base + row_off[j];
      for (uint32_t b = lane; b < o1 - o0; b += 32u) dst[b] = src[b];
    }
    return;
  }
  for (uint32_t j = warp; j < k; j += 8u) {
    const uint32_t key = row_key[j];
    if (key == 0xFFFFFFFFu) continue;
    const uint32_t start = dict_offset(v, key), end = dict_offset(v, key + 1u);
    if (start == end) continue;
    warp_decode(v.fsst + start, end - start, g.out_bytes + byte_base + row_off[j], s_sym, s_len, lane);
  }
}


// One CTA per entry for host-planned gets; a range of entries per CTA for device-planned reads, for the reason given at
// k_str_lengths. Entries with up to sparse_max survivors belong to k_str_decode_sparse there.
__global__ void __launch_bounds__(256) k_str_decode(StrGatherIo g, uint32_t n_entries, uint32_t per_cta) {
  __shared__ uint64_t s_sym[256];
  __shared__ __align__(16) uint8_t s_len[256];
  __shared__ uint32_t s_wtot[8];
  const uint32_t e_lo = blockIdx.x * per_cta, e_hi = min(n_entries, e_lo + per_cta);
  if (g.k_hint) {
    bool mine = false;
    for (uint32_t e = e_lo + threadIdx.x; e < e_hi; e += 256u) mine |= g.k_hint[2u * e] > g.sparse_max;
    if (!__syncthreads_or(mine) || g.plan->overflow) return;
  }
  uint64_t table_cache = 0;
  for (uint32_t e = e_lo; e < e_hi; ++e) {
    if (g.k_hint && g.k_hint[2u * e] <= g.sparse_max) continue;
    str_decode_entry(g, e, s_sym, s_len, s_wtot, table_cache);
    __syncthreads();
  }
}

// The rows k_str_lengths_sparse sized: one warp per entry again. The eight entries of a CTA nearly always share their
// compressor (one per column or row group), so its symbol table is loaded into shared memory once per CTA; a warp whose entry
// uses another table reads that one from global memory.
__global__ void __launch_bounds__(256) k_str_decode_sparse(StrGatherIo g, uint32_t n_entries) {
  __shared__ uint64_t s_sym[256];
  __shared__ __align__(16) uint8_t s_len[256];
  __shared__ uint64_t s_tab[8];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t e = blockIdx.x * 8u + warp;
  const uint32_t k = e < n_entries ? g.k_hint[2u * e] : 0u;
  const bool mine = k != 0u && k <= g.sparse_max;
  if (!__syncthreads_or(mine) || g.plan->overflow) return;
  const uint8_t* blob = nullptr;
  uint32_t resid_off = 0, fsst_off = 0;
  uint64_t table_ptr = 0;
  if (mine) {
    blob = g.io.refs[e].blob;
    const uint32_t hw = __ldg(reinterpret_cast<const uint32_t*>(blob) + lane);
    resid_off = __shfl_sync(kFullMask, hw, 11);
    fsst_off = __shfl_sync(kFullMask, hw, 13);
    table_ptr = static_cast<uint64_t>(__shfl_sync(kFullMask, hw, 20)) | (static_cast<uint64_t>(__shfl_sync(kFullMask, hw, 21)) << 32);
  }
  if (lane == 0) s_tab[warp] = table_ptr;
  __syncthreads();
  uint64_t cta_table = 0;
#pragma unroll
  for (int w = 7; w >= 0; --w)
    if (s_tab[w]) cta_table = s_tab[w];
  load_fsst_table(reinterpret_cast<const FsstTable*>(cta_table), s_sym, s_len);
  __syncthreads();
  if (!mine) return;
  const FsstTable* gt = reinterpret_cast<const FsstTable*>(table_ptr);
  const uint64_t* sym = table_ptr == cta_table ? s_sym : gt->symbols;
  const uint8_t* len = table_ptr == cta_table ? s_len : gt->lens;
  StrView v{};
  v.h = reinterpret_cast<const StrHeader*>(blob);
  v.resid = blob + resid_off;
  v.fsst = blob + fsst_off;
  const uint64_t rb = g.row_base[e];
  const uint32_t* row_off = g.row_off_base + rb + e;
  const uint32_t* row_key = g.row_key_base + rb;
  const uint32_t byte_base = static_cast<uint32_t>(g.byte_base[e]);
  int32_t* out_offsets = g.out_offsets + rb;
  for (uint32_t j = lane; j < k; j += 32u) out_offsets[j] = static_cast<int32_t>(byte_base + row_off[j]);
  for (uint32_t j = 0; j < k; ++j) {
    const uint32_t key = row_key[j];
    const uint32_t start = dict_offset(v, key), end = dict_offset(v, key + 1u);
    if (start == end) continue;
    warp_decode(v.fsst + start, end - start, g.out_bytes + byte_base + row_off[j], sym, len, static_cast<int>(lane));
  }
}

// grid of the two gather kernels: one CTA per entry when the host planned the get; for device-planned reads about sixteen
// CTAs per SM's worth of entry ranges, so that a list whose entries all have rows still fills the machine
// ------------------------------------------------------------------------------------------------
// get / filter of a SELECTIVE scan in one pass: the survivors of every entry, their offsets and their decoded bytes, written
// at their final positions of the concatenated Arrow array by ONE kernel.
//
// The device-planned read above is six dependent launches (row plan, lengths x 2, byte plan, decode x 2): right for reads
// that move data, but a selective LIKE leaves a handful of rows per batch and the read then costs more than the predicate
// (launches and drains). Where each entry's rows and bytes start is a
// prefix sum over the entries; here it is a single-pass chained scan (decoupled look-back) across the CTAs of the same
// kernel that decodes: a CTA takes eight entries (a warp each), sizes their survivors, publishes its (rows, bytes)
// aggregate, reads its predecessors' until it meets an inclusive prefix, and writes. CTAs take their position from a ticket
// so that every predecessor a CTA waits for is already running. Any number of survivors per entry is handled — up to 64 are
// kept in shared memory between the two phases, more are sized and then decoded again by the lane that owns them — but the
// host only picks this kernel when the previous read of the scan was sparse.
// Status word: flag (2 bits: 1 = aggregate, 2 = inclusive prefix) | rows (30 bits) | bytes (32 bits), both saturating —
// a saturated total is over every capacity and reported as such.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kOnePassKeep = 64;
constexpr unsigned long long kOpRowsMax = (1ull << 30) - 1ull, kOpBytesMax = 0xffffffffull;

__device__ __forceinline__ unsigned long long ld_relaxed_gpu(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_gpu(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long op_pack(uint32_t flag, unsigned long long rows, unsigned long long bytes) {
  rows = rows > kOpRowsMax ? kOpRowsMax : rows;
  bytes = bytes > kOpBytesMax ? kOpBytesMax : bytes;
  return (static_cast<unsigned long long>(flag) << 62) | (rows << 32) | bytes;
}

// One entry as the read sees it (header words pulled apart once per phase).
struct OpEntry {
  StrView v;
  const uint16_t* keys;
  const uint64_t* pk;
  const uint32_t* sel;
  const FsstTable* table;
  uint32_t n_words, per, tail, spl;
};
__device__ __forceinline__ OpEntry op_entry(const uint8_t* blob, const uint32_t* sel, uint32_t lane) {
  OpEntry x{};
  const uint32_t hw = __ldg(reinterpret_cast<const uint32_t*>(blob) + lane);
  const uint32_t n = __shfl_sync(kFullMask, hw, 2);
  x.spl = __shfl_sync(kFullMask, hw, 6);
  x.table = reinterpret_cast<const FsstTable*>(static_cast<uint64_t>(__shfl_sync(kFullMask, hw, 20)) |
                                               (static_cast<uint64_t>(__shfl_sync(kFullMask, hw, 21)) << 32));
  x.v.h = reinterpret_cast<const StrHeader*>(blob);
  x.v.resid = blob + __shfl_sync(kFullMask, hw, 11);
  x.v.fsst = blob + __shfl_sync(kFullMask, hw, 13);
  x.keys = reinterpret_cast<const uint16_t*>(blob + __shfl_sync(kFullMask, hw, 8));
  x.pk = reinterpret_cast<const uint64_t*>(blob + __shfl_sync(kFullMask, hw, 9));
  x.sel = sel;
  // lane L owns the selection words [L * per, (L + 1) * per): set bits in order = rows in order
  x.n_words = (n + 31u) >> 5;
  x.per = (x.n_words + 31u) / 32u;
  x.tail = n & 31u;
  return x;
}
__device__ __forceinline__ uint32_t op_sel_word(const OpEntry& x, uint32_t wi) {
  uint32_t sw = x.sel[wi];
  if (wi == x.n_words - 1u && x.tail) sw &= (1u << x.tail) - 1u;
  return sw;
}
__device__ __forceinline__ uint32_t op_value_len(const OpEntry& x, uint32_t key, uint32_t* start_out, uint32_t* end_out) {
  const uint32_t l = static_cast<uint32_t>(x.pk[key] >> 56);
  const uint32_t start = dict_offset(x.v, key), end = dict_offset(x.v, key + 1u);
  *start_out = start;
  *end_out = end;
  if (start == end) return 0u;  // empty value (fsst_buffer.rs:100-113)
  return l == 255u ? decoded_length(x.v.fsst, start, end, x.table->lens) : x.spl + l;
}
// Visits the lane's surviving rows in order: f(row position inside the entry, key).
template <typename F>
__device__ __forceinline__ void op_lane_rows(const OpEntry& x, uint32_t lane, uint32_t first_pos, F&& f) {
  uint32_t pos = first_pos;
  for (uint32_t q = 0; q < x.per; ++q) {
    const uint32_t wi = lane * x.per + q;
    if (wi >= x.n_words) break;
    uint32_t sw = op_sel_word(x, wi);
    while (sw) {
      const uint32_t b = __ffs(sw) - 1u;
      sw &= sw - 1u;
      f(pos++, static_cast<uint32_t>(x.keys[wi * 32u + b]));
    }
  }
}
__device__ __forceinline__ uint32_t op_lane_count(const OpEntry& x, uint32_t lane) {
  uint32_t c = 0;
  for (uint32_t q = 0; q < x.per; ++q) {
    const uint32_t wi = lane * x.per + q;
    if (wi >= x.n_words) break;
    c += __popc(op_sel_word(x, wi));
  }
  return c;
}
__device__ __forceinline__ unsigned long long warp_excl_scan64(unsigned long long v, uint32_t lane, unsigned long long* total) {
  unsigned long long incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long y = __shfl_up_sync(kFullMask, incl, d);
    if (lane >= static_cast<uint32_t>(d)) incl += y;
  }
  *total = __shfl_sync(kFullMask, incl, 31);
  return incl - v;
}

// A CTA takes 32 consecutive entries, four per warp: a selective scan leaves most of them without a survivor, and a warp
// that steps over its empty entries keeps the grid within ONE wave of the GPU for a 12 k-entry list (382 CTAs). That matters
// because nothing can be written before every predecessor has sized its survivors — with one entry per warp the kernel ran
// as three waves, each waiting for its slowest chain of dependent loads (polls of predecessors' status words).
constexpr uint32_t kOpPerWarp = 4, kOpPerCta = 8u * kOpPerWarp;

__global__ void __launch_bounds__(256) k_str_read_onepass(StrGatherIo g, uint32_t n_entries, unsigned long long cap_rows,
                                                          unsigned long long cap_bytes, ScanPlanHdr* hdr,
                                                          unsigned long long* status, uint32_t* ticket) {
  __shared__ uint32_t s_off[8][kOpPerWarp][kOnePassKeep + 1], s_key[8][kOpPerWarp][kOnePassKeep];
  __shared__ uint32_t s_rows[kOpPerCta], s_bytes[kOpPerCta];
  __shared__ uint32_t s_cta;
  __shared__ unsigned long long s_lb_rows[8], s_lb_bytes[8];
  __shared__ uint32_t s_lb_has[8];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_cta = atomicAdd(ticket, 1u);
  __syncthreads();
  const uint32_t cta = s_cta, n_cta = gridDim.x;
  const uint32_t e0 = cta * kOpPerCta + warp * kOpPerWarp;
  // what the warp's entries start from, requested together: lane j < 4 holds entry e0 + j
  uint32_t my_k = 0;
  const uint8_t* my_blob = nullptr;
  uint64_t my_sel_off = 0;
  if (lane < kOpPerWarp && e0 + lane < n_entries) {
    my_k = g.k_hint[2u * (e0 + lane)];
    my_blob = g.io.refs[e0 + lane].blob;
    my_sel_off = g.io.sel_off[e0 + lane];
  }
  uint32_t k[kOpPerWarp];
  unsigned long long total[kOpPerWarp];

  // ---- phase 1: the survivors of each entry and their decoded lengths ----
#pragma unroll
  for (uint32_t t = 0; t < kOpPerWarp; ++t) {
    k[t] = __shfl_sync(kFullMask, my_k, t);
    total[t] = 0;
    if (k[t]) {  // warp-uniform
      const uint8_t* blob = reinterpret_cast<const uint8_t*>(__shfl_sync(kFullMask, reinterpret_cast<unsigned long long>(my_blob), t));
      const OpEntry x = op_entry(blob, g.io.sel_base + __shfl_sync(kFullMask, static_cast<unsigned long long>(my_sel_off), t), lane);
      const uint32_t lane_rows = op_lane_count(x, lane);
      const uint32_t lane_row0 = warp_incl_scan(lane_rows, static_cast<int>(lane)) - lane_rows;
      const bool keep = k[t] <= kOnePassKeep;
      unsigned long long lane_bytes = 0;
      if (lane_rows)
        op_lane_rows(x, lane, lane_row0, [&](uint32_t pos, uint32_t key) {
          uint32_t st, en;
          const uint32_t len = op_value_len(x, key, &st, &en);
          if (keep && pos < kOnePassKeep) {
            s_off[warp][t][pos] = len;
            s_key[warp][t][pos] = key;
          }
          lane_bytes += len;
        });
      __syncwarp();
      if (keep) {  // lengths -> offsets inside the entry
        uint32_t carry = 0;
        for (uint32_t base = 0; base < k[t]; base += 32u) {
          const uint32_t j = base + lane;
          const uint32_t len = j < k[t] ? s_off[warp][t][j] : 0u;
          const uint32_t incl = warp_incl_scan(len, static_cast<int>(lane));
          if (j < k[t]) s_off[warp][t][j] = carry + incl - len;
          carry += __shfl_sync(kFullMask, incl, 31);
        }
        total[t] = carry;
      } else {
        warp_excl_scan64(lane_bytes, lane, &total[t]);
      }
    }
    if (lane == 0) {
      s_rows[warp * kOpPerWarp + t] = k[t];
      s_bytes[warp * kOpPerWarp + t] = total[t] > kOpBytesMax ? 0xffffffffu : static_cast<uint32_t>(total[t]);
    }
  }
  __syncthreads();

  // ---- the chained scan across CTAs ----
  // Every thread looks at one predecessor per round (256 status words at a time, nearest first); all threads compute the same
  // sums from the same shared words, so nothing is broadcast afterwards.
  unsigned long long agg_rows = 0, agg_bytes = 0;
#pragma unroll
  for (uint32_t w = 0; w < kOpPerCta; ++w) {
    agg_rows += s_rows[w];
    agg_bytes += s_bytes[w];
  }
  if (threadIdx.x == 0 && cta != 0u) st_relaxed_gpu(status + cta, op_pack(1u, agg_rows, agg_bytes));
  unsigned long long ex_rows = 0, ex_bytes = 0;
  for (int64_t j = static_cast<int64_t>(cta) - 1; j >= 0; j -= 256) {
    const int64_t idx = j - static_cast<int64_t>(threadIdx.x);
    unsigned long long w = 2ull << 62;  // before the first CTA: an inclusive prefix of nothing
    if (idx >= 0) {
      w = ld_relaxed_gpu(status + idx);
      while ((w >> 62) == 0ull) {  // a predecessor still sizing its entries
        __nanosleep(32);
        w = ld_relaxed_gpu(status + idx);
      }
    }
    const uint32_t m2 = __ballot_sync(kFullMask, (w >> 62) == 2ull);
    const uint32_t first = m2 ? static_cast<uint32_t>(__ffs(m2)) - 1u : 32u;  // the nearest predecessor of this warp's 32 holding a prefix
    unsigned long long r = lane <= first ? ((w >> 32) & kOpRowsMax) : 0ull, b = lane <= first ? (w & kOpBytesMax) : 0ull;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      r += __shfl_xor_sync(kFullMask, r, d);
      b += __shfl_xor_sync(kFullMask, b, d);
    }
    if (lane == 0) {
      s_lb_rows[warp] = r;
      s_lb_bytes[warp] = b;
      s_lb_has[warp] = m2 != 0u;
    }
    __syncthreads();
    bool found = false;
#pragma unroll
    for (int w8 = 0; w8 < 8; ++w8) {
      if (!found) {
        ex_rows += s_lb_rows[w8];
        ex_bytes += s_lb_bytes[w8];
        found = s_lb_has[w8] != 0u;
      }
    }
    __syncthreads();  // the shared words are rewritten by the next round
    if (found) break;
  }
  if (threadIdx.x == 0) {
    st_relaxed_gpu(status + cta, op_pack(2u, ex_rows + agg_rows, ex_bytes + agg_bytes));
    if (cta == n_cta - 1u) {  // the grand totals: header and closing offset
      const unsigned long long rows = ex_rows + agg_rows, bytes = ex_bytes + agg_bytes;
      hdr->n_hit = 0;
      hdr->rows = rows;
      hdr->bytes = bytes;
      hdr->nulls = 0;
      hdr->ulen_words = 0;
      hdr->vwords = 0;
      if (rows > cap_rows || rows >= kOpRowsMax) atomicMax(&hdr->overflow, 1u);
      else if (bytes > cap_bytes || bytes > 0x7fffffffull) atomicMax(&hdr->overflow, 2u);
      else g.out_offsets[rows] = static_cast<int32_t>(bytes);
    }
  }

  // ---- phase 2: offsets and bytes at their final positions ----
  unsigned long long row_base = ex_rows, byte_base = ex_bytes;
  for (uint32_t w = 0; w < warp * kOpPerWarp; ++w) {
    row_base += s_rows[w];
    byte_base += s_bytes[w];
  }
#pragma unroll
  for (uint32_t t = 0; t < kOpPerWarp; ++t) {
    if (!k[t]) continue;
    const unsigned long long rb = row_base, bb = byte_base;
    row_base += k[t];
    byte_base += s_bytes[warp * kOpPerWarp + t];
    if (rb + k[t] > cap_rows || bb + total[t] > cap_bytes || bb + total[t] > 0x7fffffffull) continue;  // the last CTA reports it
    const uint8_t* blob = reinterpret_cast<const uint8_t*>(__shfl_sync(kFullMask, reinterpret_cast<unsigned long long>(my_blob), t));
    const OpEntry x = op_entry(blob, g.io.sel_base + __shfl_sync(kFullMask, static_cast<unsigned long long>(my_sel_off), t), lane);
    int32_t* out_offsets = g.out_offsets + rb;
    uint8_t* out_bytes = g.out_bytes + bb;
    if (k[t] <= kOnePassKeep) {
      // (the symbol table is read through L1: neighbouring entries share it)
      for (uint32_t j = lane; j < k[t]; j += 32u) out_offsets[j] = static_cast<int32_t>(bb + s_off[warp][t][j]);
      for (uint32_t j = 0; j < k[t]; ++j) {
        const uint32_t key = s_key[warp][t][j];
        const uint32_t start = dict_offset(x.v, key), end = dict_offset(x.v, key + 1u);
        if (start == end) continue;
        warp_decode(x.v.fsst + start, end - start, out_bytes + s_off[warp][t][j], x.table->symbols, x.table->lens, static_cast<int>(lane));
      }
    } else {
      // more survivors than the warp keeps: each lane sizes its own rows again, then decodes them itself
      const uint32_t lane_rows = op_lane_count(x, lane);
      const uint32_t lane_row0 = warp_incl_scan(lane_rows, static_cast<int>(lane)) - lane_rows;
      unsigned long long lane_bytes = 0, unused;
      op_lane_rows(x, lane, lane_row0, [&](uint32_t, uint32_t key) {
        uint32_t st, en;
        lane_bytes += op_value_len(x, key, &st, &en);
      });
      unsigned long long off = warp_excl_scan64(lane_bytes, lane, &unused);
      op_lane_rows(x, lane, lane_row0, [&](uint32_t pos, uint32_t key) {
        uint32_t st, en;
        const uint32_t len = op_value_len(x, key, &st, &en);
        out_offsets[pos] = static_cast<int32_t>(bb + off);
        uint8_t* o = out_bytes + off;
        if (len) decode_visit(x.v.fsst, st, en, x.table->symbols, x.table->lens, [&](uint32_t byte) {
          *o++ = static_cast<uint8_t>(byte);
          return true;
        });
        off += len;
      });
    }
  }
}

// `d_status`: (grid + 1) 64-bit words of scratch owned by the caller's read state (status words, then the ticket).
cudaError_t launch_str_read_onepass(uint32_t n_entries, const StrGatherIo& g, uint64_t cap_rows, uint64_t cap_bytes, ScanPlanHdr* d_hdr,
                                    unsigned long long* d_status, cudaStream_t s) {
  if (n_entries == 0) return cudaErrorInvalidValue;
  const uint32_t grid = (n_entries + kOpPerCta - 1u) / kOpPerCta;
  cudaError_t e = cudaMemsetAsync(d_status, 0, (static_cast<size_t>(grid) + 1u) * 8u, s);
  if (e != cudaSuccess) return e;
  e = cudaMemsetAsync(d_hdr, 0, sizeof(ScanPlanHdr), s);
  if (e != cudaSuccess) return e;
  k_str_read_onepass<<<grid, 256, 0, s>>>(g, n_entries, cap_rows, cap_bytes, d_hdr, d_status,
                                          reinterpret_cast<uint32_t*>(d_status + grid));
  return cudaGetLastError();
}

static inline uint32_t gather_per_cta(uint32_t n_entries, const StrGatherIo& g) { return g.k_hint ? (n_entries + 2367u) / 2368u : 1u; }

cudaError_t launch_str_decode(uint32_t n_entries, const StrGatherIo& g, cudaStream_t s) {
  if (n_entries == 0) return cudaSuccess;
  if (g.k_hint && g.sparse_max) k_str_decode_sparse<<<(n_entries + 7u) / 8u, 256, 0, s>>>(g, n_entries);
  const uint32_t per_cta = gather_per_cta(n_entries, g);
  k_str_decode<<<(n_entries + per_cta - 1u) / per_cta, 256, 0, s>>>(g, n_entries, per_cta);
  return cudaGetLastError();
}

}  // namespace lc

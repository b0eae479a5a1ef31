// k_num.cu — ALP floats and u64 decimals on top of the bit-packed integer entry (sm_90a).
//
// Reference semantics restated (all under /root/reference/src/core/src/liquid_array/):
//   float encode   get_best_exponents + encode_arrow_array            float_array.rs:609-751
//   float decode   LiquidFloatArray::to_arrow_array (+ patches)        float_array.rs:293-316
//   float filter / try_eval_predicate: trait defaults (decode, arrow filter, DataFusion compare)   mod.rs:116-130
//   decimal        LiquidDecimalArray::{fits_u64, from_decimal_array, to_arrow_array}   decimal_array.rs:127-178, 293-309
//
// A float entry is an integer entry whose packed words hold the ALP-encoded signed integers minus their minimum;
// a decimal entry is a u64 integer entry. k_int_scan<DECODE> (k_int.cu) therefore does the unpacking and the
// selection -> write-offset compaction for both; the kernels here are the thin, purely HBM-bound passes on either
// side of it: integers -> floats in place + patches, float compares on the decoded values, and the 128/256-bit
// widening of decimals. No tensor cores: there is no contraction anywhere on this path.
#include <type_traits>

#include "alp_math.cuh"
#include "squeeze_math.cuh"
#include "device_utils.cuh"
#include "kernels.h"

namespace lc {

namespace {
constexpr long long kI64Max = 0x7fffffffffffffffLL;
constexpr long long kI64Min = -kI64Max - 1;

__device__ __forceinline__ long long warp_min_ll(long long v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const long long o = __shfl_xor_sync(kFullMask, v, d);
    v = o < v ? o : v;
  }
  return v;
}
__device__ __forceinline__ long long warp_max_ll(long long v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const long long o = __shfl_xor_sync(kFullMask, v, d);
    v = o > v ? o : v;
  }
  return v;
}

// (e, f) of position `idx` in the loop `for e in 0..MAX { for f in 0..e { .. } }`
__device__ __forceinline__ void combo_exponents(uint32_t idx, uint32_t* e_out, uint32_t* f_out) {
  uint32_t e = 1;
  while (idx >= e) {
    idx -= e;
    ++e;
  }
  *e_out = e;
  *f_out = idx;
}
}  // namespace

// ------------------------------------------------------------------------------------------------
// get_best_exponents: one CTA per (e, f) pair encodes the sample and reports the size the reference's
// get_array_memory_size would give for it (only the terms that differ between pairs: packed words + patch vectors).
// ------------------------------------------------------------------------------------------------
template <typename F>
__global__ void __launch_bounds__(256) k_alp_search(AlpEncIo io) {
  using A = Alp<F>;
  using I = typename A::I;
  using U = typename A::U;
  __shared__ long long s_ll[8][4];
  __shared__ uint32_t s_u[8][2];
  uint32_t e, f;
  combo_exponents(blockIdx.x, &e, &f);
  const F* __restrict__ v = reinterpret_cast<const F*>(io.values);
  uint32_t m = 0, pc = 0;
  long long ok_min = kI64Max, ok_max = kI64Min, all_min = kI64Max, all_max = kI64Min;
  for (uint32_t i = threadIdx.x; i < io.sample_cnt; i += 256u) {
    const uint32_t row = io.sample_step ? i * io.sample_step : i;
    // the strided sample keeps only non-null slots (`.filter(|s| s.is_some())`); an array of <= 1024 rows is
    // encoded as it is, null slots included
    if (io.sample_step && io.validity && !((io.validity[row >> 5] >> (row & 31u)) & 1u)) continue;
    const F x = v[row];
    const I enc = A::encode(x, e, f);
    const F dec = A::decode(enc, e, f);
    const long long w = static_cast<long long>(enc);
    ++m;
    all_min = w < all_min ? w : all_min;
    all_max = w > all_max ? w : all_max;
    if (dec == x) {  // `decoded.eq(&v)`: IEEE equality, so NaN is always a patch and -0.0 never is
      ok_min = w < ok_min ? w : ok_min;
      ok_max = w > ok_max ? w : ok_max;
    } else {
      ++pc;
    }
  }
  ok_min = warp_min_ll(ok_min);
  ok_max = warp_max_ll(ok_max);
  all_min = warp_min_ll(all_min);
  all_max = warp_max_ll(all_max);
  m = warp_sum(m);
  pc = warp_sum(pc);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    s_ll[warp][0] = ok_min;
    s_ll[warp][1] = ok_max;
    s_ll[warp][2] = all_min;
    s_ll[warp][3] = all_max;
    s_u[warp][0] = m;
    s_u[warp][1] = pc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) {
      ok_min = s_ll[w][0] < ok_min ? s_ll[w][0] : ok_min;
      ok_max = s_ll[w][1] > ok_max ? s_ll[w][1] : ok_max;
      all_min = s_ll[w][2] < all_min ? s_ll[w][2] : all_min;
      all_max = s_ll[w][3] > all_max ? s_ll[w][3] : all_max;
      m += s_u[w][0];
      pc += s_u[w][1];
    }
    unsigned long long size = 0;
    if (m) {
      // patched slots take the first good value before min/max are taken (float_array.rs:663-690), unless every
      // slot is a patch
      const bool partial = pc > 0 && pc < m;
      const I lo = static_cast<I>(partial ? ok_min : all_min), hi = static_cast<I>(partial ? ok_max : all_max);
      const U sub = static_cast<U>(static_cast<U>(hi) - static_cast<U>(lo));  // max.sub_wrapping(min) as unsigned
      const uint32_t W = bit_width_of_u64(static_cast<unsigned long long>(sub));
      const uint32_t chunks = (m + 1023u) / 1024u;
      size = static_cast<unsigned long long>(chunks) * 128ull * W;
      if (pc) {
        // Vec::resize_with(patch_count + 1) on an empty Vec: capacity max(4, patch_count + 1), for the u64 indices
        // and the native values alike
        const unsigned long long cap = pc + 1u > 4u ? pc + 1u : 4u;
        size += cap * (8ull + sizeof(F));
      }
    }
    io.sizes[blockIdx.x] = size;
    if (blockIdx.x == 0) {
      io.res->n_patches = 0;
      io.res->first_ok = 0xFFFFFFFFu;
    }
  }
}

// encode_arrow_array, pass 1: every slot encoded with the best pair (first minimum in loop order), patch flags as
// bit words, patch count, first slot that is not a patch.
template <typename F>
__global__ void __launch_bounds__(256) k_alp_encode(AlpEncIo io) {
  using A = Alp<F>;
  using I = typename A::I;
  __shared__ uint32_t s_ef[2];
  if (threadIdx.x == 0) {
    uint32_t best = 0;
    unsigned long long best_size = io.sizes[0];
    for (uint32_t c = 1; c < alp_n_combos<F>(); ++c) {
      const unsigned long long sz = io.sizes[c];
      if (sz < best_size) {  // strict: ties keep the earlier pair (float_array.rs:738-741)
        best_size = sz;
        best = c;
      }
    }
    uint32_t e, f;
    combo_exponents(best, &e, &f);
    s_ef[0] = e;
    s_ef[1] = f;
    if (blockIdx.x == 0) {
      io.res->e = e;
      io.res->f = f;
    }
  }
  __syncthreads();
  const uint32_t e = s_ef[0], f = s_ef[1];
  const F* __restrict__ v = reinterpret_cast<const F*>(io.values);
  I* __restrict__ enc_out = reinterpret_cast<I*>(io.enc);
  const uint32_t n = io.n, n_pad = (n + 31u) & ~31u;
  const int lane = threadIdx.x & 31;
  for (uint32_t i = blockIdx.x * 256u + threadIdx.x; i < n_pad; i += gridDim.x * 256u) {
    const bool in = i < n;
    bool exc = false;
    if (in) {
      const F x = v[i];
      const I enc = A::encode(x, e, f);
      exc = !(A::decode(enc, e, f) == x);
      enc_out[i] = enc;
    }
    const uint32_t xm = __ballot_sync(kFullMask, exc);
    const uint32_t om = __ballot_sync(kFullMask, in && !exc);
    if (lane == 0) {
      io.exc_words[i >> 5] = xm;
      if (xm) atomicAdd(&io.res->n_patches, static_cast<uint32_t>(__popc(xm)));
      if (om) atomicMin(&io.res->first_ok, i + static_cast<uint32_t>(__ffs(om) - 1));
    }
  }
}

// encode_arrow_array, pass 2 (one CTA, rows in order): patch list in ascending row order, patched slots replaced by
// the fill value, then min / max of what will be packed.
template <typename F>
__global__ void __launch_bounds__(1024) k_alp_patches(AlpEncIo io) {
  using I = typename Alp<F>::I;
  __shared__ uint32_t s_wtot[32];
  __shared__ long long s_mn[32], s_mx[32];
  const uint32_t n = io.n, pc = io.res->n_patches, first_ok = io.res->first_ok;
  I* __restrict__ enc = reinterpret_cast<I*>(io.enc);
  const F* __restrict__ v = reinterpret_cast<const F*>(io.values);
  F* __restrict__ pv = reinterpret_cast<F*>(io.patch_val);
  const bool fill_on = pc > 0 && pc < n;  // float_array.rs:663
  const I fill = fill_on ? enc[first_ok] : static_cast<I>(0);  // a good slot: never overwritten below
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t carry = 0;
  long long mn = kI64Max, mx = kI64Min;
  for (uint32_t base = 0; base < n; base += 1024u) {
    const uint32_t i = base + threadIdx.x;
    const bool in = i < n;
    const bool flag = in && ((io.exc_words[i >> 5] >> (i & 31u)) & 1u);
    const uint32_t bal = __ballot_sync(kFullMask, flag);
    if (lane == 0) s_wtot[warp] = __popc(bal);
    __syncthreads();
    uint32_t wbase = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < 32; ++w) {
      const uint32_t t = s_wtot[w];
      if (w < warp) wbase += t;
      tot += t;
    }
    if (in) {
      I w = enc[i];
      if (flag) {
        const uint32_t pos = carry + wbase + __popc(bal & lanemask_lt());
        io.patch_idx[pos] = i;
        pv[pos] = v[i];
        if (fill_on) {
          w = fill;
          enc[i] = fill;
        }
      }
      const long long wl = static_cast<long long>(w);
      mn = wl < mn ? wl : mn;
      mx = wl > mx ? wl : mx;
    }
    carry += tot;
    __syncthreads();  // s_wtot is rewritten next round
  }
  mn = warp_min_ll(mn);
  mx = warp_max_ll(mx);
  if (lane == 0) {
    s_mn[warp] = mn;
    s_mx[warp] = mx;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 32; ++w) {
      mn = s_mn[w] < mn ? s_mn[w] : mn;
      mx = s_mx[w] > mx ? s_mx[w] : mx;
    }
    io.res->min = mn;
    io.res->max = mx;
  }
}

cudaError_t launch_alp_encode(const AlpEncIo& io, cudaStream_t s) {
  if (io.n == 0) return cudaSuccess;
  uint32_t grid = (io.n + 255u) / 256u;
  if (grid > kGridStrideCap) grid = kGridStrideCap;
  if (io.is_f64) {
    k_alp_search<double><<<alp_n_combos<double>(), 256, 0, s>>>(io);
    k_alp_encode<double><<<grid, 256, 0, s>>>(io);
    k_alp_patches<double><<<1, 1024, 0, s>>>(io);
  } else {
    k_alp_search<float><<<alp_n_combos<float>(), 256, 0, s>>>(io);
    k_alp_encode<float><<<grid, 256, 0, s>>>(io);
    k_alp_patches<float><<<1, 1024, 0, s>>>(io);
  }
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// to_arrow_array / filter, second half: k_int_scan<DECODE> left `reference + packed` (the ALP integers) of the
// selected rows at out_off; convert in place, then drop the patches of the selected rows at their ranks.
// ------------------------------------------------------------------------------------------------
template <typename F>
__global__ void __launch_bounds__(256) k_alp_finish(ScanIo io) {
  using A = Alp<F>;
  using I = typename A::I;
  __shared__ uint32_t s_tot[8];
  __shared__ uint32_t s_word[256];
  __shared__ uint32_t s_off[256];
  const uint32_t ent = blockIdx.x;
  const EntryRef ref = io.refs[ent];
  const IntHeader* __restrict__ h = reinterpret_cast<const IntHeader*>(ref.blob);
  const uint32_t k = io.counts[static_cast<size_t>(ent) * io.counts_stride];
  I* __restrict__ out = reinterpret_cast<I*>(io.out_base) + io.out_off[ent];
  const uint32_t e = h->alp_ef & 0xffu, f = (h->alp_ef >> 8) & 0xffu;
  for (uint32_t i = threadIdx.x; i < k; i += 256u) out[i] = A::bits(A::decode(out[i], e, f));
  const uint32_t pc = h->n_patches;
  if (pc == 0 || h->bit_width == 0) return;
  __syncthreads();  // the patches land on slots other threads converted
  const uint32_t* __restrict__ pidx = reinterpret_cast<const uint32_t*>(ref.blob + h->patch_idx_off);
  const I* __restrict__ pval = reinterpret_cast<const I*>(ref.blob + h->patch_val_off);
  const uint32_t* sel = nullptr;
  if (io.sel_base) {
    const uint64_t so = io.sel_off[ent];
    if (so != kNoSel) sel = io.sel_base + so;
  }
  if (!sel) {  // every row selected: rank == row
    for (uint32_t p = threadIdx.x; p < pc; p += 256u) out[pidx[p]] = pval[p];
    return;
  }
  const uint32_t n = h->n, n_words = (n + 31u) >> 5, tail = n & 31u;
  uint32_t carry = 0;
  for (uint32_t w0 = 0; w0 < n_words; w0 += 256u) {
    const uint32_t wi = w0 + threadIdx.x;
    uint32_t sw = 0;
    if (wi < n_words) {
      sw = sel[wi];
      if (wi == n_words - 1u && tail) sw &= (1u << tail) - 1u;
    }
    uint32_t tot;
    const uint32_t excl = block_excl_scan_256(__popc(sw), s_tot, &tot);
    s_word[threadIdx.x] = sw;
    s_off[threadIdx.x] = carry + excl;
    __syncthreads();
    for (uint32_t p = threadIdx.x; p < pc; p += 256u) {
      const uint32_t row = pidx[p];
      const uint32_t lw = (row >> 5) - w0;  // wraps for rows before this tile
      if (lw < 256u) {
        const uint32_t word = s_word[lw], bit = row & 31u;
        if ((word >> bit) & 1u) out[s_off[lw] + __popc(word & ((1u << bit) - 1u))] = pval[p];
      }
    }
    carry += tot;
    __syncthreads();
  }
}

cudaError_t launch_alp_finish(uint32_t n_entries, const ScanIo& io, uint32_t tbits, cudaStream_t s) {
  if (n_entries == 0) return cudaSuccess;
  if (tbits == 64) k_alp_finish<double><<<n_entries, 256, 0, s>>>(io);
  else k_alp_finish<float><<<n_entries, 256, 0, s>>>(io);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// `col <op> literal` on decoded floats. arrow-ord orders floats by IEEE totalOrder (NaN == NaN, -0.0 < +0.0), which
// on the two's complement key of alp_math.cuh is a plain signed integer compare. Nulls come out false.
//   PRED:   values = the selected rows, compacted; mask word i covers values 32i..32i+31; AND the compact validity
//   REFINE: values = all rows; selection := selection & valid & cmp in place
// ------------------------------------------------------------------------------------------------
template <typename F>
__global__ void __launch_bounds__(256) k_float_cmp(FloatCmpIo io) {
  using A = Alp<F>;
  using I = typename A::I;
  __shared__ uint32_t s_cnt;
  const uint32_t ent = blockIdx.x;
  const EntryRef ref = io.refs[ent];
  const IntHeader* __restrict__ h = reinterpret_cast<const IntHeader*>(ref.blob);
  const uint32_t m = io.refine ? ref.rows : io.vals_counts[static_cast<size_t>(ent) * io.vals_stride];
  const I* __restrict__ vals = reinterpret_cast<const I*>(io.vals_base) + io.vals_off[ent];
  const uint32_t* and1 = nullptr;  // validity
  const uint32_t* and2 = nullptr;  // running selection
  if (io.refine) {
    if (h->has_nulls) and1 = reinterpret_cast<const uint32_t*>(ref.blob + h->validity_off);
    if (io.sel_base) {
      const uint64_t so = io.sel_off[ent];
      if (so != kNoSel) and2 = io.sel_base + so;
    }
  } else if (h->has_nulls && io.and_base) {
    and1 = io.and_base + io.and_off[ent];
  }
  uint32_t* __restrict__ out = io.out_base + io.out_off[ent];
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  const I lit = static_cast<I>(io.lit_key);
  const int op = io.op;
  const uint32_t n_words = (m + 31u) >> 5, tail = m & 31u;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t cnt = 0;
  for (uint32_t w = warp; w < n_words; w += 8u) {
    const uint32_t i = w * 32u + lane;
    bool hit = false;
    if (i < m) {
      const I key = A::order_key(vals[i]);
      hit = op == 0 ? key == lit : op == 1 ? key != lit : op == 2 ? key < lit : op == 3 ? key <= lit : op == 4 ? key > lit : key >= lit;
    }
    uint32_t cw = __ballot_sync(kFullMask, hit);
    if (lane == 0) {
      if (w == n_words - 1u && tail) cw &= (1u << tail) - 1u;
      if (and1) cw &= and1[w];
      if (and2) cw &= and2[w];
      out[w] = cw;
      cnt += __popc(cw);
    }
  }
  if (lane == 0 && cnt) atomicAdd(&s_cnt, cnt);
  __syncthreads();
  if (threadIdx.x == 0 && io.counts) {
    uint32_t* c = io.counts + static_cast<size_t>(ent) * io.counts_stride;
    if (io.refine) {
      c[0] = s_cnt;
      c[1] = 0;
    } else {
      c[2] = s_cnt;
    }
  }
}

cudaError_t launch_float_cmp(uint32_t n_entries, const FloatCmpIo& io, uint32_t tbits, cudaStream_t s) {
  if (n_entries == 0) return cudaSuccess;
  if (tbits == 64) k_float_cmp<double><<<n_entries, 256, 0, s>>>(io);
  else k_float_cmp<float><<<n_entries, 256, 0, s>>>(io);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// decimals: Decimal128 / Decimal256 little-endian two's complement <-> u64
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_dec_narrow(const unsigned long long* __restrict__ in, const uint32_t* __restrict__ validity,
                                                    uint32_t n, uint32_t words, unsigned long long* __restrict__ out,
                                                    uint32_t* __restrict__ flag) {
  for (uint32_t i = blockIdx.x * 256u + threadIdx.x; i < n; i += gridDim.x * 256u) {
    const bool ok = validity ? ((validity[i >> 5] >> (i & 31u)) & 1u) : true;
    unsigned long long lo = 0;
    if (ok) {  // fits_u64 looks at valid slots only (decimal_array.rs:127-132); null slots are stored as 0
      lo = in[static_cast<size_t>(i) * words];
      unsigned long long hi = 0;
      for (uint32_t k = 1; k < words; ++k) hi |= in[static_cast<size_t>(i) * words + k];
      if (hi) atomicOr(flag, 1u);  // negative or beyond u64::MAX
    }
    out[i] = lo;
  }
}

__global__ void __launch_bounds__(256) k_dec_widen(const unsigned long long* __restrict__ in, uint64_t n, uint32_t words,
                                                   unsigned long long* __restrict__ out) {
  // one thread per OUTPUT word: coalesced stores; `*v as i128` / i256::from_i128 of a u64 is a zero extension
  const uint64_t total = n * words;
  for (uint64_t g = static_cast<uint64_t>(blockIdx.x) * 256u + threadIdx.x; g < total; g += static_cast<uint64_t>(gridDim.x) * 256u) {
    const uint64_t i = g / words;
    out[g] = (g - i * words) == 0 ? in[i] : 0ull;
  }
}

// LQDA keeps patch indices as u64 (float_array.rs:483-496); the entry keeps them as u32. narrow also checks that every
// index is a row of the entry (an index past the end would make k_alp_finish write out of bounds).
__global__ void __launch_bounds__(256) k_widen_u32(const uint32_t* __restrict__ in, uint32_t n, unsigned long long* __restrict__ out) {
  for (uint32_t i = blockIdx.x * 256u + threadIdx.x; i < n; i += gridDim.x * 256u) out[i] = in[i];
}
__global__ void __launch_bounds__(256) k_narrow_u64(const unsigned long long* __restrict__ in, uint32_t n, unsigned long long limit,
                                                    uint32_t* __restrict__ out, uint32_t* __restrict__ flag) {
  for (uint32_t i = blockIdx.x * 256u + threadIdx.x; i < n; i += gridDim.x * 256u) {
    const unsigned long long v = in[i];
    if (v >= limit) atomicOr(flag, 1u);
    out[i] = static_cast<uint32_t>(v);
  }
}

// Squeeze (LiquidPrimitiveArray::squeeze, liquid_array/primitive_array.rs:419-496): the decoded values of a full entry
// become `reference + code`, code = the offset clamped at the sentinel (Clamp, :427-438) or its bucket index
// (Quantize, :472-481), ready for k_int_pack at the halved width. In place, one value per thread, wrapping arithmetic on
// the unsigned twin like the reference's add_wrapping / sub_wrapping.
template <typename U>
__global__ void __launch_bounds__(256) k_squeeze_map(U* __restrict__ vals, uint32_t n, U ref, uint32_t quantize, unsigned long long limit,
                                                     unsigned long long bucket_width) {
  for (uint32_t i = blockIdx.x * 256u + threadIdx.x; i < n; i += gridDim.x * 256u) {
    const unsigned long long off = static_cast<unsigned long long>(static_cast<U>(vals[i] - ref));
    vals[i] = static_cast<U>(ref + static_cast<U>(squeeze_code(off, quantize, limit, bucket_width)));
  }
}

cudaError_t launch_squeeze_map(void* d_vals, uint32_t n, uint32_t tbits, unsigned long long ref, uint32_t quantize,
                               unsigned long long limit, unsigned long long bucket_width, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  uint32_t grid = (n + 255u) / 256u;
  if (grid > kGridStrideCap) grid = kGridStrideCap;
  switch (tbits) {
    case 8: k_squeeze_map<uint8_t><<<grid, 256, 0, s>>>(static_cast<uint8_t*>(d_vals), n, static_cast<uint8_t>(ref), quantize, limit, bucket_width); break;
    case 16: k_squeeze_map<uint16_t><<<grid, 256, 0, s>>>(static_cast<uint16_t*>(d_vals), n, static_cast<uint16_t>(ref), quantize, limit, bucket_width); break;
    case 32: k_squeeze_map<uint32_t><<<grid, 256, 0, s>>>(static_cast<uint32_t*>(d_vals), n, static_cast<uint32_t>(ref), quantize, limit, bucket_width); break;
    default: k_squeeze_map<unsigned long long><<<grid, 256, 0, s>>>(static_cast<unsigned long long*>(d_vals), n, ref, quantize, limit, bucket_width); break;
  }
  return cudaGetLastError();
}

// ---- Date32 / Timestamp columns squeezed to one date component (liquid_array/squeezed_date32_array.rs); the per-value
// arithmetic lives in squeeze_math.cuh ----
// from_liquid_date32 (:63-141) / from_liquid_timestamp (:144-223): decoded days (T = int32, ticks_per_day = 0) or
// timestamp ticks (T = int64; div_euclid by the unit's ticks per day, `as i32`) -> the component of every row
template <typename T>
__global__ void __launch_bounds__(256) k_date_component(const T* __restrict__ in, uint32_t n, uint32_t field, long long ticks_per_day,
                                                        int32_t* __restrict__ out) {
  for (uint32_t i = blockIdx.x * 256u + threadIdx.x; i < n; i += gridDim.x * 256u) {
    const int32_t days = ticks_per_day ? days_of_ticks(static_cast<long long>(in[i]), ticks_per_day) : static_cast<int32_t>(in[i]);
    out[i] = date_component(field, days);
  }
}

// to_arrow_date32_lossy (:326-356) / to_arrow_timestamp_lossy (:299-321): a date whose component is the stored one —
// Year -> (y,1,1), Month -> (1970,m,1), Day -> (1970,1,d), DayOfWeek -> 1970-01-04 + dow (saturating); null rows hold 0.
// ticks_per_day = 0 writes int32 days, otherwise int64 ticks at midnight of that date.
__global__ void __launch_bounds__(256) k_date_lossy(const int32_t* __restrict__ comp, const uint32_t* __restrict__ valid, uint32_t n,
                                                    uint32_t field, long long ticks_per_day, void* __restrict__ out) {
  for (uint32_t i = blockIdx.x * 256u + threadIdx.x; i < n; i += gridDim.x * 256u) {
    const bool ok = valid ? ((valid[i >> 5] >> (i & 31u)) & 1u) : true;
    const int32_t days = ok ? lossy_days(field, comp[i]) : 0;
    if (ticks_per_day) static_cast<long long*>(out)[i] = static_cast<long long>(days) * ticks_per_day;
    else static_cast<int32_t*>(out)[i] = days;
  }
}

cudaError_t launch_date_component(const void* d_in, uint32_t n, uint32_t in_bits, uint32_t field, long long ticks_per_day,
                                  int32_t* d_out, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  uint32_t grid = (n + 255u) / 256u;
  if (grid > kGridStrideCap) grid = kGridStrideCap;
  if (in_bits == 64) k_date_component<long long><<<grid, 256, 0, s>>>(static_cast<const long long*>(d_in), n, field, ticks_per_day, d_out);
  else k_date_component<int32_t><<<grid, 256, 0, s>>>(static_cast<const int32_t*>(d_in), n, field, 0, d_out);
  return cudaGetLastError();
}

cudaError_t launch_date_lossy(const int32_t* d_comp, const uint32_t* d_valid, uint32_t n, uint32_t field, long long ticks_per_day,
                              void* d_out, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  uint32_t grid = (n + 255u) / 256u;
  if (grid > kGridStrideCap) grid = kGridStrideCap;
  k_date_lossy<<<grid, 256, 0, s>>>(d_comp, d_valid, n, field, ticks_per_day, d_out);
  return cudaGetLastError();
}

cudaError_t launch_widen_u32(const uint32_t* d_in, uint32_t n, unsigned long long* d_out, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  uint32_t grid = (n + 255u) / 256u;
  if (grid > kGridStrideCap) grid = kGridStrideCap;
  k_widen_u32<<<grid, 256, 0, s>>>(d_in, n, d_out);
  return cudaGetLastError();
}

cudaError_t launch_narrow_u64(const unsigned long long* d_in, uint32_t n, unsigned long long limit, uint32_t* d_out, uint32_t* d_flag,
                              cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  uint32_t grid = (n + 255u) / 256u;
  if (grid > kGridStrideCap) grid = kGridStrideCap;
  k_narrow_u64<<<grid, 256, 0, s>>>(d_in, n, limit, d_out, d_flag);
  return cudaGetLastError();
}

cudaError_t launch_dec_narrow(const void* d_in, const uint32_t* d_validity, uint32_t n, uint32_t width_bytes,
                              unsigned long long* d_out, uint32_t* d_flag, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  uint32_t grid = (n + 255u) / 256u;
  if (grid > kGridStrideCap) grid = kGridStrideCap;
  k_dec_narrow<<<grid, 256, 0, s>>>(static_cast<const unsigned long long*>(d_in), d_validity, n, width_bytes / 8u, d_out, d_flag);
  return cudaGetLastError();
}

cudaError_t launch_dec_widen(const unsigned long long* d_in, uint64_t n, uint32_t width_bytes, void* d_out, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  const uint64_t total = n * (width_bytes / 8u);
  uint64_t grid = (total + 255u) / 256u;
  if (grid > 4u * kGridStrideCap) grid = 4u * kGridStrideCap;  // 4 waves
  k_dec_widen<<<static_cast<uint32_t>(grid), 256, 0, s>>>(d_in, n, width_bytes / 8u, static_cast<unsigned long long*>(d_out));
  return cudaGetLastError();
}

}  // namespace lc

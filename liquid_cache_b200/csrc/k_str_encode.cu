// k_str_encode.cu — byte-view insert on the device: Arrow strings -> liquid byte-view sections.
//
// Reference semantics restated (all under /root/reference/src/core/src/):
//   u16 dictionary, uniques in first-occurrence order, null rows -> null key     utils/mod.rs:52-154
//   shared prefix = LCP of all unique values                                     byte_view_array/conversions.rs:269-307
//   per unique: FSST compress, PrefixKey {7 suffix bytes, len (255 = >=255)},    conversions.rs:309-373,
//               fingerprint = OR of 1 << (byte & 31) over the whole value        raw/fsst_buffer.rs:173-187, fingerprint.rs:19-26
//   CompactOffsets: f64 least-squares line through (i, offsets[i]) rounded to    raw/fsst_buffer.rs:267-359
//               i32, residuals stored as i8 / i16 / i32 by range
//
// Pipeline (one stream, no host round trip in between):
//   k_dict_insert   thread per row: hash, open-addressed table keyed by value (length + bytes), the slot keeps the SMALLEST row
//                   index holding that value (atomicCAS to claim, atomicMin to lower) -> first-occurrence leaders
//   k_dict_finish   one CTA: leader flags -> block scans -> unique ids in first-occurrence order, u16 keys
//   k_uniq_pass1    thread per unique: LCP with unique 0 (atomicMin), greedy FSST length, fingerprint, length stats
//   k_offsets       one CTA: exclusive scan of compressed lengths, line fit in the reference's summation order
//                   (one thread, round-to-nearest f64 ops without contraction), residual range -> width
//   k_uniq_pass2    thread per unique: FSST bytes at their final offsets, PrefixKeys against the final shared prefix
// The FSST matcher is the one fsst_host.cc trains with (lossy 3-byte hash for 3..8 byte symbols, 2-byte table,
// 1-byte fallback, escape), so the compressed form only depends on the column chunk's table.
#include "device_utils.cuh"
#include "entry_layout.h"
#include "kernels.h"

namespace lc {

namespace {

constexpr uint32_t kEmpty = 0xFFFFFFFFu;

__device__ __forceinline__ bool row_valid(const StrEncIo& io, uint32_t r) {
  return io.valid == nullptr || ((io.valid[r >> 5] >> (r & 31u)) & 1u);
}

__device__ __forceinline__ unsigned long long hash_value(const uint8_t* p, uint32_t len) {
  unsigned long long h = 0xcbf29ce484222325ull ^ (static_cast<unsigned long long>(len) * 0x9E3779B97F4A7C15ull);
  for (uint32_t i = 0; i < len; ++i) {
    h ^= p[i];
    h *= 0x100000001b3ull;
  }
  h ^= h >> 32;
  h *= 0xd6e8feb86659fd93ull;
  return h ^ (h >> 29);
}

__device__ __forceinline__ bool bytes_equal(const uint8_t* a, const uint8_t* b, uint32_t len) {
  for (uint32_t i = 0; i < len; ++i)
    if (a[i] != b[i]) return false;
  return true;
}

__device__ __forceinline__ void k_dict_insert_body(const StrEncIo& io, uint32_t bx, uint32_t gx) {
  for (uint32_t r = bx * blockDim.x + threadIdx.x; r < io.n; r += gx * blockDim.x) {
    if (!row_valid(io, r)) {
      io.row_slot[r] = kEmpty;
      continue;
    }
    const uint8_t* p = io.pool + io.row_off[r];
    const uint32_t len = io.row_len[r];
    const unsigned long long h = hash_value(p, len);
    uint32_t s = static_cast<uint32_t>(h) & io.table_mask;
    // Slots only ever go empty -> row, and a slot's row is only replaced by a smaller row of the SAME value, so a
    // (possibly stale) read of a slot still names a row whose value is the slot's value. Values are immutable inputs.
    const volatile uint32_t* vt = io.table;
    for (;;) {
      uint32_t cur = vt[s];
      if (cur == kEmpty) {
        cur = atomicCAS(&io.table[s], kEmpty, r);
        if (cur == kEmpty) break;  // claimed
      }
      if (io.row_len[cur] == len && bytes_equal(io.pool + io.row_off[cur], p, len)) {
        atomicMin(&io.table[s], r);
        break;
      }
      s = (s + 1u) & io.table_mask;
    }
    io.row_slot[r] = s;
  }
}

// One CTA of 1024 threads.
__device__ __forceinline__ void k_dict_finish_body(const StrEncIo& io, uint32_t bx, uint32_t gx) {
  __shared__ uint32_t warp_tot[32];
  __shared__ uint32_t carry, nulls;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    carry = 0;
    nulls = 0;
  }
  __syncthreads();
  for (uint32_t base = 0; base < io.n; base += 1024u) {
    const uint32_t r = base + threadIdx.x;
    uint32_t first = 0, lead = kEmpty;
    bool is_null = false;
    if (r < io.n) {
      const uint32_t s = io.row_slot[r];
      if (s == kEmpty) {
        is_null = true;
      } else {
        lead = io.table[s];
        first = lead == r;
      }
      io.leader[r] = lead;
    }
    const uint32_t incl = warp_incl_scan(first, lane);
    const uint32_t nb = __popc(__ballot_sync(kFullMask, is_null));
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    uint32_t before = 0, tile = 0;
    for (uint32_t w = 0; w < 32; ++w) {
      const uint32_t t = warp_tot[w];
      if (w < warp) before += t;
      tile += t;
    }
    const uint32_t uid = carry + before + incl - first;
    if (first) {
      if (uid < 65536u) {  // beyond that the batch is rejected; do not scribble past the arrays' intent
        io.uniq_row[uid] = r;
        io.row_slot[r] = uid;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) carry += tile;
    if (lane == 0 && nb) atomicAdd(&nulls, nb);
    __syncthreads();
  }
  const uint32_t U = carry;
  if (threadIdx.x == 0) {
    StrEncResult* res = io.res;
    res->n_unique = U;
    res->null_count = nulls;
    res->error = U > 65536u ? 1u : 0u;
    res->shared_prefix_len = U ? io.row_len[io.uniq_row[0]] : 0u;  // lowered by k_uniq_pass1
    res->max_value_len = 0;
    res->uncompressed_bytes = 0;
    res->comp_bytes = 0;
  }
  if (U > 65536u) return;
  __threadfence_block();
  __syncthreads();
  for (uint32_t r = threadIdx.x; r < io.n; r += 1024u) {
    const uint32_t lead = io.leader[r];
    io.keys[r] = lead == kEmpty ? static_cast<uint16_t>(0) : static_cast<uint16_t>(io.row_slot[lead]);
  }
}

// ---- FSST greedy matcher (same decisions as fsst_compress_host) -----------------------------------
__device__ __forceinline__ uint32_t fsst_hash3(unsigned long long w) {
  const unsigned long long h = (w & 0xFFFFFFull) * 2971215073ull;
  return static_cast<uint32_t>((h ^ (h >> 15)) & 2047u);
}

__device__ __forceinline__ unsigned long long load_le(const uint8_t* p, uint32_t avail) {
  unsigned long long w = 0;
  const uint32_t m = avail < 8u ? avail : 8u;
  for (uint32_t i = 0; i < m; ++i) w |= static_cast<unsigned long long>(p[i]) << (8u * i);
  return w;
}

// Walks one value; EMIT(code) / EMIT_ESC(byte) see the output in order. Returns the compressed length.
template <bool WRITE>
__device__ __forceinline__ uint32_t fsst_compress_value(const FsstEncTable* __restrict__ e, const uint8_t* p, uint32_t len,
                                                        uint8_t* out) {
  uint32_t o = 0, rem = len;
  while (rem) {
    const unsigned long long w = load_le(p, rem);
    uint32_t l = 0;
    int code = -1;
    if (rem >= 3u) {
      const uint32_t h = fsst_hash3(w);
      const uint32_t m = e->hash_meta[h];
      const uint32_t ml = m >> 8;
      if (ml && ml <= rem) {
        const unsigned long long lm = ml >= 8u ? ~0ull : ((1ull << (8u * ml)) - 1ull);
        if ((w & lm) == e->hash_sym[h]) {
          code = static_cast<int>(m & 0xFFu);
          l = ml;
        }
      }
    }
    if (code < 0) {
      uint32_t m = e->short_code[w & 0xFFFFu];
      if ((m >> 8) == 2u && rem < 2u) m = e->one_byte[w & 0xFFu];
      const uint32_t ml = m >> 8;
      if (ml) {
        code = static_cast<int>(m & 0xFFu);
        l = ml;
      }
    }
    if (code >= 0) {
      if (WRITE) out[o] = static_cast<uint8_t>(code);
      o += 1u;
      p += l;
      rem -= l;
    } else {
      if (WRITE) {
        out[o] = 255;
        out[o + 1] = p[0];
      }
      o += 2u;
      p += 1;
      rem -= 1u;
    }
  }
  return o;
}

__device__ __forceinline__ void k_uniq_pass1_body(const StrEncIo& io, uint32_t bx, uint32_t gx) {
  StrEncResult* res = io.res;
  const uint32_t U = res->n_unique;
  if (res->error) return;
  const uint32_t u = bx * blockDim.x + threadIdx.x;
  uint32_t len = 0;
  if (u < U) {
    const uint32_t r = io.uniq_row[u];
    const uint8_t* p = io.pool + io.row_off[r];
    len = io.row_len[r];
    // shared prefix: LCP(all) = min over uniques of LCP(unique, unique 0)
    const uint32_t r0 = io.uniq_row[0];
    const uint8_t* p0 = io.pool + io.row_off[r0];
    const uint32_t l0 = io.row_len[r0];
    const uint32_t m = len < l0 ? len : l0;
    uint32_t c = 0;
    while (c < m && p[c] == p0[c]) ++c;
    if (c < l0) atomicMin(&res->shared_prefix_len, c);
    io.clen[u] = fsst_compress_value<false>(io.enc, p, len, nullptr);
    if (io.fps) {
      uint32_t bits = 0;
      unsigned long long bl[kBloomWords] = {0ull, 0ull, 0ull, 0ull};
      for (uint32_t b = 0; b < len; ++b) {
        bits |= 1u << (p[b] & 31u);
        if (b + 2u < len) {
          const uint32_t t = trigram_bit(p[b], p[b + 1u], p[b + 2u]);
          bl[t >> 6] |= 1ull << (t & 63u);
        }
      }
      io.fps[u] = bits;
      ulonglong2* dst = reinterpret_cast<ulonglong2*>(io.blooms + static_cast<size_t>(u) * kBloomWords);
      dst[0] = make_ulonglong2(bl[0], bl[1]);
      dst[1] = make_ulonglong2(bl[2], bl[3]);
    }
  }
  // length statistics: warp-reduce, one atomic per warp
  uint32_t mx = len;
  unsigned long long sum = len;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const uint32_t omx = __shfl_xor_sync(kFullMask, mx, d);
    mx = omx > mx ? omx : mx;
    sum += __shfl_xor_sync(kFullMask, sum, d);
  }
  if ((threadIdx.x & 31u) == 0 && sum) {
    atomicMax(&res->max_value_len, mx);
    atomicAdd(&res->uncompressed_bytes, sum);
  }
}

// One CTA of 1024 threads: offsets, line fit, residuals.
__device__ __forceinline__ void k_offsets_body(const StrEncIo& io, uint32_t bx, uint32_t gx) {
  __shared__ uint32_t warp_tot[32];
  __shared__ unsigned long long carry64;
  __shared__ int32_t s_slope, s_intercept, s_min, s_max;
  __shared__ uint32_t s_ob;
  StrEncResult* res = io.res;
  if (res->error) return;
  const uint32_t U = res->n_unique;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    carry64 = 0;
    s_min = 2147483647;
    s_max = -2147483647 - 1;
  }
  __syncthreads();
  // exclusive scan of clen -> offsets[0..U]
  for (uint32_t base = 0; base < U; base += 1024u) {
    const uint32_t u = base + threadIdx.x;
    const uint32_t v = u < U ? io.clen[u] : 0u;
    const uint32_t incl = warp_incl_scan(v, lane);
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    uint32_t before = 0, tile = 0;
    for (uint32_t w = 0; w < 32; ++w) {
      const uint32_t t = warp_tot[w];
      if (w < warp) before += t;
      tile += t;
    }
    const unsigned long long off = carry64 + before + incl - v;
    if (u < U) io.offsets[u] = static_cast<uint32_t>(off);
    __syncthreads();
    if (threadIdx.x == 0) carry64 += tile;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    if (carry64 > 0xFFFFFFF0ull) res->error = 2u;
    io.offsets[U] = static_cast<uint32_t>(carry64);
    res->comp_bytes = static_cast<uint32_t>(carry64);
    // fit_line (fsst_buffer.rs:267-296) in the reference's order: sum_y, then sum_xy, each left to right
    const unsigned long long n = static_cast<unsigned long long>(U) + 1ull;
    int32_t slope = 0, intercept = 0;
    if (n <= 1ull) {
      intercept = static_cast<int32_t>(io.offsets[0]);
    } else {
      const double nf = static_cast<double>(n);
      const double sum_x = static_cast<double>(n * (n - 1ull) / 2ull);
      double sum_y = 0.0, sum_xy = 0.0;
      for (unsigned long long i = 0; i < n; ++i) sum_y = __dadd_rn(sum_y, static_cast<double>(io.offsets[i]));
      for (unsigned long long i = 0; i < n; ++i)
        sum_xy = __dadd_rn(sum_xy, __dmul_rn(static_cast<double>(i), static_cast<double>(io.offsets[i])));
      const double sum_x_sq = static_cast<double>(n * (n - 1ull) * (2ull * n - 1ull) / 6ull);
      const double num = __dsub_rn(__dmul_rn(nf, sum_xy), __dmul_rn(sum_x, sum_y));
      const double den = __dsub_rn(__dmul_rn(nf, sum_x_sq), __dmul_rn(sum_x, sum_x));
      const double sl = __ddiv_rn(num, den);
      const double ic = __ddiv_rn(__dsub_rn(sum_y, __dmul_rn(sl, sum_x)), nf);
      auto sat = [](double v) -> int32_t {
        const double r = round(v);
        if (!(r == r)) return 0;
        if (r >= 2147483647.0) return 2147483647;
        if (r <= -2147483648.0) return -2147483647 - 1;
        return static_cast<int32_t>(r);
      };
      slope = sat(sl);
      intercept = sat(ic);
    }
    s_slope = slope;
    s_intercept = intercept;
    res->slope = slope;
    res->intercept = intercept;
  }
  __syncthreads();
  if (res->error) return;
  // residual range (fsst_buffer.rs:298-359): offsets[i] - (slope * i + intercept), wrapping i32 arithmetic
  int32_t mn = 2147483647, mx = -2147483647 - 1;
  for (uint32_t i = threadIdx.x; i <= U; i += 1024u) {
    const uint32_t predicted = static_cast<uint32_t>(s_slope) * i + static_cast<uint32_t>(s_intercept);
    const int32_t r = static_cast<int32_t>(io.offsets[i] - predicted);
    mn = r < mn ? r : mn;
    mx = r > mx ? r : mx;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const int32_t omn = __shfl_xor_sync(kFullMask, mn, d), omx = __shfl_xor_sync(kFullMask, mx, d);
    mn = omn < mn ? omn : mn;
    mx = omx > mx ? omx : mx;
  }
  if (lane == 0) {
    atomicMin(&s_min, mn);
    atomicMax(&s_max, mx);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    s_ob = (s_min >= -128 && s_max <= 127) ? 1u : (s_min >= -32768 && s_max <= 32767) ? 2u : 4u;
    res->offset_bytes = s_ob;
  }
  __syncthreads();
  const uint32_t ob = s_ob;
  for (uint32_t i = threadIdx.x; i <= U; i += 1024u) {
    const uint32_t predicted = static_cast<uint32_t>(s_slope) * i + static_cast<uint32_t>(s_intercept);
    const int32_t r = static_cast<int32_t>(io.offsets[i] - predicted);
    if (ob == 1u) reinterpret_cast<int8_t*>(io.resid)[i] = static_cast<int8_t>(r);
    else if (ob == 2u) reinterpret_cast<int16_t*>(io.resid)[i] = static_cast<int16_t>(r);
    else reinterpret_cast<int32_t*>(io.resid)[i] = r;
  }
}

__device__ __forceinline__ void k_uniq_pass2_body(const StrEncIo& io, uint32_t bx, uint32_t gx) {
  const StrEncResult* res = io.res;
  if (res->error) return;
  const uint32_t U = res->n_unique;
  const uint32_t u = bx * blockDim.x + threadIdx.x;
  if (u >= U) return;
  const uint32_t r = io.uniq_row[u];
  const uint8_t* p = io.pool + io.row_off[r];
  const uint32_t len = io.row_len[r];
  fsst_compress_value<true>(io.enc, p, len, io.comp + io.offsets[u]);
  // PrefixKey::new(suffix) (fsst_buffer.rs:173-187)
  const uint32_t spl = res->shared_prefix_len;
  const uint32_t sl = len > spl ? len - spl : 0u;
  const uint32_t cp = sl < 7u ? sl : 7u;
  unsigned long long k = 0;
  for (uint32_t b = 0; b < cp; ++b) k |= static_cast<unsigned long long>(p[spl + b]) << (8u * b);
  k |= static_cast<unsigned long long>(sl >= 255u ? 255u : sl) << 56;
  io.pkeys[u] = k;
}

// Every stage exists twice: for ONE batch (work item passed by value) and for a LIST of batches (blockIdx.y, or blockIdx.x
// for the one-CTA stages, picks the work item), so a whole row group runs through the same five launches.
__global__ void k_dict_insert(StrEncIo io) { k_dict_insert_body(io, blockIdx.x, gridDim.x); }
__global__ void k_dict_insert_many(const StrEncIo* __restrict__ ios) { k_dict_insert_body(ios[blockIdx.y], blockIdx.x, gridDim.x); }
__global__ void __launch_bounds__(1024) k_dict_finish(StrEncIo io) { k_dict_finish_body(io, 0, 1); }
__global__ void __launch_bounds__(1024) k_dict_finish_many(const StrEncIo* __restrict__ ios) { k_dict_finish_body(ios[blockIdx.x], 0, 1); }
__global__ void k_uniq_pass1(StrEncIo io) { k_uniq_pass1_body(io, blockIdx.x, gridDim.x); }
__global__ void k_uniq_pass1_many(const StrEncIo* __restrict__ ios) { k_uniq_pass1_body(ios[blockIdx.y], blockIdx.x, gridDim.x); }
__global__ void __launch_bounds__(1024) k_offsets(StrEncIo io) { k_offsets_body(io, 0, 1); }
__global__ void __launch_bounds__(1024) k_offsets_many(const StrEncIo* __restrict__ ios) { k_offsets_body(ios[blockIdx.x], 0, 1); }
__global__ void k_uniq_pass2(StrEncIo io) { k_uniq_pass2_body(io, blockIdx.x, gridDim.x); }
__global__ void k_uniq_pass2_many(const StrEncIo* __restrict__ ios) { k_uniq_pass2_body(ios[blockIdx.y], blockIdx.x, gridDim.x); }

}  // namespace

cudaError_t launch_str_encode(const StrEncIo& io, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(io.table, 0xFF, (static_cast<size_t>(io.table_mask) + 1u) * sizeof(uint32_t), s);
  if (e != cudaSuccess) return e;
  const uint32_t n = io.n;
  if (n) {
    const uint32_t grid = (n + 255u) / 256u;
    k_dict_insert<<<grid < kGridStrideCap ? grid : kGridStrideCap, 256, 0, s>>>(io);
  }
  k_dict_finish<<<1, 1024, 0, s>>>(io);
  const uint32_t ugrid = n ? (n + 127u) / 128u : 1u;  // U <= n is only known on the device
  k_uniq_pass1<<<ugrid, 128, 0, s>>>(io);
  k_offsets<<<1, 1024, 0, s>>>(io);
  k_uniq_pass2<<<ugrid, 128, 0, s>>>(io);
  return cudaGetLastError();
}

// The same pipeline over a list of batches: `d_ios` holds one work item per batch (device memory), `d_tables` is the
// contiguous range of all their hash tables (filled with the empty marker here), `max_n` the largest row count.
cudaError_t launch_str_encode_many(const StrEncIo* d_ios, uint32_t n_batches, uint32_t max_n, uint32_t* d_tables,
                                   size_t table_words, cudaStream_t s) {
  if (n_batches == 0) return cudaSuccess;
  cudaError_t e = cudaMemsetAsync(d_tables, 0xFF, table_words * sizeof(uint32_t), s);
  if (e != cudaSuccess) return e;
  if (max_n) {
    uint32_t gx = (max_n + 255u) / 256u;
    if (gx > 64u) gx = 64u;  // rows beyond are covered by the grid-stride loop
    k_dict_insert_many<<<dim3(gx, n_batches), 256, 0, s>>>(d_ios);
  }
  k_dict_finish_many<<<n_batches, 1024, 0, s>>>(d_ios);
  const uint32_t ugrid = max_n ? (max_n + 127u) / 128u : 1u;
  k_uniq_pass1_many<<<dim3(ugrid, n_batches), 128, 0, s>>>(d_ios);
  k_offsets_many<<<n_batches, 1024, 0, s>>>(d_ios);
  k_uniq_pass2_many<<<dim3(ugrid, n_batches), 128, 0, s>>>(d_ios);
  return cudaGetLastError();
}

// The trigram sets are built one 256-bit row per dictionary value (k_uniq_pass1) and stored as 256 planes over the dictionary
// (entry_layout.h): a 32 x 256 bit transposition per stripe of 32 values, done with ballots — lane j holds value j's row, the
// ballot over bit t of the rows IS plane t's word for the stripe. One CTA per entry, a warp per stripe.
__device__ __forceinline__ void bloom_rows_to_planes(const unsigned long long* __restrict__ rows, uint32_t U, uint32_t* __restrict__ planes) {
  const uint32_t pw = bloom_plane_words(U);
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u, n_warps = blockDim.x >> 5;
  for (uint32_t s = warp; s < pw; s += n_warps) {
    const uint32_t i = s * 32u + lane;
    ulonglong2 lo = make_ulonglong2(0ull, 0ull), hi = lo;
    if (i < U) {
      const ulonglong2* src = reinterpret_cast<const ulonglong2*>(rows + static_cast<size_t>(i) * kBloomWords);
      lo = src[0];
      hi = src[1];
    }
    const unsigned long long r[4] = {lo.x, lo.y, hi.x, hi.y};
#pragma unroll
    for (uint32_t q = 0; q < 8; ++q) {
      const uint32_t w = static_cast<uint32_t>(r[q >> 1] >> ((q & 1u) * 32u));
      uint32_t mine = 0;
#pragma unroll
      for (uint32_t b = 0; b < 32; ++b) {
        const uint32_t bw = __ballot_sync(kFullMask, (w >> b) & 1u);
        if (lane == b) mine = bw;
      }
      planes[static_cast<size_t>(q * 32u + lane) * pw + s] = mine;
    }
  }
}

__global__ void __launch_bounds__(256) k_bloom_planes(const unsigned long long* __restrict__ rows, const StrEncResult* __restrict__ res,
                                                      uint32_t* __restrict__ planes) {
  bloom_rows_to_planes(rows, res->n_unique, planes);
}

cudaError_t launch_bloom_planes(const unsigned long long* d_rows, const StrEncResult* d_res, uint32_t* d_planes, cudaStream_t s) {
  k_bloom_planes<<<1, 256, 0, s>>>(d_rows, d_res, d_planes);
  return cudaGetLastError();
}

// Entry blob of one batch from the pipeline's work areas (see StrAsmWork). 16-byte copies where source and length allow.
__global__ void __launch_bounds__(256) k_str_assemble(const StrAsmWork* __restrict__ works) {
  const StrAsmWork& w = works[blockIdx.x];
  uint8_t* blob = w.blob;
  if (threadIdx.x < sizeof(StrHeader) / 4) reinterpret_cast<uint32_t*>(blob)[threadIdx.x] = reinterpret_cast<const uint32_t*>(&w.hdr)[threadIdx.x];
  uint32_t prev_end = sizeof(StrHeader);
  for (uint32_t q = 0; q <= w.n_segs; ++q) {
    const bool last = q == w.n_segs;
    const uint32_t dst = last ? w.blob_bytes : w.segs[q].dst_off;
    // zero the gap [prev_end, dst): section padding reads as zero
    for (uint32_t o = prev_end + threadIdx.x; o < dst; o += 256u) blob[o] = 0;
    if (last) break;
    const uint8_t* src = w.segs[q].src;
    const uint32_t bytes = w.segs[q].bytes;
    if (w.hdr.bloom_off != 0u && dst == w.hdr.bloom_off) {  // the trigram sets: rows in the work area, planes in the blob
      bloom_rows_to_planes(reinterpret_cast<const unsigned long long*>(src), w.hdr.n_unique, reinterpret_cast<uint32_t*>(blob + dst));
    } else if ((reinterpret_cast<uintptr_t>(src) & 15u) == 0) {
      const uint32_t v16 = bytes >> 4;
      const uint4* s4 = reinterpret_cast<const uint4*>(src);
      uint4* d4 = reinterpret_cast<uint4*>(blob + dst);
      for (uint32_t i = threadIdx.x; i < v16; i += 256u) d4[i] = s4[i];
      for (uint32_t o = (v16 << 4) + threadIdx.x; o < bytes; o += 256u) blob[dst + o] = src[o];
    } else {
      for (uint32_t o = threadIdx.x; o < bytes; o += 256u) blob[dst + o] = src[o];
    }
    prev_end = dst + bytes;
  }
}

cudaError_t launch_str_assemble(const StrAsmWork* d_works, uint32_t n_batches, cudaStream_t s) {
  if (n_batches == 0) return cudaSuccess;
  k_str_assemble<<<n_batches, 256, 0, s>>>(d_works);
  return cudaGetLastError();
}

}  // namespace lc

// k_bits.cu — boolean_buffer_and_then on the device, plus the small result-assembly kernels (validity concatenation,
// sparse mask transfer, Utf8View views).
// Reference: /root/reference/src/datafusion/src/utils.rs:17-83 (semantics), :104-236 (the BMI2 PDEP
// routine, the only hand-written intrinsic in the reference). out bit p = left[p] AND the
// rank_left(p)-th bit of right, where right has popcount(left) bits. On the GPU the "deposit" is a
// rank computed from a prefix sum of per-word popcounts plus __popc(word & lanemask_lt).
#include "device_utils.cuh"
#include "fixed_math.cuh"
#include "kernels.h"

namespace lc {

__global__ void __launch_bounds__(256) k_and_then(const uint32_t* __restrict__ left, uint32_t left_bits,
                                                  const uint32_t* __restrict__ right, uint32_t* __restrict__ out) {
  __shared__ uint32_t s_tot[8];
  __shared__ uint32_t s_word[256];
  __shared__ uint32_t s_off[256];
  const uint32_t n_words = (left_bits + 31u) >> 5;
  const uint32_t tail = left_bits & 31u;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t carry = 0;
  for (uint32_t w0 = 0; w0 < n_words; w0 += 256u) {
    const uint32_t wi = w0 + threadIdx.x;
    uint32_t lw = 0;
    if (wi < n_words) {
      lw = left[wi];
      if (wi == n_words - 1u && tail) lw &= (1u << tail) - 1u;
    }
    uint32_t tot;
    const uint32_t excl = block_excl_scan_256(__popc(lw), s_tot, &tot);
    s_word[threadIdx.x] = lw;
    s_off[threadIdx.x] = carry + excl;
    __syncthreads();
    for (uint32_t j = 0; j < 32; ++j) {
      const uint32_t lwi = warp * 32u + j;
      if (w0 + lwi >= n_words) break;
      const uint32_t word = s_word[lwi];
      bool bit = false;
      if ((word >> lane) & 1u) {
        const uint32_t r = s_off[lwi] + __popc(word & lanemask_lt());
        bit = (right[r >> 5] >> (r & 31u)) & 1u;
      }
      const uint32_t o = __ballot_sync(kFullMask, bit);
      if (lane == 0) out[w0 + lwi] = o;
    }
    carry += tot;
    __syncthreads();
  }
}

// Concatenate per-entry validity bit strings (entry i: k_i bits starting at word valid_off[i] of valid_base, the
// layout the DECODE kernels write) into ONE bitmap of `rows` bits on the device — the Arrow validity buffer of the
// concatenated result, so a device-resident get() never visits the host (lc_scan_read_device).
// One thread per output word; entries without nulls (counts[i*stride+1] == 0) read as all ones.
__global__ void k_concat_validity(const uint32_t* __restrict__ valid_base, const uint64_t* __restrict__ valid_off,
                                  const uint64_t* __restrict__ row_base, const uint32_t* __restrict__ counts,
                                  uint32_t counts_stride, uint32_t n_entries, uint64_t rows, uint32_t* __restrict__ out) {
  const uint64_t w = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const uint64_t r0 = w * 32ull;
  if (r0 >= rows) return;
  // last entry whose first row is <= r0
  uint32_t lo = 0, hi = n_entries;
  while (hi - lo > 1u) {
    const uint32_t mid = (lo + hi) >> 1;
    if (row_base[mid] <= r0) lo = mid;
    else hi = mid;
  }
  uint32_t e = lo, filled = 0, word = 0;
  const uint32_t want = rows - r0 < 32ull ? static_cast<uint32_t>(rows - r0) : 32u;
  while (filled < want && e < n_entries) {
    const uint64_t b = row_base[e];
    const uint64_t end = e + 1u < n_entries ? row_base[e + 1u] : rows;
    const uint64_t pos = r0 + filled;
    if (pos >= end) {
      ++e;
      continue;
    }
    const uint32_t local = static_cast<uint32_t>(pos - b);
    const uint32_t avail = static_cast<uint32_t>(end - pos);
    const uint32_t take = avail < want - filled ? avail : want - filled;
    uint32_t bits = kFullMask;
    if (counts[static_cast<size_t>(e) * counts_stride + 1u] != 0u) {
      const uint32_t* vw = valid_base + valid_off[e];
      const uint32_t wi = local >> 5, sh = local & 31u;
      const uint32_t w0 = vw[wi];
      const uint32_t w1 = (sh + take > 32u) ? vw[wi + 1u] : 0u;
      bits = __funnelshift_r(w0, w1, sh);
    }
    if (take < 32u) bits &= (1u << take) - 1u;
    word |= bits << filled;
    filled += take;
  }
  out[w] = word;
}

// Sparse selection upload: the area was zero-filled, drop the few non-zero words in ({word index << 32 | word}).
__global__ void k_scatter_words(const unsigned long long* __restrict__ pairs, uint64_t n, uint32_t* __restrict__ base) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) base[pairs[i] >> 32] = static_cast<uint32_t>(pairs[i]);
}

// Sparse mask download: collect the non-zero words of a mask area as {word index << 32 | word}; counter[0] counts all of
// them, only the first `budget` are stored (the caller falls back to a dense copy when there are more).
__global__ void k_gather_nonzero(const uint32_t* __restrict__ words, uint64_t n_words, unsigned long long* __restrict__ pairs,
                                 uint64_t budget, unsigned long long* __restrict__ counter) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const uint32_t v = i < n_words ? words[i] : 0u;
  const uint32_t m = __ballot_sync(kFullMask, v != 0u);
  if (m == 0u) return;
  if (v != 0u) {  // exactly the lanes of m
    const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
    unsigned long long base = 0;
    if (lane == leader) base = atomicAdd(counter, static_cast<unsigned long long>(__popc(m)));
    base = __shfl_sync(m, base, leader);
    const unsigned long long idx = base + __popc(m & lanemask_lt());
    if (idx < budget) pairs[idx] = (static_cast<unsigned long long>(i) << 32) | v;
  }
}

// Utf8View / BinaryView result: one 16-byte view per row over the single data buffer the decode kernel filled
// ({length, 12 inline bytes} up to 12 bytes, else {length, 4-byte prefix, buffer index 0, offset}); null rows get an
// all-zero view. What arrow's cast Dictionary -> Utf8View leaves the reference's caller with (byte_view_array/mod.rs:287-290).
__global__ void __launch_bounds__(256) k_build_views(const int32_t* __restrict__ off, uint32_t total_bytes,
                                                     const uint8_t* __restrict__ data, const uint32_t* __restrict__ valid,
                                                     uint64_t rows, uint4* __restrict__ views) {
  const uint64_t r = static_cast<uint64_t>(blockIdx.x) * 256u + threadIdx.x;
  if (r >= rows) return;
  uint4 v = make_uint4(0u, 0u, 0u, 0u);
  const bool ok = valid ? ((valid[r >> 5] >> (r & 31u)) & 1u) : true;
  if (ok) {
    const uint32_t b = static_cast<uint32_t>(off[r]);
    const uint32_t e = r + 1u < rows ? static_cast<uint32_t>(off[r + 1u]) : total_bytes;
    const uint32_t len = e - b;
    uint32_t w[3] = {0u, 0u, 0u};
    const uint32_t take = len <= 12u ? len : 4u;
    for (uint32_t i = 0; i < take; ++i) w[i >> 2] |= static_cast<uint32_t>(data[b + i]) << (8u * (i & 3u));
    v.x = len;
    v.y = w[0];
    if (len <= 12u) {
      v.z = w[1];
      v.w = w[2];
    } else {
      v.z = 0u;  // buffer index
      v.w = b;   // offset
    }
  }
  views[r] = v;
}

// LiquidFixedLenByteArray keeps its 16 / 32-byte values in ORDER-PRESERVING form: the little-endian two's complement
// integer byte-reversed (big-endian) with the sign bit flipped, so that unsigned lexicographic byte order — what the
// byte-view comparison kernels implement — is the numeric order of the decimals. In place, one thread per value.
__global__ void __launch_bounds__(256) k_fixed_to_ordered(uint8_t* __restrict__ pool, uint32_t n, uint32_t width) {
  const uint32_t r = blockIdx.x * 256u + threadIdx.x;
  if (r >= n) return;
  fixed_to_ordered_inplace(pool + static_cast<size_t>(r) * width, width);
}

cudaError_t launch_fixed_to_ordered(uint8_t* d_pool, uint32_t n, uint32_t width, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  k_fixed_to_ordered<<<(n + 255u) / 256u, 256, 0, s>>>(d_pool, n, width);
  return cudaGetLastError();
}

// LiquidFixedLenByteArray result: the decoded values (variable-length form: offsets + bytes, null rows empty; order-preserving
// form, see k_fixed_to_ordered) back as little-endian integers at their fixed stride, null slots zero. One thread per 4
// bytes of output.
__global__ void __launch_bounds__(256) k_fixed_from_var(const int32_t* __restrict__ off, uint32_t total_bytes,
                                                        const uint8_t* __restrict__ data, const uint32_t* __restrict__ valid,
                                                        uint64_t rows, uint32_t width, uint32_t* __restrict__ out) {
  const uint64_t t = static_cast<uint64_t>(blockIdx.x) * 256u + threadIdx.x;
  const uint32_t words_per_row = width >> 2;
  const uint64_t r = t / words_per_row;
  if (r >= rows) return;
  const uint32_t wdx = static_cast<uint32_t>(t % words_per_row);
  const bool ok = valid ? ((valid[r >> 5] >> (r & 31u)) & 1u) : true;
  uint32_t v = 0;
  if (ok) {
    const uint32_t b = static_cast<uint32_t>(off[r]);
    const uint32_t e = r + 1u < rows ? static_cast<uint32_t>(off[r + 1u]) : total_bytes;
    if (e - b == width) {  // always, for an entry built from fixed-width values
      v = fixed_le_word(data + b, width, wdx);
    }
  }
  out[t] = v;
}

cudaError_t launch_fixed_from_var(const int32_t* d_offsets, uint32_t total_bytes, const uint8_t* d_data, const uint32_t* d_validity,
                                  uint64_t rows, uint32_t width, void* d_out, cudaStream_t s) {
  if (rows == 0) return cudaSuccess;
  const uint64_t threads = rows * (width >> 2);
  k_fixed_from_var<<<static_cast<uint32_t>((threads + 255) / 256), 256, 0, s>>>(d_offsets, total_bytes, d_data, d_validity, rows, width,
                                                                               static_cast<uint32_t*>(d_out));
  return cudaGetLastError();
}

cudaError_t launch_build_views(const int32_t* d_offsets, uint32_t total_bytes, const uint8_t* d_data, const uint32_t* d_validity,
                               uint64_t rows, void* d_views, cudaStream_t s) {
  if (rows == 0) return cudaSuccess;
  k_build_views<<<static_cast<uint32_t>((rows + 255) / 256), 256, 0, s>>>(d_offsets, total_bytes, d_data, d_validity, rows,
                                                                           static_cast<uint4*>(d_views));
  return cudaGetLastError();
}

cudaError_t launch_gather_nonzero(const uint32_t* d_words, uint64_t n_words, unsigned long long* d_pairs, uint64_t budget,
                                  unsigned long long* d_counter, cudaStream_t s) {
  if (n_words == 0) return cudaSuccess;
  k_gather_nonzero<<<static_cast<uint32_t>((n_words + 255) / 256), 256, 0, s>>>(d_words, n_words, d_pairs, budget, d_counter);
  return cudaGetLastError();
}

cudaError_t launch_scatter_words(const unsigned long long* d_pairs, uint64_t n, uint32_t* d_base, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  k_scatter_words<<<static_cast<uint32_t>((n + 255) / 256), 256, 0, s>>>(d_pairs, n, d_base);
  return cudaGetLastError();
}

cudaError_t launch_concat_validity(const uint32_t* d_valid_base, const uint64_t* d_valid_off, const uint64_t* d_row_base,
                                   const uint32_t* d_counts, uint32_t counts_stride, uint32_t n_entries, uint64_t rows,
                                   uint32_t* d_out, cudaStream_t s) {
  if (rows == 0 || n_entries == 0) return cudaSuccess;
  const uint64_t words = (rows + 31) / 32;
  k_concat_validity<<<static_cast<uint32_t>((words + 127) / 128), 128, 0, s>>>(d_valid_base, d_valid_off, d_row_base,
                                                                               d_counts, counts_stride, n_entries, rows, d_out);
  return cudaGetLastError();
}

cudaError_t launch_and_then(const uint32_t* d_left, uint32_t left_bits, const uint32_t* d_right, uint32_t* d_out,
                            cudaStream_t s) {
  if (left_bits == 0) return cudaSuccess;
  k_and_then<<<1, 256, 0, s>>>(d_left, left_bits, d_right, d_out);
  return cudaGetLastError();
}

// lc_scan_filter_or: the merge that closes one disjunct. `term` holds the rows of the disjunct's remainder that passed
// every one of its terms, `acc` the rows accepted by the disjuncts before it, `sel` the running selection (sel_all: every
// row). Not last: acc := acc | term, term := sel & ~acc (where the next disjunct starts). Last: sel := acc | term and
// counts[2i] its popcount (counts[2i + 1] = 0, the stride-2 layout of the REFINE kernels). One warp per batch, 16-byte
// words; bits at or past rows[i], and the padding up to the batch's 4-word boundary, are written as zero whatever the
// refine kernels left there.
__global__ void __launch_bounds__(256) k_sel_or(uint32_t* __restrict__ sel, uint32_t sel_all, uint32_t* __restrict__ term,
                                                uint32_t* __restrict__ acc, const uint64_t* __restrict__ word_off,
                                                const uint32_t* __restrict__ rows, uint32_t n, uint32_t first, uint32_t last,
                                                uint32_t* __restrict__ counts) {
  const uint32_t b = blockIdx.x * 8u + (threadIdx.x >> 5);
  if (b >= n) return;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t r = rows[b];
  const uint32_t full = r >> 5, tail = r & 31u;
  const uint32_t vecs = (((r + 31u) >> 5) + 3u) >> 2;
  const uint64_t base = word_off[b] >> 2;  // batches start on a 4-word boundary
  uint4* T = reinterpret_cast<uint4*>(term) + base;
  uint4* A = reinterpret_cast<uint4*>(acc) + base;
  uint4* S = reinterpret_cast<uint4*>(sel) + base;
  uint32_t survivors = 0;
  for (uint32_t v = lane; v < vecs; v += 32u) {
    uint32_t valid[4];
#pragma unroll
    for (uint32_t j = 0; j < 4; ++j) {
      const uint32_t w = v * 4u + j;
      valid[j] = w < full ? kFullMask : (w == full && tail ? (1u << tail) - 1u : 0u);
    }
    const uint4 t = T[v];
    const uint4 a = first ? make_uint4(0u, 0u, 0u, 0u) : A[v];
    const uint4 u = make_uint4((a.x | t.x) & valid[0], (a.y | t.y) & valid[1], (a.z | t.z) & valid[2], (a.w | t.w) & valid[3]);
    if (last) {
      S[v] = u;
      survivors += __popc(u.x) + __popc(u.y) + __popc(u.z) + __popc(u.w);
    } else {
      A[v] = u;
      const uint4 s = sel_all ? make_uint4(valid[0], valid[1], valid[2], valid[3]) : S[v];
      T[v] = make_uint4(s.x & ~u.x & valid[0], s.y & ~u.y & valid[1], s.z & ~u.z & valid[2], s.w & ~u.w & valid[3]);
    }
  }
  if (last) {
    survivors = warp_sum(survivors);
    if (lane == 0) {
      counts[2u * b] = survivors;
      counts[2u * b + 1u] = 0u;
    }
  }
}

cudaError_t launch_sel_or(uint32_t* d_sel, bool sel_all, uint32_t* d_term, uint32_t* d_acc, const uint64_t* d_word_off,
                          const uint32_t* d_rows, uint32_t n, bool first, bool last, uint32_t* d_counts, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  k_sel_or<<<(n + 7u) / 8u, 256, 0, s>>>(d_sel, sel_all ? 1u : 0u, d_term, d_acc, d_word_off, d_rows, n, first ? 1u : 0u,
                                         last ? 1u : 0u, d_counts);
  return cudaGetLastError();
}

}  // namespace lc

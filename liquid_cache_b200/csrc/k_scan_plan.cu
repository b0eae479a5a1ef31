// k_scan_plan.cu — the bookkeeping of a get-with-selection done ON THE DEVICE, so that reading the survivors of a scan
// costs the host one synchronisation instead of three.
//
// read_from_cache (src/datafusion/src/reader/runtime/liquid_cache_reader.rs:342-391) reads every projected column with the
// final selection; the reference learns each batch's row count from the BooleanBuffer it holds. Here the selection lives in
// HBM, and what the decode kernels need before they can run — where each entry's rows, validity words, dictionary-length
// scratch and bytes start in the concatenated result — are prefix sums over per-entry counts that are themselves on the
// device. Round 1 fetched the counts, summed on the host and uploaded the offsets (twice for byte views: rows, then bytes).
// These two single-CTA kernels do the sums in place; the host only reads a 64-byte header together with the result.
#include "device_utils.cuh"
#include "kernels.h"

namespace lc {

// 1024 threads; thread t owns a short contiguous run of entries: serial over the run, block-wide over the runs.
template <int NV>
__device__ __forceinline__ void block_scan_runs(uint64_t (&v)[NV], uint64_t (&excl)[NV], uint64_t (&total)[NV], uint64_t* smem /*[NV][32]*/) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < NV; ++q) {
    uint64_t x = v[q];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint64_t y = __shfl_up_sync(kFullMask, x, d);
      if (lane >= static_cast<uint32_t>(d)) x += y;
    }
    if (lane == 31u) smem[q * 32 + warp] = x;
    excl[q] = x - v[q];
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int q = 0; q < NV; ++q) {
      const uint64_t w = smem[q * 32 + lane];
      uint64_t x = w;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint64_t y = __shfl_up_sync(kFullMask, x, d);
        if (lane >= static_cast<uint32_t>(d)) x += y;
      }
      smem[q * 32 + lane] = x - w;  // exclusive base of each warp
      if (lane == 31u) smem[NV * 32 + q] = x;  // grand total
    }
  }
  __syncthreads();
#pragma unroll
  for (int q = 0; q < NV; ++q) {
    excl[q] += smem[q * 32 + warp];
    total[q] = smem[NV * 32 + q];
  }
}

// Both kernels walk the entries in tiles of 4096 — four consecutive entries per thread, loads of the next tile issued before
// the block scan of the current one — so that a 12 k-entry list is three short rounds of coalesced traffic. (One
// contiguous run of n / 1024 entries per thread would be twelve dependent, uncoalesced loads deep.)
constexpr uint32_t kPlanPer = 4, kPlanTile = 1024 * kPlanPer;

// counts2[2i] = rows of entry i that survived (MODE_REFINE's count). Writes, for every entry: row_base (rows before it),
// vword_off (validity words before it, 4-word aligned per entry as the decode kernels lay them out), ulen_off (dictionary
// length scratch before it; only entries with survivors take space). Refuses (hdr->overflow) when a capacity is too small.
__global__ void __launch_bounds__(1024) k_scan_plan_rows(const uint32_t* __restrict__ counts2, const uint32_t* __restrict__ n_unique,
                                                         uint32_t n, uint64_t cap_rows, uint64_t cap_ulen, uint64_t* row_base,
                                                         uint64_t* vword_off, uint64_t* ulen_off, ScanPlanHdr* hdr) {
  __shared__ uint64_t smem[3 * 32 + 3];
  __shared__ uint32_t s_hits;
  if (threadIdx.x == 0) s_hits = 0;
  uint64_t carry[3] = {0, 0, 0};
  uint32_t hits = 0;
  uint32_t k[kPlanPer], u[kPlanPer], nk[kPlanPer], nu[kPlanPer];
  auto load = [&](uint32_t tile0, uint32_t (&kk)[kPlanPer], uint32_t (&uu)[kPlanPer]) {
#pragma unroll
    for (uint32_t j = 0; j < kPlanPer; ++j) {
      const uint32_t i = tile0 + threadIdx.x * kPlanPer + j;
      kk[j] = i < n ? counts2[2u * i] : 0u;
      uu[j] = (i < n && n_unique) ? n_unique[i] : 0u;
    }
  };
  load(0, nk, nu);
  for (uint32_t tile0 = 0; tile0 < n; tile0 += kPlanTile) {
#pragma unroll
    for (uint32_t j = 0; j < kPlanPer; ++j) {
      k[j] = nk[j];
      u[j] = nu[j];
    }
    if (tile0 + kPlanTile < n) load(tile0 + kPlanTile, nk, nu);
    uint64_t v[3] = {0, 0, 0};
#pragma unroll
    for (uint32_t j = 0; j < kPlanPer; ++j) {
      v[0] += k[j];
      v[1] += ((k[j] + 31u) / 32u + 3u) & ~3u;
      if (k[j]) {
        ++hits;
        v[2] += (u[j] + 3u) & ~3u;
      }
    }
    uint64_t excl[3], total[3];
    block_scan_runs<3>(v, excl, total, smem);
    uint64_t r = carry[0] + excl[0], w = carry[1] + excl[1], q = carry[2] + excl[2];
#pragma unroll
    for (uint32_t j = 0; j < kPlanPer; ++j) {
      const uint32_t i = tile0 + threadIdx.x * kPlanPer + j;
      if (i < n) {
        row_base[i] = r;
        vword_off[i] = w;
        ulen_off[i] = q;
      }
      r += k[j];
      w += ((k[j] + 31u) / 32u + 3u) & ~3u;
      if (k[j]) q += (u[j] + 3u) & ~3u;
    }
#pragma unroll
    for (int t = 0; t < 3; ++t) carry[t] += total[t];
    __syncthreads();  // the scan's shared words are reused by the next tile
  }
  // entries with survivors (for the record; the decode kernels skip the others by their count)
  uint32_t h = hits;
  for (int d = 16; d > 0; d >>= 1) h += __shfl_xor_sync(kFullMask, h, d);
  if ((threadIdx.x & 31u) == 0 && h) atomicAdd(&s_hits, h);
  __syncthreads();
  if (threadIdx.x == 0) {
    hdr->n_hit = s_hits;
    hdr->rows = carry[0];
    hdr->vwords = carry[1];
    hdr->ulen_words = carry[2];
    hdr->bytes = 0;
    hdr->nulls = 0;
    hdr->overflow = (carry[0] > cap_rows || carry[2] > cap_ulen) ? 1u : 0u;
  }
}

// counts4[4i + 2] = decoded bytes of entry i's surviving rows (k_str_lengths; 0 where no row survived),
// counts4[4i + 1] = nulls among them. Writes byte_base and the closing offset of the concatenated array.
__global__ void __launch_bounds__(1024) k_scan_plan_bytes(const uint32_t* __restrict__ counts4, uint32_t n, uint64_t cap_bytes,
                                                          uint64_t* byte_base, int32_t* out_offsets, ScanPlanHdr* hdr) {
  __shared__ uint64_t smem[2 * 32 + 2];
  if (hdr->overflow) return;
  uint64_t carry[2] = {0, 0};
  uint32_t b[kPlanPer], z[kPlanPer], nb[kPlanPer], nz[kPlanPer];
  auto load = [&](uint32_t tile0, uint32_t (&bb)[kPlanPer], uint32_t (&zz)[kPlanPer]) {
#pragma unroll
    for (uint32_t j = 0; j < kPlanPer; ++j) {
      const uint32_t i = tile0 + threadIdx.x * kPlanPer + j;
      const uint4 c = i < n ? reinterpret_cast<const uint4*>(counts4)[i] : make_uint4(0, 0, 0, 0);  // one 16-byte record per entry
      bb[j] = c.z;
      zz[j] = c.y;
    }
  };
  load(0, nb, nz);
  for (uint32_t tile0 = 0; tile0 < n; tile0 += kPlanTile) {
#pragma unroll
    for (uint32_t j = 0; j < kPlanPer; ++j) {
      b[j] = nb[j];
      z[j] = nz[j];
    }
    if (tile0 + kPlanTile < n) load(tile0 + kPlanTile, nb, nz);
    uint64_t v[2] = {0, 0};
#pragma unroll
    for (uint32_t j = 0; j < kPlanPer; ++j) {
      v[0] += b[j];
      v[1] += z[j];
    }
    uint64_t excl[2], total[2];
    block_scan_runs<2>(v, excl, total, smem);
    uint64_t r = carry[0] + excl[0];
#pragma unroll
    for (uint32_t j = 0; j < kPlanPer; ++j) {
      const uint32_t i = tile0 + threadIdx.x * kPlanPer + j;
      if (i < n) byte_base[i] = r;
      r += b[j];
    }
    carry[0] += total[0];
    carry[1] += total[1];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    hdr->bytes = carry[0];
    hdr->nulls = carry[1];
    if (carry[0] > cap_bytes || carry[0] > 0x7fffffffull) hdr->overflow = 2u;
    else out_offsets[hdr->rows] = static_cast<int32_t>(carry[0]);
  }
}

cudaError_t launch_scan_plan_rows(const uint32_t* d_counts2, const uint32_t* d_n_unique, uint32_t n, uint64_t cap_rows, uint64_t cap_ulen,
                                  uint64_t* d_row_base, uint64_t* d_vword_off, uint64_t* d_ulen_off, ScanPlanHdr* d_hdr, cudaStream_t s) {
  k_scan_plan_rows<<<1, 1024, 0, s>>>(d_counts2, d_n_unique, n, cap_rows, cap_ulen, d_row_base, d_vword_off, d_ulen_off, d_hdr);
  return cudaGetLastError();
}

cudaError_t launch_scan_plan_bytes(const uint32_t* d_counts4, uint32_t n, uint64_t cap_bytes, uint64_t* d_byte_base,
                                   int32_t* d_out_offsets, ScanPlanHdr* d_hdr, cudaStream_t s) {
  k_scan_plan_bytes<<<1, 1024, 0, s>>>(d_counts4, n, cap_bytes, d_byte_base, d_out_offsets, d_hdr);
  return cudaGetLastError();
}

}  // namespace lc

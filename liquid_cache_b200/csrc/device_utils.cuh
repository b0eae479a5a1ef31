// device_utils.cuh — sm_90a device helpers: TMA bulk copy + mbarrier, warp scans, bit sinks.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace lc {

constexpr uint32_t kFullMask = 0xffffffffu;

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// 32-bit load from a shared-memory address (smem_u32): keeps the hot loops on LDS with 32-bit address math.
// Not volatile: the compiler may schedule it freely; callers order it after barriers through data dependences.
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}

// ---- mbarrier + cp.async.bulk (TMA 1-D bulk copy, SASS: UBLKCP) -------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  // make the init visible to the async proxy before a bulk copy signals the barrier
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// global -> shared bulk copy; dst/src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0;
  const uint32_t addr = smem_u32(bar);
  while (!done) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
  }
}

// ---- warp helpers --------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t lanemask_lt() {
  uint32_t m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t t = __shfl_up_sync(kFullMask, v, d);
    if (lane >= d) v += t;
  }
  return v;
}

__device__ __forceinline__ uint32_t warp_sum(uint32_t v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(kFullMask, v, d);
  return v;
}

// Block-wide exclusive scan for a 256-thread CTA. `warp_tot` is 8 words of shared memory.
// Returns the exclusive prefix of `v`; *total gets the block sum. Contains two __syncthreads().
__device__ __forceinline__ uint32_t block_excl_scan_256(uint32_t v, uint32_t* warp_tot, uint32_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t incl = warp_incl_scan(v, lane);
  __syncthreads();  // warp_tot may still be read from a previous round
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  uint32_t base = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < 8; ++w) {
    uint32_t t = warp_tot[w];
    if (w < warp) base += t;
    tot += t;
  }
  *total = tot;
  return base + incl - v;
}

// Compact the per-lane 2-bit payload of the lanes selected by `selw` to the low lanes
// (a warp-wide PEXT): returns {bit0 stream, bit1 stream} as two k-bit words, k = popc(selw).
// `scratch` is 32 bytes of shared memory private to the warp.
__device__ __forceinline__ void warp_pext2(uint32_t payload, uint32_t selw, int lane, uint8_t* scratch,
                                           uint32_t* out0, uint32_t* out1) {
  if (selw == kFullMask) {
    *out0 = __ballot_sync(kFullMask, payload & 1u);
    *out1 = __ballot_sync(kFullMask, payload & 2u);
    return;
  }
  const uint32_t rank = __popc(selw & lanemask_lt());
  if ((selw >> lane) & 1u) scratch[rank] = static_cast<uint8_t>(payload);
  __syncwarp();
  const uint32_t k = __popc(selw);
  const uint32_t b = (static_cast<uint32_t>(lane) < k) ? scratch[lane] : 0u;
  *out0 = __ballot_sync(kFullMask, b & 1u);
  *out1 = __ballot_sync(kFullMask, b & 2u);
  __syncwarp();
}

// Append a k-bit string at bit position `pos` of a zero-initialised shared-memory bit buffer.
// Called by ONE lane; neighbouring warps may touch the same word, hence the atomics.
__device__ __forceinline__ void bits_append(uint32_t* buf, uint32_t pos, uint32_t k, uint32_t bits) {
  if (k == 0) return;
  const uint32_t w = pos >> 5, sh = pos & 31u;
  atomicOr(&buf[w], bits << sh);
  if (sh + k > 32u) atomicOr(&buf[w + 1], bits >> (32u - sh));
}

}  // namespace lc

// k_int_bits.cu — integer predicates with FULL-LENGTH outputs (MODE_REFINE: selection &= valid & cmp; MODE_PRED over all
// rows), the shape every conjunct of a scan has: register-resident FastLanes unpack, one warp per 1024-row chunk.
//
// Reference semantics restated (under /root/reference/src/core/src/liquid_array/): try_eval_predicate = decode, arrow
// filter, compare (primitive_array.rs:370-379, mod.rs:265-280, raw/bit_pack_array.rs:127-169); the caller's nulls->false
// and boolean_buffer_and_then (datafusion/src/cache/column.rs:134-137, datafusion/src/utils.rs:62-83) are the AND with
// validity and selection at the end of each chunk. The compare runs in the packed domain (int_plan.cuh).
//
// Why not the staged kernel (k_int_scan) here: on narrow columns (W = 12 .. 20: dates, EventTime, ids) an entry is only
// 12-20 KB, and a CTA that stages it by TMA, plans, synchronises and hands each of its 8 warps ONE chunk spends most of
// its time in the per-entry bookkeeping rather than on the bytes. A chunk of a
// W-bit column is W rows of 128 bytes and every thread needs exactly W 32-bit words of it (breg_math.cuh), so a warp can
// pull its chunk straight into registers with W coalesced loads (each instruction covers one or two whole 128-byte
// lines: the access pattern a TMA tile would give, without the shared-memory round trip and its barriers) and run the 32
// steps as straight-line code with immediate shifts and masks: ~6 instructions per 32 rows. Warps are independent — no
// __syncthreads, no mbarrier — so the SM overlaps the loads of some chunks with the ALU work of others by itself.
// Per-entry header words and the next task's blob pointer are fetched one / two tasks ahead (software pipeline in
// registers), so the only exposed latency per chunk is its own data.
#include <cstddef>
#include <cstdlib>

#include "breg_math.cuh"
#include "device_utils.cuh"
#include "int_plan.cuh"
#include "kernels.h"

namespace lc {

struct GlobalLoader {
  const uint8_t* p;
  __device__ __forceinline__ uint32_t ld8(uint32_t o) const { return __ldg(p + o); }
  __device__ __forceinline__ uint32_t ld16(uint32_t o) const { return __ldg(reinterpret_cast<const uint16_t*>(p + o)); }
  __device__ __forceinline__ uint32_t ld32(uint32_t o) const { return __ldg(reinterpret_cast<const uint32_t*>(p + o)); }
  __device__ __forceinline__ void ld64(uint32_t o, uint32_t* lo, uint32_t* hi) const {
    const uint2 v = __ldg(reinterpret_cast<const uint2*>(p + o));
    *lo = v.x;
    *hi = v.y;
  }
};

// chunks a warp keeps in flight for a W-bit field of a T-bit column: as many as fit ~40 registers of packed words
template <uint32_t T, uint32_t W>
__host__ __device__ constexpr uint32_t chunks_in_flight() {
  constexpr uint32_t regs = BregGeom<T, W>::SUB * BregGeom<T, W>::NW;
  return regs <= 10u ? 4u : (regs <= 20u ? 2u : 1u);
}

// Membership of one packed value in a warp's set. Not inlined: the 32 unrolled steps of every (T, W) instantiation call it
// instead of each carrying a copy of the search (which multiplies the build time of this file for no gain in speed).
__device__ __noinline__ bool in_warp_set(uint32_t u, const uint32_t* set, uint32_t n) {
  return in_sorted<uint32_t>(u, n, [&](uint32_t i) { return set[i]; });
}

// The per-row test of a chunk, before negation: the range of a comparison, or (IN lists, SET) membership in the entry's
// in-window list values, ascending packed offsets in the warp's slice of shared memory (set_n == 0: the entry's plan
// lowered to a range after all).
template <bool SET>
struct RowTest {
  URange<uint32_t> g;
  const uint32_t* set;
  uint32_t set_n;
  __device__ __forceinline__ bool operator()(uint32_t u) const {
    if constexpr (SET) {
      if (set_n) return in_warp_set(u, set, set_n);
    }
    return (u - g.lo) <= g.span;
  }
};

// One group of chunks [c0, c1) of an entry: every chunk's mask word is finished (negation, validity,
// selection, tail), stored, and its survivors counted. Returns the survivors of the group (per lane, to be summed).
// A group that ends inside a CH-wide step (entries whose chunk count is not a multiple of CH) re-reads its last chunk
// in the surplus slots and drops their words.
template <uint32_t T, uint32_t W, bool SET>
__device__ __forceinline__ uint32_t bits_group(const uint8_t* packed, uint32_t c0, uint32_t c1, uint32_t lane, uint32_t ordl,
                                               const RowTest<SET>& rt, uint32_t n, const uint32_t* sel, const uint32_t* valid,
                                               uint32_t* out_bits, uint32_t* out_valid, uint32_t* strip) {
  const URange<uint32_t>& g = rt.g;
  constexpr uint32_t CH = chunks_in_flight<T, W>();
  using G = BregGeom<T, W>;
  const uint32_t n_words = (n + 31u) >> 5;
  uint32_t survivors = 0;
  for (uint32_t c = c0; c < c1; c += CH) {
    // (asking the next round's lines into L2 ahead of time — one prefetch per lane — is a variant not taken)
    // the packed words of the CH chunks first: nothing they need is still in flight (the header came one task ahead) ...
    uint32_t a[CH][G::SUB][G::NW];
#pragma unroll
    for (uint32_t q = 0; q < CH; ++q) {
      const uint32_t cq = c + q < c1 ? c + q : c1 - 1u;
      breg_load<T, W>(lane, a[q], GlobalLoader{packed + static_cast<size_t>(cq) * (128u * W)});
    }
    // ... then their selection / validity words (`sel` hangs off a per-entry offset that may itself still be arriving);
    // both are consumed after the 32 steps
    uint32_t sw[CH], vw[CH];
#pragma unroll
    for (uint32_t q = 0; q < CH; ++q) {
      const uint32_t wi = (c + q) * 32u + ordl;
      sw[q] = kFullMask;
      vw[q] = kFullMask;
      if (c + q < c1 && wi < n_words) {
        if (sel) sw[q] = sel[wi];
        if (valid) vw[q] = __ldg(valid + wi);
      }
    }
#pragma unroll
    for (uint32_t q = 0; q < CH; ++q) {
      // step s's ballot is mask word out_word(s): lane 0 parks it in the warp's 32-word strip of shared memory and lane s
      // picks it up afterwards (one predicated store per step instead of a compare + select per step in every lane)
#pragma unroll
      for (uint32_t s = 0; s < 32; ++s) {
        const uint32_t u = breg_value<T, W>(a[q], s);
        const uint32_t cw = __ballot_sync(kFullMask, rt(u));
        if (lane == 0) strip[s] = cw;
      }
      __syncwarp();
      const uint32_t mine = strip[lane];
      __syncwarp();
      const uint32_t wi = (c + q) * 32u + ordl;
      if (c + q < c1 && wi < n_words) {
        uint32_t v = vw[q];
        if (wi == n_words - 1u && (n & 31u)) v &= (1u << (n & 31u)) - 1u;  // rows past n in the padded last chunk
        const uint32_t cw = (g.neg ? ~mine : mine) & v & sw[q];
        out_bits[wi] = cw;
        if (out_valid) out_valid[wi] = v;
        survivors += __popc(cw);
      }
    }
  }
  return survivors;
}

template <uint32_t T, bool SET>
__device__ __forceinline__ uint32_t bits_group_w(uint32_t W, const uint8_t* packed, uint32_t c0, uint32_t c1, uint32_t lane,
                                                 uint32_t ordl, const RowTest<SET>& g, uint32_t n, const uint32_t* sel,
                                                 const uint32_t* valid, uint32_t* out_bits, uint32_t* out_valid, uint32_t* strip) {
  switch (W) {
#define LC_W(k) \
  case k:       \
    if constexpr (k <= T) return bits_group<T, k, SET>(packed, c0, c1, lane, ordl, g, n, sel, valid, out_bits, out_valid, strip); \
    break;
    LC_W(1) LC_W(2) LC_W(3) LC_W(4) LC_W(5) LC_W(6) LC_W(7) LC_W(8) LC_W(9) LC_W(10) LC_W(11) LC_W(12) LC_W(13) LC_W(14) LC_W(15) LC_W(16)
    LC_W(17) LC_W(18) LC_W(19) LC_W(20) LC_W(21) LC_W(22) LC_W(23) LC_W(24) LC_W(25) LC_W(26) LC_W(27) LC_W(28) LC_W(29) LC_W(30) LC_W(31) LC_W(32)
#undef LC_W
  }
  return 0;
}

// Header words of one entry, as the pipeline carries them (all lanes hold the same values: broadcast loads).
struct HdrRegs {
  uint32_t w1;        // phys | tbits << 8 | bit_width << 16 | has_nulls << 24
  uint32_t n;
  uint64_t reference;
  uint32_t validity_off, packed_off, null_count, is_signed;
  uint32_t sq_lo, sq_hi, sq_kind;  // squeezed entries: bucket width words + kind (int_bucket_width)
};

__device__ __forceinline__ void load_hdr(const uint8_t* blob, HdrRegs& r) {
  const uint32_t* h32 = reinterpret_cast<const uint32_t*>(blob);
  r.w1 = __ldg(h32 + 1);
  r.n = __ldg(h32 + 2);
  r.reference = __ldg(reinterpret_cast<const unsigned long long*>(blob + 16));
  r.validity_off = __ldg(h32 + 6);
  r.packed_off = __ldg(h32 + 7);
  r.null_count = __ldg(h32 + 9);
  r.is_signed = __ldg(h32 + 10);
  r.sq_lo = __ldg(h32 + 13);
  r.sq_hi = __ldg(h32 + 14);
  r.sq_kind = __ldg(h32 + 15);
}
static_assert(offsetof(IntHeader, n) == 8 && offsetof(IntHeader, reference) == 16 && offsetof(IntHeader, validity_off) == 24 &&
                  offsetof(IntHeader, packed_off) == 28 && offsetof(IntHeader, null_count) == 36 &&
                  offsetof(IntHeader, is_signed) == 40 && offsetof(IntHeader, patch_idx_off) == 52 &&
                  offsetof(IntHeader, patch_val_off) == 56 && offsetof(IntHeader, squeeze_kind) == 60,
              "k_int_bits reads the header by word offset");

// Tasks: (entry e, group g of `1 << cshift` chunks) = (t >> gshift, t & (gpe - 1)) for t = global warp id, + total warps, ...;
// gpe = groups of the longest entry of the list rounded up to a power of two (1 for 8192-row batches in groups of eight
// chunks), shorter entries have idle tasks. The warps of a CTA take consecutive tasks, i.e. the groups of neighbouring entries. Per task the
// header is read once and the predicate planned once; the header of the warp's next task and the blob pointer of the
// one after are already in flight (software pipeline in registers).
// SET: IN / NOT IN lists (pred.op, values in `in`), planned per task by plan_int_in's two steps — the warp counts the list
// values below / inside the entry's window with one vote per 32 values, lower_in_slice picks constant, range or set, and a
// set is copied into the warp's slice of shared memory as packed offsets. The rows are still read in one pass.
template <int OCC, bool SET>
__global__ void __launch_bounds__(256, OCC) k_int_bits(ScanIo io, IntPredDesc pred, uint32_t n_entries, uint32_t gshift, uint32_t cshift, int mode,
                                                     IntInList in) {
  __shared__ uint32_t s_strip[8][32];  // per warp: the 32 ballots of a chunk, transposed through shared memory
  __shared__ uint32_t s_set[SET ? 8 : 1][SET ? kInListMaxValues : 1];  // per warp: the set of its current task
  const uint32_t lane = threadIdx.x & 31u;
  uint32_t* strip = s_strip[threadIdx.x >> 5];
  const uint32_t warps_total = gridDim.x * 8u;
  const uint32_t n_tasks = n_entries << gshift;
  const uint32_t gmask = (1u << gshift) - 1u;
  uint32_t t = blockIdx.x * 8u + (threadIdx.x >> 5);
  if (t >= n_tasks) return;
  const uint8_t* blob0 = io.refs[t >> gshift].blob;
  HdrRegs h0;
  load_hdr(blob0, h0);
  const uint8_t* blob1 = (t + warps_total < n_tasks) ? io.refs[(t + warps_total) >> gshift].blob : nullptr;
  for (; t < n_tasks; t += warps_total) {
    const uint32_t e = t >> gshift, grp = t & gmask;
    const uint32_t t1 = t + warps_total, t2 = t1 + warps_total;
    HdrRegs h1 = h0;
    if (t1 < n_tasks) load_hdr(blob1, h1);                                         // arrives while this group is worked on
    const uint8_t* blob2 = (t2 < n_tasks) ? io.refs[t2 >> gshift].blob : nullptr;

    const uint32_t tbits = (h0.w1 >> 8) & 0xffu, W = (h0.w1 >> 16) & 0xffu, n = h0.n;
    const uint32_t n_chunks = (n + 1023u) >> 10;
    const uint32_t gsz = 1u << cshift;
    const uint32_t c0 = grp * gsz, c1 = c0 + gsz < n_chunks ? c0 + gsz : n_chunks;
    if (c0 < n_chunks) {
      const uint32_t ordl = tbits >= 32u ? breg_out_word<32>(lane) : (tbits == 16u ? breg_out_word<16>(lane) : lane);
      const uint32_t* sel = nullptr;
      if (io.sel_base) {
        const uint64_t so = io.sel_off[e];
        if (so != kNoSel) sel = io.sel_base + so;
      }
      uint32_t* out_bits = reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(io.out_base) + io.out_off[e] * 4u);
      uint32_t* out_valid = (mode == MODE_PRED && io.valid_base && (h0.w1 >> 24)) ? io.valid_base + io.valid_off[e] : nullptr;
      const uint32_t* valid = (h0.w1 >> 24) ? reinterpret_cast<const uint32_t*>(blob0 + h0.validity_off) : nullptr;
      // plan: (op, literal) in the packed domain of THIS entry (the same for all lanes)
      IntHeader hh{};
      hh.tbits = static_cast<uint8_t>(tbits);
      hh.bit_width = static_cast<uint8_t>(W);
      hh.reference = h0.reference;
      hh.is_signed = h0.is_signed;
      hh.patch_idx_off = h0.sq_lo;
      hh.patch_val_off = h0.sq_hi;
      hh.squeeze_kind = static_cast<uint8_t>(h0.sq_kind & 0xffu);
      RowTest<SET> g;
      g.set = nullptr;
      g.set_n = 0;
      if constexpr (SET) {
        uint32_t below = 0, inside = 0;
        if (W != 0u) {
          for (uint32_t i = lane; i < in.n; i += 32u) {
            const int where = in_value_window(&hh, __ldg(reinterpret_cast<const unsigned long long*>(in.v) + i));
            below += where < 0 ? 1u : 0u;
            inside += where == 0 ? 1u : 0u;
          }
          below = warp_sum(below);
          inside = warp_sum(inside);
        }
        if (lower_in_slice<uint32_t>(&hh, pred.op, in, below, below + inside, &g.g)) {
          uint32_t* set = s_set[threadIdx.x >> 5];
          const uint32_t ref = static_cast<uint32_t>(window_ref(&hh));
          __syncwarp();  // the previous task's lookups are done
          for (uint32_t i = lane; i < inside; i += 32u) set[i] = static_cast<uint32_t>(in.v[below + i]) - ref;
          __syncwarp();
          g.set = set;
          g.set_n = inside;
        }
      } else {
        int32_t kind = UC_FALSE;
        uint64_t thr64 = 0;
        plan_int_pred(&hh, pred, &kind, &thr64);
        g.g = make_range<uint32_t>(kind, thr64);
      }
      uint32_t survivors = 0;
      if (W != 0u) {
        const uint8_t* packed = blob0 + h0.packed_off;
        switch (tbits) {
          case 8: survivors = bits_group_w<8>(W, packed, c0, c1, lane, ordl, g, n, sel, valid, out_bits, out_valid, strip); break;
          case 16: survivors = bits_group_w<16>(W, packed, c0, c1, lane, ordl, g, n, sel, valid, out_bits, out_valid, strip); break;
          case 32: survivors = bits_group_w<32>(W, packed, c0, c1, lane, ordl, g, n, sel, valid, out_bits, out_valid, strip); break;
          default: survivors = bits_group_w<64>(W, packed, c0, c1, lane, ordl, g, n, sel, valid, out_bits, out_valid, strip); break;
        }
      } else {  // W == 0: entirely null, nothing packed (bit_pack_array.rs:18): every mask bit is false
        const uint32_t n_words = (n + 31u) >> 5;
        for (uint32_t c = c0; c < c1; ++c) {
          const uint32_t wi = c * 32u + lane;
          if (wi < n_words) {
            out_bits[wi] = 0;
            if (out_valid) {
              uint32_t v = valid ? __ldg(valid + wi) : kFullMask;
              if (wi == n_words - 1u && (n & 31u)) v &= (1u << (n & 31u)) - 1u;
              out_valid[wi] = v;
            }
          }
        }
      }
      if (io.counts) {  // zeroed by the host before the launch
        survivors = warp_sum(survivors);
        uint32_t* cnt = io.counts + static_cast<size_t>(e) * io.counts_stride;
        if (lane == 0) {
          if (mode == MODE_REFINE) {
            if (survivors) atomicAdd(cnt, survivors);
          } else {
            if (grp == 0) {
              cnt[0] = n;
              cnt[1] = h0.null_count;
            }
            if (survivors) atomicAdd(cnt + 2, survivors);
          }
        }
      }
    }
    h0 = h1;
    blob0 = blob1;
    blob1 = blob2;
  }
}

// The host guarantees: every entry is an integer-shaped blob with tbits in {8,16,32,64}, bit_width <= 32, and the counts
// array (if any) is zeroed on the stream before this launch.
cudaError_t launch_int_bits(int mode, uint32_t n_entries, const ScanIo& io, const IntPredDesc& pred, uint32_t max_rows,
                            cudaStream_t s, const IntInList& in) {
  if (n_entries == 0) return cudaSuccess;
  static int n_sm = 0;
  if (!n_sm) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  }
  const uint32_t cpe = max_rows ? (max_rows + 1023u) / 1024u : 1u;
  // register budget: 3 CTAs per SM (80 registers) by default; LC_INT_OCC=4 selects the 64-register build (experiments)
  static const int occ_pref = [] {
    const char* e = std::getenv("LC_INT_OCC");
    return (e && e[0] == '4') ? 4 : 3;
  }();
  static int per_sm = 0;
  if (!per_sm) {
    cudaError_t e = occ_pref == 4 ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_int_bits<4, false>, 256, 0)
                                  : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_int_bits<3, false>, 256, 0);
    if (e != cudaSuccess) return e;
    if (per_sm < 1) per_sm = 1;
  }
  uint32_t grid = static_cast<uint32_t>(n_sm * per_sm);  // persistent: every resident warp loops over the tasks
  // A task is a group of eight chunks — a whole 8192-row batch: header read and predicate planned once per batch. Groups
  // of two spread the tasks more evenly over the resident warps but plan four times as often; LC_INT_GROUP=2 / 4 select
  // the smaller groups.
  static const uint32_t cshift_pref = [] {
    const char* e = std::getenv("LC_INT_GROUP");
    return (e && e[0] == '2') ? 1u : ((e && e[0] == '4') ? 2u : 3u);
  }();
  const uint32_t cshift = cshift_pref;
  uint32_t gshift = 0;
  while (((1u << cshift) << gshift) < cpe) ++gshift;
  const uint64_t n_tasks = static_cast<uint64_t>(n_entries) << gshift;
  if (n_tasks > 0x7fffffffull) return cudaErrorInvalidValue;
  const uint32_t need = static_cast<uint32_t>((n_tasks + 7u) / 8u);
  if (grid > need) grid = need;
  const bool set = pred.op == kOpIn || pred.op == kOpNotIn;
  if (set) {
    // IN lists: the default 80-register build only (LC_INT_OCC does not apply), which holds 8 KB more shared memory per
    // CTA: its own residency, the same persistent grid shape
    static int per_sm_set = 0;
    if (!per_sm_set) {
      cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_set, k_int_bits<3, true>, 256, 0);
      if (e != cudaSuccess) return e;
      if (per_sm_set < 1) per_sm_set = 1;
    }
    uint32_t grid_set = static_cast<uint32_t>(n_sm * per_sm_set);
    if (grid_set > need) grid_set = need;
    k_int_bits<3, true><<<grid_set, 256, 0, s>>>(io, pred, n_entries, gshift, cshift, mode, in);
  } else if (occ_pref == 4) {
    k_int_bits<4, false><<<grid, 256, 0, s>>>(io, pred, n_entries, gshift, cshift, mode, in);
  } else {
    k_int_bits<3, false><<<grid, 256, 0, s>>>(io, pred, n_entries, gshift, cshift, mode, in);
  }
  return cudaGetLastError();
}

}  // namespace lc

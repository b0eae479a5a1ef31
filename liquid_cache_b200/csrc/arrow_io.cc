// arrow_io.cc — Arrow C Data Interface import (borrowed) and export (caller-owned) helpers.
// Accepted input types = the dtype dispatch of transcode_liquid_inner_with_hint
// (/root/reference/src/core/src/cache/transcode.rs:46-290): integers, dates, timestamps, floats, decimals, byte views.
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <unordered_map>
#include <vector>

#include "host_common.h"

namespace lc {

// Result buffers. Small ones come from the C heap. From 1 MiB on they are PAGE-LOCKED blocks recycled through a
// process-wide pool: a device-to-host copy into pageable memory is staged by the driver (a multi-MB result such as the
// 43 MB one of the l_shipdate scan then costs more than the scan), while a pinned destination takes the DMA directly.
// Page-locking is itself slow, hence the pool: the
// Arrow release callback hands the block back (no CUDA call), and the next result of that size class reuses it.
// The pool outlives every context on purpose — an exported array may be released after its lc_ctx is gone.
namespace {
struct PinnedPool {
  std::mutex mu;
  std::unordered_map<uint8_t*, uint64_t> live;                 // handed-out block -> capacity
  std::unordered_map<uint64_t, std::vector<uint8_t*>> idle;    // capacity (power of two) -> blocks
  uint64_t idle_bytes = 0;
};
PinnedPool& pinned_pool() {
  static PinnedPool* p = new PinnedPool();  // never destroyed: release callbacks may run during interpreter shutdown
  return *p;
}
constexpr uint64_t kPinnedMin = 1ull << 20;
constexpr uint64_t kPinnedIdleMax = 8ull << 30;  // full-column string reads of the sweep are > 1 GiB each
}  // namespace

uint8_t* host_alloc(uint64_t bytes, bool force_pinned) {
  if (bytes >= kPinnedMin || force_pinned) {
    uint64_t cap = force_pinned ? 4096 : kPinnedMin;  // asynchronous downloads need a page-locked destination whatever its size
    while (cap < bytes) cap <<= 1;
    PinnedPool& pool = pinned_pool();
    {
      std::lock_guard<std::mutex> l(pool.mu);
      auto it = pool.idle.find(cap);
      if (it != pool.idle.end() && !it->second.empty()) {
        uint8_t* p = it->second.back();
        it->second.pop_back();
        pool.idle_bytes -= cap;
        pool.live.emplace(p, cap);
        return p;
      }
    }
    void* p = nullptr;
    if (cudaHostAlloc(&p, cap, cudaHostAllocDefault) == cudaSuccess) {
      std::lock_guard<std::mutex> l(pool.mu);
      pool.live.emplace(static_cast<uint8_t*>(p), cap);
      return static_cast<uint8_t*>(p);
    }
    cudaGetLastError();  // no page-locked memory to be had: fall through to the heap
  }
  void* p = nullptr;
  if (posix_memalign(&p, 64, bytes ? round_up(bytes, 64) : 64) != 0) return nullptr;
  return static_cast<uint8_t*>(p);
}

void host_free(uint8_t* p) {
  if (!p) return;
  PinnedPool& pool = pinned_pool();
  uint64_t cap = 0;
  {
    std::lock_guard<std::mutex> l(pool.mu);
    auto it = pool.live.find(p);
    if (it == pool.live.end()) {
      cap = 0;
    } else {
      cap = it->second;
      pool.live.erase(it);
      if (pool.idle_bytes + cap <= kPinnedIdleMax) {
        pool.idle[cap].push_back(p);
        pool.idle_bytes += cap;
        return;
      }
    }
  }
  if (cap) {
    if (cudaFreeHost(p) != cudaSuccess) cudaGetLastError();  // e.g. driver already shut down: the OS reclaims it
  } else {
    std::free(p);
  }
}

void copy_bits(const uint8_t* src, int64_t off, int64_t n, uint8_t* dst, uint64_t dst_bytes) {
  std::memset(dst, 0, dst_bytes);
  if (n <= 0) return;
  const int64_t nbytes = (n + 7) / 8;
  if ((off & 7) == 0) {
    std::memcpy(dst, src + (off >> 3), static_cast<size_t>(nbytes));
  } else {
    const uint8_t* s = src + (off >> 3);
    const int sh = static_cast<int>(off & 7);
    const int64_t src_bytes = (off + n + 7) / 8 - (off >> 3);
    for (int64_t i = 0; i < nbytes; ++i) {
      uint32_t lo = s[i];
      uint32_t hi = (i + 1 < src_bytes) ? s[i + 1] : 0;
      dst[i] = static_cast<uint8_t>((lo >> sh) | (hi << (8 - sh)));
    }
  }
  if (n & 7) dst[nbytes - 1] &= static_cast<uint8_t>((1u << (n & 7)) - 1u);
}

uint64_t popcount_bits(const uint8_t* bits, uint64_t n) {
  uint64_t cnt = 0;
  const uint64_t full = n / 64;
  for (uint64_t i = 0; i < full; ++i) {
    uint64_t w;
    std::memcpy(&w, bits + i * 8, 8);
    cnt += static_cast<uint64_t>(__builtin_popcountll(w));
  }
  for (uint64_t i = full * 64; i < n; ++i) cnt += (bits[i >> 3] >> (i & 7)) & 1u;
  return cnt;
}

static bool parse_int_format(const std::string& f, uint8_t* phys, uint8_t* tbits, bool* is_signed) {
  struct Row { const char* f; uint8_t phys, tbits; bool sg; };
  static const Row rows[] = {
      {"c", PT_I8, 8, true},      {"s", PT_I16, 16, true},     {"i", PT_I32, 32, true},   {"l", PT_I64, 64, true},
      {"C", PT_U8, 8, false},     {"S", PT_U16, 16, false},    {"I", PT_U32, 32, false},  {"L", PT_U64, 64, false},
      {"tdD", PT_DATE32, 32, true}, {"tdm", PT_DATE64, 64, true},
      {"tss:", PT_TS_S, 64, true},  {"tsm:", PT_TS_MS, 64, true}, {"tsu:", PT_TS_US, 64, true}, {"tsn:", PT_TS_NS, 64, true},
  };
  for (const Row& r : rows) {
    if (f == r.f) {
      *phys = r.phys; *tbits = r.tbits; *is_signed = r.sg;
      return true;
    }
  }
  return false;
}

int parse_arrow_input(const ArrowSchema* schema, const ArrowArray* array, ArrowIn* out) {
  if (!schema || !array || !schema->format) {
    set_error("null schema/array");
    return LC_ERR_INVALID;
  }
  const std::string f = schema->format;
  out->format = f;
  out->length = array->length;
  out->offset = array->offset;
  out->null_count = array->null_count;
  if (array->length < 0 || array->length > 0x7fffffffLL) {
    set_error("array length %lld not supported", (long long)array->length);
    return LC_ERR_UNSUPPORTED_TYPE;
  }
  const uint8_t* validity = array->n_buffers > 0 ? static_cast<const uint8_t*>(array->buffers[0]) : nullptr;
  out->validity = validity;
  if (out->null_count < 0) {
    out->null_count =
        validity ? array->length - static_cast<int64_t>([&] {
          uint64_t c = 0;
          for (int64_t i = 0; i < array->length; ++i) c += bit_get(validity, array->offset + i);
          return c;
        }())
                 : 0;
  }
  if (!validity) out->null_count = 0;

  if (schema->dictionary) {
    // Dictionary<UInt16, Utf8|Binary> only (transcode.rs:259-283)
    const std::string vf = schema->dictionary->format ? schema->dictionary->format : "";
    if (f != "S" || (vf != "u" && vf != "z") || !array->dictionary) {
      set_error("unsupported dictionary type (index %s, value %s)", f.c_str(), vf.c_str());
      return LC_ERR_UNSUPPORTED_TYPE;
    }
    out->kind = ArrowIn::K_DICT;
    out->byte_type = (vf == "u") ? BT_DICT16_UTF8 : BT_DICT16_BINARY;
    out->dict_value_format = vf;
    out->dict_keys = static_cast<const uint16_t*>(array->buffers[1]);
    const ArrowArray* d = array->dictionary;
    out->dict_len = d->length;
    out->dict_offset = d->offset;
    out->dict_validity = d->n_buffers > 0 ? static_cast<const uint8_t*>(d->buffers[0]) : nullptr;
    out->dict_offsets = static_cast<const int32_t*>(d->buffers[1]);
    out->dict_data = static_cast<const uint8_t*>(d->buffers[2]);
    return LC_OK;
  }
  if (parse_int_format(f, &out->phys, &out->tbits, &out->is_signed)) {
    out->kind = ArrowIn::K_INT;
    out->values = array->buffers[1];
    return LC_OK;
  }
  if (f == "f" || f == "g") {  // Float32 / Float64 -> ALP (transcode.rs:107-112)
    out->kind = ArrowIn::K_FLOAT;
    out->phys = f == "f" ? PT_F32 : PT_F64;
    out->tbits = f == "f" ? 32 : 64;
    out->is_signed = true;
    out->values = array->buffers[1];
    return LC_OK;
  }
  if (f.size() > 2 && f[0] == 'd' && f[1] == ':') {  // "d:precision,scale[,bitwidth]" (transcode.rs:113-154)
    int precision = 0, scale = 0, bw = 128;
    const int got = std::sscanf(f.c_str(), "d:%d,%d,%d", &precision, &scale, &bw);
    if (got >= 2 && (bw == 128 || bw == 256)) {
      out->kind = ArrowIn::K_DECIMAL;
      out->phys = PT_U64;
      out->tbits = 64;
      out->is_signed = false;
      out->dec_width = static_cast<uint32_t>(bw / 8);
      out->values = array->buffers[1];
      return LC_OK;
    }
  }
  if (f == "u" || f == "z") {
    out->kind = ArrowIn::K_BYTES;
    out->byte_type = (f == "u") ? BT_UTF8 : BT_BINARY;
    out->values = array->buffers[1];
    out->data = static_cast<const uint8_t*>(array->buffers[2]);
    return LC_OK;
  }
  if (f == "vu" || f == "vz") {
    out->kind = ArrowIn::K_VIEW;
    out->byte_type = (f == "vu") ? BT_UTF8_VIEW : BT_BINARY_VIEW;
    out->values = array->buffers[1];  // 16-byte views
    // buffers: [validity, views, data_0 .. data_{k-1}, variadic_sizes]
    out->n_view_buffers = array->n_buffers - 3;
    out->view_buffers = array->buffers + 2;
    return LC_OK;
  }
  // Boolean, Decimal32/64, tz-timestamps, large types, nested ...
  set_error("unsupported arrow type '%s'", f.c_str());
  return LC_ERR_UNSUPPORTED_TYPE;
}

// ---- export ------------------------------------------------------------------------------------
struct SchemaPriv {
  std::string format;
  ArrowSchema dict;
  ArrowSchema* dict_ptr;
  std::string dict_format;
};

static void release_schema(ArrowSchema* s) {
  if (!s || !s->release) return;
  SchemaPriv* p = static_cast<SchemaPriv*>(s->private_data);
  if (s->dictionary && s->dictionary->release) s->dictionary->release(s->dictionary);
  delete p;
  s->release = nullptr;
}

static void release_dict_schema(ArrowSchema* s) {
  if (s) s->release = nullptr;  // storage lives in the parent's SchemaPriv
}

void export_schema(const std::string& format, const std::string& dict_value_format, ArrowSchema* out) {
  SchemaPriv* p = new SchemaPriv();
  p->format = format;
  p->dict_format = dict_value_format;
  std::memset(out, 0, sizeof(*out));
  out->format = p->format.c_str();
  out->name = "";
  out->metadata = nullptr;
  out->flags = ARROW_FLAG_NULLABLE;
  out->n_children = 0;
  out->children = nullptr;
  out->dictionary = nullptr;
  if (!dict_value_format.empty()) {
    std::memset(&p->dict, 0, sizeof(p->dict));
    p->dict.format = p->dict_format.c_str();
    p->dict.name = "";
    p->dict.flags = ARROW_FLAG_NULLABLE;
    p->dict.release = release_dict_schema;
    out->dictionary = &p->dict;
  }
  out->release = release_schema;
  out->private_data = p;
}

struct ArrayPriv {
  std::vector<HostBuf> bufs;
  std::vector<const void*> ptrs;
  ArrowArray dict;
  bool has_dict = false;
};

static void release_array(ArrowArray* a) {
  if (!a || !a->release) return;
  ArrayPriv* p = static_cast<ArrayPriv*>(a->private_data);
  if (p->has_dict && p->dict.release) p->dict.release(&p->dict);
  for (auto& b : p->bufs)
    if (b.p) host_free(b.p);
  delete p;
  a->release = nullptr;
}

void export_array(int64_t length, int64_t null_count, std::vector<HostBuf> buffers, ArrowArray* dictionary,
                  ArrowArray* out) {
  ArrayPriv* p = new ArrayPriv();
  p->bufs = std::move(buffers);
  for (auto& b : p->bufs) p->ptrs.push_back(b.p);
  std::memset(out, 0, sizeof(*out));
  out->length = length;
  out->null_count = null_count;
  out->offset = 0;
  out->n_buffers = static_cast<int64_t>(p->ptrs.size());
  out->buffers = p->ptrs.data();
  out->n_children = 0;
  out->children = nullptr;
  out->dictionary = nullptr;
  if (dictionary) {
    p->dict = *dictionary;  // move
    dictionary->release = nullptr;
    p->has_dict = true;
    out->dictionary = &p->dict;
  }
  out->release = release_array;
  out->private_data = p;
}

}  // namespace lc

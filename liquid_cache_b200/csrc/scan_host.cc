// scan_host.cc — batched get / eval_predicate over lists of HBM-resident entries.
// Host side does planning (per-entry predicate constants, output offsets) and exactly one H2D of the
// work list + selections and one D2H of the results per call; all per-row work is in the kernels.
// Reference call sites: LiquidCache::read_arrow_array / eval_predicate_internal
// (/root/reference/src/core/src/cache/core.rs:595-634, 862-930).
#include <algorithm>
#include <cstring>
#include <atomic>
#include <chrono>
#include <mutex>
#include <cstdlib>

#include "host_common.h"
#include "host_pool.h"

namespace lc {

namespace {

// per-entry selection bookkeeping shared by every batched call
struct SelPlan {
  std::vector<const uint8_t*> bits;  // nullptr = dense
  std::vector<uint32_t> k;           // selected rows
  std::vector<uint64_t> word_off;    // offset (in u32 words) of the entry's selection in the upload area
  uint64_t sel_words = 0;
  uint64_t total_k = 0;
  bool sparse = false;        // the staged words are nearly all zero: only {word index, word} pairs are uploaded
  uint64_t sparse_pairs = 0;
};

// Host selections: every bitmap is copied ONCE into the context's pinned staging area (word aligned, tail bits
// cleared, zero padded) and counted on the way, split over the host pool — the bitmaps usually come straight out of
// a device-to-host copy, so this walk is DRAM bound on one core. The staged words go to the device with one copy
// (upload_selection). A selection that turns out to be all ones is treated as dense.
int plan_selection(lc_ctx* ctx, const uint32_t* entry_rows, uint64_t n, const uint8_t* const* sel_bits, SelPlan* p,
                   const DevSel* dev = nullptr) {
  p->bits.assign(n, nullptr);
  p->k.assign(n, 0);
  p->word_off.assign(n, 0);
  if (dev) {  // selections are already on the device; only the counts matter here
    for (uint64_t i = 0; i < n; ++i) {
      p->k[i] = dev->all_rows ? entry_rows[i] : dev->k[i];
      p->total_k += p->k[i];
    }
    return LC_OK;
  }
  if (!sel_bits) {
    for (uint64_t i = 0; i < n; ++i) {
      p->k[i] = entry_rows[i];
      p->total_k += p->k[i];
    }
    return LC_OK;
  }
  for (uint64_t i = 0; i < n; ++i) {
    p->bits[i] = sel_bits[i];
    if (sel_bits[i]) {
      p->word_off[i] = p->sel_words;
      p->sel_words += round_up((entry_rows[i] + 31) / 32, 4);
    }
  }
  const uint64_t need = p->sel_words * 4 + 64 + (p->sel_words / 16) * 8 + 128;  // dense words + room for sparse pairs
  if (need > ctx->L()->sel_stage_cap) {
    if (ctx->L()->sel_stage) cudaFreeHost(ctx->L()->sel_stage);
    ctx->L()->sel_stage = nullptr;
    ctx->L()->sel_stage_cap = 0;
    uint64_t cap = 1ull << 20;
    while (cap < need) cap *= 2;
    if (cudaHostAlloc(reinterpret_cast<void**>(&ctx->L()->sel_stage), cap, cudaHostAllocDefault) != cudaSuccess) {
      cudaGetLastError();
      set_error("selection staging: cudaHostAlloc of %llu bytes failed", (unsigned long long)cap);
      return LC_ERR_OOM;
    }
    ctx->L()->sel_stage_cap = cap;
  }
  uint8_t* stage = ctx->L()->sel_stage;
  // While staging, every range of entries also notes its non-zero words. Selections that come out of a selective
  // predicate are nearly all zero (config 2: ~1.6 set bits per 8192-bit bitmap), and then only the {word index, word}
  // pairs cross PCIe (a few KB instead of MBs); the device zero-fills the area and scatters them.
  std::mutex pairs_mu;
  std::vector<uint64_t> pairs;  // (word index << 32) | word
  const uint64_t pair_budget = p->sel_words / 16;  // beyond this the dense copy is as cheap
  std::atomic<bool> too_many{false};
  parallel_for(n, 64, [&](uint64_t b, uint64_t e) {
    std::vector<uint64_t> local;
    for (uint64_t i = b; i < e; ++i) {
      const uint32_t rows = entry_rows[i];
      if (!p->bits[i]) {
        p->k[i] = rows;
        continue;
      }
      const uint64_t words = round_up((rows + 31) / 32, 4);
      uint8_t* dst = stage + p->word_off[i] * 4;
      copy_bits(p->bits[i], 0, rows, dst, words * 4);
      const uint32_t* w32 = reinterpret_cast<const uint32_t*>(dst);
      uint32_t k = 0;
      const bool note = !too_many.load(std::memory_order_relaxed);
      // `words` is a multiple of four and the staging area is 16-byte aligned per entry: look at 64 bytes at a time and
      // go word by word only where something is set (a selection behind a selective predicate is nearly all zero)
      uint64_t w = 0;
      for (; w + 16 <= words; w += 16) {
        const uint64_t* q = reinterpret_cast<const uint64_t*>(w32 + w);
        if ((q[0] | q[1] | q[2] | q[3] | q[4] | q[5] | q[6] | q[7]) == 0) continue;
        for (uint64_t t = w; t < w + 16; ++t) {
          const uint32_t v = w32[t];
          if (v == 0) continue;
          k += static_cast<uint32_t>(__builtin_popcount(v));
          if (note) local.push_back(((p->word_off[i] + t) << 32) | v);
        }
      }
      for (; w < words; ++w) {
        const uint32_t v = w32[w];  // padding is zero
        if (v == 0) continue;
        k += static_cast<uint32_t>(__builtin_popcount(v));
        if (note) local.push_back(((p->word_off[i] + w) << 32) | v);
      }
      if (local.size() > pair_budget) too_many.store(true, std::memory_order_relaxed);
      p->k[i] = k;
      if (k == rows) p->bits[i] = nullptr;  // dense after all: the kernels take their no-selection path
    }
    if (!local.empty() && !too_many.load(std::memory_order_relaxed)) {
      std::lock_guard<std::mutex> l(pairs_mu);
      pairs.insert(pairs.end(), local.begin(), local.end());
    }
  });
  for (uint64_t i = 0; i < n; ++i) p->total_k += p->k[i];
  if (!too_many.load() && pairs.size() <= pair_budget && p->sel_words >= 4096) {
    // park the pairs behind the dense words in the pinned staging area
    const uint64_t off = round_up(p->sel_words * 4, 64);
    if (off + pairs.size() * 8 + 64 <= ctx->L()->sel_stage_cap) {
      if (!pairs.empty()) std::memcpy(stage + off, pairs.data(), pairs.size() * 8);
      p->sparse = true;
      p->sparse_pairs = pairs.size();
    }
  }
  return LC_OK;
}

// One host-to-device copy of everything plan_selection staged.
int upload_selection(lc_ctx* ctx, const SelPlan& p, uint8_t* d_sel, cudaStream_t s) {
  if (p.sel_words == 0) return LC_OK;
  if (p.sparse) {
    const uint64_t bytes = p.sparse_pairs * 8;
    if (bytes > ctx->L()->d_pairs_cap) {
      if (ctx->L()->d_pairs) cudaFree(ctx->L()->d_pairs);
      ctx->L()->d_pairs = nullptr;
      ctx->L()->d_pairs_cap = 0;
      uint64_t cap = 1ull << 16;
      while (cap < bytes) cap *= 2;
      if (cudaMalloc(reinterpret_cast<void**>(&ctx->L()->d_pairs), cap) != cudaSuccess) {
        cudaGetLastError();
        set_error("cudaMalloc of %llu bytes for sparse selections failed", (unsigned long long)cap);
        return LC_ERR_OOM;
      }
      ctx->L()->d_pairs_cap = cap;
    }
    LC_CUDA_OK(cudaMemsetAsync(d_sel, 0, p.sel_words * 4, s));
    if (bytes == 0) return LC_OK;
    LC_CUDA_OK(cudaMemcpyAsync(ctx->L()->d_pairs, ctx->L()->sel_stage + round_up(p.sel_words * 4, 64), bytes, cudaMemcpyHostToDevice, s));
    LC_CUDA_OK(launch_scatter_words(reinterpret_cast<const unsigned long long*>(ctx->L()->d_pairs), p.sparse_pairs,
                                    reinterpret_cast<uint32_t*>(d_sel), s));
    ctx->kernel_launches++;
    ctx->h2d_bytes += bytes;
    return LC_OK;
  }
  LC_CUDA_OK(cudaMemcpyAsync(d_sel, ctx->L()->sel_stage, p.sel_words * 4, cudaMemcpyHostToDevice, s));
  ctx->h2d_bytes += p.sel_words * 4;
  return LC_OK;
}

// KMP failure links of the LIKE needle
void kmp_fail(const uint8_t* nd, uint32_t m, uint16_t* fail) {
  if (!m) return;
  fail[0] = 0;
  uint32_t q = 0;
  for (uint32_t i = 1; i < m; ++i) {
    while (q > 0 && nd[q] != nd[i]) q = fail[q - 1];
    if (nd[q] == nd[i]) ++q;
    fail[i] = static_cast<uint16_t>(q);
  }
}

}  // namespace

// substring_pattern_bytes (byte_view_array/fingerprint.rs:59-73): '%x%' with x non-empty, no % or _.
// A backslash would make arrow's LIKE take the escape-aware regex path, so it is declined as well.
static int like_inner(const uint8_t* pat, uint64_t len, const uint8_t** inner, uint32_t* inner_len) {
  if (len < 3 || pat[0] != '%' || pat[len - 1] != '%') {
    set_error("LIKE pattern is not of the form %%x%%");
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  for (uint64_t i = 1; i + 1 < len; ++i) {
    if (pat[i] == '%' || pat[i] == '_' || pat[i] == '\\') {
      set_error("LIKE pattern has wildcards or escapes inside");
      return LC_ERR_UNSUPPORTED_EXPR;
    }
  }
  *inner = pat + 1;
  *inner_len = static_cast<uint32_t>(len - 2);
  return LC_OK;
}

// `decimal_col <op> literal` on LiquidFixedLenByteArray entries. The reference has no predicate for this type (the
// LiquidArray default decodes, filters and lets DataFusion compare, liquid_array/mod.rs:116-130); here the values are stored
// in order-preserving byte form (k_bits.cu k_fixed_to_ordered), so the comparison IS the byte-view comparison
// (comparisons.rs:21-151 semantics: equality on prefix keys + compressed bytes, ordering byte-wise) against the literal
// in the same form. The literal arrives as LC_LIT_I128 at the column's scale; a Decimal256 column sign-extends it.
struct FixedNeedle {
  lc_predicate pred{};
  uint8_t bytes[32];
};
static int lower_fixed_pred(Entry* const* entries, uint64_t n, const lc_predicate* pred, FixedNeedle* out) {
  const uint32_t w = entries[0]->fixed_width;
  for (uint64_t i = 0; i < n; ++i)
    if (entries[i]->fixed_width != w || entries[i]->arrow_format != entries[0]->arrow_format) {
      set_error("eval_predicate_many: fixed-length decimal entries of different types (or mixed with other entries) in one call");
      return LC_ERR_INVALID;
    }
  if (pred->op < LC_OP_EQ || pred->op > LC_OP_GE) {
    set_error("operator %d is not supported on decimal columns", pred->op);
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  if (pred->lit_kind == LC_LIT_BYTES && pred->lit_len == w) {
    fixed_needle(0, 0, pred->lit_bytes, w, out->bytes);  // the literal as the column's own little-endian integer
  } else if (pred->lit_kind == LC_LIT_I128) {
    fixed_needle(pred->lit_u64, pred->lit_i64, nullptr, w, out->bytes);
  } else {
    set_error("decimal column needs an LC_LIT_I128 literal (or its little-endian bytes)");
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  out->pred = *pred;
  out->pred.lit_kind = LC_LIT_BYTES;
  out->pred.lit_bytes = out->bytes;
  out->pred.lit_len = w;
  return LC_OK;
}

// Everything a predicate launch over byte-view entries needs, built on the host.
struct StrLaunch {
  StrPredDesc desc;
  std::vector<uint8_t> needle_blob;  // needle padded to 4 + KMP links
  const uint8_t* needle = nullptr;   // bytes the per-entry planning compares against
  uint32_t m = 0;
};

static bool is_in_list(const lc_predicate* pred) { return pred->op == LC_OP_IN || pred->op == LC_OP_NOT_IN; }

// `col [NOT] IN (list)` on byte-view entries: the list checked (Arrow Utf8 layout), sorted and deduplicated, and laid out
// again the same way — int32 offsets[k + 1], then the bytes — as the buffer k_str_scan plans its needles from.
static int prepare_str_in_list(const lc_predicate* pred, StrLaunch* L) {
  if (pred->lit_kind != LC_LIT_BYTES) {
    set_error("IN list on a byte-view column needs LC_LIT_BYTES values");
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  const uint64_t n = pred->lit_len;
  if (n > kInListMaxValues) {
    set_error("IN list of %llu values: at most %u run on the device", (unsigned long long)n, kInListMaxValues);
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  if (!pred->lit_bytes) {
    set_error("IN list without its offsets");
    return LC_ERR_INVALID;
  }
  std::vector<int32_t> off(n + 1);
  std::memcpy(off.data(), pred->lit_bytes, (n + 1) * 4);
  if (off[0] != 0) {
    set_error("IN list: offsets[0] is %d, not 0", off[0]);
    return LC_ERR_INVALID;
  }
  for (uint64_t i = 0; i < n; ++i)
    if (off[i + 1] < off[i]) {
      set_error("IN list: offsets decrease at value %llu", (unsigned long long)i);
      return LC_ERR_INVALID;
    }
  if (static_cast<uint64_t>(off[n]) > kInListMaxBytes) {
    set_error("IN list of %d value bytes: at most %u run on the device", off[n], kInListMaxBytes);
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  const char* bytes = reinterpret_cast<const char*>(pred->lit_bytes) + (n + 1) * 4;
  std::vector<std::string> vals;
  vals.reserve(n);
  for (uint64_t i = 0; i < n; ++i) vals.emplace_back(bytes + off[i], static_cast<size_t>(off[i + 1] - off[i]));
  std::sort(vals.begin(), vals.end());
  vals.erase(std::unique(vals.begin(), vals.end()), vals.end());
  const uint32_t k = static_cast<uint32_t>(vals.size());
  L->needle_blob.assign(4u * (k + 1u), 0);
  int32_t o = 0;
  for (uint32_t i = 0; i <= k; ++i) {
    std::memcpy(L->needle_blob.data() + 4u * i, &o, 4);
    if (i < k) o += static_cast<int32_t>(vals[i].size());
  }
  for (const std::string& v : vals) L->needle_blob.insert(L->needle_blob.end(), v.begin(), v.end());
  L->needle_blob.resize((L->needle_blob.size() + 3u) & ~size_t(3), 0);
  L->desc.list_n = k;
  L->desc.needle_len = 0;
  L->needle = nullptr;
  L->m = 0;
  return LC_OK;
}

static int prepare_str_pred(const lc_predicate* pred, StrLaunch* L) {
  std::memset(&L->desc, 0, sizeof(L->desc));
  L->desc.op = pred->op;
  const int op = pred->op;
  if (op == LC_OP_CONST_TRUE || op == LC_OP_CONST_FALSE) return LC_OK;
  if (is_in_list(pred)) return prepare_str_in_list(pred, L);
  if (pred->lit_kind != LC_LIT_BYTES || (!pred->lit_bytes && pred->lit_len)) {
    set_error("byte-view column needs a bytes literal");
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  const uint8_t* nd = pred->lit_bytes;
  uint64_t m = pred->lit_len;
  if (op == LC_OP_LIKE || op == LC_OP_NOT_LIKE) {
    uint32_t il;
    LC_TRY(like_inner(pred->lit_bytes, pred->lit_len, &nd, &il));
    m = il;
    uint32_t fp = 0;
    for (uint32_t i = 0; i < il; ++i) {
      fp |= 1u << (nd[i] & 31u);
      if (i + 2 < il) {
        const uint32_t t = trigram_bit(nd[i], nd[i + 1], nd[i + 2]);
        L->desc.needle_bloom[t >> 6] |= 1ull << (t & 63u);
      }
    }
    L->desc.needle_fp = fp;
    // the same bits as a list of filter planes; a long needle keeps its first 32 (any subset is a necessary condition)
    L->desc.n_planes = 0;
    for (uint32_t t = 0; t < kBloomPlanes && L->desc.n_planes < 32u; ++t)
      if ((L->desc.needle_bloom[t >> 6] >> (t & 63u)) & 1ull) L->desc.planes[L->desc.n_planes++] = static_cast<uint8_t>(t);
  }
  if (m > kMaxNeedle) {
    set_error("needle longer than %u bytes", kMaxNeedle);
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  L->needle = nd;
  L->m = static_cast<uint32_t>(m);
  L->desc.needle_len = L->m;
  const uint32_t padded = (L->m + 3u) & ~3u;
  L->needle_blob.assign(padded + 2u * L->m + 16u, 0);
  if (L->m) std::memcpy(L->needle_blob.data(), nd, L->m);
  if (op == LC_OP_LIKE || op == LC_OP_NOT_LIKE)
    kmp_fail(nd, L->m, reinterpret_cast<uint16_t*>(L->needle_blob.data() + padded));
  return LC_OK;
}

// ---- entry reference lists -----------------------------------------------------------------------
// The device-side list of {blob, sizes} for a handle list is cached per context (keyed by a hash of the handle
// array) so that repeated scans over the same column chunk upload nothing but a few scalars.
struct RefList {
  uint64_t key = 0;
  uint64_t n = 0;
  EntryRef* d_refs = nullptr;
  uint32_t* d_n_unique = nullptr;  // byte views: dictionary size per entry, behind d_refs in the same allocation
  // byte views: the distinct FSST symbol tables of the list, each entry's index into them, and room for one LIKE step table
  // (8 KB) per symbol table — k_like_steps fills it for the needle of a launch (same allocation as d_refs)
  uint64_t* d_tables = nullptr;
  uint32_t* d_entry_table = nullptr;
  uint8_t* d_like_steps = nullptr;
  uint32_t n_tables = 0;
  uint32_t max_blob = 0, max_head = 0, max_head_like = 0, max_unique = 1, max_meta = 0;  // max_meta: header .. offset residuals
  uint32_t max_rows = 0;
  bool int_bits_ok = true;  // integer lists: every entry has fields of at most 32 bits (k_int_bits covers the list)
  uint64_t epoch = 0;
  uint64_t last_use = 0;
  // host-side facts about the list, gathered once when it is built so that the per-call loops walk plain arrays
  // instead of chasing 10^4 Entry pointers (each a cache miss)
  std::shared_ptr<std::vector<uint32_t>> rows;      // rows per entry
  std::shared_ptr<std::vector<uint32_t>> n_unique;  // dictionary size per entry (byte views)
  std::shared_ptr<std::vector<const Entry*>> entries;  // the list itself: the key only pre-filters, the match is exact
  bool same_liquid_type = true, same_arrow_type = true, same_width = true, any_nulls = false, any_fixed = false;
  // did the last predicate over this list produce nearly-empty masks? (0 unknown, 1 sparse, 2 dense) — picks between
  // the sparse mask download and the chunked dense one before the answer is known
  mutable int mask_hint = 0;
  mutable uint64_t pairs_hint = 4096;  // non-zero mask words of the last sparse download over this list
  // the needle whose Shift-And step tables d_like_steps holds (and the stream that wrote them): the same LIKE over the same
  // list — the next query of a session, the next step of a bench — launches no k_like_steps
  mutable std::string steps_needle;
  mutable cudaStream_t steps_stream = nullptr;
};

struct RefCache {
  std::vector<RefList> lists;
  uint64_t tick = 0;
};

// The cache hangs off the context (opaque pointer in lc_ctx) and is only touched under the context's lock, so
// contexts used from different threads never share state.
static RefCache& ref_cache_of(lc_ctx* ctx) {
  if (!ctx->L()->ref_cache) ctx->L()->ref_cache = new RefCache();
  return *static_cast<RefCache*>(ctx->L()->ref_cache);
}

void drop_ref_cache(lc_ctx* ctx) {
  if (!ctx->L()->ref_cache) return;
  RefCache* rc = static_cast<RefCache*>(ctx->L()->ref_cache);
  for (auto& l : rc->lists)
    if (l.d_refs) cudaFree(l.d_refs);
  delete rc;
  ctx->L()->ref_cache = nullptr;
}

static int get_ref_list(lc_ctx* ctx, Entry* const* entries, uint64_t n, const RefList** out) {
  static_assert(sizeof(Entry*) == sizeof(uint64_t), "entry lists hash as 64-bit words");
  RefCache& rc = ref_cache_of(ctx);
  rc.tick++;
  // The list the validation cache handed this call (lc_lane::tok_*) is immutable while it lives: if it is the one whose
  // hash was computed last time — same address, length and generation, nothing created or dropped since — the key is
  // known and the contents need no second look (two passes over 100 KB per call of a 12 k-entry column otherwise).
  lc_lane* L = ctx->L();
  const uint64_t gen = g_validated_gen.load(std::memory_order_acquire);
  const bool tokened = n >= 64 && entries == L->tok_ptr && n == L->tok_n && L->tok_gen == gen;
  if (tokened && L->fast_ptr == entries && L->fast_n == n && L->fast_gen == gen && L->fast_epoch == ctx->epoch) {
    for (auto& l : rc.lists) {
      if (l.key == L->fast_key && l.n == n && l.epoch == ctx->epoch) {
        l.last_use = rc.tick;
        *out = &l;
        return LC_OK;
      }
    }
  }
  const uint64_t h = hash_words(reinterpret_cast<const uint64_t*>(entries), n);
  if (tokened) {
    L->fast_ptr = entries;
    L->fast_n = n;
    L->fast_gen = gen;
    L->fast_key = h;
    L->fast_epoch = ctx->epoch;
  }
  for (auto& l : rc.lists) {
    if (l.key == h && l.n == n && l.epoch == ctx->epoch && std::memcmp(l.entries->data(), entries, n * sizeof(Entry*)) == 0) {
      l.last_use = rc.tick;
      *out = &l;
      return LC_OK;
    }
  }
  // build + upload
  std::vector<EntryRef> refs(n);
  RefList nl;
  nl.key = h;
  nl.n = n;
  nl.epoch = ctx->epoch;
  nl.last_use = rc.tick;
  nl.rows = std::make_shared<std::vector<uint32_t>>(n);
  nl.n_unique = std::make_shared<std::vector<uint32_t>>(n, 0);
  nl.entries = std::make_shared<std::vector<const Entry*>>(entries, entries + n);
  const Entry* proto = entries[0];
  for (uint64_t i = 0; i < n; ++i) {
    const Entry* e = entries[i];
    if (e->squeeze_kind && !ctx->L()->squeeze_internal) {
      set_error("entry %llu of the list is squeezed: squeezed entries answer through lc_to_arrow / lc_eval_predicate", (unsigned long long)i);
      return LC_ERR_INVALID;
    }
    (*nl.rows)[i] = e->n;
    nl.max_rows = std::max(nl.max_rows, e->n);
    if (!is_int_blob(e->liquid_type) || e->ih.bit_width > 32) nl.int_bits_ok = false;
    nl.any_fixed = nl.any_fixed || e->fixed_width != 0;
    if (e->liquid_type != proto->liquid_type) nl.same_liquid_type = false;
    if (e->arrow_format != proto->arrow_format || e->dict_value_format != proto->dict_value_format) nl.same_arrow_type = false;
    if (is_int_blob(e->liquid_type)) {
      if (is_int_blob(proto->liquid_type) && e->ih.tbits != proto->ih.tbits) nl.same_width = false;
      nl.any_nulls = nl.any_nulls || e->ih.null_count != 0;
    } else {
      (*nl.n_unique)[i] = e->sh.n_unique;
      nl.any_nulls = nl.any_nulls || e->sh.null_count != 0;
    }
    refs[i].blob = e->d_blob;
    refs[i].blob_bytes = e->blob_bytes;
    refs[i].rows = e->n;
    if (is_int_blob(e->liquid_type)) {
      refs[i].head_bytes = e->blob_bytes;
      refs[i].sp_end = refs[i].pk_off = refs[i].rows_off = e->blob_bytes;
    } else {
      refs[i].head_bytes = e->sh.head_bytes;
      refs[i].sp_end = e->sh.sp_end;
      refs[i].pk_off = e->sh.prefix_keys_off;
      refs[i].rows_off = e->sh.rows_off;
      nl.max_head = std::max(nl.max_head, e->sh.head_bytes);
      nl.max_head_like = std::max(nl.max_head_like, e->sh.head_bytes - (e->sh.rows_off - e->sh.prefix_keys_off));
      nl.max_unique = std::max(nl.max_unique, e->sh.n_unique);
      nl.max_meta = std::max(nl.max_meta, e->sh.prefix_keys_off);
    }
    nl.max_blob = std::max(nl.max_blob, e->blob_bytes);
  }
  // distinct symbol tables (entries of one column chunk share theirs)
  std::vector<uint64_t> tables;
  std::vector<uint32_t> entry_table(n, 0);
  if (!is_int_blob(proto->liquid_type)) {
    std::unordered_map<uint64_t, uint32_t> seen;
    for (uint64_t i = 0; i < n; ++i) {
      const uint64_t t = entries[i]->sh.table_ptr;
      auto it = seen.find(t);
      if (it == seen.end()) {
        it = seen.emplace(t, static_cast<uint32_t>(tables.size())).first;
        tables.push_back(t);
      }
      entry_table[i] = it->second;
    }
  }
  nl.n_tables = static_cast<uint32_t>(tables.size());
  const uint64_t o_nu = round_up(n * sizeof(EntryRef) + 64, 256), o_tab = o_nu + round_up(n * 4, 256);
  const uint64_t o_et = o_tab + round_up(tables.size() * 8 + 8, 256), o_steps = o_et + round_up(n * 4, 256);
  const uint64_t total = o_steps + tables.size() * 8192ull + 256;
  if (cudaMalloc(reinterpret_cast<void**>(&nl.d_refs), total) != cudaSuccess) {
    cudaGetLastError();
    set_error("cudaMalloc for the entry list failed");
    return LC_ERR_OOM;
  }
  uint8_t* base = reinterpret_cast<uint8_t*>(nl.d_refs);
  LC_CUDA_OK(cudaMemcpyAsync(nl.d_refs, refs.data(), n * sizeof(EntryRef), cudaMemcpyHostToDevice, ctx->L()->stream));
  nl.d_n_unique = reinterpret_cast<uint32_t*>(base + o_nu);
  LC_CUDA_OK(cudaMemcpyAsync(nl.d_n_unique, nl.n_unique->data(), n * 4, cudaMemcpyHostToDevice, ctx->L()->stream));
  nl.d_tables = reinterpret_cast<uint64_t*>(base + o_tab);
  nl.d_entry_table = reinterpret_cast<uint32_t*>(base + o_et);
  nl.d_like_steps = base + o_steps;
  if (!tables.empty()) {
    LC_CUDA_OK(cudaMemcpyAsync(nl.d_tables, tables.data(), tables.size() * 8, cudaMemcpyHostToDevice, ctx->L()->stream));
    LC_CUDA_OK(cudaMemcpyAsync(nl.d_entry_table, entry_table.data(), n * 4, cudaMemcpyHostToDevice, ctx->L()->stream));
  }
  LC_CUDA_OK(cudaStreamSynchronize(ctx->L()->stream));  // `refs` is pageable host memory
  ctx->h2d_bytes += n * sizeof(EntryRef);
  // evict: stale epochs first, then least recently used beyond 16 lists
  for (size_t i = 0; i < rc.lists.size();) {
    if (rc.lists[i].epoch != ctx->epoch) {
      cudaFree(rc.lists[i].d_refs);
      rc.lists.erase(rc.lists.begin() + i);
    } else {
      ++i;
    }
  }
  if (rc.lists.size() >= 16) {
    size_t lru = 0;
    for (size_t i = 1; i < rc.lists.size(); ++i)
      if (rc.lists[i].last_use < rc.lists[lru].last_use) lru = i;
    cudaFree(rc.lists[lru].d_refs);
    rc.lists.erase(rc.lists.begin() + lru);
  }
  rc.lists.push_back(nl);
  *out = &rc.lists.back();
  return LC_OK;
}

// `col [NOT] IN (list)` on integer / date / timestamp entries: the values in the column's domain, sorted in the column's
// order (signed or unsigned, the same for every entry of the list) without duplicates, as 8-byte words ready to upload.
// Values no entry can hold (negative on an unsigned column, above i64::MAX on a signed one) are dropped.
static int make_int_in_list(const lc_predicate* pred, Entry* const* entries, uint64_t n, IntPredDesc* out,
                            std::vector<uint8_t>* blob) {
  if (entries[0]->liquid_type != LC_LIQUID_INTEGER) {
    set_error("IN lists run on integer, date, timestamp and byte-view columns only");
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  if (pred->lit_kind != LC_LIT_I64 && pred->lit_kind != LC_LIT_U64) {
    set_error("IN list on an integer column needs LC_LIT_I64 or LC_LIT_U64 values");
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  if (pred->lit_len > kInListMaxValues) {
    set_error("IN list of %llu values: at most %u run on the device", (unsigned long long)pred->lit_len, kInListMaxValues);
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  if (pred->lit_len && !pred->lit_bytes) {
    set_error("IN list without its values");
    return LC_ERR_INVALID;
  }
  const bool is_signed = entries[0]->ih.is_signed != 0;
  for (uint64_t i = 1; i < n; ++i)
    if ((entries[i]->ih.is_signed != 0) != is_signed) {
      set_error("IN list over signed and unsigned integer entries in one call");
      return LC_ERR_INVALID;
    }
  std::vector<uint64_t> v;
  v.reserve(pred->lit_len);
  for (uint64_t i = 0; i < pred->lit_len; ++i) {
    uint64_t x;
    std::memcpy(&x, pred->lit_bytes + 8 * i, 8);
    const bool neg_i64 = pred->lit_kind == LC_LIT_I64 && static_cast<int64_t>(x) < 0;
    const bool big_u64 = pred->lit_kind == LC_LIT_U64 && x > 0x7fffffffffffffffull;
    if ((is_signed && big_u64) || (!is_signed && neg_i64)) continue;
    v.push_back(x);
  }
  if (is_signed)
    std::sort(v.begin(), v.end(), [](uint64_t a, uint64_t b) { return static_cast<int64_t>(a) < static_cast<int64_t>(b); });
  else
    std::sort(v.begin(), v.end());
  v.erase(std::unique(v.begin(), v.end()), v.end());
  blob->resize(v.size() * 8);
  if (!v.empty()) std::memcpy(blob->data(), v.data(), v.size() * 8);
  out->op = pred->op;
  out->lit_kind = is_signed ? LC_LIT_I64 : LC_LIT_U64;
  out->lit_i = 0;
  out->lit_u = 0;
  return LC_OK;
}

static int make_int_pred(const lc_predicate* pred, const Entry* proto, IntPredDesc* out) {
  if (pred->op < LC_OP_EQ || pred->op > LC_OP_GE) {
    set_error("operator %d is not supported on integer columns", pred->op);
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  out->op = pred->op;
  if (proto->liquid_type == LC_LIQUID_DECIMAL) {
    // Decimal128/256 compare as signed 128/256-bit integers; every stored value is in [0, u64::MAX], so a literal
    // outside that window folds to a constant on either side (the literal arrives with the column's scale)
    out->lit_i = 0;
    out->lit_u = 0;
    if (pred->lit_kind == LC_LIT_BYTES && (pred->lit_len == 16 || pred->lit_len == 32) && pred->lit_len == proto->dec_width) {
      // the literal as the column's own little-endian integer (Decimal256 literals beyond 128 bits travel like this)
      const uint8_t* b = pred->lit_bytes;
      const bool negative = (b[pred->lit_len - 1] & 0x80u) != 0;
      bool upper = false;
      for (uint64_t i = 8; i < pred->lit_len; ++i) upper = upper || b[i] != 0;
      if (negative) {
        out->lit_kind = LC_LIT_I64;
        out->lit_i = -1;
      } else if (upper) {
        out->lit_kind = kLitAboveAll;
      } else {
        out->lit_kind = LC_LIT_U64;
        std::memcpy(&out->lit_u, b, 8);
      }
      return LC_OK;
    }
    if (pred->lit_kind != LC_LIT_I128) {
      set_error("decimal column needs an LC_LIT_I128 literal (or its little-endian bytes)");
      return LC_ERR_UNSUPPORTED_EXPR;
    }
    if (pred->lit_i64 == 0) {
      out->lit_kind = LC_LIT_U64;
      out->lit_u = pred->lit_u64;
    } else if (pred->lit_i64 < 0) {
      out->lit_kind = LC_LIT_I64;
      out->lit_i = -1;
    } else {
      out->lit_kind = kLitAboveAll;
    }
    return LC_OK;
  }
  if (pred->lit_kind == kLitSentinelPublic) {  // squeeze_host.cc only: rows of a clamped entry at the sentinel
    out->op = LC_OP_EQ;
    out->lit_kind = kLitSentinel;
    out->lit_i = 0;
    out->lit_u = 0;
    return LC_OK;
  }
  if (pred->lit_kind != LC_LIT_I64 && pred->lit_kind != LC_LIT_U64) {
    set_error("integer column needs an integer literal");
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  out->lit_kind = pred->lit_kind;
  out->lit_i = pred->lit_i64;
  out->lit_u = pred->lit_u64;
  return LC_OK;
}

// `float_col <op> literal`: the literal's key in arrow-ord's total order, in the column's own float type
// (DataFusion has already coerced the literal to that type; alp_math.cuh order_key is the device twin).
static int make_float_pred(const lc_predicate* pred, uint32_t tbits, int32_t* op, long long* key) {
  if (pred->op < LC_OP_EQ || pred->op > LC_OP_GE) {
    set_error("operator %d is not supported on float columns", pred->op);
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  if (pred->lit_kind != LC_LIT_F64) {
    set_error("float column needs an LC_LIT_F64 literal");
    return LC_ERR_UNSUPPORTED_EXPR;
  }
  *op = pred->op;
  double d;
  std::memcpy(&d, &pred->lit_u64, 8);
  if (tbits == 64) {
    int64_t b;
    std::memcpy(&b, &d, 8);
    *key = b ^ static_cast<int64_t>(static_cast<uint64_t>(b >> 63) >> 1);
  } else {
    const float f = static_cast<float>(d);
    int32_t b;
    std::memcpy(&b, &f, 4);
    *key = b ^ static_cast<int32_t>(static_cast<uint32_t>(b >> 31) >> 1);
  }
  return LC_OK;
}

namespace {
struct Tracer {  // LC_TRACE=1: wall-clock split of a call, printed to stderr
  bool on;
  std::chrono::steady_clock::time_point t0;
  const char* what;
  explicit Tracer(const char* w) : on(std::getenv("LC_TRACE") != nullptr), t0(std::chrono::steady_clock::now()), what(w) {}
  void mark(const char* stage) {
    if (!on) return;
    auto t1 = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[lc_trace] %s: %s %.3f ms\n", what, stage, std::chrono::duration<double, std::milli>(t1 - t0).count());
    t0 = t1;
  }
};
}  // namespace


// ---- float columns: decode the selected rows, compare the decoded values ------------------------------
// The reference evaluates float predicates exactly this way (trait default: filter, then DataFusion's compare on
// the Arrow array, liquid_array/mod.rs:116-130); here the three steps are k_int_scan<DECODE> (unpack + compaction),
// k_alp_finish (ALP integers -> floats, patches) and k_float_cmp (total-order compare, nulls -> false).
static int eval_predicate_float(lc_ctx* ctx, Entry* const* entries, uint64_t n, const RefList* rl, const lc_predicate* pred,
                                const uint8_t* const* sel_bits, const PredOut& out) {
  const uint32_t tbits = entries[0]->ih.tbits, tb = tbits / 8;
  if (!rl->same_width) {
    set_error("eval_predicate_many: Float32 and Float64 entries in one call");
    return LC_ERR_INVALID;
  }
  int32_t op = 0;
  long long key = 0;
  LC_TRY(make_float_pred(pred, tbits, &op, &key));
  SelPlan sp;
  LC_TRY(plan_selection(ctx, rl->rows->data(), n, sel_bits, &sp));
  std::vector<uint64_t> row_base(n), word_off(n);
  uint64_t rows = 0, words = 0;
  for (uint64_t i = 0; i < n; ++i) {
    row_base[i] = rows;
    rows += sp.k[i];
    word_off[i] = words;
    words += round_up((sp.k[i] + 31) / 32, 4);
  }
  const uint64_t up_offs = round_up(n * 8 * 3, 256);
  const uint64_t up_sel = round_up(sp.sel_words * 4, 256);
  const uint64_t up_total = up_offs + up_sel;
  const uint64_t dn_counts = round_up(n * 16, 256);
  const uint64_t dn_bits = round_up(words * 4 + 16, 256);
  const uint64_t dn_total = dn_counts + 2 * dn_bits;
  const uint64_t val_bytes = round_up(rows * tb + 16, 256);
  Scratch& sc = ctx->L()->scratch;
  LC_TRY(sc.reserve(up_total + dn_total + val_bytes + 1024, up_total + dn_total + 1024));
  uint8_t* h_up = sc.host(up_total);
  uint8_t* h_dn = sc.host(dn_total);
  uint8_t* d_up = sc.dev(up_total);
  uint8_t* d_dn = sc.dev(dn_total);
  uint8_t* d_vals = sc.dev(val_bytes);
  if (!h_up || !h_dn || !d_up || !d_dn || !d_vals) {
    set_error("eval_predicate: scratch exhausted");
    return LC_ERR_OOM;
  }
  uint64_t* a = reinterpret_cast<uint64_t*>(h_up);
  for (uint64_t i = 0; i < n; ++i) {
    a[i] = sp.bits[i] ? sp.word_off[i] : kNoSel;
    a[n + i] = row_base[i];
    a[2 * n + i] = word_off[i];
  }
  cudaStream_t s = ctx->L()->stream;
  LC_CUDA_OK(cudaMemcpyAsync(d_up, h_up, up_offs, cudaMemcpyHostToDevice, s));
  ctx->h2d_bytes += up_offs;
  LC_TRY(upload_selection(ctx, sp, d_up + up_offs, s));
  const uint64_t* offs = reinterpret_cast<const uint64_t*>(d_up);
  ScanIo io{};
  io.refs = rl->d_refs;
  io.sel_base = sp.sel_words ? reinterpret_cast<const uint32_t*>(d_up + up_offs) : nullptr;
  io.sel_off = offs;
  io.out_base = d_vals;
  io.out_off = offs + n;
  io.valid_base = reinterpret_cast<uint32_t*>(d_dn + dn_counts + dn_bits);
  io.valid_off = offs + 2 * n;
  io.counts = reinterpret_cast<uint32_t*>(d_dn);
  io.counts_stride = 4;
  IntPredDesc ip{};
  if (ctx->L()->timing_on) cudaEventRecord(ctx->L()->ev_a, s);
  LC_CUDA_OK(launch_int_scan(MODE_DECODE, static_cast<uint32_t>(n), io, ip, rl->max_blob, s));
  LC_CUDA_OK(launch_alp_finish(static_cast<uint32_t>(n), io, tbits, s));
  FloatCmpIo c{};
  c.refs = rl->d_refs;
  c.vals_base = d_vals;
  c.vals_off = offs + n;
  c.vals_counts = io.counts;
  c.vals_stride = 4;
  c.refine = 0;
  c.and_base = io.valid_base;
  c.and_off = offs + 2 * n;
  c.out_base = reinterpret_cast<uint32_t*>(d_dn + dn_counts);
  c.out_off = offs + 2 * n;
  c.counts = io.counts;
  c.counts_stride = 4;
  c.op = op;
  c.lit_key = key;
  LC_CUDA_OK(launch_float_cmp(static_cast<uint32_t>(n), c, tbits, s));
  if (ctx->L()->timing_on) {
    cudaEventRecord(ctx->L()->ev_b, s);
    ctx->L()->timing_valid = true;
  }
  ctx->kernel_launches += 3;
  LC_CUDA_OK(cudaMemcpyAsync(h_dn, d_dn, dn_total, cudaMemcpyDeviceToHost, s));
  LC_CUDA_OK(cudaStreamSynchronize(s));
  ctx->d2h_bytes += dn_total;
  const uint32_t* h_counts = reinterpret_cast<const uint32_t*>(h_dn);
  const uint8_t* h_mask = h_dn + dn_counts;
  const uint8_t* h_valid = h_dn + dn_counts + dn_bits;
  for (uint64_t i = 0; i < n; ++i) {
    const uint32_t k = h_counts[4 * i], nulls = h_counts[4 * i + 1];
    if (k != sp.k[i]) {
      set_error("internal: selected-row count mismatch on entry %llu (%u vs %u)", (unsigned long long)i, k, sp.k[i]);
      return LC_ERR_INVALID;
    }
    const uint64_t bytes = static_cast<uint64_t>((k + 31) / 32) * 4;
    const uint64_t bo = out.byte_offsets ? out.byte_offsets[i] : 0;
    std::memcpy(out.values + bo, h_mask + word_off[i] * 4, bytes);
    if (out.validity) {
      if (nulls) std::memcpy(out.validity + bo, h_valid + word_off[i] * 4, bytes);
      else std::memset(out.validity + bo, 0xFF, bytes);
    }
    if (out.true_count) out.true_count[i] = h_counts[4 * i + 2];
    if (out.len) out.len[i] = k;
    if (out.null_count) out.null_count[i] = nulls;
  }
  return LC_OK;
}

// Device pipeline flavour: every row is decoded (the values live in scratch for the duration of the launch), then
// selection := selection & valid & cmp in place.
static int refine_float(lc_ctx* ctx, Entry* const* entries, uint64_t n, const RefList* rl, const lc_predicate* pred,
                        uint32_t* d_sel_base, const uint64_t* d_word_off, bool all_rows, uint32_t* d_counts) {
  const uint32_t tbits = entries[0]->ih.tbits, tb = tbits / 8;
  if (!rl->same_width) {
    set_error("scan_filter: Float32 and Float64 entries in one call");
    return LC_ERR_INVALID;
  }
  int32_t op = 0;
  long long key = 0;
  LC_TRY(make_float_pred(pred, tbits, &op, &key));
  std::vector<uint64_t> row_base(n);
  uint64_t rows = 0;
  for (uint64_t i = 0; i < n; ++i) {
    row_base[i] = rows;
    rows += (*rl->rows)[i];
  }
  const uint64_t b_rb = round_up(n * 8, 256), b_cnt = round_up(n * 16, 256), b_vals = round_up(rows * tb + 16, 256);
  Scratch& sc = ctx->L()->scratch;
  LC_TRY(sc.reserve(b_rb + b_cnt + b_vals + 1024, 1024));
  uint8_t* d_rb = sc.dev(b_rb);
  uint8_t* d_cnt = sc.dev(b_cnt);
  uint8_t* d_vals = sc.dev(b_vals);
  if (!d_rb || !d_cnt || !d_vals) {
    set_error("scan_filter: scratch exhausted");
    return LC_ERR_OOM;
  }
  cudaStream_t s = ctx->L()->stream;
  // pageable source: the runtime stages it before returning, so `row_base` may go out of scope
  LC_CUDA_OK(cudaMemcpyAsync(d_rb, row_base.data(), n * 8, cudaMemcpyHostToDevice, s));
  ctx->h2d_bytes += n * 8;
  ScanIo io{};
  io.refs = rl->d_refs;
  io.sel_base = nullptr;  // every row
  io.sel_off = d_word_off;
  io.out_base = d_vals;
  io.out_off = reinterpret_cast<const uint64_t*>(d_rb);
  io.valid_base = nullptr;
  io.valid_off = nullptr;
  io.counts = reinterpret_cast<uint32_t*>(d_cnt);
  io.counts_stride = 4;
  IntPredDesc ip{};
  if (ctx->L()->timing_on) cudaEventRecord(ctx->L()->ev_a, s);
  LC_CUDA_OK(launch_int_scan(MODE_DECODE, static_cast<uint32_t>(n), io, ip, rl->max_blob, s));
  LC_CUDA_OK(launch_alp_finish(static_cast<uint32_t>(n), io, tbits, s));
  FloatCmpIo c{};
  c.refs = rl->d_refs;
  c.vals_base = d_vals;
  c.vals_off = io.out_off;
  c.refine = 1;
  c.sel_base = all_rows ? nullptr : d_sel_base;
  c.sel_off = d_word_off;
  c.out_base = d_sel_base;
  c.out_off = d_word_off;
  c.counts = d_counts;
  c.counts_stride = 2;
  c.op = op;
  c.lit_key = key;
  LC_CUDA_OK(launch_float_cmp(static_cast<uint32_t>(n), c, tbits, s));
  if (ctx->L()->timing_on) {
    cudaEventRecord(ctx->L()->ev_b, s);
    ctx->L()->timing_valid = true;
  }
  ctx->kernel_launches += 3;
  return LC_OK;
}

// ---- eval_predicate --------------------------------------------------------------------------------
int eval_predicate_batch(lc_ctx* ctx, Entry* const* entries, uint64_t n, const lc_predicate* pred,
                         const uint8_t* const* sel_bits, const PredOut& out) {
  if (n == 0) return LC_OK;
  Tracer tr("eval_predicate");
  const RefList* rl;
  LC_TRY(get_ref_list(ctx, entries, n, &rl));
  if (!rl->same_liquid_type) {
    set_error("eval_predicate_many: entries of different liquid types in one call");
    return LC_ERR_INVALID;
  }
  FixedNeedle fixed;
  if (rl->any_fixed) {
    LC_TRY(lower_fixed_pred(entries, n, pred, &fixed));
    pred = &fixed.pred;
  }
  if (entries[0]->liquid_type == LC_LIQUID_FLOAT) return eval_predicate_float(ctx, entries, n, rl, pred, sel_bits, out);
  const bool is_int = is_int_blob(entries[0]->liquid_type);
  SelPlan sp;
  LC_TRY(plan_selection(ctx, rl->rows->data(), n, sel_bits, &sp));
  StrLaunch sl;
  IntPredDesc ip{};
  std::vector<uint8_t> int_list;  // IN lists on integer entries
  if (is_int && is_in_list(pred)) LC_TRY(make_int_in_list(pred, entries, n, &ip, &int_list));
  else if (is_int) LC_TRY(make_int_pred(pred, entries[0], &ip));
  else LC_TRY(prepare_str_pred(pred, &sl));
  const std::vector<uint8_t>& needle_blob = is_int ? int_list : sl.needle_blob;

  // upload: sel_off[n] | out_off[n] | needle (or IN list) | selection words ; download: counts[2n] | mask words | validity words
  const uint64_t up_offs = round_up(n * 16, 256);
  const uint64_t up_needle = round_up(needle_blob.size(), 256);
  const uint64_t up_sel = round_up(sp.sel_words * 4, 256);
  const uint64_t up_total = up_offs + up_needle + up_sel;
  const bool any_nulls = rl->any_nulls;
  const bool want_valid = any_nulls && out.validity != nullptr;
  // The device lays the masks out exactly as the caller's buffer is laid out (byte_offsets) whenever those
  // offsets are word aligned and ascending, so the whole result moves with ONE copy.
  std::vector<uint64_t> out_word_off(n);
  uint64_t out_words = 0;
  bool mirror = out.byte_offsets != nullptr || n == 1;
  const uint64_t first_off = out.byte_offsets ? out.byte_offsets[0] : 0;
  if (mirror) {
    uint64_t prev_end = first_off;
    for (uint64_t i = 0; i < n && mirror; ++i) {
      const uint64_t bo = out.byte_offsets ? out.byte_offsets[i] : 0;
      if ((bo & 3) || bo < prev_end) mirror = false;
      out_word_off[i] = (bo - first_off) / 4;
      prev_end = bo + static_cast<uint64_t>((sp.k[i] + 31) / 32) * 4;
      out_words = (prev_end - first_off) / 4;
    }
    if (out_words * 4 > (sp.total_k / 8 + n * 64) * 4 + (64u << 20)) mirror = false;  // absurdly sparse layout
  }
  if (!mirror) {
    out_words = 0;
    for (uint64_t i = 0; i < n; ++i) {
      out_word_off[i] = out_words;
      out_words += round_up((sp.k[i] + 31) / 32, 4);
    }
  }
  const uint64_t dn_counts = round_up(n * 16, 256);
  const uint64_t dn_bits = round_up(out_words * 4 + 16, 256);
  const uint64_t dn_total = dn_counts + (want_valid ? 2 : 1) * dn_bits;
  cudaPointerAttributes pa;
  const bool direct = mirror && cudaPointerGetAttributes(&pa, out.values) == cudaSuccess && pa.type == cudaMemoryTypeHost;
  cudaGetLastError();
  Scratch& sc = ctx->L()->scratch;
  LC_TRY(sc.reserve(up_total + dn_total + 1024, up_total + (direct ? dn_counts : dn_total) + 1024));
  uint8_t* h_up = sc.host(up_total);
  uint8_t* h_dn = sc.host(direct ? dn_counts : dn_total);
  uint8_t* d_up = sc.dev(up_total);
  uint8_t* d_dn = sc.dev(dn_total);
  if (!h_up || !h_dn || !d_up || !d_dn) {
    set_error("eval_predicate: scratch exhausted");
    return LC_ERR_OOM;
  }
  uint64_t* h_sel_off = reinterpret_cast<uint64_t*>(h_up);
  uint64_t* h_out_off = h_sel_off + n;
  for (uint64_t i = 0; i < n; ++i) {
    h_sel_off[i] = sp.bits[i] ? sp.word_off[i] : kNoSel;
    h_out_off[i] = out_word_off[i];
  }
  if (!needle_blob.empty()) std::memcpy(h_up + up_offs, needle_blob.data(), needle_blob.size());
  const IntInList in_list{reinterpret_cast<const uint64_t*>(d_up + up_offs), static_cast<uint32_t>(int_list.size() / 8), 0};
  ScanIo io{};
  io.refs = rl->d_refs;
  io.sel_base = sp.sel_words ? reinterpret_cast<const uint32_t*>(d_up + up_offs + up_needle) : nullptr;
  io.sel_off = reinterpret_cast<const uint64_t*>(d_up);
  io.out_base = d_dn + dn_counts;
  io.out_off = reinterpret_cast<const uint64_t*>(d_up) + n;
  io.valid_base = want_valid ? reinterpret_cast<uint32_t*>(d_dn + dn_counts + dn_bits) : nullptr;
  io.valid_off = io.out_off;
  io.counts = reinterpret_cast<uint32_t*>(d_dn);
  io.counts_stride = 4;
  cudaStream_t s = ctx->L()->stream;
  tr.mark("plan + fill");
  LC_CUDA_OK(cudaMemcpyAsync(d_up, h_up, up_offs + up_needle, cudaMemcpyHostToDevice, s));
  ctx->h2d_bytes += up_offs + up_needle;
  LC_TRY(upload_selection(ctx, sp, d_up + up_offs + up_needle, s));
  // With page-locked caller buffers the launch is cut into chunks of entries: the masks of chunk c cross PCIe on
  // the copy stream while chunk c+1 is being evaluated (mask download ~ kernel time for 1 KB per 8192 rows).
  const uint64_t span = out_words * 4;
  static const int chunk_pref = [] {
    const char* e = std::getenv("LC_EVAL_CHUNKS");
    const int v = e ? std::atoi(e) : 4;
    return v < 1 ? 1 : (v > 4 ? 4 : v);
  }();
  // Nearly-empty masks (a selective predicate) are downloaded as {word index, word} pairs: the mask area is zeroed
  // first, a gather kernel collects the non-zero words, and the host zero-fills the caller's buffer and drops them
  // in. Whether that pays is only known afterwards, so the list remembers how the last predicate turned out.
  // ... and it has the host zero-fill the whole mask area (12.5 MB for a 100 M-row column): with fewer than four host
  // threads to spread that over — ranks sharing one container's CPU quota — the plain download, which costs the host
  // nothing and overlaps the kernel chunk by chunk, is the better deal.
  const bool try_sparse = direct && !want_valid && span >= (1u << 16) && rl->mask_hint != 2 && host_pool_threads() >= 4u;
  const int n_chunks = (direct && n >= 2048 && span && !try_sparse) ? chunk_pref : 1;
  if (try_sparse) LC_CUDA_OK(cudaMemsetAsync(d_dn + dn_counts, 0, span, s));
  if (n_chunks > 1 && !ctx->L()->copy_stream) {
    LC_CUDA_OK(cudaStreamCreateWithFlags(&ctx->L()->copy_stream, cudaStreamNonBlocking));
    for (cudaEvent_t& e : ctx->L()->ev_chunk) LC_CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  }
  if (!is_int) {
    sl.desc.needle = d_up + up_offs;
    sl.desc.prof = ctx->prof_on ? ctx->d_prof : nullptr;
  }
  const bool like = !is_int && (pred->op == LC_OP_LIKE || pred->op == LC_OP_NOT_LIKE);
  if (like && sl.desc.needle_len >= 1 && sl.desc.needle_len <= 31 && rl->n_tables) {
    // the streaming LIKE kernel walks candidates through one Shift-And step table per FSST symbol table of the list
    // (kept from the previous call over this list when the needle is the same)
    const std::string needle_key(reinterpret_cast<const char*>(sl.needle_blob.data()), sl.needle_blob.size());
    if (rl->steps_needle != needle_key || rl->steps_stream != s) {
      LC_CUDA_OK(launch_like_steps(rl->d_tables, rl->n_tables, sl.desc, rl->d_like_steps, s));
      ctx->kernel_launches++;
      rl->steps_needle = needle_key;
      rl->steps_stream = s;
    }
    sl.desc.like_steps = rl->d_like_steps;
    sl.desc.entry_table = rl->d_entry_table;
  }
  // all rows of narrow integer entries: the register-resident kernel (its true-counts are added per chunk: zero them first)
  const bool int_bits = is_int && rl->int_bits_ok && io.sel_base == nullptr;
  if (int_bits) LC_CUDA_OK(cudaMemsetAsync(d_dn, 0, n * 16, s));
  if (ctx->L()->timing_on) cudaEventRecord(ctx->L()->ev_a, s);
  for (int c = 0; c < n_chunks; ++c) {
    const uint64_t c0 = n * c / n_chunks, c1 = n * (c + 1) / n_chunks;
    ScanIo ioc = io;
    ioc.refs += c0;
    ioc.sel_off += c0;
    ioc.out_off += c0;
    ioc.valid_off += c0;
    ioc.counts += c0 * io.counts_stride;
    if (is_int && int_bits) {
      LC_CUDA_OK(launch_int_bits(MODE_PRED, static_cast<uint32_t>(c1 - c0), ioc, ip, rl->max_rows, s, in_list));
    } else if (is_int) {
      LC_CUDA_OK(launch_int_scan(MODE_PRED, static_cast<uint32_t>(c1 - c0), ioc, ip, rl->max_blob, s, in_list));
    } else {
      StrPredDesc dc = sl.desc;
      if (dc.entry_table) dc.entry_table += c0;
      LC_CUDA_OK(launch_str_scan(MODE_PRED, static_cast<uint32_t>(c1 - c0), ioc, dc,
                                 like ? rl->max_head_like : rl->max_head, rl->max_unique, rl->max_meta, s));
    }
    ctx->kernel_launches++;
    if (n_chunks > 1) {
      const uint64_t b0 = out_word_off[c0] * 4, b1 = (c1 < n ? out_word_off[c1] * 4 : span);
      LC_CUDA_OK(cudaEventRecord(ctx->L()->ev_chunk[c], s));
      LC_CUDA_OK(cudaStreamWaitEvent(ctx->L()->copy_stream, ctx->L()->ev_chunk[c], 0));
      if (b1 > b0) {
        LC_CUDA_OK(cudaMemcpyAsync(out.values + first_off + b0, d_dn + dn_counts + b0, b1 - b0, cudaMemcpyDeviceToHost,
                                   ctx->L()->copy_stream));
        if (want_valid)
          LC_CUDA_OK(cudaMemcpyAsync(out.validity + first_off + b0, d_dn + dn_counts + dn_bits + b0, b1 - b0,
                                     cudaMemcpyDeviceToHost, ctx->L()->copy_stream));
      }
    }
  }
  if (ctx->L()->timing_on) {
    cudaEventRecord(ctx->L()->ev_b, s);
    ctx->L()->timing_valid = true;
  }
  bool sparse_done = false;
  if (try_sparse) {
    const uint64_t budget = out_words / 16;
    const uint64_t need = 16 + budget * 8;
    if (need > ctx->L()->d_pairs_cap) {
      if (ctx->L()->d_pairs) cudaFree(ctx->L()->d_pairs);
      ctx->L()->d_pairs = nullptr;
      ctx->L()->d_pairs_cap = 0;
      uint64_t cap = 1ull << 16;
      while (cap < need) cap *= 2;
      if (cudaMalloc(reinterpret_cast<void**>(&ctx->L()->d_pairs), cap) != cudaSuccess) {
        cudaGetLastError();
        set_error("cudaMalloc of %llu bytes for sparse masks failed", (unsigned long long)cap);
        return LC_ERR_OOM;
      }
      ctx->L()->d_pairs_cap = cap;
    }
    unsigned long long* d_counter = reinterpret_cast<unsigned long long*>(ctx->L()->d_pairs);
    unsigned long long* d_pairs = d_counter + 2;
    unsigned long long* h_counter = reinterpret_cast<unsigned long long*>(h_up);  // pinned, its upload is long done
    // staging for the pairs: room for the whole budget, so that nothing is allocated once the results are known
    if (budget * 8 + 64 > ctx->L()->sel_stage_cap) {
      LC_CUDA_OK(cudaStreamSynchronize(s));  // the selection upload may still be reading the old block
      if (ctx->L()->sel_stage) cudaFreeHost(ctx->L()->sel_stage);
      ctx->L()->sel_stage = nullptr;
      ctx->L()->sel_stage_cap = 0;
      uint64_t cap = 1ull << 20;
      while (cap < budget * 8 + 64) cap *= 2;
      if (cudaHostAlloc(reinterpret_cast<void**>(&ctx->L()->sel_stage), cap, cudaHostAllocDefault) != cudaSuccess) {
        cudaGetLastError();
        set_error("cudaHostAlloc of %llu bytes failed", (unsigned long long)cap);
        return LC_ERR_OOM;
      }
      ctx->L()->sel_stage_cap = cap;
    }
    LC_CUDA_OK(cudaMemsetAsync(d_counter, 0, 16, s));
    LC_CUDA_OK(launch_gather_nonzero(reinterpret_cast<const uint32_t*>(d_dn + dn_counts), out_words, d_pairs, budget, d_counter, s));
    ctx->kernel_launches++;
    LC_CUDA_OK(cudaMemcpyAsync(h_dn, d_dn, dn_counts, cudaMemcpyDeviceToHost, s));
    LC_CUDA_OK(cudaMemcpyAsync(h_counter, d_counter, 8, cudaMemcpyDeviceToHost, s));
    // The pairs come down SPECULATIVELY with the counts — as many as the last predicate over this list produced, and a
    // margin — so that the call waits for the device once; and the caller's mask area is zero-filled on the host while the
    // kernels are still running, not after them (neither depends on the answer).
    const uint64_t spec_pairs = std::min<uint64_t>(budget, rl->pairs_hint + rl->pairs_hint / 4 + 512);
    if (spec_pairs) LC_CUDA_OK(cudaMemcpyAsync(ctx->L()->sel_stage, d_pairs, spec_pairs * 8, cudaMemcpyDeviceToHost, s));
    parallel_for(span, 1u << 20, [&](uint64_t b, uint64_t e) { std::memset(out.values + first_off + b, 0, e - b); });
    LC_CUDA_OK(cudaStreamSynchronize(s));
    const uint64_t found = *h_counter;
    ctx->d2h_bytes += dn_counts + 8 + spec_pairs * 8;
    if (found <= budget) {
      if (found > spec_pairs) {  // more non-zero words than last time: fetch the rest (a second round trip)
        LC_CUDA_OK(cudaMemcpyAsync(ctx->L()->sel_stage + spec_pairs * 8, d_pairs + spec_pairs, (found - spec_pairs) * 8,
                                   cudaMemcpyDeviceToHost, s));
        LC_CUDA_OK(cudaStreamSynchronize(s));
        ctx->d2h_bytes += (found - spec_pairs) * 8;
      }
      const unsigned long long* hp = reinterpret_cast<const unsigned long long*>(ctx->L()->sel_stage);
      uint32_t* dst = reinterpret_cast<uint32_t*>(out.values + first_off);
      for (uint64_t i = 0; i < found; ++i) dst[hp[i] >> 32] = static_cast<uint32_t>(hp[i]);
      rl->pairs_hint = found;
      rl->mask_hint = 1;
      sparse_done = true;
    } else {
      rl->mask_hint = 2;  // dense after all: plain download now (over the zeros), chunked overlap next time
    }
  }
  if (sparse_done) {
    // counts and masks are already on the host
  } else if (direct) {
    // the caller's buffers are page-locked: results land in them straight from the device
    LC_CUDA_OK(cudaMemcpyAsync(h_dn, d_dn, dn_counts, cudaMemcpyDeviceToHost, s));
    if (n_chunks == 1) {
      if (span) LC_CUDA_OK(cudaMemcpyAsync(out.values + first_off, d_dn + dn_counts, span, cudaMemcpyDeviceToHost, s));
      if (want_valid && span)
        LC_CUDA_OK(cudaMemcpyAsync(out.validity + first_off, d_dn + dn_counts + dn_bits, span, cudaMemcpyDeviceToHost, s));
    }
    ctx->d2h_bytes += dn_counts + span * (want_valid ? 2 : 1);
  } else {
    LC_CUDA_OK(cudaMemcpyAsync(h_dn, d_dn, dn_total, cudaMemcpyDeviceToHost, s));
    ctx->d2h_bytes += dn_total;
  }
  if (n_chunks > 1) LC_CUDA_OK(cudaStreamSynchronize(ctx->L()->copy_stream));
  LC_CUDA_OK(cudaStreamSynchronize(s));
  tr.mark(direct ? "upload + kernel + direct D2H" : "upload + kernel + staged D2H");

  const uint32_t* h_counts = reinterpret_cast<const uint32_t*>(h_dn);
  const uint8_t* h_mask = h_dn + dn_counts;
  const uint8_t* h_valid = h_dn + dn_counts + dn_bits;
  if (mirror && !direct && span) {
    std::memcpy(out.values + first_off, h_mask, span);
    if (want_valid) std::memcpy(out.validity + first_off, h_valid, span);
  }
  uint64_t total_true = 0;
  for (uint64_t i = 0; i < n; ++i) {
    const uint32_t k = h_counts[4 * i], nulls = h_counts[4 * i + 1];
    if (k != sp.k[i]) {
      set_error("internal: selected-row count mismatch on entry %llu (%u vs %u)", (unsigned long long)i, k, sp.k[i]);
      return LC_ERR_INVALID;
    }
    if (out.true_count) out.true_count[i] = h_counts[4 * i + 2];
    total_true += h_counts[4 * i + 2];
    const uint64_t bytes = static_cast<uint64_t>((k + 31) / 32) * 4;
    const uint64_t bo = out.byte_offsets ? out.byte_offsets[i] : 0;
    if (!mirror) {
      std::memcpy(out.values + bo, h_mask + out_word_off[i] * 4, bytes);
      if (want_valid && nulls) std::memcpy(out.validity + bo, h_valid + out_word_off[i] * 4, bytes);
    }
    if (out.validity && nulls == 0 && any_nulls) std::memset(out.validity + bo, 0xFF, bytes);
    if (out.len) out.len[i] = k;
    if (out.null_count) out.null_count[i] = nulls;
  }
  if (rl->mask_hint == 2 && total_true < out_words / 32) rl->mask_hint = 0;  // selective again: retry the sparse download
  tr.mark("per-entry results");
  // no entry has nulls: validity (if the caller wants it at all) is all ones
  if (out.validity && !any_nulls) {
    if (mirror && span)
      parallel_for(span, 1u << 20, [&](uint64_t b, uint64_t e) { std::memset(out.validity + first_off + b, 0xFF, e - b); });
    else
      for (uint64_t i = 0; i < n; ++i)
        std::memset(out.validity + (out.byte_offsets ? out.byte_offsets[i] : 0), 0xFF, static_cast<uint64_t>((sp.k[i] + 31) / 32) * 4);
  }
  return LC_OK;
}

// ---- device pipeline: selection := selection & valid & predicate (no host round trip of bits) ----
int refine_batch(lc_ctx* ctx, Entry* const* entries, uint64_t n, const lc_predicate* pred, uint32_t* d_sel_base,
                 const uint64_t* d_word_off, bool all_rows, uint32_t* d_counts) {
  if (n == 0) return LC_OK;
  const RefList* rl;
  LC_TRY(get_ref_list(ctx, entries, n, &rl));
  if (!rl->same_liquid_type) {
    set_error("scan_filter: entries of different liquid types in one call");
    return LC_ERR_INVALID;
  }
  FixedNeedle fixed;
  if (rl->any_fixed) {
    LC_TRY(lower_fixed_pred(entries, n, pred, &fixed));
    pred = &fixed.pred;
  }
  if (entries[0]->liquid_type == LC_LIQUID_FLOAT)
    return refine_float(ctx, entries, n, rl, pred, d_sel_base, d_word_off, all_rows, d_counts);
  const bool is_int = is_int_blob(entries[0]->liquid_type);
  StrLaunch sl;
  IntPredDesc ip{};
  std::vector<uint8_t> int_list;  // IN lists on integer entries
  if (is_int && is_in_list(pred)) LC_TRY(make_int_in_list(pred, entries, n, &ip, &int_list));
  else if (is_int) LC_TRY(make_int_pred(pred, entries[0], &ip));
  else LC_TRY(prepare_str_pred(pred, &sl));
  cudaStream_t s = ctx->L()->stream;
  // The needle (or IN list) is the only thing that travels: a few bytes from pageable memory (the runtime stages such
  // copies before returning) into a small buffer the context keeps for this purpose.
  const std::vector<uint8_t>& needle_blob = is_int ? int_list : sl.needle_blob;
  uint8_t* d_nd = nullptr;
  if (!needle_blob.empty()) {
    if (!ctx->L()->d_needle) {
      if (cudaMalloc(reinterpret_cast<void**>(&ctx->L()->d_needle), std::max<size_t>(2 * (kMaxNeedle + 16) * 2, kInListBlobCap)) != cudaSuccess) {
        cudaGetLastError();
        set_error("cudaMalloc for the needle buffer failed");
        return LC_ERR_OOM;
      }
    }
    d_nd = ctx->L()->d_needle;
    const std::string needle_key(reinterpret_cast<const char*>(needle_blob.data()), needle_blob.size());
    if (ctx->L()->needle_in_buffer != needle_key || ctx->L()->needle_stream != s) {  // the buffer already holds it otherwise
      LC_CUDA_OK(cudaMemcpyAsync(d_nd, needle_blob.data(), needle_blob.size(), cudaMemcpyHostToDevice, s));
      ctx->h2d_bytes += needle_blob.size();
      ctx->L()->needle_in_buffer = needle_key;
      ctx->L()->needle_stream = s;
    }
  }
  const IntInList in_list{reinterpret_cast<const uint64_t*>(d_nd), static_cast<uint32_t>(int_list.size() / 8), 0};
  ScanIo io{};
  io.refs = rl->d_refs;
  io.sel_base = all_rows ? nullptr : d_sel_base;
  io.sel_off = d_word_off;
  io.out_base = d_sel_base;
  io.out_off = d_word_off;
  io.valid_base = nullptr;
  io.valid_off = nullptr;
  io.counts = d_counts;
  io.counts_stride = 2;
  if (is_int) {
    if (rl->int_bits_ok && d_counts) LC_CUDA_OK(cudaMemsetAsync(d_counts, 0, n * 8, s));  // k_int_bits adds per chunk
    if (ctx->L()->timing_on) cudaEventRecord(ctx->L()->ev_a, s);
    if (rl->int_bits_ok) LC_CUDA_OK(launch_int_bits(MODE_REFINE, static_cast<uint32_t>(n), io, ip, rl->max_rows, s, in_list));
    else LC_CUDA_OK(launch_int_scan(MODE_REFINE, static_cast<uint32_t>(n), io, ip, rl->max_blob, s, in_list));
  } else {
    const std::string needle_key(reinterpret_cast<const char*>(sl.needle_blob.data()), sl.needle_blob.size());
    sl.desc.needle = d_nd;
    sl.desc.prof = ctx->prof_on ? ctx->d_prof : nullptr;
    const bool like = (pred->op == LC_OP_LIKE || pred->op == LC_OP_NOT_LIKE);
    if (like && sl.desc.needle_len >= 1 && sl.desc.needle_len <= 31 && rl->n_tables) {
      if (rl->steps_needle != needle_key || rl->steps_stream != s) {
        LC_CUDA_OK(launch_like_steps(rl->d_tables, rl->n_tables, sl.desc, rl->d_like_steps, s));
        ctx->kernel_launches++;
        rl->steps_needle = needle_key;
        rl->steps_stream = s;
      }
      sl.desc.like_steps = rl->d_like_steps;
      sl.desc.entry_table = rl->d_entry_table;
    }
    if (ctx->L()->timing_on) cudaEventRecord(ctx->L()->ev_a, s);
    LC_CUDA_OK(launch_str_scan(MODE_REFINE, static_cast<uint32_t>(n), io, sl.desc, like ? rl->max_head_like : rl->max_head,
                               rl->max_unique, rl->max_meta, s));
  }
  if (ctx->L()->timing_on) {
    cudaEventRecord(ctx->L()->ev_b, s);
    ctx->L()->timing_valid = true;
  }
  ctx->kernel_launches++;
  return LC_OK;
}

// ---- reads planned on the device -------------------------------------------------------------------
// The survivors of a device-resident selection are sized, placed and decoded against capacities chosen before their counts
// are known (k_scan_plan.cu, k_str_read_onepass); the 64-byte ScanPlanHdr (rows, bytes, overflow) says whether the
// capacities sufficed. Used by the selective byte-view get (to_arrow_batch), scan_read_fused and scan_read_async.
struct PlannedRead {
  const uint32_t* sel_base;  // selection words
  const uint64_t* sel_off;   // per entry: word offset into sel_base
  const uint32_t* k2;        // per entry: surviving rows, at stride 2
  uint64_t cap_rows, cap_bytes, cap_ulen;
  bool onepass;              // byte views: the whole read is ONE kernel (k_str_read_onepass)
  uint8_t* scratch;          // device, planned_layout(...).bytes
  void* d_values;
  int32_t* d_offsets;        // byte views: int32[cap_rows + 1]; integers: nullptr
  ScanPlanHdr* d_hdr;
};

static uint64_t carve(uint64_t* o, uint64_t bytes) {
  const uint64_t at = *o;
  *o += round_up(bytes, 256);
  return at;
}

// Offsets of the pieces of a read's device scratch; `bytes` is the total.
struct PlannedLayout {
  uint64_t status = 0, rowb = 0, vw = 0, ul = 0, bb = 0, cnt = 0, rowoff = 0, rowkey = 0, ulen = 0, bytes = 0;
};
static PlannedLayout planned_layout(uint64_t n, bool is_str, bool onepass, uint64_t cap_rows, uint64_t cap_ulen) {
  PlannedLayout l;
  if (onepass) {  // the status words of its chained scan are all the one-pass kernel needs
    l.status = carve(&l.bytes, ((n + 7) / 8 + 2) * 8);
    return l;
  }
  l.rowb = carve(&l.bytes, n * 8);
  l.vw = carve(&l.bytes, n * 8);
  l.ul = carve(&l.bytes, n * 8);
  l.bb = carve(&l.bytes, n * 8);
  l.cnt = carve(&l.bytes, n * 16);
  if (is_str) {
    l.rowoff = carve(&l.bytes, (cap_rows + n) * 4 + 16);
    l.rowkey = carve(&l.bytes, cap_rows * 4 + 16);
    l.ulen = carve(&l.bytes, cap_ulen * 4 + 16);
  }
  return l;
}

// Enqueues the read on the lane's stream without synchronising: the one-pass kernel, or the row plan followed by the
// integer decode or by the four byte-view launches (sparse lengths, lengths, byte plan, decode).
static int enqueue_planned_read(lc_ctx* ctx, const RefList* rl, uint64_t n, const PlannedRead& pr) {
  cudaStream_t s = ctx->L()->stream;
  const uint32_t nn = static_cast<uint32_t>(n);
  const bool is_str = pr.d_offsets != nullptr;
  const PlannedLayout l = planned_layout(n, is_str, pr.onepass, pr.cap_rows, pr.cap_ulen);
  uint8_t* d = pr.scratch;
  StrGatherIo g{};
  g.io.refs = rl->d_refs;
  g.io.sel_base = pr.sel_base;
  g.io.sel_off = pr.sel_off;
  g.k_hint = pr.k2;
  g.out_offsets = pr.d_offsets;
  g.out_bytes = static_cast<uint8_t*>(pr.d_values);
  if (pr.onepass) {
    LC_CUDA_OK(launch_str_read_onepass(nn, g, pr.cap_rows, pr.cap_bytes, pr.d_hdr, reinterpret_cast<unsigned long long*>(d + l.status), s));
    ctx->kernel_launches++;
    return LC_OK;
  }
  uint64_t* d_rowb = reinterpret_cast<uint64_t*>(d + l.rowb);
  uint64_t* d_vw = reinterpret_cast<uint64_t*>(d + l.vw);
  uint64_t* d_ul = reinterpret_cast<uint64_t*>(d + l.ul);
  uint64_t* d_bb = reinterpret_cast<uint64_t*>(d + l.bb);
  uint32_t* d_cnt = reinterpret_cast<uint32_t*>(d + l.cnt);
  LC_CUDA_OK(cudaMemsetAsync(d_cnt, 0, n * 16, s));
  LC_CUDA_OK(launch_scan_plan_rows(pr.k2, is_str ? rl->d_n_unique : nullptr, nn, pr.cap_rows, pr.cap_ulen, d_rowb, d_vw, d_ul, pr.d_hdr, s));
  ctx->kernel_launches++;
  g.io.out_off = d_rowb;
  g.io.valid_off = d_vw;
  g.io.counts = d_cnt;
  g.io.counts_stride = 4;
  if (!is_str) {
    g.io.out_base = pr.d_values;
    g.io.abort_flag = &pr.d_hdr->overflow;  // survivors beyond the capacity: the kernel returns without writing
    LC_CUDA_OK(launch_int_scan(MODE_DECODE, nn, g.io, IntPredDesc{}, rl->max_blob, s));
    ctx->kernel_launches++;
    return LC_OK;
  }
  g.row_off_base = reinterpret_cast<uint32_t*>(d + l.rowoff);
  g.row_key_base = reinterpret_cast<uint32_t*>(d + l.rowkey);
  g.ulen_base = reinterpret_cast<uint32_t*>(d + l.ulen);
  g.row_base = d_rowb;
  g.ulen_off = d_ul;
  g.byte_base = d_bb;
  g.plan = pr.d_hdr;
  g.sparse_max = 64;  // entries with up to 64 survivors: one warp each, no staging (k_str_lengths_sparse)
  LC_CUDA_OK(launch_str_lengths_sparse(nn, g, s));
  LC_CUDA_OK(launch_str_lengths(nn, g, rl->max_head, s));
  LC_CUDA_OK(launch_scan_plan_bytes(d_cnt, nn, pr.cap_bytes, d_bb, g.out_offsets, pr.d_hdr, s));
  LC_CUDA_OK(launch_str_decode(nn, g, s));
  ctx->kernel_launches += 4;
  return LC_OK;
}

// The host's half of a planned read: the header, the offsets (byte views) and a speculative prefix of the values come down
// with ONE synchronisation; a result larger than that prefix is fetched whole in a second round trip (rare). `value_width`
// is the integers' bytes per value (byte views: 0, their size is in the header). When the header reports an overflow
// nothing more is fetched or counted: the caller decides.
struct PlannedHost {
  ScanPlanHdr hdr{};
  HostBlock offsets, values;
};
static int download_planned(lc_ctx* ctx, ScanPlanHdr* h_hdr, const PlannedRead& pr, uint32_t value_width, uint64_t spec_rows,
                            uint64_t spec_bytes, PlannedHost* out) {
  cudaStream_t s = ctx->L()->stream;
  const bool is_str = pr.d_offsets != nullptr;
  const uint64_t pre_rows = std::min(spec_rows, pr.cap_rows), pre_bytes = std::min(spec_bytes, pr.cap_bytes);
  if (is_str) out->offsets = HostBlock((spec_rows + 1) * 4 + 64, 0, true);
  out->values = HostBlock(spec_bytes + 64, 0, true);
  if ((is_str && !out->offsets.p) || !out->values.p) {
    set_error("host allocation failed");
    return LC_ERR_OOM;
  }
  LC_CUDA_OK(cudaMemcpyAsync(h_hdr, pr.d_hdr, sizeof(ScanPlanHdr), cudaMemcpyDeviceToHost, s));
  if (is_str) LC_CUDA_OK(cudaMemcpyAsync(out->offsets.p, pr.d_offsets, (pre_rows + 1) * 4, cudaMemcpyDeviceToHost, s));
  if (pre_bytes) LC_CUDA_OK(cudaMemcpyAsync(out->values.p, pr.d_values, pre_bytes, cudaMemcpyDeviceToHost, s));
  LC_CUDA_OK(cudaStreamSynchronize(s));
  out->hdr = *h_hdr;
  if (out->hdr.overflow) return LC_OK;
  const uint64_t rows = out->hdr.rows, bytes = is_str ? out->hdr.bytes : rows * value_width;
  ctx->d2h_bytes += sizeof(ScanPlanHdr) + (is_str ? (pre_rows + 1) * 4 : 0) + pre_bytes;
  if (rows > spec_rows || bytes > spec_bytes) {
    // offsets that covered the whole row capacity are complete (the selective get knows its rows); the rest comes again
    const bool offsets_again = is_str && spec_rows < pr.cap_rows;
    if (offsets_again) out->offsets = HostBlock((rows + 1) * 4 + 64, 0, true);
    out->values = HostBlock(bytes + 64, 0, true);
    if ((offsets_again && !out->offsets.p) || !out->values.p) {
      set_error("host allocation failed");
      return LC_ERR_OOM;
    }
    if (offsets_again) LC_CUDA_OK(cudaMemcpyAsync(out->offsets.p, pr.d_offsets, (rows + 1) * 4, cudaMemcpyDeviceToHost, s));
    LC_CUDA_OK(cudaMemcpyAsync(out->values.p, pr.d_values, bytes, cudaMemcpyDeviceToHost, s));
    LC_CUDA_OK(cudaStreamSynchronize(s));
    ctx->d2h_bytes += (offsets_again ? (rows + 1) * 4 : 0) + bytes;
  }
  if (is_str) {
    reinterpret_cast<int32_t*>(out->offsets.p)[rows] = static_cast<int32_t>(bytes);
    out->offsets.bytes = (rows + 1) * 4;
  }
  out->values.bytes = bytes;
  return LC_OK;
}

// Makes a scan's device buffer hold `need` bytes; a new allocation gets `headroom` more. LC_INTERNAL_FALLBACK when
// cudaMalloc fails.
static int grow_device(cudaStream_t s, uint8_t** buf, uint64_t* cap, uint64_t need, uint64_t headroom) {
  if (need <= *cap) return LC_OK;
  if (*buf) {
    LC_CUDA_OK(cudaStreamSynchronize(s));
    cudaFree(*buf);
    *buf = nullptr;
    *cap = 0;
  }
  if (cudaMalloc(reinterpret_cast<void**>(buf), need + headroom) != cudaSuccess) {
    cudaGetLastError();
    return LC_INTERNAL_FALLBACK;
  }
  *cap = need + headroom;
  return LC_OK;
}

// ---- get / filter ----------------------------------------------------------------------------------
static int finish_bytes_array(const Entry* proto, uint64_t rows, uint64_t nulls, HostBlock validity, HostBlock offsets,
                              HostBlock views, HostBlock data, ArrowSchema* out_schema, ArrowArray* out_array);

int to_arrow_batch(lc_ctx* ctx, Entry* const* entries, uint64_t n, const uint8_t* const* sel_bits,
                   const DevSel* dev_sel, ArrowSchema* out_schema, ArrowArray* out_array, const DeviceOut* dev_out) {
  Tracer tr("to_arrow");
  if (n == 0) {
    set_error("to_arrow: empty entry list");
    return LC_ERR_INVALID;
  }
  const Entry* proto = entries[0];
  const RefList* rl;
  LC_TRY(get_ref_list(ctx, entries, n, &rl));
  if (!rl->same_liquid_type || !rl->same_arrow_type) {
    set_error("to_arrow_many: entries have different arrow types");
    return LC_ERR_INVALID;
  }
  tr.mark("entry list + type check");
  SelPlan sp;
  LC_TRY(plan_selection(ctx, rl->rows->data(), n, sel_bits, &sp, dev_sel));
  tr.mark("stage selection");
  const bool is_int = is_int_blob(proto->liquid_type);
  cudaStream_t s = ctx->L()->stream;
  Scratch& sc = ctx->L()->scratch;

  std::vector<uint64_t> vword_off(n), row_base(n);
  uint64_t vwords = 0, rows = 0;
  for (uint64_t i = 0; i < n; ++i) {
    vword_off[i] = vwords;
    vwords += round_up((sp.k[i] + 31) / 32, 4);
    row_base[i] = rows;
    rows += sp.k[i];
  }
  if (rows > 0x7fffffffull) {
    set_error("result has more than 2^31 rows");
    return LC_ERR_INVALID;
  }
  tr.mark("plan");
  // upload: sel_off[n] | out_off[n] (ints: element offsets; strings: row_base) | valid_off[n] | ulen_off[n] |
  //         byte_base[n] (strings, second upload) | selection words
  const uint64_t up_offs = round_up(n * 8 * 6, 256);
  const uint64_t up_sel = round_up(sp.sel_words * 4, 256);
  const uint64_t up_total = up_offs + up_sel;
  const uint64_t dn_counts = round_up(n * 16, 256);
  const uint64_t dn_valid = round_up(vwords * 4, 256);
  const uint64_t dn_total = dn_counts + dn_valid;

  auto fill_offsets = [&](uint8_t* h_up, const std::vector<uint64_t>* ulen_off) {
    uint64_t* a = reinterpret_cast<uint64_t*>(h_up);
    for (uint64_t i = 0; i < n; ++i) {
      a[i] = dev_sel ? (dev_sel->all_rows ? kNoSel : dev_sel->word_off[i]) : (sp.bits[i] ? sp.word_off[i] : kNoSel);
      a[n + i] = row_base[i];
      a[2 * n + i] = vword_off[i];
      a[3 * n + i] = ulen_off ? (*ulen_off)[i] : 0;
      a[4 * n + i] = 0;
    }
  };
  auto make_io = [&](uint8_t* d_up, uint8_t* d_dn, void* out_base) {
    ScanIo io{};
    io.refs = rl->d_refs;
    const uint64_t* offs = reinterpret_cast<const uint64_t*>(d_up);
    if (dev_sel) io.sel_base = dev_sel->all_rows ? nullptr : dev_sel->d_base;
    else io.sel_base = sp.sel_words ? reinterpret_cast<const uint32_t*>(d_up + up_offs) : nullptr;
    io.sel_off = offs;
    io.out_base = out_base;
    io.out_off = offs + n;
    io.valid_base = reinterpret_cast<uint32_t*>(d_dn + dn_counts);
    io.valid_off = offs + 2 * n;
    io.counts = reinterpret_cast<uint32_t*>(d_dn);
    io.counts_stride = 4;
    return io;
  };
  // Validity of the concatenated result: the per-entry compact bit strings the kernels wrote are joined at bit
  // granularity ON THE DEVICE (k_concat_validity; entries without nulls read as all ones) and the finished bitmap is
  // copied to the host — no host loop over rows or entries.
  const uint64_t cat_bytes = round_up(((rows + 31) / 32) * 4 + 16, 256);
  auto concat_validity_device = [&](const ScanIo& io, uint8_t* d_up, uint8_t* d_cat, HostBlock* validity) -> int {
    *validity = HostBlock(round_up((rows + 7) / 8, 4), (rows + 7) / 8);
    if (!validity->p) {
      set_error("host allocation failed");
      return LC_ERR_OOM;
    }
    const uint64_t* offs = reinterpret_cast<const uint64_t*>(d_up);
    LC_CUDA_OK(launch_concat_validity(io.valid_base, offs + 2 * n, offs + n, io.counts, 4, static_cast<uint32_t>(n), rows,
                                      reinterpret_cast<uint32_t*>(d_cat), s));
    ctx->kernel_launches++;
    LC_CUDA_OK(cudaMemcpyAsync(validity->p, d_cat, round_up(validity->bytes, 4), cudaMemcpyDeviceToHost, s));
    ctx->d2h_bytes += validity->bytes;
    return LC_OK;
  };

  if (is_int) {
    const uint32_t tb = proto->ih.tbits / 8;
    const bool is_float = proto->liquid_type == LC_LIQUID_FLOAT;
    const bool is_dec = proto->liquid_type == LC_LIQUID_DECIMAL;
    const uint32_t out_tb = is_dec ? proto->dec_width : tb;  // bytes per value of the Arrow result
    if (!rl->same_width) {
      set_error("to_arrow_many: mixed integer widths");
      return LC_ERR_INVALID;
    }
    const uint64_t val_bytes = round_up(rows * tb, 256);
    const uint64_t wide_bytes = is_dec ? round_up(rows * out_tb, 256) : 0;
    LC_TRY(sc.reserve(up_total + dn_total + val_bytes + wide_bytes + cat_bytes + 1024, up_total + dn_total + 1024));
    uint8_t* h_up = sc.host(up_total);
    uint8_t* h_dn = sc.host(dn_total);
    uint8_t* d_up = sc.dev(up_total);
    uint8_t* d_dn = sc.dev(dn_total);
    uint8_t* d_vals = sc.dev(val_bytes);
    uint8_t* d_wide = is_dec ? sc.dev(wide_bytes) : nullptr;
    uint8_t* d_cat = sc.dev(cat_bytes);
    if (!h_up || !h_dn || !d_up || !d_dn || !d_vals || (is_dec && !d_wide) || !d_cat) {
      set_error("to_arrow: scratch exhausted");
      return LC_ERR_OOM;
    }
    if (dev_out && !dev_out->d_values && !rl->any_nulls) {
      // size query over entries without nulls: everything asked for follows from the selection counts
      if (dev_out->out_rows) *dev_out->out_rows = rows;
      if (dev_out->out_value_bytes) *dev_out->out_value_bytes = rows * out_tb;
      if (dev_out->out_null_count) *dev_out->out_null_count = 0;
      return LC_OK;
    }
    fill_offsets(h_up, nullptr);
    const ScanIo io = make_io(d_up, d_dn, d_vals);
    IntPredDesc ip{};
    LC_CUDA_OK(cudaMemcpyAsync(d_up, h_up, up_offs, cudaMemcpyHostToDevice, s));
    ctx->h2d_bytes += up_offs;
    if (!dev_sel) LC_TRY(upload_selection(ctx, sp, d_up + up_offs, s));
    LC_CUDA_OK(launch_int_scan(MODE_DECODE, static_cast<uint32_t>(n), io, ip, rl->max_blob, s));
    ctx->kernel_launches++;
    if (is_float) {
      // the decode left the ALP integers of the selected rows: -> floats in place, then their patches
      LC_CUDA_OK(launch_alp_finish(static_cast<uint32_t>(n), io, proto->ih.tbits, s));
      ctx->kernel_launches++;
    }
    const uint8_t* d_result = d_vals;  // what travels: native values, or the decimals widened to 128/256 bits
    if (dev_out) {
      // device-resident result: counts come back (null count), values and validity stay in HBM
      LC_CUDA_OK(cudaMemcpyAsync(h_dn, d_dn, dn_counts, cudaMemcpyDeviceToHost, s));
      LC_CUDA_OK(cudaStreamSynchronize(s));
      ctx->d2h_bytes += dn_counts;
      const uint32_t* hc = reinterpret_cast<const uint32_t*>(h_dn);
      uint64_t nulls = 0;
      for (uint64_t i = 0; i < n; ++i) nulls += hc[4 * i + 1];
      if (dev_out->out_rows) *dev_out->out_rows = rows;
      if (dev_out->out_value_bytes) *dev_out->out_value_bytes = rows * out_tb;
      if (dev_out->out_null_count) *dev_out->out_null_count = nulls;
      if (!dev_out->d_values) return LC_OK;  // size query
      if (dev_out->values_cap < rows * out_tb) {
        set_error("read_device: values buffer of %llu bytes, need %llu", (unsigned long long)dev_out->values_cap,
                  (unsigned long long)(rows * out_tb));
        return LC_ERR_INVALID;
      }
      if (is_dec) {
        LC_CUDA_OK(launch_dec_widen(reinterpret_cast<const unsigned long long*>(d_vals), rows, out_tb, dev_out->d_values, s));
        ctx->kernel_launches++;
      } else if (rows) {
        LC_CUDA_OK(cudaMemcpyAsync(dev_out->d_values, d_vals, rows * tb, cudaMemcpyDeviceToDevice, s));
      }
      if (nulls && dev_out->d_validity) {
        const uint64_t* offs = reinterpret_cast<const uint64_t*>(d_up);
        LC_CUDA_OK(launch_concat_validity(io.valid_base, offs + 2 * n, offs + n, io.counts, 4, static_cast<uint32_t>(n), rows,
                                          static_cast<uint32_t*>(dev_out->d_validity), s));
        ctx->kernel_launches++;
      }
      LC_CUDA_OK(cudaStreamSynchronize(s));
      return LC_OK;
    }
    if (is_dec) {
      LC_CUDA_OK(launch_dec_widen(reinterpret_cast<const unsigned long long*>(d_vals), rows, out_tb, d_wide, s));
      ctx->kernel_launches++;
      d_result = d_wide;
    }
    HostBlock values(rows * out_tb, rows * out_tb);
    if (!values.p) {
      set_error("host allocation of %llu bytes failed", (unsigned long long)(rows * out_tb));
      return LC_ERR_OOM;
    }
    LC_CUDA_OK(cudaMemcpyAsync(h_dn, d_dn, dn_counts, cudaMemcpyDeviceToHost, s));
    if (rows) LC_CUDA_OK(cudaMemcpyAsync(values.p, d_result, rows * out_tb, cudaMemcpyDeviceToHost, s));
    LC_CUDA_OK(cudaStreamSynchronize(s));
    ctx->d2h_bytes += dn_counts + rows * out_tb;
    const uint32_t* h_counts = reinterpret_cast<const uint32_t*>(h_dn);
    uint64_t nulls = 0;
    for (uint64_t i = 0; i < n; ++i) {
      if (h_counts[4 * i] != sp.k[i]) {
        set_error("internal: selected-row count mismatch on entry %llu", (unsigned long long)i);
        return LC_ERR_INVALID;
      }
      nulls += h_counts[4 * i + 1];
    }
    HostBlock validity;
    if (nulls) {  // second, small round trip only when the result has nulls
      LC_TRY(concat_validity_device(io, d_up, d_cat, &validity));
      LC_CUDA_OK(cudaStreamSynchronize(s));
    }
    export_schema(proto->arrow_format, "", out_schema);
    std::vector<HostBuf> bufs{validity.release(), values.release()};
    export_array(static_cast<int64_t>(rows), static_cast<int64_t>(nulls), std::move(bufs), nullptr, out_array);
    return LC_OK;
  }

  // ---------------- byte-view, a handful of rows per batch: ONE kernel, ONE synchronisation ----------------
  // What the reader does after a selective predicate (liquid_cache_reader.rs:342-391: only batches with survivors, each with
  // its mask as the selection): the row counts are known here, the decoded bytes are not — k_str_read_onepass sizes, places
  // (chained scan across its CTAs) and decodes in one launch, and the host downloads the 64-byte header together with the
  // offsets and a speculative prefix of the bytes (sized by what such reads have needed so far).
  {
    bool sparse_ok = !dev_sel && !dev_out && rows != 0 && rows <= 16ull * n && !rl->any_nulls && !rl->any_fixed &&
                     (proto->sh.arrow_type == BT_UTF8 || proto->sh.arrow_type == BT_BINARY);
    uint64_t bound = 0;
    for (uint64_t i = 0; i < n && sparse_ok; ++i) {
      if (!sp.bits[i]) sparse_ok = false;  // an all-ones selection takes every row of the batch
      bound += static_cast<uint64_t>(sp.k[i]) * entries[i]->sh.max_value_len;
    }
    if (sparse_ok && bound <= (256ull << 20)) {
      const uint64_t cap_bytes = bound;
      const uint64_t up_tab = round_up(n * 16, 256);  // word_off[n] (u64) | k[n] at stride 2 (u32 pairs)
      const uint64_t up_sel1 = round_up(sp.sel_words * 4, 256);
      const uint64_t dv_plan = planned_layout(n, true, true, rows, 0).bytes;
      const uint64_t dv_off = round_up((rows + 1) * 4, 256), dv_val = round_up(cap_bytes + 16, 256);
      LC_TRY(sc.reserve(up_tab + up_sel1 + dv_plan + 256 + dv_off + dv_val + 1024, up_tab + 256 + 1024));
      uint8_t* h_up = sc.host(up_tab);
      ScanPlanHdr* h_hdr = reinterpret_cast<ScanPlanHdr*>(sc.host(256));
      uint8_t* d_up = sc.dev(up_tab + up_sel1);
      uint8_t* d_plan = sc.dev(dv_plan);
      ScanPlanHdr* d_hdr = reinterpret_cast<ScanPlanHdr*>(sc.dev(256));
      int32_t* d_off = reinterpret_cast<int32_t*>(sc.dev(dv_off));
      uint8_t* d_val = sc.dev(dv_val);
      if (!h_up || !h_hdr || !d_up || !d_plan || !d_hdr || !d_off || !d_val) {
        set_error("to_arrow: scratch exhausted");
        return LC_ERR_OOM;
      }
      uint64_t* h_word_off = reinterpret_cast<uint64_t*>(h_up);
      uint32_t* h_k2 = reinterpret_cast<uint32_t*>(h_up + n * 8);
      for (uint64_t i = 0; i < n; ++i) {
        h_word_off[i] = sp.word_off[i];
        h_k2[2 * i] = sp.k[i];
        h_k2[2 * i + 1] = 0;
      }
      LC_CUDA_OK(cudaMemcpyAsync(d_up, h_up, n * 16, cudaMemcpyHostToDevice, s));
      ctx->h2d_bytes += n * 16;
      LC_TRY(upload_selection(ctx, sp, d_up + up_tab, s));
      PlannedRead pr{};
      pr.sel_base = reinterpret_cast<const uint32_t*>(d_up + up_tab);
      pr.sel_off = reinterpret_cast<const uint64_t*>(d_up);
      pr.k2 = reinterpret_cast<const uint32_t*>(d_up + n * 8);
      pr.cap_rows = rows;
      pr.cap_bytes = cap_bytes;
      pr.onepass = true;
      pr.scratch = d_plan;
      pr.d_values = d_val;
      pr.d_offsets = d_off;
      pr.d_hdr = d_hdr;
      LC_TRY(enqueue_planned_read(ctx, rl, n, pr));
      double& ratio = ctx->L()->onepass_bytes_per_row;
      const uint64_t spec = std::min<uint64_t>(cap_bytes, static_cast<uint64_t>(static_cast<double>(rows) * ratio * 1.25) + 4096);
      PlannedHost res;
      LC_TRY(download_planned(ctx, h_hdr, pr, 0, rows, spec, &res));
      tr.mark("one-pass read + its download");
      if (res.hdr.overflow || res.hdr.rows != rows) {  // cannot happen with an upper bound as the capacity: refuse rather than guess
        set_error("internal: one-pass read reported rows %llu (expected %llu), overflow %u", (unsigned long long)res.hdr.rows,
                  (unsigned long long)rows, res.hdr.overflow);
        return LC_ERR_INVALID;
      }
      ratio = std::max(8.0, static_cast<double>(res.values.bytes) / static_cast<double>(rows));
      return finish_bytes_array(proto, rows, 0, HostBlock{}, std::move(res.offsets), HostBlock{}, std::move(res.values), out_schema,
                                out_array);
    }
  }

  // ---------------- byte-view: pass 1 (lengths), host prefix sums, pass 2 (decode) ----------------
  uint64_t ulen_words = 0;
  std::vector<uint64_t> ulen_off(n);
  for (uint64_t i = 0; i < n; ++i) {
    ulen_off[i] = ulen_words;
    ulen_words += round_up((*rl->n_unique)[i], 4);
  }
  const uint64_t dv_rowoff = round_up((rows + n) * 4 + 16, 256);  // k_i + 1 per entry
  const uint64_t dv_rowkey = round_up(rows * 4 + 16, 256);
  const uint64_t dv_ulen = round_up(ulen_words * 4 + 16, 256);
  LC_TRY(sc.reserve(up_total + dn_total + dv_rowoff + dv_rowkey + dv_ulen + cat_bytes + 1024, up_total + dn_total + 1024));
  uint8_t* h_up = sc.host(up_total);
  uint8_t* h_dn = sc.host(dn_total);
  uint8_t* d_up = sc.dev(up_total);
  uint8_t* d_dn = sc.dev(dn_total);
  uint8_t* d_rowoff = sc.dev(dv_rowoff);
  uint8_t* d_rowkey = sc.dev(dv_rowkey);
  uint8_t* d_ulen = sc.dev(dv_ulen);
  uint8_t* d_cat = sc.dev(cat_bytes);
  if (!h_up || !h_dn || !d_up || !d_dn || !d_rowoff || !d_rowkey || !d_ulen || !d_cat) {
    set_error("to_arrow: scratch exhausted");
    return LC_ERR_OOM;
  }
  fill_offsets(h_up, &ulen_off);
  StrGatherIo g{};
  g.io = make_io(d_up, d_dn, nullptr);
  g.row_off_base = reinterpret_cast<uint32_t*>(d_rowoff);
  g.row_key_base = reinterpret_cast<uint32_t*>(d_rowkey);
  g.ulen_base = reinterpret_cast<uint32_t*>(d_ulen);
  g.row_base = reinterpret_cast<const uint64_t*>(d_up) + n;
  g.ulen_off = reinterpret_cast<const uint64_t*>(d_up) + 3 * n;
  g.byte_base = reinterpret_cast<const uint64_t*>(d_up) + 4 * n;
  g.dict_base = reinterpret_cast<const uint64_t*>(d_up) + 5 * n;
  LC_CUDA_OK(cudaMemcpyAsync(d_up, h_up, up_offs, cudaMemcpyHostToDevice, s));
  ctx->h2d_bytes += up_offs;
  if (!dev_sel) LC_TRY(upload_selection(ctx, sp, d_up + up_offs, s));
  tr.mark("fill + upload");
  LC_CUDA_OK(launch_str_lengths(static_cast<uint32_t>(n), g, rl->max_head, s));
  ctx->kernel_launches++;
  LC_CUDA_OK(cudaMemcpyAsync(h_dn, d_dn, dn_total, cudaMemcpyDeviceToHost, s));
  LC_CUDA_OK(cudaStreamSynchronize(s));
  tr.mark("lengths kernel + counts D2H");
  ctx->d2h_bytes += dn_total;
  const uint32_t* h_counts = reinterpret_cast<const uint32_t*>(h_dn);
  uint64_t nulls = 0, total_bytes = 0;
  uint64_t* h_byte_base = reinterpret_cast<uint64_t*>(h_up) + 4 * n;
  uint64_t* h_dict_base = reinterpret_cast<uint64_t*>(h_up) + 5 * n;  // adjacent: one upload carries both
  uint64_t dict_bytes = 0;
  constexpr uint64_t kDictScratchMax = 1ull << 30;
  for (uint64_t i = 0; i < n; ++i) {
    if (h_counts[4 * i] != sp.k[i]) {
      set_error("internal: selected-row count mismatch on entry %llu", (unsigned long long)i);
      return LC_ERR_INVALID;
    }
    nulls += h_counts[4 * i + 1];
    h_byte_base[i] = total_bytes;
    total_bytes += h_counts[4 * i + 2];
    // dense entries (as many rows selected as there are dictionary values, or more) decode their dictionary once
    const uint64_t ub = round_up(entries[i]->sh.uncompressed_bytes + 16, 256);
    if (sp.k[i] >= (*rl->n_unique)[i] && (*rl->n_unique)[i] > 0 && dict_bytes + ub <= kDictScratchMax) {
      h_dict_base[i] = dict_bytes;
      dict_bytes += ub;
    } else {
      h_dict_base[i] = ~0ull;
    }
  }
  if (total_bytes > 0x7fffffffull) {
    set_error("decoded values exceed 2 GiB (int32 offsets); split the call");
    return LC_ERR_INVALID;
  }
  if (dev_out && proto->fixed_width) {
    set_error("read_device: decimals outside u64 (LiquidFixedLenByteArray) are read through lc_to_arrow / lc_scan_read");
    return LC_ERR_UNSUPPORTED_TYPE;
  }
  if (dev_out) {
    if (dev_out->out_rows) *dev_out->out_rows = rows;
    if (dev_out->out_value_bytes) *dev_out->out_value_bytes = total_bytes;
    if (dev_out->out_null_count) *dev_out->out_null_count = nulls;
    if (!dev_out->d_values && !dev_out->d_offsets) return LC_OK;  // size query
    if (!dev_out->d_offsets || (total_bytes && !dev_out->d_values) || dev_out->values_cap < total_bytes) {
      set_error("read_device: need an offsets buffer of %llu int32 and %llu value bytes", (unsigned long long)(rows + 1),
                (unsigned long long)total_bytes);
      return LC_ERR_INVALID;
    }
    g.out_offsets = static_cast<int32_t*>(dev_out->d_offsets);
    g.out_bytes = static_cast<uint8_t*>(dev_out->d_values);
    // byte_base[n] and the closing offset travel from the pinned upload area (idle since the sync above)
    int32_t* h_last = reinterpret_cast<int32_t*>(h_up);  // sel_off[0] slot: no longer needed on the host
    *h_last = static_cast<int32_t>(total_bytes);
    uint8_t* d_dict = nullptr;
    if (dict_bytes && cudaMallocAsync(reinterpret_cast<void**>(&d_dict), dict_bytes, s) != cudaSuccess) {
      cudaGetLastError();
      d_dict = nullptr;  // no room for decoded dictionaries: every row decodes its own value
    }
    g.dict_scratch = d_dict;
    LC_CUDA_OK(cudaMemcpyAsync(d_up + 4 * n * 8, h_byte_base, 2 * n * 8, cudaMemcpyHostToDevice, s));
    LC_CUDA_OK(launch_str_decode(static_cast<uint32_t>(n), g, s));
    if (d_dict) cudaFreeAsync(d_dict, s);
    LC_CUDA_OK(cudaMemcpyAsync(g.out_offsets + rows, h_last, 4, cudaMemcpyHostToDevice, s));
    ctx->kernel_launches++;
    if (nulls && dev_out->d_validity) {
      const uint64_t* offs = reinterpret_cast<const uint64_t*>(d_up);
      LC_CUDA_OK(launch_concat_validity(g.io.valid_base, offs + 2 * n, offs + n, g.io.counts, 4, static_cast<uint32_t>(n), rows,
                                        static_cast<uint32_t*>(dev_out->d_validity), s));
      ctx->kernel_launches++;
    }
    LC_CUDA_OK(cudaStreamSynchronize(s));
    ctx->h2d_bytes += n * 8 + 4;
    return LC_OK;
  }
  const uint8_t bt = proto->sh.arrow_type;
  // Utf8View / BinaryView ship 16-byte views, LiquidFixedLenByteArray ships the values at their fixed stride: both are
  // built on the device from the decoded (offsets, bytes) and take the place of the offsets in the download
  const uint32_t fixed_w = proto->fixed_width;
  const bool want_views = bt == BT_UTF8_VIEW || bt == BT_BINARY_VIEW || fixed_w != 0;
  const uint64_t off_bytes = (rows + 1) * 4;
  const uint64_t view_bytes = fixed_w ? rows * fixed_w : want_views ? rows * 16 : 0;
  const uint64_t res_bytes = round_up(off_bytes, 256) + round_up(total_bytes + 16, 256) + round_up(view_bytes + 16, 256);
  uint8_t* d_res = nullptr;
  if (cudaMallocAsync(reinterpret_cast<void**>(&d_res), res_bytes, s) != cudaSuccess) {
    cudaGetLastError();
    set_error("cudaMallocAsync of %llu result bytes failed", (unsigned long long)res_bytes);
    return LC_ERR_OOM;
  }
  tr.mark("prefix sums + cudaMallocAsync");
  g.out_offsets = reinterpret_cast<int32_t*>(d_res);
  g.out_bytes = d_res + round_up(off_bytes, 256);
  uint8_t* d_views = g.out_bytes + round_up(total_bytes + 16, 256);
  // view types ship 16-byte views built on the device instead of the offsets
  HostBlock offsets = want_views ? HostBlock() : HostBlock(off_bytes, off_bytes);
  HostBlock views = want_views ? HostBlock(view_bytes + 16, view_bytes) : HostBlock();
  HostBlock data(total_bytes ? total_bytes : 1, total_bytes);
  HostBlock validity;
  if ((!want_views && !offsets.p) || (want_views && !views.p) || !data.p) {
    cudaFreeAsync(d_res, s);
    set_error("host allocation failed");
    return LC_ERR_OOM;
  }
  // second (small) upload: byte_base[n] and dict_base[n]
  uint8_t* d_dict = nullptr;
  if (dict_bytes && cudaMallocAsync(reinterpret_cast<void**>(&d_dict), dict_bytes, s) != cudaSuccess) {
    cudaGetLastError();
    d_dict = nullptr;  // no room for decoded dictionaries: every row decodes its own value
  }
  g.dict_scratch = d_dict;
  cudaError_t ce = cudaMemcpyAsync(d_up + 4 * n * 8, h_byte_base, 2 * n * 8, cudaMemcpyHostToDevice, s);
  if (ce == cudaSuccess) ce = launch_str_decode(static_cast<uint32_t>(n), g, s);
  if (d_dict) cudaFreeAsync(d_dict, s);
  int rc = LC_OK;
  if (ce == cudaSuccess && nulls) rc = concat_validity_device(g.io, d_up, d_cat, &validity);
  if (ce == cudaSuccess && rc == LC_OK && want_views) {
    ce = fixed_w ? launch_fixed_from_var(g.out_offsets, static_cast<uint32_t>(total_bytes), g.out_bytes,
                                         nulls ? reinterpret_cast<const uint32_t*>(d_cat) : nullptr, rows, fixed_w, d_views, s)
                 : launch_build_views(g.out_offsets, static_cast<uint32_t>(total_bytes), g.out_bytes,
                                      nulls ? reinterpret_cast<const uint32_t*>(d_cat) : nullptr, rows, d_views, s);
    ctx->kernel_launches++;
    if (ce == cudaSuccess && rows) ce = cudaMemcpyAsync(views.p, d_views, view_bytes, cudaMemcpyDeviceToHost, s);
  } else if (ce == cudaSuccess && rc == LC_OK && rows) {
    ce = cudaMemcpyAsync(offsets.p, g.out_offsets, rows * 4, cudaMemcpyDeviceToHost, s);
  }
  if (ce == cudaSuccess && rc == LC_OK && total_bytes && !fixed_w)
    ce = cudaMemcpyAsync(data.p, g.out_bytes, total_bytes, cudaMemcpyDeviceToHost, s);
  cudaFreeAsync(d_res, s);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);
  if (ce != cudaSuccess) {
    set_error("CUDA error in byte-view decode: %s", cudaGetErrorString(ce));
    return LC_ERR_CUDA;
  }
  LC_TRY(rc);
  tr.mark("decode kernel + result D2H");
  ctx->kernel_launches++;
  ctx->h2d_bytes += n * 8;
  ctx->d2h_bytes += (want_views ? view_bytes : rows * 4) + (fixed_w ? 0 : total_bytes);
  if (!want_views) reinterpret_cast<int32_t*>(offsets.p)[rows] = static_cast<int32_t>(total_bytes);
  return finish_bytes_array(proto, rows, nulls, std::move(validity), std::move(offsets), std::move(views), std::move(data), out_schema,
                            out_array);
}

// ---- get over a device-resident selection with ONE host synchronisation ----------------------------------------
// lc_scan_read used to cost three round trips: the survivor counts (to size everything), the decoded lengths (to size
// the bytes), the result. Here the two sizing steps are prefix sums on the device (k_scan_plan.cu) and the kernels run
// back to back against capacities taken from the previous read of the same scan; the host downloads a 64-byte header
// together with a speculative prefix of the result (again sized by the previous read) and only goes back for more when
// this read turned out larger. A capacity that is too small makes the kernels return at once (ScanPlanHdr.overflow) and
// the call falls back to the host-planned path, which also teaches the next call its sizes.
// Covers Utf8 / Binary byte views and plain integers without nulls; everything else takes the host-planned path.
int scan_read_fused(lc_ctx* ctx, FusedRead* fr, Entry* const* entries, uint64_t n, const uint32_t* d_sel, const uint64_t* d_word_off,
                    const uint32_t* d_counts2, uint64_t total_rows_in, ArrowSchema* out_schema, ArrowArray* out_array,
                    FusedDeviceOut* dev_out) {
  if (!fr->have_spec) return LC_INTERNAL_FALLBACK;
  const RefList* rl;
  LC_TRY(get_ref_list(ctx, entries, n, &rl));
  const Entry* proto = entries[0];
  if (!rl->same_liquid_type || !rl->same_arrow_type || rl->any_nulls || rl->any_fixed) return LC_INTERNAL_FALLBACK;
  const bool is_int = proto->liquid_type == LC_LIQUID_INTEGER;
  const bool is_str = proto->liquid_type == LC_LIQUID_BYTE_VIEW &&
                      (proto->sh.arrow_type == BT_UTF8 || proto->sh.arrow_type == BT_BINARY);
  if (!is_int && !is_str) return LC_INTERNAL_FALLBACK;
  if (is_int && !rl->same_width) return LC_INTERNAL_FALLBACK;
  // integers decode through the staged scan kernel, which reads every entry of the list: only worth it when a fair share
  // of the rows survives (the host-planned path reads just the batches with survivors)
  if (is_int && fr->spec_rows * 64 < total_rows_in) return LC_INTERNAL_FALLBACK;
  const uint32_t tb = is_int ? proto->ih.tbits / 8 : 0;
  cudaStream_t s = ctx->L()->stream;
  Tracer tr("scan_read_fused");

  PlannedRead pr{};
  pr.sel_base = d_sel;
  pr.sel_off = d_word_off;
  pr.k2 = d_counts2;
  pr.cap_rows = fr->spec_rows + fr->spec_rows / 2 + 4096;
  pr.cap_bytes = is_int ? pr.cap_rows * tb : fr->spec_bytes + fr->spec_bytes / 2 + (64u << 10);
  pr.cap_ulen = is_int ? 0 : fr->spec_ulen + fr->spec_ulen / 2 + (64u << 10);
  // the previous read of this scan left a handful of survivors per entry: one kernel does the whole read (k_str_read_onepass)
  pr.onepass = is_str && fr->spec_rows <= 8ull * n;
  // one device allocation, carved: the read's scratch | header | offsets | values (a borrowed result stays here)
  uint64_t o = planned_layout(n, is_str, pr.onepass, pr.cap_rows, pr.cap_ulen).bytes;
  const uint64_t o_hdr = carve(&o, 256);
  const uint64_t o_off = is_str ? carve(&o, (pr.cap_rows + 1) * 4) : 0;
  const uint64_t o_val = carve(&o, pr.cap_bytes + 16);
  LC_TRY(grow_device(s, &fr->d_buf, &fr->d_cap, o, o / 4));
  if (!fr->h_hdr && cudaHostAlloc(reinterpret_cast<void**>(&fr->h_hdr), 256, cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    return LC_INTERNAL_FALLBACK;
  }
  uint8_t* d = fr->d_buf;
  pr.scratch = d;
  pr.d_values = d + o_val;
  pr.d_offsets = is_str ? reinterpret_cast<int32_t*>(d + o_off) : nullptr;
  pr.d_hdr = reinterpret_cast<ScanPlanHdr*>(d + o_hdr);
  LC_TRY(enqueue_planned_read(ctx, rl, n, pr));
  tr.mark("launches");
  PlannedHost res;
  if (dev_out) {  // the result stays in the scan's device buffer (valid until the next read of this scan)
    LC_CUDA_OK(cudaMemcpyAsync(fr->h_hdr, pr.d_hdr, sizeof(ScanPlanHdr), cudaMemcpyDeviceToHost, s));
    LC_CUDA_OK(cudaStreamSynchronize(s));
    res.hdr = *fr->h_hdr;
    if (!res.hdr.overflow) ctx->d2h_bytes += sizeof(ScanPlanHdr);
  } else {
    const uint64_t spec_rows = fr->spec_rows + fr->spec_rows / 8 + 64;
    const uint64_t spec_bytes = is_int ? spec_rows * tb : fr->spec_bytes + fr->spec_bytes / 8 + 4096;
    LC_TRY(download_planned(ctx, fr->h_hdr, pr, tb, spec_rows, spec_bytes, &res));
  }
  tr.mark("download");
  if (res.hdr.overflow) {  // a capacity was short: the kernels did nothing; let the host-planned path answer and re-teach the sizes
    fr->have_spec = false;
    return LC_INTERNAL_FALLBACK;
  }
  const uint64_t rows = res.hdr.rows, bytes = is_int ? rows * tb : res.hdr.bytes;
  fr->spec_rows = rows;
  fr->spec_bytes = is_int ? 0 : bytes;
  if (!pr.onepass) fr->spec_ulen = res.hdr.ulen_words;  // the one-pass kernel uses no dictionary-length scratch: keep what the general path learnt
  if (dev_out) {
    dev_out->d_values = pr.d_values;
    dev_out->d_offsets = pr.d_offsets;
    dev_out->rows = rows;
    dev_out->value_bytes = bytes;
    return LC_OK;
  }
  export_schema(proto->arrow_format, "", out_schema);
  std::vector<HostBuf> bufs(1);  // no validity: the list has no nulls
  if (is_str) bufs.push_back(res.offsets.release());
  bufs.push_back(res.values.release());
  export_array(static_cast<int64_t>(rows), 0, std::move(bufs), nullptr, out_array);
  return LC_OK;
}

// The same device-planned read, FULLY ASYNCHRONOUS: the result lands in caller-owned device buffers of stated capacities
// and the 64-byte plan header (rows, bytes, overflow) in caller-owned device memory; nothing is downloaded and the stream is
// not synchronised. This is what a consumer on the device wants — the NCCL gather of every rank's filtered batch runs right
// behind it on the same stream and one tiny header download ends the step (bench.py, dist.py::DeviceGather).
int scan_read_async(lc_ctx* ctx, FusedRead* fr, Entry* const* entries, uint64_t n, const uint32_t* d_sel, const uint64_t* d_word_off,
                    const uint32_t* d_counts2, void* d_values, uint64_t values_cap, void* d_offsets, uint64_t rows_cap, void* d_header) {
  const RefList* rl;
  LC_TRY(get_ref_list(ctx, entries, n, &rl));
  const Entry* proto = entries[0];
  if (!rl->same_liquid_type || !rl->same_arrow_type || rl->any_nulls || rl->any_fixed) return LC_INTERNAL_FALLBACK;
  const bool is_int = proto->liquid_type == LC_LIQUID_INTEGER;
  const bool is_str = proto->liquid_type == LC_LIQUID_BYTE_VIEW &&
                      (proto->sh.arrow_type == BT_UTF8 || proto->sh.arrow_type == BT_BINARY);
  if ((!is_int && !is_str) || (is_int && !rl->same_width) || (is_str && !d_offsets) || !d_values || !d_header) return LC_INTERNAL_FALLBACK;
  const uint32_t tb = is_int ? proto->ih.tbits / 8 : 0;
  PlannedRead pr{};
  pr.sel_base = d_sel;
  pr.sel_off = d_word_off;
  pr.k2 = d_counts2;
  pr.cap_rows = is_int ? std::min<uint64_t>(rows_cap, values_cap / tb) : rows_cap;
  pr.cap_bytes = is_int ? 0 : std::min<uint64_t>(values_cap, 0x7fffffffull);
  // dictionary-length scratch: at most min(n, cap_rows) entries have survivors, each at most the list's largest dictionary
  pr.cap_ulen = is_int ? 0 : std::min<uint64_t>(n, pr.cap_rows) * round_up(rl->max_unique, 4);
  // A selective scan (the caller's row capacity says so: at most a handful of survivors per entry on average) is read by
  // ONE kernel — sizes, chained scan across its CTAs, decode (k_str_read_onepass) — instead of the general sequence.
  pr.onepass = is_str && rows_cap <= 16ull * n;
  const uint64_t o = planned_layout(n, is_str, pr.onepass, pr.cap_rows, pr.cap_ulen).bytes;
  LC_TRY(grow_device(ctx->L()->stream, &fr->a_buf, &fr->a_cap, o, o / 8));
  pr.scratch = fr->a_buf;
  pr.d_values = d_values;
  pr.d_offsets = is_str ? static_cast<int32_t*>(d_offsets) : nullptr;
  pr.d_hdr = static_cast<ScanPlanHdr*>(d_header);
  return enqueue_planned_read(ctx, rl, n, pr);
}

void fused_read_learn(FusedRead* fr, const ArrowArray* arr, int64_t value_bytes, uint64_t ulen_words) {
  fr->spec_rows = static_cast<uint64_t>(arr->length);
  fr->spec_bytes = value_bytes > 0 ? static_cast<uint64_t>(value_bytes) : 0;
  fr->spec_ulen = std::max<uint64_t>(fr->spec_ulen, ulen_words);
  fr->have_spec = true;
}

void fused_read_free(FusedRead* fr) {
  if (fr->a_buf) cudaFree(fr->a_buf);
  if (fr->d_buf) cudaFree(fr->d_buf);
  if (fr->h_hdr) cudaFreeHost(fr->h_hdr);
  *fr = FusedRead();
}

// Turn (validity, int32 offsets, bytes) into the ORIGINAL arrow type of the column:
// Utf8 / Binary as is; Utf8View / BinaryView by building 16-byte views over the single data buffer;
// Dictionary<UInt16,_> by re-encoding (what arrow's cast dictionary -> original type leaves the caller with,
// byte_view_array/mod.rs:287-290).
static int finish_bytes_array(const Entry* proto, uint64_t rows, uint64_t nulls, HostBlock validity, HostBlock offsets,
                              HostBlock views, HostBlock data, ArrowSchema* out_schema, ArrowArray* out_array) {
  const uint8_t bt = proto->sh.arrow_type;
  const int32_t* off = reinterpret_cast<const int32_t*>(offsets.p);
  if (bt == BT_DECIMAL128 || bt == BT_DECIMAL256) {
    // LiquidFixedLenByteArray::to_arrow_array (fix_len_byte_array.rs:87-95): the decimal array itself; `views` holds the
    // values at their fixed stride (null slots zero)
    export_schema(proto->arrow_format, "", out_schema);
    std::vector<HostBuf> bufs{validity.release(), views.release()};
    export_array(static_cast<int64_t>(rows), static_cast<int64_t>(nulls), std::move(bufs), nullptr, out_array);
    return LC_OK;
  }
  if (bt == BT_UTF8 || bt == BT_BINARY) {
    export_schema(bt == BT_UTF8 ? "u" : "z", "", out_schema);
    std::vector<HostBuf> bufs{validity.release(), offsets.release(), data.release()};
    export_array(static_cast<int64_t>(rows), static_cast<int64_t>(nulls), std::move(bufs), nullptr, out_array);
    return LC_OK;
  }
  if (bt == BT_UTF8_VIEW || bt == BT_BINARY_VIEW) {
    // the views came off the device (k_build_views); only the variadic-sizes buffer is made here
    HostBlock sizes(8, 8);
    if (!sizes.p) {
      set_error("host allocation failed");
      return LC_ERR_OOM;
    }
    const int64_t sz = static_cast<int64_t>(data.bytes);
    std::memcpy(sizes.p, &sz, 8);
    export_schema(bt == BT_UTF8_VIEW ? "vu" : "vz", "", out_schema);
    std::vector<HostBuf> bufs{validity.release(), views.release(), data.release(), sizes.release()};
    export_array(static_cast<int64_t>(rows), static_cast<int64_t>(nulls), std::move(bufs), nullptr, out_array);
    return LC_OK;
  }
  // Dictionary<UInt16, Utf8|Binary>: first-occurrence re-encode of the decoded rows
  std::unordered_map<std::string, uint16_t> seen;
  std::vector<std::string> order;
  HostBlock keys(rows * 2 + 2, rows * 2);
  if (!keys.p) {
    set_error("host allocation failed");
    return LC_ERR_OOM;
  }
  std::memset(keys.p, 0, rows * 2 + 2);
  for (uint64_t r = 0; r < rows; ++r) {
    const bool ok = !validity.p || bit_get(validity.p, static_cast<int64_t>(r));
    if (!ok) continue;
    std::string sv(reinterpret_cast<const char*>(data.p) + off[r], static_cast<size_t>(off[r + 1] - off[r]));
    auto it = seen.find(sv);
    uint16_t key;
    if (it == seen.end()) {
      if (order.size() >= 65536) {
        set_error("more than 65536 distinct values in a dictionary result");
        return LC_ERR_UNSUPPORTED_TYPE;
      }
      key = static_cast<uint16_t>(order.size());
      seen.emplace(sv, key);
      order.push_back(std::move(sv));
    } else {
      key = it->second;
    }
    reinterpret_cast<uint16_t*>(keys.p)[r] = key;
  }
  uint64_t dbytes = 0;
  for (auto& sv : order) dbytes += sv.size();
  HostBlock doff((order.size() + 1) * 4, (order.size() + 1) * 4);
  HostBlock ddata(dbytes ? dbytes : 1, dbytes);
  if (!doff.p || !ddata.p) {
    set_error("host allocation failed");
    return LC_ERR_OOM;
  }
  int32_t* dof = reinterpret_cast<int32_t*>(doff.p);
  uint64_t p = 0;
  for (size_t i = 0; i < order.size(); ++i) {
    dof[i] = static_cast<int32_t>(p);
    std::memcpy(ddata.p + p, order[i].data(), order[i].size());
    p += order[i].size();
  }
  dof[order.size()] = static_cast<int32_t>(p);
  ArrowArray dict_arr;
  std::vector<HostBuf> dbufs{HostBuf{nullptr, 0}, doff.release(), ddata.release()};
  export_array(static_cast<int64_t>(order.size()), 0, std::move(dbufs), nullptr, &dict_arr);
  export_schema("S", bt == BT_DICT16_UTF8 ? "u" : "z", out_schema);
  std::vector<HostBuf> bufs{validity.release(), keys.release()};
  export_array(static_cast<int64_t>(rows), static_cast<int64_t>(nulls), std::move(bufs), &dict_arr, out_array);
  return LC_OK;
}

}  // namespace lc

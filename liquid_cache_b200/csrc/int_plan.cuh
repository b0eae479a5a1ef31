// int_plan.cuh — how `col <op> literal` becomes a test on the unsigned PACKED value of an integer entry: the planner and the
// range form every scan loop of k_int.cu evaluates. Host + device, so that the same code is exercised on the CPU against
// plain comparisons and the squeezed-array oracle (tests/cpp/int_plan_host.cc, tests/test_int_plan_cpu.py).
#pragma once
#include <cstdint>

#include "entry_layout.h"
#include "kernels.h"

#ifdef __CUDACC__
#define LC_PL_HD __host__ __device__ __forceinline__
#else
#define LC_PL_HD inline
#endif

namespace lc {

// Every comparison of the unsigned packed value against the threshold is one range test:
//   cmp(u) = ((u - lo) <= span) != neg
template <typename C>
struct URange {
  C lo, span;
  bool neg;
};

template <typename C>
LC_PL_HD URange<C> make_range(int32_t kind, uint64_t thr64) {
  const C mx = static_cast<C>(~static_cast<C>(0));
  const C thr = static_cast<C>(thr64);
  URange<C> g;
  g.lo = 0;
  g.span = mx;
  g.neg = false;
  switch (kind) {
    case UC_FALSE: g.neg = true; break;
    case UC_TRUE: break;
    case UC_EQ: g.lo = thr; g.span = 0; break;
    case UC_NE: g.lo = thr; g.span = 0; g.neg = true; break;
    case UC_LT: if (thr == 0) g.neg = true; else g.span = static_cast<C>(thr - 1); break;
    case UC_LE: g.span = thr; break;
    case UC_GT: if (thr == mx) g.neg = true; else { g.lo = static_cast<C>(thr + 1); g.span = static_cast<C>(mx - g.lo); } break;
    default: g.lo = thr; g.span = static_cast<C>(mx - thr); break;
  }
  return g;
}

// Where one literal lies against the window of an entry. All valid values satisfy reference <= v <= reference + umax
// (umax = 2^W - 1) in the column's own ordering: -1 below the window, +1 above it, 0 inside with *d = literal - reference.
// No 128-bit arithmetic needed: once lit >= reference is known, (lit - reference) fits in 64 unsigned bits.
LC_PL_HD int lit_window(const IntHeader* h, uint64_t umax, int32_t lit_kind, int64_t lit_i, uint64_t lit_u, uint64_t* d) {
  *d = 0;
  if (lit_kind == kLitAboveAll) return 1;  // decimal literal beyond u64::MAX (scan_host.cc make_int_pred)
  if (h->is_signed) {
    const int sh = 64 - h->tbits;
    const long long ref = static_cast<long long>(h->reference << sh) >> sh;
    if (lit_kind == 1 /*U64*/ && lit_u > 0x7fffffffffffffffull) return 1;
    const long long lit = lit_kind == 1 ? static_cast<long long>(lit_u) : lit_i;
    if (lit < ref) return -1;
    *d = static_cast<uint64_t>(lit) - static_cast<uint64_t>(ref);
    return *d > umax ? 1 : 0;
  }
  const uint64_t ref = h->reference;
  if (lit_kind == 0 /*I64*/ && lit_i < 0) return -1;
  const uint64_t lit = lit_kind == 0 ? static_cast<uint64_t>(lit_i) : lit_u;
  if (lit < ref) return -1;
  *d = lit - ref;
  return *d > umax ? 1 : 0;
}

LC_PL_HD uint64_t window_umax(const IntHeader* h) {
  const uint32_t W = h->bit_width;
  return W == 64 ? ~0ull : ((1ull << W) - 1ull);
}

// The entry's reference as a 64-bit pattern of the column's domain (signed references are stored in their own width):
// the packed offset of an in-window list value v is v - window_ref(h), modulo 2^64.
LC_PL_HD uint64_t window_ref(const IntHeader* h) {
  if (!h->is_signed) return h->reference;
  const int sh = 64 - h->tbits;
  return static_cast<uint64_t>(static_cast<long long>(h->reference << sh) >> sh);
}

// (op, literal) -> compare in the unsigned packed domain u = v - reference: a literal outside the window folds to a
// constant and one inside becomes an unsigned threshold.
LC_PL_HD void plan_int_pred(const IntHeader* h, const IntPredDesc& p, int32_t* ucmp, uint64_t* thr) {
  *thr = 0;
  if (h->bit_width == 0) {  // all null: values never matter
    *ucmp = UC_FALSE;
    return;
  }
  const uint64_t umax = window_umax(h);
  if (p.lit_kind == kLitSentinel) {  // which rows of a clamped entry sit at the sentinel (squeeze_host.cc)
    *thr = umax;
    *ucmp = UC_EQ;
    return;
  }
  uint64_t d = 0;
  const int where = lit_window(h, umax, p.lit_kind, p.lit_i, p.lit_u, &d);
  bool below = where < 0, above = where > 0;
  if (h->squeeze_kind == 2 && !below && p.lit_kind != kLitAboveAll) {
    // quantized entry (hybrid_primitive_array.rs:564-650): the words are bucket indices b = offset / bucket_width; compare
    // them with the literal's bucket q. b < q / b > q are the operator's two sides, exactly what `b <op> q` gives; inside
    // bucket q the same expression is right whenever the host let the call through (the literal sits on the bucket edge
    // that decides the operator, or no selected row is in bucket q — squeeze_host.cc checks that first with `= literal`,
    // which lands here as b == q).
    d = d / int_bucket_width(*h);  // d was the literal's offset from the reference
    above = d > umax;              // (the test above compared that offset with the code range: redo it for the bucket)
  }
  const int op = p.op;
  if (below) {
    *ucmp = (op == 1 || op == 4 || op == 5) ? UC_TRUE : UC_FALSE;  // NE, GT, GE
  } else if (above) {
    *ucmp = (op == 1 || op == 2 || op == 3) ? UC_TRUE : UC_FALSE;  // NE, LT, LE
  } else {
    *thr = d;
    *ucmp = op == 0 ? UC_EQ : op == 1 ? UC_NE : op == 2 ? UC_LT : op == 3 ? UC_LE : op == 4 ? UC_GT : UC_GE;
  }
}

// `col [NOT] IN (list)` on one (full, not squeezed) entry. p.v is sorted in the column's order without duplicates, so
// the values inside the entry's window are one slice [a, b) of it and their packed offsets v - window_ref ascend.
LC_PL_HD int in_value_window(const IntHeader* h, uint64_t v) {
  uint64_t d = 0;
  return lit_window(h, window_umax(h), h->is_signed ? 0 : 1, static_cast<int64_t>(v), v, &d);
}

// The slice by two binary searches (k_int_bits counts the same two numbers with a warp vote instead).
LC_PL_HD void in_window_slice(const IntHeader* h, const IntInList& p, uint32_t* a, uint32_t* b) {
  uint32_t lo = 0, hi = p.n;  // first value not below the window
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (in_value_window(h, p.v[mid]) < 0) lo = mid + 1u;
    else hi = mid;
  }
  *a = lo;
  hi = p.n;  // first value above the window
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (in_value_window(h, p.v[mid]) <= 0) lo = mid + 1u;
    else hi = mid;
  }
  *b = lo;
}

// The slice [a, b) lowers to
//   empty                         -> a constant (false for IN, true for NOT IN)
//   one value / consecutive run   -> the range test of `=` / `BETWEEN`, so those lists cost what the comparison costs
//   anything else                 -> a set test over the slice: returns true, g->neg says NOT IN, lo / span are unused
template <typename C>
LC_PL_HD bool lower_in_slice(const IntHeader* h, int32_t op, const IntInList& p, uint32_t a, uint32_t b, URange<C>* g) {
  const bool neg = op == kOpNotIn;
  if (h->bit_width == 0 || a == b) {  // all null (the rows are null whatever the list says) / nothing in the window
    *g = make_range<C>((neg && h->bit_width != 0) ? UC_TRUE : UC_FALSE, 0);
    return false;
  }
  const uint64_t ref = window_ref(h);
  const uint64_t d0 = p.v[a] - ref, d1 = p.v[b - 1u] - ref;
  g->lo = static_cast<C>(d0);
  g->span = static_cast<C>(d1 - d0);
  g->neg = neg;
  return d1 - d0 != static_cast<uint64_t>(b - 1u - a);  // distinct ascending values: consecutive iff the span is the count
}

template <typename C>
LC_PL_HD bool plan_int_in(const IntHeader* h, int32_t op, const IntInList& p, URange<C>* g, uint32_t* a, uint32_t* b) {
  *a = *b = 0;
  if (h->bit_width != 0) in_window_slice(h, p, a, b);
  return lower_in_slice<C>(h, op, p, *a, *b, g);
}

// The set test of plan_int_in: is the packed value u one of the n ascending offsets s[0..n)? (lower bound by halving)
template <typename C, typename Get>
LC_PL_HD bool in_sorted(C u, uint32_t n, Get s) {
  uint32_t lo = 0, len = n;
  while (len > 0) {
    const uint32_t half = len >> 1;
    if (s(lo + half) < u) {
      lo += half + 1u;
      len -= half + 1u;
    } else {
      len = half;
    }
  }
  return lo < n && s(lo) == u;
}

}  // namespace lc

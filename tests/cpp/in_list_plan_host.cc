// The IN-list planner of the integer kernels (liquid_cache_b200/csrc/int_plan.cuh: plan_int_in + in_sorted) compiled for
// the HOST: given an entry header and a sorted, duplicate-free list in the column's domain, which of a list of packed
// values are members — evaluated as k_int_bits / k_int_scan do (range test, or lookup among the slice's packed offsets).
// Checked against brute-force membership in tests/test_in_list_cpu.py.
#include <cstdint>
#include <cstring>

#include "liquid_cache_b200/csrc/int_plan.cuh"

extern "C" {

// header: tbits, bit_width, is_signed, reference (raw bits); list[n_list] sorted in the column's order; negated: NOT IN.
// packed[n] -> out[n] (0 / 1). Returns 0 constant, 1 range, 2 set; *a, *b the slice of the list inside the window.
int ilp_eval(uint32_t tbits, uint32_t bit_width, uint32_t is_signed, uint64_t reference, const uint64_t* list, uint32_t n_list,
             int32_t negated, const uint64_t* packed, uint32_t n, uint8_t* out, uint32_t* a_out, uint32_t* b_out) {
  lc::IntHeader h;
  std::memset(&h, 0, sizeof(h));
  h.tbits = static_cast<uint8_t>(tbits);
  h.bit_width = static_cast<uint8_t>(bit_width);
  h.is_signed = is_signed;
  h.reference = reference;
  const lc::IntInList in{list, n_list, 0};
  const int32_t op = negated ? lc::kOpNotIn : lc::kOpIn;
  uint32_t a = 0, b = 0;
  int shape;
  const uint64_t ref = lc::window_ref(&h);
  if (bit_width <= 32) {  // k_int_bits: 32-bit packed domain
    lc::URange<uint32_t> g;
    const bool set = lc::plan_int_in<uint32_t>(&h, op, in, &g, &a, &b);
    shape = set ? 2 : (a == b ? 0 : 1);
    for (uint32_t i = 0; i < n; ++i) {
      const uint32_t u = static_cast<uint32_t>(packed[i]);
      const bool hit = set ? lc::in_sorted<uint32_t>(u, b - a, [&](uint32_t k) { return static_cast<uint32_t>(list[a + k] - ref); })
                           : (u - g.lo) <= g.span;
      out[i] = (hit != g.neg) ? 1 : 0;
    }
  } else {  // k_int_scan: 64-bit packed domain
    lc::URange<uint64_t> g;
    const bool set = lc::plan_int_in<uint64_t>(&h, op, in, &g, &a, &b);
    shape = set ? 2 : (a == b ? 0 : 1);
    for (uint32_t i = 0; i < n; ++i) {
      const uint64_t u = packed[i];
      const bool hit = set ? lc::in_sorted<uint64_t>(u, b - a, [&](uint32_t k) { return list[a + k] - ref; }) : (u - g.lo) <= g.span;
      out[i] = (hit != g.neg) ? 1 : 0;
    }
  }
  *a_out = a;
  *b_out = b;
  return shape;
}
}

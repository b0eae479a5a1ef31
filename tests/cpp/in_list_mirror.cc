// `col [NOT] IN (list)` through the C++ mirror of the front door (liquid_cache_b200/csrc/liquid_cache.hpp): one integer
// and one string IN list, with a copied expression that must carry its own list. Exit codes as tests/cpp/quickstart.cc:
// 0 all answers right, 3 no CUDA device, 1 a wrong answer.
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "liquid_cache_b200/csrc/liquid_cache.hpp"

namespace lc = liquid_cache;

namespace {

struct Owned {
  std::vector<const void*> bufs;
  std::vector<uint8_t> validity, data;
  std::vector<int32_t> offsets;
  std::string format;
};
void release_schema(ArrowSchema* s) {
  delete static_cast<Owned*>(s->private_data);
  s->release = nullptr;
}
void release_array(ArrowArray* a) {
  delete static_cast<Owned*>(a->private_data);
  a->release = nullptr;
}
void make_schema(const char* format, ArrowSchema* out) {
  Owned* o = new Owned();
  o->format = format;
  std::memset(out, 0, sizeof(*out));
  out->format = o->format.c_str();
  out->name = "";
  out->flags = ARROW_FLAG_NULLABLE;
  out->release = release_schema;
  out->private_data = o;
}
void make_i32(const std::vector<int32_t>& v, ArrowSchema* s, ArrowArray* a) {
  make_schema("i", s);
  Owned* o = new Owned();
  o->data.resize(v.size() * 4);
  std::memcpy(o->data.data(), v.data(), o->data.size());
  o->bufs = {nullptr, o->data.data()};
  std::memset(a, 0, sizeof(*a));
  a->length = static_cast<int64_t>(v.size());
  a->n_buffers = 2;
  a->buffers = o->bufs.data();
  a->release = release_array;
  a->private_data = o;
}
void make_utf8(const std::vector<const char*>& v, ArrowSchema* s, ArrowArray* a) {  // nullptr = NULL
  make_schema("u", s);
  Owned* o = new Owned();
  o->validity.assign((v.size() + 7) / 8, 0);
  o->offsets.push_back(0);
  int64_t nulls = 0;
  for (size_t i = 0; i < v.size(); ++i) {
    if (v[i]) {
      o->validity[i / 8] |= static_cast<uint8_t>(1u << (i % 8));
      o->data.insert(o->data.end(), v[i], v[i] + std::strlen(v[i]));
    } else {
      ++nulls;
    }
    o->offsets.push_back(static_cast<int32_t>(o->data.size()));
  }
  o->bufs = {nulls ? o->validity.data() : nullptr, o->offsets.data(), o->data.data()};
  std::memset(a, 0, sizeof(*a));
  a->length = static_cast<int64_t>(v.size());
  a->null_count = nulls;
  a->n_buffers = 3;
  a->buffers = o->bufs.data();
  a->release = release_array;
  a->private_data = o;
}
std::string mask_string(const lc::BooleanArray& m) {  // 'T' / 'F' / 'N' per row
  std::string s;
  for (uint64_t i = 0; i < m.len; ++i) {
    const bool valid = m.null_count == 0 || ((m.validity[i / 8] >> (i % 8)) & 1);
    s += !valid ? 'N' : ((m.values[i / 8] >> (i % 8)) & 1) ? 'T' : 'F';
  }
  return s;
}
int failures = 0;
void expect(bool ok, const char* what) {
  if (!ok) {
    std::fprintf(stderr, "WRONG: %s\n", what);
    ++failures;
  }
}

}  // namespace

int main() {
  std::unique_ptr<lc::LiquidCache> cache;
  try {
    cache.reset(lc::LiquidCacheBuilder().with_batch_size(8192).build());
  } catch (const lc::GpuError& e) {
    std::fprintf(stderr, "no device: %s\n", e.what());
    return 3;
  }
  try {
    ArrowSchema s;
    ArrowArray a;
    make_i32({-1, 6, 3, 6, -7, 100}, &s, &a);
    cache->insert(1, &s, &a).run();
    a.release(&a);
    s.release(&s);
    lc::BooleanArray mask;
    lc::LiquidExpr in = lc::LiquidExpr::in_list_i64({6, -1, 42});
    lc::LiquidExpr copy = in;  // the copy owns its own list
    in = lc::LiquidExpr::in_list_i64({100});
    expect(cache->eval_predicate(1, copy).read(&mask) && mask_string(mask) == "TTFTFF", "int32 IN (6, -1, 42)");
    expect(cache->eval_predicate(1, lc::LiquidExpr::in_list_i64({6, -1, 42}, true)).read(&mask) && mask_string(mask) == "FFTFTT",
           "int32 NOT IN (6, -1, 42)");

    make_utf8({"MAIL", "SHIP", nullptr, "AIR", "TRUCK", "MAIL"}, &s, &a);
    cache->insert(2, &s, &a).run();
    a.release(&a);
    s.release(&s);
    expect(cache->eval_predicate(2, lc::LiquidExpr::in_list_bytes({"MAIL", "SHIP"})).read(&mask) && mask_string(mask) == "TTNFFT",
           "l_shipmode IN ('MAIL', 'SHIP')");
    expect(cache->eval_predicate(2, lc::LiquidExpr::in_list_bytes({"MAIL", "SHIP"}, true)).read(&mask) && mask_string(mask) == "FFNTTF",
           "l_shipmode NOT IN ('MAIL', 'SHIP')");
    std::printf("cpp in_list: %d wrong answers\n", failures);
  } catch (const std::exception& e) {
    std::fprintf(stderr, "exception: %s\n", e.what());
    return 1;
  }
  return failures ? 1 : 0;
}

/* lc_scan_filter_or through the C header alone (plain C11): the reference's three-column OR (a = 2 OR b = 40 OR c = 600)
 * and a DNF with an AND group, on one 8-row batch. Exit codes as tests/cpp/quickstart.cc: 0 all answers right, 3 no CUDA
 * device, 1 a wrong answer. */
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "include/lc_gpu.h"

static void no_release_schema(struct ArrowSchema* s) { s->release = NULL; }
static void no_release_array(struct ArrowArray* a) { a->release = NULL; }

static int encode_i32(lc_ctx* ctx, const int32_t* v, int64_t n, lc_handle* out) {
  static const void* bufs[2];
  struct ArrowSchema s;
  struct ArrowArray a;
  memset(&s, 0, sizeof(s));
  memset(&a, 0, sizeof(a));
  s.format = "i";
  s.name = "";
  s.flags = ARROW_FLAG_NULLABLE;
  s.release = no_release_schema;
  bufs[0] = NULL;
  bufs[1] = v;
  a.length = n;
  a.n_buffers = 2;
  a.buffers = bufs;
  a.release = no_release_array;
  return lc_encode(ctx, &s, &a, LC_HINT_NONE, 0, out);
}

static lc_predicate int_pred(int32_t op, int64_t v) {
  lc_predicate p;
  memset(&p, 0, sizeof(p));
  p.op = op;
  p.lit_kind = LC_LIT_I64;
  p.lit_i64 = v;
  return p;
}

static int failures = 0;

static void expect_rc(int rc, int want, const char* what) {
  if (rc != want) {
    fprintf(stderr, "WRONG: %s returned %d (%s)\n", what, rc, lc_last_error());
    ++failures;
  }
}

/* the selection of the scan's only batch as a bit string, and its count */
static void expect_rows(lc_scan* scan, const char* want, const char* what) {
  uint8_t bits[8] = {0};
  uint64_t count = 0, total = 0;
  char got[9];
  int i;
  if (lc_scan_selection(scan, 0, bits) != LC_OK || lc_scan_counts(scan, &count, &total) != LC_OK) {
    fprintf(stderr, "WRONG: %s: %s\n", what, lc_last_error());
    ++failures;
    return;
  }
  for (i = 0; i < 8; ++i) got[i] = ((bits[0] >> i) & 1) ? '1' : '0';
  got[8] = '\0';
  uint64_t want_count = 0;
  for (i = 0; i < 8; ++i) want_count += want[i] == '1';
  if (strcmp(got, want) != 0 || count != want_count || total != want_count) {
    fprintf(stderr, "WRONG: %s: got %s (%llu) want %s\n", what, got, (unsigned long long)count, want);
    ++failures;
  }
}

int main(void) {
  lc_ctx* ctx = NULL;
  if (lc_ctx_create(0, 0, &ctx) != LC_OK) {
    fprintf(stderr, "no device: %s\n", lc_last_error());
    return 3;
  }
  const int32_t a[8] = {1, 2, 3, 4, 5, 6, 7, 8};
  const int32_t b[8] = {10, 20, 30, 40, 50, 60, 70, 80};
  const int32_t c[8] = {100, 200, 300, 400, 500, 600, 700, 800};
  lc_handle ha, hb, hc;
  if (encode_i32(ctx, a, 8, &ha) != LC_OK || encode_i32(ctx, b, 8, &hb) != LC_OK || encode_i32(ctx, c, 8, &hc) != LC_OK) {
    fprintf(stderr, "encode: %s\n", lc_last_error());
    return 1;
  }
  const uint64_t rows = 8;
  lc_scan* scan = NULL;
  if (lc_scan_begin(ctx, 1, &rows, &scan) != LC_OK) {
    fprintf(stderr, "scan: %s\n", lc_last_error());
    return 1;
  }
  /* evaluate_three_column_or: a = 2 OR b = 40 OR c = 600 -> rows 1, 3, 5 */
  const lc_handle* terms[3] = {&ha, &hb, &hc};
  lc_predicate preds[3] = {int_pred(LC_OP_EQ, 2), int_pred(LC_OP_EQ, 40), int_pred(LC_OP_EQ, 600)};
  expect_rc(lc_scan_filter_or(scan, 3, terms, preds, NULL), LC_OK, "three-column OR");
  expect_rows(scan, "01010100", "a = 2 OR b = 40 OR c = 600");
  /* (a >= 2 AND a <= 4) OR b = 80 -> rows 1, 2, 3, 7 */
  lc_scan_reset(scan);
  const lc_handle* dnf_terms[3] = {&ha, &ha, &hb};
  lc_predicate dnf[3] = {int_pred(LC_OP_GE, 2), int_pred(LC_OP_LE, 4), int_pred(LC_OP_EQ, 80)};
  const uint32_t group[3] = {0, 0, 1};
  expect_rc(lc_scan_filter_or(scan, 3, dnf_terms, dnf, group), LC_OK, "DNF");
  expect_rows(scan, "01110001", "(a >= 2 AND a <= 4) OR b = 80");
  /* a malformed group is refused and leaves the selection as it was */
  const uint32_t bad_group[3] = {0, 2, 2};
  expect_rc(lc_scan_filter_or(scan, 3, dnf_terms, dnf, bad_group), LC_ERR_INVALID, "a malformed group");
  expect_rows(scan, "01110001", "after a refused call");
  lc_scan_end(scan);
  lc_release(ctx, ha);
  lc_release(ctx, hb);
  lc_release(ctx, hc);
  lc_ctx_destroy(ctx);
  printf("c scan_or: %d wrong answers\n", failures);
  return failures ? 1 : 0;
}

// sortkey.cuh — the normalised sort key (sort.cu): one definition of row order and equality, shared by the sort, the merge
// and the window boundaries (window.cu).
#pragma once
#include "common.cuh"

namespace b2 {

constexpr int SORT_MAX_KEYS = 16;
struct SortCol {
  const void* data;
  const uint32_t* valid;
  const int32_t* offsets;
  int32_t dtype, width;
  int32_t ascending, nulls_first;
  int32_t key_off;    // first byte of this column inside the row key
  int32_t key_len;    // bytes (null byte included)
  int32_t has_null_byte;
  int32_t str_max;    // strings: padded length
};
struct SortPlan {
  int32_t ncols;
  int32_t key_bytes;
  SortCol c[SORT_MAX_KEYS];
};

// byte `b` (0 = most significant) of column c's normalised key for `row`
__device__ __forceinline__ uint32_t norm_byte(const SortCol& c, int64_t row, int b) {
  const bool valid = row_valid(c.valid, row);
  uint32_t out;
  if (c.has_null_byte && b == 0) {
    // nulls_first: null -> 0, valid -> 1 ; nulls_last: null -> 1, valid -> 0   (not affected by desc)
    return valid ? (c.nulls_first ? 1u : 0u) : (c.nulls_first ? 0u : 1u);
  }
  if (!valid) return 0;
  const int vb = b - c.has_null_byte;  // byte inside the value part
  if (c.dtype == B2_STRING) {
    const int32_t s = c.offsets[row], len = c.offsets[row + 1] - s;
    if (vb < c.str_max) out = vb < len ? reinterpret_cast<const uint8_t*>(c.data)[s + vb] : 0u;
    else out = ((uint32_t)len >> (8 * (3 - (vb - c.str_max)))) & 255u;  // 4-byte big-endian length tiebreak
  } else if (c.width == 16) {
    const uint64_t* p = reinterpret_cast<const uint64_t*>(c.data) + 2 * row;
    uint64_t hi = p[1] ^ 0x8000000000000000ull, lo = p[0];
    out = vb < 8 ? (uint32_t)(hi >> (8 * (7 - vb))) & 255u : (uint32_t)(lo >> (8 * (15 - vb))) & 255u;
  } else {
    uint64_t u;
    switch (c.dtype) {
      case B2_FLOAT32: {
        float f = reinterpret_cast<const float*>(c.data)[row];
        uint32_t x = (f != f) ? 0x7fc00000u : (f == 0.0f ? 0u : __float_as_uint(f));
        x = (x & 0x80000000u) ? ~x : (x | 0x80000000u);
        u = x;
      } break;
      case B2_FLOAT64: {
        double d = reinterpret_cast<const double*>(c.data)[row];
        uint64_t x = (d != d) ? 0x7ff8000000000000ull : (d == 0.0 ? 0ull : (uint64_t)__double_as_longlong(d));
        u = (x & 0x8000000000000000ull) ? ~x : (x | 0x8000000000000000ull);
      } break;
      default:
        switch (c.width) {
          case 1: u = (uint8_t)(reinterpret_cast<const uint8_t*>(c.data)[row] ^ 0x80u); break;
          case 2: u = (uint16_t)(reinterpret_cast<const uint16_t*>(c.data)[row] ^ 0x8000u); break;
          case 4: u = reinterpret_cast<const uint32_t*>(c.data)[row] ^ 0x80000000u; break;
          default: u = reinterpret_cast<const uint64_t*>(c.data)[row] ^ 0x8000000000000000ull; break;
        }
    }
    out = (uint32_t)(u >> (8 * (c.width - 1 - vb))) & 255u;
  }
  return c.ascending ? out : (out ^ 255u);
}

// bytes [8*chunk, 8*chunk+8) of the row key of `row` (byte 8*chunk most significant)
__device__ __forceinline__ uint64_t key_chunk(const SortPlan& plan, int64_t row, int chunk) {
  uint64_t k = 0;
  const int b0 = chunk * 8;
  for (int ci = 0; ci < plan.ncols; ci++) {
    const SortCol& c = plan.c[ci];
    const int lo = max(b0, c.key_off), hi = min(b0 + 8, c.key_off + c.key_len);
    for (int b = lo; b < hi; b++) k |= (uint64_t)norm_byte(c, row, b - c.key_off) << (8 * (7 - (b - b0)));
  }
  return k;
}

SortPlan make_sort_plan(const Table* t, const b2_order_by_arg* keys, int nkeys, bool force_null_byte = false, const int32_t* str_max = nullptr);
std::vector<SortPlan> shared_sort_plans(const std::vector<const Table*>& ts, const b2_order_by_arg* keys, int nkeys);

}  // namespace b2

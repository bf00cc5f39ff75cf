// crb_grid_common.cuh — device code shared by the grid planners' kernels (crb_grid.cu: one map; crb_grid_many.cu: a
// map per query): the motion model, the restated libstdc++ heap and the reference's rounding of points to cells.  See
// crb_grid.cu for what each piece restates.
#pragma once

#include <float.h>

#include "crb_common.cuh"

namespace {

// get_motion_model :99-108, in its order; the diagonal cost is (float)std::sqrt(2)
__constant__ int c_mx[8] = {1, 0, -1, 0, -1, -1, 1, 1};
__constant__ int c_my[8] = {0, 1, 0, -1, -1, 1, -1, 1};
constexpr float kDiag = 1.41421354f;

__device__ __forceinline__ float grid_nan() { return __int_as_float(0x7fc00000); }

struct Entry {  // one heap element; 8-byte aligned so that an entry moves in one load and one store
  float key;
  uint32_t cd;  // cell << 3 | move
};
static_assert(sizeof(Entry) == 8, "heap entry is 8 bytes");

// comp(a, b) of the reference's priority_queue: a->key > b->key
__device__ __forceinline__ void heap_sift_up(Entry* h, int64_t hole, int64_t top, Entry v) {
  int64_t parent = (hole - 1) / 2;
  while (hole > top && h[parent].key > v.key) {
    h[hole] = h[parent];
    hole = parent;
    parent = (hole - 1) / 2;
  }
  h[hole] = v;
}

__device__ __forceinline__ void heap_push(Entry* h, int64_t& len, Entry v) {
  heap_sift_up(h, len, 0, v);
  ++len;
}

// pop_heap + pop_back: returns the top, len shrinks by one
__device__ __forceinline__ Entry heap_pop(Entry* h, int64_t& len) {
  const Entry top = h[0];
  --len;
  if (len > 0) {
    const Entry v = h[len];
    int64_t hole = 0, child = 0;
    while (child < (len - 1) / 2) {
      child = 2 * (child + 1);
      if (h[child].key > h[child - 1].key) --child;
      h[hole] = h[child];
      hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
      child = 2 * (child + 1);
      h[hole] = h[child - 1];
      hole = child - 1;
    }
    heap_sift_up(h, hole, 0, v);
  }
  return top;
}

// (int)std::round(p / reso) with p / reso a float quotient and roundf; false when the result is not a finite value
// inside the int range (the reference's conversion is undefined there)
__device__ __forceinline__ bool grid_cell_f(float p, float reso, int& c) {
  const float r = roundf(__fdiv_rn(p, reso));
  if (!(r >= -2147483648.0f && r < 2147483648.0f)) return false;
  c = __float2int_rz(r);
  return true;
}

// (int)std::round(o * 1.0 / reso), in double
__device__ __forceinline__ bool grid_cell_d(float o, float reso, int& c) {
  const double r = round(__ddiv_rn((double)o, (double)reso));
  if (!(r >= -2147483648.0 && r < 2147483648.0)) return false;
  c = __double2int_rz(r);
  return true;
}

}  // namespace

// Grow-only planner workspace of the context, shared by both planners (the first 256 bytes hold the query counter).
int crb_grid_ws_reserve(crb_ctx* ctx, size_t bytes);
// CRB_OK, or CRB_ERR_NO_DEVICE (and the error string) without a usable CUDA device.
int crb_grid_require_device(const char* fn);

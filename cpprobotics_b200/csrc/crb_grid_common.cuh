// crb_grid_common.cuh — device code shared by the grid planners' kernels (crb_grid.cu: one map; crb_grid_many.cu: a
// map per query): the motion model, the restated libstdc++ heap, the reference's rounding of points to cells, the
// obstacle map's per-cell test and the search of one query.  See crb_grid.cu for what each piece restates.
#pragma once

#include <float.h>

#include "crb_common.cuh"

#define GRID_MAP_BLOCK 256
#define GRID_PLAN_BLOCK 128

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

// calc_obstacle_map for the cell (x, y) (one thread per cell, every thread of the block calls it): whether an obstacle
// lies within thr cells of it.  Obstacle k is (ox[k * stride], oy[k * stride]); the block rounds the obstacles to cells
// a tile of GRID_MAP_BLOCK at a time into s_ob / s_ok.
__device__ __forceinline__ bool grid_cell_blocked(int64_t x, int64_t y, int64_t n_obs, const float* ox, const float* oy,
                                                  int64_t stride, float reso, float thr, int2* s_ob, int* s_ok) {
  bool blocked = false;
  for (int64_t k0 = 0; k0 < n_obs; k0 += GRID_MAP_BLOCK) {
    const int64_t k = k0 + threadIdx.x;
    int ix = 0, iy = 0;
    const bool ok = k < n_obs && grid_cell_d(ox[k * stride], reso, ix) && grid_cell_d(oy[k * stride], reso, iy);
    __syncthreads();  // the previous tile is no longer read
    s_ob[threadIdx.x] = make_int2(ix, iy);
    s_ok[threadIdx.x] = ok;
    __syncthreads();
    const int m = n_obs - k0 < GRID_MAP_BLOCK ? (int)(n_obs - k0) : GRID_MAP_BLOCK;
    for (int j = 0; j < m && !blocked; ++j) {
      if (!s_ok[j]) continue;
      // std::sqrt(std::pow(ox - x, 2) + std::pow(oy - y, 2)) in double, narrowed to the float d; the squares of
      // integer differences are exact
      const double dx = (double)(s_ob[j].x - x), dy = (double)(s_ob[j].y - y);
      const float d = __double2float_rn(__dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy))));
      blocked = d <= thr;
    }
  }
  return blocked;
}

// Slot layout: heap | g (A* only) | state, each 256-byte aligned, for a map of `cells` cells (the heap at offset 0).
__host__ __device__ __forceinline__ void grid_slot_layout(bool astar, int64_t cells, int64_t& g_off, int64_t& state_off,
                                                          int64_t& slot_bytes) {
  g_off = ((8 * cells + 1) * (int64_t)sizeof(Entry) + 255) / 256 * 256;
  state_off = g_off + (astar ? (cells * (int64_t)sizeof(float) + 255) / 256 * 256 : 0);
  slot_bytes = (state_off + cells + 255) / 256 * 256;
}

// The queries of a plan launch and where their outputs go (crb.h): query q plans from (sg[q], sg[n + q]) to
// (sg[2 n + q], sg[3 n + q]); path is NULL when max_pts is 0.
struct GridQueries {
  int64_t n;
  const float* sg;
  int max_pts;
  float* path;
  int32_t* path_len;
  float* cost;
  int32_t* n_visited;
  int32_t* status;
};

// Query q (of n) of a_star_planning (ALGO = CRB_GRID_ASTAR) or dijkstra_star_planning on `map`, the W x H = cells
// cells of box at resolution reso, in a slot's heap, g (A* only) and state; writes the query's outputs.  map_ok false
// stands for a bad map entry: CRB_GRID_BAD_MAP, and nothing of the map or the slot is touched.  box, reso and map are
// references so that crb_grid_plan_kernel reads them from its parameters where they are used: taken by value, they
// change that kernel's machine code.
template <int ALGO>
__device__ __forceinline__ void grid_plan_query(const GridQueries& a, int64_t n, int64_t q, bool map_ok, const crb_grid_box& box,
                                                int W, int H, int64_t cells, const float& reso, const uint8_t* const& map,
                                                Entry* heap, float* g, uint8_t* st) {
  int sx, sy, gx, gy;
  int32_t status = CRB_GRID_NO_PATH, nvis = 0, plen = 0;
  float cost = grid_nan();
  if (!map_ok) {
    status = CRB_GRID_BAD_MAP;
  } else if (!(grid_cell_f(a.sg[q], reso, sx) && grid_cell_f(a.sg[n + q], reso, sy) &&
               grid_cell_f(a.sg[2 * n + q], reso, gx) && grid_cell_f(a.sg[3 * n + q], reso, gy))) {
    status = CRB_GRID_BAD_POINT;
  } else {
    // box-relative cells (64-bit: a cell far outside the box must not wrap into it)
    const int64_t rsx = (int64_t)sx - box.min_x, rsy = (int64_t)sy - box.min_y;
    const int64_t rgx = (int64_t)gx - box.min_x, rgy = (int64_t)gy - box.min_y;
    if (rsx < 0 || rsx >= W || rsy < 0 || rsy >= H) {
      status = CRB_GRID_START_OUTSIDE;
    } else {
      const bool goal_in = rgx >= 0 && rgx < W && rgy >= 0 && rgy < H;
      const int64_t goal_cell = goal_in ? rgx * H + rgy : -1;
      // fresh cell state (and path costs) for this query, 16 bytes per store
      {
        uint4* s4 = (uint4*)st;
        const int64_t n4 = (cells + 15) / 16;
        for (int64_t i = 0; i < n4; ++i) s4[i] = make_uint4(0u, 0u, 0u, 0u);
        if (ALGO == CRB_GRID_ASTAR) {
          const uint32_t fm = __float_as_uint(FLT_MAX);
          uint4* g4 = (uint4*)g;
          const int64_t m4 = (cells + 3) / 4;
          for (int64_t i = 0; i < m4; ++i) g4[i] = make_uint4(fm, fm, fm, fm);
        }
      }
      const int64_t start = rsx * H + rsy;
      if (ALGO == CRB_GRID_ASTAR) g[start] = 0.0f;
      int64_t len = 0;
      heap_push(heap, len, Entry{0.0f, (uint32_t)start << 3});
      bool first = true;
      while (len > 0) {
        const Entry e = heap_pop(heap, len);
        const int64_t cell = e.cd >> 3;
        if (st[cell] & 0x80) continue;  // a duplicate of a visited cell
        st[cell] = first ? 0x88 : (uint8_t)(0x80 | (e.cd & 7));
        first = false;
        ++nvis;
        if (cell == goal_cell) {
          status = CRB_GRID_FOUND;
          cost = e.key;
          break;
        }
        const int cx = (int)(cell / H), cy = (int)(cell - (int64_t)cx * H);
        float gc = 0.0f, h = 0.0f;
        if (ALGO == CRB_GRID_ASTAR) {
          gc = g[cell];
          // calc_heristic(ngoal, node): w * std::sqrt(pow(dx, 2) + pow(dy, 2)) in double (w = 1), narrowed
          const double dx = (double)(rgx - cx), dy = (double)(rgy - cy);
          h = __double2float_rn(__dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy))));
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int nx = cx + c_mx[i], ny = cy + c_my[i];
          if (nx < 0 || nx >= W || ny < 0 || ny >= H) continue;  // verify_node: the box
          const int64_t nc = (int64_t)nx * H + ny;
          if (__ldg(map + nc)) continue;                          // verify_node: the map
          if (st[nc] & 0x80) continue;                            // visited
          const float step = i < 4 ? 1.0f : kDiag;
          if (ALGO == CRB_GRID_ASTAR) {
            const float ng = __fadd_rn(gc, step);
            if (ng < g[nc]) {
              g[nc] = ng;
              heap_push(heap, len, Entry{__fadd_rn(ng, h), ((uint32_t)nc << 3) | (uint32_t)i});
            }
          } else {
            heap_push(heap, len, Entry{__fadd_rn(e.key, step), ((uint32_t)nc << 3) | (uint32_t)i});
          }
        }
      }
      if (status == CRB_GRID_FOUND) {
        // calc_final_path: the goal, then parent after parent down to the start
        int64_t c = goal_cell;
        for (;;) {
          if (a.path && plen < a.max_pts) {
            const int x = (int)(c / H), y = (int)(c - (c / H) * H);
            a.path[(2 * (int64_t)plen) * n + q] = __fmul_rn(__int2float_rn(x + box.min_x), reso);
            a.path[(2 * (int64_t)plen + 1) * n + q] = __fmul_rn(__int2float_rn(y + box.min_y), reso);
          }
          ++plen;
          const uint8_t s = st[c];
          if (s & 0x08) break;
          c -= (int64_t)c_mx[s & 7] * H + c_my[s & 7];
        }
      }
    }
  }
  if (status != CRB_GRID_FOUND) plen = 0;
  if (a.path_len) a.path_len[q] = plen;
  if (a.cost) a.cost[q] = cost;
  if (a.n_visited) a.n_visited[q] = status == CRB_GRID_NO_PATH || status == CRB_GRID_FOUND ? nvis : 0;
  if (a.status) a.status[q] = status;
}

}  // namespace

// Grow-only planner workspace of the context, shared by both planners (the first 256 bytes hold the query counter).
int crb_grid_ws_reserve(crb_ctx* ctx, size_t bytes);

// crb_grid.cu — grid A* and Dijkstra for many start / goal queries on one obstacle map, for sm_90a.
//
// Replaces calc_obstacle_map, a_star_planning and dijkstra_star_planning of src/a_star.cpp and src/dijkstra.cpp
// (the two files differ in about 12 lines: the key, and A*'s path_cost relaxation).  Bit-exact with the reference
// built for x86-64: every float and double operation is an explicitly rounded intrinsic, so the TU's -fmad setting
// does not matter, and the priority queue is the libstdc++ binary heap restated step by step (push: sift-up while
// the parent's key is greater; pop: the last entry is saved, the hole walks down to a leaf taking the right child
// unless its key is greater than the left one's, the lone left child of an even-sized heap is taken, and the saved
// entry sifts back up).  Ties are everywhere on a grid, and which parent a cell keeps is decided by that order.
// Queries that each plan on their own map: crb_grid_many.cu, on the same device code (crb_grid_common.cuh).
//
// Mapping.
//   crb_grid_map_kernel: one thread per cell; the obstacles are rounded to cells once per block, a tile at a time, in
//     shared memory, and every thread of the block tests its cell against the tile.
//   crb_grid_plan_kernel: one thread per query, running the reference's search serially (the pop order is the
//     result, so there is nothing to split inside a query).  The kernel is persistent: each lane owns one workspace
//     slot and takes its next query from an atomic counter, so a lane whose query ends early starts another instead
//     of waiting for the rest of its warp.  A slot holds
//       heap  [8 * cells + 1] 8-byte entries: float key, cell << 3 | move (every visited cell pushes at most 8)
//       g     [cells] float, A*'s path_cost (FLT_MAX = never reached)
//       state [cells] uint8: bit 7 visited, bit 3 the start, bits 0-2 the move that reached the cell from its parent
//     and the parent of a cell is cell - offset[move], so no pointer or parent array is kept.
#include "crb_grid_common.cuh"

__global__ void __launch_bounds__(GRID_MAP_BLOCK)
crb_grid_map_kernel(int64_t n_obs, const float* __restrict__ ox, const float* __restrict__ oy, float reso, float thr,
                    crb_grid_box box, int64_t cells, uint8_t* __restrict__ map) {
  __shared__ int2 s_ob[GRID_MAP_BLOCK];
  __shared__ int s_ok[GRID_MAP_BLOCK];
  const int64_t c = (int64_t)blockIdx.x * GRID_MAP_BLOCK + threadIdx.x;
  const int64_t H = (int64_t)box.max_y - box.min_y;
  const int64_t x = c < cells ? box.min_x + c / H : 0, y = c < cells ? box.min_y + c % H : 0;
  const bool blocked = grid_cell_blocked(x, y, n_obs, ox, oy, 1, reso, thr, s_ob, s_ok);
  if (c < cells) map[c] = blocked ? 1 : 0;
}

struct GridPlanArgs {
  crb_grid_box box;
  const uint8_t* map;
  float reso;
  GridQueries q;
  unsigned long long* counter;
  char* ws;
  size_t slot_bytes;
  int64_t slots;
  int64_t heap_off, g_off, state_off;  // byte offsets inside a slot
};

template <int ALGO>
__global__ void __launch_bounds__(GRID_PLAN_BLOCK) crb_grid_plan_kernel(const GridPlanArgs a) {
  const int64_t lane = (int64_t)blockIdx.x * GRID_PLAN_BLOCK + threadIdx.x;
  if (lane >= a.slots) return;
  char* slot = a.ws + lane * a.slot_bytes;
  Entry* heap = (Entry*)(slot + a.heap_off);
  float* g = (float*)(slot + a.g_off);
  uint8_t* st = (uint8_t*)(slot + a.state_off);
  const int64_t n = a.q.n;
  const int W = a.box.max_x - a.box.min_x, H = a.box.max_y - a.box.min_y;
  const int64_t cells = (int64_t)W * H;
  for (;;) {
    const int64_t q = (int64_t)atomicAdd(a.counter, 1ull);
    if (q >= n) return;
    grid_plan_query<ALGO>(a.q, n, q, true, a.box, W, H, cells, a.reso, a.map, heap, g, st);
  }
}

namespace {

// W, H and W * H of a box inside the limits, or false after setting the error string
bool grid_box_dims(const crb_grid_box* b, const char* fn, int64_t& W, int64_t& H) {
  if (b == nullptr) {
    crb_set_error("%s: invalid argument: box is NULL", fn);
    return false;
  }
  W = (int64_t)b->max_x - b->min_x;
  H = (int64_t)b->max_y - b->min_y;
  if (W < 1 || H < 1) {
    crb_set_error("%s: invalid argument: the box is empty", fn);
    return false;
  }
  if (W > CRB_GRID_MAX_SIDE || H > CRB_GRID_MAX_SIDE || W * H > CRB_GRID_MAX_CELLS) {
    crb_set_error("%s: invalid argument: the box exceeds CRB_GRID_MAX_SIDE or CRB_GRID_MAX_CELLS", fn);
    return false;
  }
  return true;
}

bool grid_reso_ok(float reso) { return isfinite(reso) && reso > 0.0f; }

int grid_slots(crb_ctx* ctx, int algo, int64_t cells, int64_t n, int64_t& slots, int64_t& slot_bytes) {
  int per_sm = 0;
  CRB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(
      &per_sm, algo == CRB_GRID_ASTAR ? (const void*)crb_grid_plan_kernel<CRB_GRID_ASTAR>
                                      : (const void*)crb_grid_plan_kernel<CRB_GRID_DIJKSTRA>,
      GRID_PLAN_BLOCK, 0));
  int64_t go, so;
  grid_slot_layout(algo == CRB_GRID_ASTAR, cells, go, so, slot_bytes);
  const int64_t resident = (int64_t)(per_sm > 0 ? per_sm : 1) * GRID_PLAN_BLOCK * ctx->sm_count;
  int64_t by_budget = (int64_t)(CRB_GRID_WS_BUDGET / (size_t)slot_bytes);
  if (by_budget < 1) by_budget = 1;
  slots = n < resident ? n : resident;
  if (slots > by_budget) slots = by_budget;
  if (slots < 1) slots = 1;
  return CRB_OK;
}

}  // namespace

// Grow-only planner workspace of the context (the first 256 bytes hold the query counter); crb_grid_many.cu's planner
// shares it.
int crb_grid_ws_reserve(crb_ctx* ctx, size_t bytes) {
  if (ctx->grid_ws_cap >= bytes) return CRB_OK;
  if (ctx->grid_ws) {
    CRB_CUDA(cudaStreamSynchronize(ctx->stream));
    CRB_CUDA(cudaFree(ctx->grid_ws));
    ctx->grid_ws = nullptr;
    ctx->grid_ws_cap = 0;
  }
  const cudaError_t e = cudaMalloc(&ctx->grid_ws, bytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    ctx->grid_ws = nullptr;
    crb_set_error("crb_grid_plan_batched: cudaMalloc of %zu workspace bytes: %s", bytes, cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? CRB_ERR_ALLOC : CRB_ERR_CUDA;
  }
  ctx->grid_ws_cap = bytes;
  return CRB_OK;
}

extern "C" {

int crb_grid_box_of_obstacles(int64_t n_obs, const float* ox, const float* oy, float reso, crb_grid_box* box) {
  CRB_REQUIRE(n_obs >= 1, "n_obs must be >= 1");
  CRB_REQUIRE(ox && oy && box, "ox, oy or box is NULL");
  CRB_REQUIRE(grid_reso_ok(reso), "reso must be finite and > 0");
  int mnx = INT32_MAX, mxx = INT32_MIN, mny = INT32_MAX, mxy = INT32_MIN;
  for (int64_t k = 0; k < n_obs; ++k) {
    const double rx = round((double)ox[k] * 1.0 / (double)reso), ry = round((double)oy[k] * 1.0 / (double)reso);
    CRB_REQUIRE(rx >= -2147483648.0 && rx < 2147483648.0 && ry >= -2147483648.0 && ry < 2147483648.0,
                "an obstacle is non-finite or rounds outside the int range");
    const int x = (int)rx, y = (int)ry;
    mnx = x < mnx ? x : mnx;
    mxx = x > mxx ? x : mxx;
    mny = y < mny ? y : mny;
    mxy = y > mxy ? y : mxy;
  }
  box->min_x = mnx;
  box->min_y = mny;
  box->max_x = mxx;
  box->max_y = mxy;
  return CRB_OK;
}

int crb_grid_obstacle_map(crb_ctx* ctx, int64_t n_obs, const float* ox, const float* oy, float reso, float rr,
                          const crb_grid_box* box, uint8_t* map) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(n_obs >= 0, "n_obs must be >= 0");
  CRB_REQUIRE(grid_reso_ok(reso), "reso must be finite and > 0");
  CRB_REQUIRE(isfinite(rr), "rr must be finite");
  int64_t W, H;
  if (!grid_box_dims(box, __func__, W, H)) return CRB_ERR_INVALID_ARG;
  CRB_REQUIRE(map != nullptr && (n_obs == 0 || (ox && oy)), "ox, oy or map is NULL");
  const int rc = crb_require_device(__func__);
  if (rc != CRB_OK) return rc;
  CRB_DEVICE_GUARD(ctx);
  const int64_t cells = W * H;
  // vr / reso: the float quotient the reference compares with
  const float thr = rr / reso;
  crb_grid_map_kernel<<<crb_grid_for(cells, GRID_MAP_BLOCK), GRID_MAP_BLOCK, 0, ctx->stream>>>(
      n_obs, ox, oy, reso, thr, *box, cells, map);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

int crb_grid_plan_slots(crb_ctx* ctx, int algo, const crb_grid_box* box, int64_t n, int64_t* slots) {
  CRB_REQUIRE(ctx != nullptr && slots != nullptr, "ctx or slots is NULL");
  CRB_REQUIRE(algo == CRB_GRID_ASTAR || algo == CRB_GRID_DIJKSTRA, "algo must be CRB_GRID_ASTAR or CRB_GRID_DIJKSTRA");
  CRB_REQUIRE(n >= 0, "n must be >= 0");
  int64_t W, H;
  if (!grid_box_dims(box, __func__, W, H)) return CRB_ERR_INVALID_ARG;
  const int rc = crb_require_device(__func__);
  if (rc != CRB_OK) return rc;
  CRB_DEVICE_GUARD(ctx);
  int64_t sb;
  return grid_slots(ctx, algo, W * H, n, *slots, sb);
}

int crb_grid_plan_batched(crb_ctx* ctx, int algo, const crb_grid_box* box, const uint8_t* map, float reso, int64_t n,
                          const float* sg, int max_pts, float* path, int32_t* path_len, float* cost,
                          int32_t* n_visited, int32_t* status) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(algo == CRB_GRID_ASTAR || algo == CRB_GRID_DIJKSTRA, "algo must be CRB_GRID_ASTAR or CRB_GRID_DIJKSTRA");
  CRB_REQUIRE(grid_reso_ok(reso), "reso must be finite and > 0");
  CRB_REQUIRE(n >= 0 && n <= INT64_MAX / 4, "n out of range");
  CRB_REQUIRE(max_pts >= 0, "max_pts must be >= 0");
  CRB_REQUIRE(n <= INT64_MAX / 2 / (max_pts > 0 ? max_pts : 1), "n * max_pts out of range");
  int64_t W, H;
  if (!grid_box_dims(box, __func__, W, H)) return CRB_ERR_INVALID_ARG;
  CRB_REQUIRE(n == 0 || (map && sg), "map or sg is NULL");
  CRB_REQUIRE(n == 0 || max_pts == 0 || path, "path is NULL with max_pts > 0");
  const int rc = crb_require_device(__func__);
  if (rc != CRB_OK) return rc;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  GridPlanArgs a;
  a.box = *box;
  a.map = map;
  a.reso = reso;
  a.q = GridQueries{n, sg, max_pts, max_pts > 0 ? path : nullptr, path_len, cost, n_visited, status};
  int64_t slot_bytes;
  int r = grid_slots(ctx, algo, W * H, n, a.slots, slot_bytes);
  if (r != CRB_OK) return r;
  a.slot_bytes = (size_t)slot_bytes;
  a.heap_off = 0;
  grid_slot_layout(algo == CRB_GRID_ASTAR, W * H, a.g_off, a.state_off, slot_bytes);
  r = crb_grid_ws_reserve(ctx, 256 + (size_t)a.slots * a.slot_bytes);
  if (r != CRB_OK) return r;
  a.counter = (unsigned long long*)ctx->grid_ws;
  a.ws = (char*)ctx->grid_ws + 256;
  CRB_CUDA(cudaMemsetAsync(a.counter, 0, sizeof(unsigned long long), ctx->stream));
  const int blocks = crb_grid_for(a.slots, GRID_PLAN_BLOCK);
  if (algo == CRB_GRID_ASTAR)
    crb_grid_plan_kernel<CRB_GRID_ASTAR><<<blocks, GRID_PLAN_BLOCK, 0, ctx->stream>>>(a);
  else
    crb_grid_plan_kernel<CRB_GRID_DIJKSTRA><<<blocks, GRID_PLAN_BLOCK, 0, ctx->stream>>>(a);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

}  // extern "C"

// crb_grid_many.cu — grid A* and Dijkstra with a map per query, for sm_90a: calc_obstacle_map for many maps in one
// launch, and a_star_planning / dijkstra_star_planning for queries that each name their own map.
//
// The maps live back to back in one byte store described by a map table (crb.h): boxes, reso and map_off per map.
// Every entry is device data, checked on the device before anything it points at is read.  The kernels are
// crb_grid.cu's, generalised to read their box, resolution and map from the table (the computation, the heap and the
// rounding are the same code, crb_grid_common.cuh), so each map and each query's outputs are bitwise those of the
// single-map entry points on that map.  crb_grid.cu's kernels are kept as they were for the single-map entry points:
// with every query on one map, these kernels took 0.4 % longer on the scatter 128^2 map with Dijkstra, beyond the
// run-to-run spread of 0.2 %, on an H100 (DESIGN.md §3).
//
// Mapping.
//   crb_grid_map_many_kernel: blocks indexed by (256-cell tile, map), so every valid map is built in full whatever the
//     other entries hold and no block searches map_off; a block past its map's cells leaves at once.
//   crb_grid_plan_many_kernel: crb_grid_plan_kernel's persistent lanes and slots; the slots are sized for the call's
//     max_cells, and each query lays its slot out (heap 8 * W * H + 1 entries, A*'s g, state) for its own map.
#include "crb_grid_common.cuh"

#define GRID_MAP_BLOCK 256
#define GRID_PLAN_BLOCK 128

namespace {

// A map table (crb.h): map m has box boxes[m], resolution reso[m] and bytes [map_off[m], map_off[m + 1]) of maps.
struct GridTable {
  const crb_grid_box* boxes;
  const float* reso;
  const int64_t* map_off;
  int32_t n_maps;
  int64_t n_cells, max_cells;
};

// Entry m of a table, checked before anything it points at is read: false for an index outside [0, n_maps), a box
// outside the limits or with more than max_cells cells, inconsistent offsets, or a reso that is not finite and > 0
__device__ __forceinline__ bool grid_table_entry(const GridTable& t, int64_t m, crb_grid_box& box, float& reso,
                                                 int64_t& off) {
  if (m < 0 || m >= t.n_maps) return false;
  const crb_grid_box b = t.boxes[m];
  const int64_t W = (int64_t)b.max_x - b.min_x, H = (int64_t)b.max_y - b.min_y;
  if (W < 1 || H < 1 || W > CRB_GRID_MAX_SIDE || H > CRB_GRID_MAX_SIDE || W * H > t.max_cells) return false;
  const int64_t lo = t.map_off[m], hi = t.map_off[m + 1];
  if (lo < 0 || hi < lo || hi > t.n_cells || hi - lo != W * H) return false;
  const float r = t.reso[m];
  if (!(isfinite(r) && r > 0.0f)) return false;
  box = b;
  reso = r;
  off = lo;
  return true;
}

// Slot layout: heap | g (A* only) | state, each 256-byte aligned, for a map of `cells` cells.  A query lays its slot
// out for its own map; the host sizes the slots for the largest map a call may use.
__host__ __device__ __forceinline__ void grid_slot_layout(bool astar, int64_t cells, int64_t& g_off, int64_t& state_off,
                                                          int64_t& slot_bytes) {
  g_off = ((8 * cells + 1) * (int64_t)sizeof(Entry) + 255) / 256 * 256;
  state_off = g_off + (astar ? (cells * (int64_t)sizeof(float) + 255) / 256 * 256 : 0);
  slot_bytes = (state_off + cells + 255) / 256 * 256;
}

}  // namespace

struct GridMapArgs {
  const float* ob;  // [n_rows][2] rows (ox, oy)
  int64_t n_rows;
  const int64_t* ob_off;
  int32_t n_sets;
  const int32_t* ob_of;  // [n_maps] the list of each map
  const float* rr;       // [n_maps]
  GridTable t;
  uint8_t* maps;
  int32_t* map_status;
};

// crb_grid_map_kernel's computation, block (tile, m) building the cells [256 * tile, 256 * tile + 256) of map m:
// gridDim.y blocks stride over the maps and block (0, m) writes map m's status.  Blocks past a map's cells, and every
// block of a bad entry, leave at once; nothing of a map is read before its entry and list reference are checked.
__global__ void __launch_bounds__(GRID_MAP_BLOCK) crb_grid_map_many_kernel(const GridMapArgs a) {
  __shared__ int2 s_ob[GRID_MAP_BLOCK];
  __shared__ int s_ok[GRID_MAP_BLOCK];
  for (int64_t mi = blockIdx.y; mi < a.t.n_maps; mi += gridDim.y) {
    crb_grid_box box = {0, 0, 1, 1};
    float reso = 1.0f;
    int64_t ob0 = 0, ob1 = 0, off = 0;
    bool ok = grid_table_entry(a.t, mi, box, reso, off);
    const float rr = ok ? a.rr[mi] : 0.0f;
    ok = ok && isfinite(rr) && crb_obstacle_list(mi, a.ob_off, a.n_sets, a.ob_of, a.n_rows, INT64_MAX, ob0, ob1);
    if (a.map_status && blockIdx.x == 0 && threadIdx.x == 0) a.map_status[mi] = ok ? CRB_GRID_MAP_OK : CRB_GRID_MAP_BAD;
    if (!ok) continue;  // the whole block: nothing of this map is written
    // vr / reso: the float quotient the reference compares with
    const float thr = __fdiv_rn(rr, reso);
    const int64_t H = (int64_t)box.max_y - box.min_y;
    const int64_t cells = ((int64_t)box.max_x - box.min_x) * H;
    if ((int64_t)blockIdx.x * GRID_MAP_BLOCK >= cells) continue;
    const int64_t n_obs = ob1 - ob0;
    const float* ob = a.ob + 2 * ob0;
    const int64_t c = (int64_t)blockIdx.x * GRID_MAP_BLOCK + threadIdx.x;
    const int64_t x = c < cells ? box.min_x + c / H : 0, y = c < cells ? box.min_y + c % H : 0;
    bool blocked = false;
    for (int64_t k0 = 0; k0 < n_obs; k0 += GRID_MAP_BLOCK) {
      const int64_t k = k0 + threadIdx.x;
      int ix = 0, iy = 0;
      const bool ok = k < n_obs && grid_cell_d(ob[2 * k], reso, ix) && grid_cell_d(ob[2 * k + 1], reso, iy);
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
    if (c < cells) a.maps[off + c] = blocked ? 1 : 0;
  }
}

struct GridPlanManyArgs {
  const uint8_t* maps;
  GridTable t;
  const int32_t* map_of;  // [n] the map of each query
  int64_t n;
  const float* sg;
  int max_pts;
  float* path;
  int32_t* path_len;
  float* cost;
  int32_t* n_visited;
  int32_t* status;
  unsigned long long* counter;
  char* ws;
  int64_t slot_bytes;
  int64_t slots;
};

// crb_grid_plan_kernel's search, each query on its own map: the entry is checked before the map is read, and the slot
// (sized by the host for max_cells) is laid out for the query's own W * H.  __maxnreg__(56) (launched with
// GRID_PLAN_BLOCK threads) keeps A* from the 16-byte spill ptxas otherwise chooses at 48 registers.
template <int ALGO>
__global__ void __maxnreg__(56) crb_grid_plan_many_kernel(const GridPlanManyArgs a) {
  const int64_t lane = (int64_t)blockIdx.x * GRID_PLAN_BLOCK + threadIdx.x;
  if (lane >= a.slots) return;
  char* slot = a.ws + lane * a.slot_bytes;
  const int64_t n = a.n;
  for (;;) {
    const int64_t q = (int64_t)atomicAdd(a.counter, 1ull);
    if (q >= n) return;
    crb_grid_box box = {0, 0, 1, 1};
    float reso = 1.0f;
    int64_t off = 0;
    const bool map_ok = grid_table_entry(a.t, a.map_of[q], box, reso, off);
    const uint8_t* map = a.maps + off;
    const int W = box.max_x - box.min_x, H = box.max_y - box.min_y;
    const int64_t cells = (int64_t)W * H;
    int64_t g_off, state_off, slot_end;
    grid_slot_layout(ALGO == CRB_GRID_ASTAR, cells, g_off, state_off, slot_end);
    Entry* heap = (Entry*)slot;
    float* g = (float*)(slot + g_off);
    uint8_t* st = (uint8_t*)(slot + state_off);
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
}

namespace {

int grid_many_slots(crb_ctx* ctx, int algo, int64_t max_cells, int64_t n, int64_t& slots, int64_t& slot_bytes) {
  int per_sm = 0;
  CRB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(
      &per_sm, algo == CRB_GRID_ASTAR ? (const void*)crb_grid_plan_many_kernel<CRB_GRID_ASTAR>
                                      : (const void*)crb_grid_plan_many_kernel<CRB_GRID_DIJKSTRA>,
      GRID_PLAN_BLOCK, 0));
  int64_t go, so;
  grid_slot_layout(algo == CRB_GRID_ASTAR, max_cells, go, so, slot_bytes);
  const int64_t resident = (int64_t)(per_sm > 0 ? per_sm : 1) * GRID_PLAN_BLOCK * ctx->sm_count;
  int64_t by_budget = (int64_t)(CRB_GRID_WS_BUDGET / (size_t)slot_bytes);
  if (by_budget < 1) by_budget = 1;
  slots = n < resident ? n : resident;
  if (slots > by_budget) slots = by_budget;
  if (slots < 1) slots = 1;
  return CRB_OK;
}

// Host checks of a map table's scalars (the entries are device data, checked per map or query on the device)
bool grid_table_scalars_ok(int32_t n_maps, int64_t n_cells, int64_t max_cells, const char* fn) {
  if (n_maps < 1 || n_cells < 0 || max_cells < 1 || max_cells > CRB_GRID_MAX_CELLS) {
    crb_set_error("%s: invalid argument: need n_maps >= 1, n_cells >= 0 and 1 <= max_cells <= CRB_GRID_MAX_CELLS", fn);
    return false;
  }
  return true;
}

}  // namespace

extern "C" {

int crb_grid_obstacle_map_many(crb_ctx* ctx, const float* ob, int64_t n_rows, const int64_t* ob_off, int32_t n_sets,
                               const int32_t* ob_of, const float* rr, const crb_grid_box* boxes, const float* reso,
                               const int64_t* map_off, int32_t n_maps, int64_t n_cells, int64_t max_cells,
                               uint8_t* maps, int32_t* map_status) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  if (!grid_table_scalars_ok(n_maps, n_cells, max_cells, __func__)) return CRB_ERR_INVALID_ARG;
  CRB_REQUIRE(n_sets >= 1 && n_rows >= 0, "need n_sets >= 1 and n_rows >= 0");
  CRB_REQUIRE(boxes && reso && map_off, "boxes, reso or map_off is NULL");
  CRB_REQUIRE(ob_off && ob_of && rr && (ob || n_rows == 0), "ob, ob_off, ob_of or rr is NULL");
  CRB_REQUIRE(maps || n_cells == 0, "maps is NULL");
  const int rc = crb_grid_require_device(__func__);
  if (rc != CRB_OK) return rc;
  CRB_DEVICE_GUARD(ctx);
  GridMapArgs a = {};
  a.ob = ob;
  a.n_rows = n_rows;
  a.ob_off = ob_off;
  a.n_sets = n_sets;
  a.ob_of = ob_of;
  a.rr = rr;
  a.t = GridTable{boxes, reso, map_off, n_maps, n_cells, max_cells};
  a.maps = maps;
  a.map_status = map_status;
  const dim3 grid(crb_grid_for(max_cells, GRID_MAP_BLOCK), n_maps < 65535 ? n_maps : 65535);
  crb_grid_map_many_kernel<<<grid, GRID_MAP_BLOCK, 0, ctx->stream>>>(a);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

int crb_grid_plan_many_slots(crb_ctx* ctx, int algo, int64_t max_cells, int64_t n, int64_t* slots) {
  CRB_REQUIRE(ctx != nullptr && slots != nullptr, "ctx or slots is NULL");
  CRB_REQUIRE(algo == CRB_GRID_ASTAR || algo == CRB_GRID_DIJKSTRA, "algo must be CRB_GRID_ASTAR or CRB_GRID_DIJKSTRA");
  CRB_REQUIRE(n >= 0, "n must be >= 0");
  CRB_REQUIRE(max_cells >= 1 && max_cells <= CRB_GRID_MAX_CELLS, "max_cells must be in [1, CRB_GRID_MAX_CELLS]");
  const int rc = crb_grid_require_device(__func__);
  if (rc != CRB_OK) return rc;
  CRB_DEVICE_GUARD(ctx);
  int64_t sb;
  return grid_many_slots(ctx, algo, max_cells, n, *slots, sb);
}

int crb_grid_plan_many_batched(crb_ctx* ctx, int algo, const crb_grid_box* boxes, const float* reso,
                               const int64_t* map_off, int32_t n_maps, const uint8_t* maps, int64_t n_cells,
                               int64_t max_cells, int64_t n, const int32_t* map_of, const float* sg, int max_pts,
                               float* path, int32_t* path_len, float* cost, int32_t* n_visited, int32_t* status) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(algo == CRB_GRID_ASTAR || algo == CRB_GRID_DIJKSTRA, "algo must be CRB_GRID_ASTAR or CRB_GRID_DIJKSTRA");
  if (!grid_table_scalars_ok(n_maps, n_cells, max_cells, __func__)) return CRB_ERR_INVALID_ARG;
  CRB_REQUIRE(n >= 0 && n <= INT64_MAX / 4, "n out of range");
  CRB_REQUIRE(max_pts >= 0, "max_pts must be >= 0");
  CRB_REQUIRE(n <= INT64_MAX / 2 / (max_pts > 0 ? max_pts : 1), "n * max_pts out of range");
  CRB_REQUIRE(n == 0 || (boxes && reso && map_off && map_of && sg), "boxes, reso, map_off, map_of or sg is NULL");
  CRB_REQUIRE(n == 0 || n_cells == 0 || maps, "maps is NULL");
  CRB_REQUIRE(n == 0 || max_pts == 0 || path, "path is NULL with max_pts > 0");
  const int rc = crb_grid_require_device(__func__);
  if (rc != CRB_OK) return rc;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  GridPlanManyArgs a = {};
  a.maps = maps;
  a.t = GridTable{boxes, reso, map_off, n_maps, n_cells, max_cells};
  a.map_of = map_of;
  a.n = n;
  a.sg = sg;
  a.max_pts = max_pts;
  a.path = max_pts > 0 ? path : nullptr;
  a.path_len = path_len;
  a.cost = cost;
  a.n_visited = n_visited;
  a.status = status;
  int r = grid_many_slots(ctx, algo, max_cells, n, a.slots, a.slot_bytes);
  if (r != CRB_OK) return r;
  r = crb_grid_ws_reserve(ctx, 256 + (size_t)a.slots * (size_t)a.slot_bytes);
  if (r != CRB_OK) return r;
  a.counter = (unsigned long long*)ctx->grid_ws;
  a.ws = (char*)ctx->grid_ws + 256;
  CRB_CUDA(cudaMemsetAsync(a.counter, 0, sizeof(unsigned long long), ctx->stream));
  const int blocks = crb_grid_for(a.slots, GRID_PLAN_BLOCK);
  if (algo == CRB_GRID_ASTAR)
    crb_grid_plan_many_kernel<CRB_GRID_ASTAR><<<blocks, GRID_PLAN_BLOCK, 0, ctx->stream>>>(a);
  else
    crb_grid_plan_many_kernel<CRB_GRID_DIJKSTRA><<<blocks, GRID_PLAN_BLOCK, 0, ctx->stream>>>(a);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

}  // extern "C"

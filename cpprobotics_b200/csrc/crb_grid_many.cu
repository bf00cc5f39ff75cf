// crb_grid_many.cu — grid A* and Dijkstra with a map per query, for sm_90a: calc_obstacle_map for many maps in one
// launch, and a_star_planning / dijkstra_star_planning for queries that each name their own map.
//
// The maps live back to back in one byte store described by a map table (crb.h): boxes, reso and map_off per map.
// Every entry is device data, checked on the device before anything it points at is read.  Each kernel runs the same
// per-cell and per-query body as crb_grid.cu's (grid_cell_blocked and grid_plan_query, crb_grid_common.cuh) and
// differs only in reading its box, resolution and map from the table, so each map and each query's outputs are
// bitwise those of the single-map entry points on that map.  The single-map entry points keep their own kernels: with
// every query on one map, these kernels took 0.4 % longer on the scatter 128^2 map with Dijkstra, beyond the
// run-to-run spread of 0.2 %, on an H100 (DESIGN.md §3).
//
// Mapping.
//   crb_grid_map_many_kernel: blocks indexed by (256-cell tile, map), so every valid map is built in full whatever the
//     other entries hold and no block searches map_off; a block past its map's cells leaves at once.
//   crb_grid_plan_many_kernel: crb_grid_plan_kernel's persistent lanes and slots; the slots are sized for the call's
//     max_cells, and each query lays its slot out (heap 8 * W * H + 1 entries, A*'s g, state) for its own map.
#include "crb_grid_common.cuh"

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

// calc_obstacle_map, block (tile, m) building the cells [256 * tile, 256 * tile + 256) of map m:
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
    const bool blocked = grid_cell_blocked(x, y, n_obs, ob, ob + 1, 2, reso, thr, s_ob, s_ok);
    if (c < cells) a.maps[off + c] = blocked ? 1 : 0;
  }
}

struct GridPlanManyArgs {
  const uint8_t* maps;
  GridTable t;
  const int32_t* map_of;  // [n] the map of each query
  GridQueries q;
  unsigned long long* counter;
  char* ws;
  int64_t slot_bytes;
  int64_t slots;
};

// The search, each query on its own map: the entry is checked before the map is read, and the slot (sized by the host
// for max_cells) is laid out for the query's own W * H.  __maxnreg__(56) (launched with
// GRID_PLAN_BLOCK threads) keeps A* from the 16-byte spill ptxas otherwise chooses at 48 registers.
template <int ALGO>
__global__ void __maxnreg__(56) crb_grid_plan_many_kernel(const GridPlanManyArgs a) {
  const int64_t lane = (int64_t)blockIdx.x * GRID_PLAN_BLOCK + threadIdx.x;
  if (lane >= a.slots) return;
  char* slot = a.ws + lane * a.slot_bytes;
  const int64_t n = a.q.n;
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
    grid_plan_query<ALGO>(a.q, n, q, map_ok, box, W, H, cells, reso, map, (Entry*)slot, (float*)(slot + g_off),
                          (uint8_t*)(slot + state_off));
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
  const int rc = crb_require_device(__func__);
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
  const int rc = crb_require_device(__func__);
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
  const int rc = crb_require_device(__func__);
  if (rc != CRB_OK) return rc;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  GridPlanManyArgs a = {};
  a.maps = maps;
  a.t = GridTable{boxes, reso, map_off, n_maps, n_cells, max_cells};
  a.map_of = map_of;
  a.q = GridQueries{n, sg, max_pts, max_pts > 0 ? path : nullptr, path_len, cost, n_visited, status};
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

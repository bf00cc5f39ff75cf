/* crb_oracle_grid.c — CPU restatement of src/a_star.cpp and src/dijkstra.cpp: the obstacle cells and box (:115-140),
 * calc_obstacle_map (:48-78), and the two searches with calc_final_path (:31-45), in plain C.
 *
 * The reference's std::priority_queue<Node*, vector, cmp> with cmp = left->key > right->key is restated as the
 * libstdc++ binary heap it is built on (push_heap, pop_heap, __adjust_heap), so ties pop in the same order; the
 * tests pin this restatement against the host's std::priority_queue.  Per-cell arrays are indexed relative to the
 * box, (x - min_x, y - min_y), which inside the reference's defined domain (a square box; for A* min = 0) is the
 * reference's computation, and outside it defines the result (crb.h).  Statuses as crb.h's CRB_GRID_*. */
#include "crb_oracle_grid.h"

#include <float.h>
#include <math.h>
#include <omp.h>
#include <stdlib.h>
#include <string.h>

enum { ASTAR = 0, DIJKSTRA = 1 };
enum { FOUND = 0, NO_PATH = 1, START_OUTSIDE = 2, BAD_POINT = 3 };

/* get_motion_model :99-108 */
static const int MX[8] = {1, 0, -1, 0, -1, -1, 1, 1};
static const int MY[8] = {0, 1, 0, -1, -1, 1, -1, 1};
#define DIAG 1.41421354f /* (float)std::sqrt(2) */

typedef struct {
  float key;
  uint32_t cd; /* cell << 3 | move (or an id in crb_oracle_grid_heap_run) */
} entry;

/* __push_heap: sift the value up from hole while comp(parent, value), i.e. parent.key > value.key */
static void sift_up(entry* h, int64_t hole, int64_t top, entry v) {
  int64_t parent = (hole - 1) / 2;
  while (hole > top && h[parent].key > v.key) {
    h[hole] = h[parent];
    hole = parent;
    parent = (hole - 1) / 2;
  }
  h[hole] = v;
}

/* priority_queue::push: push_back, then push_heap */
static void heap_push(entry* h, int64_t* len, entry v) {
  sift_up(h, *len, 0, v);
  ++*len;
}

/* priority_queue::pop: pop_heap (the last element saved, the top moved to the back, __adjust_heap from the root over
 * the shorter range), then pop_back.  __adjust_heap walks the hole down taking the right child unless
 * comp(right, left), takes the lone left child of an even-length range, then sifts the saved value up. */
static entry heap_pop(entry* h, int64_t* len) {
  const entry top = h[0];
  const int64_t n = --*len;
  if (n > 0) {
    const entry v = h[n];
    int64_t hole = 0, child = 0;
    while (child < (n - 1) / 2) {
      child = 2 * (child + 1);
      if (h[child].key > h[child - 1].key) --child;
      h[hole] = h[child];
      hole = child;
    }
    if ((n & 1) == 0 && child == (n - 2) / 2) {
      child = 2 * (child + 1);
      h[hole] = h[child - 1];
      hole = child - 1;
    }
    sift_up(h, hole, 0, v);
  }
  return top;
}

int64_t crb_oracle_grid_heap_run(int64_t n_ops, const uint8_t* op, const float* keys, int32_t* popped) {
  entry* h = (entry*)malloc(sizeof(entry) * (size_t)(n_ops > 0 ? n_ops : 1));
  int64_t len = 0, k = 0;
  for (int64_t i = 0; i < n_ops; ++i) {
    if (op[i]) {
      entry e = {keys[i], (uint32_t)i};
      heap_push(h, &len, e);
    } else {
      if (len == 0) {
        k = -1;
        break;
      }
      popped[k++] = (int32_t)heap_pop(h, &len).cd;
    }
  }
  free(h);
  return k;
}

/* (int)std::round(p / reso): a float quotient and roundf; 0 when the result is not finite and inside the int range */
static int cell_f(float p, float reso, int* c) {
  const float r = roundf(p / reso);
  if (!(r >= -2147483648.0f && r < 2147483648.0f)) return 0;
  *c = (int)r;
  return 1;
}

/* (int)std::round(o * 1.0 / reso), in double */
static int cell_d(float o, float reso, int* c) {
  const double r = round((double)o * 1.0 / (double)reso);
  if (!(r >= -2147483648.0 && r < 2147483648.0)) return 0;
  *c = (int)r;
  return 1;
}

int crb_oracle_grid_box(int64_t n_obs, const float* ox, const float* oy, float reso, int32_t* box) {
  if (n_obs < 1 || !isfinite(reso) || !(reso > 0.0f)) return -1;
  int mnx = INT32_MAX, mxx = INT32_MIN, mny = INT32_MAX, mxy = INT32_MIN;
  for (int64_t k = 0; k < n_obs; ++k) {
    int x, y;
    if (!cell_d(ox[k], reso, &x) || !cell_d(oy[k], reso, &y)) return -1;
    mnx = x < mnx ? x : mnx;
    mxx = x > mxx ? x : mxx;
    mny = y < mny ? y : mny;
    mxy = y > mxy ? y : mxy;
  }
  box[0] = mnx;
  box[1] = mny;
  box[2] = mxx;
  box[3] = mxy;
  return 0;
}

void crb_oracle_grid_map(int64_t n_obs, const float* ox, const float* oy, float reso, float rr, const int32_t* box,
                         uint8_t* map) {
  const int64_t W = (int64_t)box[2] - box[0], H = (int64_t)box[3] - box[1];
  const float thr = rr / reso; /* vr / reso */
  int* cx = (int*)malloc(sizeof(int) * (size_t)(n_obs > 0 ? n_obs : 1));
  int* cy = (int*)malloc(sizeof(int) * (size_t)(n_obs > 0 ? n_obs : 1));
  char* ok = (char*)malloc((size_t)(n_obs > 0 ? n_obs : 1));
  for (int64_t k = 0; k < n_obs; ++k) ok[k] = (char)(cell_d(ox[k], reso, &cx[k]) && cell_d(oy[k], reso, &cy[k]));
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < W; ++i) {
    const int64_t x = box[0] + i;
    for (int64_t j = 0; j < H; ++j) {
      const int64_t y = box[1] + j;
      uint8_t b = 0;
      for (int64_t k = 0; k < n_obs; ++k) {
        if (!ok[k]) continue;
        /* std::sqrt(std::pow(ox - x, 2) + std::pow(oy - y, 2)) in double, narrowed to float (the `break`: an OR) */
        const double dx = (double)(cx[k] - x), dy = (double)(cy[k] - y);
        const float d = (float)sqrt(dx * dx + dy * dy);
        if (d <= thr) {
          b = 1;
          break;
        }
      }
      map[i * H + j] = b;
    }
  }
  free(cx);
  free(cy);
  free(ok);
}

typedef struct {
  entry* heap;
  float* g;
  uint8_t* st; /* bit 7 visited, bit 3 the start, bits 0-2 the move from the parent */
} work;

static int work_alloc(work* w, int algo, int64_t cells) {
  w->heap = (entry*)malloc(sizeof(entry) * (size_t)(8 * cells + 1));
  w->g = algo == ASTAR ? (float*)malloc(sizeof(float) * (size_t)cells) : NULL;
  w->st = (uint8_t*)malloc((size_t)cells);
  return w->heap && w->st && (algo != ASTAR || w->g);
}

static void work_free(work* w) {
  free(w->heap);
  free(w->g);
  free(w->st);
}

typedef struct {
  int32_t status, n_visited, path_len;
  float cost;
  int64_t goal_cell;
} result;

/* one query; the expansion trace goes to txy (absolute cells) when given */
static result solve(int algo, const int32_t* box, const uint8_t* map, float reso, float sx, float sy, float gx,
                    float gy, const work* w, int32_t* txy, int64_t cap, int64_t* tlen) {
  result r = {NO_PATH, 0, 0, NAN, -1};
  const int64_t W = (int64_t)box[2] - box[0], H = (int64_t)box[3] - box[1], cells = W * H;
  int isx, isy, igx, igy;
  if (!(cell_f(sx, reso, &isx) && cell_f(sy, reso, &isy) && cell_f(gx, reso, &igx) && cell_f(gy, reso, &igy))) {
    r.status = BAD_POINT;
    return r;
  }
  const int64_t rsx = (int64_t)isx - box[0], rsy = (int64_t)isy - box[1];
  const int64_t rgx = (int64_t)igx - box[0], rgy = (int64_t)igy - box[1];
  if (rsx < 0 || rsx >= W || rsy < 0 || rsy >= H) {
    r.status = START_OUTSIDE;
    return r;
  }
  const int64_t goal = (rgx >= 0 && rgx < W && rgy >= 0 && rgy < H) ? rgx * H + rgy : -1;
  memset(w->st, 0, (size_t)cells);
  if (algo == ASTAR)
    for (int64_t i = 0; i < cells; ++i) w->g[i] = FLT_MAX;
  const int64_t start = rsx * H + rsy;
  if (algo == ASTAR) w->g[start] = 0.0f;
  int64_t len = 0, nt = 0;
  entry e0 = {0.0f, (uint32_t)start << 3};
  heap_push(w->heap, &len, e0);
  int first = 1;
  while (len > 0) {
    const entry e = heap_pop(w->heap, &len);
    const int64_t cell = e.cd >> 3;
    if (w->st[cell] & 0x80) continue;
    w->st[cell] = first ? 0x88 : (uint8_t)(0x80 | (e.cd & 7));
    first = 0;
    ++r.n_visited;
    if (cell == goal) {
      r.status = FOUND;
      r.cost = e.key;
      r.goal_cell = goal;
      break;
    }
    const int64_t cx = cell / H, cy = cell % H;
    float gc = 0.0f, h = 0.0f;
    if (algo == ASTAR) {
      gc = w->g[cell];
      /* calc_heristic(ngoal, node) :95-97, at the expanded node */
      const double dx = (double)(rgx - cx), dy = (double)(rgy - cy);
      h = (float)(1.0 * sqrt(dx * dx + dy * dy));
    }
    for (int i = 0; i < 8; ++i) {
      const int64_t nx = cx + MX[i], ny = cy + MY[i];
      if (nx < 0 || nx >= W || ny < 0 || ny >= H) continue;
      const int64_t nc = nx * H + ny;
      if (map[nc]) continue;
      if (w->st[nc] & 0x80) continue;
      if (txy) {
        if (nt < cap) {
          txy[2 * nt] = (int32_t)(nx + box[0]);
          txy[2 * nt + 1] = (int32_t)(ny + box[1]);
        }
        ++nt;
      }
      const float step = i < 4 ? 1.0f : DIAG;
      if (algo == ASTAR) {
        const float ng = gc + step;
        if (ng < w->g[nc]) {
          w->g[nc] = ng;
          entry en = {ng + h, ((uint32_t)nc << 3) | (uint32_t)i};
          heap_push(w->heap, &len, en);
        }
      } else {
        entry en = {e.key + step, ((uint32_t)nc << 3) | (uint32_t)i};
        heap_push(w->heap, &len, en);
      }
    }
  }
  if (tlen) *tlen = nt;
  return r;
}

void crb_oracle_grid_plan(int algo, const int32_t* box, const uint8_t* map, float reso, int64_t n, const float* sg,
                          int max_pts, float* path, int32_t* path_len, float* cost, int32_t* n_visited,
                          int32_t* status, int nthreads) {
  const int64_t H = (int64_t)box[3] - box[1], cells = ((int64_t)box[2] - box[0]) * H;
  if (nthreads <= 0) nthreads = omp_get_max_threads();
#pragma omp parallel num_threads(nthreads)
  {
    work w;
    const int ok = work_alloc(&w, algo, cells);
#pragma omp for schedule(dynamic, 16)
    for (int64_t q = 0; q < n; ++q) {
      if (!ok) continue;
      result r = solve(algo, box, map, reso, sg[q], sg[n + q], sg[2 * n + q], sg[3 * n + q], &w, NULL, 0, NULL);
      int32_t plen = 0;
      if (r.status == FOUND) {
        /* calc_final_path: the goal, then its parents down to the start, (float)x * reso */
        int64_t c = r.goal_cell;
        for (;;) {
          if (path && plen < max_pts) {
            path[(2 * (int64_t)plen) * n + q] = (float)(c / H + box[0]) * reso;
            path[(2 * (int64_t)plen + 1) * n + q] = (float)(c % H + box[1]) * reso;
          }
          ++plen;
          const uint8_t s = w.st[c];
          if (s & 0x08) break;
          c -= MX[s & 7] * H + MY[s & 7];
        }
      }
      if (path_len) path_len[q] = plen;
      if (cost) cost[q] = r.cost;
      if (n_visited) n_visited[q] = r.n_visited;
      if (status) status[q] = r.status;
    }
    work_free(&w);
  }
}

int64_t crb_oracle_grid_trace(int algo, const int32_t* box, const uint8_t* map, float reso, float sx, float sy,
                              float gx, float gy, int32_t* txy, int64_t cap) {
  const int64_t cells = ((int64_t)box[2] - box[0]) * ((int64_t)box[3] - box[1]);
  work w;
  if (!work_alloc(&w, algo, cells)) {
    work_free(&w);
    return -1;
  }
  int64_t nt = 0;
  const result r = solve(algo, box, map, reso, sx, sy, gx, gy, &w, txy, cap, &nt);
  work_free(&w);
  return r.status == FOUND || r.status == NO_PATH ? nt : -1;
}

/* crb_oracle_grid.h — CPU checker for the grid planners of src/a_star.cpp and src/dijkstra.cpp (libcrb's
 * crb_grid_*).  Boxes are int32[4] = (min_x, min_y, max_x, max_y), the layout of crb_grid_box. */
#ifndef CRB_ORACLE_GRID_H_
#define CRB_ORACLE_GRID_H_
#include <stdint.h>

/* :115-140: 0, or -1 when n < 1, reso is not finite and > 0, or an obstacle rounds outside the int range */
int crb_oracle_grid_box(int64_t n_obs, const float* ox, const float* oy, float reso, int32_t* box);
/* calc_obstacle_map :48-78 into map [W*H], cell (x, y) at (x - min_x) * H + (y - min_y) */
void crb_oracle_grid_map(int64_t n_obs, const float* ox, const float* oy, float reso, float rr, const int32_t* box,
                         uint8_t* map);
/* the planners for n queries, crb_grid_plan_batched's layout and statuses; OpenMP over queries (nthreads 0 = all) */
void crb_oracle_grid_plan(int algo, const int32_t* box, const uint8_t* map, float reso, int64_t n, const float* sg,
                          int max_pts, float* path, int32_t* path_len, float* cost, int32_t* n_visited,
                          int32_t* status, int nthreads);
/* one query's expansion trace: every neighbour that passes verify_node and the visited check, in order, as absolute
 * cells (x, y) into txy [2 * cap]; returns the trace's full length, or -1 for a status other than FOUND / NO_PATH */
int64_t crb_oracle_grid_trace(int algo, const int32_t* box, const uint8_t* map, float reso, float sx, float sy,
                              float gx, float gy, int32_t* txy, int64_t cap);
/* the restated heap on its own: op[i] = 1 pushes keys[i] with id i, op[i] = 0 pops; the popped ids in order go to
 * popped (the number of pops is returned; a pop of an empty heap returns -1) */
int64_t crb_oracle_grid_heap_run(int64_t n_ops, const uint8_t* op, const float* keys, int32_t* popped);
#endif

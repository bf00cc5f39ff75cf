/* crb_oracle_rrt.h — CPU checker for RRT::planning of include/rrt.h (libcrb's crb_rrt_plan_batched): libstdc++'s
 * std::mt19937, uniform_int_distribution<int> and uniform_real_distribution<float>, glibc 2.39's atan2f and the
 * planner, written out with no libm or libstdc++ call in the generator, the distributions or atan2f. */
#ifndef CRB_ORACLE_RRT_H_
#define CRB_ORACLE_RRT_H_
#include <stdint.h>

/* the first n outputs of std::mt19937 seeded with seed */
void crb_oracle_rrt_mt_run(uint32_t seed, int64_t n, uint32_t* out);
/* the distributions fed from a fixed list of generator outputs u [n_u] (the crafted values of a test): kind 0 draws
 * uniform_int_distribution<int>(0, 100), kind 1 uniform_real_distribution<float>(a, b) as float bits, until fewer
 * than one draw's worth of values may remain.  out [k] gets the results, used [k] the values each draw consumed;
 * returns k */
int64_t crb_oracle_rrt_dist_run(int kind, float a, float b, int64_t n_u, const uint32_t* u, uint32_t* out,
                                int32_t* used);
/* glibc 2.39's __atanf and atan2f restated */
float crb_oracle_rrt_atanf(float x);
float crb_oracle_rrt_atan2f(float y, float x);
/* mismatches of crb_oracle_rrt_atanf against the host atanf over the bit patterns [lo_bits, hi_bits) (OpenMP) */
int64_t crb_oracle_rrt_atanf_census(uint32_t lo_bits, uint32_t hi_bits);
/* mismatches of crb_oracle_rrt_atan2f against the host atan2f over n pairs (y[i], x[i]) (OpenMP) */
int64_t crb_oracle_rrt_atan2f_pairs(int64_t n, const float* y, const float* x);
/* mismatches of crb_oracle_rrt_atanf against got [hi_bits - lo_bits] (the device's results) */
int64_t crb_oracle_rrt_atanf_check(uint32_t lo_bits, uint32_t hi_bits, const float* got);
/* mismatches of crb_oracle_rrt_atan2f against got [n] */
int64_t crb_oracle_rrt_atan2f_check(int64_t n, const float* y, const float* x, const float* got);

/* crb_rrt_plan_batched for n queries with crb_rrt_params' fields spelled out, its layouts, statuses and truncation;
 * draws [n] (or NULL) gets the number of generator outputs each query consumed, branches [n] (or NULL) bit 0 when a
 * uniform_int_distribution draw was redrawn and bit 1 when generate_canonical's 1.0 was mapped to nextafterf(1, 0).  OpenMP over queries (nthreads 0 =
 * all). */
void crb_oracle_rrt_plan(float rand_min, float rand_max, float expand_dis, int32_t goal_sample_rate, int32_t max_iter,
                         const float* ob, int32_t n_ob, int64_t n, const float* se, const uint32_t* seed, int32_t max_pts,
                         float* path, int32_t* path_len, int32_t max_nodes, float* tree, int32_t* parent,
                         int32_t* n_nodes, int32_t* n_iter, int32_t* status, int64_t* draws, int32_t* branches,
                         int nthreads);
#endif

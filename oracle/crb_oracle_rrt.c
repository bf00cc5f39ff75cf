/* crb_oracle_rrt.c — C restatement of RRT::planning (include/rrt.h:75-159, GetNearestNode :161-174, CollisionCheck
 * :176-181) for many seeded queries: the CPU checker of libcrb's crb_rrt_plan_batched.
 *
 * What the reference computes, built with GCC 13 / libstdc++ for x86-64 and glibc 2.39:
 *   - goal_gen is std::mt19937 (result_type is 64-bit there), restated below: seeding, twist, tempering.
 *   - goal_dis(goal_gen), a uniform_int_distribution<int>(0, 100), takes Lemire's path (_S_nd<uint64_t>): one 32x7-bit
 *     product, redrawn while its low word is below 2^32 mod 101 = 68; the result is the high word.
 *   - area_dis(goal_gen), a uniform_real_distribution<float>, is generate_canonical<float, 24>: one draw, (float)u / 2^32,
 *     with 1.0 (u >= 2^32 - 128) mapped to nextafterf(1, 0); then u01 * (b - a) + a in float.
 *   - std::pow(float, 2) promotes to double; a float's square is exact there.  The collision and goal tests take the
 *     double sqrt.  std::atan2 / std::cos / std::sin on floats are glibc's atan2f (restated below), cosf and sinf
 *     (crb_oracle_libm_sincosf of crb_oracle.c).
 * Built with -ffp-contract=off: every float expression rounds as written. */
#include "crb_oracle_rrt.h"

#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <omp.h>

#include "crb_oracle.h"

/* include/crb.h */
#define RRT_FOUND 0
#define RRT_MAX_ITER 1
#define RRT_BAD_INPUT 2

static uint32_t bits_of(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
}
static float float_of(uint32_t u) {
  float f;
  memcpy(&f, &u, 4);
  return f;
}

/* ---- std::mt19937 ------------------------------------------------------------------------------------------------ */
typedef struct {
  uint32_t x[624];
  int p;
  int64_t draws;
  int32_t branches; /* bit 0: a uniform_int_distribution redraw, bit 1: generate_canonical's 1.0 -> nextafterf */
} mt_t;

static void mt_seed(mt_t* m, uint32_t s) {
  m->x[0] = s;
  for (int i = 1; i < 624; ++i) m->x[i] = 1812433253u * (m->x[i - 1] ^ (m->x[i - 1] >> 30)) + (uint32_t)i;
  m->p = 624;
  m->draws = 0;
  m->branches = 0;
}

static void mt_twist(mt_t* m) {
  uint32_t* x = m->x;
  for (int k = 0; k < 624; ++k) {
    const uint32_t y = (x[k] & 0x80000000u) | (x[(k + 1) % 624] & 0x7fffffffu);
    x[k] = x[k < 227 ? k + 397 : k - 227] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
  }
  m->p = 0;
}

static uint32_t mt_next(mt_t* m) {
  if (m->p >= 624) mt_twist(m);
  uint32_t z = m->x[m->p++];
  z ^= z >> 11;
  z ^= (z << 7) & 0x9d2c5680u;
  z ^= (z << 15) & 0xefc60000u;
  z ^= z >> 18;
  m->draws++;
  return z;
}

void crb_oracle_rrt_mt_run(uint32_t seed, int64_t n, uint32_t* out) {
  mt_t* m = (mt_t*)malloc(sizeof(mt_t));
  mt_seed(m, seed);
  for (int64_t i = 0; i < n; ++i) out[i] = mt_next(m);
  free(m);
}

/* ---- the two distributions, on any source of 32-bit values ------------------------------------------------------ */
typedef uint32_t (*draw_fn)(void* src);

/* uniform_int_distribution<int>(0, 100): _S_nd<uint64_t>(g, 101); *branches (or NULL) gets bit 0 on a redraw */
static int uid_0_100(draw_fn g, void* src, int32_t* branches) {
  uint64_t prod = (uint64_t)g(src) * 101u;
  uint32_t low = (uint32_t)prod;
  if (low < 101u) {
    if (branches && low < 68u) *branches |= 1;
    while (low < 68u) { /* -101 % 101 in 32 bits */
      prod = (uint64_t)g(src) * 101u;
      low = (uint32_t)prod;
    }
  }
  return (int)(prod >> 32);
}

/* uniform_real_distribution<float>(a, b): generate_canonical<float, 24> then u01 * (b - a) + a; *branches (or NULL)
 * gets bit 1 when the canonical value rounds to 1 */
static float ureal(draw_fn g, void* src, float a, float b, int32_t* branches) {
  const float sum = 0.0f + (float)g(src) * 1.0f;
  float r = sum / 4294967296.0f;
  if (r >= 1.0f) {
    r = float_of(0x3f7fffffu);
    if (branches) *branches |= 2;
  }
  return r * (b - a) + a;
}

static uint32_t draw_mt(void* m) { return mt_next((mt_t*)m); }

typedef struct {
  const uint32_t* u;
  int64_t n, pos;
  int dry; /* a value past the end was asked for */
} list_src;
static uint32_t draw_list(void* s) {
  list_src* l = (list_src*)s;
  if (l->pos < l->n) return l->u[l->pos++];
  l->dry = 1;
  return 0xffffffffu; /* ends a redraw loop: (2^32 - 1) * 101 has the low word 2^32 - 101 */
}

int64_t crb_oracle_rrt_dist_run(int kind, float a, float b, int64_t n_u, const uint32_t* u, uint32_t* out,
                                int32_t* used) {
  list_src l = {u, n_u, 0, 0};
  int64_t k = 0;
  while (l.pos < n_u) {
    const int64_t p0 = l.pos;
    const uint32_t r = kind == 0 ? (uint32_t)uid_0_100(draw_list, &l, NULL) : bits_of(ureal(draw_list, &l, a, b, NULL));
    if (l.dry) break;
    out[k] = r;
    used[k++] = (int32_t)(l.pos - p0);
  }
  return k;
}

/* ---- glibc 2.39's atanf / atan2f: fdlibm's binary32 s_atanf.c and e_atan2f.c (Sun Microsystems, freely
 * redistributable), every operation in float ---------------------------------------------------------------------- */
static const float atanhi[] = {4.6364760399e-01f, 7.8539812565e-01f, 9.8279368877e-01f, 1.5707962513e+00f};
static const float atanlo[] = {5.0121582440e-09f, 3.7748947079e-08f, 3.4473217170e-08f, 7.5497894159e-08f};
static const float aT[] = {3.3333334327e-01f, -2.0000000298e-01f, 1.4285714924e-01f, -1.1111110449e-01f,
                           9.0908870101e-02f, -7.6918758452e-02f, 6.6610731184e-02f, -5.8335702866e-02f,
                           4.9768779427e-02f, -3.6531571299e-02f, 1.6285819933e-02f};

float crb_oracle_rrt_atanf(float x) {
  const int32_t hx = (int32_t)bits_of(x);
  const int32_t ix = hx & 0x7fffffff;
  int id;
  if (ix >= 0x4c000000) { /* |x| >= 2^25 */
    if (ix > 0x7f800000) return x + x;
    return hx > 0 ? atanhi[3] + atanlo[3] : -atanhi[3] - atanlo[3];
  }
  if (ix < 0x3ee00000) { /* |x| < 0.4375 */
    if (ix < 0x31000000) return x; /* |x| < 2^-29 */
    id = -1;
  } else {
    x = fabsf(x);
    if (ix < 0x3f980000) {   /* |x| < 1.1875 */
      if (ix < 0x3f300000) { /* 7/16 <= |x| < 11/16 */
        id = 0;
        x = (2.0f * x - 1.0f) / (2.0f + x);
      } else { /* 11/16 <= |x| < 19/16 */
        id = 1;
        x = (x - 1.0f) / (x + 1.0f);
      }
    } else {
      if (ix < 0x401c0000) { /* |x| < 2.4375 */
        id = 2;
        x = (x - 1.5f) / (1.0f + 1.5f * x);
      } else { /* 2.4375 <= |x| < 2^25 */
        id = 3;
        x = -1.0f / x;
      }
    }
  }
  const float z = x * x;
  const float w = z * z;
  const float s1 = z * (aT[0] + w * (aT[2] + w * (aT[4] + w * (aT[6] + w * (aT[8] + w * aT[10])))));
  const float s2 = w * (aT[1] + w * (aT[3] + w * (aT[5] + w * (aT[7] + w * aT[9]))));
  if (id < 0) return x - x * (s1 + s2);
  const float r = atanhi[id] - ((x * (s1 + s2) - atanlo[id]) - x);
  return hx < 0 ? -r : r;
}

float crb_oracle_rrt_atan2f(float y, float x) {
  const float tiny = 1.0e-30f, pi_o_4 = 7.8539818525e-01f, pi_o_2 = 1.5707963705e+00f, pi = 3.1415927410e+00f,
              pi_lo = -8.7422776573e-08f;
  const int32_t hx = (int32_t)bits_of(x), ix = hx & 0x7fffffff;
  const int32_t hy = (int32_t)bits_of(y), iy = hy & 0x7fffffff;
  if (ix > 0x7f800000 || iy > 0x7f800000) return x + y; /* NaN */
  if (hx == 0x3f800000) return crb_oracle_rrt_atanf(y); /* x = 1 */
  const int m = ((hy >> 31) & 1) | ((hx >> 30) & 2);   /* 2 * sign(x) + sign(y) */
  if (iy == 0) {
    switch (m) {
      case 0:
      case 1: return y;
      case 2: return pi + tiny;
      default: return -pi - tiny;
    }
  }
  if (ix == 0) return hy < 0 ? -pi_o_2 - tiny : pi_o_2 + tiny;
  if (ix == 0x7f800000) {
    if (iy == 0x7f800000) {
      switch (m) {
        case 0: return pi_o_4 + tiny;
        case 1: return -pi_o_4 - tiny;
        case 2: return 3.0f * pi_o_4 + tiny;
        default: return -3.0f * pi_o_4 - tiny;
      }
    }
    switch (m) {
      case 0: return 0.0f;
      case 1: return -0.0f;
      case 2: return pi + tiny;
      default: return -pi - tiny;
    }
  }
  if (iy == 0x7f800000) return hy < 0 ? -pi_o_2 - tiny : pi_o_2 + tiny;
  const int32_t k = (iy - ix) >> 23;
  float z;
  if (k > 60) z = pi_o_2 + 0.5f * pi_lo; /* |y / x| > 2^60 */
  else if (hx < 0 && k < -60) z = 0.0f;   /* |y| / x < -2^60 */
  else z = crb_oracle_rrt_atanf(fabsf(y / x));
  switch (m) {
    case 0: return z;
    case 1: return float_of(bits_of(z) ^ 0x80000000u);
    case 2: return pi - (z - pi_lo);
    default: return (z - pi_lo) - pi;
  }
}

static int differ(float a, float b) { return bits_of(a) != bits_of(b) && !(isnan(a) && isnan(b)); }

int64_t crb_oracle_rrt_atanf_census(uint32_t lo_bits, uint32_t hi_bits) {
  int64_t bad = 0;
#pragma omp parallel for reduction(+ : bad) schedule(static, 1 << 16)
  for (int64_t u = lo_bits; u < (int64_t)hi_bits; ++u) {
    const float x = float_of((uint32_t)u);
    volatile float h = atanf(x);
    bad += differ(h, crb_oracle_rrt_atanf(x));
  }
  return bad;
}

int64_t crb_oracle_rrt_atan2f_pairs(int64_t n, const float* y, const float* x) {
  int64_t bad = 0;
#pragma omp parallel for reduction(+ : bad) schedule(static, 1 << 14)
  for (int64_t i = 0; i < n; ++i) {
    volatile float h = atan2f(y[i], x[i]);
    bad += differ(h, crb_oracle_rrt_atan2f(y[i], x[i]));
  }
  return bad;
}

int64_t crb_oracle_rrt_atanf_check(uint32_t lo_bits, uint32_t hi_bits, const float* got) {
  int64_t bad = 0;
#pragma omp parallel for reduction(+ : bad) schedule(static, 1 << 16)
  for (int64_t u = lo_bits; u < (int64_t)hi_bits; ++u)
    bad += differ(got[u - lo_bits], crb_oracle_rrt_atanf(float_of((uint32_t)u)));
  return bad;
}

int64_t crb_oracle_rrt_atan2f_check(int64_t n, const float* y, const float* x, const float* got) {
  int64_t bad = 0;
#pragma omp parallel for reduction(+ : bad) schedule(static, 1 << 14)
  for (int64_t i = 0; i < n; ++i) bad += differ(got[i], crb_oracle_rrt_atan2f(y[i], x[i]));
  return bad;
}

/* ---- RRT::planning ----------------------------------------------------------------------------------------------- */
/* (float)(pow(dx, 2) + pow(dy, 2)) with float dx, dy: the squares are exact in double */
static double sq2(float dx, float dy) { return (double)dx * (double)dx + (double)dy * (double)dy; }

static void put_point(float* path, int64_t n, int64_t q, int32_t max_pts, int32_t k, float x, float y) {
  if (path && k < max_pts) {
    path[(2 * (int64_t)k) * n + q] = x;
    path[(2 * (int64_t)k + 1) * n + q] = y;
  }
}

void crb_oracle_rrt_plan(float rand_min, float rand_max, float expand_dis, int32_t goal_sample_rate, int32_t max_iter,
                         const float* ob, int32_t n_ob, int64_t n, const float* se, const uint32_t* seed, int32_t max_pts,
                         float* path, int32_t* path_len, int32_t max_nodes, float* tree, int32_t* parent,
                         int32_t* n_nodes, int32_t* n_iter, int32_t* status, int64_t* draws, int32_t* branches,
                         int nthreads) {
  int ob_ok = 1;
  for (int32_t j = 0; j < 3 * n_ob; ++j) ob_ok &= isfinite(ob[j]) != 0;
  if (nthreads <= 0) nthreads = omp_get_max_threads();
#pragma omp parallel num_threads(nthreads)
  {
    mt_t* m = (mt_t*)malloc(sizeof(mt_t));
    float* nx = (float*)malloc(sizeof(float) * 2 * ((size_t)max_iter + 1));
    float* ny = nx + max_iter + 1;
    int32_t* par = (int32_t*)malloc(sizeof(int32_t) * ((size_t)max_iter + 1));
#pragma omp for schedule(dynamic, 16)
    for (int64_t q = 0; q < n; ++q) {
      const float sx = se[q], sy = se[n + q], gx = se[2 * n + q], gy = se[3 * n + q];
      mt_seed(m, seed[q]);
      int32_t st = RRT_MAX_ITER, nn = 0, it = 0, plen = 0;
      if (!(ob_ok && isfinite(sx) && isfinite(sy) && isfinite(gx) && isfinite(gy))) {
        st = RRT_BAD_INPUT;
      } else {
        nx[0] = sx;
        ny[0] = sy;
        par[0] = -1;
        nn = 1;
        while (it < max_iter) {
          ++it;
          float rx, ry;
          if (uid_0_100(draw_mt, m, &m->branches) > goal_sample_rate) {
            rx = ureal(draw_mt, m, rand_min, rand_max, &m->branches);
            ry = ureal(draw_mt, m, rand_min, rand_max, &m->branches);
          } else {
            rx = gx;
            ry = gy;
          }
          /* GetNearestNode: strict < from FLT_MAX, the first minimum wins and NaN never does */
          float best = FLT_MAX;
          int32_t bi = -1;
          for (int32_t i = 0; i < nn; ++i) {
            const float d = (float)sq2(nx[i] - rx, ny[i] - ry);
            if (d < best) {
              best = d;
              bi = i;
            }
          }
          if (bi < 0) { /* the reference would read node_list[-1] */
            st = RRT_BAD_INPUT;
            break;
          }
          const float theta = crb_oracle_rrt_atan2f(ry - ny[bi], rx - nx[bi]);
          float sn, cs;
          crb_oracle_libm_sincosf(theta, &sn, &cs);
          const float px = nx[bi] + expand_dis * cs, py = ny[bi] + expand_dis * sn;
          int hit = 0;
          for (int32_t j = 0; j < n_ob && !hit; ++j)
            hit = sqrt(sq2(ob[3 * j] - px, ob[3 * j + 1] - py)) <= (double)ob[3 * j + 2];
          if (hit) continue;
          nx[nn] = px;
          ny[nn] = py;
          par[nn] = bi;
          ++nn;
          if (sqrt(sq2(px - gx, py - gy)) <= (double)expand_dis) {
            st = RRT_FOUND;
            break;
          }
        }
      }
      if (st == RRT_FOUND) {
        /* end, then node_list.back() and its parents down to (not including) the start, then start */
        put_point(path, n, q, max_pts, plen++, gx, gy);
        for (int32_t c = nn - 1; par[c] >= 0; c = par[c]) put_point(path, n, q, max_pts, plen++, nx[c], ny[c]);
        put_point(path, n, q, max_pts, plen++, sx, sy);
      }
      const int32_t w = nn < max_nodes ? nn : max_nodes;
      for (int32_t k = 0; k < w; ++k) {
        if (tree) {
          tree[(2 * (int64_t)k) * n + q] = nx[k];
          tree[(2 * (int64_t)k + 1) * n + q] = ny[k];
        }
        if (parent) parent[(int64_t)k * n + q] = par[k];
      }
      if (path_len) path_len[q] = plen;
      if (n_nodes) n_nodes[q] = nn;
      if (n_iter) n_iter[q] = it;
      if (status) status[q] = st;
      if (draws) draws[q] = m->draws;
      if (branches) branches[q] = m->branches;
    }
    free(par);
    free(nx);
    free(m);
  }
}

// crb_rrt.cu — RRT::planning (include/rrt.h:75-159) for many seeded start / goal queries, on one obstacle list or on
// an obstacle list per query (crb.h's obstacle store), for sm_90a.
//
// Bit-exact with the reference built for x86-64 with GCC 13 / libstdc++ and glibc 2.39, after goal_gen.seed(seed):
//   - goal_gen, a std::mt19937: libstdc++'s seeding, twist and tempering.  Both distributions draw from it (area_gen
//     is never used).  goal_dis, uniform_int_distribution<int>(0, 100), takes Lemire's path because mt19937's
//     result_type is 64-bit there: u * 101 in 64 bits, redrawn while the low word is below 2^32 mod 101 = 68, the high
//     word is the result.  area_dis, uniform_real_distribution<float>, is generate_canonical<float, 24> on one draw,
//     (float)u / 2^32 with 1.0 mapped to nextafterf(1, 0), then u01 * (b - a) + a in float.
//   - GetNearestNode's std::pow(float, 2) promotes to double, where a float's square is exact, so
//     (float)(pow(dx, 2) + pow(dy, 2)) is one double fma and a narrowing.  The collision and goal tests keep the
//     double sqrt.  std::atan2 / std::cos / std::sin on floats are glibc's atan2f, cosf, sinf (crb_common.cuh).
//   - Every float and double operation is an explicitly rounded intrinsic, so the TU's -fmad setting does not matter.
//
// Mapping: one warp per query.  A query's iterations are serial (each draw depends on the tree so far), but inside an
// iteration the warp splits the nearest-node scan (lane-strided strict-< passes, then a (distance, index) butterfly that
// keeps the first minimum), the obstacle test (lane-strided, then a vote) and the generator's twist (20 steps of 32
// words, in the order that keeps every read of the sequential twist).  The draws, atan2f and sincosf are computed by
// every lane alike, so control flow stays uniform.  Warps are persistent: one warp per block, each takes its next query
// from an atomic counter, because query lengths differ by 2x and more.  Both entry points run the same kernel: a
// query's obstacles are rows [b, e) of the store (every query on [0, n_ob) for the shared list), read lane-strided
// from global memory through its own base pointer, and checked finite once per query.
//
// Shared memory per warp (dynamic, sized from max_iter): the generator's 624 words, then node coordinates (float2) and
// parent indices (int16) for max_iter + 1 nodes.  Parents stay in shared memory rather than only in the optional global
// output: the path is walked from them, and the caller may ask for no tree at all.
#include <float.h>

#include "crb_common.cuh"

namespace {

constexpr int kMtN = 624;
constexpr unsigned kFull = 0xffffffffu;

struct RrtArgs {
  float rand_min, rand_max, e;
  int32_t gsr, max_iter;
  const float* ob;
  int64_t n_rows;
  const int64_t* ob_off;  // NULL: every query on rows [0, n_rows)
  int32_t n_sets;
  const int32_t* ob_of;
  int64_t n;
  const float* se;
  const uint32_t* seed;
  int32_t max_pts;
  float* path;
  int32_t* path_len;
  int32_t max_nodes;
  float* tree;
  int32_t* parent;
  int32_t* n_nodes;
  int32_t* n_iter;
  int32_t* status;
  unsigned long long* counter;
};

size_t rrt_smem_bytes(int32_t max_iter) {
  const size_t nodes = (size_t)max_iter + 1;
  return (kMtN * 4 + nodes * 8 + nodes * 2 + 15) / 16 * 16;
}

// libstdc++'s _M_gen_rand by the warp: word k becomes x[k + 397 or k - 227] ^ f(x[k], x[k + 1]), where words below k
// are already new and words above k still old.  Lanes take 32 consecutive words per step and read before any of them
// writes; the word at k - 227 was written at least seven steps earlier and the one at k + 397 is written seven later.
__device__ __forceinline__ void mt_twist(uint32_t* x, int lane) {
  for (int base = 0; base < kMtN; base += 32) {
    const int k = base + lane;
    uint32_t v = 0;
    if (k < kMtN) {
      const uint32_t y = (x[k] & 0x80000000u) | (x[k == kMtN - 1 ? 0 : k + 1] & 0x7fffffffu);
      v = x[k < 227 ? k + 397 : k - 227] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    __syncwarp();
    if (k < kMtN) x[k] = v;
    __syncwarp();
  }
}

// the next output, the same in every lane
__device__ __forceinline__ uint32_t mt_next(uint32_t* x, int& p, int lane) {
  if (p >= kMtN) {
    mt_twist(x, lane);
    p = 0;
  }
  uint32_t z = x[p++];
  z ^= z >> 11;
  z ^= (z << 7) & 0x9d2c5680u;
  z ^= (z << 15) & 0xefc60000u;
  z ^= z >> 18;
  return z;
}

// uniform_int_distribution<int>(0, 100)
__device__ __forceinline__ int uid_0_100(uint32_t* x, int& p, int lane) {
  uint64_t prod = (uint64_t)mt_next(x, p, lane) * 101u;
  while ((uint32_t)prod < 68u) prod = (uint64_t)mt_next(x, p, lane) * 101u;
  return (int)(prod >> 32);
}

// uniform_real_distribution<float>(a, b)
__device__ __forceinline__ float ureal(uint32_t* x, int& p, int lane, float a, float b) {
  float r = __fmul_rn(__uint2float_rn(mt_next(x, p, lane)), 0x1p-32f);  // (float)u / 2^32: exact scaling
  if (r >= 1.0f) r = __uint_as_float(0x3f7fffffu);
  return __fadd_rn(__fmul_rn(r, __fsub_rn(b, a)), a);
}

// (pow(dx, 2) + pow(dy, 2)) in double for float dx, dy: both squares are exact
__device__ __forceinline__ double sq2(float dx, float dy) {
  const double x = (double)dx, y = (double)dy;
  return __fma_rn(x, x, __dmul_rn(y, y));
}

}  // namespace

// Launched with 32 threads per block.  The query's obstacle base and count, held in registers through the loop, would
// take ptxas from 58 to 64 registers; the cap keeps 58 with no spill.
__global__ void __maxnreg__(58) crb_rrt_plan_kernel(const RrtArgs a) {
  extern __shared__ __align__(16) uint32_t smem[];
  uint32_t* mt = smem;
  float2* node = (float2*)(smem + kMtN);
  int16_t* par = (int16_t*)(node + a.max_iter + 1);
  const int lane = threadIdx.x;
  const int64_t n = a.n;
  const float e = a.e;
  for (;;) {
    unsigned long long qq = 0;
    if (lane == 0) qq = atomicAdd(a.counter, 1ull);
    const int64_t q = (int64_t)__shfl_sync(kFull, qq, 0);
    if (q >= n) return;
    const float sx = a.se[q], sy = a.se[n + q], gx = a.se[2 * n + q], gy = a.se[3 * n + q];
    // the query's obstacles, then every value of them finite, or the query is BAD_INPUT
    int64_t ob0, ob1;
    const bool ref_ok = crb_obstacle_list(q, a.ob_off, a.n_sets, a.ob_of, a.n_rows, INT32_MAX / 3, ob0, ob1);
    const float* ob = a.ob + 3 * ob0;
    const int32_t n_ob = (int32_t)(ob1 - ob0);
    bool ob_ok = true;
    for (int j = lane; j < 3 * n_ob; j += 32) ob_ok &= isfinite(__ldg(ob + j));
    ob_ok = __all_sync(kFull, ob_ok);
    // goal_gen.seed(s): every lane runs the recurrence, lane k % 32 stores word k
    {
      uint32_t v = a.seed[q];
      if (lane == 0) mt[0] = v;
      for (int k = 1; k < kMtN; ++k) {
        v = 1812433253u * (v ^ (v >> 30)) + (uint32_t)k;
        if ((k & 31) == lane) mt[k] = v;
      }
      __syncwarp();
    }
    int p = kMtN;
    int32_t st = CRB_RRT_MAX_ITER_REACHED, nn = 0, it = 0;
    if (!ref_ok) {
      st = CRB_RRT_BAD_OBSTACLES;
    } else if (!(ob_ok && isfinite(sx) && isfinite(sy) && isfinite(gx) && isfinite(gy))) {
      st = CRB_RRT_BAD_INPUT;
    } else {
      if (lane == 0) {
        node[0] = make_float2(sx, sy);
        par[0] = -1;
      }
      nn = 1;
      __syncwarp();
      while (it < a.max_iter) {
        ++it;
        float rx = gx, ry = gy;
        if (uid_0_100(mt, p, lane) > a.gsr) {
          rx = ureal(mt, p, lane, a.rand_min, a.rand_max);
          ry = ureal(mt, p, lane, a.rand_min, a.rand_max);
        }
        // GetNearestNode: strict < from FLT_MAX, so the first minimum wins and NaN never does
        float bd = FLT_MAX;
        int bi = INT32_MAX;
#pragma unroll 4
        for (int i = lane; i < nn; i += 32) {
          const float2 nd = node[i];
          const float d = __double2float_rn(sq2(__fsub_rn(nd.x, rx), __fsub_rn(nd.y, ry)));
          if (d < bd) {
            bd = d;
            bi = i;
          }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
          const float od = __shfl_xor_sync(kFull, bd, off);
          const int oi = __shfl_xor_sync(kFull, bi, off);
          if (od < bd || (od == bd && oi < bi)) {
            bd = od;
            bi = oi;
          }
        }
        if (bi == INT32_MAX) {  // no winner: the reference would read node_list[-1]
          st = CRB_RRT_BAD_INPUT;
          break;
        }
        const float2 nb = node[bi];
        const float theta = crb_atan2f_libm(__fsub_rn(ry, nb.y), __fsub_rn(rx, nb.x));
        float sn, cs;
        crb_sincosf_libm(theta, sn, cs);
        const float px = __fadd_rn(nb.x, __fmul_rn(e, cs)), py = __fadd_rn(nb.y, __fmul_rn(e, sn));
        // CollisionCheck: the new point only
        bool hit = false;
        for (int j = lane; j < n_ob; j += 32) {
          const float ox = __ldg(ob + 3 * j), oy = __ldg(ob + 3 * j + 1), r = __ldg(ob + 3 * j + 2);
          hit |= __dsqrt_rn(sq2(__fsub_rn(ox, px), __fsub_rn(oy, py))) <= (double)r;
        }
        if (__any_sync(kFull, hit)) continue;
        if (lane == 0) {
          node[nn] = make_float2(px, py);
          par[nn] = (int16_t)bi;
        }
        ++nn;
        __syncwarp();
        if (__dsqrt_rn(sq2(__fsub_rn(px, gx), __fsub_rn(py, gy))) <= (double)e) {
          st = CRB_RRT_FOUND;
          break;
        }
      }
    }
    // node_list in insertion order
    const int32_t w = nn < a.max_nodes ? nn : a.max_nodes;
    for (int k = lane; k < w; k += 32) {
      if (a.tree) {
        const float2 nd = node[k];
        a.tree[(2 * (int64_t)k) * n + q] = nd.x;
        a.tree[(2 * (int64_t)k + 1) * n + q] = nd.y;
      }
      if (a.parent) a.parent[(int64_t)k * n + q] = par[k];
    }
    if (lane == 0) {
      int32_t plen = 0;
      if (st == CRB_RRT_FOUND) {
        // the goal, then node_list.back() and its parents down to node 0, the start (which the reference appends as
        // `start`: the same point)
        float x = gx, y = gy;
        for (int c = nn - 1;; c = par[c]) {
          if (a.path && plen < a.max_pts) {
            a.path[(2 * (int64_t)plen) * n + q] = x;
            a.path[(2 * (int64_t)plen + 1) * n + q] = y;
          }
          ++plen;
          if (c < 0) break;
          x = node[c].x;
          y = node[c].y;
        }
      }
      if (a.path_len) a.path_len[q] = plen;
      if (a.n_nodes) a.n_nodes[q] = nn;
      if (a.n_iter) a.n_iter[q] = it;
      if (a.status) a.status[q] = st;
    }
    __syncwarp();  // the next query overwrites the generator and the nodes
  }
}

extern "C" {

void crb_rrt_default_params(crb_rrt_params* p) {
  // include/rrt.h:61 (expand_dis 1.0, goal_sample_rate 5, max_iter 500); src/rrt.cpp:30 rand_area {-2, 15}
  p->rand_min = -2.0f;
  p->rand_max = 15.0f;
  p->expand_dis = 1.0f;
  p->goal_sample_rate = 5;
  p->max_iter = 500;
}

}  // extern "C"

// The argument checks both entry points share (everything but the obstacles).
static int rrt_check_args(crb_ctx* ctx, const crb_rrt_params* prm, int64_t n, const float* se, const uint32_t* seed,
                          int32_t max_pts, int32_t max_nodes) {
  CRB_REQUIRE(ctx != nullptr && prm != nullptr, "ctx or prm is NULL");
  CRB_REQUIRE(isfinite(prm->rand_min) && isfinite(prm->rand_max) && prm->rand_min <= prm->rand_max,
              "rand_min and rand_max must be finite with rand_min <= rand_max");
  CRB_REQUIRE(isfinite(prm->expand_dis), "expand_dis must be finite");
  CRB_REQUIRE(prm->max_iter >= 1 && prm->max_iter <= CRB_RRT_MAX_ITER, "max_iter must be in [1, CRB_RRT_MAX_ITER]");
  CRB_REQUIRE(n >= 0 && n <= INT64_MAX / 4, "n out of range");
  CRB_REQUIRE(max_pts >= 0 && max_nodes >= 0, "max_pts and max_nodes must be >= 0");
  CRB_REQUIRE(n <= INT64_MAX / 2 / ((max_pts > max_nodes ? max_pts : max_nodes) + 1), "n * max_pts out of range");
  CRB_REQUIRE(n == 0 || (se && seed), "se or seed is NULL");
  return CRB_OK;
}

// No device, no computation (crb_require_device); then the launch, n > 0.
static int rrt_launch(crb_ctx* ctx, const char* fn, const crb_rrt_params* prm, const float* ob, int64_t n_rows,
                      const int64_t* ob_off, int32_t n_sets, const int32_t* ob_of, int64_t n, const float* se,
                      const uint32_t* seed, int32_t max_pts, float* path, int32_t* path_len, int32_t max_nodes,
                      float* tree, int32_t* parent, int32_t* n_nodes, int32_t* n_iter, int32_t* status) {
  const int rc = crb_require_device(fn);
  if (rc != CRB_OK) return rc;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  if (ctx->rrt_counter == nullptr) CRB_CUDA(cudaMalloc(&ctx->rrt_counter, sizeof(unsigned long long)));
  const size_t smem = rrt_smem_bytes(prm->max_iter);
  CRB_CUDA(cudaFuncSetAttribute(crb_rrt_plan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  CRB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, crb_rrt_plan_kernel, 32, smem));
  const int64_t resident = (int64_t)(per_sm > 0 ? per_sm : 1) * ctx->sm_count;
  RrtArgs a;
  a.rand_min = prm->rand_min;
  a.rand_max = prm->rand_max;
  a.e = prm->expand_dis;
  a.gsr = prm->goal_sample_rate;
  a.max_iter = prm->max_iter;
  a.ob = ob;
  a.n_rows = n_rows;
  a.ob_off = ob_off;
  a.n_sets = n_sets;
  a.ob_of = ob_of;
  a.n = n;
  a.se = se;
  a.seed = seed;
  a.max_pts = max_pts;
  a.path = max_pts > 0 ? path : nullptr;
  a.path_len = path_len;
  a.max_nodes = max_nodes;
  a.tree = max_nodes > 0 ? tree : nullptr;
  a.parent = max_nodes > 0 ? parent : nullptr;
  a.n_nodes = n_nodes;
  a.n_iter = n_iter;
  a.status = status;
  a.counter = (unsigned long long*)ctx->rrt_counter;
  CRB_CUDA(cudaMemsetAsync(a.counter, 0, sizeof(unsigned long long), ctx->stream));
  crb_rrt_plan_kernel<<<(unsigned)(n < resident ? n : resident), 32, smem, ctx->stream>>>(a);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

extern "C" {

int crb_rrt_plan_batched(crb_ctx* ctx, const crb_rrt_params* prm, const float* ob, int32_t n_ob, int64_t n,
                         const float* se, const uint32_t* seed, int32_t max_pts, float* path, int32_t* path_len,
                         int32_t max_nodes, float* tree, int32_t* parent, int32_t* n_nodes, int32_t* n_iter,
                         int32_t* status) {
  int rc = rrt_check_args(ctx, prm, n, se, seed, max_pts, max_nodes);
  if (rc != CRB_OK) return rc;
  CRB_REQUIRE(n_ob >= 0 && n_ob <= INT32_MAX / 3, "n_ob out of range");
  CRB_REQUIRE(n == 0 || n_ob == 0 || ob, "ob is NULL");
  return rrt_launch(ctx, __func__, prm, ob, n_ob, nullptr, 1, nullptr, n, se, seed, max_pts, path, path_len, max_nodes,
                    tree, parent, n_nodes, n_iter, status);
}

int crb_rrt_plan_many_batched(crb_ctx* ctx, const crb_rrt_params* prm, const float* ob, int64_t n_rows,
                              const int64_t* ob_off, int32_t n_sets, const int32_t* ob_of, int64_t n, const float* se,
                              const uint32_t* seed, int32_t max_pts, float* path, int32_t* path_len, int32_t max_nodes,
                              float* tree, int32_t* parent, int32_t* n_nodes, int32_t* n_iter, int32_t* status) {
  int rc = rrt_check_args(ctx, prm, n, se, seed, max_pts, max_nodes);
  if (rc != CRB_OK) return rc;
  CRB_REQUIRE(n_sets >= 1 && n_rows >= 0, "n_sets must be >= 1 and n_rows >= 0");
  CRB_REQUIRE(n == 0 || (ob_off && ob_of && (ob || n_rows == 0)), "ob, ob_off or ob_of is NULL");
  return rrt_launch(ctx, __func__, prm, ob, n_rows, ob_off, n_sets, ob_of, n, se, seed, max_pts, path, path_len,
                    max_nodes, tree, parent, n_nodes, n_iter, status);
}

}  // extern "C"

// crb_mpc_tasks.cu — resident-slot MPC solver for sm_90a: persistent CTAs, roll-outs in shared memory,
// sweeps regrouped by kind.
//
// Same solver, same bits as crb_mpc_solve_kernel (crb_mpc.cu) and oracle/crb_oracle_mpc.c; replaces
// mpc_solve() + FG_EVAL, src/model_predictive_control.cpp:188-346.  What changes is WHERE a problem lives
// and WHO advances it:
//
//   * One persistent CTA per SM.  A CTA owns S problem SLOTS.  Both roll-out buffers of a slot (X, U: the
//     data every sweep reads and writes with a dependent chain behind it) and its scalar state stay in
//     SHARED MEMORY for the whole solve (976 B per slot at T = 20, up to MPC_TASK_SLOTS per SM).  The stage gains and
//     the translated reference (written once per backward sweep / once per problem, read by the next
//     forward sweeps) go to a per-CTA slab of 80-byte stage records in global memory that the CTA reuses for
//     every problem it ever solves (SMs x S x 1.5 KB), kept in L2 by an evict_last policy.  The first version
//     of the solver streamed a 2.3 KB per-problem workspace through HBM ~20 times per solve; here DRAM sees
//     mostly the inputs and the outputs.
//   * A problem is advanced one SWEEP at a time (refill = retire + load + initial roll-out, backward,
//     forward); between sweeps everything it needs is in its slot, so ANY thread can run its next sweep.
//     Each warp repeatedly takes up to 32 slots that wait for the same kind of sweep and runs that sweep
//     with one problem per lane.  An adaptive solver diverges badly under a fixed problem-to-lane map
//     (4..15 outer iterations, 1..5 line-search passes: 16.5 of 32 lanes active in the first version);
//     regrouped, the lanes of a warp always execute the same sweep kind for the same stage count.
//   * Problems are pulled from a global counter 32 at a time, so the CTAs balance themselves and the
//     inputs of a refill are coalesced 128-byte rows of the SoA arrays.
//
// Scheduling state per CTA (shared memory): one ring queue of waiting slots per sweep kind and one lock
// word.  A warp enters ONE short critical section per task: it appends the slots of the sweep it just
// finished to the queues of the kinds they wait for next, then takes up to 32 slots from the fullest
// queue.  (The first version scanned a phase word per slot with 40 ballots under the lock, and warps spent
// much of their time in that scan and in the lock's spin loop.)  Warps that find nothing wait on a
// sequence word that every post bumps, not on the lock.  All waiting loops are bounded: on overrun the
// kernel raises the error word in the slab header instead of hanging the GPU.
#include "crb_common.cuh"
#include "crb_mpc_core.cuh"
#include "crb_mpc_tasks.cuh"

#define MPC_TASK_QS 256  // ring size of the per-kind queues (power of two >= slots per CTA)
// Slots per CTA at most.  The per-CTA stage-record slabs (SMs x S x (T-1) x 80 B) must leave the 50 MB L2 room
// for the streaming inputs and outputs: at T = 20 the ~230 slots that shared memory holds make a 46 MB slab.
// Measured on an H100 SXM (400 W limit), 2^16 problems, T = 20: 52 M solves/s at 160 slots vs 44 M at 230.
#define MPC_TASK_SLOTS 160

struct MpcTaskArgs {
  int64_t count, ld_in, ld_out;
  int T, S, slot_words;
  int fill_min;                // scheduler: do not start a sweep with fewer slots than this while others are in flight
  const float* x0;
  const float* xref;
  const float* u_init;
  unsigned long long* header;  // [0] next problem index, [1] error word
  const int32_t* perm;         // hinted order: the k-th problem to start is perm[k] (NULL: index order)
  float* slab;                 // [grid][S][T-1][MPC_REC]
  float* sol;
  float* u0;
  float* cost;
  int32_t* status;
  int32_t* iters;
};

// Scheduling state of one CTA (shared memory, after the slots).  Everything except `seq` is read and
// written under `lock` only.
struct alignas(16) MpcSched {  // 16-byte multiple: the cp.async rings follow it
  int q[3][MPC_TASK_QS];  // slots waiting for a REFILL / BW / FW sweep (ring buffers)
  int head[3], tail[3];   // monotonic positions into q[k]
  int inflight;           // warps that are executing a task
  int lock;
  int seq;                // bumped whenever work is posted: idle warps watch it instead of the lock
};
static_assert(sizeof(MpcSched) % 16 == 0, "record rings must start 16-byte aligned");

__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

// RING_BULK = false (default): records staged by cp.async commit groups; true (CRB_MPC_RING=bulk): by one 80-byte
// cp.async.bulk (TMA) per lane and stage on mbarriers.  The TMA engine is built for tiles, and 32 separate 80-byte
// descriptors per warp and stage cost more than 160 LDGSTS lanes; kept as a compile-time variant (a run-time
// branch costs registers and code size).
template <bool RING_BULK>
__global__ void __launch_bounds__(MPC_TASK_MAX_WARPS * 32, 1)
crb_mpc_tasks_kernel(const __grid_constant__ MpcTaskArgs A, const __grid_constant__ MpcP p) {
  extern __shared__ __align__(16) float smem[];
  const int S = A.S, T = A.T, N = T - 1, SW = A.slot_words;
  const int lane = threadIdx.x & 31;
  MpcSched* const sc = reinterpret_cast<MpcSched*>(smem + (size_t)S * SW);
  volatile int* const vhead = sc->head;
  volatile int* const vtail = sc->tail;
  for (int s = threadIdx.x; s < S; s += blockDim.x) {
    sc->q[0][s] = s;  // every slot starts empty and waits for a refill
    reinterpret_cast<int*>(smem + (size_t)s * SW + mpc_slot_tr_words(T))[MPC_SW_PROB] = -1;
  }
  if (threadIdx.x == 0) {
    sc->head[0] = sc->head[1] = sc->head[2] = 0;
    sc->tail[0] = S; sc->tail[1] = sc->tail[2] = 0;
    sc->inflight = 0; sc->lock = 0; sc->seq = 0;
  }
  __syncthreads();
  float* const slab = A.slab + (size_t)blockIdx.x * S * N * MPC_REC;
  const int tr_words = mpc_slot_tr_words(T);
  const unsigned FULL = 0xffffffffu;

  const unsigned long long pol = mpc_policy_evict_last();
  // this warp's record ring (forward sweeps), after the scheduling state
  const unsigned ring = (unsigned)__cvta_generic_to_shared(reinterpret_cast<char*>(sc + 1) +
                                                           (size_t)(threadIdx.x >> 5) * MPC_RING_BYTES) +
                        (unsigned)lane * 16u;
  // TMA form of the ring: [stage][lane][80 B] in the same bytes, one mbarrier per stage after all the rings
  const int nwarps_k = blockDim.x >> 5;
  const unsigned ring_bulk = RING_BULK ? (unsigned)__cvta_generic_to_shared(reinterpret_cast<char*>(sc + 1) +
                                                                              (size_t)(threadIdx.x >> 5) * MPC_RING_BYTES) +
                                               (unsigned)lane * 80u
                                         : 0u;
  const unsigned mbar = (unsigned)__cvta_generic_to_shared(reinterpret_cast<char*>(sc + 1) +
                                                           (size_t)nwarps_k * MPC_RING_BYTES) +
                        (unsigned)(threadIdx.x >> 5) * (MPC_RING_D * 8u);
  unsigned rounds[MPC_RING_D] = {0u, 0u, 0u};
  if (RING_BULK) {
    if (lane == 0) {
#pragma unroll
      for (int s = 0; s < MPC_RING_D; ++s)
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 32;" :: "r"(mbar + 8u * (unsigned)s) : "memory");
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
  }
  bool have_post = false, active = false;
  int patience = 2;
  int slot = 0, next = MPC_PH_DEAD;
  for (;;) {
    // ---- one critical section per task: publish the finished sweep's slots, take the next batch -------
    // the whole warp polls together (lane 0 does the atomic, everybody sleeps): no divergent spin loop
    int got = 0;
    for (int tries = 0;; ++tries) {
      int old = 1;
      if (lane == 0) old = atomicCAS(&sc->lock, 0, 1);
      old = __shfl_sync(FULL, old, 0);
      if (old == 0) { got = 1; break; }
      if (tries > (1 << 22)) { if (lane == 0) atomicExch(&A.header[1], 1ull); break; }
      __nanosleep(tries < 4 ? 40 : 200);
    }
    if (!got) break;  // never hang the GPU on a scheduling bug: raise the error word and leave
    __threadfence_block();
    if (have_post) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const bool mine = active && next == k + 1;
        const unsigned m = __ballot_sync(FULL, mine);
        if (m) {
          const int base = vtail[k];
          if (mine) sc->q[k][(base + __popc(m & lanemask_lt())) & (MPC_TASK_QS - 1)] = slot;
          __syncwarp();
          if (lane == 0) vtail[k] = base + __popc(m);
        }
      }
      if (lane == 0) {
        *(volatile int*)&sc->inflight = *(volatile int*)&sc->inflight - 1;
        *(volatile int*)&sc->seq = *(volatile int*)&sc->seq + 1;
      }
      __syncwarp();
    }
    const int h0 = vhead[0], h1 = vhead[1], h2 = vhead[2];
    const int c_refill = vtail[0] - h0, c_bw = vtail[1] - h1, c_fw = vtail[2] - h2;
    int kind = MPC_PH_FW, best = c_fw, hk = h2;
    if (c_bw > best) { kind = MPC_PH_BW; best = c_bw; hk = h1; }
    if (c_refill > best) { kind = MPC_PH_REFILL; best = c_refill; hk = h0; }
    // A thin batch costs a whole sweep of the warp's time.  When the fullest queue has fewer than `A.fill_min` slots,
    // other warps are in flight (their posts will refill the queues) and the patience is not used up, take
    // nothing now and look again after the next post.
    int infl = *(volatile int*)&sc->inflight;
    const bool hold = best > 0 && best < A.fill_min && infl >= 2 && patience > 0;
    const int taken = hold ? 0 : (best < 32 ? best : 32);
    active = lane < taken;
    slot = active ? *(volatile int*)&sc->q[kind - 1][(hk + lane) & (MPC_TASK_QS - 1)] : 0;
    const int seen = *(volatile int*)&sc->seq;
    __syncwarp();
    if (lane == 0 && taken > 0) {
      vhead[kind - 1] = hk + taken;
      *(volatile int*)&sc->inflight = infl + 1;
    }
    __threadfence_block();
    __syncwarp();
    if (lane == 0) atomicExch(&sc->lock, 0);
    have_post = false;
    if (taken == 0) {
      if (hold) --patience;
      if (infl == 0 && best == 0) break;  // nothing waits and nobody is working: this CTA is done
      int spins = 0;         // wait for the next post without touching the lock
      while (*(volatile int*)&sc->seq == seen) {
        __nanosleep(400);
        if (++spins > (1 << 23)) { if (lane == 0) atomicExch(&A.header[1], 2ull); break; }
      }
      if (spins > (1 << 23)) break;
      continue;
    }
    patience = 2;
    MpcSlot sl;
    sl.tr = smem + (size_t)slot * SW;
    sl.sw = sl.tr + tr_words;
    sl.rec = slab + (size_t)slot * N * MPC_REC;
    sl.pol = pol;
    sl.ring = ring;
    sl.ring_bulk = ring_bulk;
    sl.mbar = mbar;

    next = MPC_PH_DEAD;
    if (kind == MPC_PH_BW) {
      if (active) next = mpc_task_bw(sl, T, p);
    } else if (kind == MPC_PH_FW) {
      if (RING_BULK) {   // every lane walks the ring protocol (mbarrier arrivals); idle lanes touch nothing else
#pragma unroll
        for (int s = 0; s < MPC_RING_D; ++s) sl.rounds[s] = rounds[s];
        next = mpc_task_fw<true>(sl, T, p, active);
#pragma unroll
        for (int s = 0; s < MPC_RING_D; ++s) rounds[s] = sl.rounds[s];
      } else if (active) {
        next = mpc_task_fw<false>(sl, T, p);
      }
    } else {
      // retire what the slot holds, then pull the next problems: consecutive indices for consecutive
      // lanes, so the loads of a refill are coalesced rows of x0 / xref
      if (active && mpc_sw_int(sl, MPC_SW_PROB) >= 0)
        mpc_task_retire(sl, T, p, A.ld_out, A.sol, A.u0, A.cost, A.status, A.iters);
      unsigned long long base = 0;
      if (lane == 0) base = atomicAdd(&A.header[0], (unsigned long long)taken);
      base = __shfl_sync(FULL, base, 0);
      int64_t i = (int64_t)base + lane;
      // hinted order: the k-th problem to start is perm[k] (problems sorted by decreasing hint, crb_mpc_hint_perm_kernel)
      if (A.perm != nullptr && active && i < A.count) i = (int64_t)__ldg(A.perm + i);
      if (active) {
        if (i < A.count) {
          next = mpc_task_init(sl, T, p, i, A.ld_in, A.x0, A.xref, A.u_init);
        } else {
          mpc_sw_int(sl, MPC_SW_PROB) = -1;  // the batch is exhausted: the slot stays empty
          next = MPC_PH_DEAD;
        }
      }
    }
    __threadfence_block();  // the sweep's results are visible before the slots are queued again
    have_post = true;
  }
}

// ---- hinted order: the long problems first, the rest in (almost) index order -------------------------------------
// Two small launches in front of the solver: the histogram of the clamped hints, then the scatter.  The ~15 % of the
// problems with the largest hints (hint >= thr, mpc_hint_threshold) are sorted by decreasing hint and start first;
// all the others form ONE bin behind them.  A position is (problems in earlier bins) + (arrival rank in the bin);
// the rank comes from one warp-aggregated atomicAdd per bin and warp, so the lanes of a warp stay together and the
// big bin keeps runs of consecutive indices: the solver's refills of those problems still read coalesced rows of
// x0 / xref.  (A full sort by hint scattered every refill over 32 rows: 4-8 % slower at 2^20 problems, where there
// is no tail to win back.)  The order inside a bin depends on the run; the results do not.
__global__ void __launch_bounds__(256) crb_mpc_hint_hist_kernel(int64_t count, const int32_t* __restrict__ hint,
                                                                unsigned* __restrict__ hist) {
  __shared__ unsigned sh[MPC_HINT_BINS];
  if (threadIdx.x < MPC_HINT_BINS) sh[threadIdx.x] = 0u;
  __syncthreads();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
    atomicAdd(&sh[mpc_hint_clamp(hint[i])], 1u);
  __syncthreads();
  if (threadIdx.x < MPC_HINT_BINS && sh[threadIdx.x]) atomicAdd(&hist[threadIdx.x], sh[threadIdx.x]);
}

__global__ void __launch_bounds__(256) crb_mpc_hint_perm_kernel(int64_t count, const int32_t* __restrict__ hint,
                                                                const unsigned* __restrict__ hist,
                                                                unsigned* __restrict__ cursor,
                                                                int32_t* __restrict__ perm) {
  __shared__ unsigned first[MPC_HINT_BINS];   // first position of the bin: number of problems in earlier bins
  __shared__ int s_thr;
  if (threadIdx.x == 0) s_thr = mpc_hint_threshold(hist, count);
  __syncthreads();
  const int thr = s_thr;
  if (threadIdx.x < MPC_HINT_BINS) {
    // bins thr .. 63 in decreasing order, then bin 0 = everything below thr
    unsigned f = 0u;
    const int me = (int)threadIdx.x;
    if (me >= thr) {
      for (int b = MPC_HINT_BINS - 1; b > me; --b) f += hist[b];
    } else {
      for (int b = MPC_HINT_BINS - 1; b >= thr; --b) f += hist[b];
    }
    first[threadIdx.x] = f;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t rounds = (count + stride - 1) / stride;   // the same trip count for every thread: full-warp intrinsics
  for (int64_t r = 0; r < rounds; ++r) {
    const int64_t i = r * stride + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int h = i < count ? mpc_hint_clamp(hint[i]) : -1;
    if (h >= 0 && h < thr) h = 0;                               // one bin for everything below the threshold
    const unsigned grp = __match_any_sync(0xffffffffu, h);      // the lanes of this warp in the same bin
    const int leader = __ffs(grp) - 1;
    unsigned off = 0u;
    if (lane == leader && h >= 0) off = atomicAdd(&cursor[h], (unsigned)__popc(grp));
    off = __shfl_sync(0xffffffffu, off, leader);
    if (h >= 0) perm[first[h] + off + (unsigned)__popc(grp & lanemask_lt())] = (int32_t)i;
  }
}

// Launch geometry for `count` problems of horizon T: warps per CTA, slots per CTA, CTAs, shared memory.
struct MpcTaskGeom {
  int nwarps, S, grid;
  size_t smem;
};
static bool mpc_tasks_geometry(int sm_count, int T, int64_t count, MpcTaskGeom* g) {
  const size_t smem_cap = 227 * 1024;
  static int env_warps = -1, env_slots = -1;  // A/B knobs (process-wide, read once)
  if (env_warps < 0) {
    const char* e = getenv("CRB_MPC_WARPS");
    env_warps = e ? atoi(e) : 0;
    const char* f = getenv("CRB_MPC_SLOTS");
    env_slots = f ? atoi(f) : 0;
  }
  int nwarps = env_warps > 0 ? env_warps : MPC_TASK_MAX_WARPS;
  if (nwarps > MPC_TASK_MAX_WARPS) nwarps = MPC_TASK_MAX_WARPS;
  // shared memory: slots, scheduling state, one record ring per warp.  Fewer warps leave more slots waiting
  // (fuller warps of one kind); the default takes the most warps that keep >= 24 slots waiting.
  int S = 0;
  size_t fixed = 0;
  for (;; --nwarps) {
    fixed = sizeof(MpcSched) + (size_t)nwarps * MPC_RING_BYTES + (size_t)nwarps * MPC_RING_D * 8;
    size_t s = (smem_cap - fixed) / ((size_t)mpc_slot_words(T) * sizeof(float));
    if (s > MPC_TASK_SLOTS) s = MPC_TASK_SLOTS;
    S = (int)s;
    if (env_slots > 0 && env_slots < S) S = env_slots;
    if (nwarps == 1) break;
    if (env_warps > 0 ? nwarps * 32 <= S : nwarps * 32 + 24 <= S) break;
  }
  if (S < 32) return false;
  // one CTA per SM; fewer when the batch has less than one task per warp
  int64_t grid = (count + (int64_t)nwarps * 32 - 1) / ((int64_t)nwarps * 32);
  if (grid > sm_count) grid = sm_count;
  if (grid < 1) grid = 1;
  g->nwarps = nwarps;
  g->S = S;
  g->grid = (int)grid;
  g->smem = (size_t)S * mpc_slot_words(T) * sizeof(float) + fixed;
  return true;
}

// header (768 B: counters, hint histogram, bin cursors) + slab of stage records + the start order (one int per
// problem) + 256 B of alignment slack
#define MPC_TASK_HEADER_BYTES 768
static size_t mpc_tasks_slab_bytes(const MpcTaskGeom& g, int T) {
  return ((size_t)g.grid * g.S * (size_t)(T - 1) * MPC_REC * sizeof(float) + 255) & ~(size_t)255;
}
size_t crb_mpc_tasks_scratch_bytes(int sm_count, int T, int64_t count) {
  MpcTaskGeom g;
  if (!mpc_tasks_geometry(sm_count, T, count, &g)) return MPC_TASK_HEADER_BYTES + 256;
  return MPC_TASK_HEADER_BYTES + 256 + mpc_tasks_slab_bytes(g, T) + (size_t)count * sizeof(int32_t);
}

int crb_mpc_tasks_launch(crb_ctx* ctx, cudaStream_t st, int64_t count, int64_t ld, int T,
                         const float* x0, const float* xref, const float* u_init, void* scratch,
                         int64_t ld_out, float* sol, float* u0, float* cost, int32_t* status,
                         int32_t* iters, const MpcP& p, const int32_t* hint) {
  CRB_REQUIRE(count < ((int64_t)1 << 31), "more than 2^31 problems in one launch");
  MpcTaskGeom g;
  if (!mpc_tasks_geometry(ctx->sm_count, T, count, &g)) {
    crb_set_error("crb_mpc_tasks_launch: T = %d does not fit the resident-slot kernel", T);
    return CRB_ERR_UNSUPPORTED;
  }
  if (!ctx->mpc_tasks_attr_set) {
    CRB_CUDA(cudaFuncSetAttribute(crb_mpc_tasks_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  227 * 1024));
    CRB_CUDA(cudaFuncSetAttribute(crb_mpc_tasks_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  227 * 1024));
    ctx->mpc_tasks_attr_set = 1;
  }
  char* base = (char*)(((uintptr_t)scratch + 255) & ~(uintptr_t)255);
  MpcTaskArgs a;
  a.count = count; a.ld_in = ld; a.ld_out = ld_out;
  a.T = T; a.S = g.S; a.slot_words = mpc_slot_words(T);
  {
    // CRB_MPC_FILL (A/B, read once; default 0 = off): hold back batches thinner than this many slots.  Off by
    // default: the idle wait is worth more than the fuller warp.
    static int fill = -1;
    if (fill < 0) {
      const char* e = getenv("CRB_MPC_FILL");
      fill = e ? atoi(e) : 0;
      if (fill < 0 || fill > 32) fill = 0;
    }
    a.fill_min = fill;
  }
  static int bulk = -1;   // CRB_MPC_RING=bulk selects the TMA form of the record ring (A/B, read once)
  if (bulk < 0) {
    const char* e = getenv("CRB_MPC_RING");
    bulk = (e && e[0] == 'b') ? 1 : 0;
  }
  a.x0 = x0; a.xref = xref; a.u_init = u_init;
  a.header = (unsigned long long*)base;
  a.slab = (float*)(base + MPC_TASK_HEADER_BYTES);
  a.sol = sol; a.u0 = u0; a.cost = cost; a.status = status; a.iters = iters;
  a.perm = nullptr;
  CRB_CUDA(cudaMemsetAsync(base, 0, MPC_TASK_HEADER_BYTES, st));
  // With many SM-generations of problems there is no tail to win back and the 15 % scattered refills cost more
  // than they save: the hints are used up to 6 generations (6 x CTAs x slots problems).
  if (hint != nullptr && count <= 6 * (int64_t)g.grid * g.S) {
    int32_t* perm = (int32_t*)(base + MPC_TASK_HEADER_BYTES + mpc_tasks_slab_bytes(g, T));
    unsigned* hist = (unsigned*)(base + 256);
    unsigned* cursor = (unsigned*)(base + 512);
    int hg = (int)((count + 2047) / 2048);
    if (hg > 4 * ctx->sm_count) hg = 4 * ctx->sm_count;
    if (hg < 1) hg = 1;
    crb_mpc_hint_hist_kernel<<<hg, 256, 0, st>>>(count, hint, hist);
    crb_mpc_hint_perm_kernel<<<hg, 256, 0, st>>>(count, hint, hist, cursor, perm);
    ctx->launches += 2;
    a.perm = perm;
  }
  if (bulk)
    crb_mpc_tasks_kernel<true><<<(unsigned)g.grid, g.nwarps * 32, g.smem, st>>>(a, p);
  else
    crb_mpc_tasks_kernel<false><<<(unsigned)g.grid, g.nwarps * 32, g.smem, st>>>(a, p);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

// crb_ctx.cu — context, memory helpers, timers and default parameter blocks of libcrb.
#include <stdarg.h>

#include "crb_common.cuh"

static thread_local char g_err[512] = "";

void crb_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" {

int crb_abi_version(void) { return CRB_ABI_VERSION; }
const char* crb_last_error_string(void) { return g_err; }

int crb_init(crb_ctx** out, int device_id) {
  CRB_REQUIRE(out != nullptr, "out is NULL");
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    crb_set_error("crb_init: no usable CUDA device (%s); libcrb has no CPU fallback",
                  e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
    return CRB_ERR_NO_DEVICE;
  }
  int prev = -1;
  CRB_CUDA(cudaGetDevice(&prev));
  if (device_id < 0) device_id = prev;
  CRB_REQUIRE(device_id < count, "device_id out of range");
  cudaDeviceProp prop;
  CRB_CUDA(cudaGetDeviceProperties(&prop, device_id));
  if (prop.major != 9 || prop.minor != 0) {
    crb_set_error("crb_init: device %d is sm_%d%d; libcrb is built for sm_90a only", device_id,
                  prop.major, prop.minor);
    return CRB_ERR_UNSUPPORTED;
  }
  crb_ctx* c = new crb_ctx();
  memset(c, 0, sizeof(*c));
  c->device = device_id;
  c->sm_count = prop.multiProcessorCount;
  c->comm_world = 1;
  // everything below runs with device_id current; the caller's current device is restored on every path and a
  // partially built context is torn down instead of leaked
  cudaError_t err = cudaSetDevice(device_id);
  if (err == cudaSuccess) err = cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking);
  c->stream = c->own_stream;
  if (err == cudaSuccess) err = cudaEventCreate(&c->ev_start);
  if (err == cudaSuccess) err = cudaEventCreate(&c->ev_stop);
  for (int i = 0; i < CRB_N_PIPE && err == cudaSuccess; ++i)
    err = cudaStreamCreateWithFlags(&c->pipe_stream[i], cudaStreamNonBlocking);
  if (err == cudaSuccess) err = cudaMallocHost(&c->host_scratch, 4096);
  if (err == cudaSuccess) err = cudaMalloc(&c->tickets, 64 * sizeof(unsigned));
  if (err == cudaSuccess) err = cudaMemset(c->tickets, 0, 64 * sizeof(unsigned));
  if (err != cudaSuccess) {
    crb_set_error("crb_init: %s", cudaGetErrorString(err));
    crb_destroy(c);
    if (prev >= 0) cudaSetDevice(prev);
    return err == cudaErrorMemoryAllocation ? CRB_ERR_ALLOC : CRB_ERR_CUDA;
  }
  if (prev >= 0 && prev != device_id) cudaSetDevice(prev);
  *out = c;
  return CRB_OK;
}

int crb_destroy(crb_ctx* ctx) {
  if (!ctx) return CRB_OK;
  int prev = -1;
  if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
  cudaSetDevice(ctx->device);
  if (ctx->comm) crb_comm_destroy(ctx);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  if (ctx->own_stream) cudaStreamSynchronize(ctx->own_stream);
  for (int i = 0; i < CRB_N_PIPE; ++i) {
    if (ctx->pipe_stream[i]) {
      cudaStreamSynchronize(ctx->pipe_stream[i]);
      cudaStreamDestroy(ctx->pipe_stream[i]);
    }
    if (ctx->pipe_buf[i]) cudaFree(ctx->pipe_buf[i]);
  }
  if (ctx->scratch) cudaFree(ctx->scratch);
  if (ctx->mpc_ws) cudaFree(ctx->mpc_ws);
  if (ctx->host_scratch) cudaFreeHost(ctx->host_scratch);
  if (ctx->tickets) cudaFree(ctx->tickets);
  if (ctx->ev_start) cudaEventDestroy(ctx->ev_start);
  if (ctx->ev_stop) cudaEventDestroy(ctx->ev_stop);
  if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
  cudaGetLastError();
  if (prev >= 0 && prev != ctx->device) cudaSetDevice(prev);
  delete ctx;
  return CRB_OK;
}

int crb_set_stream(crb_ctx* ctx, void* cuda_stream) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  ctx->stream = (cudaStream_t)cuda_stream;
  return CRB_OK;
}
int crb_use_own_stream(crb_ctx* ctx) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  ctx->stream = ctx->own_stream;
  return CRB_OK;
}
void* crb_get_stream(crb_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

int crb_sync(crb_ctx* ctx) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_CUDA(cudaStreamSynchronize(ctx->stream));
  return CRB_OK;
}
int64_t crb_launch_count(crb_ctx* ctx) { return ctx ? ctx->launches : -1; }

int crb_host_alloc(void** out, size_t bytes) {
  CRB_REQUIRE(out != nullptr, "out is NULL");
  CRB_CUDA(cudaMallocHost(out, bytes ? bytes : 1));
  return CRB_OK;
}
int crb_host_free(void* p) {
  if (p) CRB_CUDA(cudaFreeHost(p));
  return CRB_OK;
}
int crb_device_alloc(crb_ctx* ctx, void** out, size_t bytes) {
  CRB_REQUIRE(ctx != nullptr && out != nullptr, "ctx/out is NULL");
  CRB_DEVICE_GUARD(ctx);
  CRB_CUDA(cudaMalloc(out, bytes ? bytes : 1));
  return CRB_OK;
}
int crb_device_free(crb_ctx* ctx, void* p) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_DEVICE_GUARD(ctx);
  if (p) CRB_CUDA(cudaFree(p));
  return CRB_OK;
}
int crb_memcpy_h2d(crb_ctx* ctx, void* dst_dev, const void* src_host, size_t bytes) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_CUDA(cudaMemcpyAsync(dst_dev, src_host, bytes, cudaMemcpyHostToDevice, ctx->stream));
  return CRB_OK;
}
int crb_memcpy_d2h(crb_ctx* ctx, void* dst_host, const void* src_dev, size_t bytes) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_CUDA(cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CRB_CUDA(cudaStreamSynchronize(ctx->stream));
  return CRB_OK;
}
int crb_timer_start(crb_ctx* ctx) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_CUDA(cudaEventRecord(ctx->ev_start, ctx->stream));
  return CRB_OK;
}
int crb_timer_stop_ms(crb_ctx* ctx, float* ms_out) {
  CRB_REQUIRE(ctx != nullptr && ms_out != nullptr, "ctx/ms_out is NULL");
  CRB_CUDA(cudaEventRecord(ctx->ev_stop, ctx->stream));
  CRB_CUDA(cudaEventSynchronize(ctx->ev_stop));
  CRB_CUDA(cudaEventElapsedTime(ms_out, ctx->ev_start, ctx->ev_stop));
  return CRB_OK;
}

// ---- default parameter blocks (the constants that live in the reference's main()s) -------------
void crb_ekf_default_params(crb_ekf_params* p) {
  // src/extended_kalman_filter.cpp:17 DT; :142-146 Q (doubles narrowed into a Matrix4f); :149-151 R
  memset(p, 0, sizeof(*p));
  p->dt = 0.1;
  p->Q[0] = (float)(0.1 * 0.1);
  p->Q[5] = (float)(0.1 * 0.1);
  p->Q[10] = (float)((1.0 / 180 * 3.14159265358979323846) * (1.0 / 180 * 3.14159265358979323846));
  p->Q[15] = (float)(0.1 * 0.1);
  p->R[0] = 1.0f;
  p->R[3] = 1.0f;
}

void crb_pf_default_params(crb_pf_params* p) {
  // src/particle_filter.cpp:18 DT; :19 PI; :217 Q = 0.1*0.1; :228-230 Rsim; :183 u
  memset(p, 0, sizeof(*p));
  p->dt = 0.1;
  p->pi = 3.141592653;
  p->Q = (float)(0.1 * 0.1);
  p->rsim_diag[0] = (float)1.0;
  p->rsim_diag[1] =
      (float)((30.0 / 180 * 3.14159265358979323846) * (30.0 / 180 * 3.14159265358979323846));
  p->u[0] = 1.0f;
  p->u[1] = 0.1f;
}

void crb_mpc_default_params(crb_mpc_params* p) {
  // src/model_predictive_control.cpp:26-39 macros, :202-210 / :247-250 weights
  memset(p, 0, sizeof(*p));
  p->dt = (float)0.2;
  p->wb = (float)2.5;
  p->max_steer = (float)(45.0 / 180 * 3.14159265358979323846);
  p->max_accel = (float)1.0;
  p->max_speed = (float)(55.0 / 3.6);
  p->min_speed = (float)(-20.0 / 3.6);
  p->w_a = 0.01f;
  p->w_delta = 0.01f;
  p->w_da = 0.01f;
  p->w_ddelta = 1.0f;
  p->w_x = 1.0f;
  p->w_y = 1.0f;
  p->w_yaw = 0.5f;
  p->w_v = 0.5f;
  p->max_iter = 50;   // IPOPT's max_iter option (:326); MAX_ITER 3 / DU_TH 0.1 (:30-31) are unused macros
  p->du_th = 1.0e-4f;
  p->max_ls = 4;
  p->j_tol = 1.0e-6f;
}

}  // extern "C"

int crb_ctx_pipe_reserve(crb_ctx* ctx, int slot, size_t bytes) {
  CRB_DEVICE_GUARD(ctx);
  if (ctx->pipe_cap[slot] >= bytes) return CRB_OK;
  if (ctx->pipe_buf[slot]) {
    CRB_CUDA(cudaStreamSynchronize(ctx->pipe_stream[slot]));
    CRB_CUDA(cudaFree(ctx->pipe_buf[slot]));
    ctx->pipe_buf[slot] = nullptr;
    ctx->pipe_cap[slot] = 0;
  }
  CRB_CUDA(cudaMalloc(&ctx->pipe_buf[slot], bytes));
  ctx->pipe_cap[slot] = bytes;
  return CRB_OK;
}

int crb_ctx_scratch_reserve(crb_ctx* ctx, size_t bytes) {
  CRB_DEVICE_GUARD(ctx);
  if (ctx->scratch_cap >= bytes) return CRB_OK;
  if (ctx->scratch) {
    CRB_CUDA(cudaStreamSynchronize(ctx->stream));
    CRB_CUDA(cudaFree(ctx->scratch));
    ctx->scratch = nullptr;
    ctx->scratch_cap = 0;
  }
  CRB_CUDA(cudaMalloc(&ctx->scratch, bytes));
  ctx->scratch_cap = bytes;
  return CRB_OK;
}

int crb_ctx_mpc_ws_reserve(crb_ctx* ctx, size_t bytes) {
  CRB_DEVICE_GUARD(ctx);
  if (ctx->mpc_ws_cap >= bytes) return CRB_OK;
  if (ctx->mpc_ws) {
    CRB_CUDA(cudaStreamSynchronize(ctx->stream));
    CRB_CUDA(cudaFree(ctx->mpc_ws));
    ctx->mpc_ws = nullptr;
    ctx->mpc_ws_cap = 0;
  }
  CRB_CUDA(cudaMalloc(&ctx->mpc_ws, bytes));
  ctx->mpc_ws_cap = bytes;
  return CRB_OK;
}

// cg_api.cu -- context management for the C ABI (include/catgrasp_b200.h).
#include "cg_common.cuh"
#include <stdlib.h>

extern "C" const char *cg_version(void) { return "catgrasp_b200 0.1 (sm_90a)"; }

extern "C" int cg_ctx_create(int device, cg_ctx **out) {
  if (!out) return CG_EINVAL;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n) return CG_ECUDA;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return CG_ECUDA;
  if (prop.major != 9 || prop.minor != 0) {
    // no multi-backend dispatch: this library only carries sm_90a code
    fprintf(stderr, "catgrasp_b200: device %d is sm_%d%d, this library is sm_90a-only\n", device, prop.major,
            prop.minor);
    return CG_EUNSUPPORTED;
  }
  if (cudaSetDevice(device) != cudaSuccess) return CG_ECUDA;
  cg_ctx *ctx = new cg_ctx();
  ctx->device = device;
  ctx->num_sms = prop.multiProcessorCount;
  const char *tr = getenv("CG_TRACE");
  ctx->trace = tr && tr[0] == '1';
  if (cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete ctx;
    return CG_ECUDA;
  }
  ctx->stream = ctx->own_stream;
  if (cudaMalloc(&ctx->ovf_flag, 4) != cudaSuccess || cudaMemset(ctx->ovf_flag, 0, 4) != cudaSuccess) {
    cudaStreamDestroy(ctx->own_stream);
    delete ctx;
    return CG_ECUDA;
  }
  *out = ctx;
  return CG_OK;
}

// engines 2 and 3 clamp 128->1024 inputs to the fp16 range; *out = 1 if that happened since the last call (clears the flag)
extern "C" int cg_ctx_fp16_overflow(cg_ctx *ctx, int *out) {
  if (!ctx || !out) return CG_EINVAL;
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  uint32_t h = 0;
  CG_CUDA(ctx, cudaMemcpyAsync(&h, ctx->ovf_flag, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (h) CG_CUDA(ctx, cudaMemsetAsync(ctx->ovf_flag, 0, 4, ctx->stream));
  *out = (int)h;
  return CG_OK;
}

extern "C" void cg_ctx_destroy(cg_ctx *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->switch_event) cudaEventDestroy(ctx->switch_event);
  if (ctx->ovf_flag) cudaFree(ctx->ovf_flag);
  if (ctx->ws) cudaFree(ctx->ws);
  if (ctx->io) cudaFree(ctx->io);
  cudaStreamDestroy(ctx->own_stream);
  delete ctx;
}

// The context's workspaces (ws / io arenas) are reused by consecutive calls.  When the caller moves the context to a
// different stream, work already enqueued on the previous stream may still be reading them: order the new stream behind
// the old one with an event (no host synchronisation).
static int switch_stream(cg_ctx *ctx, cudaStream_t next) {
  if (next == ctx->stream) return CG_OK;
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  if (!ctx->switch_event) CG_CUDA(ctx, cudaEventCreateWithFlags(&ctx->switch_event, cudaEventDisableTiming));
  // the previous stream may be a caller-owned stream that has been destroyed since: its work is complete then, and
  // recording on a dead handle is an error we can ignore
  if (cudaEventRecord(ctx->switch_event, ctx->stream) == cudaSuccess)
    CG_CUDA(ctx, cudaStreamWaitEvent(next, ctx->switch_event, 0));
  else
    cudaGetLastError();
  ctx->stream = next;
  return CG_OK;
}

extern "C" int cg_ctx_set_stream(cg_ctx *ctx, void *cuda_stream) {
  if (!ctx) return CG_EINVAL;
  // NULL is a real stream: the CUDA legacy default stream (what torch uses unless told otherwise)
  return switch_stream(ctx, static_cast<cudaStream_t>(cuda_stream));
}

extern "C" int cg_ctx_use_own_stream(cg_ctx *ctx) {
  if (!ctx) return CG_EINVAL;
  return switch_stream(ctx, ctx->own_stream);
}

extern "C" int cg_ctx_synchronize(cg_ctx *ctx) {
  if (!ctx) return CG_EINVAL;
  CG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return CG_OK;
}

extern "C" const char *cg_last_error(cg_ctx *ctx) { return ctx ? ctx->err.c_str() : "null context"; }
extern "C" int64_t cg_ctx_launch_count(cg_ctx *ctx) { return ctx ? ctx->launches : 0; }
extern "C" void cg_ctx_reset_launch_count(cg_ctx *ctx) { if (ctx) ctx->launches = 0; }

extern "C" int cg_ctx_set_engine(cg_ctx *ctx, int engine) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, engine >= 0 && engine <= 3,
             "engine must be 0 (fp32 SIMT), 1 (wgmma 3-pass), 2 (wgmma 2-pass) or 3 (wgmma 1-pass)");
  ctx->engine = engine;
  return CG_OK;
}
extern "C" int cg_ctx_get_engine(cg_ctx *ctx) { return ctx ? ctx->engine : CG_EINVAL; }

static int grow(cg_ctx *ctx, void **p, size_t *cur, size_t bytes) {
  if (bytes <= *cur) return CG_OK;
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  // the arena may still be in use by enqueued work
  CG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (*p) {
    cudaFree(*p);
    *p = nullptr;
    *cur = 0;
  }
  size_t want = bytes + bytes / 4;
  cudaError_t e = cudaMalloc(p, want);
  if (e != cudaSuccess) {
    cudaGetLastError();
    want = bytes;
    e = cudaMalloc(p, want);
  }
  if (e != cudaSuccess) {
    ctx->err = std::string("workspace allocation failed: ") + cudaGetErrorString(e);
    cudaGetLastError();
    return CG_ENOMEM;
  }
  *cur = want;
  return CG_OK;
}

int cg_ws_reserve(cg_ctx *ctx, size_t bytes) { return grow(ctx, &ctx->ws, &ctx->ws_bytes, bytes); }
int cg_io_reserve(cg_ctx *ctx, size_t bytes) { return grow(ctx, &ctx->io, &ctx->io_bytes, bytes); }

extern "C" int cg_ctx_fill_workspaces(cg_ctx *ctx, int byte) {
  if (!ctx) return CG_EINVAL;
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  if (ctx->ws) CG_CUDA(ctx, cudaMemsetAsync(ctx->ws, byte, ctx->ws_bytes, ctx->stream));
  if (ctx->io) CG_CUDA(ctx, cudaMemsetAsync(ctx->io, byte, ctx->io_bytes, ctx->stream));
  return CG_OK;
}

// CG_TRACE diagnostics: durations between consecutive post-launch events on the context's stream, grouped by call site
void cg_trace_mark(cg_ctx *ctx, const char *where) {
  cudaEvent_t e;
  if (cudaEventCreate(&e) != cudaSuccess) return;
  cudaEventRecord(e, ctx->stream);
  ctx->trace_events.emplace_back(where, e);
  if (ctx->trace_events.size() < 3000) return;
  cudaEventSynchronize(e);
  std::vector<std::pair<std::string, std::pair<int, double>>> agg;
  for (size_t i = 1; i < ctx->trace_events.size(); i++) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ctx->trace_events[i - 1].second, ctx->trace_events[i].second);
    const char *w = strrchr(ctx->trace_events[i].first, '/');
    std::string key = w ? w + 1 : ctx->trace_events[i].first;
    bool found = false;
    for (auto &a : agg)
      if (a.first == key) { a.second.first++; a.second.second += ms; found = true; break; }
    if (!found) agg.push_back({key, {1, (double)ms}});
  }
  fprintf(stderr, "[cg trace] %zu launches (time since the previous launch's end, incl. gaps)\n", ctx->trace_events.size());
  for (auto &a : agg)
    fprintf(stderr, "[cg trace] %-28s n=%5d total=%9.3f ms avg=%8.2f us\n", a.first.c_str(), a.second.first, a.second.second,
            1e3 * a.second.second / a.second.first);
  for (auto &t : ctx->trace_events) cudaEventDestroy(t.second);
  ctx->trace_events.clear();
}

extern "C" int cg_ctx_profile(cg_ctx *ctx, int enable) {
  if (!ctx) return CG_EINVAL;
  ctx->prof = enable != 0;
  return CG_OK;
}

extern "C" int cg_ctx_profile_read(cg_ctx *ctx, double *ms_total, int64_t *launches) {
  if (!ctx || !ms_total || !launches) return CG_EINVAL;
  double tot = 0.0;
  for (auto &pr : ctx->prof_events) {
    CG_CUDA(ctx, cudaEventSynchronize(pr.second));
    float ms = 0.f;
    CG_CUDA(ctx, cudaEventElapsedTime(&ms, pr.first, pr.second));
    tot += ms;
    cudaEventDestroy(pr.first);
    cudaEventDestroy(pr.second);
  }
  *ms_total = tot;
  *launches = (int64_t)ctx->prof_events.size();
  ctx->prof_events.clear();
  return CG_OK;
}

// cg_common.cuh -- shared internals of libcatgrasp_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <string>
#include <utility>
#include <vector>
#include "../../include/catgrasp_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libcatgrasp_b200 is written for sm_90a (H100) only"
#endif

constexpr int CG_MAX_DEVICES = 64;   // per-device one-time kernel attributes are tracked in arrays of this size

struct cg_ctx {
  int device = 0;
  cudaStream_t own_stream = nullptr;
  cudaStream_t stream = nullptr;
  std::string err;
  int64_t launches = 0;
  // 0 = fp32 SIMT, 1 = wgmma bf16 3-pass, 2 = wgmma fp16 2-pass, 3 = wgmma single fp16 pass (default)
  int engine = 3;
  cudaEvent_t switch_event = nullptr;   // orders a newly selected stream behind the previous one (shared workspaces)
  uint32_t *ovf_flag = nullptr;   // device word: engine 2 or 3 saw a 128->1024 input above the fp16 range (clamped)
  int num_sms = 132;
  // optional event-pair timing of trunk launches (bench roofline)
  bool prof = false;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_events;
  // CG_TRACE=1 (diagnostics): an event after every launch; per-call-site durations are printed to stderr every 3000 launches
  bool trace = false;
  std::vector<std::pair<const char *, cudaEvent_t>> trace_events;
  // grow-only device workspace, carved per call
  void *ws = nullptr;
  size_t ws_bytes = 0;
  // second device arena for *_host entry points' device copies of I/O (carved only by cg_io_stage)
  void *io = nullptr;
  size_t io_bytes = 0;
  bool io_held = false;   // a cg_io_stage compute step is running: its pieces of io must stay where they are
};

#define CG_CUDA(ctx, call)                                                        \
  do {                                                                            \
    cudaError_t _e = (call);                                                      \
    if (_e != cudaSuccess) {                                                      \
      (ctx)->err = std::string(#call) + ": " + cudaGetErrorString(_e);            \
      return CG_ECUDA;                                                            \
    }                                                                             \
  } while (0)

#define CG_REQUIRE(ctx, cond, msg)                                                \
  do {                                                                            \
    if (!(cond)) {                                                                \
      (ctx)->err = std::string("invalid argument: ") + (msg);                     \
      return CG_EINVAL;                                                           \
    }                                                                             \
  } while (0)

void cg_trace_mark(cg_ctx *ctx, const char *where);
#define CG_STR2(x) #x
#define CG_STR(x) CG_STR2(x)

#define CG_LAUNCH_CHECK(ctx)                                                      \
  do {                                                                            \
    (ctx)->launches++;                                                            \
    if ((ctx)->trace) cg_trace_mark((ctx), __FILE__ ":" CG_STR(__LINE__));        \
    cudaError_t _e = cudaGetLastError();                                          \
    if (_e != cudaSuccess) {                                                      \
      (ctx)->err = std::string("kernel launch: ") + cudaGetErrorString(_e);       \
      return CG_ECUDA;                                                            \
    }                                                                             \
  } while (0)

// one Sdf3D grid resident in HBM: made by cg_sdf_create (cg_collide.cu) from a host grid or by cg_sdf_from_mesh
// (cg_sdf_build.cu) from a triangle mesh
struct cg_sdf {
  cg_ctx *ctx;
  float *grid;  // device, data[i][j][k]
  int nx, ny, nz;
  float origin[3];
  float res;
  int border_nonneg;   // every cell on the six boundary faces is >= 0 (true for padded grids, make_sdf.py:30)
  float border_min;    // smallest value on the six boundary faces
};
// border_nonneg / border_min of a host copy of the grid (decides the filter's out-of-box shortcut)
void cg_sdf_border_stats(cg_sdf *s, const float *grid_host);

int cg_ws_reserve(cg_ctx *ctx, size_t bytes);   // grow-only (cg_api.cu); call sites use cg_ws_carve / cg_io_stage
int cg_io_reserve(cg_ctx *ctx, size_t bytes);

// Bump allocator over an arena: each piece starts at the next multiple of 256 bytes from the base.  An arena over
// nullptr only measures: take() returns nullptr, and `off` ends at the bytes the same takes need in a real arena.
struct cg_arena {
  char *base;
  size_t off = 0;
  explicit cg_arena(void *b) : base(static_cast<char *>(b)) {}
  template <typename T>
  T *take(size_t n) {
    off = (off + 255) & ~size_t(255);
    T *p = base ? reinterpret_cast<T *>(base + off) : nullptr;
    off += n * sizeof(T);
    return p;
  }
};

// cg_ws_carve / cg_io_carve(ctx, layout): layout(cg_arena &) makes one call's take()s and stores the pointers.  It runs
// over a measuring arena, the context's ws (*_dev internals) or io (cg_io_stage) arena grows to the bytes measured, and
// it runs again over that arena.  Growing frees the arena: code that holds pieces of a carve must not call anything
// that carves the same arena.  An io carve while a cg_io_stage compute step holds io is refused.
template <typename Layout>
int cg_carve(cg_ctx *ctx, bool io, Layout &layout) {
  if (io && ctx->io_held) {
    ctx->err = "internal error: the compute step of a *_host call carved the io arena that holds its pieces";
    return CG_EINVAL;
  }
  cg_arena measure(nullptr);
  layout(measure);
  const int rc = io ? cg_io_reserve(ctx, measure.off) : cg_ws_reserve(ctx, measure.off);
  if (rc) return rc;
  cg_arena ar(io ? ctx->io : ctx->ws);
  layout(ar);
  if (ar.off == measure.off) return CG_OK;
  ctx->err = "internal error: a workspace layout carved a different size than it measured";
  return CG_EINVAL;
}
template <typename Layout> int cg_ws_carve(cg_ctx *ctx, Layout &&layout) { return cg_carve(ctx, false, layout); }
template <typename Layout> int cg_io_carve(cg_ctx *ctx, Layout &&layout) { return cg_carve(ctx, true, layout); }

// The io pieces of a *_host call, in declaration order: in(host, n) is copied from the host before the compute step,
// out(host, n) back to the host after it unless host is null, take<T>(n) is scratch.  0-element pieces copy nothing.
struct cg_io_pieces {
  struct Copy { void *dst; const void *src; size_t bytes; };
  cg_arena *ar = nullptr;
  std::vector<Copy> h2d, d2h;
  template <typename T> T *take(size_t n) { return ar->take<T>(n); }
  template <typename T> T *in(const T *host, size_t n) {
    T *d = take<T>(n);
    h2d.push_back({d, host, n * sizeof(T)});
    return d;
  }
  template <typename T> T *out(T *host, size_t n) {
    T *d = take<T>(n);
    if (host) d2h.push_back({host, d, n * sizeof(T)});
    return d;
  }
};

// cg_io_stage(ctx, layout, compute), what every *_host entry point does: carve layout(cg_io_pieces &) over io, enqueue
// the inputs' copies on ctx->stream, compute(), the outputs' copies, and synchronise.  A failing compute()'s status is
// returned with nothing copied back.  compute() may carve ws but not io, which holds its pieces: that is refused.
template <typename Layout, typename Compute>
int cg_io_stage(cg_ctx *ctx, Layout &&layout, Compute &&compute) {
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  cg_io_pieces io;
  int rc = cg_io_carve(ctx, [&](cg_arena &ar) { io = cg_io_pieces{&ar, {}, {}}; layout(io); });
  if (rc) return rc;
  for (const auto &c : io.h2d)
    if (c.bytes) CG_CUDA(ctx, cudaMemcpyAsync(c.dst, c.src, c.bytes, cudaMemcpyHostToDevice, ctx->stream));
  ctx->io_held = true;
  rc = compute();
  ctx->io_held = false;
  if (rc) return rc;
  for (const auto &c : io.d2h)
    if (c.bytes) CG_CUDA(ctx, cudaMemcpyAsync(c.dst, c.src, c.bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return CG_OK;
}

// one owning device allocation: freed when it goes out of scope unless release() hands it on
struct DevBuf {
  void *p = nullptr;
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  ~DevBuf() { if (p) cudaFree(p); }
  void *release() { return std::exchange(p, nullptr); }
};

// cudaMalloc into b: CG_ENOMEM when the device is out of memory, CG_ECUDA on any other error
inline int dev_alloc(cg_ctx *ctx, DevBuf &b, size_t bytes) {
  const cudaError_t e = cudaMalloc(&b.p, bytes);
  if (e == cudaErrorMemoryAllocation) {
    cudaGetLastError();
    ctx->err = "out of device memory";
    return CG_ENOMEM;
  }
  CG_CUDA(ctx, e);
  return CG_OK;
}

// ---- order-preserving float <-> uint key (for atomicMax on floats) --------
__host__ __device__ __forceinline__ uint32_t cg_f2key(float f) {
#ifdef __CUDA_ARCH__
  uint32_t b = __float_as_uint(f);
#else
  uint32_t b;
  memcpy(&b, &f, 4);
#endif
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__host__ __device__ __forceinline__ float cg_key2f(uint32_t k) {
  uint32_t b = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
#ifdef __CUDA_ARCH__
  return __uint_as_float(b);
#else
  float f;
  memcpy(&f, &b, 4);
  return f;
#endif
}

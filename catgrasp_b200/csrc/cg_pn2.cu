// cg_pn2.cu -- PointNet++ sampling / grouping primitives (pointnet2.py:14-149).
//
// These are HBM/L2-bound index kernels: no tensor cores.  Distances follow the
// reference's floating-point forms exactly where the result feeds a comparison:
//   FPS        : direct form  ((dx*dx + dy*dy) + dz*dz), pointnet2.py:71
//   ball query : expanded form -2*<s,d> + |s|^2 + |d|^2,  pointnet2.py:30-32
#include <cooperative_groups.h>
#include <stdlib.h>

#include "cg_common.cuh"

namespace cgr = cooperative_groups;

namespace {

__device__ __forceinline__ float sq_direct(float x, float y, float z, float cx, float cy, float cz) {
  const float dx = __fsub_rn(x, cx), dy = __fsub_rn(y, cy), dz = __fsub_rn(z, cz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ float sq_expanded(float sx, float sy, float sz, float ss, float dx, float dy, float dz) {
  // dist = -2 * (src . dst); dist += sum(src^2); dist += sum(dst^2)
  const float dot = fmaf(sz, dz, fmaf(sy, dy, __fmul_rn(sx, dx)));
  const float dd = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
  return __fadd_rn(__fadd_rn(__fmul_rn(-2.f, dot), ss), dd);
}

// ---------------------------------------------------------------- FPS ------
// One CTA per cloud.  Running min-distances live in shared memory; coordinates
// too when they fit (16 B/point), else they are re-read through L1/L2.
constexpr int FPS_T = 1024;

template <bool XYZ_IN_SMEM>
__global__ void __launch_bounds__(FPS_T, 1) fps_kernel(const float *__restrict__ xyz, int N, int npoint,
                                                       const int32_t *__restrict__ start_idx,
                                                       int32_t *__restrict__ out_idx) {
  extern __shared__ __align__(16) float sm[];
  float *dist = sm;                       // [N]
  float *sx = sm + N;                     // [3N] (only when XYZ_IN_SMEM)
  __shared__ float red_v[32];
  __shared__ int red_i[32];
  __shared__ int far_s;
  const int b = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const float *P = xyz + (size_t)b * N * 3;
  for (int i = tid; i < N; i += FPS_T) dist[i] = 1e10f;    // pointnet2.py:65
  if (XYZ_IN_SMEM)
    for (int i = tid; i < 3 * N; i += FPS_T) sx[i] = P[i];
  if (tid == 0) far_s = start_idx ? start_idx[b] : 0;      // :66 (explicit instead of torch.randint)
  __syncthreads();
  const float *Q = XYZ_IN_SMEM ? sx : P;
  for (int it = 0; it < npoint; it++) {
    const int far = far_s;
    if (tid == 0) out_idx[(size_t)b * npoint + it] = far;  // :69
    const float cx = Q[3 * far], cy = Q[3 * far + 1], cz = Q[3 * far + 2];
    float best = -1.f;
    int besti = 0x7fffffff;
    for (int i = tid; i < N; i += FPS_T) {
      const float d = sq_direct(Q[3 * i], Q[3 * i + 1], Q[3 * i + 2], cx, cy, cz);  // :71
      float dm = dist[i];
      if (d < dm) { dm = d; dist[i] = d; }                 // :72-73
      if (dm > best) { best = dm; besti = i; }             // first maximum (lowest index) per thread
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
      if (ov > best || (ov == best && oi < besti)) { best = ov; besti = oi; }
    }
    if (lane == 0) { red_v[wid] = best; red_i[wid] = besti; }   // previous round's readers passed its last barrier
    __syncthreads();
    if (wid == 0) {
      best = red_v[lane];
      besti = red_i[lane];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
        if (ov > best || (ov == best && oi < besti)) { best = ov; besti = oi; }
      }
      if (lane == 0) far_s = besti;                        // :74 torch.max -> first max index
    }
    __syncthreads();
  }
}

// Cluster-cooperative FPS: a thread-block cluster (8 CTAs, 16 where the device allows it) per cloud.  Every thread keeps
// its PPT points AND their running min-distances in registers for the whole kernel, so a round touches no memory
// except the hand-over of one 24-byte candidate per CTA: warp redux -> CTA (shared memory) -> all CTAs of the cluster
// (distributed shared memory), signalled by remote mbarrier arrivals (release/acquire at cluster scope; a full
// barrier.cluster per round measured 1.9 us/round, 3x the exchange itself).  The candidate carries the point's coordinates, so the
// next round starts without a dependent global load.  Semantics are the reference's (pointnet2.py:54-75): direct-form
// fp32 distances, strict `dist < distance` update, first (lowest-index) maximum.
constexpr int FPSC_T = 256;
constexpr int FPSC_MAXC = 16;

struct FpsCand {
  float v, x, y, z;
  int i;
  int pad[3];
};

__device__ __forceinline__ uint32_t fps_smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
// (value desc, index asc) winner of a warp with two redux instructions: distances are >= 0, so their bit patterns order
// like unsigned integers (-2 marks an unused slot and maps to 0)
__device__ __forceinline__ void fps_warp_winner(float v, int i, uint32_t &wbits, int &wi) {
  const uint32_t bits = v < 0.f ? 0u : __float_as_uint(v) + 1u;
  wbits = __reduce_max_sync(0xffffffffu, bits);
  wi = (int)__reduce_min_sync(0xffffffffu, bits == wbits ? (uint32_t)i : 0xffffffffu);
}

template <int PPT>
__global__ void __launch_bounds__(FPSC_T, 1) fps_cluster_kernel(const float *__restrict__ xyz, int N, int npoint,
                                                                const int32_t *__restrict__ start_idx,
                                                                int32_t *__restrict__ out_idx) {
  cgr::cluster_group cluster = cgr::this_cluster();
  const int csize = (int)cluster.num_blocks(), crank = (int)cluster.block_rank();
  const int b = blockIdx.x / csize;
  __shared__ FpsCand rec[2][FPSC_MAXC];            // written by every CTA of the cluster (slot = writer's rank)
  __shared__ FpsCand wred[FPSC_T / 32];
  __shared__ unsigned long long xbar[2];           // one arrival per CTA of the cluster and round (parity = round & 1)
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const float *P = xyz + (size_t)b * N * 3;
  const int Ttot = csize * FPSC_T, gtid = crank * FPSC_T + tid;
  float px[PPT], py[PPT], pz[PPT], pd[PPT];
#pragma unroll
  for (int k = 0; k < PPT; k++) {
    const int i = gtid + k * Ttot;
    if (i < N) {
      px[k] = P[3 * i]; py[k] = P[3 * i + 1]; pz[k] = P[3 * i + 2];
      pd[k] = 1e10f;                                        // pointnet2.py:65
    } else {
      px[k] = py[k] = pz[k] = 0.f;
      pd[k] = -2.f;                                         // never selected, never updated (d >= 0 < -2 is false)
    }
  }
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(fps_smem_u32(&xbar[0])), "r"(csize));
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(fps_smem_u32(&xbar[1])), "r"(csize));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  int far = start_idx ? start_idx[b] : 0;                   // :66 (explicit instead of torch.randint)
  float cx = P[3 * far], cy = P[3 * far + 1], cz = P[3 * far + 2];
  cluster.sync();                                           // barriers initialised in every CTA before remote arrivals
  for (int it = 0; it < npoint; it++) {
    if (crank == 0 && tid == 0) out_idx[(size_t)b * npoint + it] = far;   // :69
    if (it == npoint - 1) break;
    float bv = -1.f, bx = 0.f, by = 0.f, bz = 0.f;
    int bi = 0x7fffffff;
#pragma unroll
    for (int k = 0; k < PPT; k++) {
      const float d = sq_direct(px[k], py[k], pz[k], cx, cy, cz);        // :71
      if (d < pd[k]) pd[k] = d;                                          // :72-73
      if (pd[k] > bv) { bv = pd[k]; bi = gtid + k * Ttot; bx = px[k]; by = py[k]; bz = pz[k]; }   // k ascending = index ascending
    }
    uint32_t wb;
    int wi;
    fps_warp_winner(bv, bi, wb, wi);
    if (bi == wi) { wred[wid].v = bv; wred[wid].i = bi; wred[wid].x = bx; wred[wid].y = by; wred[wid].z = bz; }   // one lane
    __syncthreads();
    const int buf = it & 1;
    if (wid == 0) {
      FpsCand c;
      c.v = -2.f; c.i = 0x7fffffff; c.x = c.y = c.z = 0.f;
      if (lane < FPSC_T / 32) c = wred[lane];
      uint32_t cb;
      int ci;
      fps_warp_winner(c.v, c.i, cb, ci);
      const int src = __ffs(__ballot_sync(0xffffffffu, c.i == ci)) - 1;
      const float v = __shfl_sync(0xffffffffu, c.v, src), x = __shfl_sync(0xffffffffu, c.x, src),
                  y = __shfl_sync(0xffffffffu, c.y, src), z = __shfl_sync(0xffffffffu, c.z, src);
      if (lane < csize) {     // lane r delivers this CTA's candidate into CTA r's slot [crank] and arrives on CTA r's barrier
        FpsCand *dst = cluster.map_shared_rank(&rec[buf][crank], lane);
        dst->v = v; dst->x = x; dst->y = y; dst->z = z; dst->i = ci;
        uint32_t rbar;
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rbar) : "r"(fps_smem_u32(&xbar[buf])), "r"(lane));
        asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(rbar) : "memory");
      }
    }
    {   // every thread waits for the csize arrivals of this round (acquire at cluster scope: the records are visible)
      const uint32_t bar = fps_smem_u32(&xbar[buf]), parity = ((uint32_t)it >> 1) & 1u;
      uint32_t ok;
      do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(bar), "r"(parity)
            : "memory");
      } while (!ok);
    }
    float gv = -2.f;
    int gi = 0x7fffffff;
    for (int r = 0; r < csize; r++) {
      const float ov = rec[buf][r].v;
      const int oi = rec[buf][r].i;
      if (ov > gv || (ov == gv && oi < gi)) { gv = ov; gi = oi; cx = rec[buf][r].x; cy = rec[buf][r].y; cz = rec[buf][r].z; }
    }
    far = gi;                                               // :74 torch.max -> first max index
    // wred is rewritten next round only after every thread passed this round's barrier wait; rec[buf] / xbar[buf] are
    // reused two rounds later, after every CTA has completed round it + 1, i.e. after all of them finished reading here
  }
  cluster.sync();             // no CTA exits while a peer may still write into its shared memory
}

// ---------------------------------------------------------- ball query ------
// One warp per centroid; 32 points per step, ballot + prefix popcount keeps the
// reference's "nsample smallest indices" order without a sort.
constexpr int BQ_WARPS = 8;

__global__ void __launch_bounds__(BQ_WARPS * 32) ball_query_kernel(float r2, int nsample,
                                                                    const float *__restrict__ xyz,
                                                                    const float *__restrict__ new_xyz, int B, int N,
                                                                    int S, int32_t *__restrict__ out_idx) {
  const long w = (long)blockIdx.x * BQ_WARPS + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= (long)B * S) return;
  const int b = (int)(w / S);
  const float *P = xyz + (size_t)b * N * 3;
  const float sx = new_xyz[w * 3], sy = new_xyz[w * 3 + 1], sz = new_xyz[w * 3 + 2];
  const float ss = __fadd_rn(__fadd_rn(__fmul_rn(sx, sx), __fmul_rn(sy, sy)), __fmul_rn(sz, sz));
  int32_t *out = out_idx + w * nsample;
  int cnt = 0;
  int first = N;   // an empty ball leaves N everywhere (reference behaviour, SURVEY Appendix A2)
  for (int base = 0; base < N && cnt < nsample; base += 32) {
    const int i = base + lane;
    bool in = false;
    if (i < N) {
      const float d = sq_expanded(sx, sy, sz, ss, P[3 * i], P[3 * i + 1], P[3 * i + 2]);
      in = !(d > r2);                                      // pointnet2.py:93
    }
    const unsigned m = __ballot_sync(0xffffffffu, in);
    if (m) {
      if (cnt == 0) first = base + __ffs(m) - 1;
      const int slot = cnt + __popc(m & ((1u << lane) - 1u));
      if (in && slot < nsample) out[slot] = i;
      cnt += __popc(m);
    }
  }
  if (cnt > nsample) cnt = nsample;
  for (int s = cnt + lane; s < nsample; s += 32) out[s] = first;   // :95-97
}

// ------------------------------------------------------ dense helpers ------
// (B,S,3) x (B,N,3) -> (B,S,N): a CTA produces a 64 x 256 tile; the 64 source rows and their squared norms sit in
// shared memory, every thread owns one destination point and streams 64 coalesced stores (the kernel is bound by the
// S*N*4 output bytes).
constexpr int SQ_TS = 64, SQ_TN = 256;
__global__ void __launch_bounds__(SQ_TN) square_distance_kernel(const float *__restrict__ src, const float *__restrict__ dst, int B,
                                                                int S, int N, float *__restrict__ out) {
  __shared__ float4 ss[SQ_TS];
  const int b = blockIdx.z, s0 = blockIdx.y * SQ_TS, n = blockIdx.x * SQ_TN + threadIdx.x;
  if (threadIdx.x < SQ_TS && s0 + threadIdx.x < S) {
    const float *s = src + ((size_t)b * S + s0 + threadIdx.x) * 3;
    ss[threadIdx.x] = make_float4(s[0], s[1], s[2],
                                  __fadd_rn(__fadd_rn(__fmul_rn(s[0], s[0]), __fmul_rn(s[1], s[1])), __fmul_rn(s[2], s[2])));
  }
  __syncthreads();
  if (n >= N) return;
  const float *d = dst + ((size_t)b * N + n) * 3;
  const float dx = d[0], dy = d[1], dz = d[2];
  const int cnt = min(SQ_TS, S - s0);
  float *o = out + ((size_t)b * S + s0) * N + n;
  for (int i = 0; i < cnt; i++) {
    const float4 s = ss[i];
    o[(size_t)i * N] = sq_expanded(s.x, s.y, s.z, s.w, dx, dy, dz);
  }
}

__global__ void index_points_kernel(const float *__restrict__ points, const int32_t *__restrict__ idx, int B, int N,
                                    int C, int S, float *__restrict__ out) {
  const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long total = (long)B * S * C;
  if (t >= total) return;
  const int c = (int)(t % C);
  const long bs = t / C;
  const int b = (int)(bs / S);
  const int id = idx[bs];
  out[t] = (id >= 0 && id < N) ? points[((size_t)b * N + id) * C + c] : 0.f;
}

__global__ void group_points_kernel(const float *__restrict__ xyz, const float *__restrict__ points,
                                    const float *__restrict__ new_xyz, const int32_t *__restrict__ idx, int B, int N,
                                    int D, int S, int K, float *__restrict__ out) {
  const int Cc = 3 + D;
  const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long total = (long)B * S * K * Cc;
  if (t >= total) return;
  const int c = (int)(t % Cc);
  const long bsk = t / Cc;
  const long bs = bsk / K;
  const int b = (int)(bs / S);
  const int id = idx[bsk];
  float v = 0.f;
  if (id >= 0 && id < N) {
    if (c < 3) v = __fsub_rn(xyz[((size_t)b * N + id) * 3 + c], new_xyz[bs * 3 + c]);   // pointnet2.py:119
    else v = points[((size_t)b * N + id) * D + (c - 3)];                                 // :122-123
  }
  out[t] = v;
}

}  // namespace

extern "C" int cg_fps_dev(cg_ctx *ctx, const float *xyz, int B, int N, int npoint, const int32_t *start_idx,
                          int32_t *out_idx) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, xyz && out_idx && B > 0 && N > 0 && npoint > 0, "fps: bad arguments");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  // cluster size: 16 CTAs (non-portable) when the device can co-schedule them, else 8; points per thread in registers
  static int csize_dev[CG_MAX_DEVICES] = {};
  if (csize_dev[ctx->device] == 0) {
    int cs = 8;
    const void *fns[4] = {(const void *)fps_cluster_kernel<4>, (const void *)fps_cluster_kernel<8>,
                          (const void *)fps_cluster_kernel<16>, (const void *)fps_cluster_kernel<32>};
    bool ok16 = true;
    for (const void *f : fns)
      if (cudaFuncSetAttribute(f, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess) ok16 = false;
    if (ok16) {
      cudaLaunchConfig_t q = {};
      q.gridDim = dim3(16); q.blockDim = dim3(FPSC_T);
      cudaLaunchAttribute at;
      at.id = cudaLaunchAttributeClusterDimension;
      at.val.clusterDim.x = 16; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
      q.attrs = &at; q.numAttrs = 1;
      int ncl = 0;
      if (cudaOccupancyMaxActiveClusters(&ncl, fps_cluster_kernel<8>, &q) == cudaSuccess && ncl >= 1) cs = 16;
    }
    cudaGetLastError();
    csize_dev[ctx->device] = cs;
  }
  // Cluster size: cost model per round ~ base(csize) + 0.025 x points per thread, base = 0.70 / 0.83 / 1.0 / 1.45
  // for 2 / 4 / 8 / 16 CTAs (the cross-CTA exchange is the floor: remote store + remote mbarrier arrive + acquire wait,
  // and it grows with the cluster); pick the cheapest size whose points fit the 32-registers-per-thread budget.
  int csize = csize_dev[ctx->device];
  {
    const int sizes[4] = {2, 4, 8, 16};
    const double base[4] = {0.70, 0.83, 1.0, 1.45};
    double best = 1e30;
    for (int k = 0; k < 4; k++) {
      if (sizes[k] > csize_dev[ctx->device]) break;
      const long ppt = ((long)N + (long)sizes[k] * FPSC_T - 1) / ((long)sizes[k] * FPSC_T);
      if (ppt > 32) continue;
      const double cost = base[k] + 0.025 * (double)ppt;
      if (cost < best) { best = cost; csize = sizes[k]; }
    }
  }
#ifdef CG_EXPERIMENTS
  if (getenv("CG_FPS_CLUSTER")) csize = atoi(getenv("CG_FPS_CLUSTER"));   // developer builds: cluster-size sweep
#endif
  const long per_thread = ((long)N + (long)csize * FPSC_T - 1) / ((long)csize * FPSC_T);
  CG_REQUIRE(ctx, per_thread <= 32, "fps: N too large (max 32 points per thread x 256 threads x cluster size)");
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(B * csize));
  cfg.blockDim = dim3(FPSC_T);
  cfg.stream = ctx->stream;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = (unsigned)csize; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  if (per_thread <= 4) CG_CUDA(ctx, cudaLaunchKernelEx(&cfg, fps_cluster_kernel<4>, xyz, N, npoint, start_idx, out_idx));
  else if (per_thread <= 8) CG_CUDA(ctx, cudaLaunchKernelEx(&cfg, fps_cluster_kernel<8>, xyz, N, npoint, start_idx, out_idx));
  else if (per_thread <= 16) CG_CUDA(ctx, cudaLaunchKernelEx(&cfg, fps_cluster_kernel<16>, xyz, N, npoint, start_idx, out_idx));
  else CG_CUDA(ctx, cudaLaunchKernelEx(&cfg, fps_cluster_kernel<32>, xyz, N, npoint, start_idx, out_idx));
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

// the round-1 single-CTA kernel (kept for comparison in scripts/bench_primitives.py)
extern "C" int cg_fps_single_cta_dev(cg_ctx *ctx, const float *xyz, int B, int N, int npoint, const int32_t *start_idx,
                                     int32_t *out_idx) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, xyz && out_idx && B > 0 && N > 0 && npoint > 0, "fps: bad arguments");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t full = (size_t)N * 16, dist_only = (size_t)N * 4;
  const size_t cap = 220 * 1024;
  CG_REQUIRE(ctx, dist_only <= cap, "fps (single CTA): N too large for the shared-memory distance array (max 56320)");
  static bool attr_set[CG_MAX_DEVICES] = {};   // the attribute is per device
  if (!attr_set[ctx->device]) {
    CG_CUDA(ctx, cudaFuncSetAttribute(fps_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cap));
    CG_CUDA(ctx, cudaFuncSetAttribute(fps_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cap));
    attr_set[ctx->device] = true;
  }
  if (full <= cap)
    fps_kernel<true><<<B, FPS_T, full, ctx->stream>>>(xyz, N, npoint, start_idx, out_idx);
  else
    fps_kernel<false><<<B, FPS_T, dist_only, ctx->stream>>>(xyz, N, npoint, start_idx, out_idx);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

extern "C" int cg_ball_query_dev(cg_ctx *ctx, float radius2, int nsample, const float *xyz, const float *new_xyz,
                                 int B, int N, int S, int32_t *out_idx) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, xyz && new_xyz && out_idx && B > 0 && N > 0 && S > 0 && nsample > 0, "ball_query: bad arguments");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const long warps = (long)B * S;
  ball_query_kernel<<<(unsigned)((warps + BQ_WARPS - 1) / BQ_WARPS), BQ_WARPS * 32, 0, ctx->stream>>>(
      radius2, nsample, xyz, new_xyz, B, N, S, out_idx);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

extern "C" int cg_square_distance_dev(cg_ctx *ctx, const float *src, const float *dst, int B, int S, int N,
                                      float *out) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, src && dst && out && B > 0 && S > 0 && N > 0, "square_distance: bad arguments");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  CG_REQUIRE(ctx, B <= 65535 && (S + SQ_TS - 1) / SQ_TS <= 65535, "square_distance: B or S too large for one launch");
  dim3 grid((N + SQ_TN - 1) / SQ_TN, (S + SQ_TS - 1) / SQ_TS, B);
  square_distance_kernel<<<grid, SQ_TN, 0, ctx->stream>>>(src, dst, B, S, N, out);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

extern "C" int cg_index_points_dev(cg_ctx *ctx, const float *points, const int32_t *idx, int B, int N, int C, int S,
                                   float *out) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, points && idx && out && B > 0 && N > 0 && C > 0 && S > 0, "index_points: bad arguments");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const long total = (long)B * S * C;
  index_points_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>(points, idx, B, N, C, S, out);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

extern "C" int cg_group_points_dev(cg_ctx *ctx, const float *xyz, const float *points, const float *new_xyz,
                                   const int32_t *idx, int B, int N, int D, int S, int K, float *out) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, xyz && new_xyz && idx && out && B > 0 && N > 0 && S > 0 && K > 0 && D >= 0, "group_points: bad arguments");
  CG_REQUIRE(ctx, D == 0 || points, "group_points: points required when D > 0");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const long total = (long)B * S * K * (3 + D);
  group_points_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>(xyz, points, new_xyz, idx, B, N, D, S, K,
                                                                           out);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

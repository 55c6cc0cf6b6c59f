// cg_sa.cu -- PointNet++ set-abstraction / feature-propagation stacks on top of the sampling/grouping primitives of
// cg_pn2.cu (north_star: "per-group MLP+max-pool on tensor cores only where the group x channel tile is a genuine
// dense contraction (vectorised FMA otherwise)").
//
// The reference ships only the primitives (/root/reference/pointnet2.py:101-149) and cites the upstream module family
// in its model docstrings (:274,:304); the modules restated here are that family's PointNetSetAbstraction /
// PointNetFeaturePropagation:
//   SA:  sample_and_group -> (B,S,K,3+D) -> [1x1 conv + BN + ReLU] x L over all B*S*K rows -> max over K -> (B,S,C_L)
//   FP:  3 nearest neighbours of every dense point among the S sparse points (expanded-form square_distance, :14-33),
//        weights (1/(d+1e-8)) / sum, weighted sum of their features -> concat skip features -> [conv + BN + ReLU] x L
// Every layer is launched through cg_linear_launch: a layer with a tensor-core image (K a multiple of 64, >= 64 output
// channels) and >= 64 rows runs on wgmma (linear_tc_kernel, bf16 hi/lo x3, fp32 accumulate); the first layer of an SA
// stack (K = 3 + D, typically 6) is an FMA kernel -- it is not a tensor-core shape.
#include <float.h>
#include <memory>

#include "cg_net.cuh"

struct cg_mlp {
  cg_ctx *ctx;
  std::vector<cg_layer> L;   // device weights (BN folded by the host), each layer's tensor-core image owned here
};

namespace {

// x (G,K,C) -> out (G,C): max over the K rows of every group; thread = (group, channel), coalesced over channels
__global__ void group_max_kernel(const float *__restrict__ x, int G, int K, int C, float *__restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)G * C) return;
  const int g = (int)(idx / C), c = (int)(idx - (long long)g * C);
  const float *p = x + ((size_t)g * K) * C + c;
  float m = -FLT_MAX;
  for (int k = 0; k < K; k++) m = fmaxf(m, p[(size_t)k * C]);
  out[idx] = m;
}

// 3 nearest of the S sparse points for every dense point.  One thread per dense point; the sparse cloud is staged
// through shared memory in tiles.  Distance = the reference's expanded form, same fp32 operation order as
// square_distance_kernel (cg_pn2.cu): dot = fma(z,z', fma(y,y', x*x')), d = ((-2*dot) + |a|^2) + |b|^2.
// Selection = the first three entries of a stable ascending sort (ties -> lower index), which is what torch.sort
// returns for distinct distances; exact ties between different sparse points are measure-zero for real clouds.
// S == 2: the module family keeps the two neighbours it has (sort()[:, :, :3] of two columns), so the weights are
// normalised over two and the third slot is written as index 0, weight 0.
constexpr int NN_T = 128, NN_TILE = 1024;
__global__ void three_nn_kernel(const float *__restrict__ xyz1, const float *__restrict__ xyz2, int N, int S,
                                int32_t *__restrict__ out_idx, float *__restrict__ out_w) {
  __shared__ float sx[NN_TILE], sy[NN_TILE], sz[NN_TILE], sn[NN_TILE];
  const int b = blockIdx.y;
  const int n = blockIdx.x * NN_T + threadIdx.x;
  const float *q = xyz1 + ((size_t)b * N + (n < N ? n : N - 1)) * 3;
  const float qx = q[0], qy = q[1], qz = q[2];
  const float qn = __fadd_rn(__fadd_rn(__fmul_rn(qx, qx), __fmul_rn(qy, qy)), __fmul_rn(qz, qz));
  float d0 = FLT_MAX, d1 = FLT_MAX, d2 = FLT_MAX;
  int i0 = 0, i1 = 0, i2 = 0;
  for (int s0 = 0; s0 < S; s0 += NN_TILE) {
    const int cnt = min(NN_TILE, S - s0);
    __syncthreads();
    for (int i = threadIdx.x; i < cnt; i += NN_T) {
      const float *p = xyz2 + ((size_t)b * S + s0 + i) * 3;
      const float x = p[0], y = p[1], z = p[2];
      sx[i] = x; sy[i] = y; sz[i] = z;
      sn[i] = __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
    }
    __syncthreads();
    for (int i = 0; i < cnt; i++) {
      const float dot = __fmaf_rn(qz, sz[i], __fmaf_rn(qy, sy[i], __fmul_rn(qx, sx[i])));
      const float d = __fadd_rn(__fadd_rn(__fmul_rn(-2.f, dot), qn), sn[i]);
      if (d < d2) {
        const int id = s0 + i;
        if (d < d1) {
          d2 = d1; i2 = i1;
          if (d < d0) { d1 = d0; i1 = i0; d0 = d; i0 = id; }
          else { d1 = d; i1 = id; }
        } else { d2 = d; i2 = id; }
      }
    }
  }
  if (n >= N) return;
  // dist_recip = 1 / (d + 1e-8); weight = dist_recip / sum(dist_recip)   (fp32, torch operation order)
  const float r0 = __fdiv_rn(1.f, __fadd_rn(d0, 1e-8f)), r1 = __fdiv_rn(1.f, __fadd_rn(d1, 1e-8f));
  float norm = __fadd_rn(r0, r1), w2 = 0.f;
  if (S >= 3) {
    const float r2 = __fdiv_rn(1.f, __fadd_rn(d2, 1e-8f));
    norm = __fadd_rn(norm, r2);
    w2 = __fdiv_rn(r2, norm);
  }
  const size_t o = ((size_t)b * N + n) * 3;
  out_idx[o] = i0; out_idx[o + 1] = i1; out_idx[o + 2] = i2;
  out_w[o] = __fdiv_rn(r0, norm); out_w[o + 1] = __fdiv_rn(r1, norm); out_w[o + 2] = w2;
}

// out[b][n][off + c] = sum_j w[b][n][j] * points2[b][idx[b][n][j]][c]   (sum order j = 0,1,2 like torch.sum over dim 2;
// j = 0,1 when S == 2) and out[b][n][c] = points1[b][n][c] for the skip features; one warp per dense point, lanes over
// channels.
__global__ void three_interp_kernel(const float *__restrict__ points1, int D1, const float *__restrict__ points2, int D2,
                                    const int32_t *__restrict__ idx, const float *__restrict__ w, int B, int N, int S,
                                    float *__restrict__ out) {
  const long long wid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= (long long)B * N) return;
  const int b = (int)(wid / N);
  const int32_t *id = idx + wid * 3;
  const float *ww = w + wid * 3;
  const int i0 = id[0], i1 = id[1], i2 = id[2];
  const float w0 = ww[0], w1 = ww[1], w2 = ww[2];
  const float *p0 = points2 + ((size_t)b * S + i0) * D2, *p1 = points2 + ((size_t)b * S + i1) * D2,
              *p2 = points2 + ((size_t)b * S + i2) * D2;
  float *o = out + (size_t)wid * (D1 + D2);
  if (points1)
    for (int c = lane; c < D1; c += 32) o[c] = points1[(size_t)wid * D1 + c];
  for (int c = lane; c < D2; c += 32) {
    const float v = __fadd_rn(__fmul_rn(p0[c], w0), __fmul_rn(p1[c], w1));
    o[D1 + c] = S >= 3 ? __fadd_rn(v, __fmul_rn(p2[c], w2)) : v;
  }
}

int run_mlp(cg_mlp *m, const float *x, long long R, float *out_last, float **last_buf) {
  cg_ctx *ctx = m->ctx;
  const int nlayers = (int)m->L.size();
  int maxc = 0;
  for (const cg_layer &l : m->L) maxc = l.C > maxc ? l.C : maxc;
  float *pp[2];
  int rc = cg_ws_carve(ctx, [&](cg_arena &ar) { for (float *&p : pp) p = ar.take<float>((size_t)R * maxc); });
  if (rc) return rc;
  const float *cur = x;
  for (int i = 0; i < nlayers; i++) {
    float *dst = (i == nlayers - 1 && out_last) ? out_last : pp[i & 1];
    if ((rc = cg_linear_launch(ctx, m->L[i], cur, (int)R, dst, CG_FC_RELU))) return rc;
    cur = dst;
  }
  if (last_buf) *last_buf = const_cast<float *>(cur);
  return CG_OK;
}

}  // namespace

extern "C" int cg_mlp_create(cg_ctx *ctx, int nlayers, const int *dims, const float *const *Wt_host,
                             const float *const *b_host, cg_mlp **out) {
  if (!ctx || !out) return CG_EINVAL;
  CG_REQUIRE(ctx, nlayers >= 1 && nlayers <= 8 && dims && Wt_host && b_host, "mlp_create: bad arguments");
  for (int i = 0; i <= nlayers; i++) CG_REQUIRE(ctx, dims[i] > 0 && dims[i] <= 4096, "mlp_create: channel count out of range");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  // null layers, so that every error return below frees what exists so far
  std::unique_ptr<cg_mlp, void (*)(cg_mlp *)> m(new cg_mlp(), cg_mlp_destroy);
  m->ctx = ctx;
  m->L.assign(nlayers, cg_layer{});
  for (int i = 0; i < nlayers; i++) {
    cg_layer &l = m->L[i];
    l.K = dims[i];
    l.C = dims[i + 1];
    float *W = nullptr, *b = nullptr;
    const size_t nw = (size_t)l.K * l.C;
    CG_CUDA(ctx, cudaMalloc(&W, nw * sizeof(float)));
    l.Wt = W;
    CG_CUDA(ctx, cudaMalloc(&b, (size_t)l.C * sizeof(float)));
    l.b = b;
    CG_CUDA(ctx, cudaMemcpyAsync(W, Wt_host[i], nw * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    CG_CUDA(ctx, cudaMemcpyAsync(b, b_host[i], (size_t)l.C * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    const int rc = cg_linear_tc_image(ctx, Wt_host[i], l.K, l.C, &l.tc);
    if (rc != CG_OK) return rc;
  }
  CG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  *out = m.release();
  return CG_OK;
}

extern "C" void cg_mlp_destroy(cg_mlp *m) {
  if (!m) return;
  cudaSetDevice(m->ctx->device);
  for (const cg_layer &l : m->L) {
    cudaFree(const_cast<float *>(l.Wt));
    cudaFree(const_cast<float *>(l.b));
    cudaFree(const_cast<void *>(l.tc));
  }
  delete m;
}

extern "C" int cg_shared_mlp_dev(cg_mlp *m, const float *x, int64_t R, float *out) {
  if (!m) return CG_EINVAL;
  cg_ctx *ctx = m->ctx;
  CG_REQUIRE(ctx, x && out && R > 0 && R < (1ll << 31), "shared_mlp: bad arguments");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  return run_mlp(m, x, R, out, nullptr);
}

extern "C" int cg_group_mlp_max_dev(cg_mlp *m, const float *grouped, int G, int K, float *out) {
  if (!m) return CG_EINVAL;
  cg_ctx *ctx = m->ctx;
  CG_REQUIRE(ctx, grouped && out && G > 0 && K > 0 && (long long)G * K < (1ll << 31), "group_mlp_max: bad arguments");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  float *last = nullptr;
  int rc = run_mlp(m, grouped, (long long)G * K, nullptr, &last);
  if (rc) return rc;
  const int C = m->L.back().C;
  const long long total = (long long)G * C;
  group_max_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>(last, G, K, C, out);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

extern "C" int cg_three_interp_dev(cg_ctx *ctx, const float *xyz1, const float *xyz2, const float *points1, int D1,
                                   const float *points2, int D2, int B, int N, int S, float *out, int32_t *out_idx,
                                   float *out_weight) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, xyz1 && xyz2 && points2 && out && B > 0 && N > 0 && S >= 2 && D2 > 0 && D1 >= 0,
             "three_interp: bad arguments (S >= 2 required; S == 1 is a plain broadcast)");
  CG_REQUIRE(ctx, (points1 != nullptr) == (D1 > 0), "three_interp: points1 / D1 mismatch");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  int32_t *idx = out_idx;
  float *w = out_weight;
  if (!idx || !w) {
    const size_t n3 = (size_t)B * N * 3;
    int32_t *ti; float *tw;
    int rc = cg_ws_carve(ctx, [&](cg_arena &ar) { ti = ar.take<int32_t>(n3); tw = ar.take<float>(n3); });
    if (rc) return rc;
    if (!idx) idx = ti;
    if (!w) w = tw;
  }
  dim3 g1((N + NN_T - 1) / NN_T, B);
  three_nn_kernel<<<g1, NN_T, 0, ctx->stream>>>(xyz1, xyz2, N, S, idx, w);
  CG_LAUNCH_CHECK(ctx);
  const long long warps = (long long)B * N;
  three_interp_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, ctx->stream>>>(points1, D1, points2, D2, idx, w, B, N, S,
                                                                                   out);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

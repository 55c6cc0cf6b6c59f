// cg_linear_tc.cu -- fully-connected layers on wgmma (bf16 hi/lo x3, fp32 accumulate in registers).
//
//   Y[M][N] = act( X[M][K] @ Wt[K][N] + bias[row / bias_row_div][N] )      K % 64 == 0
//
// replaces nn.Linear / Conv1d(k=1) + folded BN (+ReLU) of the PointNet heads (pointnet2.py:176-183, :214-221,
// :295-298, :323-327) for M >= 64 rows.  One CTA = 128 rows x 128 output columns, one warpgroup per 64 rows; K runs
// through a 3-stage ring of 64-wide K-blocks: the weight block arrives as a bulk copy of the host-prepared swizzled
// image (B operand), the activations are read as fp32 (or as the trunk's order-preserving keys) straight into the
// A-operand register fragments, split into bf16 hi/lo on the way.
#include <algorithm>

#include "cg_net.cuh"
#include "cg_tc_ptx.cuh"

namespace {
using namespace cg_ptx;

constexpr uint32_t PIECE = 16384;             // [128 rows x 64 bf16]
constexpr int STAGES = 3;
constexpr uint32_t STAGE_BYTES = 2 * PIECE;   // B hi, B lo of one 64-wide K-block
constexpr int LT = 256;                       // two consumer warpgroups: rows 0-63 / 64-127 of the tile

struct Bars {
  unsigned long long full[STAGES], empty[STAGES];
};
constexpr size_t LSMEM = STAGES * STAGE_BYTES + sizeof(Bars);

__global__ void __launch_bounds__(LT, 1) linear_tc_kernel(const float *__restrict__ X, int M, int K,
                                                          const unsigned char *__restrict__ wimg,
                                                          const float *__restrict__ bias, int N, int relu,
                                                          int bias_row_div, int x_is_keys, float *__restrict__ Y) {
  // no static shared memory in this kernel: the dynamic window starts 1024-byte aligned (checked)
  extern __shared__ __align__(1024) unsigned char smem[];
  if ((smem_u32(smem) & 1023u) != 0u) __trap();
  Bars &S = *reinterpret_cast<Bars *>(smem + STAGES * STAGE_BYTES);
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  const int g = lane >> 2, q = lane & 3;
  const long long tile = cg_row_tile();
  if (tile * 128 >= M) return;                // before any barrier: the whole CTA leaves
  const int n0 = blockIdx.x * 128, m0 = (int)tile * 128;
  const int nkb = K >> 6;
  const uint32_t smem_s = smem_u32(smem);
  const unsigned char *src = wimg + (size_t)blockIdx.x * nkb * STAGE_BYTES;   // this column tile's K-blocks
  if (tid == 0) {
    for (int s = 0; s < STAGES; s++) {
      mbar_init(smem_u32(&S.full[s]), 1);
      mbar_init(smem_u32(&S.empty[s]), LT / 32);
    }
    mbar_init_fence();
    for (int kb = 0; kb < nkb && kb < STAGES; kb++) {
      mbar_expect_tx(smem_u32(&S.full[kb]), STAGE_BYTES);
      bulk_g2s(smem_s + (uint32_t)kb * STAGE_BYTES, src + (size_t)kb * STAGE_BYTES, STAGE_BYTES, smem_u32(&S.full[kb]));
    }
  }
  __syncthreads();
  // this thread's rows of the A fragments: m0 + 16 * warp + g and + 8
  const int ma = m0 + 16 * warp + g, mb = ma + 8;
  const bool la = ma < M, lb = mb < M;
  const float *xa = X + (size_t)(la ? ma : 0) * K + 2 * q, *xb = X + (size_t)(lb ? mb : 0) * K + 2 * q;
  auto ld2 = [&](const float *p, bool live) {
    if (!live) return make_float2(0.f, 0.f);
    float2 v = *reinterpret_cast<const float2 *>(p);
    if (x_is_keys) v = make_float2(cg_key2f(__float_as_uint(v.x)), cg_key2f(__float_as_uint(v.y)));
    return v;
  };
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; i++) acc[i] = 0.f;
  for (int kb = 0; kb < nkb; kb++) {
    const int s = kb % STAGES;
    // A fragments of the 4 k-steps of this K-block, straight from the fp32 rows (split into bf16 hi / lo)
    uint32_t ah[4][4], al[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ks++) {
      const int k = kb * 64 + ks * 16;
      const float2 v0 = ld2(xa + k, la), v1 = ld2(xb + k, lb), v2 = ld2(xa + k + 8, la), v3 = ld2(xb + k + 8, lb);
      split_bf16x2(v0.x, v0.y, ah[ks][0], al[ks][0]);
      split_bf16x2(v1.x, v1.y, ah[ks][1], al[ks][1]);
      split_bf16x2(v2.x, v2.y, ah[ks][2], al[ks][2]);
      split_bf16x2(v3.x, v3.y, ah[ks][3], al[ks][3]);
    }
    mbar_wait(smem_u32(&S.full[s]), ((uint32_t)(kb / STAGES)) & 1u);
    const uint32_t b_s = smem_s + (uint32_t)s * STAGE_BYTES;
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ks++) {
      const uint64_t bh = wg_desc(b_s + 32u * ks), bl = wg_desc(b_s + PIECE + 32u * ks);
      wg_m64n128<false>(acc, al[ks], bh, 1u);
      wg_m64n128<false>(acc, ah[ks], bl, 1u);
      wg_m64n128<false>(acc, ah[ks], bh, 1u);
    }
    wg_commit();
    wg_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&S.empty[s]));
    if (tid == 0 && kb + STAGES < nkb) {   // refill the stage once all eight warps have read it
      mbar_wait(smem_u32(&S.empty[s]), ((uint32_t)(kb / STAGES)) & 1u);
      mbar_expect_tx(smem_u32(&S.full[s]), STAGE_BYTES);
      bulk_g2s(b_s, src + (size_t)(kb + STAGES) * STAGE_BYTES, STAGE_BYTES, smem_u32(&S.full[s]));
    }
  }
  // ---------------- epilogue: D[row][col] -> + bias, ReLU -> Y ----------------
#pragma unroll
  for (int r = 0; r < 2; r++) {
    const int m = r ? mb : ma;
    if (!(r ? lb : la)) continue;
    const float *brow = bias ? (bias + (size_t)(bias_row_div > 0 ? m / bias_row_div : 0) * N) : nullptr;
#pragma unroll
    for (int i = 0; i < 16; i++)
#pragma unroll
      for (int e = 0; e < 2; e++) {
        const int n = n0 + 8 * i + 2 * q + e;
        if (n < N) {
          float o = acc[4 * i + 2 * r + e] + (brow ? brow[n] : 0.f);
          if (relu) o = fmaxf(o, 0.f);
          Y[(size_t)m * N + n] = o;
        }
      }
  }
}

unsigned short bf16_rne(float f) {
  uint32_t x;
  memcpy(&x, &f, 4);
  const uint32_t lsb = (x >> 16) & 1u;
  x += 0x7fffu + lsb;
  return (unsigned short)(x >> 16);
}
float bf16_to_f(unsigned short h) {
  uint32_t x = (uint32_t)h << 16;
  float f;
  memcpy(&f, &x, 4);
  return f;
}

}  // namespace

void cg_pack_bf16x2_block(const float *Wt, int C, int c0, int rows, int k0, unsigned char *hi, unsigned char *lo) {
  for (int r = 0; r < rows; r++)
    for (int kk = 0; kk < 64; kk++) {
      const float w = Wt[(size_t)(k0 + kk) * C + c0 + r];
      const unsigned short h = bf16_rne(w), l = bf16_rne(w - bf16_to_f(h));
      const size_t off = row_chunk_off(r, kk >> 3) + (size_t)(kk & 7) * 2;
      memcpy(hi + off, &h, 2);
      memcpy(lo + off, &l, 2);
    }
}

// image layout: [column tile (128 outputs)][K-block][hi 16 KB | lo 16 KB], rows past N are zero
int cg_linear_tc_image(cg_ctx *ctx, const float *Wt_host, int K, int N, const void **img) {
  *img = nullptr;
  if (K % 64 != 0 || N < 64) return CG_OK;
  const int ntile = (N + 127) / 128, nkb = K / 64;
  const size_t bytes = (size_t)ntile * nkb * 2 * PIECE;
  std::vector<unsigned char> h(bytes, 0);
  for (int t = 0; t < ntile; t++)
    for (int kb = 0; kb < nkb; kb++) {
      unsigned char *hi = h.data() + ((size_t)t * nkb + kb) * 2 * PIECE;
      cg_pack_bf16x2_block(Wt_host, N, 128 * t, std::min(128, N - 128 * t), 64 * kb, hi, hi + PIECE);
    }
  CG_CUDA(ctx, cudaFuncSetAttribute(linear_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LSMEM));
  void *d = nullptr;
  CG_CUDA(ctx, cudaMalloc(&d, bytes));
  *img = d;
  CG_CUDA(ctx, cudaMemcpyAsync(d, h.data(), bytes, cudaMemcpyHostToDevice, ctx->stream));
  CG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // h goes out of scope
  return CG_OK;
}

int cg_linear_tc_launch(cg_ctx *ctx, const float *X, int M, int K, const void *img, const float *bias, int N, int relu,
                        int bias_row_div, int x_is_keys, float *Y) {
  const dim3 grid = cg_row_tile_grid((N + 127) / 128, ((long long)M + 127) / 128);
  linear_tc_kernel<<<grid, LT, LSMEM, ctx->stream>>>(X, M, K, static_cast<const unsigned char *>(img), bias, N, relu,
                                                     bias_row_div, x_is_keys, Y);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

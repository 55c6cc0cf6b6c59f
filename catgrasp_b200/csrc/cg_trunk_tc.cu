// cg_trunk_tc.cu -- tensor-core "trunk" kernel (engines 1, 2, 3): the fused per-point shared-MLP chain + max of
// cg_trunk_simt.cu with every layer that is a genuine dense contraction on Hopper's wgmma.
//
//   layer            wgmma (m64nNk16, fp32 accumulators in registers)                          epilogue
//   6 -> 64          fp32 FMA (K = 6 is not a tensor-core shape), computed in the A-fragment layout -> X1
//   64 -> 64 (L1)    D1[pt][ch] = X1[pt][k] (registers) . W1[ch][k] (smem)   bf16 hi/lo x3, N = 64    bias/ReLU -> X2
//   64 -> 128 (L2)   D2[pt][ch] = X2[pt][k] (registers) . W2[ch][k] (smem)   bf16 hi/lo x3, N = 128   bias/ReLU -> X3
//   128 -> 1024 (L3) D3[pt][ch] = X3[pt][k] (registers) . W3[ch][k] (smem ring), 8 chunks of 128   max over points
//
// The accumulator fragment of one layer is the A-operand fragment of the next (cg_tc_ptx.cuh), so the activations of a
// tile never touch shared memory: shared memory holds only the resident W1 / W2 and a ring through which a producer
// warp streams W3 with cp.async.bulk, completion counted on mbarriers.
//
// Precision of L3 (PASSES, the template parameter; L1 / L2 are always near-fp32):
//   3 (engine 1)  W3 and X3 split x = hi + lo in bf16, products lo*hi + hi*lo + hi*hi (lo*lo ~ 2^-16 dropped): near-fp32
//   2 (engine 2)  W3 one fp16 term, X3 fp16 hi + lo
//   1 (engine 3)  W3 and X3 one fp16 term each.
// On both fp16 engines X3 values above the fp16 range are clamped to 65504 AND reported through
// cg_trunk_args::ovf_flag so that the host can re-run on engine 1.
//
// Persistent grid: one CTA per SM.  The B x ntiles tiles are numbered candidate-major and CTA i runs the contiguous
// range [i T / G, (i + 1) T / G), so ranges differ by at most one tile and may start or end inside a candidate (the
// global max is an atomicMax on order-preserving keys, so a candidate split over CTAs needs nothing else).
//
// CTA = 384 threads: two consumer warpgroups (points 0-63 / 64-127 of each 128-point tile; each runs the whole layer
// chain for its points), one producer warp and three helper warps.  The two consumer warpgroups are independent except
// for the shared W3 ring, so one warpgroup's FMA layer, epilogues and max reduction overlap the other's tensor-core
// work; warpgroup 1 starts one front (input + FMA + L1 + L2) behind warpgroup 0 so that their fronts do not coincide.
// The helpers keep per-candidate work off the consumers' path: the next candidate's pose inverse, T3 and T64 operand
// image, and the global fold (bias, ReLU, atomicMax) of each finished candidate's running max.
#include <limits.h>
#include <stdlib.h>

#include <algorithm>

#include "cg_tc_ptx.cuh"
#include "cg_trunk_common.cuh"

namespace {
using namespace cg_trunk;
using namespace cg_ptx;

constexpr int NCW = 8;                      // consumer warps (two warpgroups)
constexpr int PROD_WARP = NCW;              // warp 8: W1 / W2 / W3 producer
constexpr int HELP_WARP = NCW + 1;          // warps 9-11: per-candidate helpers
constexpr int NHELP = 3 * 32;
constexpr int NTC = (NCW + 4) * 32;         // 384 threads
constexpr int NCHUNK = 8;                   // 1024 output channels / 128
constexpr uint32_t PIECE = 16384;           // [128 rows x 64 x 16-bit] one swizzled K-block
// shared-memory map
constexpr uint32_t W1_OFF = 0;              // [hi 8 KB | lo 8 KB]: shared W1, or the current candidate's T64 operand
constexpr uint32_t W2_OFF = PIECE;          // [hi 16 KB | lo 16 KB]
constexpr uint32_t RING_OFF = 3 * PIECE;    // 128 KB of W3 slots (one slot = one 64-wide K-block of a 128-channel chunk)
constexpr uint32_t RING_BYTES = 8 * PIECE;
constexpr uint32_t SACC_OFF = RING_OFF + RING_BYTES;   // running max: float2 per (warpgroup, half-chunk, warp, lane)
constexpr uint32_t SACC_BYTES = 2 * 2 * NCHUNK * 4 * 32 * 8;
constexpr uint32_t KEYS_OFF = SACC_OFF + SACC_BYTES;   // per-candidate max keys [2][1024], by candidate parity
constexpr uint32_t KEYS_BYTES = 2 * 1024 * 4;
constexpr uint32_t MISC_OFF = KEYS_OFF + KEYS_BYTES;
constexpr int NSLOT_MAX = 8;
// operand image built by cg_tc_prepare
constexpr uint32_t IMG_W3B = NCHUNK * 2 * 2 * PIECE;   // bf16: [chunk][kb][hi 16 KB | lo 16 KB]
constexpr uint32_t IMG_W2 = 2 * PIECE, IMG_W1 = PIECE;
constexpr uint32_t IMG_W2_OFF = IMG_W3B, IMG_W1_OFF = IMG_W3B + IMG_W2;
constexpr uint32_t IMG_W3H_OFF = IMG_W1_OFF + IMG_W1;  // fp16: [chunk][kb] 16 KB
constexpr uint32_t IMG_W3H = NCHUNK * 2 * PIECE;

struct Misc {
  float w0[6 * 64];
  float bias0[64];
  float bias1[64];
  float bias2[128];
  double pinv[12];
  double mean[6];
  double sden[6];
  float T3[12];
  unsigned long long full_bar[NSLOT_MAX];    // producer -> consumers: W3 slot landed
  unsigned long long empty_bar[NSLOT_MAX];   // consumers -> producer: every consumer warp is done reading the slot
  unsigned long long w_bar;                  // resident W1 / W2 landed
  // Per-candidate hand-offs; k counts the candidates of the CTA's range.  pinv, T3 and the T64 image exist once: the
  // helpers rewrite them for candidate k + 1 between the consumers' last front of candidate k and their first of k + 1.
  unsigned long long cand_bar;               // helpers -> consumers: pinv / T3 / T64 image of candidate k written
  unsigned long long front_bar;              // consumers -> helpers: every consumer is past the last front of k
  unsigned long long keys_bar[2];            // consumers -> helpers: candidate k's max is in keys[k & 1]
};

constexpr size_t SMEM_BYTES = MISC_OFF + sizeof(Misc);
static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB per-CTA shared memory of sm_90");

// One step of the transposing column-max butterfly of the L3 reduction: the lanes with bit STEP set keep the upper
// half of their STEP columns, the others the lower half, and each takes the max with its partner's copy.  STEP is a
// template parameter so that every index into x is a constant and x stays in registers.
template <int STEP>
__device__ __forceinline__ void max_butterfly_step(float *x, int lane) {
  const bool up = (lane & STEP) != 0;
#pragma unroll
  for (int k = 0; k < STEP / 2; k++) {
    const float send = up ? x[k] : x[k + STEP / 2];
    const float keep = up ? x[k + STEP / 2] : x[k];
    x[k] = fmaxf(keep, __shfl_xor_sync(0xffffffffu, send, STEP));
  }
}

#ifdef CG_EXPERIMENTS
// Phase timeline (developer builds, CG_TRUNK_TIMELINE=1): every consumer warp of TL_CTAS sampled CTAs (spread over
// the grid) sums clock64() cycles per phase over its tiles and writes one record of TL_REC words: the TL_NPHASE
// sums, its tile count and its total cycles.  TL_L3_WAIT and TL_RING lie inside TL_L3.
enum { TL_START, TL_INPUT, TL_FRONT, TL_L3, TL_L3_WAIT, TL_RING, TL_NPHASE };
constexpr int TL_CTAS = 8, TL_REC = 8;
__host__ __device__ constexpr int TL_STRIDE(int B) { return B >= TL_CTAS ? B / TL_CTAS : 1; }
#define TL_PARAM , unsigned long long *tl
#define TL_ARG(p) , p
#else
#define TL_PARAM
#define TL_ARG(p)
#endif

template <int PASSES>
__global__ void __launch_bounds__(NTC, 1) trunk_tc_kernel(const cg_trunk_args a TL_PARAM) {
  constexpr int NSLOT = PASSES == 3 ? 4 : 8;
  constexpr uint32_t SLOT_BYTES = PASSES == 3 ? 2 * PIECE : PIECE;
  constexpr bool F16 = PASSES < 3;
  // the operand tiles need 1024-byte alignment (SWIZZLE_128B atoms); the kernel has no static shared memory
  extern __shared__ __align__(1024) unsigned char smem[];
  if ((smem_u32(smem) & 1023u) != 0u) __trap();
  Misc &S = *reinterpret_cast<Misc *>(smem + MISC_OFF);
  float2 *sacc = reinterpret_cast<float2 *>(smem + SACC_OFF);
  uint32_t *keys = reinterpret_cast<uint32_t *>(smem + KEYS_OFF);
  // warp index through a shuffle: the compiler then knows it is warp-uniform and the role branches are not divergent
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  const int N = a.N;
  const int ntiles = (N + TP - 1) / TP;
  // this CTA's tiles [t_begin, t_begin + my_tiles) of the candidate-major numbering t = b * ntiles + j; the launch
  // makes gridDim.x <= B * ntiles, so every range holds at least one tile
  const long long T = (long long)a.B * ntiles;
  const int t_begin = (int)(blockIdx.x * T / gridDim.x);
  const int my_tiles = (int)((blockIdx.x + 1) * T / gridDim.x) - t_begin;
  const int b_first = t_begin / ntiles;
  const int ncand = (t_begin + my_tiles - 1) / ntiles - b_first + 1;
  const unsigned char *img = static_cast<const unsigned char *>(a.tc_img);
  const bool has_l1 = a.stage1_mode != 0;
  const uint32_t smem_s = smem_u32(smem);
  const uint32_t w1_s = smem_s + W1_OFF, w2_s = smem_s + W2_OFF, ring_s = smem_s + RING_OFF;
  const uint32_t misc_s = smem_s + MISC_OFF;
  const uint32_t full_s = misc_s + (uint32_t)offsetof(Misc, full_bar), empty_s = misc_s + (uint32_t)offsetof(Misc, empty_bar);
  const uint32_t wbar_s = misc_s + (uint32_t)offsetof(Misc, w_bar);
  const uint32_t cand_s = misc_s + (uint32_t)offsetof(Misc, cand_bar), front_s = misc_s + (uint32_t)offsetof(Misc, front_bar);
  const uint32_t keys_s = misc_s + (uint32_t)offsetof(Misc, keys_bar);

  // ---- one-time setup --------------------------------------------------------------------------------------
  for (int i = tid; i < 6 * 64; i += NTC) S.w0[i] = a.l0.Wt[i];
  if (tid < 64) {
    S.bias0[tid] = a.l0.b[tid];
    S.bias1[tid] = (a.stage1_mode == 1) ? a.l1.b[tid] : 0.f;
  }
  if (tid < 128) S.bias2[tid] = a.l2.b[tid];
  if (a.in.x_direct == nullptr && tid < 6) {
    S.mean[tid] = a.in.mean ? a.in.mean[tid] : 0.0;
    S.sden[tid] = a.in.stdv ? 1.0 / (a.in.stdv[tid] + 1e-15) : 1.0;   // reciprocal: the hot loop multiplies
  }
  for (int i = tid; i < (int)(SACC_BYTES / 8); i += NTC) sacc[i] = make_float2(-INFINITY, -INFINITY);
  for (int i = tid; i < 2 * 1024; i += NTC) keys[i] = 0u;   // below the key of every float
  if (tid == 0) {
    for (int i = 0; i < NSLOT; i++) {
      mbar_init(full_s + 8u * i, 1);
      mbar_init(empty_s + 8u * i, NCW);
    }
    mbar_init(wbar_s, 1);
    mbar_init(cand_s, NHELP);
    mbar_init(front_s, NCW * 32);
    mbar_init(keys_s, NCW * 32);
    mbar_init(keys_s + 8u, NCW * 32);
    mbar_init_fence();
  }
  __syncthreads();

  if (warp == PROD_WARP) {
    // ======================= producer: resident W2 (+ shared W1), then W3 slot by slot =======================
    // one W3 stream over the whole range: the ring does not drain at candidate boundaries
    if (lane == 0) {
      mbar_expect_tx(wbar_s, IMG_W2 + (a.stage1_mode == 1 ? IMG_W1 : 0u));
      bulk_g2s(w2_s, img + IMG_W2_OFF, IMG_W2, wbar_s);
      if (a.stage1_mode == 1) bulk_g2s(w1_s, img + IMG_W1_OFF, IMG_W1, wbar_s);
      const unsigned char *w3src = img + (PASSES == 3 ? 0u : IMG_W3H_OFF);
      const int total = my_tiles * NCHUNK * 2;
      for (int gs = 0; gs < total; gs++) {
        const int s = gs % NSLOT;
        mbar_wait(empty_s + 8u * s, (((uint32_t)(gs / NSLOT)) & 1u) ^ 1u);   // the first round passes immediately
        mbar_expect_tx(full_s + 8u * s, SLOT_BYTES);
        bulk_g2s(ring_s + (uint32_t)s * SLOT_BYTES, w3src + (size_t)(gs % (NCHUNK * 2)) * SLOT_BYTES, SLOT_BYTES,
                 full_s + 8u * s);
      }
    }
    return;
  }

  if (warp >= HELP_WARP) {
    // ======================= helpers: per-candidate constants and the global fold =======================
    // Candidate k's inputs are loaded (and T64 converted) before waiting for the consumers to leave candidate k - 1,
    // so that only the shared-memory stores sit between the consumers' last front of k - 1 and their first of k.
    // The fold of candidate k - 1 follows the hand-over of k; the consumers cannot fill keys[(k - 1) & 1] again
    // before the hand-over of k + 1, which comes after that fold.
    const int ht = tid - HELP_WARP * 32;
    for (int k = 0; k <= ncand; k++) {
      if (k < ncand) {
        const int b = b_first + k;
        // T64 as the B operand of L1:  B[j][kk] = T64[kk][j]  (pointnet2.py:257).  Unit u = (row j, 8-wide K chunk
        // kc) is one 16-byte chunk of the hi and of the lo image; a warp's 32 rows read 32 consecutive floats.
        constexpr int TU = (64 * 8 + NHELP - 1) / NHELP;
        uint32_t t64h[TU][4], t64l[TU][4];
        if (a.stage1_mode == 2) {
          const float *Tb = a.T64 + (size_t)b * 4096;
#pragma unroll
          for (int i = 0; i < TU; i++) {
            const int u = ht + NHELP * i;
            if (u < 512) {
              float v[8];
#pragma unroll
              for (int e = 0; e < 8; e++) v[e] = __ldg(Tb + (8 * (u >> 6) + e) * 64 + (u & 63));
#pragma unroll
              for (int e = 0; e < 4; e++) split_bf16x2(v[2 * e], v[2 * e + 1], t64h[i][e], t64l[i][e]);
            }
          }
        }
        double pinv[12];
        const bool do_pinv = a.in.x_direct == nullptr && ht == 0;
        if (do_pinv) pose_inverse(a.in.poses + (size_t)b * 16, pinv);
        const float t3 = (a.T3 && ht < 9) ? a.T3[b * 9 + ht] : 0.f;
        if (k > 0) mbar_wait(front_s, (uint32_t)(k - 1) & 1u);
        if (a.stage1_mode == 2) {
#pragma unroll
          for (int i = 0; i < TU; i++) {
            const int u = ht + NHELP * i;
            if (u < 512) {
              const uint32_t off = row_chunk_off(u & 63, u >> 6);
              *reinterpret_cast<uint4 *>(smem + W1_OFF + off) =
                  make_uint4(t64h[i][0], t64h[i][1], t64h[i][2], t64h[i][3]);
              *reinterpret_cast<uint4 *>(smem + W1_OFF + 8192 + off) =
                  make_uint4(t64l[i][0], t64l[i][1], t64l[i][2], t64l[i][3]);
            }
          }
          fence_proxy_async();
        }
        if (do_pinv) {
#pragma unroll
          for (int i = 0; i < 12; i++) S.pinv[i] = pinv[i];
        }
        if (ht < 9) S.T3[ht] = t3;
        mbar_arrive(cand_s);
      }
      if (k > 0) {
        // candidate k - 1: bias and ReLU commute with the max (both are monotone), so they follow it
        const int kp = k - 1;
        mbar_wait(keys_s + 8u * (kp & 1), ((uint32_t)kp >> 1) & 1u);
        uint32_t *kb = keys + (kp & 1) * 1024;
        uint32_t *g = a.gmax_keys + (size_t)(b_first + kp) * 1024;
        for (int ch = ht; ch < 1024; ch += NHELP) {
          float m = cg_key2f(kb[ch]) + __ldg(&a.l3.b[ch]);
          if (a.relu3) m = fmaxf(m, 0.f);
          atomicMax(&g[ch], cg_f2key(m));
          kb[ch] = 0u;
        }
      }
    }
    return;
  }

  // ======================= consumer warpgroups =======================
  const int wg = warp >> 2, w4 = warp & 3, g = lane >> 2, q = lane & 3;
  float vmax = 0.f;   // largest 128->1024 input seen by this thread (post-ReLU, fp16 engines): reported if beyond the fp16 range
#ifdef CG_EXPERIMENTS
  // phase timeline of the sampled CTAs (scripts/trunk_timeline.py): cycles per phase summed over this warp's tiles
  const bool tl_on = tl != nullptr && blockIdx.x % TL_STRIDE(gridDim.x) == 0 &&
                     (int)(blockIdx.x / TL_STRIDE(gridDim.x)) < TL_CTAS;
  unsigned long long tl_sum[TL_NPHASE] = {}, tl_t0 = clock64(), tl_t = tl_t0, tl_s;
#define TL_MARK(phase)                   \
  do {                                   \
    const unsigned long long _t = clock64(); \
    tl_sum[phase] += _t - tl_t;          \
    tl_t = _t;                           \
  } while (0)
#define TL_SPAN_BEGIN() (tl_s = clock64())
#define TL_SPAN_END(phase) (tl_sum[phase] += clock64() - tl_s)
#else
#define TL_MARK(phase) ((void)0)
#define TL_SPAN_BEGIN() ((void)0)
#define TL_SPAN_END(phase) ((void)0)
#endif
  mbar_wait(wbar_s, 0u);

  // The input of a point row is fetched one tile ahead (fetch_id / fetch_row during the previous tile's L3) and
  // finished (finish_row) when its tile starts, so the dependent id -> cloud-row loads are off the critical path.
  // Row n >= N of candidate b duplicates a valid point of b: it cannot change a max.  x_direct rows travel as exact
  // float -> double.
  auto fetch_id = [&](int b, int n) -> int {
    if (n >= N) n = N - 1;
    return (a.in.x_direct == nullptr && a.in.ids) ? __ldg(a.in.ids + (size_t)b * N + n) : n;
  };
  auto fetch_row = [&](int b, int id, double *r) {
    if (a.in.x_direct) {
      const float *xr = a.in.x_direct + ((size_t)b * N + id) * 6;
#pragma unroll
      for (int k = 0; k < 6; k++) r[k] = __ldg(xr + k);
    } else {
      const double *px = a.in.cloud_xyz + (size_t)id * 3;
      const double *pn = a.in.cloud_nrm + (size_t)id * 3;
#pragma unroll
      for (int k = 0; k < 3; k++) {
        r[k] = __ldg(px + k);
        r[3 + k] = __ldg(pn + k);
      }
    }
  };
  // input row (6 floats after pose transform / normalisation / T3)
  auto finish_row = [&](const double *r, float *v) {
    if (a.in.x_direct) {
#pragma unroll
      for (int k = 0; k < 6; k++) v[k] = (float)r[k];
    } else {
      const double x = r[0], y = r[1], z = r[2];
      const double nx = r[3], ny = r[4], nz = r[5];
      const double *R = S.pinv;
      double w[6];
      w[0] = R[0] * x + R[1] * y + R[2] * z + R[9];
      w[1] = R[3] * x + R[4] * y + R[5] * z + R[10];
      w[2] = R[6] * x + R[7] * y + R[8] * z + R[11];
      w[3] = R[0] * nx + R[1] * ny + R[2] * nz;
      w[4] = R[3] * nx + R[4] * ny + R[5] * nz;
      w[5] = R[6] * nx + R[7] * ny + R[8] * nz;
#pragma unroll
      for (int k = 0; k < 6; k++) v[k] = (float)((w[k] - S.mean[k]) * S.sden[k]);
    }
    if (a.T3) {  // xyz @ T3 (pointnet2.py:248), normals pass through (:245-250)
      const float x = v[0], y = v[1], z = v[2];
      v[0] = fmaf(z, S.T3[6], fmaf(y, S.T3[3], x * S.T3[0]));
      v[1] = fmaf(z, S.T3[7], fmaf(y, S.T3[4], x * S.T3[1]));
      v[2] = fmaf(z, S.T3[8], fmaf(y, S.T3[5], x * S.T3[2]));
    }
  };

  // W3 ring slot and mbarrier phase of K-block kb of chunk c of the current tile
  uint32_t gslot = 0;   // W3 slots consumed before the current tile
  auto slot_of = [&](int c, int kb) { return (gslot + 2u * c + kb) % NSLOT; };
  auto phase_of = [&](int c, int kb) { return ((gslot + 2u * c + kb) / NSLOT) & 1u; };

  const int prow = wg * 64 + w4 * 16 + g;   // this thread's rows of a tile: prow and prow + 8
  // Half-chunks per unrolled L3 group (below), and whether the whole input rows of the next tile are prefetched during
  // L3 or only their ids: the 24 registers of two float64 rows fit beside the L3 pipeline of engine 3 only.
  constexpr int L3_GROUP = PASSES == 1 ? 8 : 4;
  constexpr bool ROW_PREFETCH = PASSES == 1;
  double r0[6], r1[6];   // raw input rows of the next tile
  int id0, id1;
  {
    const int j = t_begin - b_first * ntiles;
    id0 = fetch_id(b_first, j * TP + prow);
    id1 = fetch_id(b_first, j * TP + prow + 8);
    if (ROW_PREFETCH) {
      fetch_row(b_first, id0, r0);
      fetch_row(b_first, id1, r1);
    }
  }
  // Warpgroup 1 starts its first tile when warpgroup 0 has finished the front layers of its own (named barrier 2), so
  // that one warpgroup's front runs under the other's L3 instead of leaving the tensor pipe idle for both.
  if (wg == 1) asm volatile("bar.sync 2, 256;" ::: "memory");
  TL_MARK(TL_START);
  for (int it = 0; it < my_tiles; it++) {
    // tile j of candidate b, candidate ci of the range; the candidate's first / last tile in this range
    const int b = (t_begin + it) / ntiles, j = t_begin + it - b * ntiles, ci = b - b_first;
    const bool cand_first = it == 0 || j == 0, cand_last = it + 1 == my_tiles || j + 1 == ntiles;
    const int p0 = j * TP + prow;   // this thread's rows: points p0 and p0 + 8
    if (cand_first) mbar_wait(cand_s, (uint32_t)ci & 1u);   // pinv / T3 / T64 image of candidate b
    // ---- 6 -> 64 (+bias, ReLU) straight into the D-fragment layout of a 64-column tile ----
    float d64[32];
    {
      float v0[6], v1[6];
      if (!ROW_PREFETCH) {
        fetch_row(b, id0, r0);
        fetch_row(b, id1, r1);
      }
      finish_row(r0, v0);
      finish_row(r1, v1);
      TL_MARK(TL_INPUT);
#pragma unroll
      for (int m = 0; m < 8; m++)
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int c = 8 * m + 2 * q + e;
          float o0 = S.bias0[c], o1 = o0;
#pragma unroll
          for (int k = 0; k < 6; k++) {
            const float w = S.w0[k * 64 + c];
            o0 = fmaf(v0[k], w, o0);
            o1 = fmaf(v1[k], w, o1);
          }
          d64[4 * m + e] = fmaxf(o0, 0.f);
          d64[4 * m + 2 + e] = fmaxf(o1, 0.f);
        }
    }
    uint32_t xh[8][4], xl[8][4];   // A fragments of the current layer input (up to K = 128), bf16 / fp16 hi + lo
    // ---- L1: 64 -> 64 (STNkd shared conv, or the per-candidate T64 feature transform) ----
    if (has_l1) {
      d_to_a<4, false>(d64, xh, xl);
      wg_fence_regs<16>(xh[0]);
      wg_fence_regs<16>(xl[0]);
      wg_fence_regs<32>(d64);
      wg_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ks++) {
        const uint64_t bh = wg_desc(w1_s + 32u * ks), bl = wg_desc(w1_s + 8192u + 32u * ks);
        wg_m64n64<false>(d64, xl[ks], bh, ks > 0 ? 1u : 0u);
        wg_m64n64<false>(d64, xh[ks], bl, 1u);
        wg_m64n64<false>(d64, xh[ks], bh, 1u);
      }
      wg_commit();
      wg_wait<0>();
      wg_fence_regs<32>(d64);
      wg_fence_regs<16>(xh[0]);
      wg_fence_regs<16>(xl[0]);
#pragma unroll
      for (int i = 0; i < 32; i++) {
        if (a.stage1_mode == 1) d64[i] = fmaxf(d64[i] + S.bias1[8 * (i >> 2) + 2 * q + (i & 1)], 0.f);
      }
      if (a.pf_out) {   // PointNetSeg point feature (pointnet2.py:261)
#pragma unroll
        for (int r = 0; r < 2; r++) {
          const int n = p0 + 8 * r;
          if (n < N) {
            float *dst = a.pf_out + ((size_t)b * N + n) * 64 + 2 * q;
#pragma unroll
            for (int m = 0; m < 8; m++)
              *reinterpret_cast<float2 *>(dst + 8 * m) = make_float2(d64[4 * m + 2 * r], d64[4 * m + 2 * r + 1]);
          }
        }
      }
    }
    // the last read of candidate b's pinv / T3 / T64 image in this range is done: the helpers may replace them
    if (cand_last) mbar_arrive(front_s);
    // ---- L2: 64 -> 128 ----
    float acc[64];
    d_to_a<4, false>(d64, xh, xl);
    wg_fence_regs<16>(xh[0]);
    wg_fence_regs<16>(xl[0]);
    wg_fence_regs<64>(acc);
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ks++) {
      const uint64_t bh = wg_desc(w2_s + 32u * ks), bl = wg_desc(w2_s + PIECE + 32u * ks);
      wg_m64n128<false>(acc, xl[ks], bh, ks > 0 ? 1u : 0u);
      wg_m64n128<false>(acc, xh[ks], bl, 1u);
      wg_m64n128<false>(acc, xh[ks], bh, 1u);
    }
    wg_commit();
    wg_wait<0>();
    wg_fence_regs<64>(acc);
    wg_fence_regs<16>(xh[0]);
    wg_fence_regs<16>(xl[0]);
    // warpgroup 0's front of the first tile is done: release warpgroup 1 (see above)
    if (it == 0 && wg == 0) asm volatile("bar.arrive 2, 256;" ::: "memory");
    TL_MARK(TL_FRONT);
#pragma unroll
    for (int i = 0; i < 64; i++) acc[i] = fmaxf(acc[i] + S.bias2[8 * (i >> 2) + 2 * q + (i & 1)], 0.f);
    if (PASSES == 1) {
#pragma unroll
      for (int j = 0; j < 8; j++)
#pragma unroll
        for (int r = 0; r < 4; r++) {
          const float x0 = acc[8 * j + 2 * r], x1 = acc[8 * j + 2 * r + 1];
          vmax = fmaxf(vmax, fmaxf(x0, x1));
          // values beyond the fp16 range saturate to 65504 instead of becoming inf (x0 -> low half)
          asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(xh[j][r]) : "f"(x1), "f"(x0));
        }
    } else {
      if (PASSES == 2) {   // split_f16x2 clamps to the fp16 range: record what it clamps
#pragma unroll
        for (int i = 0; i < 64; i++) vmax = fmaxf(vmax, acc[i]);
      }
      d_to_a<8, F16>(acc, xh, xl);
    }
    wg_fence_regs<32>(xh[0]);
    if (PASSES != 1) wg_fence_regs<32>(xl[0]);
    // ---- L3: 128 -> 1024 in 16 half-chunks of 64 channels; max over the tile's points ----
    // Two 32-register accumulators: half-chunk h + 1 is issued before half-chunk h is reduced, so the reduction
    // overlaps the tensor cores.  Half-chunk h = channels 64h .. 64h+63 = rows 64 (h & 1) .. of chunk h / 2's W3 slots.
    // The 16 half-chunks are unrolled so that both accumulators are fixed registers: with operand fences around every
    // issue and wait ptxas then keeps exactly one wgmma group in flight during each reduction.
    auto issue = [&](int h, float *d) {
      const int c = h >> 1;
      if ((h & 1) == 0) {
        TL_SPAN_BEGIN();
        mbar_wait(full_s + 8u * slot_of(c, 0), phase_of(c, 0));
        mbar_wait(full_s + 8u * slot_of(c, 1), phase_of(c, 1));
        TL_SPAN_END(TL_RING);
      }
      wg_fence_regs<32>(d);
      wg_fence();
#pragma unroll
      for (int kb = 0; kb < 2; kb++) {
        const uint32_t ws = ring_s + slot_of(c, kb) * SLOT_BYTES + (uint32_t)(h & 1) * (PIECE / 2);
#pragma unroll
        for (int ks = 0; ks < 4; ks++) {
          const int j = kb * 4 + ks;
          const uint32_t first = (kb | ks) ? 1u : 0u;
          const uint64_t bw = wg_desc(ws + 32u * ks);
          if (PASSES == 3) {
            const uint64_t bl = wg_desc(ws + PIECE + 32u * ks);
            wg_m64n64<false>(d, xl[j], bw, first);   // x_lo * w_hi
            wg_m64n64<false>(d, xh[j], bl, 1u);      // x_hi * w_lo
            wg_m64n64<false>(d, xh[j], bw, 1u);      // x_hi * w_hi
          } else if (PASSES == 2) {
            wg_m64n64<true>(d, xl[j], bw, first);
            wg_m64n64<true>(d, xh[j], bw, 1u);
          } else {
            wg_m64n64<true>(d, xh[j], bw, first);
          }
        }
      }
      wg_commit();
      wg_fence_regs<32>(d);
    };
    // half-chunk h is complete in this warp: fold its column max into the running max; after the second half of a
    // chunk hand the chunk's two W3 slots back
    auto reduce = [&](int h, const float *d) {
      const int c = h >> 1;
      if (h & 1) {
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(empty_s + 8u * slot_of(c, 0));
          mbar_arrive(empty_s + 8u * slot_of(c, 1));
        }
      }
      // column max over this warp's 16 rows: own two rows, then a transposing butterfly over lane bits 4, 3, 2
      // (each step halves the columns a thread is responsible for).  Afterwards thread (g, q) holds the columns
      // 8g + 2q + {0, 1} of the half-chunk.
      float x[16];
#pragma unroll
      for (int i = 0; i < 8; i++) {
        x[2 * i] = fmaxf(d[4 * i], d[4 * i + 2]);
        x[2 * i + 1] = fmaxf(d[4 * i + 1], d[4 * i + 3]);
      }
      max_butterfly_step<16>(x, lane);
      max_butterfly_step<8>(x, lane);
      max_butterfly_step<4>(x, lane);
      float2 &slot = sacc[((wg * 2 * NCHUNK + h) * 4 + w4) * 32 + lane];   // private to this thread
      const float2 old = slot;
      slot = make_float2(fmaxf(old.x, x[0]), fmaxf(old.y, x[1]));
    };
    // The half-chunks run in groups of L3_GROUP, unrolled so that the two accumulators are fixed registers.  Inside a
    // group one wgmma group is in flight during each reduction; a group ends with a full wait, so that no wgmma is in
    // flight across the loop's back edge (ptxas would otherwise serialise the loop).  A fully unrolled L3 does not fit
    // the 168-register budget of a 288-thread CTA (registers are allocated per
    // warpgroup: 288 threads count as 384).
    // The next tile's input is fetched where nothing is in flight: the ids before the first group, the dependent
    // rows before the second (a last tile re-reads its own rows, clamped to the candidate's points).
    const int nt = t_begin + it + (it + 1 < my_tiles ? 1 : 0);
    const int nb = nt / ntiles, pn = (nt - nb * ntiles) * TP + prow;
    id0 = fetch_id(nb, pn);
    id1 = fetch_id(nb, pn + 8);
#pragma unroll 1
    for (int h0 = 0; h0 < 2 * NCHUNK; h0 += L3_GROUP) {
      if (ROW_PREFETCH && h0 == L3_GROUP) {
        fetch_row(nb, id0, r0);
        fetch_row(nb, id1, r1);
      }
      float acc3[2][32];   // even / odd half-chunks
      issue(h0, acc3[0]);
#pragma unroll
      for (int j = 0; j < L3_GROUP; j++) {
        if (j + 1 < L3_GROUP) issue(h0 + j + 1, acc3[(j + 1) & 1]);
        TL_SPAN_BEGIN();
        if (j + 1 < L3_GROUP) wg_wait<1>();
        else wg_wait<0>();
        TL_SPAN_END(TL_L3_WAIT);
        wg_fence_regs<32>(acc3[j & 1]);
        reduce(h0 + j, acc3[j & 1]);
      }
    }
    // the last wgmma that read the A fragments is complete: the next tile's front may overwrite them
    wg_fence_regs<32>(xh[0]);
    if (PASSES != 1) wg_fence_regs<32>(xl[0]);
    gslot += 2u * NCHUNK;
    if (cand_last) {
      // hand candidate b's running max to the helpers (keys by candidate parity) and start the next one at -inf
      uint32_t *kk = keys + (ci & 1) * 1024;
#pragma unroll 4
      for (int h = 0; h < 2 * NCHUNK; h++) {
        float2 &slot = sacc[((wg * 2 * NCHUNK + h) * 4 + w4) * 32 + lane];
        const float2 v = slot;
        atomicMax(&kk[64 * h + 2 * lane], cg_f2key(v.x));   // thread (g, q) holds columns 8g + 2q + {0, 1}
        atomicMax(&kk[64 * h + 2 * lane + 1], cg_f2key(v.y));
        slot = make_float2(-INFINITY, -INFINITY);
      }
      mbar_arrive(keys_s + 8u * (ci & 1));
    }
    TL_MARK(TL_L3);
  }
  if (F16 && vmax > 65504.f && a.ovf_flag) atomicOr(a.ovf_flag, 1u);
#ifdef CG_EXPERIMENTS
  if (tl_on && lane == 0) {
    unsigned long long *o = tl + ((size_t)(blockIdx.x / TL_STRIDE(gridDim.x)) * NCW + warp) * TL_REC;
#pragma unroll
    for (int p = 0; p < TL_NPHASE; p++) o[p] = tl_sum[p];
    o[TL_NPHASE] = (unsigned long long)my_tiles;
    o[TL_NPHASE + 1] = clock64() - tl_t0;
  }
#endif
#undef TL_MARK
#undef TL_SPAN_BEGIN
#undef TL_SPAN_END
}

}  // namespace

size_t cg_tc_image_bytes() { return (size_t)IMG_W3H_OFF + IMG_W3H; }

int cg_tc_prepare(cg_ctx *ctx, const float *Wt3, const float *Wt2, const float *Wt1, void *dst_dev, int *f16_ok) {
  CG_CUDA(ctx, cudaFuncSetAttribute(trunk_tc_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
  CG_CUDA(ctx, cudaFuncSetAttribute(trunk_tc_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
  CG_CUDA(ctx, cudaFuncSetAttribute(trunk_tc_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
  float wmax = 0.f;
  for (size_t i = 0; i < (size_t)128 * 1024; i++) wmax = fmaxf(wmax, fabsf(Wt3[i]));
  *f16_ok = (wmax < 65504.f) ? 1 : 0;   // otherwise the fp16 image would hold infinities
  std::vector<unsigned char> img(cg_tc_image_bytes(), 0);
  for (int ch = 0; ch < NCHUNK; ch++)
    for (int kb = 0; kb < 2; kb++) {
      unsigned char *hi = img.data() + (size_t)(ch * 2 + kb) * 2 * PIECE;
      cg_pack_bf16x2_block(Wt3, 1024, ch * 128, 128, kb * 64, hi, hi + PIECE);
    }
  cg_pack_bf16x2_block(Wt2, 128, 0, 128, 0, img.data() + IMG_W2_OFF, img.data() + IMG_W2_OFF + PIECE);
  if (Wt1) cg_pack_bf16x2_block(Wt1, 64, 0, 64, 0, img.data() + IMG_W1_OFF, img.data() + IMG_W1_OFF + 8192);
  // fp16 single-term W3 for the fp16 engines: [chunk][kb] 16 KB
  for (int ch = 0; ch < NCHUNK; ch++)
    for (int r = 0; r < 128; r++)
      for (int k = 0; k < 128; k++) {
        const __half h = __float2half_rn(Wt3[(size_t)k * 1024 + ch * 128 + r]);
        unsigned short bits;
        memcpy(&bits, &h, 2);
        const size_t off = (size_t)IMG_W3H_OFF + (size_t)(ch * 2 + (k >> 6)) * PIECE + row_chunk_off(r, (k & 63) >> 3) +
                           (size_t)(k & 7) * 2;
        memcpy(img.data() + off, &bits, 2);
      }
  CG_CUDA(ctx, cudaMemcpyAsync(dst_dev, img.data(), img.size(), cudaMemcpyHostToDevice, ctx->stream));
  CG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // img goes out of scope
  return CG_OK;
}

int cg_trunk_launch_tc(cg_ctx *ctx, const cg_trunk_args &a) {
  CG_REQUIRE(ctx, a.B > 0 && a.N > 0, "trunk: B,N must be positive");
  CG_REQUIRE(ctx, a.tc_img != nullptr, "trunk: tensor-core weight image missing");
  // persistent: one CTA per SM (or per tile, if there are fewer tiles), each over a balanced range of tiles
  const long long tiles = (long long)a.B * ((a.N + TP - 1) / TP);
  CG_REQUIRE(ctx, tiles <= INT_MAX, "trunk: too many tiles in one launch");
  const int grid = (int)std::min<long long>(ctx->num_sms, tiles);
  // W3 beyond the fp16 range: the fp16 engines fall back to the 3-pass bf16 kernel
  const int passes = !a.tc_f16_ok || ctx->engine == 1 ? 3 : (ctx->engine == 2 ? 2 : 1);
#ifdef CG_EXPERIMENTS
  static const bool timeline = getenv("CG_TRUNK_TIMELINE") && atoi(getenv("CG_TRUNK_TIMELINE")) != 0;
  unsigned long long *tl = nullptr;
  const size_t tl_words = (size_t)TL_CTAS * NCW * TL_REC;
  if (timeline) {
    CG_CUDA(ctx, cudaMallocAsync(&tl, tl_words * 8, ctx->stream));
    CG_CUDA(ctx, cudaMemsetAsync(tl, 0, tl_words * 8, ctx->stream));
  }
#endif
  if (passes == 3) trunk_tc_kernel<3><<<grid, NTC, SMEM_BYTES, ctx->stream>>>(a TL_ARG(tl));
  else if (passes == 2) trunk_tc_kernel<2><<<grid, NTC, SMEM_BYTES, ctx->stream>>>(a TL_ARG(tl));
  else trunk_tc_kernel<1><<<grid, NTC, SMEM_BYTES, ctx->stream>>>(a TL_ARG(tl));
  CG_LAUNCH_CHECK(ctx);
#ifdef CG_EXPERIMENTS
  if (timeline) {
    std::vector<unsigned long long> h(tl_words);
    CG_CUDA(ctx, cudaMemcpyAsync(h.data(), tl, tl_words * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CG_CUDA(ctx, cudaFreeAsync(tl, ctx->stream));
    CG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    // cycles per tile of one warp, averaged over the consumer warps of the sampled CTAs; the warps of a CTA run
    // concurrently, so "total" is also the CTA's cycles per tile
    double sum[TL_NPHASE + 1] = {}, tiles = 0;
    int recs = 0;
    for (int r = 0; r < TL_CTAS * NCW; r++) {
      const unsigned long long *o = &h[(size_t)r * TL_REC];
      if (o[TL_NPHASE] == 0) continue;
      for (int p = 0; p < TL_NPHASE; p++) sum[p] += (double)o[p];
      sum[TL_NPHASE] += (double)o[TL_NPHASE + 1];
      tiles += (double)o[TL_NPHASE];
      recs++;
    }
    if (recs > 0) {
      // tensor-pipe cycles of one 128-point tile at 2048 dense fp16 / bf16 MAC per clock per SM
      const double l3 = 128.0 * 128 * 1024 / 2048 * passes, l12 = 128.0 * 64 * (128 + (a.stage1_mode ? 64 : 0)) * 3 / 2048;
      const double tot = sum[TL_NPHASE] / tiles;
      fprintf(stderr,
              "[trunk-timeline] passes=%d B=%d N=%d stage1=%d tiles/CTA=%.0f warps=%d  clk/tile: start %.0f  input %.0f  "
              "front %.0f  l3 %.0f (wgmma-wait %.0f, ring-wait %.0f)  total %.0f  | tensor work %.0f clk/tile -> "
              "busy %.1f%%\n",
              passes, a.B, a.N, a.stage1_mode, tiles / recs, recs, sum[TL_START] / tiles, sum[TL_INPUT] / tiles,
              sum[TL_FRONT] / tiles, sum[TL_L3] / tiles, sum[TL_L3_WAIT] / tiles, sum[TL_RING] / tiles, tot, l3 + l12,
              100.0 * (l3 + l12) / tot);
    }
  }
#endif
  return CG_OK;
}

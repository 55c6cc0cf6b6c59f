// cg_trunk_tc.cu -- tensor-core "trunk" kernel (engines 1, 2, 3): the fused per-point shared-MLP chain + max of
// cg_trunk_simt.cu with every layer that is a genuine dense contraction on Hopper's wgmma.
//
//   layer            wgmma (m64nNk16, fp32 accumulators in registers)                          epilogue
//   6 -> 64          fp32 FMA (K = 6 is not a tensor-core shape), computed in the A-fragment layout -> X1
//   64 -> 64 (L1)    D1[pt][ch] = X1[pt][k] (registers) . W1[ch][k] (smem)   bf16 hi/lo x3, N = 64    bias/ReLU -> X2
//   64 -> 128 (L2)   D2[pt][ch] = X2[pt][k] (registers) . W2[ch][k] (smem)   bf16 hi/lo x3, N = 128   bias/ReLU -> X3 smem
//   128 -> 1024 (L3) D3[ch][pt] = W3[ch][k] (smem ring) . X3[pt][k] (smem), 8 chunks of 128 channels  max over points
//
// The front (FMA, L1, L2) runs point-major: the accumulator fragment of one layer is the A-operand fragment of the
// next (cg_tc_ptx.cuh), so X1 and X2 stay in registers.  Only X3 is staged, once per tile: L2's epilogue stores it into
// a [points x 128] K-major swizzled image that is the B operand of L3.  L3 runs channel-major with W3 as the A operand,
// straight from the ring through which a producer warp streams W3 with cp.async.bulk (completion counted on
// mbarriers), so one W3 fetch serves every point of the tile, and a channel's max over points is a row reduction
// inside the accumulator fragment.
//
// Precision of L3 (PASSES, the template parameter; L1 / L2 are always near-fp32):
//   3 (engine 1)  W3 and X3 split x = hi + lo in bf16, products hi*lo + lo*hi + hi*hi (lo*lo ~ 2^-16 dropped): near-fp32
//   2 (engine 2)  W3 one fp16 term, X3 fp16 hi + lo
//   1 (engine 3)  W3 and X3 one fp16 term each.
// On both fp16 engines X3 values above the fp16 range are clamped to 65504 AND reported through
// cg_trunk_args::ovf_flag so that the host can re-run on engine 1.
//
// Tiles: 256 points on engine 3 (the fp16 X3 image is 64 KB), 128 points on engines 1 and 2 (hi + lo images, 64 KB).
// Persistent grid: one CTA per SM.  The B x ntiles tiles are numbered candidate-major and CTA i runs the contiguous
// range [i T / G, (i + 1) T / G), so ranges differ by at most one tile and may start or end inside a candidate (the
// global max is an atomicMax on order-preserving keys, so a candidate split over CTAs needs nothing else).
//
// CTA = 384 threads: two consumer warpgroups, one producer warp and three helper warps.  Warpgroup w builds the front
// of the tile's points [w TILE / 2, (w + 1) TILE / 2) in 64-row blocks, and in L3 computes the channels 64w .. 64w+63
// of every 128-channel chunk over all the tile's points.  The helpers keep the input rows and per-candidate work off
// the consumers' path: one tile ahead they gather the tile's cloud rows and apply the float64 pose transform,
// normalisation and T3 into the shared input tile X0 [TILE][6], which the consumers read at the start of the tile's
// 6 -> 64 layer; they also write each candidate's T64 operand image and do the global fold (bias, ReLU, atomicMax) of
// each finished candidate's max.
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
// points per tile: engine 3 stages one fp16 X3 term, engines 1 and 2 a hi and a lo term in the same 64 KB
__host__ __device__ constexpr int tile_points(int passes) { return passes == 1 ? 256 : 128; }
// shared-memory map
constexpr uint32_t W1_OFF = 0;              // [hi 8 KB | lo 8 KB]: shared W1, or the current candidate's T64 operand
constexpr uint32_t W2_OFF = PIECE;          // [hi 16 KB | lo 16 KB]
constexpr uint32_t X3_OFF = 3 * PIECE;      // 64 KB X3 image: [kb][TILE rows x 64] (engine 3), [hi | lo][kb][128 x 64]
constexpr uint32_t X3_BYTES = 4 * PIECE;
constexpr uint32_t RING_OFF = X3_OFF + X3_BYTES;   // 96 KB of W3 slots (one slot = one 64-wide K-block of a chunk)
constexpr uint32_t RING_BYTES = 6 * PIECE;
constexpr uint32_t KEYS_OFF = RING_OFF + RING_BYTES;   // per-candidate max keys [2][1024], by candidate parity
constexpr uint32_t KEYS_BYTES = 2 * 1024 * 4;
constexpr uint32_t MISC_OFF = KEYS_OFF + KEYS_BYTES;
constexpr int NSLOT_MAX = 6;
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
  double mean[6];                            // input normalisation: (w - mean) * sden
  double sden[6];
  unsigned long long full_bar[NSLOT_MAX];   // producer -> consumers: W3 slot landed
  unsigned long long empty_bar[NSLOT_MAX];   // consumers -> producer: every consumer warp is done reading the slot
  unsigned long long w_bar;                  // resident W1 / W2 landed
  // X0 exists once: the helpers write the rows of tile t + 1 once every consumer has read those of tile t.
  unsigned long long x0_full;                // helpers -> consumers: X0 holds the current tile's rows
  unsigned long long x0_empty;               // consumers -> helpers: every consumer is past the tile's last X0 read
  // Per-candidate hand-offs; k counts the candidates of the CTA's range.  The T64 image exists once: the helpers
  // rewrite it for candidate k + 1 between the consumers' last L1 of candidate k and their first of k + 1.
  unsigned long long cand_bar;               // helpers -> consumers: T64 image of candidate k written
  unsigned long long front_bar;              // consumers -> helpers: every consumer is past the last L1 of k
  unsigned long long keys_bar[2];            // consumers -> helpers: candidate k's max is in keys[k & 1]
};
// the input tile X0: float [TILE][6], the 6 input values of each point; a 24-byte row stride is conflict-free for the
// 8 rows of a fragment
constexpr uint32_t X0_OFF = MISC_OFF + sizeof(Misc);
__host__ __device__ constexpr size_t smem_bytes(int passes) { return X0_OFF + (size_t)tile_points(passes) * 6 * 4; }
static_assert(smem_bytes(1) <= 232448 && smem_bytes(3) <= 232448, "exceeds the 227 KB per-CTA shared memory of sm_90");

#ifdef CG_EXPERIMENTS
// Phase timeline (developer builds, CG_TRUNK_TIMELINE=1): every consumer and helper warp of TL_CTAS sampled CTAs
// (spread over the grid) sums clock64() cycles per phase over its tiles and writes one record of TL_REC words: the
// phase sums, its tile count and its total cycles.  Consumer phases TL_*: TL_L3_WAIT and TL_RING lie inside TL_L3.
// Helper phases TH_*: building X0 (gather, transform, stores), waiting for the consumers to free X0, the T64
// hand-off and the fold.  A CTA's records: its NCW consumer warps, then its 3 helper warps.
enum { TL_START, TL_INPUT, TL_FRONT, TL_X3, TL_L3, TL_L3_WAIT, TL_RING, TL_NPHASE };
enum { TH_BUILD, TH_EMPTY, TH_CAND, TH_FOLD, TH_NPHASE };
constexpr int TL_CTAS = 8, TL_REC = TL_NPHASE + 2, TL_WARPS = NCW + 3;
__host__ __device__ constexpr int TL_STRIDE(int B) { return B >= TL_CTAS ? B / TL_CTAS : 1; }
#define TL_PARAM , unsigned long long *tl
#define TL_ARG(p) , p
#else
#define TL_PARAM
#define TL_ARG(p)
#endif

template <int PASSES>
__global__ void __launch_bounds__(NTC, 1) trunk_tc_kernel(const cg_trunk_args a TL_PARAM) {
  constexpr int TILE = tile_points(PASSES);
  constexpr int NBLK = TILE / 128;            // 64-row front blocks per warpgroup = 128-point L3 units per chunk
  constexpr int NSLOT = PASSES == 3 ? 3 : 6;
  constexpr uint32_t SLOT_BYTES = PASSES == 3 ? 2 * PIECE : PIECE;
  static_assert(NSLOT * SLOT_BYTES == RING_BYTES, "ring");
  constexpr bool F16 = PASSES < 3;
  constexpr uint32_t X3_KB = TILE * 128;      // one [TILE x 64] K-block of the X3 image
  constexpr uint32_t X3_LO = 2 * X3_KB;       // the lo term (engines 1 and 2)
  static_assert((PASSES == 1 ? 2 : 4) * X3_KB == X3_BYTES, "X3 image");
  // the operand tiles need 1024-byte alignment (SWIZZLE_128B atoms); the kernel has no static shared memory
  extern __shared__ __align__(1024) unsigned char smem[];
  if ((smem_u32(smem) & 1023u) != 0u) __trap();
  Misc &S = *reinterpret_cast<Misc *>(smem + MISC_OFF);
  uint32_t *keys = reinterpret_cast<uint32_t *>(smem + KEYS_OFF);
  // warp index through a shuffle: the compiler then knows it is warp-uniform and the role branches are not divergent
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  const int N = a.N;
  const int ntiles = (N + TILE - 1) / TILE;
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
  const uint32_t w1_s = smem_s + W1_OFF, w2_s = smem_s + W2_OFF, x3_s = smem_s + X3_OFF, ring_s = smem_s + RING_OFF;
  const uint32_t misc_s = smem_s + MISC_OFF;
  const uint32_t full_s = misc_s + (uint32_t)offsetof(Misc, full_bar), empty_s = misc_s + (uint32_t)offsetof(Misc, empty_bar);
  const uint32_t wbar_s = misc_s + (uint32_t)offsetof(Misc, w_bar);
  const uint32_t cand_s = misc_s + (uint32_t)offsetof(Misc, cand_bar), front_s = misc_s + (uint32_t)offsetof(Misc, front_bar);
  const uint32_t keys_s = misc_s + (uint32_t)offsetof(Misc, keys_bar);
  const uint32_t x0f_s = misc_s + (uint32_t)offsetof(Misc, x0_full), x0e_s = misc_s + (uint32_t)offsetof(Misc, x0_empty);
  float *x0 = reinterpret_cast<float *>(smem + X0_OFF);
  // the T64 image is the only per-candidate operand the consumers read
  const bool t64_handoff = a.stage1_mode == 2;

  // ---- one-time setup --------------------------------------------------------------------------------------
  for (int i = tid; i < 6 * 64; i += NTC) S.w0[i] = a.l0.Wt[i];
  if (tid < 64) {
    S.bias0[tid] = a.l0.b[tid];
    S.bias1[tid] = (a.stage1_mode == 1) ? a.l1.b[tid] : 0.f;
  }
  if (tid < 128) S.bias2[tid] = a.l2.b[tid];
  if (a.in.x_direct == nullptr && tid < 6) {
    S.mean[tid] = a.in.mean ? a.in.mean[tid] : 0.0;
    S.sden[tid] = a.in.stdv ? 1.0 / (a.in.stdv[tid] + 1e-15) : 1.0;   // reciprocal: every row multiplies
  }
  if (tid == 0) {
    for (int i = 0; i < NSLOT; i++) {
      mbar_init(full_s + 8u * i, 1);
      mbar_init(empty_s + 8u * i, NCW);
    }
    mbar_init(wbar_s, 1);
    mbar_init(x0f_s, NHELP);
    mbar_init(x0e_s, NCW * 32);
    mbar_init(cand_s, NHELP);
    mbar_init(front_s, NCW * 32);
    mbar_init(keys_s, NCW * 32);
    mbar_init(keys_s + 8u, NCW * 32);
    mbar_init_fence();
  }
  __syncthreads();

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
  // record of this warp (record index rec) over its `tiles` tiles
#define TL_WRITE(rec, tiles)                                                                              \
  do {                                                                                                    \
    if (tl_on && lane == 0) {                                                                             \
      unsigned long long *o = tl + ((size_t)(blockIdx.x / TL_STRIDE(gridDim.x)) * TL_WARPS + (rec)) * TL_REC; \
      for (int p = 0; p < TL_NPHASE; p++) o[p] = tl_sum[p];                                               \
      o[TL_NPHASE] = (unsigned long long)(tiles);                                                         \
      o[TL_NPHASE + 1] = clock64() - tl_t0;                                                               \
    }                                                                                                     \
  } while (0)
#else
#define TL_MARK(phase) ((void)0)
#define TL_SPAN_BEGIN() ((void)0)
#define TL_SPAN_END(phase) ((void)0)
#define TL_WRITE(rec, tiles) ((void)0)
#endif

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
    // ======================= helpers: the input tile X0, the T64 image and the global fold =======================
    // The helpers walk the CTA's tiles one ahead of the consumers.  For tile t they load and transform the rows into
    // registers, wait until every consumer has read X0 of tile t - 1 (in tile t - 1's 6 -> 64 layer) and only then
    // store; tile t - 1's L1, L2 and L3 cover the loads.  Row n >= N of candidate b duplicates a valid point of b: it
    // cannot change a max.  At the first tile of candidate k the T64 image comes first, in the same way: loaded and
    // converted, then stored once every consumer is past the last L1 of k - 1 (just after their last X0 read of k - 1).
    // The fold of k - 1 comes after X0 of k's first tile, so a fold never delays an X0; the consumers cannot fill
    // keys[(k - 1) & 1] again before X0 of k + 1's first tile, which comes after that fold.
    const int ht = tid - HELP_WARP * 32;
    constexpr int XR = (TILE + NHELP - 1) / NHELP;   // X0 rows of this thread: ht + NHELP i < TILE
    const bool xd = a.in.x_direct != nullptr;
    // the candidate's pose inverse and T3 (mean and sden are the call's, in shared memory)
    double pinv[12];
    float t3[9] = {};
    // x_direct rows travel as exact float -> double
    auto fetch_id = [&](int b, int n) -> int {
      if (n >= N) n = N - 1;
      return (!xd && a.in.ids) ? __ldg(a.in.ids + (size_t)b * N + n) : n;
    };
    auto fetch_row = [&](int b, int id, double *r) {
      if (xd) {
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
      if (xd) {
#pragma unroll
        for (int k = 0; k < 6; k++) v[k] = (float)r[k];
      } else {
        const double x = r[0], y = r[1], z = r[2];
        const double nx = r[3], ny = r[4], nz = r[5];
        const double *R = pinv;
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
        v[0] = fmaf(z, t3[6], fmaf(y, t3[3], x * t3[0]));
        v[1] = fmaf(z, t3[7], fmaf(y, t3[4], x * t3[1]));
        v[2] = fmaf(z, t3[8], fmaf(y, t3[5], x * t3[2]));
      }
    };
    // candidate kp of the range: bias and ReLU commute with the max (both are monotone), so they follow it.  Every
    // one of the 1024 keys was stored by its channel's owner before the consumers arrived on keys_bar.
    auto fold = [&](int kp) {
      mbar_wait(keys_s + 8u * (kp & 1), ((uint32_t)kp >> 1) & 1u);
      const uint32_t *kb = keys + (kp & 1) * 1024;
      uint32_t *g = a.gmax_keys + (size_t)(b_first + kp) * 1024;
      for (int ch = ht; ch < 1024; ch += NHELP) {
        float m = cg_key2f(kb[ch]) + __ldg(&a.l3.b[ch]);
        if (a.relu3) m = fmaxf(m, 0.f);
        atomicMax(&g[ch], cg_f2key(m));
      }
    };
    // the ids of this thread's rows of a tile are loaded one iteration ahead, so that a tile's build waits only for the
    // dependent cloud rows
    int ids[XR];
    auto load_ids = [&](int t) {
      const int b = t / ntiles, j = t - b * ntiles;
#pragma unroll
      for (int i = 0; i < XR; i++)
        if (ht + NHELP * i < TILE) ids[i] = fetch_id(b, j * TILE + ht + NHELP * i);
    };
    load_ids(t_begin);
#pragma unroll 1
    for (int it = 0; it < my_tiles; it++) {
      const int b = (t_begin + it) / ntiles, j = t_begin + it - b * ntiles, ci = b - b_first;
      const bool cand_first = it == 0 || j == 0;
      // the T64 image comes before the candidate's pinv / T3, so that those are not live beside it
      if (cand_first && t64_handoff) {
        // T64 as the B operand of L1:  B[j][kk] = T64[kk][j]  (pointnet2.py:257).  Unit u = (row j, 8-wide K chunk
        // kc) is one 16-byte chunk of the hi and of the lo image; a warp's 32 rows read 32 consecutive floats.
        constexpr int TU = (64 * 8 + NHELP - 1) / NHELP;
        uint32_t t64h[TU][4], t64l[TU][4];
        const float *Tb = a.T64 + (size_t)b * 4096;
#pragma unroll
        for (int i = 0; i < TU; i++) {
          const int u = ht + NHELP * i;
          if (u < 512) {
            float tv[8];
#pragma unroll
            for (int e = 0; e < 8; e++) tv[e] = __ldg(Tb + (8 * (u >> 6) + e) * 64 + (u & 63));
#pragma unroll
            for (int e = 0; e < 4; e++) split_bf16x2(tv[2 * e], tv[2 * e + 1], t64h[i][e], t64l[i][e]);
          }
        }
        if (ci > 0) mbar_wait(front_s, (uint32_t)(ci - 1) & 1u);
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
        mbar_arrive(cand_s);
        TL_MARK(TH_CAND);
      }
      if (cand_first) {
        if (!xd) pose_inverse(a.in.poses + (size_t)b * 16, pinv);
        if (a.T3) {
#pragma unroll
          for (int e = 0; e < 9; e++) t3[e] = a.T3[b * 9 + e];
        }
      }
      // ---- X0 of tile it ----
      float v[XR][6];
      {
        double r[XR][6];
#pragma unroll
        for (int i = 0; i < XR; i++)
          if (ht + NHELP * i < TILE) fetch_row(b, ids[i], r[i]);
#pragma unroll
        for (int i = 0; i < XR; i++)
          if (ht + NHELP * i < TILE) finish_row(r[i], v[i]);
      }
      TL_MARK(TH_BUILD);
      if (it > 0) mbar_wait(x0e_s, (uint32_t)(it - 1) & 1u);
      TL_MARK(TH_EMPTY);
#pragma unroll
      for (int i = 0; i < XR; i++)
        if (ht + NHELP * i < TILE) {
          float2 *dst = reinterpret_cast<float2 *>(x0 + (ht + NHELP * i) * 6);
          dst[0] = make_float2(v[i][0], v[i][1]);
          dst[1] = make_float2(v[i][2], v[i][3]);
          dst[2] = make_float2(v[i][4], v[i][5]);
        }
      mbar_arrive(x0f_s);
      if (it + 1 < my_tiles) load_ids(t_begin + it + 1);
      TL_MARK(TH_BUILD);
      if (cand_first && ci > 0) {
        fold(ci - 1);
        TL_MARK(TH_FOLD);
      }
    }
    fold(ncand - 1);
    TL_MARK(TH_FOLD);
    TL_WRITE(NCW + warp - HELP_WARP, my_tiles);
    return;
  }

  // ======================= consumer warpgroups =======================
  const int wg = warp >> 2, w4 = warp & 3, g = lane >> 2, q = lane & 3;
  float vmax = 0.f;   // largest 128->1024 input seen by this thread (post-ReLU, fp16 engines): reported if beyond the fp16 range
  mbar_wait(wbar_s, 0u);

  // W3 ring slot and mbarrier phase of K-block kb of chunk c of the current tile
  uint32_t gslot = 0;   // W3 slots consumed before the current tile
  auto slot_of = [&](int c, int kb) { return (gslot + 2u * c + kb) % NSLOT; };
  auto phase_of = [&](int c, int kb) { return ((gslot + 2u * c + kb) / NSLOT) & 1u; };

  // this thread's front rows of a tile: prow(blk) and prow(blk) + 8 of each 64-row block blk
  auto prow = [&](int blk) { return wg * (TILE / 2) + blk * 64 + w4 * 16 + g; };
  TL_MARK(TL_START);
  for (int it = 0; it < my_tiles; it++) {
    // tile j of candidate b, candidate ci of the range; the candidate's first / last tile in this range
    const int b = (t_begin + it) / ntiles, j = t_begin + it - b * ntiles, ci = b - b_first;
    const bool cand_first = it == 0 || j == 0, cand_last = it + 1 == my_tiles || j + 1 == ntiles;
    if (cand_first && t64_handoff) mbar_wait(cand_s, (uint32_t)ci & 1u);   // T64 image of candidate b
    mbar_wait(x0f_s, (uint32_t)it & 1u);   // X0 holds this tile's input rows
#pragma unroll 1
    for (int blk = 0; blk < NBLK; blk++) {
      const int p0 = j * TILE + prow(blk);   // this thread's rows: points p0 and p0 + 8
      // ---- 6 -> 64 (+bias, ReLU) straight into the D-fragment layout of a 64-column tile ----
      float d64[32];
      {
        float v0[6], v1[6];
        const float2 *x0r = reinterpret_cast<const float2 *>(x0 + prow(blk) * 6);
#pragma unroll
        for (int k = 0; k < 3; k++) {
          const float2 u0 = x0r[k], u1 = x0r[24 + k];   // rows prow and prow + 8
          v0[2 * k] = u0.x;
          v0[2 * k + 1] = u0.y;
          v1[2 * k] = u1.x;
          v1[2 * k + 1] = u1.y;
        }
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
      // this thread's last X0 read of the tile is done: the helpers may store the next tile's rows
      if (blk == NBLK - 1) mbar_arrive(x0e_s);
      uint32_t xh[4][4], xl[4][4];   // A fragments of the layer input (K = 64), bf16 hi + lo
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
      // the last read of candidate b's T64 image in this range is done: the helpers may replace it
      if (t64_handoff && cand_last && blk == NBLK - 1) mbar_arrive(front_s);
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
#pragma unroll
      for (int i = 0; i < 64; i++) acc[i] = fmaxf(acc[i] + S.bias2[8 * (i >> 2) + 2 * q + (i & 1)], 0.f);
      TL_MARK(TL_FRONT);
      // Both warpgroups' L3 wgmma of the previous tile are complete (each waited for its own before getting here):
      // the X3 image may be overwritten.  The first block's front ran under the other warpgroup's L3.
      if (blk == 0) asm volatile("bar.sync 1, 256;" ::: "memory");
      // ---- X3 -> the [TILE x 128] K-major image: accumulator pair i (channels 8i + 2q, +1) of row g (+ 8) is one
      // 32-bit word of 16-byte chunk i & 7 of K-block i >> 3 (conflict-free: the 8 rows of a step hit 8 chunks) ----
#pragma unroll
      for (int r = 0; r < 2; r++) {
        const int pr = prow(blk) + 8 * r;
#pragma unroll
        for (int i = 0; i < 16; i++) {
          const float x0 = acc[4 * i + 2 * r], x1 = acc[4 * i + 2 * r + 1];
          const uint32_t off = X3_OFF + (uint32_t)(i >> 3) * X3_KB + row_chunk_off(pr, i & 7) + 4u * q;
          uint32_t h, l;
          if (PASSES == 1) {
            vmax = fmaxf(vmax, fmaxf(x0, x1));
            // values beyond the fp16 range saturate to 65504 instead of becoming inf (x0 -> low half)
            asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h) : "f"(x1), "f"(x0));
          } else if (PASSES == 2) {   // split_f16x2 clamps to the fp16 range: record what it clamps
            vmax = fmaxf(vmax, fmaxf(x0, x1));
            split_f16x2(x0, x1, h, l);
          } else {
            split_bf16x2(x0, x1, h, l);
          }
          *reinterpret_cast<uint32_t *>(smem + off) = h;
          if (PASSES != 1) *reinterpret_cast<uint32_t *>(smem + off + X3_LO) = l;
        }
      }
    }
    // X3 is complete once every consumer thread has stored its part: make it visible to the wgmma (async) proxy
    fence_proxy_async();
    asm volatile("bar.sync 1, 256;" ::: "memory");
    TL_MARK(TL_X3);
    // ---- L3: 128 -> 1024, channel-major: D[ch][pt] = W3 (ring slot rows 64 wg ..) . X3^T ----
    // 8 * NBLK units; unit u = 128-point block u % NBLK of chunk u / NBLK, one m64n128 accumulator of 64 registers.
    // Two accumulators: unit u + 1 is issued before unit u is reduced, so the reduction overlaps the tensor cores.
    // The units of a group are unrolled so that both accumulators are fixed registers; with operand fences around
    // every issue and wait ptxas keeps exactly one wgmma group in flight during each reduction.
    // The units run in unrolled groups that end with a full wait, so that no wgmma is in flight across the loop's
    // back edge (ptxas would otherwise serialise the loop); larger groups do not fit the 168-register budget of a
    // 384-thread CTA.  Issuing the next chunk's unit while a chunk is in flight holds 4 W3 slots: the 6 fp16 slots
    // allow it, the 3 bf16 slots of engine 1 do not, so engine 1 runs unit by unit and relies on the other
    // warpgroup's wgmma to cover its reductions.  Its ring holds only 1.5 chunks, so engine 1 commits each K-block
    // as a group of its own and hands K-block 0's slot back as soon as that group is complete: the producer then
    // fetches the next chunk's second slot under the current chunk's second half.
    constexpr int NU = NCHUNK * NBLK, GROUP = PASSES == 1 ? 8 : (PASSES == 2 ? 4 : 1);
    constexpr bool EARLY_RELEASE = GROUP == 1;
    static_assert(GROUP == 1 || NSLOT >= 4, "a unit issued ahead needs the next chunk's slots as well");
    auto issue = [&](int u, float *d) {
      const int c = u / NBLK, hb = u % NBLK;
      if (hb == 0) {
        TL_SPAN_BEGIN();
        mbar_wait(full_s + 8u * slot_of(c, 0), phase_of(c, 0));
        mbar_wait(full_s + 8u * slot_of(c, 1), phase_of(c, 1));
        TL_SPAN_END(TL_RING);
      }
      wg_fence_regs<64>(d);
      wg_fence();
#pragma unroll
      for (int kb = 0; kb < 2; kb++) {
        const uint32_t ws = ring_s + slot_of(c, kb) * SLOT_BYTES + (uint32_t)wg * (PIECE / 2);
        const uint32_t xs = x3_s + (uint32_t)kb * X3_KB + (uint32_t)hb * PIECE;
#pragma unroll
        for (int ks = 0; ks < 4; ks++) {
          const uint32_t first = (kb | ks) ? 1u : 0u;
          const uint64_t aw = wg_desc(ws + 32u * ks), bx = wg_desc(xs + 32u * ks);
          if (PASSES == 3) {
            const uint64_t al = wg_desc(ws + PIECE + 32u * ks), bxl = wg_desc(xs + X3_LO + 32u * ks);
            wg_ss_m64n128<false>(d, aw, bxl, first);   // w_hi * x_lo
            wg_ss_m64n128<false>(d, al, bx, 1u);       // w_lo * x_hi
            wg_ss_m64n128<false>(d, aw, bx, 1u);       // w_hi * x_hi
          } else if (PASSES == 2) {
            wg_ss_m64n128<true>(d, aw, wg_desc(xs + X3_LO + 32u * ks), first);
            wg_ss_m64n128<true>(d, aw, bx, 1u);
          } else {
            wg_ss_m64n128<true>(d, aw, bx, first);
          }
        }
        if (EARLY_RELEASE && kb == 0) wg_commit();   // K-block 0 as a group of its own (see below)
      }
      wg_commit();
      wg_fence_regs<64>(d);
    };
    // unit u is complete in this warpgroup: the max over its points of each of this thread's rows (channels
    // 128 c + 64 wg + 16 w4 + g + 8 r) is folded over the row's quad, and the q = 0 lane, the channel's only owner in
    // the CTA, keeps the candidate's running max as a key in keys[ci & 1] (stored on the candidate's first unit of
    // the range).  After the chunk's last unit hand its two W3 slots back.
    uint32_t *kk = keys + (ci & 1) * 1024 + wg * 64 + w4 * 16 + g;
    auto reduce = [&](int u, const float *d) {
      const int c = u / NBLK, hb = u % NBLK;
      if (hb == NBLK - 1) {
        __syncwarp();
        if (lane == 0) {
          if (!EARLY_RELEASE) mbar_arrive(empty_s + 8u * slot_of(c, 0));
          mbar_arrive(empty_s + 8u * slot_of(c, 1));
        }
      }
#pragma unroll
      for (int r = 0; r < 2; r++) {
        float m = fmaxf(d[2 * r], d[2 * r + 1]);
#pragma unroll
        for (int i = 1; i < 16; i++) m = fmaxf(m, fmaxf(d[4 * i + 2 * r], d[4 * i + 2 * r + 1]));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
        if (q == 0) {
          const uint32_t key = cg_f2key(m);
          uint32_t &slot = kk[128 * c + 8 * r];
          slot = (cand_first && hb == 0) ? key : max(slot, key);
        }
      }
    };
#pragma unroll 1
    for (int u0 = 0; u0 < NU; u0 += GROUP) {
      float acc3[2][64];   // even / odd units
      issue(u0, acc3[0]);
#pragma unroll
      for (int j = 0; j < GROUP; j++) {
        if (j + 1 < GROUP) issue(u0 + j + 1, acc3[(j + 1) & 1]);
        TL_SPAN_BEGIN();
        if (EARLY_RELEASE) {
          wg_wait<1>();
          __syncwarp();
          if (lane == 0) mbar_arrive(empty_s + 8u * slot_of((u0 + j) / NBLK, 0));
        }
        if (j + 1 < GROUP) wg_wait<1>();
        else wg_wait<0>();
        TL_SPAN_END(TL_L3_WAIT);
        wg_fence_regs<64>(acc3[j & 1]);
        reduce(u0 + j, acc3[j & 1]);
      }
    }
    gslot += 2u * NCHUNK;
    // candidate b's max is complete in keys[ci & 1]: hand it to the helpers
    if (cand_last) mbar_arrive(keys_s + 8u * (ci & 1));
    TL_MARK(TL_L3);
  }
  if (F16 && vmax > 65504.f && a.ovf_flag) atomicOr(a.ovf_flag, 1u);
  TL_WRITE(warp, my_tiles);
#undef TL_MARK
#undef TL_SPAN_BEGIN
#undef TL_SPAN_END
#undef TL_WRITE
}

}  // namespace

size_t cg_tc_image_bytes() { return (size_t)IMG_W3H_OFF + IMG_W3H; }

int cg_tc_prepare(cg_ctx *ctx, const float *Wt3, const float *Wt2, const float *Wt1, void *dst_dev, int *f16_ok) {
  CG_CUDA(ctx, cudaFuncSetAttribute(trunk_tc_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes(3)));
  CG_CUDA(ctx, cudaFuncSetAttribute(trunk_tc_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes(2)));
  CG_CUDA(ctx, cudaFuncSetAttribute(trunk_tc_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes(1)));
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
  // W3 beyond the fp16 range: the fp16 engines fall back to the 3-pass bf16 kernel
  const int passes = !a.tc_f16_ok || ctx->engine == 1 ? 3 : (ctx->engine == 2 ? 2 : 1);
  // persistent: one CTA per SM (or per tile, if there are fewer tiles), each over a balanced range of tiles
  const int tp = tile_points(passes);
  const long long tiles = (long long)a.B * ((a.N + tp - 1) / tp);
  CG_REQUIRE(ctx, tiles <= INT_MAX, "trunk: too many tiles in one launch");
  const int grid = (int)std::min<long long>(ctx->num_sms, tiles);
#ifdef CG_EXPERIMENTS
  static const bool timeline = getenv("CG_TRUNK_TIMELINE") && atoi(getenv("CG_TRUNK_TIMELINE")) != 0;
  unsigned long long *tl = nullptr;
  const size_t tl_words = (size_t)TL_CTAS * TL_WARPS * TL_REC;
  if (timeline) {
    CG_CUDA(ctx, cudaMallocAsync(&tl, tl_words * 8, ctx->stream));
    CG_CUDA(ctx, cudaMemsetAsync(tl, 0, tl_words * 8, ctx->stream));
  }
#endif
  const size_t smem = smem_bytes(passes);
  if (passes == 3) trunk_tc_kernel<3><<<grid, NTC, smem, ctx->stream>>>(a TL_ARG(tl));
  else if (passes == 2) trunk_tc_kernel<2><<<grid, NTC, smem, ctx->stream>>>(a TL_ARG(tl));
  else trunk_tc_kernel<1><<<grid, NTC, smem, ctx->stream>>>(a TL_ARG(tl));
  CG_LAUNCH_CHECK(ctx);
#ifdef CG_EXPERIMENTS
  if (timeline) {
    std::vector<unsigned long long> h(tl_words);
    CG_CUDA(ctx, cudaMemcpyAsync(h.data(), tl, tl_words * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CG_CUDA(ctx, cudaFreeAsync(tl, ctx->stream));
    CG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    // cycles of one warp, averaged over the consumer (helper) warps of the sampled CTAs; the warps of a CTA run
    // concurrently, so "total" is also the CTA's cycles
    double sum[TL_NPHASE + 1] = {}, tiles = 0, hsum[TH_NPHASE + 1] = {}, htiles = 0;
    int recs = 0;
    for (int r = 0; r < TL_CTAS * TL_WARPS; r++) {
      const unsigned long long *o = &h[(size_t)r * TL_REC];
      if (o[TL_NPHASE] == 0) continue;
      if (r % TL_WARPS < NCW) {
        for (int p = 0; p < TL_NPHASE; p++) sum[p] += (double)o[p];
        sum[TL_NPHASE] += (double)o[TL_NPHASE + 1];
        tiles += (double)o[TL_NPHASE];
        recs++;
      } else {
        for (int p = 0; p < TH_NPHASE; p++) hsum[p] += (double)o[p];
        hsum[TH_NPHASE] += (double)o[TL_NPHASE + 1];
        htiles += (double)o[TL_NPHASE];
      }
    }
    if (recs > 0) {
      // per 128 points, so that tiles of 128 and 256 points compare directly; tensor-pipe cycles of 128 points at
      // 2048 dense fp16 / bf16 MAC per clock per SM
      const double p128 = tiles * (tp / 128), h128 = htiles * (tp / 128);
      const double l3 = 128.0 * 128 * 1024 / 2048 * passes, l12 = 128.0 * 64 * (128 + (a.stage1_mode ? 64 : 0)) * 3 / 2048;
      const double tot = sum[TL_NPHASE] / p128;
      fprintf(stderr,
              "[trunk-timeline] passes=%d B=%d N=%d stage1=%d tile=%d tiles/CTA=%.0f warps=%d  clk/128 pts: start %.0f  "
              "input %.0f  front %.0f  x3 %.0f  l3 %.0f (wgmma-wait %.0f, ring-wait %.0f)  total %.0f  | tensor work "
              "%.0f clk/128 pts -> busy %.1f%%  | helpers: x0 build %.0f  x0-empty wait %.0f  t64 %.0f  fold %.0f\n",
              passes, a.B, a.N, a.stage1_mode, tp, tiles / recs, recs, sum[TL_START] / p128, sum[TL_INPUT] / p128,
              sum[TL_FRONT] / p128, sum[TL_X3] / p128, sum[TL_L3] / p128, sum[TL_L3_WAIT] / p128, sum[TL_RING] / p128,
              tot, l3 + l12, 100.0 * (l3 + l12) / tot, hsum[TH_BUILD] / h128, hsum[TH_EMPTY] / h128,
              hsum[TH_CAND] / h128, hsum[TH_FOLD] / h128);
    }
  }
#endif
  return CG_OK;
}

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

// What differs between the engines, by L3's PASSES (3 = engine 1, 2 = engine 2, 1 = engine 3).
template <int P>
struct Engine {
  static constexpr int PASSES = P;
  // points per tile: engine 3 stages one fp16 X3 term, engines 1 and 2 a hi and a lo term in the same 64 KB
  static constexpr int TILE = PASSES == 1 ? 256 : 128;
  static constexpr int NBLK = TILE / 128;   // 64-row front blocks per warpgroup = 128-point L3 units per chunk
  static constexpr int NSLOT = PASSES == 3 ? 3 : 6;
  static constexpr uint32_t SLOT_BYTES = PASSES == 3 ? 2 * PIECE : PIECE;
  static_assert(NSLOT * SLOT_BYTES == RING_BYTES, "ring");
  static constexpr bool F16 = PASSES < 3;
  static constexpr uint32_t X3_KB = TILE * 128;   // one [TILE x 64] K-block of the X3 image
  static constexpr uint32_t X3_LO = 2 * X3_KB;    // the lo term (engines 1 and 2)
  static_assert((PASSES == 1 ? 2 : 4) * X3_KB == X3_BYTES, "X3 image");
  // L3 units issued per unrolled group, and whether K-block 0's slot goes back before its chunk is done (see l3)
  static constexpr int GROUP = PASSES == 1 ? 8 : (PASSES == 2 ? 4 : 1);
  static constexpr bool EARLY_RELEASE = GROUP == 1;
  static_assert(GROUP == 1 || NSLOT >= 4, "a unit issued ahead needs the next chunk's slots as well");
  static constexpr uint32_t W3_SRC = PASSES == 3 ? 0u : IMG_W3H_OFF;   // the W3 image this engine streams
  static constexpr size_t SMEM = X0_OFF + (size_t)TILE * 6 * 4;        // dynamic shared memory of a CTA
};
static_assert(Engine<1>::SMEM <= 232448 && Engine<3>::SMEM <= 232448, "exceeds the 227 KB per-CTA shared memory of sm_90");

// The CTA's tiles [t_begin, t_begin + my_tiles) of the candidate-major numbering t = b * ntiles + j; the launch makes
// gridDim.x <= B * ntiles, so every range holds at least one tile.  ncand candidates from b_first meet the range.
struct Range {
  int ntiles, t_begin, my_tiles, b_first, ncand;
  struct Tile {
    int b, j, ci;                  // tile j of candidate b, candidate ci of the range
    bool cand_first, cand_last;    // the candidate's first / last tile in this range
  };
  __device__ Range(int B, int N, int tile) {
    ntiles = (N + tile - 1) / tile;
    const long long T = (long long)B * ntiles;
    t_begin = (int)(blockIdx.x * T / gridDim.x);
    my_tiles = (int)((blockIdx.x + 1) * T / gridDim.x) - t_begin;
    b_first = t_begin / ntiles;
    ncand = (t_begin + my_tiles - 1) / ntiles - b_first + 1;
  }
  // tile it of the range
  __device__ Tile tile(int it) const {
    const int b = (t_begin + it) / ntiles, j = t_begin + it - b * ntiles;
    return {b, j, b - b_first, it == 0 || j == 0, it + 1 == my_tiles || j + 1 == ntiles};
  }
};

// The CTA's mbarriers (shared addresses of the Misc fields of the same names).  Each completes one phase per use, so
// the wait for use k (k = 0, 1, ...) is a wait for phase parity k & 1.  x0_full / x0_empty are used once per tile,
// cand_bar / front_bar once per candidate of the range, keys_bar[p] by the candidates of parity p, full / empty[s] by
// the W3 K-blocks that pass through slot s.
struct Barriers {
  uint32_t full_bar, empty_bar, w_bar, x0_full, x0_empty, cand_bar, front_bar, keys_bar;
  __device__ explicit Barriers(uint32_t misc_s)
      : full_bar(misc_s + (uint32_t)offsetof(Misc, full_bar)),
        empty_bar(misc_s + (uint32_t)offsetof(Misc, empty_bar)),
        w_bar(misc_s + (uint32_t)offsetof(Misc, w_bar)),
        x0_full(misc_s + (uint32_t)offsetof(Misc, x0_full)),
        x0_empty(misc_s + (uint32_t)offsetof(Misc, x0_empty)),
        cand_bar(misc_s + (uint32_t)offsetof(Misc, cand_bar)),
        front_bar(misc_s + (uint32_t)offsetof(Misc, front_bar)),
        keys_bar(misc_s + (uint32_t)offsetof(Misc, keys_bar)) {}
  // arrival counts: one thread or the helpers on the producer / helper side, a warp or a thread of every consumer
  // warp on the consumer side
  __device__ void init(int nslot) const {
    for (int i = 0; i < nslot; i++) {
      mbar_init(full_bar + 8u * i, 1);
      mbar_init(empty_bar + 8u * i, NCW);
    }
    mbar_init(w_bar, 1);
    mbar_init(x0_full, NHELP);
    mbar_init(x0_empty, NCW * 32);
    mbar_init(cand_bar, NHELP);
    mbar_init(front_bar, NCW * 32);
    mbar_init(keys_bar, NCW * 32);
    mbar_init(keys_bar + 8u, NCW * 32);
    mbar_init_fence();
  }
  __device__ uint32_t full_at(uint32_t s) const { return full_bar + 8u * s; }
  __device__ uint32_t empty_at(uint32_t s) const { return empty_bar + 8u * s; }
  __device__ uint32_t keys_of(int k) const { return keys_bar + 8u * (k & 1); }   // candidate k's: keys_bar[k & 1]
  // candidate k of the range is use k >> 1 of its keys barrier
  __device__ void wait_keys(int k) const { mbar_wait(keys_of(k), ((uint32_t)k >> 1) & 1u); }
};
// wait for use k of a barrier
__device__ __forceinline__ void wait_use(uint32_t bar, uint32_t k) { mbar_wait(bar, k & 1u); }
// wait for use k - 1, the release of a buffer's previous use: the first round, k = 0, passes at once, as a fresh
// mbarrier counts the phase before its first as complete
__device__ __forceinline__ void wait_prev_use(uint32_t bar, uint32_t k) { mbar_wait(bar, (k & 1u) ^ 1u); }


// Phase timeline (developer builds, CG_TRUNK_TIMELINE=1): every consumer and helper warp of TL_CTAS sampled CTAs
// (spread over the grid) sums clock64() cycles per phase over its tiles and writes one record of TL_REC words: the
// phase sums, its tile count and its total cycles.  Consumer phases TL_*: TL_L3_WAIT and TL_RING lie inside TL_L3.
// Helper phases TH_*: building X0 (gather, transform, stores), waiting for the consumers to free X0, the T64
// hand-off and the fold.  A CTA's records: its NCW consumer warps, then its 3 helper warps.  Other builds record
// nothing.
enum { TL_START, TL_INPUT, TL_FRONT, TL_X3, TL_L3, TL_L3_WAIT, TL_RING, TL_NPHASE };
enum { TH_BUILD, TH_EMPTY, TH_CAND, TH_FOLD, TH_NPHASE };
#ifdef CG_EXPERIMENTS
constexpr int TL_CTAS = 8, TL_REC = TL_NPHASE + 2, TL_WARPS = NCW + 3;
__host__ __device__ constexpr int TL_STRIDE(int B) { return B >= TL_CTAS ? B / TL_CTAS : 1; }
struct Timeline {
  unsigned long long *out;
  bool on;   // this CTA is sampled
  unsigned long long sum[TL_NPHASE] = {}, t0, t, s;
  __device__ explicit Timeline(unsigned long long *tl) {
    out = tl;
    on = tl != nullptr && blockIdx.x % TL_STRIDE(gridDim.x) == 0 && (int)(blockIdx.x / TL_STRIDE(gridDim.x)) < TL_CTAS;
    t0 = clock64();
    t = t0;
  }
  // the time since the last mark goes to phase p
  __device__ void mark(int p) {
    const unsigned long long now = clock64();
    sum[p] += now - t;
    t = now;
  }
  // the time from span_begin to span_end goes to phase p, without moving the mark
  __device__ void span_begin() { s = clock64(); }
  __device__ void span_end(int p) { sum[p] += clock64() - s; }
  // record rec of the CTA: this warp's sums over its `tiles` tiles
  __device__ void write(int rec, int tiles) const {
    if (on && (threadIdx.x & 31) == 0) {
      unsigned long long *o = out + ((size_t)(blockIdx.x / TL_STRIDE(gridDim.x)) * TL_WARPS + rec) * TL_REC;
      for (int p = 0; p < TL_NPHASE; p++) o[p] = sum[p];
      o[TL_NPHASE] = (unsigned long long)tiles;
      o[TL_NPHASE + 1] = clock64() - t0;
    }
  }
};
#else
struct Timeline {
  __device__ void mark(int) {}
  __device__ void span_begin() {}
  __device__ void span_end(int) {}
  __device__ void write(int, int) const {}
};
#endif

// ======================= producer: resident W2 (+ shared W1), then W3 slot by slot =======================
// One W3 stream over the whole range: the ring does not drain at candidate boundaries.  The CTA's gs-th W3 K-block
// goes through slot gs % NSLOT as that slot's use gs / NSLOT.
template <class E>
__device__ __forceinline__ void producer(const cg_trunk_args &a, const unsigned char *img, const Range &R,
                                         const Barriers &bar, uint32_t smem_s) {
  mbar_expect_tx(bar.w_bar, IMG_W2 + (a.stage1_mode == 1 ? IMG_W1 : 0u));
  bulk_g2s(smem_s + W2_OFF, img + IMG_W2_OFF, IMG_W2, bar.w_bar);
  if (a.stage1_mode == 1) bulk_g2s(smem_s + W1_OFF, img + IMG_W1_OFF, IMG_W1, bar.w_bar);
  const unsigned char *w3src = img + E::W3_SRC;
  const int total = R.my_tiles * NCHUNK * 2;
  for (int gs = 0; gs < total; gs++) {
    const int s = gs % E::NSLOT;
    wait_prev_use(bar.empty_at(s), (uint32_t)(gs / E::NSLOT));
    mbar_expect_tx(bar.full_at(s), E::SLOT_BYTES);
    bulk_g2s(smem_s + RING_OFF + (uint32_t)s * E::SLOT_BYTES,
             w3src + (size_t)(gs % (NCHUNK * 2)) * E::SLOT_BYTES, E::SLOT_BYTES, bar.full_at(s));
  }
}

// ======================= helpers: the input tile X0, the T64 image and the global fold =======================
template <class E>
__device__ __forceinline__ void helpers(const cg_trunk_args &a, const Range &R, const Barriers &bar,
                                        unsigned char *smem, float *x0, uint32_t *keys, int N, bool t64_handoff,
                                        Timeline &tl, int ht) {
  Misc &S = *reinterpret_cast<Misc *>(smem + MISC_OFF);
  // The helpers walk the CTA's tiles one ahead of the consumers.  For tile t they load and transform the rows into
  // registers, wait until every consumer has read X0 of tile t - 1 (in tile t - 1's 6 -> 64 layer) and only then
  // store; tile t - 1's L1, L2 and L3 cover the loads.  Row n >= N of candidate b duplicates a valid point of b: it
  // cannot change a max.  At the first tile of candidate k the T64 image comes first, in the same way: loaded and
  // converted, then stored once every consumer is past the last L1 of k - 1 (just after their last X0 read of k - 1).
  // The fold of k - 1 comes after X0 of k's first tile, so a fold never delays an X0; the consumers cannot fill
  // keys[(k - 1) & 1] again before X0 of k + 1's first tile, which comes after that fold.
  constexpr int XR = (E::TILE + NHELP - 1) / NHELP;   // X0 rows of this thread: ht + NHELP i < TILE
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
      double w[6];
      pose_transform(pinv, r[0], r[1], r[2], r[3], r[4], r[5], w);
#pragma unroll
      for (int k = 0; k < 6; k++) v[k] = (float)((w[k] - S.mean[k]) * S.sden[k]);
    }
    if (a.T3) apply_t3(t3, v);
  };
  // candidate kp of the range: bias and ReLU commute with the max (both are monotone), so they follow it.  Every
  // one of the 1024 keys was stored by its channel's owner before the consumers arrived on keys_bar.
  auto fold = [&](int kp) {
    bar.wait_keys(kp);
    const uint32_t *kb = keys + (kp & 1) * 1024;
    uint32_t *g = a.gmax_keys + (size_t)(R.b_first + kp) * 1024;
    for (int ch = ht; ch < 1024; ch += NHELP) {
      float m = cg_key2f(kb[ch]) + __ldg(&a.l3.b[ch]);
      if (a.relu3) m = fmaxf(m, 0.f);
      atomicMax(&g[ch], cg_f2key(m));
    }
  };
  // the ids of this thread's rows of tile t (of the candidate-major numbering) are loaded one iteration ahead, so that
  // a tile's build waits only for the dependent cloud rows; taking b and j from R.tile here changes the generated code
  int ids[XR];
  auto load_ids = [&](int t) {
    const int b = t / R.ntiles, j = t - b * R.ntiles;
#pragma unroll
    for (int i = 0; i < XR; i++)
      if (ht + NHELP * i < E::TILE) ids[i] = fetch_id(b, j * E::TILE + ht + NHELP * i);
  };
  load_ids(R.t_begin);
#pragma unroll 1
  for (int it = 0; it < R.my_tiles; it++) {
    const Range::Tile t = R.tile(it);
    const int b = t.b, ci = t.ci;
    const bool cand_first = t.cand_first;
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
      if (ci > 0) wait_use(bar.front_bar, (uint32_t)(ci - 1));
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
      mbar_arrive(bar.cand_bar);
      tl.mark(TH_CAND);
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
        if (ht + NHELP * i < E::TILE) fetch_row(b, ids[i], r[i]);
#pragma unroll
      for (int i = 0; i < XR; i++)
        if (ht + NHELP * i < E::TILE) finish_row(r[i], v[i]);
    }
    tl.mark(TH_BUILD);
    if (it > 0) wait_use(bar.x0_empty, (uint32_t)(it - 1));
    tl.mark(TH_EMPTY);
#pragma unroll
    for (int i = 0; i < XR; i++)
      if (ht + NHELP * i < E::TILE) {
        float2 *dst = reinterpret_cast<float2 *>(x0 + (ht + NHELP * i) * 6);
        dst[0] = make_float2(v[i][0], v[i][1]);
        dst[1] = make_float2(v[i][2], v[i][3]);
        dst[2] = make_float2(v[i][4], v[i][5]);
      }
    mbar_arrive(bar.x0_full);
    if (it + 1 < R.my_tiles) load_ids(R.t_begin + it + 1);
    tl.mark(TH_BUILD);
    if (cand_first && ci > 0) {
      fold(ci - 1);
      tl.mark(TH_FOLD);
    }
  }
  fold(R.ncand - 1);
  tl.mark(TH_FOLD);
  tl.write(NCW + ht / 32, R.my_tiles);
}

// ---- L1: 64 -> 64 of d64 in place (STNkd shared conv with bias and ReLU, or the per-candidate T64 feature
// transform), and the PointNetSeg point feature of this thread's rows p0 and p0 + 8 of candidate b (pointnet2.py:261)
__device__ __forceinline__ void layer1(const cg_trunk_args &a, const Misc &S, uint32_t w1_s, int N, int b, int p0,
                                       int q, float *d64, uint32_t (*xh)[4], uint32_t (*xl)[4]) {
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
  if (a.pf_out) {
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

// ---- L2: 64 -> 128 (+bias, ReLU) of the L1 output d64 into acc; xh / xl hold its A fragments ----
__device__ __forceinline__ void layer2(const Misc &S, uint32_t w2_s, int q, float *d64, uint32_t (*xh)[4],
                                       uint32_t (*xl)[4], float *acc) {
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
}

// X3 -> the [TILE x 128] K-major image: accumulator pair i (channels 8i + 2q, +1) of row `row` (+ 8) is one 32-bit
// word of 16-byte chunk i & 7 of K-block i >> 3 (conflict-free: the 8 rows of a step hit 8 chunks).  vmax keeps the
// largest value stored on the fp16 engines.
template <class E>
__device__ __forceinline__ void store_x3(unsigned char *smem, const float *acc, int row, int q, float &vmax) {
#pragma unroll
  for (int r = 0; r < 2; r++) {
    const int pr = row + 8 * r;
#pragma unroll
    for (int i = 0; i < 16; i++) {
      const float x0 = acc[4 * i + 2 * r], x1 = acc[4 * i + 2 * r + 1];
      const uint32_t off = X3_OFF + (uint32_t)(i >> 3) * E::X3_KB + row_chunk_off(pr, i & 7) + 4u * q;
      uint32_t h, l;
      if (E::PASSES == 1) {
        vmax = fmaxf(vmax, fmaxf(x0, x1));
        // values beyond the fp16 range saturate to 65504 instead of becoming inf (x0 -> low half)
        asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h) : "f"(x1), "f"(x0));
      } else if (E::PASSES == 2) {   // split_f16x2 clamps to the fp16 range: record what it clamps
        vmax = fmaxf(vmax, fmaxf(x0, x1));
        split_f16x2(x0, x1, h, l);
      } else {
        split_bf16x2(x0, x1, h, l);
      }
      *reinterpret_cast<uint32_t *>(smem + off) = h;
      if (E::PASSES != 1) *reinterpret_cast<uint32_t *>(smem + off + E::X3_LO) = l;
    }
  }
}

// L3 unit u of the current tile: 128-point block u % NBLK of chunk u / NBLK, one m64n128 accumulator d.  The CTA's
// W3 K-blocks run on over its range: gslot counts those consumed before the current tile, and K-block kb of chunk c
// is the CTA's K-block gslot + 2 c + kb, in slot (gslot + 2 c + kb) % NSLOT as that slot's use (..) / NSLOT.
template <class E>
__device__ __forceinline__ void l3_issue(const Barriers &bar, uint32_t smem_s, uint32_t gslot, int wg, int u,
                                         float *d, Timeline &tl) {
  const int c = u / E::NBLK, hb = u % E::NBLK;
  if (hb == 0) {
    tl.span_begin();
    wait_use(bar.full_at((gslot + 2u * c) % E::NSLOT), (gslot + 2u * c) / E::NSLOT);
    wait_use(bar.full_at((gslot + 2u * c + 1) % E::NSLOT), (gslot + 2u * c + 1) / E::NSLOT);
    tl.span_end(TL_RING);
  }
  wg_fence_regs<64>(d);
  wg_fence();
#pragma unroll
  for (int kb = 0; kb < 2; kb++) {
    const uint32_t ws = smem_s + RING_OFF + (gslot + 2u * c + kb) % E::NSLOT * E::SLOT_BYTES + (uint32_t)wg * (PIECE / 2);
    const uint32_t xs = smem_s + X3_OFF + (uint32_t)kb * E::X3_KB + (uint32_t)hb * PIECE;
#pragma unroll
    for (int ks = 0; ks < 4; ks++) {
      const uint32_t first = (kb | ks) ? 1u : 0u;
      const uint64_t aw = wg_desc(ws + 32u * ks), bx = wg_desc(xs + 32u * ks);
      if (E::PASSES == 3) {
        const uint64_t al = wg_desc(ws + PIECE + 32u * ks), bxl = wg_desc(xs + E::X3_LO + 32u * ks);
        wg_ss_m64n128<false>(d, aw, bxl, first);   // w_hi * x_lo
        wg_ss_m64n128<false>(d, al, bx, 1u);       // w_lo * x_hi
        wg_ss_m64n128<false>(d, aw, bx, 1u);       // w_hi * x_hi
      } else if (E::PASSES == 2) {
        wg_ss_m64n128<true>(d, aw, wg_desc(xs + E::X3_LO + 32u * ks), first);
        wg_ss_m64n128<true>(d, aw, bx, 1u);
      } else {
        wg_ss_m64n128<true>(d, aw, bx, first);
      }
    }
    if (E::EARLY_RELEASE && kb == 0) wg_commit();   // K-block 0 as a group of its own (see the L3 loop)
  }
  wg_commit();
  wg_fence_regs<64>(d);
}

// unit u is complete in this warpgroup: the max over its points of each of this thread's rows (channels
// 128 c + 64 wg + 16 w4 + g + 8 r) is folded over the row's quad, and the q = 0 lane, the channel's only owner in the
// CTA, keeps the candidate's running max as a key in kk, its row of keys[ci & 1] (stored on the candidate's first
// unit of the range).  After the chunk's last unit hand its two W3 slots back.
template <class E>
__device__ __forceinline__ void l3_reduce(const Barriers &bar, uint32_t gslot, int lane, int u, const float *d,
                                          uint32_t *kk, bool cand_first) {
  const int c = u / E::NBLK, hb = u % E::NBLK, q = lane & 3;
  if (hb == E::NBLK - 1) {
    __syncwarp();
    if (lane == 0) {
      if (!E::EARLY_RELEASE) mbar_arrive(bar.empty_at((gslot + 2u * c) % E::NSLOT));
      mbar_arrive(bar.empty_at((gslot + 2u * c + 1) % E::NSLOT));
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
}

template <int PASSES>
__global__ void __launch_bounds__(NTC, 1) trunk_tc_kernel(const cg_trunk_args a
#ifdef CG_EXPERIMENTS
                                                          , unsigned long long *tl_out
#endif
) {
  using E = Engine<PASSES>;
  constexpr int TILE = E::TILE, NBLK = E::NBLK, NSLOT = E::NSLOT;
  constexpr uint32_t SLOT_BYTES = E::SLOT_BYTES, X3_KB = E::X3_KB, X3_LO = E::X3_LO;
  constexpr bool F16 = E::F16;
  // the operand tiles need 1024-byte alignment (SWIZZLE_128B atoms); the kernel has no static shared memory
  extern __shared__ __align__(1024) unsigned char smem[];
  if ((smem_u32(smem) & 1023u) != 0u) __trap();
  Misc &S = *reinterpret_cast<Misc *>(smem + MISC_OFF);
  uint32_t *keys = reinterpret_cast<uint32_t *>(smem + KEYS_OFF);
  // warp index through a shuffle: the compiler then knows it is warp-uniform and the role branches are not divergent
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  const int N = a.N;
  const Range R(a.B, N, TILE);
  const unsigned char *img = static_cast<const unsigned char *>(a.tc_img);
  const bool has_l1 = a.stage1_mode != 0;
  const uint32_t smem_s = smem_u32(smem);
  const uint32_t w1_s = smem_s + W1_OFF, w2_s = smem_s + W2_OFF, x3_s = smem_s + X3_OFF, ring_s = smem_s + RING_OFF;
  const uint32_t misc_s = smem_s + MISC_OFF;
  const Barriers bar(misc_s);
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
  if (tid == 0) bar.init(NSLOT);
  __syncthreads();

#ifdef CG_EXPERIMENTS
  Timeline tl(tl_out);
#else
  Timeline tl;
#endif

  if (warp == PROD_WARP) {
    if (lane == 0) producer<E>(a, img, R, bar, smem_u32(smem));
    return;
  }

  if (warp >= HELP_WARP) {
    helpers<E>(a, R, bar, smem, x0, keys, N, t64_handoff, tl, tid - HELP_WARP * 32);
    return;
  }

  // ======================= consumer warpgroups =======================
  const int wg = warp >> 2, w4 = warp & 3, g = lane >> 2, q = lane & 3;
  float vmax = 0.f;   // largest 128->1024 input seen by this thread (post-ReLU, fp16 engines): reported if beyond the fp16 range
  wait_use(bar.w_bar, 0u);

  // W3 ring slot of K-block kb of chunk c of the current tile
  uint32_t gslot = 0;   // W3 slots consumed before the current tile
  auto slot_of = [&](int c, int kb) { return (gslot + 2u * c + kb) % NSLOT; };

  // this thread's front rows of a tile: prow(blk) and prow(blk) + 8 of each 64-row block blk
  auto prow = [&](int blk) { return wg * (TILE / 2) + blk * 64 + w4 * 16 + g; };
  tl.mark(TL_START);
  for (int it = 0; it < R.my_tiles; it++) {
    const Range::Tile t = R.tile(it);
    const int b = t.b, j = t.j, ci = t.ci;
    const bool cand_first = t.cand_first, cand_last = t.cand_last;
    if (cand_first && t64_handoff) wait_use(bar.cand_bar, (uint32_t)ci);   // T64 image of candidate b
    wait_use(bar.x0_full, (uint32_t)it);   // X0 holds this tile's input rows
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
        tl.mark(TL_INPUT);
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
      if (blk == NBLK - 1) mbar_arrive(bar.x0_empty);
      uint32_t xh[4][4], xl[4][4];   // A fragments of the layer input (K = 64), bf16 hi + lo
      // ---- L1: 64 -> 64 (STNkd shared conv, or the per-candidate T64 feature transform) ----
      if (has_l1) layer1(a, S, w1_s, N, b, p0, q, d64, xh, xl);
      // the last read of candidate b's T64 image in this range is done: the helpers may replace it
      if (t64_handoff && cand_last && blk == NBLK - 1) mbar_arrive(bar.front_bar);
      // ---- L2: 64 -> 128 ----
      float acc[64];
      layer2(S, w2_s, q, d64, xh, xl, acc);
      tl.mark(TL_FRONT);
      // Both warpgroups' L3 wgmma of the previous tile are complete (each waited for its own before getting here):
      // the X3 image may be overwritten.  The first block's front ran under the other warpgroup's L3.
      if (blk == 0) asm volatile("bar.sync 1, 256;" ::: "memory");
      store_x3<E>(smem, acc, prow(blk), q, vmax);
    }
    // X3 is complete once every consumer thread has stored its part: make it visible to the wgmma (async) proxy
    fence_proxy_async();
    asm volatile("bar.sync 1, 256;" ::: "memory");
    tl.mark(TL_X3);
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
    uint32_t *kk = keys + (ci & 1) * 1024 + wg * 64 + w4 * 16 + g;
#pragma unroll 1
    for (int u0 = 0; u0 < NCHUNK * NBLK; u0 += E::GROUP) {
      float acc3[2][64];   // even / odd units
      l3_issue<E>(bar, smem_s, gslot, wg, u0, acc3[0], tl);
#pragma unroll
      for (int j = 0; j < E::GROUP; j++) {
        if (j + 1 < E::GROUP) l3_issue<E>(bar, smem_s, gslot, wg, u0 + j + 1, acc3[(j + 1) & 1], tl);
        tl.span_begin();
        if (E::EARLY_RELEASE) {
          wg_wait<1>();
          __syncwarp();
          if (lane == 0) mbar_arrive(bar.empty_at(slot_of((u0 + j) / NBLK, 0)));
        }
        if (j + 1 < E::GROUP) wg_wait<1>();
        else wg_wait<0>();
        tl.span_end(TL_L3_WAIT);
        wg_fence_regs<64>(acc3[j & 1]);
        l3_reduce<E>(bar, gslot, lane, u0 + j, acc3[j & 1], kk, cand_first);
      }
    }
    gslot += 2u * NCHUNK;
    // candidate b's max is complete in keys[ci & 1]: hand it to the helpers
    if (cand_last) mbar_arrive(bar.keys_of(ci));
    tl.mark(TL_L3);
  }
  if (F16 && vmax > 65504.f && a.ovf_flag) atomicOr(a.ovf_flag, 1u);
  tl.write(warp, R.my_tiles);
}

}  // namespace

size_t cg_tc_image_bytes() { return (size_t)IMG_W3H_OFF + IMG_W3H; }

int cg_tc_prepare(cg_ctx *ctx, const float *Wt3, const float *Wt2, const float *Wt1, void *dst_dev, int *f16_ok) {
  CG_CUDA(ctx, cudaFuncSetAttribute(trunk_tc_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Engine<3>::SMEM));
  CG_CUDA(ctx, cudaFuncSetAttribute(trunk_tc_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Engine<2>::SMEM));
  CG_CUDA(ctx, cudaFuncSetAttribute(trunk_tc_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Engine<1>::SMEM));
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

#ifdef CG_EXPERIMENTS
// Copies back the records of one timelined launch over `tiles` tiles of `tp` points, frees tl and prints the
// averages: cycles of one warp, averaged over the consumer (helper) warps of the sampled CTAs; the warps of a CTA run
// concurrently, so "total" is also the CTA's cycles.
static int trunk_timeline_report(cg_ctx *ctx, const cg_trunk_args &a, int passes, int tp, unsigned long long *tl) {
  const size_t tl_words = (size_t)TL_CTAS * TL_WARPS * TL_REC;
  std::vector<unsigned long long> h(tl_words);
  CG_CUDA(ctx, cudaMemcpyAsync(h.data(), tl, tl_words * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CG_CUDA(ctx, cudaFreeAsync(tl, ctx->stream));
  CG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
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
  return CG_OK;
}
#endif

// one launch of the engine with L3 in PASSES passes
template <int PASSES>
static int trunk_launch(cg_ctx *ctx, const cg_trunk_args &a) {
  using E = Engine<PASSES>;
  // persistent: one CTA per SM (or per tile, if there are fewer tiles), each over a balanced range of tiles
  const long long tiles = (long long)a.B * ((a.N + E::TILE - 1) / E::TILE);
  CG_REQUIRE(ctx, tiles <= INT_MAX, "trunk: too many tiles in one launch");
  const int grid = (int)std::min<long long>(ctx->num_sms, tiles);
#ifdef CG_EXPERIMENTS
  static const bool timeline = getenv("CG_TRUNK_TIMELINE") && atoi(getenv("CG_TRUNK_TIMELINE")) != 0;
  unsigned long long *tl = nullptr;
  const size_t tl_bytes = (size_t)TL_CTAS * TL_WARPS * TL_REC * 8;
  if (timeline) {
    CG_CUDA(ctx, cudaMallocAsync(&tl, tl_bytes, ctx->stream));
    CG_CUDA(ctx, cudaMemsetAsync(tl, 0, tl_bytes, ctx->stream));
  }
  trunk_tc_kernel<PASSES><<<grid, NTC, E::SMEM, ctx->stream>>>(a, tl);
  CG_LAUNCH_CHECK(ctx);
  if (timeline) return trunk_timeline_report(ctx, a, PASSES, E::TILE, tl);
#else
  trunk_tc_kernel<PASSES><<<grid, NTC, E::SMEM, ctx->stream>>>(a);
  CG_LAUNCH_CHECK(ctx);
#endif
  return CG_OK;
}

int cg_trunk_launch_tc(cg_ctx *ctx, const cg_trunk_args &a) {
  CG_REQUIRE(ctx, a.B > 0 && a.N > 0, "trunk: B,N must be positive");
  CG_REQUIRE(ctx, a.tc_img != nullptr, "trunk: tensor-core weight image missing");
  // W3 beyond the fp16 range: the fp16 engines fall back to the 3-pass bf16 kernel
  const int passes = !a.tc_f16_ok || ctx->engine == 1 ? 3 : (ctx->engine == 2 ? 2 : 1);
  if (passes == 3) return trunk_launch<3>(ctx, a);
  else if (passes == 2) return trunk_launch<2>(ctx, a);
  else return trunk_launch<1>(ctx, a);
}

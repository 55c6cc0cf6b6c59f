// cg_net.cuh -- network weight table, trunk and fully-connected launch interfaces (internal).
#pragma once
#include "cg_common.cuh"

// One folded (conv|linear)+BN layer: Wt is [K][C] row-major (k-major), b is [C].  tc is the layer's own wgmma operand
// image (cg_linear_tc_image), owned by the net / MLP that holds the layer; null for shapes the tensor-core FC kernel
// does not take and for layers that are not launched through cg_linear_launch (the trunk layers).
struct cg_layer {
  const float *Wt;
  const float *b;
  int K, C;
  const void *tc;
};

// Weight order inside the blob (must match catgrasp_b200/weights.py:BLOB_ORDER).
enum cg_layer_id {
  L_S3_C1 = 0, L_S3_C2, L_S3_C3, L_S3_F1, L_S3_F2, L_S3_F3,   // STN3d      pointnet2.py:153-186
  L_E_C1,                                                      // encoder conv1 :252
  L_SK_C1, L_SK_C2, L_SK_C3, L_SK_F1, L_SK_F2, L_SK_F3,        // STNkd(64)  :189-224
  L_E_C2, L_E_C3,                                              // encoder conv2/3 :263-264
  L_HEAD0, L_HEAD1, L_HEAD2, L_HEAD3, L_HEAD4,                 // cls: fc1,fc2,fc3 ; seg: conv1g,conv1p,conv2,conv3,conv4
  L_COUNT
};

struct cg_net {
  cg_ctx *ctx;
  int kind, n_out;
  float *blob_dev;
  size_t blob_floats;
  cg_layer L[L_COUNT];
  // tensor-core (wgmma) bf16 hi/lo + fp16 operand images of each trunk's 128->1024, 64->128 and (STNkd) 64->64
  // layers, built at create time: [W3 | W2 | W1]; indices 0 = STN3d, 1 = STNkd, 2 = encoder
  void *tc_img[3];
  int tc_f16_ok[3];   // 128->1024 weights fit fp16 (|w| < 65504): the 2-pass engine may be used for this trunk
};

// How the first kernel of each trunk obtains its (N,6) input rows.
struct cg_input_src {
  const float *x_direct;   // (B,N,6) float32, or nullptr
  const double *cloud_xyz; // (M,3)
  const double *cloud_nrm; // (M,3)
  const double *poses;     // (B,4,4)
  const int32_t *ids;      // (B,N)
  const double *mean;      // (6) or nullptr
  const double *stdv;      // (6) or nullptr
  int M;
};

struct cg_trunk_args {
  cg_input_src in;
  int B, N;
  const float *T3;   // (B,9) or nullptr
  cg_layer l0;       // 6 -> 64  (+ReLU)
  int stage1_mode;   // 0 none, 1 shared 64->64 (+ReLU), 2 per-candidate 64x64 matrix (no bias / ReLU)
  cg_layer l1;
  const float *T64;  // (B,64,64) when stage1_mode == 2
  cg_layer l2;       // 64 -> 128 (+ReLU)
  cg_layer l3;       // 128 -> 1024
  const void *tc_img; // wgmma operand images [W3 | W2 | W1 | W3 fp16] of l3 / l2 / l1 (engines 1-3)
  int tc_f16_ok;      // engine 2 allowed for this trunk (else it runs the 3-pass kernel)
  int relu3;
  uint32_t *gmax_keys;  // (B,1024) order-preserving keys, zero-initialised by the launcher
  float *pf_out;        // (B,N,64) stage-1 output (PointNetSeg point feature) or nullptr
  uint32_t *ovf_flag;       // engines 2, 3: set to 1 when an activation had to be clamped to the fp16 range (or nullptr)
};

int cg_trunk_launch_simt(cg_ctx *ctx, const cg_trunk_args &a);
int cg_trunk_launch_tc(cg_ctx *ctx, const cg_trunk_args &a);   // engines 1-3 (wgmma)
size_t cg_tc_image_bytes();
// Wt3 [128][1024], Wt2 [64][128], Wt1 [64][64] or nullptr (folded fp32, k-major rows, host).  Also sets the trunk
// kernels' shared-memory limit on the current device, so it runs there before any trunk launch that uses the image.
int cg_tc_prepare(cg_ctx *ctx, const float *Wt3, const float *Wt2, const float *Wt1, void *dst_dev, int *f16_ok);

// Packs rows c0 .. c0+rows-1 (output channels) of the K-block k0 .. k0+63 of a host weight Wt [K][C] (k-major) into
// the swizzled [rows x 64] bf16 hi / lo operand pieces of the wgmma kernels (w = hi + lo, both round-to-nearest-even).
void cg_pack_bf16x2_block(const float *Wt, int C, int c0, int rows, int k0, unsigned char *hi, unsigned char *lo);

// Row tiles of the fully-connected kernels: gridDim.y is capped at 65535, so the tiles are spread over (y, z) and a
// launch covers up to 2^31 rows.  tile = blockIdx.z * gridDim.y + blockIdx.y; CTAs past the last tile exit at once.
inline dim3 cg_row_tile_grid(unsigned col_tiles, long long row_tiles) {
  const unsigned y = row_tiles < 65535 ? (unsigned)row_tiles : 65535u;
  return dim3(col_tiles, y, (unsigned)((row_tiles + y - 1) / y));
}
__device__ __forceinline__ long long cg_row_tile() { return (long long)blockIdx.z * gridDim.y + blockIdx.y; }

// Y[M][C] = act(X[M][K] @ L.Wt[K][C] + bias[(row / rows_per_bias)][C]), bias = row_bias if given, else L.b.
// Runs on tensor cores when the engine is >= 1, the layer has an image (L.tc) and M >= 64; else on the FMA kernels.
enum : unsigned {
  CG_FC_RELU = 1u,   // ReLU after the bias
  CG_FC_KEYS = 2u,   // X holds order-preserving uint keys (a trunk's max-pool output), decoded on load
};
// cg_linear_launch runs M <= CG_FC_FEW_ROWS rows on its few-row kernel (below the tensor-core kernel's 64), whose
// sums for a row do not depend on M
constexpr int CG_FC_FEW_ROWS = 8;
int cg_linear_launch(cg_ctx *ctx, const cg_layer &L, const float *X, int M, float *Y, unsigned flags,
                     const float *row_bias = nullptr, int rows_per_bias = 0);
// Row groups of the few-row kernel for one launch: g[i] = first row << 4 | rows (1 .. CG_FC_FEW_ROWS); n = 0 is a
// plain launch on M rows.
constexpr int CG_FC_GROUPS_PER_LAUNCH = 128;
struct cg_fc_row_groups {
  int n;
  int32_t g[CG_FC_GROUPS_PER_LAUNCH];
};
// cg_linear_launch on each of n_groups consecutive row groups of X / Y (rows[i] rows each, host array), with each
// group's bits: the groups of at most CG_FC_FEW_ROWS rows share few-row launches (CG_FC_GROUPS_PER_LAUNCH per launch),
// every other group is a cg_linear_launch of its own.  Layer bias only; fewer than 2^27 rows in all.
int cg_linear_launch_groups(cg_ctx *ctx, const cg_layer &L, const float *X, const int32_t *rows, int n_groups, float *Y,
                            unsigned flags);
// tensor-core FC path (cg_linear_tc.cu).  The image builder returns nullptr in *img for shapes the kernel does not take
// (K % 64 != 0 or N < 64); otherwise a device image the caller frees with cudaFree.  It also sets the kernel's
// shared-memory limit on the current device.
int cg_linear_tc_image(cg_ctx *ctx, const float *Wt_host, int K, int N, const void **img);
int cg_linear_tc_launch(cg_ctx *ctx, const float *X, int M, int K, const void *img, const float *bias, int N, int relu,
                        int bias_row_div, int x_is_keys, float *Y);
int cg_softmax_launch(cg_ctx *ctx, const float *logits, int B, int C, float *probs, int32_t *label);
int cg_nunocs_post_launch(cg_ctx *ctx, const float *logits, int P, int bins, float *coords,
                          float *conf_z, int32_t *out_bins);

// cg_net.cu -- network handles and forward orchestration behind the C ABI.
//
// PointNetCls  (pointnet2.py:275-299): trunk A -> FC x3 -> T3
//                                      trunk B -> FC x3 -> T64
//                                      trunk C -> FC x3 -> logits -> softmax
// PointNetSeg  (pointnet2.py:302-329): same encoder, trunk C also emits the
//   64-ch point feature; the 1088->512 conv is split into its global part
//   (computed once per cloud and used as a per-cloud bias) and its 64-ch
//   point part, which removes 4.29 of 9.72 GMAC without changing the math.
#include <memory>

#include "cg_net.cuh"

namespace {

struct LayerDim { int K, C; };

void layer_dims(int kind, int n_out, LayerDim d[L_COUNT]) {
  d[L_S3_C1] = {6, 64};     d[L_S3_C2] = {64, 128};   d[L_S3_C3] = {128, 1024};
  d[L_S3_F1] = {1024, 512}; d[L_S3_F2] = {512, 256};  d[L_S3_F3] = {256, 9};
  d[L_E_C1] = {6, 64};
  d[L_SK_C1] = {64, 64};    d[L_SK_C2] = {64, 128};   d[L_SK_C3] = {128, 1024};
  d[L_SK_F1] = {1024, 512}; d[L_SK_F2] = {512, 256};  d[L_SK_F3] = {256, 4096};
  d[L_E_C2] = {64, 128};    d[L_E_C3] = {128, 1024};
  if (kind == CG_NET_CLS) {
    d[L_HEAD0] = {1024, 512}; d[L_HEAD1] = {512, 256}; d[L_HEAD2] = {256, n_out};
    d[L_HEAD3] = {0, 0};      d[L_HEAD4] = {0, 0};
  } else {
    d[L_HEAD0] = {1024, 512}; d[L_HEAD1] = {64, 512};  d[L_HEAD2] = {512, 256};
    d[L_HEAD3] = {256, 128};  d[L_HEAD4] = {128, n_out};
  }
}

inline size_t pad64(size_t n) { return (n + 63) & ~size_t(63); }

constexpr int CHUNK_B = CG_GRASPQ_CHUNK_B;  // candidates per internal pass (bounds the T64 workspace to 256 MB)

}  // namespace

extern "C" size_t cg_net_blob_floats(int kind, int n_out) {
  LayerDim d[L_COUNT];
  layer_dims(kind, n_out, d);
  size_t n = 0;
  for (int i = 0; i < L_COUNT; i++) n += pad64((size_t)d[i].K * d[i].C) + pad64((size_t)d[i].C);
  return n;
}

extern "C" int cg_net_create(cg_ctx *ctx, int kind, int n_out, const float *blob_host, size_t blob_floats,
                             cg_net **out) {
  if (!ctx || !out) return CG_EINVAL;
  CG_REQUIRE(ctx, kind == CG_NET_CLS || kind == CG_NET_SEG, "net kind");
  CG_REQUIRE(ctx, n_out > 0 && (kind == CG_NET_SEG || n_out <= 32), "n_out");
  CG_REQUIRE(ctx, blob_host && blob_floats == cg_net_blob_floats(kind, n_out), "weight blob size mismatch");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  // value-initialised (null blob, images and layers), so that every error return below frees what exists so far
  std::unique_ptr<cg_net, void (*)(cg_net *)> net(new cg_net(), cg_net_destroy);
  net->ctx = ctx;
  net->kind = kind;
  net->n_out = n_out;
  net->blob_floats = blob_floats;
  CG_CUDA(ctx, cudaMalloc(&net->blob_dev, blob_floats * sizeof(float)));
  CG_CUDA(ctx, cudaMemcpyAsync(net->blob_dev, blob_host, blob_floats * sizeof(float), cudaMemcpyHostToDevice,
                               ctx->stream));
  LayerDim d[L_COUNT];
  layer_dims(kind, n_out, d);
  size_t off = 0;
  size_t woff[L_COUNT];
  for (int i = 0; i < L_COUNT; i++) {
    net->L[i].K = d[i].K;
    net->L[i].C = d[i].C;
    net->L[i].Wt = net->blob_dev + off;
    woff[i] = off;
    off += pad64((size_t)d[i].K * d[i].C);
    net->L[i].b = net->blob_dev + off;
    off += pad64((size_t)d[i].C);
  }
  // tensor-core operand images of the three trunks
  const int l3[3] = {L_S3_C3, L_SK_C3, L_E_C3}, l2[3] = {L_S3_C2, L_SK_C2, L_E_C2}, l1[3] = {-1, L_SK_C1, -1};
  for (int i = 0; i < 3; i++) {
    CG_CUDA(ctx, cudaMalloc(&net->tc_img[i], cg_tc_image_bytes()));
    int rc = cg_tc_prepare(ctx, blob_host + woff[l3[i]], blob_host + woff[l2[i]],
                           l1[i] >= 0 ? blob_host + woff[l1[i]] : nullptr, net->tc_img[i], &net->tc_f16_ok[i]);
    if (rc != CG_OK) return rc;
  }
  // tensor-core images of the FC / head layers (the trunk layers have theirs in tc_img)
  const int fc_layers[] = {L_S3_F1, L_S3_F2, L_SK_F1, L_SK_F2, L_SK_F3, L_HEAD0, L_HEAD1, L_HEAD2, L_HEAD3, L_HEAD4};
  for (int li : fc_layers) {
    int rc = cg_linear_tc_image(ctx, blob_host + woff[li], d[li].K, d[li].C, &net->L[li].tc);
    if (rc != CG_OK) return rc;
  }
  CG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  *out = net.release();
  return CG_OK;
}

extern "C" void cg_net_destroy(cg_net *net) {
  if (!net) return;
  cudaSetDevice(net->ctx->device);
  for (int i = 0; i < L_COUNT; i++) cudaFree(const_cast<void *>(net->L[i].tc));
  cudaFree(net->blob_dev);
  for (int i = 0; i < 3; i++) cudaFree(net->tc_img[i]);
  delete net;
}

namespace {

int trunk_launch(cg_ctx *ctx, const cg_trunk_args &a) {
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  if (ctx->prof) {
    CG_CUDA(ctx, cudaEventCreate(&e0));
    CG_CUDA(ctx, cudaEventCreate(&e1));
    CG_CUDA(ctx, cudaEventRecord(e0, ctx->stream));
  }
  int rc;
  if (ctx->engine >= 1) rc = cg_trunk_launch_tc(ctx, a);   // 3-pass bf16 / 2-pass fp16 / 1-pass fp16 on wgmma
  else rc = cg_trunk_launch_simt(ctx, a);
  if (ctx->prof) {
    CG_CUDA(ctx, cudaEventRecord(e1, ctx->stream));
    ctx->prof_events.emplace_back(e0, e1);
  }
  return rc;
}

struct EncoderWs {
  uint32_t *gmax;   // (B,1024)
  float *f1;        // (B,512)
  float *f2;        // (B,256)
  float *T3;        // (B,9)
  float *T64;       // (B,4096)
};

void encoder_ws_carve(cg_arena &ar, int B, EncoderWs &w) {
  w.gmax = ar.take<uint32_t>((size_t)B * 1024);
  w.f1 = ar.take<float>((size_t)B * 512);
  w.f2 = ar.take<float>((size_t)B * 256);
  w.T3 = ar.take<float>((size_t)B * 9);
  w.T64 = ar.take<float>((size_t)B * 4096);
}

// The FC chain after a trunk (STN3d, STNkd, cls head): layers L[l], L[l+1], L[l+2] =
// 1024 -> 512 (ReLU, from the max-pool keys in w.gmax) -> 256 (ReLU) -> out (no ReLU).
// rows > 0 launches it on groups of at most `rows` clouds (0: all B in one launch per layer).
// groups (host, n_groups entries summing to B): launch each layer on these row groups instead (cg_linear_launch_groups).
int fc_chain(cg_ctx *ctx, const cg_layer *L, int l, int B, const EncoderWs &w, float *out, int rows = 0,
             const int32_t *groups = nullptr, int n_groups = 0) {
  if (groups) {
    int rc;
    if ((rc = cg_linear_launch_groups(ctx, L[l], reinterpret_cast<const float *>(w.gmax), groups, n_groups, w.f1,
                                      CG_FC_RELU | CG_FC_KEYS)))
      return rc;
    if ((rc = cg_linear_launch_groups(ctx, L[l + 1], w.f1, groups, n_groups, w.f2, CG_FC_RELU))) return rc;
    return cg_linear_launch_groups(ctx, L[l + 2], w.f2, groups, n_groups, out, 0);
  }
  const int g = rows > 0 ? rows : B;
  for (int r0 = 0; r0 < B; r0 += g) {
    const int m = B - r0 < g ? B - r0 : g;
    int rc;
    if ((rc = cg_linear_launch(ctx, L[l], reinterpret_cast<const float *>(w.gmax + (size_t)r0 * 1024), m,
                               w.f1 + (size_t)r0 * 512, CG_FC_RELU | CG_FC_KEYS)))
      return rc;
    if ((rc = cg_linear_launch(ctx, L[l + 1], w.f1 + (size_t)r0 * 512, m, w.f2 + (size_t)r0 * 256, CG_FC_RELU)))
      return rc;
    if ((rc = cg_linear_launch(ctx, L[l + 2], w.f2 + (size_t)r0 * 256, m, out + (size_t)r0 * L[l + 2].C, 0))) return rc;
  }
  return CG_OK;
}

// Runs the PointNetEncoder (pointnet2.py:241-271) for B clouds; on return w.gmax holds the
// (B,1024) global feature as order-preserving keys; pf_out (optional) the 64-ch point feature.
// keys_out (optional, test hook): (3,B,1024) copies of the three trunks' max-pool keys.  fc_rows, fc_groups,
// n_fc_groups: fc_chain's rows, groups and n_groups.
int encoder_forward(cg_net *net, const cg_input_src &in, int B, int N, EncoderWs &w, float *pf_out,
                    uint32_t *keys_out = nullptr, int fc_rows = 0, const int32_t *fc_groups = nullptr,
                    int n_fc_groups = 0) {
  cg_ctx *ctx = net->ctx;
  const cg_layer *L = net->L;
  int rc;
  cg_trunk_args a;
  a.in = in; a.B = B; a.N = N; a.ovf_flag = ctx->ovf_flag;
  const size_t kb = (size_t)B * 1024 * 4;
  // --- trunk A: STN3d convs + max (pointnet2.py:170-175)
  CG_CUDA(ctx, cudaMemsetAsync(w.gmax, 0, (size_t)B * 1024 * 4, ctx->stream));
  a.T3 = nullptr; a.l0 = L[L_S3_C1]; a.stage1_mode = 0; a.l1 = cg_layer{nullptr, nullptr, 0, 0}; a.T64 = nullptr;
  a.l2 = L[L_S3_C2]; a.l3 = L[L_S3_C3]; a.tc_img = net->tc_img[0]; a.tc_f16_ok = net->tc_f16_ok[0]; a.relu3 = 1; a.gmax_keys = w.gmax; a.pf_out = nullptr;
  if ((rc = trunk_launch(ctx, a))) return rc;
  if (keys_out) CG_CUDA(ctx, cudaMemcpyAsync(keys_out, w.gmax, kb, cudaMemcpyDeviceToDevice, ctx->stream));
  if ((rc = fc_chain(ctx, L, L_S3_F1, B, w, w.T3, fc_rows, fc_groups, n_fc_groups))) return rc;
  // --- trunk B: encoder conv1 + STNkd convs + max (pointnet2.py:252, :208-213)
  CG_CUDA(ctx, cudaMemsetAsync(w.gmax, 0, (size_t)B * 1024 * 4, ctx->stream));
  a.T3 = w.T3; a.l0 = L[L_E_C1]; a.stage1_mode = 1; a.l1 = L[L_SK_C1];
  a.l2 = L[L_SK_C2]; a.l3 = L[L_SK_C3]; a.tc_img = net->tc_img[1]; a.tc_f16_ok = net->tc_f16_ok[1]; a.relu3 = 1;
  if ((rc = trunk_launch(ctx, a))) return rc;
  if (keys_out) CG_CUDA(ctx, cudaMemcpyAsync(keys_out + (size_t)B * 1024, w.gmax, kb, cudaMemcpyDeviceToDevice, ctx->stream));
  if ((rc = fc_chain(ctx, L, L_SK_F1, B, w, w.T64, fc_rows, fc_groups, n_fc_groups))) return rc;
  // --- trunk C: conv1, @T64, conv2, conv3(+BN, no ReLU), max (pointnet2.py:252-265)
  CG_CUDA(ctx, cudaMemsetAsync(w.gmax, 0, (size_t)B * 1024 * 4, ctx->stream));
  a.stage1_mode = 2; a.T64 = w.T64; a.l1 = cg_layer{nullptr, nullptr, 64, 64};
  a.l2 = L[L_E_C2]; a.l3 = L[L_E_C3]; a.tc_img = net->tc_img[2]; a.tc_f16_ok = net->tc_f16_ok[2]; a.relu3 = 0; a.pf_out = pf_out;
  if ((rc = trunk_launch(ctx, a))) return rc;
  if (keys_out) CG_CUDA(ctx, cudaMemcpyAsync(keys_out + (size_t)2 * B * 1024, w.gmax, kb, cudaMemcpyDeviceToDevice, ctx->stream));
  return CG_OK;
}

int cls_forward_impl(cg_net *net, const cg_input_src &in_all, int B_all, int N, float *out_logits, float *out_probs,
                     int32_t *out_label) {
  cg_ctx *ctx = net->ctx;
  CG_REQUIRE(ctx, net->kind == CG_NET_CLS, "net is not a PointNetCls");
  CG_REQUIRE(ctx, B_all > 0 && N > 0, "B,N must be positive");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const int n_out = net->n_out;
  const int Bc_max = B_all < CHUNK_B ? B_all : CHUNK_B;
  EncoderWs w;
  float *logits_ws;
  int rc = cg_ws_carve(ctx, [&](cg_arena &ar) {
    encoder_ws_carve(ar, Bc_max, w);
    logits_ws = ar.take<float>((size_t)Bc_max * n_out);
  });
  if (rc) return rc;
  for (int b0 = 0; b0 < B_all; b0 += CHUNK_B) {
    const int B = (B_all - b0 < CHUNK_B) ? (B_all - b0) : CHUNK_B;
    cg_input_src in = in_all;
    if (in.x_direct) in.x_direct += (size_t)b0 * N * 6;
    if (in.poses) in.poses += (size_t)b0 * 16;
    if (in.ids) in.ids += (size_t)b0 * N;
    if ((rc = encoder_forward(net, in, B, N, w, nullptr))) return rc;
    float *lg = out_logits ? out_logits + (size_t)b0 * n_out : logits_ws;
    if ((rc = fc_chain(ctx, net->L, L_HEAD0, B, w, lg))) return rc;
    if (out_probs || out_label) {
      if ((rc = cg_softmax_launch(ctx, lg, B, n_out, out_probs ? out_probs + (size_t)b0 * n_out : nullptr,
                                  out_label ? out_label + b0 : nullptr)))
        return rc;
    }
  }
  return CG_OK;
}

// fc_rows > 0: the per-cloud FC layers run on groups of at most fc_rows clouds (encoder_forward)
int seg_forward_impl(cg_net *net, const float *x, int B, int N, float *out_logits, int bins, float *out_coords,
                     float *out_conf, int32_t *out_bins, int fc_rows = 0) {
  cg_ctx *ctx = net->ctx;
  CG_REQUIRE(ctx, net->kind == CG_NET_SEG, "net is not a PointNetSeg");
  CG_REQUIRE(ctx, B > 0 && N > 0 && x, "seg: bad arguments");
  CG_REQUIRE(ctx, B <= CHUNK_B, "seg: too many clouds in one call");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t P = (size_t)B * N;
  const int n_out = net->n_out;
  EncoderWs w;
  float *pf, *biasg, *y1, *y2, *y3, *lg;
  int rc = cg_ws_carve(ctx, [&](cg_arena &ar) {
    encoder_ws_carve(ar, B, w);
    pf = ar.take<float>(P * 64);
    biasg = ar.take<float>((size_t)B * 512);
    y1 = ar.take<float>(P * 512);
    y2 = ar.take<float>(P * 256);
    y3 = ar.take<float>(P * 128);
    lg = out_logits ? out_logits : ar.take<float>(P * n_out);
  });
  if (rc) return rc;
  cg_input_src in;
  memset(&in, 0, sizeof(in));
  in.x_direct = x;
  if ((rc = encoder_forward(net, in, B, N, w, pf, nullptr, fc_rows))) return rc;
  const cg_layer *L = net->L;
  // global half of conv1 (pointnet2.py:270-271 tiles the global feature over N; it is constant per cloud)
  const int g = fc_rows > 0 ? fc_rows : B;
  for (int r0 = 0; r0 < B; r0 += g)
    if ((rc = cg_linear_launch(ctx, L[L_HEAD0], reinterpret_cast<const float *>(w.gmax + (size_t)r0 * 1024),
                               B - r0 < g ? B - r0 : g, biasg + (size_t)r0 * 512, CG_FC_KEYS)))
      return rc;
  if ((rc = cg_linear_launch(ctx, L[L_HEAD1], pf, (int)P, y1, CG_FC_RELU, biasg, N))) return rc;
  if ((rc = cg_linear_launch(ctx, L[L_HEAD2], y1, (int)P, y2, CG_FC_RELU))) return rc;
  if ((rc = cg_linear_launch(ctx, L[L_HEAD3], y2, (int)P, y3, CG_FC_RELU))) return rc;
  if ((rc = cg_linear_launch(ctx, L[L_HEAD4], y3, (int)P, lg, 0))) return rc;
  if (out_coords || out_conf || out_bins) {
    CG_REQUIRE(ctx, bins > 0 && bins * 3 == n_out, "nunocs: n_out != 3*bins");
    if ((rc = cg_nunocs_post_launch(ctx, lg, (int)P, bins, out_coords, out_conf, out_bins))) return rc;
  }
  return CG_OK;
}

}  // namespace

extern "C" int cg_graspq_forward_dev(cg_net *net, const double *cloud_xyz, const double *cloud_nrm, int M,
                                     const double *poses, int B, const int32_t *ids, int N, const double *mean,
                                     const double *stdv, float *out_probs, int32_t *out_label) {
  if (!net) return CG_EINVAL;
  cg_ctx *ctx = net->ctx;
  CG_REQUIRE(ctx, cloud_xyz && cloud_nrm && poses && M > 0, "graspq: null cloud/poses");
  CG_REQUIRE(ctx, ids != nullptr || N <= M, "graspq: ids required when N > M");
  CG_REQUIRE(ctx, (mean == nullptr) == (stdv == nullptr), "graspq: mean/std must come together");
  cg_input_src in;
  memset(&in, 0, sizeof(in));
  in.cloud_xyz = cloud_xyz; in.cloud_nrm = cloud_nrm; in.poses = poses; in.ids = ids;
  in.mean = mean; in.stdv = stdv; in.M = M;
  return cls_forward_impl(net, in, B, N, nullptr, out_probs, out_label);
}

extern "C" int cg_graspq_forward_many_dev(cg_net *net, const double *cloud_xyz, const double *cloud_nrm, int M_total,
                                          const double *poses, int B_total, const int32_t *ids, int N,
                                          const double *mean, const double *stdv, const int32_t *fc_groups,
                                          int n_groups, float *out_probs, int32_t *out_label) {
  if (!net) return CG_EINVAL;
  cg_ctx *ctx = net->ctx;
  CG_REQUIRE(ctx, net->kind == CG_NET_CLS, "graspq_many: net is not a PointNetCls");
  CG_REQUIRE(ctx, cloud_xyz && cloud_nrm && poses && ids && fc_groups && out_probs, "graspq_many: null argument");
  CG_REQUIRE(ctx, M_total > 0 && B_total > 0 && N > 0 && n_groups > 0, "graspq_many: bad shape");
  CG_REQUIRE(ctx, (mean == nullptr) == (stdv == nullptr), "graspq_many: mean/std must come together");
  long long sum = 0;
  for (int i = 0; i < n_groups; i++) {
    CG_REQUIRE(ctx, fc_groups[i] >= 1 && fc_groups[i] <= CG_GRASPQ_CHUNK_B, "graspq_many: a group of 1 .. CHUNK_B rows");
    sum += fc_groups[i];
  }
  CG_REQUIRE(ctx, sum == B_total, "graspq_many: the groups do not add up to B_total");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const int n_out = net->n_out;
  const int Bc_max = B_total < CHUNK_B ? B_total : CHUNK_B;
  EncoderWs w;
  float *logits;
  int rc = cg_ws_carve(ctx, [&](cg_arena &ar) {
    encoder_ws_carve(ar, Bc_max, w);
    logits = ar.take<float>((size_t)Bc_max * n_out);
  });
  if (rc) return rc;
  cg_input_src in;
  memset(&in, 0, sizeof(in));
  in.cloud_xyz = cloud_xyz; in.cloud_nrm = cloud_nrm; in.mean = mean; in.stdv = stdv; in.M = M_total;
  // passes of whole groups, at most CHUNK_B candidates each: a candidate's trunk keys do not depend on the pass, and
  // each group's FC layers get the launch (and so the bits) the group's own call gets
  for (int g0 = 0, b0 = 0; g0 < n_groups;) {
    int g1 = g0, B = 0;
    while (g1 < n_groups && B + fc_groups[g1] <= CHUNK_B) B += fc_groups[g1++];
    in.poses = poses + (size_t)b0 * 16;
    in.ids = ids + (size_t)b0 * N;
    if ((rc = encoder_forward(net, in, B, N, w, nullptr, nullptr, 0, fc_groups + g0, g1 - g0))) return rc;
    if ((rc = fc_chain(ctx, net->L, L_HEAD0, B, w, logits, 0, fc_groups + g0, g1 - g0))) return rc;
    if ((rc = cg_softmax_launch(ctx, logits, B, n_out, out_probs + (size_t)b0 * n_out,
                                out_label ? out_label + b0 : nullptr)))
      return rc;
    g0 = g1;
    b0 += B;
  }
  return CG_OK;
}

extern "C" int cg_graspq_forward_host(cg_net *net, const double *cloud_xyz, const double *cloud_nrm, int M,
                                      const double *poses, int B, const int32_t *ids, int N, const double *mean,
                                      const double *stdv, float *out_probs, int32_t *out_label) {
  if (!net) return CG_EINVAL;
  cg_ctx *ctx = net->ctx;
  CG_REQUIRE(ctx, cloud_xyz && cloud_nrm && poses && ids && out_probs, "graspq_host: null argument");
  CG_REQUIRE(ctx, M > 0 && B > 0 && N > 0, "graspq_host: bad shape");
  // The subset indices are the bulk of the input (4 B x N per candidate; 16.8 MB for 4096 x 1024).  When the caller's
  // buffer is pinned (page-locked, mapped under UVA) the trunk kernels read it in place: every index is fetched exactly
  // once per trunk launch, two tiles ahead of its use, so the PCIe / C2C transfer hides under the kernels instead of
  // sitting in front of them.  Pageable memory takes the staged copy.  The mapped address is the current device's.
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const int32_t *ids_mapped = nullptr;
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, ids) == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer != nullptr)
    ids_mapped = static_cast<const int32_t *>(at.devicePointer);
  else
    cudaGetLastError();   // an unregistered pointer is not an error here
  const double *d_xyz, *d_nrm, *d_pose, *d_mean, *d_std; const int32_t *d_ids; int32_t *d_label; float *d_probs;
  return cg_io_stage(ctx, [&](cg_io_pieces &io) {
    d_xyz = io.in(cloud_xyz, (size_t)M * 3);
    d_nrm = io.in(cloud_nrm, (size_t)M * 3);
    d_pose = io.in(poses, (size_t)B * 16);
    d_ids = ids_mapped ? ids_mapped : io.in(ids, (size_t)B * N);
    d_mean = mean ? io.in(mean, 6) : nullptr;
    d_std = stdv ? io.in(stdv, 6) : nullptr;
    d_probs = io.out(out_probs, (size_t)B * net->n_out);
    d_label = io.out(out_label, B);
  }, [&] {
    return cg_graspq_forward_dev(net, d_xyz, d_nrm, M, d_pose, B, d_ids, N, d_mean, d_std, d_probs, d_label);
  });
}

extern "C" int cg_cls_forward_dev(cg_net *net, const float *x, int B, int N, float *out_logits, float *out_probs) {
  if (!net) return CG_EINVAL;
  CG_REQUIRE(net->ctx, x != nullptr, "cls: null input");
  cg_input_src in;
  memset(&in, 0, sizeof(in));
  in.x_direct = x;
  return cls_forward_impl(net, in, B, N, out_logits, out_probs, nullptr);
}

extern "C" int cg_seg_forward_dev(cg_net *net, const float *x, int B, int N, float *out_logits) {
  if (!net) return CG_EINVAL;
  CG_REQUIRE(net->ctx, out_logits != nullptr, "seg: null output");
  return seg_forward_impl(net, x, B, N, out_logits, 0, nullptr, nullptr, nullptr);
}

extern "C" int cg_encoder_probe_dev(cg_net *net, const float *x, const double *cloud_xyz, const double *cloud_nrm,
                                    int M, const double *poses, const int32_t *ids, const double *mean,
                                    const double *stdv, int B, int N, uint32_t *out_keys, float *out_T3,
                                    float *out_T64, float *out_pf) {
  if (!net) return CG_EINVAL;
  cg_ctx *ctx = net->ctx;
  CG_REQUIRE(ctx, B > 0 && B <= CHUNK_B && N > 0, "encoder_probe: 0 < B <= 16384, N > 0");
  CG_REQUIRE(ctx, out_keys && out_T3 && out_T64, "encoder_probe: null output");
  cg_input_src in;
  memset(&in, 0, sizeof(in));
  if (x) {
    in.x_direct = x;
  } else {
    CG_REQUIRE(ctx, cloud_xyz && cloud_nrm && poses && M > 0, "encoder_probe: null cloud/poses");
    CG_REQUIRE(ctx, ids != nullptr || N <= M, "encoder_probe: ids required when N > M");
    CG_REQUIRE(ctx, (mean == nullptr) == (stdv == nullptr), "encoder_probe: mean/std must come together");
    in.cloud_xyz = cloud_xyz; in.cloud_nrm = cloud_nrm; in.poses = poses; in.ids = ids;
    in.mean = mean; in.stdv = stdv; in.M = M;
  }
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  EncoderWs w;
  int rc = cg_ws_carve(ctx, [&](cg_arena &ar) { encoder_ws_carve(ar, B, w); });
  if (rc) return rc;
  if ((rc = encoder_forward(net, in, B, N, w, out_pf, out_keys))) return rc;
  CG_CUDA(ctx, cudaMemcpyAsync(out_T3, w.T3, (size_t)B * 9 * 4, cudaMemcpyDeviceToDevice, ctx->stream));
  CG_CUDA(ctx, cudaMemcpyAsync(out_T64, w.T64, (size_t)B * 4096 * 4, cudaMemcpyDeviceToDevice, ctx->stream));
  return CG_OK;
}

extern "C" int cg_nunocs_forward_dev(cg_net *net, const float *x, int N, int bins, float *out_coords,
                                     float *out_conf_z, int32_t *out_bins) {
  if (!net) return CG_EINVAL;
  return seg_forward_impl(net, x, 1, N, nullptr, bins, out_coords, out_conf_z, out_bins);
}

extern "C" int cg_nunocs_forward_host(cg_net *net, const float *x_host, int N, int bins, float *out_coords,
                                      float *out_conf_z, int32_t *out_bins) {
  if (!net) return CG_EINVAL;
  cg_ctx *ctx = net->ctx;
  CG_REQUIRE(ctx, x_host && N > 0 && out_coords, "nunocs_host: bad arguments");
  const float *d_x; float *d_c, *d_z; int32_t *d_b;
  return cg_io_stage(ctx, [&](cg_io_pieces &io) {
    d_x = io.in(x_host, (size_t)N * 6);
    d_c = io.out(out_coords, (size_t)N * 3);
    d_z = io.out(out_conf_z, N);
    d_b = io.out(out_bins, (size_t)N * 3);
  }, [&] { return cg_nunocs_forward_dev(net, d_x, N, bins, d_c, d_z, d_b); });
}

// Objects per pass of the batched NUNOCS forward: whole objects up to CG_NUNOCS_MANY_PASS_POINTS points.  Below 64
// points a cloud's point-wise layers take another kernel at B = 1 than in a batch (cg_linear_launch), so one object.
static int nunocs_pass_objects(int B, int N) {
  if (N < 64) return 1;
  long long p = CG_NUNOCS_MANY_PASS_POINTS / N;
  if (p > CHUNK_B) p = CHUNK_B;
  if (p > B) p = B;
  return p < 1 ? 1 : (int)p;
}

extern "C" int cg_nunocs_forward_many_dev(cg_net *net, const float *x, int B, int N, int bins, float *out_coords,
                                          float *out_conf_z, int32_t *out_bins) {
  if (!net) return CG_EINVAL;
  cg_ctx *ctx = net->ctx;
  CG_REQUIRE(ctx, x && N > 0 && out_coords, "nunocs_many: bad arguments");
  CG_REQUIRE(ctx, B >= 1 && B <= CG_NUNOCS_MANY_MAX_B, "nunocs_many: 1 <= B <= CG_NUNOCS_MANY_MAX_B");
  CG_REQUIRE(ctx, net->kind == CG_NET_SEG && bins > 0 && bins * 3 == net->n_out, "nunocs_many: n_out != 3*bins");
  const int per = nunocs_pass_objects(B, N);
  for (int b0 = 0; b0 < B; b0 += per) {
    const int nb = B - b0 < per ? B - b0 : per;
    const size_t p0 = (size_t)b0 * N;
    int rc = seg_forward_impl(net, x + p0 * 6, nb, N, nullptr, bins, out_coords + p0 * 3,
                              out_conf_z ? out_conf_z + p0 : nullptr, out_bins ? out_bins + p0 * 3 : nullptr,
                              CG_FC_FEW_ROWS);   // the kernel and the sums a single cloud gets
    if (rc) return rc;
  }
  return CG_OK;
}

extern "C" int cg_nunocs_forward_many_host(cg_net *net, const float *x_host, int B, int N, int bins, float *out_coords,
                                           float *out_conf_z, int32_t *out_bins) {
  if (!net) return CG_EINVAL;
  cg_ctx *ctx = net->ctx;
  CG_REQUIRE(ctx, x_host && N > 0 && out_coords, "nunocs_many_host: bad arguments");
  CG_REQUIRE(ctx, B >= 1 && B <= CG_NUNOCS_MANY_MAX_B, "nunocs_many_host: 1 <= B <= CG_NUNOCS_MANY_MAX_B");
  const size_t P = (size_t)B * N;
  const float *d_x; float *d_c, *d_z; int32_t *d_b;
  return cg_io_stage(ctx, [&](cg_io_pieces &io) {
    d_x = io.in(x_host, P * 6);
    d_c = io.out(out_coords, P * 3);
    d_z = io.out(out_conf_z, P);
    d_b = io.out(out_bins, P * 3);
  }, [&] { return cg_nunocs_forward_many_dev(net, d_x, B, N, bins, d_c, d_z, d_b); });
}

/*
 * catgrasp_b200.h -- C ABI of libcatgrasp_b200.so (sm_90a, H100).
 *
 * This is the drop-in boundary for CaTGrasp's per-scene grasp-scoring hot
 * path and the per-pick stages around it (segmentation, NUNOCS and its 9-DoF
 * pose search, the grasp samplers and filters, affordance transfer, ranking).
 * Every entry point is `extern "C"`, takes plain pointers and sizes,
 * returns an int status (0 = ok, negative = CG_E*), and never calls exit().
 * Each entry cites the reference interface (file:line under the reference
 * checkout) that it replaces.
 *
 * Pointer conventions
 *   *_host : the function takes HOST buffers, performs H2D, compute and D2H
 *            itself on the context stream and returns after the result is in
 *            the host output buffer (the reference-facing, blocking call).
 *   *_dev  : all data pointers are DEVICE pointers owned by the caller
 *            (e.g. torch allocations), except parameters marked host; the
 *            call enqueues work on the context stream and returns without
 *            synchronising.
 * A parameter marked host or device is read there whatever the entry's name.
 * Row-major everywhere.  Poses are 4x4 row-major.
 */
#ifndef CATGRASP_B200_H
#define CATGRASP_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- status codes ------------------------------------------------------ */
#define CG_OK            0
#define CG_EINVAL       -1   /* bad argument / shape (reference: printf+exit(1),
                                my_cpp/collision_manager.cpp:17-27,57-61)     */
#define CG_ECUDA        -2   /* CUDA runtime error, see cg_last_error()       */
#define CG_ENOMEM       -3
#define CG_EUNSUPPORTED -4

typedef struct cg_ctx cg_ctx;   /* one per device; owns stream + workspace    */
typedef struct cg_net cg_net;   /* folded PointNetCls / PointNetSeg weights   */
typedef struct cg_sdf cg_sdf;   /* one Sdf3D grid resident in HBM             */

/* ---- context ----------------------------------------------------------- */
int         cg_ctx_create(int device, cg_ctx **out);
void        cg_ctx_destroy(cg_ctx *ctx);
/* Enqueue on a caller-owned cudaStream_t (passed as void*).  NULL means the
 * CUDA legacy default stream (stream 0), NOT the context's own stream; a new
 * context starts on its own non-blocking stream (cg_ctx_use_own_stream).      */
int         cg_ctx_set_stream(cg_ctx *ctx, void *cuda_stream);
int         cg_ctx_use_own_stream(cg_ctx *ctx);
int         cg_ctx_synchronize(cg_ctx *ctx);
const char *cg_last_error(cg_ctx *ctx);
const char *cg_version(void);
/* number of kernels this library launched on ctx since creation / reset.   */
int64_t     cg_ctx_launch_count(cg_ctx *ctx);
void        cg_ctx_reset_launch_count(cg_ctx *ctx);
/* GEMM engine of the fused shared-MLP "trunk":
 *   0 = fp32 SIMT (exact-order reference engine)
 *   1 = wgmma, bf16 hi/lo x hi/lo, 3 passes (near-fp32)
 *   2 = wgmma, 128->1024 layer with fp16 hi/lo activations x one fp16 weight
 *       term, 2 passes
 *   3 = wgmma, the 128->1024 layer as ONE fp16 x fp16 pass               [default]
 *   Every engine keeps grasp scores within the 1e-4 tolerance of the fp32
 *   reference (tests/test_gpu_parity.py).
 *   (2 and 3 fall back to 1 for a net whose folded weights exceed the fp16 range) */
int         cg_ctx_set_engine(cg_ctx *ctx, int engine);
int         cg_ctx_get_engine(cg_ctx *ctx);
/* Engines 2 and 3 clamp the 128->1024 layer's inputs to the fp16 range (65504).
 * *out = 1 if a clamp happened on this context since the previous call (the
 * flag is cleared); the caller should then re-run on engine 1.  Synchronises
 * the context's stream.                                                      */
int         cg_ctx_fp16_overflow(cg_ctx *ctx, int *out);
/* Optional in-stream timing of the dominant kernel (the fused shared-MLP+max
 * "trunk"): when enabled every trunk launch is bracketed by a CUDA event pair
 * on the launching stream; cg_ctx_profile_read() synchronises those events and
 * returns the summed duration and the launch count, then clears the list.   */
int         cg_ctx_profile(cg_ctx *ctx, int enable);
int         cg_ctx_profile_read(cg_ctx *ctx, double *ms_total, int64_t *launches);

/* ---- networks ----------------------------------------------------------
 * Replaces: pointnet2.py:275-299 (PointNetCls), :302-329 (PointNetSeg),
 * loaded through Utils.py:135-148 (load_model).  The host side folds every
 * BatchNorm into the preceding conv/linear and packs fp32 weights in the
 * order documented in catgrasp_b200/weights.py; `blob` is that packing.
 *   kind: 0 = PointNetCls(n_in=6, n_out), 1 = PointNetSeg(n_in=6, n_out)     */
#define CG_NET_CLS 0
#define CG_NET_SEG 1
int  cg_net_create(cg_ctx *ctx, int kind, int n_out,
                   const float *blob_host, size_t blob_floats, cg_net **out);
void cg_net_destroy(cg_net *net);
size_t cg_net_blob_floats(int kind, int n_out);

/* Grasp-Q forward over B candidates.
 * Replaces: predicter.py:67-94 (GraspPredicter.predict_batch) incl. the
 * per-candidate GraspDataset.transform (dataset_grasp.py:63-91) which is
 * fused into the first kernel: for candidate b, point n
 *     id   = ids[b*N+n]                       (host-drawn numpy RNG indices)
 *     xyz  = inv(pose_b)     * cloud_xyz[id]  (float64, like the reference)
 *     nrm  = inv(pose_b[:3,:3]) * cloud_nrm[id]
 *     in6  = ([xyz,nrm] - mean) / (std + 1e-15)   (if mean/std != NULL)
 * then PointNetCls forward + softmax in fp32.
 *   cloud_xyz, cloud_nrm : (M,3) float64      poses : (B,4,4) float64
 *   ids : (B,N) int32 in [0,M)                mean,std : (6,) float64 or NULL
 *   out_probs : (B,n_out) float32             out_label : (B,) int32 or NULL
 * out_label[b] is the argmax of the float32 probabilities written to
 * out_probs[b], the lowest class winning a tie (predicter.py:86-89 takes
 * the argmax after the softmax): logits too close for expf to separate give
 * equal probabilities and the lower class.
 */
int cg_graspq_forward_host(cg_net *net,
                           const double *cloud_xyz, const double *cloud_nrm, int M,
                           const double *poses, int B,
                           const int32_t *ids, int N,
                           const double *mean, const double *std,
                           float *out_probs, int32_t *out_label);
int cg_graspq_forward_dev(cg_net *net,
                          const double *cloud_xyz, const double *cloud_nrm, int M,
                          const double *poses, int B,
                          const int32_t *ids, int N,
                          const double *mean, const double *std,
                          float *out_probs, int32_t *out_label);

/* cg_graspq_forward_dev for the candidates of several objects in one call
 * (GraspPredicter.score_many).  cloud_xyz, cloud_nrm: the objects' clouds
 * concatenated, (M_total,3); poses (B_total,4,4); ids (B_total,N) already
 * rebased to rows of the concatenation.  fc_groups (HOST, n_groups entries of
 * 1 .. CG_GRASPQ_CHUNK_B rows, summing to B_total): consecutive row groups,
 * each the candidates one cg_graspq_forward_dev launch covers; every group's
 * FC layers take the kernel that call would take (the row count selects it),
 * so row b of the result equals, bit for bit, the row of the call on its group
 * alone.  The trunks run over whole groups in passes of at most
 * CG_GRASPQ_CHUNK_B candidates; groups of at most 8 rows share one FC launch
 * per layer.  out_probs (B_total,n_out), out_label (B_total,) or NULL.       */
#define CG_GRASPQ_CHUNK_B 16384
int cg_graspq_forward_many_dev(cg_net *net,
                               const double *cloud_xyz, const double *cloud_nrm, int M_total,
                               const double *poses, int B_total,
                               const int32_t *ids, int N,
                               const double *mean, const double *std,
                               const int32_t *fc_groups /* host */, int n_groups,
                               float *out_probs, int32_t *out_label);

/* The per-candidate point-subset draw of GraspDataset.transform
 * (dataset_grasp.py:72-73: np.random.choice(np.arange(M), size=n_pts,
 * replace=(M < n_pts)) from the GLOBAL legacy numpy generator, once per
 * candidate, in candidate order).
 *
 * cg_host_legacy_choice (HOST function, no GPU work): the same draw, bit for
 * bit, without the Python-level call per candidate.  key[624] / *pos are the
 * MT19937 state of np.random.get_state() (fields 1 and 2); both are advanced
 * exactly as numpy would advance them, so np.random.set_state() afterwards
 * leaves the host program on the reference's random stream.  The stream walk
 * is sequential (AVX-512 / AVX2 / scalar, picked at load time); the
 * permutations are replayed on `nthreads` host threads (<= 0: one per core,
 * at most 12).  out: (count, n_pts) int32.
 * cg_host_rng_isa(level) caps the instruction set (0 scalar, 1 AVX2, 2 AVX-512,
 * -1 best available) and returns the level in use -- a test hook.
 *
 * cg_draw_ids_dev (opt-in, NOT the reference's numbers): a counter-based draw
 * on the device with the same distribution -- n_pts distinct uniform indices
 * (keyed Feistel permutation of [0,M), cycle-walked) when M >= n_pts, n_pts
 * independent uniform indices when M < n_pts.  Candidate b uses the key
 * (seed, first_candidate + b), so shards of one candidate list draw the same
 * subsets as the unsharded call.  out_ids: (count, n_pts) int32 on device.   */
int cg_host_legacy_choice(uint32_t *key, int32_t *pos, int64_t M, int32_t n_pts,
                          int32_t count, int32_t *out, int32_t nthreads);
/* advance the generator over `count` candidates without producing their indices (sharded scoring) */
int cg_host_legacy_skip(uint32_t *key, int32_t *pos, int64_t M, int32_t n_pts, int32_t count);
int cg_host_rng_isa(int level);
int cg_draw_ids_dev(cg_ctx *ctx, int M, int n_pts, int count, uint64_t seed,
                    int64_t first_candidate, int32_t *out_ids);
/* cg_draw_ids_dev for n_obj objects in one launch.  Object o owns output rows
 * row_offsets[o] .. row_offsets[o+1]-1 (row_offsets: n_obj+1 ascending int64,
 * row_offsets[0] = 0, row_offsets[n_obj] = rows; an object may own none);
 * its rows are cg_draw_ids_dev(M[o], n_pts, its row count, seed[o],
 * first_candidate = 0) plus base[o] (the object's first row in a
 * concatenation of the clouds).  M, seed, row_offsets, base: device arrays.
 * out_ids: (rows, n_pts) int32 on device.                                    */
int cg_draw_ids_many_dev(cg_ctx *ctx, int n_obj, const int32_t *M, const uint64_t *seed,
                         const int64_t *row_offsets, const int32_t *base, int n_pts, int rows,
                         int32_t *out_ids);

/* PointNetCls / PointNetSeg forward on an already materialised input tensor
 * x : (B,N,6) float32 (device).  Replaces pointnet2.py:289-299 / :316-329.
 *   cls: out_logits (B,n_out) and/or out_probs (B,n_out) (either may be NULL)
 *   seg: out_logits (B,N,n_out) float32                                     */
int cg_cls_forward_dev(cg_net *net, const float *x, int B, int N,
                       float *out_logits, float *out_probs);
int cg_seg_forward_dev(cg_net *net, const float *x, int B, int N,
                       float *out_logits);
/* Encoder intermediates -- a test hook (device pointers, enqueued on the
 * context stream).  Runs the PointNet encoder of either net kind on B <= 16384
 * candidates exactly as the forward entries do and copies out, per stage:
 *   out_keys (3,B,1024) uint32: the max-pool outputs of the STN3d, STNkd and
 *            encoder trunks as order-preserving keys (the fp32 bits b map to
 *            b | 0x80000000 when b's sign bit is clear, else to ~b)
 *   out_T3 (B,9), out_T64 (B,4096) float32: the two feature transforms
 *   out_pf (B,N,64) float32: the point feature after T64, or NULL
 * Input: x (B,N,6) float32, or x == NULL and the fused grasp-Q form of
 * cg_graspq_forward_dev (ids may be NULL when N <= M; mean/std both or neither). */
int cg_encoder_probe_dev(cg_net *net, const float *x,
                         const double *cloud_xyz, const double *cloud_nrm, int M,
                         const double *poses, const int32_t *ids,
                         const double *mean, const double *std, int B, int N,
                         uint32_t *out_keys, float *out_T3, float *out_T64,
                         float *out_pf);
/* NUNOCS post-processing, predicter.py:144-150: logits (P, 3*bins) ->
 * coords (P,3) = argmax*(1/bins) - 0.5 and conf_z (P,) = softmax prob of the
 * z-axis argmax bin.  Fused variant of cg_seg_forward for B=1.              */
int cg_nunocs_forward_host(cg_net *net, const float *x_host, int N, int bins,
                           float *out_coords, float *out_conf_z, int32_t *out_bins);
int cg_nunocs_forward_dev(cg_net *net, const float *x, int N, int bins,
                          float *out_coords, float *out_conf_z, int32_t *out_bins);
/* The same for B objects of N points each (replaces predicter.py:136-150 once per object of a list):
 * x (B,N,6) -> coords (B,N,3), conf_z (B,N), bins (B,N,3).  Object b's outputs are those of
 * cg_nunocs_forward_dev on x[b], bit for bit, on every engine: the per-cloud FC layers run in groups of at
 * most 8 clouds (the few-row kernel a single cloud takes), and N < 64 runs one object per pass.  The forward
 * runs in passes of at most CG_NUNOCS_MANY_PASS_POINTS points (whole objects); CG_EINVAL before any launch
 * unless 1 <= B <= CG_NUNOCS_MANY_MAX_B and N > 0.  _dev runs on the context stream and does not synchronise. */
#define CG_NUNOCS_MANY_MAX_B 65535
#define CG_NUNOCS_MANY_PASS_POINTS (1 << 18)
int cg_nunocs_forward_many_host(cg_net *net, const float *x_host, int B, int N, int bins,
                                float *out_coords, float *out_conf_z, int32_t *out_bins);
int cg_nunocs_forward_many_dev(cg_net *net, const float *x, int B, int N, int bins,
                               float *out_coords, float *out_conf_z, int32_t *out_bins);

/* ---- SDF grid ----------------------------------------------------------
 * Replaces: meshpy/meshpy/sdf.py:217-289 (Sdf3D), sdf_file.py:59-87.
 * grid is data[i][j][k] row-major (k fastest) float32; grid coordinate of a
 * point x (SDF frame) is (x - origin) / resolution (sdf.py:252-264).        */
int  cg_sdf_create(cg_ctx *ctx, const float *grid_host, int nx, int ny, int nz,
                   const float origin[3], float resolution, cg_sdf **out);
void cg_sdf_destroy(cg_sdf *sdf);
/* Point-wise signed distance lookups at GRID coordinates (P,3) float32.
 *   mode 0: trilinear, sdf.py:292-343 (_signed_distance)
 *   mode 1: nearest cell with clamp, sdf.py:345-359 (_signed_distance_batch) */
#define CG_SDF_TRILINEAR 0
#define CG_SDF_NEAREST   1
int cg_sdf_lookup_dev(cg_sdf *sdf, const float *grid_coords, int P, int mode,
                      float *out_sd);

/* ---- SDF grid from a triangle mesh ---------------------------------------
 * Replaces: make_sdf.py:30-36 (the external SDFGen binary run on a gripper
 * mesh) and the .sdf files it writes, sdf_file.py:59-87.
 * vertices (nv,3) float64 and faces (nf,3) int32 are HOST arrays of a closed
 * mesh; the call is blocking.  Grid geometry, per axis a:
 *   n_a      = ceil((max_a - min_a) / resolution - 1e-4) + 1 + 2 * padding
 *   origin_a = float32(min_a - padding * resolution)   (float64 arithmetic)
 * Node (i,j,k) lies at origin + (i,j,k) * resolution (float64 from the float32
 * values).  Each value is the exact distance from the node to the nearest
 * triangle, computed in float64 and rounded once to float32, negative inside
 * (ray parity along x).  Errors (CG_EINVAL, no handle created): nv or nf <= 0,
 * an index out of range, a non-finite vertex, resolution <= 0 or not finite,
 * padding < 0, more than 2048 nodes along an axis, a mesh that is not closed.
 * CG_ENOMEM when the device is out of memory.                              */
int cg_sdf_from_mesh(cg_ctx *ctx, const double *vertices, int nv, const int32_t *faces, int nf,
                     float resolution, int padding, cg_sdf **out);
/* dims (nx,ny,nz), origin and resolution of a grid (sdf_file.py:59-87 header) */
int cg_sdf_geometry(const cg_sdf *sdf, int dims[3], float origin[3], float *resolution);
/* copy the grid to host memory, data[i][j][k] (k fastest); blocking          */
int cg_sdf_download(cg_sdf *sdf, float *grid_host);

/* ---- collision filter --------------------------------------------------
 * Replaces: my_cpp/common.cpp:156-321 (filterGraspPose) with the FCL
 * mesh-vs-octree test (collision_manager.cpp:93-111) substituted by the
 * gripper-SDF predicate of sdf.py:377-389 (is_any_points_inside, nearest
 * mode) or its trilinear form (sdf.py:292-343).  IK (common.cpp:214-226) is
 * NOT evaluated here: cg_filter_apply_ik_dev (below) applies it to these
 * outputs.
 *   grasp_poses (G,4,4), symmetry_tfs (S,4,4), the five 4x4 matrices:
 *       float32 row-major (the reference narrows float64 -> float at the
 *       pybind boundary, common.h:51,60).
 *   open_pts (P1,3), enclosed_pts (P2,3): float32 camera-frame points
 *       (gripper_collision_pts / gripper_enclosed_collision_pts).
 *   Outputs are indexed by pair q = i*S + j, i.e. DETERMINISTIC order
 *   (the reference's is thread-arrival order, common.cpp:303-313):
 *   out_status[q] : 0 accepted, 1 rejected by approach direction,
 *                   3 rejected by collision (2 is reserved for IK)
 *   out_offset[q] : index 0..4 of the winning lateral offset
 *                   (0,+1mm,-1mm,+2mm,-2mm; common.cpp:255-262), -1 if none
 *   out_poses[q]  : (4,4) float32 grasp_in_cam shifted by the winning offset,
 *                   all-zero when rejected (common.cpp:289-293)              */
#define CG_ST_ACCEPT    0
#define CG_ST_REJ_DIR   1
#define CG_ST_REJ_IK    2
#define CG_ST_REJ_COLL  3   /* collision (with split_coll_status and no pose adjustment: the OPEN gripper hits the object) */
#define CG_ST_REJ_COLL_ENCL 4   /* split_coll_status only: the open gripper is free, the ENCLOSED gripper hits the background */
typedef struct cg_filter_params {
  float nocs_pose[16];
  float canonical_to_nocs[16];
  float gripper_in_grasp[16];
  int   filter_approach_dir_face_camera;
  int   adjust_collision_pose;
  int   sdf_mode;          /* CG_SDF_TRILINEAR or CG_SDF_NEAREST */
  float sdf_margin;        /* a scene point collides iff sd < sdf_margin (metres).  0 = the SDF predicate of
                              meshpy/sdf.py:377-389 (point inside the gripper solid).  octo_resolution*sqrt(3)/2 makes
                              the verdict conservative w.r.t. the reference's mesh-vs-voxel test
                              (my_cpp/collision_manager.cpp:93-111): every occupied voxel cube of side
                              octo_resolution that can touch the gripper surface has its generating point within
                              that distance of the surface.                                                        */
  int   split_coll_status; /* != 0 and adjust_collision_pose == 0: report which of the reference's two tests rejected a
                              pose (CG_ST_REJ_COLL = open gripper vs object points, common.cpp:231-238;
                              CG_ST_REJ_COLL_ENCL = enclosed gripper vs background, :241-248) -- the verbose counters
                              n_open_gripper_rej / n_close_gripper_rej.  Costs the reference's scan order (open first)
                              instead of the faster background-sample-first order.  With pose adjustment the reference
                              itself counts every collision rejection as "open" (:290-294): always CG_ST_REJ_COLL.     */
} cg_filter_params;

int cg_filter_grasp_pose_host(cg_ctx *ctx, const cg_filter_params *prm,
                              const float *grasp_poses, int G,
                              const float *symmetry_tfs, int S,
                              cg_sdf *sdf_open, const float *open_pts, int P1,
                              cg_sdf *sdf_enclosed, const float *enclosed_pts, int P2,
                              uint8_t *out_status, int8_t *out_offset, float *out_poses);
int cg_filter_grasp_pose_dev(cg_ctx *ctx, const cg_filter_params *prm /* host */,
                             const float *grasp_poses, int G,
                             const float *symmetry_tfs, int S,
                             cg_sdf *sdf_open, const float *open_pts, int P1,
                             cg_sdf *sdf_enclosed, const float *enclosed_pts, int P2,
                             uint8_t *out_status, int8_t *out_offset, float *out_poses);

/* ---- IK feasibility (KUKA iiwa14) ----------------------------------------
 * Replaces: my_cpp/common.cpp:9-72 (get_ik_within_limits over the generated
 * ikfast solver, free joint 2 fixed at 0) and its use in filterGraspPose
 * (:214-226).  A closed-form float64 solver of the same chain (DESIGN.md X5).
 *
 * cg_iiwa14_ik_dev: ee_in_base (Q,4,4) float32 (device), upper / lower: HOST
 *   arrays of 7 doubles.  out_count[i] (int8) = number of solutions with
 *   lower[k] <= q[k] <= upper[k] for all 7 joints (0 for a non-finite pose and
 *   whenever lower > upper).  out_solutions (Q,8,7) float64 or NULL: every
 *   solution regardless of the limits, slot 4*s + 2*e + w with
 *     s: 0 = q0 towards the wrist centre, 1 = q0 + pi (shoulder flip)
 *     e: 0 = q3 >= 0, 1 = q3 < 0 (elbow)
 *     w: 0 = q5 >= 0 (or the lumped singular wrist), 1 = flipped wrist,
 *   angles in [-pi, pi], q2 = 0, unused slots NaN.  Q = 0 is a no-op.
 *
 * cg_filter_apply_ik_dev: the IK test of filterGraspPose as a pass over the
 *   outputs of cg_filter_grasp_pose_dev (same prm, poses, symmetries; same
 *   stream, after it).  For every pair whose status is not CG_ST_REJ_DIR it
 *   composes ee_in_base = cam_in_world * grasp_in_cam * ee_in_grasp from the
 *   UN-shifted pose in the filter's float32 order and, when no solution is
 *   within the limits, sets status CG_ST_REJ_IK, offset -1 and an all-zero pose
 *   (IK precedes the collision tests in the reference).                      */
typedef struct cg_ik_params {
  float  cam_in_world[16];
  float  ee_in_grasp[16];
  double upper[7];
  double lower[7];
} cg_ik_params;
int cg_iiwa14_ik_dev(cg_ctx *ctx, const float *ee_in_base, int Q,
                     const double upper[7] /* host */, const double lower[7] /* host */,
                     int8_t *out_count, double *out_solutions);
int cg_filter_apply_ik_dev(cg_ctx *ctx, const cg_filter_params *prm /* host */,
                           const float *grasp_poses, int G,
                           const float *symmetry_tfs, int S,
                           const cg_ik_params *ik /* host */,
                           uint8_t *status, int8_t *offset, float *out_poses);

/* ---- occupancy / occlusion grid from a depth scan ----------------------------
 * Replaces: my_cpp/common.cpp:324-431 (makeOccupancyGridFromCloudScan; the K
 * argument of the reference is computed with but never influences its output).
 * Samples form a regular grid over the padded bounding box of pts:
 *   dims[a] = int((max_a + 0.005 - (min_a - 0.005)) / resolution), origin[a] = min_a - 0.005   (float arithmetic)
 * out_flags[(xi*ny + yi)*nz + zi] = 1 iff the first occupied cell on the ray origin -> sample is not farther than
 * the sample (the reference pushes exactly these samples, in thread-arrival order; here raster order).            */
int cg_occupancy_grid_geometry(const float *pts_host, int P, float resolution, int dims[3], float origin[3]);
int cg_occupancy_from_scan_host(cg_ctx *ctx, const float *pts_host, int P, float resolution,
                                unsigned char *out_flags_host);

/* ---- NUNOCS 9-DoF RANSAC hypothesis scoring -------------------------------------
 * Replaces: aligning.py:36-81 (estimate9DTransform_worker) for H hypotheses at once.
 *   source, target (N,3) float64 correspondences; ids (H,4) int32 = the 4-subsets (host numpy RNG, aligning.py:91-97)
 *   The 4-point affine is cv2.estimateAffine3D's: the exact solution when the float32-narrowed points are affinely
 *   independent, else the minimum-norm least-squares one (singular values <= 6 DBL_EPSILON * their sum dropped).
 *   The minimum-norm solve runs when the LU solve meets a pivot < 1e-12; a system that is nonsingular by that test
 *   but whose smallest singular value is under cv2's cut (large coordinates; not for points in the unit cube)
 *   keeps the LU answer where cv2 would truncate.
 *   out_valid[h] = hypothesis passed the scale / singular-value / det / max_dimensions gates
 *   out_ratio[h] = inlier ratio at pass_threshold, out_T[h] = (4,4) float64 transform R diag(scales) | t;
 *   where out_valid[h] = 0: out_ratio[h] = 0 and out_T[h] is all zeros                                              */
int cg_ransac9d_host(cg_ctx *ctx, const double *source, const double *target, int N, const int32_t *ids, int H,
                     double pass_threshold, const double min_scale[3], const double max_scale[3],
                     const double *max_dims, double *out_ratio, double *out_T, unsigned char *out_valid);
/* The whole NUNOCS pose search in one launch on device buffers (replaces aligning.py:83-119 twice and
 * predicter.py:152-172): the same scoring as cg_ransac9d_host for n_thr (1 or 2) thresholds, each with its own H
 * subsets (ids (n_thr*H,4): rows t*H .. t*H+H-1 belong to thresholds[t]), then the selection on the device:
 *   per threshold, the winner = the first maximum of the inlier count among valid hypotheses (the host's
 *   keep[argmax(ratio[keep])]); its T is the scoring pass's, bit for bit cg_ransac9d_host's T[winner];
 *   the pose = the first threshold whose winner has det(T[:3,:3]) >= 0 and the largest ratio
 *   count(|T src - tgt| <= ratio_threshold) / N, strictly above the previous best (starting at 0).
 * out_record (n_thr*19 + 18 float64, integers stored exactly):
 *   per threshold t at t*19: [winner h or -1, its count at thresholds[t], T (4x4, zeros if none),
 *                             its count at ratio_threshold]
 *   then [chosen threshold or -1, pose (4x4, zeros if none), best_ratio].
 * Runs on the context stream and does not synchronise.                                                         */
int cg_ransac9d_pose_dev(cg_ctx *ctx, const double *source, const double *target, int N, const int32_t *ids, int H,
                         const double *thresholds /* host */, int n_thr, const double min_scale[3] /* host */,
                         const double max_scale[3] /* host */, const double *max_dims /* host */,
                         double ratio_threshold, double *out_record);
/* cg_ransac9d_pose_dev for B objects of N correspondences each (predicter.py:152-172 once per object of a list):
 * source, target (B,N,3), ids (B, n_thr*H, 4) -- object b's rows as cg_ransac9d_pose_dev's ids --, out_records
 * (B, n_thr*19 + 18): object b's record as cg_ransac9d_pose_dev writes it for source[b], target[b], ids[b], bit
 * for bit.  One CTA per (object, threshold, hypothesis); the winner keys, the completion counter and the last
 * CTA's choice are per object.  At most CG_RANSAC_MANY_PASS_PAIRS CTAs per launch (whole objects; one object
 * when n_thr*H is larger), the launches in object order.  CG_EINVAL before any launch unless
 * 1 <= B <= CG_NUNOCS_MANY_MAX_B.  Runs on the context stream and does not synchronise.                        */
#define CG_RANSAC_MANY_PASS_PAIRS (1 << 20)
int cg_ransac9d_pose_many_dev(cg_ctx *ctx, const double *source, const double *target, int B, int N,
                              const int32_t *ids, int H, const double *thresholds /* host */, int n_thr,
                              const double min_scale[3] /* host */, const double max_scale[3] /* host */,
                              const double *max_dims /* host */, double ratio_threshold, double *out_records);

/* The same two entries with aligning.py:68-79's evaluation (use_kdtree_for_eval=True, kdtree_eval_resolution =
 * resolution) in place of the residual count; the gates and the selection rules are unchanged.  For a hypothesis
 * that passes the gates, with src_t = T [source, 1] and thr its threshold:
 *   count = #{i : some voxel mean of target lies within thr of src_t[i]} + #{j : some voxel mean of src_t lies within
 *           thr of target[j]}   (cKDTree's `distance <= thr` on both voxel-thinned clouds),
 *   out_ratio = count / (2N); in the record of the pose entry, each winner's count is out of 2N (its count at
 *   ratio_threshold is still the residual count out of N, as in predict).
 * Voxels are cg_voxel_down_sample_dev's: cell floor((p - (min_bound - r*0.5)) / r), the mean of its points summed in
 * ascending index.  src_t = ((T00 x + T01 y) + T02 z) + T03 per row and distances (dx*dx + dy*dy) + dz*dz, then
 * sqrt, all float64 without FMA, so the counts are a function of T and the inputs alone.
 * CG_EINVAL before any launch: N > CG_RANSAC_KD_MAX_N, or resolution not positive and finite.  CG_EINVAL after the
 * launch: the target, or a transformed source, spans 2^21 or more voxels on an axis or is not finite.
 * Synchronisation: both entries synchronise the stream three times -- building the target's cg_cloud_index (its
 * bounds, then its cell count) and reading the kernel's error word at the end.  The device workspace holds about
 * 100 N bytes per CTA of the launch (at most 1 GiB in all, or one CTA per SM if that is larger).                   */
#define CG_RANSAC_KD_MAX_N 65536
int cg_ransac9d_kdtree_host(cg_ctx *ctx, const double *source, const double *target, int N, const int32_t *ids, int H,
                            double pass_threshold, const double min_scale[3], const double max_scale[3],
                            const double *max_dims, double resolution, double *out_ratio, double *out_T,
                            unsigned char *out_valid);
int cg_ransac9d_kdtree_pose_dev(cg_ctx *ctx, const double *source, const double *target, int N, const int32_t *ids,
                                int H, const double *thresholds /* host */, int n_thr,
                                const double min_scale[3] /* host */, const double max_scale[3] /* host */,
                                const double *max_dims /* host */, double ratio_threshold, double resolution,
                                double *out_record);

/* ---- Cone pose enumeration (device pointers, float64 like the reference's numpy) ----------
 * Replaces: dexnet/grasping/grasp_sampler.py:266-286 (PointConeGraspSampler.sample_one_surface_point: the
 *   R0 / R0 @ R_sphere @ R_inplane x approach-depth loops, Utils.py:172-179 normalizeRotation) and :191-203
 *   (center_ob_between_gripper).  Its C++ twin my_cpp/common.cpp:111-153 (augmentGraspPoses) is uncalled.
 *   surface_pts (S,3), R0 (S,9 row-major: columns approach / major / minor, computed on the host, :262),
 *   R_sphere (NS,9), R_inplane (NI,9), depths (ND) = np.arange(0, hand_depth, approach_step)
 *   out_poses64 (P,16) row-major 4x4, P = S * (1 + NS*NI) * ND, ordered (surface point, rotation, depth) like the
 *   reference's list; out_poses32 (P,16) or NULL = the same poses narrowed to float32 for cg_filter_grasp_pose_dev.
 *   CG_EINVAL, before any launch: P >= 2^31, or NS, NI > 0 with R_sphere or R_inplane NULL.                         */
int cg_cone_poses_dev(cg_ctx *ctx, const double *surface_pts, const double *R0, int S, const double *R_sphere, int NS,
                      const double *R_inplane, int NI, const double *depths, int ND, double init_bite,
                      double *out_poses64, float *out_poses32);
/* grasp_sampler.py:191-203: shift every pose along its y axis to the middle of the object's extent (pts (M,3) float64,
 * camera frame) in the grasp frame; poses are updated in place (poses32 may be NULL).  M = 0 is CG_EINVAL; P = 0
 * returns CG_OK without work.                                                                                        */
int cg_center_grasps_dev(cg_ctx *ctx, double *poses64, float *poses32, int P, const double *pts, int M);

/* ---- Affordance transfer per grasp (device pointers, float64) --------------------------------
 * Replaces: run_grasp_simulation.py:50-73 (compute_grasp_affordance_worker) + pybullet_env/env_grasp.py:243-283
 *   (get_finger_contact_area) for G grasps at once.
 *   cam_in_finger (G,16) = inv(finger_mesh_in_grasp) * inv(grasp_in_cam) per grasp (row-major 4x4, :52)
 *   pts, nrm (P,3): the canonical cloud and normals in the camera frame; affordance (P): score of each point's nearest
 *   canonical point (:62-63, gathered once per object on the host)
 *   finger_boxes (F,4) = x min, x max, z min, z max of each finger mesh (:252); grip_dirs (F) = +1 / -1 for a finger closing
 *   along +y / -y (:261-266); 1 <= F <= 4
 *   surface_tol: a point is in the patch when |y - extreme y| <= surface_tol; a negative or NaN tolerance leaves every
 *   patch empty, which drops the finger (:268-269) without reading a normal
 *   out_p (G) = p(T|G), NaN where the reference drops the grasp; out_contacts (G,4) = contact-patch sizes per finger
 *   (0 for a dropped finger).                                                                                          */
int cg_grasp_affordance_dev(cg_ctx *ctx, const double *cam_in_finger, int G, const double *pts, const double *nrm,
                            const double *affordance, int P, const double *finger_boxes /* host */,
                            const int *grip_dirs /* host */, int F,
                            double surface_tol, double *out_p, int *out_contacts);

/* ---- point-cloud preparation ---- */
/* Replaces the open3d / scipy steps of the per-pick path: Utils.py:239-251 (depth2xyzmap), open3d VoxelDownSample and
 * EstimateNormals (run_grasp_simulation.py:97, :114, :137, :173, :209, :246-247), Utils.py:205-213
 * (correct_pcd_normal_direction), cKDTree.query (:120, :131) and query_ball_point (Utils.py:482-488).
 * Points are float64 (N,3) device arrays.  Distances are d2 = (dx*dx + dy*dy) + dz*dz in float64 without FMA,
 * bit-equal to scipy's; a tie goes to the smaller point index.  No result depends on atomic arrival order.        */
#define CG_CLOUD_MAX_NN 64
typedef struct cg_cloud_index cg_cloud_index;
/* depth (H,W) float32 (depth_is_f64 = 0) or float64 -> out_xyz (H,W,3) float32: x = (u - K[2]) * z / K[0],
 * y = (v - K[5]) * z / K[4] in float64 left to right, then narrowed; depth < 0.1 in the depth's own type gives
 * (0,0,0).  K is a host array of 9 doubles (row-major 3x3).                                                        */
int cg_depth2xyz_dev(cg_ctx *ctx, const void *depth, int depth_is_f64, int H, int W, const double *K /* host */,
                     float *out_xyz);
/* Bins pts (P,3) into cells of size `cell` with origin min_bound - cell/2 (cell = floor((p - origin) / cell)), sorts
 * the points by (cell, index) and builds the ascending cell table.  The index copies the points, so pts may be freed
 * afterwards.  Synchronises the context's stream twice (the bounds, then the cell count).  Fails with CG_EINVAL on a
 * non-finite coordinate or when the cloud spans 2^21 or more cells on an axis.                                     */
int  cg_cloud_index_create(cg_ctx *ctx, const double *pts /* device */, int P, double cell, cg_cloud_index **out);
void cg_cloud_index_destroy(cg_cloud_index *index);
/* P, number of occupied cells (= the voxel count of cg_voxel_down_sample_dev), cell size, origin[3]; any may be NULL */
int  cg_cloud_index_info(const cg_cloud_index *index, int *out_points, int *out_cells, double *out_cell, double *out_origin);
/* open3d VoxelDownSample with voxel_size = the index's cell: one output per occupied cell, in ascending (ix, iy, iz)
 * order; mean = members summed in ascending point index, divided by the count; normals (P,3) or NULL: the summed
 * normal divided by its norm (a zero sum stays zero).  out_pts / out_normals hold cg_cloud_index_info's cell count. */
int  cg_voxel_down_sample_dev(const cg_cloud_index *index, const double *normals, double *out_pts, double *out_normals);
/* cKDTree(indexed points).query(query (Q,3)) restricted to max_dist: out_idx (Q) int32 = nearest point (smallest
 * index on a tie), out_dist = sqrt(d2); -1 / +inf when no point has sqrt(d2) <= max_dist.  Here and in
 * cg_cloud_radius_mask_dev, Q = 0 is a no-op whose pointers may be NULL (an empty torch tensor has no storage).    */
int  cg_cloud_nearest_dev(const cg_cloud_index *index, const double *query, int Q, double max_dist, int32_t *out_idx,
                          double *out_dist);
/* out_mask[i] = 1 when some indexed point has d2 <= r*r (compare_sqrt = 0, query_ball_point's test) or
 * sqrt(d2) <= r (compare_sqrt = 1, the `dists <= R` test on cKDTree.query's distances), else 0.                   */
int  cg_cloud_radius_mask_dev(const cg_cloud_index *index, const double *query, int Q, double r, int compare_sqrt,
                              uint8_t *out_mask);
/* Normals of the indexed points: the max_nn (<= CG_CLOUD_MAX_NN) nearest points with d2 <= radius*radius, ordered
 * by (d2, index) and including the point itself; the unit eigenvector of the smallest eigenvalue of their float64
 * covariance about the mean; (0,0,1) for fewer than 3 neighbours or a zero covariance; then oriented towards
 * view_point (host double[3]) exactly as correct_pcd_normal_direction does (n / (|n| + 1e-10), flipped when the dot
 * product with the unit view direction is < 0).  out_normals (P,3) in the caller's point order; out_nbr (P,max_nn)
 * int32 (neighbours in order, -1 padded) and out_nbr_count (P) may be NULL.                                      */
int  cg_cloud_normals_dev(const cg_cloud_index *index, double radius, int max_nn, const double *view_point /* host */,
                          double *out_normals, int32_t *out_nbr, int32_t *out_nbr_count);

/* ---- mean-shift clustering ---- */
/* sklearn MeanShift(bandwidth, seeds=None, bin_seeding=False, cluster_all=True) up to its labels (predicter.py:332).
 * index: a cg_cloud_index over X built with cell = bandwidth (its origin anchors the fixed point; an ascent step scans
 * at most 4 x 4 x 4 cells), else CG_EINVAL; X (P,3): the same points, float32 (x_is_f64 = 0) or float64, in the dtype every centre is returned in.  P <= 2^21, else
 * CG_EINVAL.  One flat-kernel ascent per point: the set d2 = (dx*dx + dy*dy) + dz*dz <= bandwidth^2 (float64, no
 * FMA), its mean summed in int64 fixed point (order-free; see cg_meanshift.cu), stopping on an empty set, on a step
 * of at most 1e-3 * bandwidth or after max_iter (>= 0) steps.  Outputs, all device memory:
 *   out_seed_centres (P,3), out_seed_counts (P) = final set size (0: empty), out_seed_iters (P) = completed steps;
 *   out_centres (P,3 capacity) = the kept modes, in (count, x, y, z) descending order after sklearn's greedy
 *   suppression of modes within bandwidth; out_n_centres (1) = how many.
 * Labels are the nearest kept centre (cg_cloud_nearest_dev over an index of out_centres).  Never synchronises.     */
int  cg_meanshift_dev(const cg_cloud_index *index, const void *X, int x_is_f64, double bandwidth, int max_iter,
                      void *out_seed_centres, int32_t *out_seed_counts, int32_t *out_seed_iters, void *out_centres,
                      int32_t *out_n_centres);

/* ---- sparse 3-D convolution (spconv 1.x semantics; cg_spconv.cu) ----
 * The layer types of PointGroup's U-Net (PointGroup/model/pointgroup/pointgroup.py): SubMConv3d k3 and k1,
 * SparseConv3d k2 s2 and SparseInverseConv3d k2.  A level is a set of distinct sites (x, y, z), each in [0, 2^21), in
 * ascending (x, y, z) order, z fastest.  Rows are int32 indices into a level; -1 is "absent".  Every output is sized
 * from a row bound the caller gives; the true count is written to a device word, and no entry synchronises.        */
/* coords (N,3) int32, each in [0, 2^21) (not checked) -> the level of its distinct sites: out_vox (N,3 capacity),
 * out_nvox (1) = V, out_p2v (N) = each point's site, out_nbr (N,27): for site v < V and k = 9 kx + 3 ky + kz the site
 * v + (kx-1, ky-1, kz-1) or -1; rows from V on are -1.                                                            */
int  cg_spconv_index_dev(cg_ctx *ctx, const int32_t *coords, int N, int32_t *out_vox, int32_t *out_nvox,
                         int32_t *out_p2v, int32_t *out_nbr);
/* The coarser level of a level with *nvox sites (rows of vox, M >= *nvox) on the spatial shape shape[3] (host): the
 * parents c >> 1 of the sites whose parent index is below (S - 2) / 2 + 1 on every axis (an odd axis drops its last
 * plane).  out_rows bounds the parents: at least min(M, the coarse shape's cell count), else CG_EINVAL.  out_vox
 * (out_rows,3 capacity), out_nvox (1) and out_nbr (out_rows,27) as cg_spconv_index_dev gives them for the parents;
 * out_down (out_rows,8): for parent p and k = 4 kx + 2 ky + kz the child 2 p + (kx, ky, kz) or -1; out_up (M,8): for
 * child c the parent at k = c - 2 parent(c) and -1 at the other seven (all eight -1 for a dropped child).          */
int  cg_spconv_down_dev(cg_ctx *ctx, const int32_t *vox, const int32_t *nvox, int M, const int32_t *shape /* host */,
                        int out_rows, int32_t *out_vox, int32_t *out_nvox, int32_t *out_nbr, int32_t *out_down,
                        int32_t *out_up);
/* Batched levels: the sites of B frames, each on its own spatial shape, in one level.  Key layout: a site (x, y, z)
 * of frame b is the key b << 3w | x << 2w | y << w | z, and a level holds its sites in ascending key order, so frame
 * by frame and, within a frame, in the (x, y, z) order above.  Width rule: w is the smallest width with 2^w >= every
 * frame's shape on every axis, the frame field takes f = bit_length(B - 1) bits, and f + 3w must be <= 63, else
 * CG_EINVAL with a message (a key is never wrapped); B = 1 keeps the one-frame layout (f = 0, w = 21).  Neighbours
 * and parents stay inside their frame's fields.  Frame b's rows are [base_b, base_b + n_b), base_b the sites of the
 * frames before it, and its sites, count n_b and every table entry equal the one-frame call's on frame b alone, plus
 * base_b (-1 stays -1).
 * cg_spconv_index_many_dev: coords (N,3) the frames' points concatenated, frame b's at rows
 * [offsets[b], offsets[b + 1]) (host, B + 1, from 0 to N), each in [0, shapes[3 b + axis]) (not checked); shapes
 * (host, B x 3) each in [1, 2^21].  Outputs as cg_spconv_index_dev's, and out_frame (N capacity) = each site's frame;
 * out_p2v names the batched rows.                                                                                 */
int  cg_spconv_index_many_dev(cg_ctx *ctx, const int32_t *coords, int N, int B, const int32_t *offsets /* host */,
                              const int32_t *shapes /* host */, int32_t *out_vox, int32_t *out_nvox,
                              int32_t *out_frame, int32_t *out_p2v, int32_t *out_nbr);
/* cg_spconv_down_dev on a batched level: vox (M,3) and frame (M) its sites and their frames, shapes (host, B x 3) the
 * frames' spatial shapes.  Each child is dropped against its own frame's coarse shape (S_b - 2) / 2 + 1.  Row bound:
 * out_rows >= max(1, min(M, the coarse shapes' cell counts summed over the frames)), else CG_EINVAL; it is a bound
 * only, the true count goes to out_nvox.  out_frame (out_rows capacity) = each parent's frame.                     */
int  cg_spconv_down_many_dev(cg_ctx *ctx, const int32_t *vox, const int32_t *frame, const int32_t *nvox, int M, int B,
                             const int32_t *shapes /* host */, int out_rows, int32_t *out_vox, int32_t *out_nvox,
                             int32_t *out_frame, int32_t *out_nbr, int32_t *out_down, int32_t *out_up);
/* out (M,Cout) rows r < *nout: (sum over k, then input channel, of W[k][ci][co] * act(in[nbr[r][k]][ci]) + bias[co])
 * + residual[r][co], one fp32 FMA chain per output, so two runs are bitwise equal.  in (rows,Cin); nbr (M,K), or NULL
 * with K = 1 for the 1x1 convolution (row r reads row r); W (K,Cin,Cout) as spconv stores (k..., Cin, Cout).  act(v) =
 * max(v * bn_scale[ci] + bn_shift[ci], 0) when both are given (the BN + ReLU before a conv), else v; an absent row
 * contributes nothing.  bias (Cout) and residual (M,Cout) may be NULL.  Rows from min(*nout, M) on are not written.
 * Every index in the first min(*nout, M) rows of nbr must be a row of in (not checked).                          */
int  cg_spconv_conv_dev(cg_ctx *ctx, const float *in, int Cin, const int32_t *nbr, int K, const int32_t *nout, int M,
                        const float *W, int Cout, const float *bn_scale, const float *bn_shift, const float *bias,
                        const float *residual, float *out);
/* PointGroup's voxelisation, pointgroup_ops mode 4 (the mean): out (V,C) rows v < min(*nvox, V) = the mean of the
 * rows of feats (N,C) whose p2v (N) is v, as voxelize_fp_cuda_ sums it: out = 0, then for each such point in
 * ascending index out = fl(out + fl(fl(1 / n) * x)) in fp32, no FMA, so the result is deterministic.  A site with no
 * point is 0; a point whose p2v is not a site below min(*nvox, V) is ignored.  Rows from min(*nvox, V) on are not
 * written.                                                                                                        */
int  cg_pointgroup_voxel_mean_dev(cg_ctx *ctx, const float *feats, int N, int C, const int32_t *p2v,
                                  const int32_t *nvox, int V, float *out);
/* PointGroup's output_layer and offset head, one site per warp: a = max(in * bn_scale + bn_shift, 0) (m channels),
 * h = max(W1^T a + b1, 0) with the head's BN folded into W1 (m,m) [in][out] and b1 (m), out_site (V,3) rows
 * v < min(*nvox, V) = W2^T h + b2 with W2 (m,3) [in][out]; each output one fp32 FMA chain over the inputs ascending,
 * then the bias.  out (N,3) = out_site[p2v[i]], NaN for a point naming no site.  m in [1, 512].                 */
int  cg_pointgroup_head_dev(cg_ctx *ctx, const float *in, int m, const int32_t *nvox, int V, const float *bn_scale,
                            const float *bn_shift, const float *W1, const float *b1, const float *W2, const float *b2,
                            const int32_t *p2v, int N, float *out_site, float *out);

/* ---- per-pick glue (csrc/cg_pick.cu; catgrasp_b200/pick.py) ---------------------------------------------------
 * Device pointers, the context's stream, no synchronisation.
 *
 * cg_segment_table_dev: run_grasp_simulation.py:217-240 and :253-259 on labels (M) int32 or int64 (labels_is_i64)
 * and points x (M,3) float32 or float64 (x_is_f64).  Labels are dense in [0, L): L is the segmenter's cluster count
 * (MeanShift's number of centres, i.e. labels.max() + 1); a label outside [0, L) belongs to no segment.  Per label l:
 * out_count[l], the exact per-axis out_min / out_max (L,3) float64 (0 for an empty label), and out_inlier[l] (uint8):
 * count >= 500 and not n / ((q0 * q1) * q2) < 0.01, q = (max - min) / 0.001 rounded in the cloud's dtype, the division
 * by the product in float64 (a zero extent gives inf: an inlier).  out_labels (M, the labels' dtype) = the label, or -1
 * where it is no inlier (:240).  out_order (L): the inlier labels by count descending, ties in descending label order
 * (reversed(sorted(..., key=count))), then -1; *out_n_kept their number.  out_offsets (L+1): out_offsets[0] = 0 and
 * out_offsets[k+1] - out_offsets[k] = the count of out_order[k] (0 past the kept ones); out_index (M): the point
 * indices of the k-th kept segment, ascending, at [out_offsets[k], out_offsets[k+1]); entries from
 * out_offsets[*out_n_kept] on are not meaningful.  M >= 0, 1 <= L < 2^30.                                        */
int  cg_segment_table_dev(cg_ctx *ctx, const void *labels, int labels_is_i64, const void *x, int x_is_f64, int M, int L,
                          void *out_labels, int32_t *out_count, double *out_min, double *out_max, uint8_t *out_inlier,
                          int32_t *out_order, int32_t *out_n_kept, int32_t *out_offsets, int32_t *out_index);
/* cg_rank_grasps_dev: run_grasp_simulation.py:311-328.  probs (G,C) float32, p_T_given_G (G) float64 ->
 * out_p_G (G) = (pred * arange(C)).sum() / denom bit for bit with numpy (float64 products, numpy's pairwise summation
 * order), denom = len(cfg_grasp['classes']) - 1 (:313; the shipped grasp-Q net has C = 10 outputs for 11 class edges,
 * so denom = C); out_p_T_G (G) = p_T_given_G * p_G; out_perm (G) int32 = Python's stable sorted(key=-p_T_G):
 * descending, equal keys (+0.0 and -0.0 included) in input order.  G >= 0, 1 <= C <= 128, denom >= 1; NaN keys are
 * not ordered.                                                                                                     */
int  cg_rank_grasps_dev(cg_ctx *ctx, const float *probs, int G, int C, int denom, const double *p_T_given_G,
                        double *out_p_G, double *out_p_T_G, int32_t *out_perm);

/* ---- PointNet++ primitives (device pointers) ---------------------------
 * Replace the free functions of pointnet2.py:14-149.  Indices are int32 on
 * the device (the Python mirror widens to int64 like the reference).        */
/* pointnet2.py:14-33  square_distance: (B,S,3),(B,N,3) -> (B,S,N)           */
int cg_square_distance_dev(cg_ctx *ctx, const float *src, const float *dst,
                           int B, int S, int N, float *out);
/* pointnet2.py:35-51  index_points: points (B,N,C), idx (B,S) -> (B,S,C)    */
int cg_index_points_dev(cg_ctx *ctx, const float *points, const int32_t *idx,
                        int B, int N, int C, int S, float *out);
/* pointnet2.py:54-75  farthest_point_sample with explicit start indices.
 * cg_fps_dev: one thread-block cluster per cloud, points + running distances in
 * registers, one distributed-shared-memory exchange per round (N <= 65536 /
 * 131072 points for cluster size 8 / 16).  cg_fps_single_cta_dev: the round-1
 * one-CTA kernel (N <= 56320), kept for comparison.                           */
int cg_fps_dev(cg_ctx *ctx, const float *xyz, int B, int N, int npoint,
               const int32_t *start_idx, int32_t *out_idx);
int cg_fps_single_cta_dev(cg_ctx *ctx, const float *xyz, int B, int N, int npoint,
                          const int32_t *start_idx, int32_t *out_idx);
/* pointnet2.py:78-98  query_ball_point (first nsample by index, pad w/ first;
 * an empty ball yields N in every slot, like the reference).  radius2 is
 * float32(radius**2), the threshold torch compares against (:93)            */
int cg_ball_query_dev(cg_ctx *ctx, float radius2, int nsample,
                      const float *xyz, const float *new_xyz,
                      int B, int N, int S, int32_t *out_idx);
/* pointnet2.py:101-129 grouping tail of sample_and_group:
 * out (B,S,K,3+D) = [xyz[idx]-new_xyz, points[idx]]                         */
int cg_group_points_dev(cg_ctx *ctx, const float *xyz, const float *points,
                        const float *new_xyz, const int32_t *idx,
                        int B, int N, int D, int S, int K, float *out);


/* ---- PointNet++ set-abstraction / feature-propagation stacks -----------------------------
 * The reference ships the primitives above and cites the upstream module family in its model
 * docstrings (pointnet2.py:274,304); these entry points are that family's
 * PointNetSetAbstraction / PointNetFeaturePropagation built on the primitives
 * (sample_and_group, pointnet2.py:101-129; square_distance, :14-33).
 *
 * cg_mlp: a stack of nlayers shared (1x1 conv + BatchNorm + ReLU) layers, BN folded by the host:
 *   dims[nlayers+1] channel counts, Wt_host[i] = [dims[i]][dims[i+1]] k-major fp32, b_host[i] = [dims[i+1]].
 * Layers whose input width is a multiple of 64 run on wgmma (bf16 hi/lo x3, fp32 accumulate) when
 * there are >= 64 rows; narrower ones (the 3+D input layer) on the FMA kernels.                        */
typedef struct cg_mlp cg_mlp;
int  cg_mlp_create(cg_ctx *ctx, int nlayers, const int *dims, const float *const *Wt_host,
                   const float *const *b_host, cg_mlp **out);
void cg_mlp_destroy(cg_mlp *mlp);
/* x (R, dims[0]) -> out (R, dims[nlayers]): the per-row MLP (feature-propagation tail).  R < 2^31 (also
 * G*K below), any row count in that range.                                                          */
int  cg_shared_mlp_dev(cg_mlp *mlp, const float *x, int64_t R, float *out);
/* grouped (G, K, dims[0]) = output of cg_group_points_dev with G = B*S -> out (G, dims[nlayers]):
 * per-row MLP over all G*K rows, then max over the K rows of every group (set abstraction).           */
int  cg_group_mlp_max_dev(cg_mlp *mlp, const float *grouped, int G, int K, float *out);
/* Feature propagation, interpolation half: for every dense point xyz1[b][n] the 3 nearest of the S
 * sparse points xyz2[b] (expanded-form distances, ties -> lower index), weights (1/(d+1e-8))/sum, and
 *   out[b][n] = [points1[b][n] (D1 skip channels, optional) | sum_j w_j * points2[b][idx_j] (D2)]
 * out (B,N,D1+D2); out_idx (B,N,3) int32 / out_weight (B,N,3) optional (NULL: scratch).  S >= 2.
 * S == 2 follows the module family, which keeps the first three of the sorted distances and so has two
 * neighbours: weights (1/(d+1e-8)) / (r0+r1), out = w0*p0 + w1*p1, and the third slot of out_idx /
 * out_weight is index 0 with weight 0 (the Python module returns (B,N,2)).  S == 1 is a plain broadcast
 * and is left to the caller.                                                                            */
int  cg_three_interp_dev(cg_ctx *ctx, const float *xyz1, const float *xyz2, const float *points1, int D1,
                         const float *points2, int D2, int B, int N, int S, float *out,
                         int32_t *out_idx, float *out_weight);

#ifdef __cplusplus
}
#endif
#endif /* CATGRASP_B200_H */

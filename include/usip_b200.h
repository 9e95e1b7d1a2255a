/* usip_b200.h -- C ABI of libusip_b200.so: the H100 (sm_90a) drop-in for the USIP detector /
 * descriptor hot path.  Plain pointers and sizes only: no torch types, no C++ in the signatures.
 *
 * Conventions (all functions):
 *   - every pointer is a DEVICE pointer unless the name says `host`; tensors are dense, row-major;
 *   - the caller owns and pre-allocates every buffer; the library keeps no global state;
 *   - `stream` is a cudaStream_t passed as void*; launches are asynchronous, nothing synchronises;
 *   - the return value is 0 on success, otherwise a cudaError_t (or -1 for invalid arguments);
 *   - "(B,C,N)" etc. are the REFERENCE layouts (channel-major), "[P,C]" are this library's internal
 *     row-major point-major activations (row = one point / one group sample, C contiguous).
 *
 * Each entry point cites the reference interface it replaces (paths relative to lijx10/USIP).
 */
#ifndef USIP_B200_H_
#define USIP_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define USIP_B200_ABI_VERSION 1
int usip_abi_version(void);
/* name of the last failing check/launch for the calling thread ("" if none); host pointer */
const char* usip_last_error(void);

/* ------------------------------------------------------------------------------------------------
 * 1. Reference operator modules (plugin API B-1)
 * ---------------------------------------------------------------------------------------------- */

/* index_max.forward_cuda_shared_mem / forward_cuda          models/index_max_ext/index_max.cpp:132-148,
 * kernels models/index_max_ext/index_max_cuda.cu:9-25,29-61.
 * data (B,C,N) f32, index (B,N) i32 in [0,K) -> out_idx (B,C,K) i32: smallest n attaining
 * max{data[b,c,n] : index[b,n]==k, data > -1000}, else 0.  No B*K shared-memory cap.
 * scratch: B*C*K u64 (packed running max), may not alias anything. */
int usip_index_max_f32(const float* data, const int32_t* index, int32_t* out_idx,
                       unsigned long long* scratch, int B, int C, int N, int K, void* stream);

/* ball_query.forward_cuda_shared_mem                        models/ball_query_ext/ball_query.cpp:33-39,
 * kernel models/ball_query_ext/ball_query_cuda.cu:10-49.
 * dist (B,M,N) f32 -> out_idx (B,M,K) i32: first K n (ascending) with dist<=radius; 0 hits -> 0;
 * u<K hits -> out[u+i] = out[i % u]. */
int usip_ball_query_dist_f32(const float* dist, float radius, int32_t* out_idx,
                             int B, int M, int N, int K, void* stream);

/* Fused replacement of models/networks.py:355-373 (distance matrix + ball_query + gather + decenter):
 * xyz (B,3,N), feat (B,S,N) (S may be 0), centers (B,3,M) ->
 *   out_idx (B,M,K) i32      (bit-identical to ball_query on torch.norm(centers-xyz))
 *   out_group (B,3+S,M,K) f32 = x_aug gathered, xyz channels minus the centre  (`x_features`) (or NULL)
 *   out_rows  [B*M*K, ld_rows] f32: the same group as point-major rows for the MLP stack (or NULL)
 * scratch: usip_ball_group_scratch_bytes() bytes, 256-byte aligned (per cloud: bucket fill counts, 2-D bucket grid of
 * 32-byte records, overflow list).  CONTRACT: its counter region must be all-zero when the call starts -- clear it ONCE with
 * usip_ball_group_scratch_init() -- and every call leaves it all-zero again (the last CTA of each cloud restores it), so a
 * scratch buffer that is kept between calls costs no memset launch.  One scratch per stream.  Without scratch (or for
 * S > 4) the reference's in-order scan runs as a single kernel.  Two launches (build, query) chained by programmatic
 * dependent launch; the query stages its candidate buckets with one tensor-map TMA per keypoint. */
int usip_ball_group_f32(const float* xyz, const float* feat, const float* centers, float radius,
                        int32_t* out_idx, float* out_group, float* out_rows, int ld_rows,
                        void* scratch, int64_t scratch_bytes, int B, int S, int N, int M, int K, void* stream);
int64_t usip_ball_group_scratch_bytes(int B, int S, int N, int M, int K);
int usip_ball_group_scratch_init(void* scratch, int64_t scratch_bytes, int B, void* stream);

/* k-nearest-POINT grouping of the ablation detector RPN_Detector_KNN      models/networks.py:556-565
 * (torch.norm + topk(k, largest=False, sorted=False) + gather + subtract the node), without the (B,M,N) matrix.
 * out_idx (B,M,K) i32: the K points nearest to each centre, EXACT, in ascending point index (the reference's order is
 * unspecified; ties at the K-th distance: lowest index first); out_group / out_rows as in usip_ball_group_f32.  K <= N.
 * A NaN or inf squared distance gets one key, larger than every finite one, so such points come last and tie among
 * themselves lowest index first (torch.topk would put NaN after inf). */
int usip_knn_group_f32(const float* xyz, const float* feat, const float* centers, int32_t* out_idx, float* out_group,
                       float* out_rows, int ld_rows, int B, int S, int N, int M, int K, void* stream);

/* Farthest point sampling of the SOM nodes          data/kitti_detector_loader.py:68-83 (FarthestSampler.sample), :144-145
 * pts (B, Ns, 3) f32 row-major (the numpy subset the reference samples from), start (B,) i32 = index of the first node
 * (the reference draws it with np.random.randint) -> out_idx (B, k) i32 in selection order, out_nodes (B, 3, k) f32 (or
 * NULL).  Bit-identical to the numpy code: float64 running distances, first arg-max.  Ns <= 8192.  Points must be finite:
 * np.minimum propagates a NaN distance, the kernel keeps the smaller value. */
int usip_fps_f32(const float* pts, const int32_t* start, int32_t* out_idx, float* out_nodes, int B, int Ns, int k,
                 void* stream);
/* usip_fps_f64: usip_fps_f32 on float64 points, pts (B, Ns, 3) f64 (data/scenenn_descriptor_loader.py samples the
 * float64 ICP'd anchor): the same distance arithmetic, arg-max and minimum, so points that are float32 values give
 * usip_fps_f32's indices.  out_nodes (B, 3, k) f32 casts of the selected points, or NULL.  Ns <= 8192; the points sit in
 * 24 * Ns bytes of shared memory. */
int usip_fps_f64(const double* pts, const int32_t* start, int32_t* out_idx, float* out_nodes, int B, int Ns, int k,
                 void* stream);

/* Training pairs on the device (csrc/pairgen.cu): the detector's data/kitti_detector_loader.py:101-259
 * (KittiLoader.__getitem__) and data/modelnet_shrec_loader.py:152-275 (ModelNet_Shrec_Loader.__getitem__), and the
 * descriptor's data/kitti_descriptor_loader.py:102-347 (KittiDescriptorLoader.__getitem__).
 * Input: a ragged batch of raw scans, scans [T, C] f32 (x, y, z, then C-3 feature columns) with row offsets (n_scans+1)
 * i64.  Clouds are numbered c = 2*pair + side (0 = src / anchor, 1 = dst / positive); scan_of_cloud (2*n_pairs) i32 names
 * the scan of every cloud.  The detector names a pair's scan twice (both sides subsample the same scan independently), the
 * descriptor names the anchor's and the positive's.  Every per-point random number is Philox4x32-10 keyed by
 * (seed, step, cloud, point, purpose), so a batch is a pure function of (seed, step).
 *
 * usip_cloud_subsample (get_instance_unaugmented_np, detector :118-145, descriptor :117-128):
 *   out_rows (2*n_pairs, N) i32: row indices into each cloud's scan.  Optional radius mask (use_radius): fp32
 *     sqrt(x*x + z*z) compared in double against `radius`.  >= N points inside: a uniform subset of N without
 *     replacement, ascending row index.  Ns < N inside: every inside row t times (t the smallest >= 1 with Ns + t*Ns >= N),
 *     ascending, then a uniform subset of the N - t*Ns remainder, ascending.  A scan with no point inside gets rows 0.
 *     (The descriptor's reference raises below N rows; its callers reject such scans.)
 *   out_cand (2*n_pairs, n_cand) i32: a uniform subset of n_cand of the N positions, ascending (the FPS candidates).
 *   out_start (2*n_pairs) i32: the FPS start index in [0, n_cand).  out_valid (2*n_pairs) i32: points inside (or NULL).
 *   max_rows >= the longest scan, at most USIP_SUBSAMPLE_MAX_ROWS; N <= usip_pair_max_scan_rows(), the longest scan
 *   the one-CTA kernel takes.  With max_rows <= usip_pair_max_scan_rows() both levels run in that kernel (one CTA per
 *   cloud, keys in shared memory).  Above it the rows run in a kernel with one 8-CTA thread-block cluster per cloud that
 *   regenerates the keys in every pass; the selection is defined as the N smallest (Philox key, row) pairs either way,
 *   so out_rows and out_valid do not depend on which kernel ran.
 * usip_cloud_gather_candidates: out_pts (2*n_pairs, n_cand, 3) f32 = xyz of rows[c, cand[c, j]] of scan_of_cloud[c] --
 *   usip_fps_f32's input.
 * usip_pair_augment (augment(), :149-216, train mode only, then transform_pc_pytorch for dst, augmentation.py:199-248):
 *   rows as above, nodes (2*n_pairs, 3, M) f32 = the FPS nodes (usip_fps_f32 out_nodes);
 *   params (n_pairs, 48) f64 per pair: [0:9] horizontal, [9:18] 3-d and [18:27] perturbation rotation matrices (row
 *     major, applied as data @ R in float64), [27] augmentation scale, [28:31] augmentation shift, [31:40] the transform's
 *     R (fp32 values), [40:43] its shift, [43] its scale, [44] the Oxford height scale (USIP_PAIR_HEIGHT_SCALE),
 *     [45] the indoor per-pair augmentation switch (usip_indoor_pair_augment; ignored here), [46:48] unused;
 *   jit_pc (2*n_pairs, N, 3), jit_sn (2*n_pairs, N, S), jit_node (2*n_pairs, M, 3) f64 clipped jitter, each NULL to draw
 *     it on the device (N(0, 0.04^2) clipped at 0.12 for pc / node, N(0, 0.01^2) clipped at 0.05 for sn);
 *   flags: USIP_PAIR_* below.  sn = columns 3:3+S of the scan, or the last column when S == 1.
 *   -> src/dst pc (n_pairs, 3, N), sn (n_pairs, S, N), node (n_pairs, 3, M), R (n_pairs, 3, 3), scale (n_pairs),
 *      shift (n_pairs, 3, 1), all f32 -- the nine tensors of ModelDetector.set_input.
 * usip_desc_pair_augment (augment(), :205-276, train mode only):
 *   params (2*n_pairs, 32) f64 per cloud: [0:31] as above, with rotations and shift of the cloud's own and [27] the
 *     pair's scale, the same value in both of its clouds;
 *   jitter arrays and flags as in usip_pair_augment (the transform flags only); sn = columns 3:3+S for every S
 *     (3 + S <= C).  Test mode (no USIP_PAIR_TRAIN): the rows and the nodes as they are.
 *   -> anc/pos pc (n_pairs, 3, N), sn (n_pairs, S, N), node (n_pairs, 3, M) f32.
 * usip_modelnet_pair_augment (data/modelnet_shrec_loader.py:182-243 ModelNet_Shrec_Loader.augment, train mode only,
 *   then transform_pc_pytorch for dst): arguments, params layout and outputs as usip_pair_augment, but
 *   jit_pc (n_pairs, N, 3), jit_sn (n_pairs, N, 3), jit_node (n_pairs, M, 3) are PER PAIR: row i of src and of dst gets
 *     the same jitter, although the two clouds subsample independently.  NULL: drawn on the device with Philox keyed by
 *     the pair, N(0, 0.01^2) clipped at 0.05 for pc and sn, N(0, 0.04^2) clipped at 0.1 for nodes;
 *   S == 3 and sn = columns 3:6 (C >= 6).  After any rotation sn is a float64 chain (rotated, jittered, times [27]);
 *     without one it is fp32, jittered and scaled in place.  sn is never shifted.  pc and nodes: as usip_pair_augment.
 * usip_indoor_pair_augment (data/match3d_detector_loader.py:110-216 and scenenn_detector_loader.py, which augment like
 *   KittiLoader with other laws, then transform_pc_pytorch for dst): arguments, params layout, arithmetic and outputs as
 *   usip_pair_augment, but
 *   - device-mode jitter is N(0, 0.01^2) clipped at 0.02 for pc, every sn column and nodes (same Philox keys);
 *   - sn = columns 3:3+S for every S, 1 <= S <= 8 and 3 + S <= C;
 *   - with USIP_PAIR_TRAIN, pair b is augmented only when params[b, 45] != 0 (SceneNN trains on its train split, which
 *     is augmented, and its val split, which is not).  An un-augmented pair gets the gathered rows and nodes, then the
 *     dst transform, exactly as in test mode; its jitter rows are never read;
 *   - USIP_PAIR_ENU_TO_CAM and USIP_PAIR_HEIGHT_SCALE are refused (-1 before any launch).
 * Oxford scans (data/oxford_detector_loader.py, oxford_descriptor_loader.py) are ENU, z up.  USIP_PAIR_ENU_TO_CAM makes
 *   usip_pair_augment and usip_desc_pair_augment first map every row and node to the camera frame, (x, y, z) ->
 *   (x, -z, y), and sn columns 0:3 alike (requires S >= 3); then they run as above.  USIP_PAIR_HEIGHT_SCALE (detector
 *   only, with USIP_PAIR_ENU_TO_CAM, applied in train mode only): before the frame change a row's z becomes
 *   fl32(z * fl32(hs)), hs = params[b, 44].
 * usip_cloud_gather_candidates_zscaled: usip_cloud_gather_candidates with z multiplied by z_scale[c] (2*n_pairs) f32 in
 *   fp32, the height-scaled FPS input of the Oxford detector.
 * usip_cloud_gather_candidates_icp_f64 (SceneNN descriptor, data/scenenn_descriptor_loader.py __getitem__): out_pts
 *   (2*n_pairs, n_cand, 3) f64, usip_fps_f64's input.  Side 1 (the positive): the exact doubles of the fp32 rows.  Side 0
 *   (the anchor): hom2cart(T @ [x y z 1]^T) with T = icp (n_pairs, 4, 4) f64 row-major of the pair, in this order: per
 *   row r of T, h_r = fl(fma(z, T[r,2], fma(y, T[r,1], x * T[r,0])) + T[r,3]) (numpy's BLAS leaves the order open),
 *   then h_0 / h_3, h_1 / h_3, h_2 / h_3, divided even when T's last row is [0 0 0 1].
 * usip_scenenn_desc_pair_augment (SceneNNDescriptorLoader.__getitem__ with augment / augment_rot_only, then
 *   transform_pc_pytorch on the positive): rows (2*n_pairs, N) as above, icp as above, cand_pts the gathered float64
 *   candidates and node_idx (2*n_pairs, M) i32 the FPS selection into them (usip_fps_f64 out_idx), n_cand <= 8192 their
 *   count; params (n_pairs, 48) f64 in usip_pair_augment's layout, the rotations, [27] scale and [28:31] shift shared by
 *   the pair's two clouds, and [45] the pair's augmentation kind: 2 full (train split), 1 rotations only (val), any other
 *   value none (test).  flags: the USIP_PAIR_ROT_* and USIP_PAIR_TRANSLATION bits; USIP_PAIR_TRAIN is ignored (the kind
 *   decides).  sn = columns 3:3+S, 3 <= S <= 8.
 *   - anchor pc: the ICP above in float64, then (kind >= 1) the rotations as data @ R and (kind 2) the scale and
 *     (USIP_PAIR_TRANSLATION) the shift, all in float64, then one cast to fp32.  anchor sn[0:3]: the same ICP map
 *     (translation included), rounded to fp32, then each rotation in float64 rounded to fp32.  Other sn columns as read.
 *   - positive pc: in float64 from its first rotation on; without one, kind 2 scales it in fp32 (fl32(x * fl32(scale)))
 *     and shifts it as fl32(x + shift).  positive sn as the anchor's, without the ICP.
 *   - nodes: cand_pts[c, node_idx[c, i]], float64 through the rotations, scale and shift, then cast.
 *   - no jitter term at all.  Then the positive's pc, sn[0:3] and nodes get the fp32 dst transform of usip_pair_augment.
 *   -> anc/pos pc (n_pairs, 3, N), sn (n_pairs, S, N), node (n_pairs, 3, M), R (n_pairs, 3, 3), scale (n_pairs),
 *      shift (n_pairs, 3, 1) f32: the eleven ModelDescriptorIndoor.set_input tensors without the keypoints and sigmas.
 *   Refused (-1 before any launch): a null icp, S < 3 or S > 8, 3 + S > C, USIP_PAIR_ENU_TO_CAM or
 *   USIP_PAIR_HEIGHT_SCALE, M > n_cand, n_pairs > 32767.
 * usip_scale_channel_f32: t (B, C, L) f32 in place, t[b, k, :] *= factor in fp32 (the descriptor batch's height
 *   scaling, oxford/train_descriptor.py).
 * Every cloud of the augment and gather calls is one grid row, so usip_pair_augment, usip_indoor_pair_augment,
 *   usip_desc_pair_augment, usip_modelnet_pair_augment, usip_scenenn_desc_pair_augment and
 *   usip_cloud_gather_candidates(_zscaled, _icp_f64) take n_pairs <= 32767 (-1 before any launch
 *   above it); usip_test_cloud_gather takes n_clouds <= 65535 and usip_scale_channel_f32 B <= 65535. */
#define USIP_PAIR_TRAIN 1
#define USIP_PAIR_ROT_HORIZONTAL 2
#define USIP_PAIR_ROT_3D 4
#define USIP_PAIR_ROT_PERTURBATION 8
#define USIP_PAIR_TRANSLATION 16
#define USIP_PAIR_ENU_TO_CAM 32
#define USIP_PAIR_HEIGHT_SCALE 64
#define USIP_SUBSAMPLE_MAX_ROWS 16777216           /* usip_cloud_subsample: the longest scan, 2^24 rows */
int usip_pair_max_scan_rows(void);
int usip_cloud_subsample(const float* scans, int C, const int64_t* offsets, const int32_t* scan_of_cloud, int max_rows,
                         int n_pairs, int N, int n_cand, int use_radius, double radius, uint64_t seed, uint64_t step,
                         int32_t* out_rows, int32_t* out_cand, int32_t* out_start, int32_t* out_valid, void* stream);
int usip_cloud_gather_candidates(const float* scans, int C, const int64_t* offsets, const int32_t* scan_of_cloud,
                                 const int32_t* rows, const int32_t* cand, float* out_pts, int n_pairs, int N,
                                 int n_cand, void* stream);
int usip_cloud_gather_candidates_zscaled(const float* scans, int C, const int64_t* offsets,
                                         const int32_t* scan_of_cloud, const int32_t* rows, const int32_t* cand,
                                         const float* z_scale, float* out_pts, int n_pairs, int N, int n_cand,
                                         void* stream);
int usip_cloud_gather_candidates_icp_f64(const float* scans, int C, const int64_t* offsets,
                                         const int32_t* scan_of_cloud, const int32_t* rows, const int32_t* cand,
                                         const double* icp, double* out_pts, int n_pairs, int N, int n_cand,
                                         void* stream);
int usip_scenenn_desc_pair_augment(const float* scans, int C, const int64_t* offsets, const int32_t* scan_of_cloud,
                                   const int32_t* rows, const double* icp, const double* cand_pts,
                                   const int32_t* node_idx, const double* params, int flags, int S, int n_pairs, int N,
                                   int M, int n_cand, float* anc_pc, float* anc_sn, float* anc_node, float* pos_pc,
                                   float* pos_sn, float* pos_node, float* R, float* scale, float* shift, void* stream);
int usip_scale_channel_f32(float* t, int B, int C, int L, int k, float factor, void* stream);
int usip_pair_augment(const float* scans, int C, const int64_t* offsets, const int32_t* scan_of_cloud,
                      const int32_t* rows, const float* nodes, const double* params, const double* jit_pc,
                      const double* jit_sn, const double* jit_node, uint64_t seed, uint64_t step, int flags, int S,
                      int n_pairs, int N, int M, float* src_pc, float* src_sn, float* src_node, float* dst_pc,
                      float* dst_sn, float* dst_node, float* R, float* scale, float* shift, void* stream);
int usip_indoor_pair_augment(const float* scans, int C, const int64_t* offsets, const int32_t* scan_of_cloud,
                             const int32_t* rows, const float* nodes, const double* params, const double* jit_pc,
                             const double* jit_sn, const double* jit_node, uint64_t seed, uint64_t step, int flags,
                             int S, int n_pairs, int N, int M, float* src_pc, float* src_sn, float* src_node,
                             float* dst_pc, float* dst_sn, float* dst_node, float* R, float* scale, float* shift,
                             void* stream);
int usip_modelnet_pair_augment(const float* scans, int C, const int64_t* offsets, const int32_t* scan_of_cloud,
                               const int32_t* rows, const float* nodes, const double* params, const double* jit_pc,
                               const double* jit_sn, const double* jit_node, uint64_t seed, uint64_t step, int flags,
                               int S, int n_pairs, int N, int M, float* src_pc, float* src_sn, float* src_node,
                               float* dst_pc, float* dst_sn, float* dst_node, float* R, float* scale, float* shift,
                               void* stream);
int usip_desc_pair_augment(const float* scans, int C, const int64_t* offsets, const int32_t* scan_of_cloud,
                           const int32_t* rows, const float* nodes, const double* params, const double* jit_pc,
                           const double* jit_sn, const double* jit_node, uint64_t seed, uint64_t step, int flags, int S,
                           int n_pairs, int N, int M, float* anc_pc, float* anc_sn, float* anc_node, float* pos_pc,
                           float* pos_sn, float* pos_node, void* stream);

/* Test-set clouds (evaluation/kitti_test_loader.py:106-139, oxford_test_loader.py:63-96; the noise of
 * evaluation/save_keypoints.py:275).  n_clouds clouds, cloud c reading scan scan_of_cloud[c]: rows (n_clouds, N) i32
 * and FPS nodes (n_clouds, 3, M) f32 (usip_cloud_subsample / usip_cloud_gather_candidates / usip_fps_f32) ->
 * pc (n_clouds, 3, N), sn (n_clouds, S, N) = scan columns 3:3+S, node (n_clouds, 3, M).  flags: 0 or
 * USIP_PAIR_ENU_TO_CAM (Oxford: pc, sn columns 0:3 and nodes to the camera frame, S >= 3).  With noise_sigma != 0, pc
 * then becomes fl32(pc + fl32(n * fl32(noise_sigma))) with n uploaded in noise (n_clouds, 3, N) f32 (torch.randn on the
 * host), or, with noise NULL, a Philox N(0, 1) keyed by (seed, step, cloud, point). */
int usip_test_cloud_gather(const float* scans, int C, const int64_t* offsets, const int32_t* scan_of_cloud,
                           const int32_t* rows, const float* nodes, const float* noise, float noise_sigma,
                           uint64_t seed, uint64_t step, int flags, int S, int n_clouds, int N, int M, float* pc,
                           float* sn, float* node, void* stream);

/* Keypoint repeatability       evaluation/matlab/eval_repeatability/eval_rep.m:142-146, for every K of a sweep at once.
 * keypoints (n_scans, 3, M) f32, order (n_scans, M) i32 (the selection order of every scan's keypoints), count
 * (n_scans,) i32 (how many of them are selectable).  pairs (P, 2) i32: the anchor and positive scan.  frames (P, 3, 3, 4)
 * f64 row-major: the anchor's frame map F_a, the positive's F_p and the ground truth T_gt.  ks: nK ascending positive
 * K values (host memory, nK <= USIP_REP_MAX_K).  For pair p and K = ks[k], with n_a = min(K, count[anc]) and
 * n_p = min(K, count[pos]):  a_i = F_a * kp[anc][:, order[anc][i]] (i < n_a),  q_j = T_gt * (F_p * kp[pos][:,
 * order[pos][j]]) (j < n_p), each matrix-vector product ((m0 x + m1 y) + m2 z) + m3 in fp64 without contraction;
 * inliers[p, k] = #{i : sqrt(min_j ((dx^2 + dy^2) + dz^2)) < radius} and n_anc[p, k] = n_a.  One CTA per pair;
 * min(M, ks[nK-1]) must not exceed USIP_REP_MAX_KEYPOINTS, radius must be > 0. */
#define USIP_REP_MAX_K 32
#define USIP_REP_MAX_KEYPOINTS 4096
int usip_repeatability_f64(const float* keypoints, const int32_t* order, const int32_t* count, int n_scans, int M,
                           const int32_t* pairs, const double* frames, int P, const int32_t* ks, int nK, double radius,
                           int32_t* inliers, int32_t* n_anc, void* stream);

/* Outdoor registration    evaluation/matlab/eval_outdoor/{kitti/evaluate_kitti.m, oxford/evaluate_oxford.m}: descriptor
 * matching, then RANSAC (external/ransacfitRt.m, ransac.m, estimateRigidTransform.m), for every pair, every K of a
 * keypoint-count sweep and every trial budget of a maxTrials sweep.  Both kernels run one CTA per (pair, K) and refuse
 * more than USIP_REG_MAX_KEYPOINTS rows per scan (their shared memory).
 *
 * usip_desc_match_f64: desc (n_scans, L, D) f32, each scan's rows in selection order; count (n_scans,) i32; pairs
 * (P, 2) i32 (anchor scan, positive scan); ks: nK ascending positive K values (host memory, nK <= USIP_REP_MAX_K).  For
 * pair p and K = ks[kk] the anchor set is rows 0..n_a-1 of the anchor scan, n_a = min(K, count, L), and likewise the
 * positive set.  d^2(i, j) = sum_c (a_c - b_c)^2 in fp64 with c ascending and no contraction; candidates are ordered
 * by (d^2, index), so the lowest index wins a tie, and a NaN d^2 (a non-finite descriptor value) orders as +inf: every
 * row gets its min(k, n) neighbours whatever the values.
 *   k == 1 (KITTI): one-way 1-NN; match i = (i, nearest positive) for i < n_a, in anchor order (none if n_pos = 0).
 *   k in 2..8 (Oxford): the k nearest positives of every anchor united with the k nearest anchors of every positive
 *   (all rows when a set has fewer than k), unique rows sorted by anchor, then positive: MATLAB's union(.., 'rows').
 * -> matches (P, nK, cap, 2) i32 (anchor row, positive row), cap = L for k == 1 and 2*k*L otherwise, and n_matches
 * (P, nK) i32.  D must not exceed USIP_REG_MAX_DIM.
 *
 * usip_ransac_rt_f64: xyz (n_scans, L, 3) f32 in the rows' order of desc; count, pairs as above; frames (P, 3, 3, 4)
 * f64 (F_a, F_p, T_gt as usip_repeatability_f64; T_gt is not read); matches / n_matches of usip_desc_match_f64 (cap
 * as there); trials: nT ascending trial budgets (host memory, 1 <= nT <= USIP_REG_MAX_SWEEP, 1 <= trials[i] <=
 * USIP_REG_MAX_TRIALS); threshold > 0.  x1 = F_a * anchor row, x2 = F_p * positive row (((m0 x + m1 y) + m2 z) + m3),
 * and the model is x1 = R x2 + t.
 *   Trial j (0-based) reads three uniforms u in [0, 1): row j of uniforms ((trials[nT-1] + 1, 3) f64) when given, else
 *   Philox4x32-10 with counter (j, 0, 0x52414e53, 0) and key (seed lo, seed hi), u_i = word_i * 2^-32 (i = 0, 1, 2):
 *   every pair and K sees the same stream, as ransac.m's rng(0) does.  usip_ransac_uniforms writes them.
 *   Sample of n = npts matches: i0 = min(floor(u0 n), n-1); i1 = min(floor(u1 (n-1)), n-2), then i1 += 1 if i1 >= i0;
 *   i2 = min(floor(u2 (n-2)), n-3), then i2 += 1 if i2 >= min(i0, i1), then i2 += 1 if i2 >= max(i0, i1); products
 *   in fp64.
 *   Fit (estimateRigidTransform.m): centroids ((0 + p_0) + p_1) + ... then / n; B = sum of A_i^T A_i over the points in
 *   order, A_i = [0, (y-x)^T; x-y, [y+x]_x] of the centred pair, entry (r, c) ((A0r A0c + A1r A1c) + A2r A2c) + A3r A3c;
 *   cyclic Jacobi on B, pairs (0,1) (0,2) (0,3) (1,2) (1,3) (2,3), 8 sweeps, a rotation skipped when its off-diagonal
 *   entry is exactly 0 (theta = (a_qq - a_pp) / (2 a_pq), t = sign(theta) / (|theta| + sqrt(theta^2 + 1)), sign(0) =
 *   1, c = 1 / sqrt(t^2 + 1), s = t c); the eigenvector of the smallest diagonal entry (lowest index on a tie) goes
 *   to quat2rot.m unnormalised; t = xbar - R ybar.  Inlier: sqrt((dx^2 + dy^2) + dz^2) < threshold, strictly.
 *   Stop (ransac.m): on ninliers >= bestscore the trial becomes the best and N = max(log(1 - 0.99) / log(clamp(1 -
 *   (f f) f, eps, 1 - eps)), 10), f = ninliers / npts; then trialcount += 1; the loop ends when trialcount > maxTrials
 *   or N <= trialcount.  One stream serves the whole sweep: each budget's result is the loop state where that loop
 *   ends.  Trials run 256 at a time and one thread replays the update in trial order, so the result is the sequential
 *   loop's.  `log` is CUDA's, within 1 ulp of a correctly rounded one, so a stop can differ from another libm's only
 *   when N lies within an ulp of an integer; every other step is correctly rounded.
 *   Finish (ransacfitRt.m): the best trial's inliers are refitted as above (status 0), unless fewer than 3 (status 2,
 *   Rt zero).  npts < 3: status 1, no model; npts == 3: fitted directly, trialcount 0, n_inliers 3.  A match index
 *   outside its scan's rows gives status 3.
 * -> Rt (P, nK, nT, 3, 4) f64; n_inliers (the best trial's count), trialcount, best_trial (-1 without trials) and
 * status, each (P, nK, nT) i32. */
#define USIP_REG_MAX_KEYPOINTS 1024
#define USIP_REG_MAX_DIM 512
#define USIP_REG_MAX_MATCH_K 8
#define USIP_REG_MAX_SWEEP 16
#define USIP_REG_MAX_TRIALS 100000
int usip_desc_match_f64(const float* desc, const int32_t* count, int n_scans, int L, int D, const int32_t* pairs,
                        int P, const int32_t* ks, int nK, int k, int32_t* matches, int32_t* n_matches, void* stream);
int usip_ransac_rt_f64(const float* xyz, const int32_t* count, int n_scans, int L, const int32_t* pairs,
                       const double* frames, int P, int nK, const int32_t* matches, const int32_t* n_matches, int cap,
                       const int32_t* trials, int nT, double threshold, uint64_t seed, const double* uniforms,
                       double* Rt, int32_t* n_inliers, int32_t* trialcount, int32_t* best_trial, int32_t* status,
                       void* stream);
/* the uniforms of trials 0..T-1 of usip_ransac_rt_f64's Philox stream -> out (T, 3) f64 */
int usip_ransac_uniforms(uint64_t seed, int T, double* out, void* stream);

/* Information matrix of the registration      evaluation/matlab/eval_indoor/3dmatch/register2Fragments.m:77-88.
 * The inputs of usip_ransac_rt_f64 (same values: the matches, the trial sweep, threshold, seed and uniforms), plus its
 * best_trial and status (P, nK, nT) i32.  For each (pair, K, budget) with status 0 the best trial's model is derived
 * again from the same uniforms (sample and 3-point fit as in usip_ransac_rt_f64; npts == 3: all three matches), its
 * inliers are taken in ascending match order, and info = sum over them, in that order, of A^T A with
 * A = [I3 | [[0, 2z, -2y], [-2z, 0, 2x], [2y, -2x, 0]]], (x, y, z) = F_a * the anchor row (fragment 1's keypoint);
 * entry (r, c) of A^T A is ((A0r A0c + A1r A1c) + A2r A2c), all fp64 without contraction.  n_info = the inlier count,
 * which equals usip_ransac_rt_f64's n_inliers.  status != 0: info zero and n_info 0 (register2Fragments.m's catch: no
 * inliers).  A status-0 entry whose best trial lies outside the stream or does not fit the matches: info zero, n_info -1.
 * -> info (P, nK, nT, 6, 6) f64 row-major, n_info (P, nK, nT) i32. */
int usip_ransac_info_f64(const float* xyz, const int32_t* count, int n_scans, int L, const int32_t* pairs,
                         const double* frames, int P, int nK, const int32_t* matches, const int32_t* n_matches, int cap,
                         const int32_t* trials, int nT, double threshold, uint64_t seed, const double* uniforms,
                         const int32_t* best_trial, const int32_t* status, double* info, int32_t* n_info, void* stream);

/* Fragment overlap      register2Fragments.m:134-137 (ratioAligned(1)), for J (fragment a, fragment b, map) jobs at once.
 * xyz (sum of rows, 3) f32: every fragment's rows packed (columns 0:3 of its .npy), device; offsets (n_frags + 1) i64,
 * HOST memory, offsets[0] = 0, fragment f = rows [offsets[f], offsets[f+1]); jobs (J, 2) i32, HOST memory: fragment a
 * (the reference's fragment 1) and fragment b; Rt (J, 3, 4) f64, device: x_a = R x_b + t, as usip_ransac_rt_f64 returns
 * it.  -> hits (J,) i32, device.
 *   Rule: every point of b is mapped in fp64 without contraction, ((r0 x + r1 y) + r2 z) + t per row, then rounded once
 *   to fp32: b'.  A point p of a is a hit iff some b' has sqrtf(d2) < radius, d2 = (dx dx + dy dy) + dz dz in fp32
 *   round-to-nearest without FMA, radius fp32; tested as d2 <= t_lim, t_lim the largest fp32 with sqrtf(t_lim) <
 *   radius, found on the host.  A point with a non-finite coordinate, in a or in b, is never a hit (it still counts in
 *   a's rows).  hits[j] = the number of points of a that are hits: an existence count, so no search order shows.
 *   Search: each fragment is counting-sorted into a uniform cell grid over its finite rows (at most 2 rows + 64 cells;
 *   edge 1.01 radius, grown by 1.25 until the cells fit; rows outside clamp into border cells).  A query p goes into
 *   b's frame as q = R^T (p - t) (fp64) and scans every cell the box [q - r', q + r'] touches.  Margin: with delta =
 *   max |(R^T R - I)_ik| (+ 2^-40), bmax = max |coordinate| of b's finite rows and B = max_i (sum_k |R_ik| bmax +
 *   |t_i|) >= |b'_i|, a passing b' lies within D = radius (1 + 2^-20) of p (the fp32 d2 is at most 5 roundings below
 *   the true square) and b' lies within 2^-23 B of R b + t (one fp32 rounding per coordinate, sqrt(3) 2^-24 B in norm,
 *   plus the fp64 map's error); so |q - b| <= (D + 2^-23 B)(1 + 2 delta) + 6 delta bmax (|R^T w| <= ||R|| |w| and
 *   ||R^T R - I||_F <= 3 delta), and r' adds 2^-40 (|p|_inf + |t|_inf + bmax) for q's own fp64 error.  The bound holds
 *   for any R (a far-from-rigid R only widens the search); a non-finite r' or q scans every cell.
 *   Refused before any launch: a job naming a fragment out of range, a fragment with no rows or more than
 *   USIP_OVERLAP_MAX_ROWS, more than 65535 fragments, radius <= 0 or non-finite, scratch smaller than
 *   usip_fragment_overlap_scratch_bytes(offsets[n_frags], n_frags, J) or not 16-byte aligned.  Six kernels per call:
 *   box, grid set-up, count, scan, scatter, query. */
#define USIP_OVERLAP_MAX_ROWS (1 << 26)
size_t usip_fragment_overlap_scratch_bytes(int64_t total_rows, int n_frags, int J);
int usip_fragment_overlap_f32(const float* xyz, const int64_t* offsets, int n_frags, const int32_t* jobs,
                              const double* Rt, int J, float radius, void* scratch, size_t scratch_bytes,
                              int32_t* hits, void* stream);

/* Radius non-maximum suppression of the detected keypoints    evaluation/save_keypoints.py:180-216 (nms)
 * keypoints (B,3,M) f32, sigmas (B,M) f32 -> out_idx (B,M) i32: original indices of the kept keypoints in the order the
 * reference emits them (ascending sigma, ties by index), padded with -1; out_count (B,) i32.  radius < 0.01: pass-through
 * (0..M-1, count M) like the reference.  NaN sigmas come first, in index order among themselves (np.argmin returns the
 * first NaN), and each suppresses its neighbours as usual.  M <= 8533 (6 * 4 * M bytes of shared memory). */
int usip_nms_f32(const float* keypoints, const float* sigmas, float radius, int32_t* out_idx, int32_t* out_count,
                 int B, int M, void* stream);

/* operations.knn_gather_by_indexing                         models/operations.py:271-287
 * src (B,C,N), idx (B,M,K) i32 -> out (B,C,M,K): out[b,c,m,k] = src[b,c,idx[b,m,k]]. */
int usip_knn_gather_f32(const float* src, const int32_t* idx, float* out,
                        int B, int C, int N, int M, int K, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 2. Grouping front-end of RPN_Detector.forward            models/networks.py:85-108, util/som.py:17-54
 * ---------------------------------------------------------------------------------------------- */

/* som.query_topk(k=1): nearest node per point, fp32 (dx*dx+dy*dy)+dz*dz, ties -> smallest m.
 * xyz (B,3,N), node (B,3,M) -> min_idx (B,N) i32, count (B,M) i32 (must be zeroed by the caller). */
int usip_som_assign_f32(const float* xyz, const float* node, int32_t* min_idx, int32_t* count,
                        int B, int N, int M, void* stream);

/* The same result through a cell grid over the M <= 1024 nodes of each cloud (csrc/nngrid.cu): the nodes are counting-sorted
 * into ~M/2 cells, every point searches the cell shells around it until nothing outside can be closer -- ~50 distance
 * evaluations per point instead of M.  scratch: usip_som_assign_grid_scratch_bytes(B, M) bytes, 16-byte aligned. */
size_t usip_som_assign_grid_scratch_bytes(int B, int M);
int usip_som_assign_grid_f32(const float* xyz, const float* node, int32_t* min_idx, int32_t* count, void* scratch,
                             size_t scratch_bytes, int B, int N, int M, void* stream);

/* Stable counting sort of the points of every cloud by node id.
 *   seg_off (B,M+1) i32 : rows [seg_off[m], seg_off[m+1]) of cloud b belong to node m
 *   perm    (B,N)   i32 : sorted position -> original point index n (ascending n inside a node)
 *   row_seg (B,N)   i32 : b*M + node id of each sorted row
 * scratch: B * ceil(N/256) * M i32.  M <= 50176; a larger M is refused before any launch. */
int usip_cluster_sort(const int32_t* min_idx, int32_t* seg_off, int32_t* perm, int32_t* row_seg,
                      int32_t* scratch, int B, int N, int M, void* stream);

/* networks.py:87-108: cluster mean (sum/(count+1e-5), empty -> 0), decentre, concat sn.
 *   cluster_mean (B,3,M) f32 ; x_aug [B*N, ldx] (sorted rows; cols 0..2 = x - mean[node], 3..3+S-1 = sn,
 *   remaining cols up to ldx zero). */
int usip_cluster_mean_decenter(const float* xyz, const float* feat, const int32_t* seg_off,
                               const int32_t* perm, float* cluster_mean, float* x_aug, int ldx,
                               int B, int S, int N, int M, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 3. Shared-MLP stack: conv1x1 (+bias) with fused BN/ReLU prologue and BN-stat / group-max epilogue
 *    models/layers.py:248-303 (EquivariantLayer), 172-216 (MyConv2d), 23-121 (MyBatchNorm*)
 * ---------------------------------------------------------------------------------------------- */
typedef struct usip_layer_desc {
  const float* X;  int32_t ldx;        /* [P,Cin] input (pre-activation of the previous layer)       */
  int32_t P, Cin, Cout;
  const float* W;  int32_t ldw;        /* [Cout,Cin] weight rows, row stride ldw (conv weight layout)  */
  int32_t w_transposed;                /* 1: W is stored [Cin,Cout] (row stride ldw) -- dgrad uses the
                                          forward weight as-is: G_in = G_out * W                        */
  const float* bias;                   /* [Cout] or NULL                                              */
  const float* in_scale;               /* [Cin] or NULL: a = x*in_scale+in_shift (folded BatchNorm)   */
  const float* in_shift;
  int32_t in_relu;                     /* apply ReLU after the affine                                 */
  const float* addend; int32_t ld_add; /* optional [G,Cout] term added per row group                  */
  const int32_t* add_index;            /* row -> g  (NULL: g = row / add_group)                       */
  int32_t add_group;
  float* Y; int32_t ldy;               /* [P,Cout] output (NULL: not written)                         */
  float* stat_partial;                 /* [usip_layer_stat_slots(desc),2,Cout] partial (sum, sumsq) rows, or NULL */
  float* gmax; float* gmin;            /* [P/group,Cout] per-group max / min of Y, or NULL            */
  int32_t* garg_max; int32_t* garg_min;/* [P/group,Cout] row-in-group of the max / min, or NULL       */
  int32_t group;
  int32_t precision;                   /* 0 = fp32 SIMT, 1 = 3xTF32 wgmma (Cin%32==0, Cout%64==0) */
  void* tc_workspace;                  /* precision 1: >= usip_layer_tc_workspace_bytes(Cin,Cout) bytes */
  int64_t tc_workspace_bytes;
  int32_t tc_weights_packed;           /* 1: tc_workspace already holds the packed weights of this W  */
  int32_t debug_flags;                 /* precision option of the tensor-core kernel, 0 = 3xTF32: 8 = plain single-pass TF32
                                          (hi x hi product only, ~5e-4 relative: the backward-precision option of the train
                                          step).  Other bits are ignored. */
  unsigned long long* debug_clocks;    /* unused, keep NULL (kept for the layout of the descriptor) */
} usip_layer_desc;

int usip_layer_fwd(const usip_layer_desc* d, void* stream);
/* Packs the tensor-core weight tiles of n layers (precision != 0 descriptors: W, ldw, w_transposed, Cin, Cout, P, group /
 * gmax / gmin, debug_flags and tc_workspace are read) in ONE launch, exactly as usip_layer_fwd does on a call with
 * tc_weights_packed == 0; afterwards those layers may be launched with tc_weights_packed = 1.  The train step uses it to
 * re-pack all weight matrices after the optimizer update (26 launches -> 1). */
int usip_layer_tc_pack_many(const usip_layer_desc* descs, int n, void* stream);
/* number of [2,Cout] partial rows usip_layer_fwd writes into stat_partial for this descriptor (P, Cout, precision,
   group and whether group outputs are requested must already be filled in): one per 128-row tile for the SIMT kernel,
   one per (CTA, 32-row quarter) for the persistent tensor-core kernel.  usip_bn_finalize sums them in a fixed order. */
int usip_layer_stat_slots(const usip_layer_desc* desc);
int usip_layer_tile_rows(void);
/* bytes of tc_workspace (hi/lo TF32 split of W, pre-swizzled into wgmma operand tiles) */
int64_t usip_layer_tc_workspace_bytes(int Cin, int Cout);

/* Training-mode BatchNorm finalisation (F.batch_norm, layers.py:69-71): reduce the per-tile partials,
 * produce the folded affine scale = gamma/sqrt(var+eps), shift = beta - mean*scale, update running stats
 * (momentum, unbiased var) and save mean / invstd for the backward pass.
 * The partials are fp32 (sum y, sum y^2) per tile and var = E[y^2] - E[y]^2 in float64, so the variance loses digits to
 * cancellation when a channel's |mean| is large against its std: from the SIMT layer's partials the relative error of
 * invstd stays below 2.5e-7 + 4e-8 (|mean|/std)^2 (measured on an H100 80GB HBM3 at 700 W over 65573 rows: 5.8e-8,
 * 8.1e-7, 4.5e-6 and 6.2e-5 at |mean|/std = 0, 10, 30 and 100). */
int usip_bn_finalize(const float* stat_partial, int ntiles, int64_t count, int C,
                     const float* gamma, const float* beta, float eps, float momentum,
                     float* running_mean, float* running_var, float* scale, float* shift,
                     float* save_mean, float* save_invstd, void* stream);
/* Eval-mode: scale/shift from the running statistics. */
int usip_bn_eval_affine(const float* gamma, const float* beta, const float* running_mean,
                        const float* running_var, float eps, int C, float* scale, float* shift, void* stream);

/* Segmented max over the sorted rows of every node (index_max + gather of networks.py:117-120,130-133):
 * X [B*N, ldx] -> pooled [B*M, ldp] (empty node -> 0), arg [B*M, C] i32 = global sorted row (or -1).
 * C, ldx, ldp multiples of 4; X, pooled, arg 16-byte aligned (section 5). */
int usip_segmax(const float* X, int ldx, const int32_t* seg_off, const int32_t* perm,
                float* pooled, int ldp, int32_t* arg, int B, int N, int M, int C, void* stream);

/* Node kNN, layers.py:417-421: ascending sqrt-distance, ties by index.  pts (B,3,M) -> knn (B,M,K) i32. */
int usip_knn_nodes(const float* pts, int32_t* knn_idx, int B, int M, int K, void* stream);

/* First kNN-fusion layer without materialising the (B,3+C,M,K) group tensor (layers.py:422-432):
 * Y[(b,m,k),:] = Z[b*M+knn[b,m,k],:] + Wxyz * (pts[b,:,knn]-pts[b,:,m]) + bias ; + BN stat partials.
 * Cout, ldz, ldy multiples of 4; Z and Y 16-byte aligned (section 5). */
int usip_knn_combine(const float* Z, int ldz, const float* pts, const int32_t* knn_idx,
                     const float* W, int ldw, const float* bias, float* Y, int ldy, float* stat_partial,
                     int B, int M, int K, int Cout, void* stream);

/* out[q, c] = relu(scale[c]*(scale[c]>=0 ? gmax : gmin)[q,c] + shift[c])  == max_k relu(bn(y_k)) */
int usip_group_select(const float* gmax, const float* gmin, const float* scale, const float* shift,
                      float* out, int ldo, int Q, int C, void* stream);

/* Groups larger than the layer epilogue's 128 rows: out_max[q, c] = max over r < ratio of gmax[q*ratio + r, c] (and
 * out_min likewise from gmin, when both are given) for Q_out x C outputs, rows contiguous ([Q_out*ratio, C] in,
 * [Q_out, C] out).  Same comparison as the epilogue's group max (strict >, strict <, from -inf / +inf; NaN never wins)
 * and the result of one in-order scan, so it is deterministic.  The indoor descriptor uses it for its 448-row balls
 * (64-row sub-groups, ratio 7) and for the per-cloud global max over its M keypoints (ratio M).  No arg outputs: see
 * usip_group_max_combine_arg. */
int usip_group_max_combine(const float* gmax, const float* gmin, float* out_max, float* out_min, int ratio, int Q_out,
                           int C, void* stream);
/* The same combine with arg outputs, for the backward of the indoor descriptor.  out_amax [Q_out, C] i32 is the row of
 * out_max in the whole group: r * sub + amax[q*ratio + r, c], where r < ratio is the first input row holding the max
 * (row 0 when none beats -inf: all -inf / NaN) and amax the row-in-sub-group args of the layer epilogue; with amax NULL
 * (the global max over keypoints) it is r.  out_amin likewise from gmin / amin.  With ties at the first index inside each
 * sub-group, the arg is the first index of the max over all ratio * sub rows.  gmax, out_max, out_amax are required;
 * gmin, out_min, out_amin come together; amin comes with amax (and gmin); sub >= 1 with args. */
int usip_group_max_combine_arg(const float* gmax, const float* gmin, const int32_t* amax, const int32_t* amin,
                               float* out_max, float* out_min, int32_t* out_amax, int32_t* out_amin, int ratio, int sub,
                               int Q_out, int C, void* stream);

/* networks.py:151-154: keypoints (B,3,M) = out[:, :3] + cluster_mean ; sigmas (B,M) = softplus(out[:,3]) + lb */
int usip_head_finalize(const float* out4, int ld, const float* cluster_mean, float sigma_lower_bound,
                       float* keypoints, float* sigmas, int B, int M, void* stream);

/* networks.py:383: out (B,C,M) = X[q,:] / (||X[q,:]||_2 + 1e-5); norm_out [B*M] optional (saved for backward) */
int usip_l2norm_to_bcm(const float* X, int ldx, float* out, float* norm_out, int B, int M, int C, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 4. Losses                                                  models/losses.py:44-143
 * ---------------------------------------------------------------------------------------------- */
/* min_j ||a_i - b_j||_2 and argmin (first index on exact ties).  a (B,3,Ma), b (B,3,Nb) ->
 * min_d (B,Ma) f32, arg (B,Ma) i32.  packed: B*Ma u64 scratch. */
int usip_pairwise_min_f32(const float* a, const float* b, float* min_d, int32_t* arg,
                          unsigned long long* packed, int B, int Ma, int Nb, void* stream);

/* The same result (bit-identical min_d and arg, same tie rule) for FEW queries against a LARGE point set -- the
 * keypoint-on-point-cloud searches of keypoint_detector.py:187-197 (512 keypoints against 16384 points per cloud): the
 * cloud is counting-sorted into a cell grid (one CTA per cloud) and every query scans the cell shells around it until
 * nothing outside can be closer.  scratch: usip_pairwise_min_grid_scratch_bytes(B, Nb) bytes, 16-byte aligned, contents
 * irrelevant on entry. */
size_t usip_pairwise_min_grid_scratch_bytes(int B, int Nb);
int usip_pairwise_min_grid_f32(const float* a, const float* b, float* min_d, int32_t* arg, void* scratch,
                               size_t scratch_bytes, int B, int Ma, int Nb, void* stream);

/* ChamferLoss_Brute sigma branch (losses.py:79-97) from the two pairwise-min results:
 * out[0]=loss, out[1]=chamfer_pure, out[2]=chamfer_weighted. */
int usip_chamfer_prob_reduce(const float* d_sd, const int32_t* i_sd, const float* d_ds, const int32_t* i_ds,
                             const float* sig_src, const float* sig_dst, float* out3, int B, int M, int N,
                             void* stream);

/* keypoint_detector.py:182-184: out = R @ kp * scale + shift   (kp (B,3,M), R (B,3,3), scale (B), shift (B,3)) */
int usip_transform_points(const float* kp, const float* R, const float* scale, const float* shift,
                          float* out, int B, int M, void* stream);

/* mean over (B,M) of d times alpha -> out[0]  (keypoint_detector.py:193-197) */
int usip_mean_scale(const float* d, int64_t n, float alpha, float* out, void* stream);


/* DescPairScanLoss (models/losses.py:190-237): min_j ||a[:,i] - b[:,j]||_2 over C-dim descriptors, a (B,C,Ma), b (B,C,Nb) */
int usip_desc_pairmin_f32(const float* a, const float* b, float* min_d, int32_t* arg, int B, int C, int Ma, int Nb,
                          void* stream);
/* loss (B,M) = w * clamp(dpos - dneg + gamma, 0), w = clamp(sigma_max - sigma, 0)/mean; active (B) = mean(> 0) */
int usip_desc_triplet(const float* dpos, const float* dneg, const float* sigma, float gamma, float sigma_max,
                      float* loss, float* active, int B, int M, void* stream);

/* backward of DescPairScanLoss (losses.py:199-233) with upstream gradient g_loss (B,M): anc (B,C,M), pos (B,C,Mp),
 * neg (B,C,Mn), saved (dpos, ipos, dneg, ineg) of usip_desc_pairmin_f32; g_anc / g_pos / g_neg are ACCUMULATED into
 * (pre-zero them). */
int usip_desc_triplet_bwd(const float* anc, const float* pos, const float* neg, const float* dpos, const int32_t* ipos,
                          const float* dneg, const int32_t* ineg, const float* sigma, float gamma, float sigma_max,
                          const float* g_loss, float* g_anc, float* g_pos, float* g_neg, int B, int C, int M, int Mp,
                          int Mn, void* stream);
/* DescCGFLoss (models/losses.py:240-369), the indoor descriptor's triplet loss, without its (B,M,M) and (B,C,M,M)
 * intermediates.  anc_kp (B,3,M) already in the positive frame, pos_kp (B,3,M), anc_desc / pos_desc (B,D,M), sigma (B,M),
 * the reference's three draws u_near, u_out (B,M,M) and u_sel (B,M), all contiguous.  For each anchor m, over the positive
 * keypoints j (d = sqrt((dx*dx + dy*dy) + dz*dz) in fp32 without contraction, mask = d <= radius), first index on ties:
 *   near = argmax (mask ? u_near : 0),  far = argmax -(d + (mask ? 1000 : 0)),  out = argmax (!mask ? u_out : 0)
 * and only those three descriptor distances.  Per cloud (fixed-order sums): scaling = M / (count + 1),
 * w = clamp(sigma_max - sigma, 0) / mean, neg = u_sel < 0.5 ? d_far : d_out,
 * before_clamp = (d_near - neg + gamma) * mask, loss (B,M) = w * clamp(before_clamp, 0) * scaling,
 * active (B) = #(before_clamp > 1e-5) / (count + 1).  Saved for the backward: sel (B,M,4) i32 = near, far, out, flags
 * (bit 0 mask, bit 1 u_sel < 0.5), aux (B,M,4) f32 = d_near, d_far, d_out, before_clamp, cloud (B,2) f32 = scaling, mean
 * weight; sel and aux 16-byte aligned.  Limits: M <= USIP_CGF_MAX_M (the positive keypoints are staged in shared
 * memory), D a multiple of 4 in [4, USIP_CGF_MAX_D] (the backward keeps D/32 channels per lane in registers). */
#define USIP_CGF_MAX_M 2048
#define USIP_CGF_MAX_D 512
int usip_desc_cgf_f32(const float* anc_kp, const float* pos_kp, const float* anc_desc, const float* pos_desc,
                      const float* sigma, const float* u_near, const float* u_out, const float* u_sel, float radius,
                      float gamma, float sigma_max, float* loss, float* active, int32_t* sel, float* aux, float* cloud,
                      int B, int M, int D, void* stream);
/* backward of usip_desc_cgf_f32 for the upstream gradient g_loss (B,M): g_anc, g_pos (B,D,M) OVERWRITTEN.  Per anchor,
 * coef = ((g * scaling) * w) * [before_clamp >= 0] * mask (torch's clamp passes the gradient at 0); the pairs near, far,
 * out receive coef, -coef * [u_sel < 0.5], -coef * [u_sel >= 0.5] times (a - p) / d, exactly 0 where d == 0.  g_pos is
 * gathered positive-major (each positive keypoint walks the anchors in order): bit-reproducible, no atomics. */
int usip_desc_cgf_bwd(const float* anc_desc, const float* pos_desc, const float* sigma, const int32_t* sel,
                      const float* aux, const float* cloud, const float* g_loss, float sigma_max, float* g_anc,
                      float* g_pos, int B, int M, int D, void* stream);
/* backward of usip_l2norm_to_bcm: g (B,C,M), raw rows Y [B*M, C] -> GY [B*M, C]                     networks.py:383 */
int usip_l2norm_bwd(const float* g, const float* Y, int ldy, float* GY, int ldg, int B, int M, int C, void* stream);

/* PointOnSurfaceLoss                                                                   models/losses.py:146-183
 * kp (B,3,M), pc (B,3,N), sn (B,S,N) (first 3 channels = normal), arg (B,M) = nearest point (usip_pairwise_min_f32).
 * loss != NULL: loss (B,M) = (n . (kp-p)/(||kp-p|| + 1e-7))^2;  g_kp != NULL: g_kp (B,3,M) = g (B,M) * dloss/dkp. */
int usip_point_on_surface(const float* kp, const float* pc, const float* sn, const int32_t* arg, const float* g,
                          float* loss, float* g_kp, int B, int M, int N, int S, void* stream);

/* ---- backward of the loss kernels (autograd of models/losses.py / keypoint_detector.py:182-184) ---- */
/* grad of sum_i g_i*gscale*min_d_i: grad_a (B,3,Ma) overwritten, grad_b (B,3,Nb) ACCUMULATED (pre-zero) or NULL */
int usip_pairwise_min_bwd(const float* a, const float* b, const float* min_d, const int32_t* arg,
                          const float* g, float gscale, float* grad_a, float* grad_b,
                          int B, int Ma, int Nb, void* stream);
/* all four grads ACCUMULATE into pre-zeroed buffers; gout = d loss_total / d chamfer_loss (device scalar) */
int usip_chamfer_prob_bwd(const float* src, const float* dst, const float* sig_src, const float* sig_dst,
                          const float* d_sd, const int32_t* i_sd, const float* d_ds, const int32_t* i_ds,
                          const float* gout, float* g_src, float* g_dst, float* g_sig_src, float* g_sig_dst,
                          int B, int M, int N, void* stream);
int usip_transform_points_bwd(const float* g_out, const float* R, const float* scale, float* g_kp,
                              int B, int M, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 5. Backward pass of the fused plan (autograd of models/networks.py:75-162 / layers.py re-derived)
 *
 * Alignment: these kernels move 16-byte vectors, so the following operands must be 16-byte aligned (and their leading
 * dimensions multiples of 4 floats); a misaligned one is rejected with -1 before any launch:
 *   usip_bn_bwd_reduce      G, Y, scale, shift, mean, invstd, part
 *   usip_bn_bwd_apply       G, Y, GY, scale, shift, mean, invstd, c1, c2
 *   usip_groupmax_bwd_apply Y, gz, argsel, GY, scale, mean, invstd, c1, c2
 *   usip_group_sum          G, out
 *   usip_seg_sum            G, out
 *   usip_head_bwd           G
 *   usip_knn_combine_bwd    GY  (GZ may be unaligned or have ld % 4 != 0: it then takes scalar atomics)
 * Two forward calls of sections 2 and 3 follow the same rule:
 *   usip_segmax             X, pooled, arg
 *   usip_knn_combine        Z, Y
 * A column view at an offset that is not a multiple of 4 floats is therefore not accepted by these calls.
 * usip_index_max_f32 accepts any alignment: it moves 16-byte vectors only when data and index are 16-byte aligned and
 * N % 4 == 0, and loads scalars otherwise.
 * ---------------------------------------------------------------------------------------------- */
/* train-mode BatchNorm(+ReLU) backward: partial sums of g_z and g_z*xhat per 128-row tile ([ntiles,2,C]) */
int usip_bn_bwd_reduce(const float* G, int ldg, const float* Y, int ldy, const float* scale, const float* shift,
                       const float* mean, const float* invstd, int relu, float* part, int P, int C, void* stream);
/* -> g_gamma, g_beta (optionally accumulated) and the per-channel constants c1 = g_beta/n, c2 = g_gamma/n */
int usip_bn_bwd_finalize(const float* part, int ntiles, int64_t count, int C, float* g_gamma, float* g_beta,
                         float* c1, float* c2, int accumulate, void* stream);
/* g_y = scale*(g*1[z>0] - c1 - xhat*c2); GY may alias G */
int usip_bn_bwd_apply(const float* G, int ldg, const float* Y, int ldy, const float* scale, const float* shift,
                      const float* mean, const float* invstd, const float* c1, const float* c2, int relu,
                      float* GY, int ldo, int P, int C, void* stream);
/* group-max layers (max_k relu(bn(y_k)), layers.py:433,438) */
int usip_groupmax_bwd_select(const float* Gout, int ldg, const float* gmax, const float* gmin, const int32_t* amax,
                             const int32_t* amin, const float* scale, const float* shift, const float* mean,
                             const float* invstd, float* gz, int32_t* argsel, float* part, int Q, int C, void* stream);
int usip_groupmax_scatter_add(float* G, int ldg, const float* gsrc, const int32_t* argsel, int K, int Q, int C,
                              void* stream);
int usip_groupmax_bwd_apply(const float* Y, int ldy, const float* gz, const int32_t* argsel, const float* scale,
                            const float* mean, const float* invstd, const float* c1, const float* c2, float* GY,
                            int ldo, int K, int P, int C, void* stream);
int usip_group_sum(const float* G, int ldg, float* out, int ldo, int K, int Q, int C, void* stream);
int usip_seg_sum(const float* G, int ldg, const int32_t* seg_off, float* out, int ldo, int B, int N, int M, int C,
                 void* stream);
/* arg-max un-pooling (backward of usip_segmax): G[arg[q,c], c] (+)= gp[q,c] */
int usip_unpool_scatter(float* G, int ldg, const float* gp, int ldp, const int32_t* arg, int Q, int C,
                        int accumulate, void* stream);
/* backward of usip_knn_combine: GZ (pre-zeroed) += scatter of GY by neighbour; gW[:,0:3] += GY^T delta_xyz */
int usip_knn_combine_bwd(const float* GY, int ldg, const float* pts, const int32_t* knn_idx, float* GZ, int ldz,
                         float* gW, int ldw, int B, int M, int K, int C, void* stream);
/* out[c] += sum_r G[r,c] */
int usip_colsum(const float* G, int ldg, float* out, int P, int C, void* stream);
int usip_head_bwd(const float* g_kp, const float* g_sig, const float* out4, int ld, float* G, int B, int M,
                  void* stream);
/* gW[Cout,Cin] += GY[P,Cout]^T * act(X)[P,Cin], act = optional folded BN affine + ReLU (same prologue as forward);
 * precision 1: wgmma 3xTF32 (MN-major operands transposed to K-major in shared memory; precision 4: the same kernel as plain single-pass TF32) when Cout>=64, Cout%4==0, Cin%64==0, P>=4096 (a 64-wide layer fills half of the
 * 128-row tile (two m64 wgmma row blocks) with zero rows); Cin<=8 has an HBM-bound row-streaming kernel; otherwise the register-tiled fp32 SIMT kernel */
int usip_wgrad(const float* GY, int ldg, const float* X, int ldx, const float* in_scale, const float* in_shift,
               int in_relu, float* gW, int ldw, int P, int Cout, int Cin, int precision, void* stream);

/* ---- parameter update (replaces torch.optim.Adam at models/keypoint_detector.py:42-45,207; keypoint_descriptor.py:32-35) ----
 * Adam(betas, eps, weight_decay 0) over flat fp32 buffers of n elements (n % 4 == 0, 16-byte aligned).  `lr_dev` (1 float)
 * and `step_dev` (1 int64, steps taken so far; incremented by the kernel) live in device memory so the launch can be part
 * of a CUDA graph; `arrive` is a zero-initialised uint32 scratch word.  g is multiplied by grad_scale first (1/world for a
 * summed data-parallel gradient). */
int usip_adam_step(float* p, const float* g, float* m, float* v, const float* lr_dev, int64_t* step_dev, uint32_t* arrive,
                   float beta1, float beta2, float eps, float grad_scale, int64_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* USIP_B200_H_ */

/*
 * pn2_api.h — C ABI of libpn2_b200.so: the PointNet++ set-abstraction / feature-propagation
 * geometry ops as hand-written sm_90a CUDA kernels.
 *
 * This is the drop-in boundary for charlesq34/pointnet2's tf_ops/{sampling,grouping,
 * 3d_interpolation}.  Every entry point replaces one of the free "Launcher"/"_cpu" functions the
 * reference's TensorFlow OpKernels call (cited per function, paths relative to the reference
 * root) and keeps that function's scalar/pointer argument order, with a trailing CUDA stream.
 *
 * Conventions (all entry points):
 *   - plain C, no torch/TF types: sizes are `int`, tensors are raw pointers, `stream` is a
 *     cudaStream_t passed as void* (NULL = legacy default stream, as the reference uses).
 *   - device entry points (pn2_*): every pointer is a DEVICE pointer to a dense row-major
 *     float32 / int32 tensor.  The library allocates nothing, frees nothing and never
 *     synchronises; launches are asynchronous on `stream`.  Stateless and re-entrant.
 *   - gradients accumulate with float atomics into a buffer the CALLER has zero-filled, exactly
 *     like the reference (tf_sampling.cpp:174, tf_grouping.cpp:204, tf_interpolate.cpp:258).
 *   - return value: 0 on success, otherwise a cudaError_t (argument errors return
 *     cudaErrorInvalidValue = 1).  pn2_error_string() translates.
 *   - limits: every tensor must have fewer than 2^31 elements per batch entry; n, m < 2^31
 *     (totals are indexed with 64 bits: gather / concat / interpolate are tested beyond 2^32 elements);
 *     ops that put the batch on gridDim.y (ball query, three_nn, the row kernels) take b <= 65535.
 *   - the pn2_set_* tuning hooks store one atomic word each: they may be called from any thread at any
 *     time; a launch sees either the old or the new setting, never a mixture.
 */
#ifndef PN2_API_H_
#define PN2_API_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PN2_API_VERSION 2

/* ---- sampling (replaces tf_ops/sampling/tf_sampling_g.cu launchers) ---------------------- */

/* farthestpointsamplingLauncher(b,n,m,inp,temp,out), tf_sampling_g.cu:203-205.
 * inp (b,n,3) f32; out (b,m) i32.  out[:,0] = 0; selection order and tie-break identical to the
 * reference kernel (:105-170): argmax of the running min squared distance under
 * (value desc, k mod 512 asc, k asc).  `temp` is the reference's (32,n) float scratch
 * (tf_sampling_g.cu:202).  Clouds of up to 425984 points (16 CTAs x 512 threads x 52 points) keep the
 * running minimum in registers and never touch it (temp may be NULL); larger clouds take the reference's
 * global-scratch layout and need pn2_fps_scratch_bytes(b, n) bytes there (cudaErrorInvalidValue if temp
 * is NULL then). */
int pn2_fps(int b, int n, int m, const float* inp, float* temp, int* out, void* stream);

/* Bytes of `temp` pn2_fps / pn2_fps_gather need for (b, n): 0 up to n = 425984, else
 * min(b,32)*n*sizeof(float). */
size_t pn2_fps_scratch_bytes(int b, int n);

/* Same as pn2_fps, also emitting new_xyz (b,m,3) = inp gathered at out (FPS + gather_point in one
 * launch; the pair sample_and_group always issues, utils/pointnet_util.py:40). new_xyz may be NULL. */
int pn2_fps_gather(int b, int n, int m, const float* inp, float* temp, int* out, float* new_xyz, void* stream);

/* Variable-size clouds.  The *_ragged entries take a padded batch: xyz (b,n,3) with n the row stride, and
 * lengths (b,) int32, a DEVICE array: cloud i is its first lengths[i] rows.  Cloud i then gets exactly what the
 * entry without lengths computes on that cloud alone called with n = lengths[i], bit for bit; the padding rows are
 * never read (they may hold NaN, inf or anything else).  The library never reads `lengths` on the host, so every
 * call stays asynchronous and capturable in a CUDA graph: each kernel clamps the value it reads to [1, n], and the
 * kernel variant (and so the cost) is chosen from n.  lengths == NULL means every cloud has n points. */

/* pn2_fps_gather on ragged clouds: out (b,m) indices < lengths[i]; new_xyz (b,m,3) or NULL.  temp as for
 * pn2_fps_gather: pn2_fps_scratch_bytes(b, n) bytes. */
int pn2_fps_gather_ragged(int b, int n, int m, const float* inp, const int* lengths, float* temp, int* out,
                          float* new_xyz, void* stream);

/* probsampleLauncher(b,n,m,inp_p,inp_r,temp,out), tf_sampling_g.cu:198-201 (ProbSample op,
 * tf_sampling.cpp:66-92).  inp_p (b,n) f32 unnormalised probabilities; inp_r (b,m) f32 uniform
 * draws in [0,1]; temp (b,n) f32 caller-provided scratch that receives the cumulative sums (the
 * reference's allocate_temp, tf_sampling.cpp:86); out (b,m) i32 = index of the first cumulative sum
 * >= inp_r * sum.  The float32 cumulative sum keeps the reference's association, so indices are
 * bit-exact.  One CTA per row: b <= 2^31-1. */
int pn2_prob_sample(int b, int n, int m, const float* inp_p, const float* inp_r, float* temp, int* out, void* stream);

/* gatherpointLauncher(b,n,m,inp,idx,out), tf_sampling_g.cu:206-208. out (b,m,3). */
int pn2_gather_point(int b, int n, int m, const float* inp, const int* idx, float* out, void* stream);

/* scatteraddpointLauncher(b,n,m,out_g,idx,inp_g), tf_sampling_g.cu:209-211.
 * inp_g (b,n,3) must be zero-filled by the caller. */
int pn2_gather_point_grad(int b, int n, int m, const float* out_g, const int* idx, float* inp_g, void* stream);
/* The same gradient WITHOUT atomics: pn2_group_point_grad_det with c = 3, nsample = 1, i.e. inp_g[b,i,:] is the
 * sum of out_g[b,j,:] over the j with idx[b,j] == i in ascending j.  inp_g (b,n,3) is overwritten.
 * workspace: pn2_group_point_grad_det_workspace_bytes(b, n, m, 1). */
int pn2_gather_point_grad_det(int b, int n, int m, const float* out_g, const int* idx, float* inp_g,
                              void* workspace, size_t workspace_bytes, void* stream);

/* ---- grouping (replaces tf_ops/grouping/tf_grouping_g.cu launchers) ----------------------- */

/* queryBallPointLauncher(b,n,m,radius,nsample,xyz1,xyz2,idx,pts_cnt), tf_grouping_g.cu:125-128.
 * xyz1 (b,n,3) data, xyz2 (b,m,3) queries; idx (b,m,nsample) i32, pts_cnt (b,m) i32.
 * First nsample hits in ascending index order, row padded with the first hit.  Rows with no hit
 * (undefined in the reference) are written as zeros with pts_cnt = 0. */
int pn2_query_ball_point(int b, int n, int m, float radius, int nsample, const float* xyz1,
                         const float* xyz2, int* idx, int* pts_cnt, void* stream);

/* Same operation and bit-identical results through a uniform grid (cell edge >= 1.01 radius: each query
 * only tests its 3x3x3 cell neighbourhood).  Clouds of 2048 <= n <= 9700 points are served by the
 * shared-memory grid kernel of pn2_ball_group (one launch, no workspace used).  Larger clouds use a
 * caller-provided device workspace of at least pn2_query_ball_point_workspace_bytes(b, n) bytes:
 * clouds whose balls are sparse are binned into a grid in that workspace;
 * the other clouds (dense or badly skewed ones, and any call with workspace == NULL or n < 2048)
 * take the brute-force path above, as does the whole batch when fewer than a quarter of its clouds
 * qualify and any cloud with a NaN coordinate (the reference counts a NaN point as a hit in every
 * ball, which only the scan reproduces).  workspace_bytes == 0 from the size query means "not applicable". */
size_t pn2_query_ball_point_workspace_bytes(int b, int n);
int pn2_query_ball_point_ws(int b, int n, int m, float radius, int nsample, const float* xyz1,
                            const float* xyz2, int* idx, int* pts_cnt, void* workspace,
                            size_t workspace_bytes, void* stream);

/* pn2_query_ball_point_ws in two halves: the grid build needs only the data points (xyz1), so it can
 * run on a second stream while farthest point sampling is still producing the queries; the second
 * half needs the queries.  Both return cudaErrorInvalidValue where pn2_query_ball_point_ws would
 * have fallen back to brute force (no workspace / n < 2048 / radius <= 1e-20). */
int pn2_ball_grid_build(int b, int n, float radius, int nsample, const float* xyz1, void* workspace,
                        size_t workspace_bytes, void* stream);
int pn2_query_ball_point_prebuilt(int b, int n, int m, float radius, int nsample, const float* xyz1,
                                  const float* xyz2, int* idx, int* pts_cnt, const void* workspace,
                                  size_t workspace_bytes, void* stream);

/* pn2_query_ball_point_ws on ragged data clouds (see pn2_fps_gather_ragged): lengths1 (b,) device int32, the
 * lengths of xyz1; the queries xyz2 are dense.  Same paths (chosen from n) and the same workspace query,
 * pn2_query_ball_point_workspace_bytes(b, n).  Every index in idx is < lengths1[i]. */
int pn2_query_ball_point_ragged(int b, int n, int m, float radius, int nsample, const float* xyz1,
                                const int* lengths1, const float* xyz2, int* idx, int* pts_cnt, void* workspace,
                                size_t workspace_bytes, void* stream);

/* groupPointLauncher(b,n,c,m,nsample,points,idx,out), tf_grouping_g.cu:133-136.
 * points (b,n,c); idx (b,m,nsample); out (b,m,nsample,c). */
int pn2_group_point(int b, int n, int c, int m, int nsample, const float* points, const int* idx,
                    float* out, void* stream);

/* groupPointGradLauncher(b,n,c,m,nsample,grad_out,idx,grad_points), tf_grouping_g.cu:137-141.
 * grad_points (b,n,c) must be zero-filled by the caller. */
int pn2_group_point_grad(int b, int n, int c, int m, int nsample, const float* grad_out,
                         const int* idx, float* grad_points, void* stream);

/* The same gradient WITHOUT atomics, for reproducible training: an inverse index (which entries e = j*nsample + k
 * point at each data point) is built in `workspace` (pn2_group_point_grad_det_workspace_bytes(b,n,m,nsample) bytes),
 * then each data point's rows are added in ascending e, the order group_point_grad_cpu (query_ball_point.cpp:70-84)
 * adds them: the result is run-to-run deterministic and bit-identical to that function for any list length.
 * grad_points (b,n,c) is overwritten (rows no entry references become 0): no zero-fill needed.
 * m*nsample >= 2^31 or a workspace that is too small returns cudaErrorInvalidValue without a launch. */
size_t pn2_group_point_grad_det_workspace_bytes(int b, int n, int m, int nsample);
int pn2_group_point_grad_det(int b, int n, int c, int m, int nsample, const float* grad_out, const int* idx,
                             float* grad_points, void* workspace, size_t workspace_bytes, void* stream);

/* selectionSortLauncher(b,n,m,k,dist,outi,out), tf_grouping_g.cu:129-132 (select_top_k).
 * dist (b,m,n); outi (b,m,n) i32, out (b,m,n) f32: the first k columns hold the k smallest values
 * of each row, ascending, and their indices, as k rounds of selection sort with swaps produce;
 * columns >= k hold the permuted remainder exactly as the reference leaves it. */
int pn2_selection_sort(int b, int n, int m, int k, const float* dist, int* outi, float* out, void* stream);

/* knn_point(k, xyz1, xyz2), tf_grouping.py:48-73, without the (b,m,n) distance matrix the reference's
 * graph materialises: xyz1 (b,n,3) data, xyz2 (b,m,3) queries -> val (b,m,k) f32 squared distances
 * ascending, idx (b,m,k) i32.  Bit-identical to the first k columns of selectionSortLauncher
 * (tf_grouping_g.cu:83-123, :129-132) applied to dist[b,j,i] = ((dx*dx + dy*dy) + dz*dz), every product
 * and sum rounded on its own — including the order the selection sort's SWAPS give to equal distances.
 * 1 <= k <= min(n, 128); otherwise cudaErrorInvalidValue (use pn2_selection_sort on a matrix). */
int pn2_knn_point(int b, int n, int m, int k, const float* xyz1, const float* xyz2, float* val, int* idx,
                  void* stream);

/* pn2_knn_point on ragged clouds (see pn2_fps_gather_ragged): lengths1 (b,) device int32, the lengths of the data
 * clouds xyz1, and lengths2 (b,) device int32, the lengths of the query clouds xyz2; either may be NULL (every cloud
 * has n points / m queries).  Each value is clamped to [1, n] (lengths1) or [1, m] (lengths2) on the device; the
 * kernel (and so the cost) is chosen from n and k.  With len_i = lengths1[i], k_i = min(k, len_i) and qlen_i =
 * lengths2[i], every query row j < qlen_i of cloud i holds:
 *   - columns [0, k_i): bit for bit what pn2_knn_point(k_i) returns for the truncated cloud xyz1[i, :len_i] and that
 *     query, ties and NaN / inf distances included;
 *   - columns [k_i, k) (a cloud shorter than k): column 0 again, in val and idx, as the ball query pads a short row
 *     with its first hit (a max-pool over the row is unchanged, and group_point on idx gives the grouped points).
 * Query rows j >= qlen_i are never read and hold idx 0 / val +inf (the missing-neighbour filler of
 * pn2_three_nn_ragged).  Padding rows of xyz1 and xyz2 may hold NaN, inf or anything else.  Still 1 <= k <=
 * min(n, 128).  lengths1 = lengths2 = NULL is pn2_knn_point; self-kNN of a ragged batch passes the same lengths twice. */
int pn2_knn_point_ragged(int b, int n, int m, int k, const float* xyz1, const int* lengths1, const float* xyz2,
                         const int* lengths2, float* val, int* idx, void* stream);

/* ---- 3d_interpolation (replaces the CPU functions of tf_interpolate.cpp; now on the GPU) -- */

/* threenn_cpu(b,n,m,xyz1,xyz2,dist,idx), tf_interpolate.cpp:60-103.
 * xyz1 (b,n,3) unknown, xyz2 (b,m,3) known; dist (b,n,3) f32 SQUARED distances ascending,
 * idx (b,n,3) i32; ties -> lower index; m < 3 -> (+inf, 0) fill.  Bit-exact with the reference's
 * x86 arithmetic (no contraction). */
int pn2_three_nn(int b, int n, int m, const float* xyz1, const float* xyz2, float* dist, int* idx, void* stream);

/* threeinterpolate_cpu(b,m,c,n,points,idx,weight,out), tf_interpolate.cpp:107-127.
 * points (b,m,c); idx, weight (b,n,3); out (b,n,c). */
int pn2_three_interpolate(int b, int m, int c, int n, const float* points, const int* idx,
                          const float* weight, float* out, void* stream);

/* threeinterpolate_grad_cpu(b,n,c,m,grad_out,idx,weight,grad_points), tf_interpolate.cpp:131-153.
 * grad_points (b,m,c) must be zero-filled by the caller. */
int pn2_three_interpolate_grad(int b, int n, int c, int m, const float* grad_out, const int* idx,
                               const float* weight, float* grad_points, void* stream);

/* The same gradient WITHOUT atomics: an inverse index (which unknown points reference each known point) is
 * built in `workspace` (pn2_three_interpolate_grad_det_workspace_bytes(b,n,m) bytes), then one warp per
 * known point adds its contributions in ascending (j, t) order — the order threeinterpolate_grad_cpu adds
 * them, every product and sum rounded on its own — so the result is run-to-run deterministic AND, for known
 * points referenced by at most 256 (j, t) pairs (every point of a non-degenerate layer), bit-identical to the
 * reference's CPU function; longer lists are summed in 8 consecutive pieces combined in order (deterministic,
 * equal to the sequential sum up to rounding).  grad_points (b,m,c) is overwritten: no zero-fill needed. */
size_t pn2_three_interpolate_grad_det_workspace_bytes(int b, int n, int m);
int pn2_three_interpolate_grad_det(int b, int n, int c, int m, const float* grad_out, const int* idx,
                                   const float* weight, float* grad_points, void* workspace,
                                   size_t workspace_bytes, void* stream);

/* ---- fused callers' glue (utils/pointnet_util.py) ------------------------------------------ */

/* sample_and_group's grouping tail, utils/pointnet_util.py:45-54 (SSG) and :179-186 (MSG), in
 * one pass: out[b,j,k,:] = concat of (xyz[idx]-new_xyz[j]) and points[idx] in the order chosen.
 *   xyz (b,n,3), new_xyz (b,m,3), points (b,n,c) or NULL (c = 0), idx (b,m,nsample)
 *   out (b,m,nsample,3+c);  grouped_xyz (b,m,nsample,3) or NULL (the 4th return of
 *   sample_and_group);  xyz_first != 0: [xyz, feats] (SSG, :50), else [feats, xyz] (MSG, :184). */
int pn2_group_concat(int b, int n, int c, int m, int nsample, const float* xyz, const float* new_xyz,
                     const float* points, const int* idx, int xyz_first, float* out,
                     float* grouped_xyz, void* stream);

/* pointnet_fp_module's front end, utils/pointnet_util.py:211-216, in one pass over the unknown
 * points: three_nn -> dist=max(dist,1e-10); w=(1/dist)/sum(1/dist) -> three_interpolate.
 *   xyz1 (b,n,3), xyz2 (b,m,3), points2 (b,m,c) -> out (b,n,c).
 *   dist/idx/weight (b,n,3) outputs are optional (NULL to skip). */
int pn2_three_nn_interpolate(int b, int n, int m, int c, const float* xyz1, const float* xyz2,
                             const float* points2, float* out, float* dist, int* idx, float* weight,
                             void* stream);

/* The whole front end of pointnet_fp_module, utils/pointnet_util.py:211-219, in one pass: the above plus the
 * concat with the dense level's own features: out (b,n,c2+c1) = [interpolated points2 (c2) | points1 (c1)].
 * points1 (b,n,c1) may be NULL with c1 = 0.  Values equal three_nn -> weights -> three_interpolate -> concat. */
int pn2_fp_interpolate_concat(int b, int n, int m, int c2, int c1, const float* xyz1, const float* xyz2,
                              const float* points1, const float* points2, float* out, void* stream);

/* ---- 16-bit features (mixed precision) ----------------------------------------------------------
 * The ops that carry FEATURES also take bfloat16 or float16 feature tensors.  Each typed entry point
 * takes the feature element type as its first argument and otherwise the arguments of the untyped entry
 * of the same name, feature pointers as void*.  Coordinates, weights, distances and indices stay
 * float32 / int32.  Arithmetic is float32: features are upcast exactly, every result is the float32
 * result of the untyped op rounded once (round to nearest even) to the feature type, and copied
 * features are copied bit for bit.  With PN2_F32 a typed entry computes exactly what the untyped one
 * does.  An unknown dtype code or a NULL tensor returns cudaErrorInvalidValue without a launch. */
#define PN2_F32 0
#define PN2_BF16 1
#define PN2_F16 2

int pn2_group_point_typed(int dtype, int b, int n, int c, int m, int nsample, const void* points, const int* idx,
                          void* out, void* stream);
/* The scatter-add runs into `accum` (b,n,c) float32, zero-filled by the caller; grad_points (b,n,c) in `dtype`
 * then receives accum rounded once.  accum may be NULL for PN2_F32 (grad_points is accumulated into, zero-filled
 * by the caller, as in pn2_group_point_grad). */
int pn2_group_point_grad_typed(int dtype, int b, int n, int c, int m, int nsample, const void* grad_out,
                               const int* idx, void* grad_points, float* accum, void* stream);
/* float32 sums in the same order as the untyped entry, rounded once; no accumulator.
 * workspace: pn2_group_point_grad_det_workspace_bytes(b, n, m, nsample) */
int pn2_group_point_grad_det_typed(int dtype, int b, int n, int c, int m, int nsample, const void* grad_out,
                                   const int* idx, void* grad_points, void* workspace, size_t workspace_bytes,
                                   void* stream);
/* points and out in `dtype`; the xyz channels of out are the float32 differences rounded once;
 * grouped_xyz stays float32. */
int pn2_group_concat_typed(int dtype, int b, int n, int c, int m, int nsample, const float* xyz,
                           const float* new_xyz, const void* points, const int* idx, int xyz_first, void* out,
                           float* grouped_xyz, void* stream);
int pn2_three_interpolate_typed(int dtype, int b, int m, int c, int n, const void* points, const int* idx,
                                const float* weight, void* out, void* stream);
/* workspace: pn2_three_interpolate_grad_det_workspace_bytes(b, n, m), as for the untyped entry */
int pn2_three_interpolate_grad_det_typed(int dtype, int b, int n, int c, int m, const void* grad_out,
                                         const int* idx, const float* weight, void* grad_points, void* workspace,
                                         size_t workspace_bytes, void* stream);
int pn2_three_nn_interpolate_typed(int dtype, int b, int n, int m, int c, const float* xyz1, const float* xyz2,
                                   const void* points2, void* out, float* dist, int* idx, float* weight,
                                   void* stream);
int pn2_fp_interpolate_concat_typed(int dtype, int b, int n, int m, int c2, int c1, const float* xyz1,
                                    const float* xyz2, const void* points1, const void* points2, void* out,
                                    void* stream);

/* Interpolation onto ragged clouds (see pn2_fps_gather_ragged): lengths1 (b,) device int32, the lengths of the UNKNOWN
 * side (xyz1, points1, and the n rows of idx / weight / dist / out / grad_out); the known side (xyz2, points, points2) is
 * dense.  Every real row j < lengths1[i] of every output is bit for bit what the entry without lengths computes for it.
 * Padding rows are never read (xyz1, points1 and grad_out may hold NaN or inf there) and hold a fixed filler:
 * idx 0 and dist +inf (the missing-neighbour filler), weight 0, and 0 in every feature output (the points1 half of
 * pn2_fp_interpolate_concat_ragged_typed included).  The gradients into the known features equal those of the call on
 * the truncated clouds: bit for bit for the deterministic one (same workspace formula), within float-atomic rounding for
 * the atomic one.  lengths1 == NULL is the entry without lengths.  lengths1 goes after xyz1, or after weight where there
 * is no xyz1. */
int pn2_three_nn_ragged(int b, int n, int m, const float* xyz1, const int* lengths1, const float* xyz2, float* dist,
                        int* idx, void* stream);
int pn2_three_nn_interpolate_ragged_typed(int dtype, int b, int n, int m, int c, const float* xyz1, const int* lengths1,
                                          const float* xyz2, const void* points2, void* out, float* dist, int* idx,
                                          float* weight, void* stream);
int pn2_fp_interpolate_concat_ragged_typed(int dtype, int b, int n, int m, int c2, int c1, const float* xyz1,
                                           const int* lengths1, const float* xyz2, const void* points1,
                                           const void* points2, void* out, void* stream);
int pn2_three_interpolate_ragged_typed(int dtype, int b, int m, int c, int n, const void* points, const int* idx,
                                       const float* weight, const int* lengths1, void* out, void* stream);
/* float32, float atomics: grad_points (b,m,c) zero-filled by the caller, as for pn2_three_interpolate_grad */
int pn2_three_interpolate_grad_ragged(int b, int n, int c, int m, const float* grad_out, const int* idx,
                                      const float* weight, const int* lengths1, float* grad_points, void* stream);
/* workspace: pn2_three_interpolate_grad_det_workspace_bytes(b, n, m), n the padded size */
int pn2_three_interpolate_grad_det_ragged_typed(int dtype, int b, int n, int c, int m, const void* grad_out,
                                                const int* idx, const float* weight, const int* lengths1,
                                                void* grad_points, void* workspace, size_t workspace_bytes,
                                                void* stream);

/* ---- learned layers: masked batch norm + ReLU (the ragged rows of the segmentation nets) ---------------------------
 * x (rows, c) in `dtype`, keep (rows,) uint8 (a torch bool mask viewed as bytes): batch norm whose training statistics
 * come from the rows with keep[r] != 0 only, followed by ReLU:
 *   y = keep ? max(0, (x - mean) * (invstd * gamma) + beta) : 0,   invstd = rsqrt(var + eps), var biased.
 * Padding rows (keep[r] == 0) of x and dy are never read (they may hold NaN or inf); those of y and dx are written 0.
 * Statistics, gamma, beta, dgamma, dbeta and the running buffers are float32 whatever `dtype` is; arithmetic is float32.
 * The mean and variance are an exact two-pass over register-held groups of rows merged with Chan's formula, never
 * E[x^2] - mean^2.  The row partition depends on (rows, c) only and every sum has a fixed order, with no float atomics:
 * results are bit-identical from run to run and device to device.  Nothing is read back to the host.
 * Forward: writes save_mean / save_invstd (c floats each); when running_mean / running_var are given (both or neither)
 * updates them from the real rows as torch's BatchNorm1d would from a batch of them alone: unbiased variance
 * var * cnt / max(cnt - 1, 1), weight `momentum`, or 1 / *num_batches_tracked (read on the device, already incremented by
 * the caller) when momentum < 0.  gamma / beta may be NULL (affine = False).
 * No real row at all (rows > 0, every keep 0): the mean is 0 / 0 as in layers.masked_batch_norm, so save_mean,
 * save_invstd, running_mean and running_var become NaN; y is all 0, and the backward writes dx 0 and dgamma = dbeta = 0.
 * Backward (y and the saved statistics from the forward): g = keep ? dy * [y > 0] : 0, xhat = (x - mean) * invstd,
 *   dx = keep ? gamma * invstd * (g - sum(g) / cnt - xhat * sum(g * xhat) / cnt) : 0,  dgamma = sum(g * xhat),
 *   dbeta = sum(g)   (sums over the real rows; dgamma / dbeta may be NULL, gamma NULL means 1).
 * Both take a device workspace of pn2_masked_bn_workspace_bytes(rows, c) bytes (16-byte aligned).  rows == 0 launches
 * nothing.  An unknown dtype, a NULL required tensor, c <= 0, rows < 0 or a short workspace return cudaErrorInvalidValue
 * without a launch. */
size_t pn2_masked_bn_workspace_bytes(int rows, int c);
int pn2_masked_bn_relu_forward_typed(int dtype, int rows, int c, const void* x, const unsigned char* keep, const float* gamma,
                                     const float* beta, float eps, float momentum, const long long* num_batches_tracked,
                                     float* running_mean, float* running_var, void* y, float* save_mean, float* save_invstd,
                                     void* workspace, size_t workspace_bytes, void* stream);
int pn2_masked_bn_relu_backward_typed(int dtype, int rows, int c, const void* dy, const void* x, const void* y,
                                      const unsigned char* keep, const float* gamma, const float* save_mean,
                                      const float* save_invstd, void* dx, float* dgamma, float* dbeta, void* workspace,
                                      size_t workspace_bytes, void* stream);

/* The same batch norm + ReLU followed by a max over each cloud's real rows (tf_util.max_pool2d over [num_point, 1],
 * models/pointnet_cls_basic.py:52), without writing the (b, n, c) ReLU output.  x (b, n, c) in `dtype`, keep (b*n) bytes as
 * above (row j of cloud i is real when keep[i*n + j] != 0).  b*n < 2^31.
 * Forward: the statistics, save_mean / save_invstd and the running statistics come from the kernels of
 * pn2_masked_bn_relu_forward_typed on the b*n rows, so they are bit-identical to it.  Then, per (cloud i, column k),
 * out[i, k] = max over the real rows j of y[i, j, k] (y computed and rounded to `dtype` exactly as that entry writes it,
 * values compared as order-preserving keys, so NaN wins) and argmax[i, k] (int32) = the FIRST such row j: where TF's
 * MaxPoolGrad sends the gradient.  A cloud without a real row gets out 0 and argmax -1.
 * Backward (out, argmax and the saved statistics from the forward): g[i, k] = out[i, k] > 0 ? dout[i, k] : 0 at row
 * argmax[i, k] of cloud i and 0 on every other row; dbeta = sum_i g, dgamma = sum_i g * xhat(argmax row), both in
 * ascending i; dx = keep ? gamma * invstd * (g - dbeta / cnt - xhat * dgamma / cnt) : 0 over all b*n rows, cnt the real
 * rows.  No float atomics: bit-identical from run to run.
 * Both take a device workspace of pn2_masked_bn_relu_max_workspace_bytes(b, n, c) bytes (16-byte aligned).  b == 0
 * launches nothing; an unknown dtype, a NULL required pointer, b < 0, n <= 0, c <= 0 or a short workspace return
 * cudaErrorInvalidValue without a launch. */
size_t pn2_masked_bn_relu_max_workspace_bytes(int b, int n, int c);
int pn2_masked_bn_relu_max_forward_typed(int dtype, int b, int n, int c, const void* x, const unsigned char* keep,
                                         const float* gamma, const float* beta, float eps, float momentum,
                                         const long long* num_batches_tracked, float* running_mean, float* running_var,
                                         void* out, int* argmax, float* save_mean, float* save_invstd, void* workspace,
                                         size_t workspace_bytes, void* stream);
int pn2_masked_bn_relu_max_backward_typed(int dtype, int b, int n, int c, const void* dout, const void* x, const void* out,
                                          const int* argmax, const unsigned char* keep, const float* gamma,
                                          const float* save_mean, const float* save_invstd, void* dx, float* dgamma,
                                          float* dbeta, void* workspace, size_t workspace_bytes, void* stream);

/* ---- learned layers: the inference tail of a set-abstraction level (utils/pointnet_util.py:45-54 + :115-124, MSG
 * :179-191) in one launch -----------------------------------------------------------------------------------------------
 * For every group (i, j) of b x m:   row k = concat(xyz[i, idx[i,j,k]] - new_xyz[i,j], points[i, idx[i,j,k]]) in the order
 * xyz_first chooses (as pn2_group_concat; use_xyz == 0 with points: the features alone), then for each of nlayers <= 4
 * layers   row = act((row . W^T + bias - mean) * gamma / sqrt(var + eps) + beta),   and out[i, j, :] = max over k of row.
 * No tensor of b*m*nsample rows is written.  xyz (b,n,3) f32; new_xyz (b,m,3) f32 or NULL (zeros); points (b,n,c) in
 * `dtype` or NULL (c is then taken as 0); idx (b,m,nsample) i32 with every index < n, or NULL (row k is point k; needs
 * nsample == n: the one group that holds the whole cloud).  Per layer l, HOST arrays of nlayers entries holding DEVICE
 * pointers to the module's own float32 tensors: widths[l] = C_out (<= 1024; C_in of layer 0 is c + 3 or c, <= 1027),
 * weight[l] (C_out, C_in) row-major, bias[l] (C_out) or NULL, and for the batch norm bn_mean[l] / bn_var[l] (the running
 * statistics; bn_mean == NULL or bn_mean[l] == NULL: the layer has none), bn_weight[l] / bn_bias[l] (NULL: not affine),
 * bn_eps[l]; relu[l] != 0: act = max(., 0), else the identity.  The kernel derives the per-channel scale and shift
 * itself: there is no folded copy of the parameters that could go stale.
 * out: group (i, j) is written at out + (i*m + j) * out_row_stride, widths[nlayers-1] elements of `dtype`, so one scale
 * of a multi-scale level can write its slice of the concatenated (b, m, sum of widths) tensor.
 * PN2_F32: FP32 fused multiply-adds in ascending channel order.  PN2_BF16 / PN2_F16: tensor-core products of the 16-bit
 * rows with the weights rounded to the 16-bit type, float32 accumulation; the centred xyz are rounded once (as
 * pn2_group_concat_typed), and each layer's result is rounded once after the affine and the activation, in float32.
 * Every output depends on its own group alone and every sum has a fixed order: the same bits on every run, whatever b is
 * and whatever the other groups hold.  NaN propagates through the maximum as in torch.  b == 0 or m == 0 launches
 * nothing; invalid arguments return cudaErrorInvalidValue without a launch. */
int pn2_sa_mlp_max_typed(int dtype, int b, int n, int c, int m, int nsample, const float* xyz, const float* new_xyz,
                         const void* points, const int* idx, int xyz_first, int use_xyz, int nlayers, const int* widths,
                         const float* const* weight, const float* const* bias, const float* const* bn_weight,
                         const float* const* bn_bias, const float* const* bn_mean, const float* const* bn_var,
                         const float* bn_eps, const int* relu, void* out, long long out_row_stride, void* stream);

/* pn2_sa_mlp_max_all_typed: the one group of every cloud (idx == NULL, nsample == n, m == 1), with per-cloud row counts.
 * Arguments and arithmetic as pn2_sa_mlp_max_typed; new_xyz (b,1,3) or NULL; lengths (b,) device int32 or NULL: rows
 * j >= lengths[i], clamped to [1, n], are padding and never read (they may hold NaN).  xyz may be NULL when the rows take
 * no coordinates (use_xyz == 0 with points).  out row i at out + i * out_row_stride.
 * When a cloud has more row tiles than the machine needs, they are dealt out to several CTAs, which atomicMax their
 * partial key maxima into the workspace (zeroed on the stream first); a second launch turns the keys into values.  The
 * split count is a function of b, n, the widths and the SM count, never of the values or the lengths, and the maximum of
 * exact keys does not depend on it: the output is bit-identical to pn2_sa_mlp_max_typed's one-CTA walk and to each
 * cloud computed alone.  Workspace: pn2_sa_mlp_max_all_workspace_bytes(b, widths[nlayers-1]) bytes, 16-byte aligned,
 * required whatever the split.  Nothing is read back to the host: the call can be captured in a CUDA graph.  b == 0
 * launches nothing; invalid arguments return cudaErrorInvalidValue without a launch. */
size_t pn2_sa_mlp_max_all_workspace_bytes(int b, int c_out);
int pn2_sa_mlp_max_all_typed(int dtype, int b, int n, int c, const float* xyz, const float* new_xyz, const void* points,
                             const int* lengths, int xyz_first, int use_xyz, int nlayers, const int* widths,
                             const float* const* weight, const float* const* bias, const float* const* bn_weight,
                             const float* const* bn_bias, const float* const* bn_mean, const float* const* bn_var,
                             const float* bn_eps, const int* relu, void* out, long long out_row_stride, void* workspace,
                             size_t workspace_bytes, void* stream);

/* ---- learned layers, row by row: feature-propagation tails and heads at inference (utils/pointnet_util.py:199-229)
 * ------------------------------------------------------------------------------------------------------------------------
 * The layers of pn2_sa_mlp_max_typed (same per-layer HOST arrays of DEVICE pointers, same arithmetic, nlayers <= 4,
 * widths <= 1024), applied to every row with one output row per input row and no pooling; layer 0 takes up to 1536 inputs.
 * Row r of the result is written at out + r * out_row_stride (widths[nlayers-1] elements of `dtype`).  Every output row
 * depends on its own input row alone and every sum has a fixed order: the same bits whatever the row count and whatever
 * the other rows hold.  Padding rows are never read and are written as 0.  Nothing is read back to the host, so both
 * calls can be captured in a CUDA graph.  Invalid arguments return cudaErrorInvalidValue without a launch.
 *
 * pn2_fp_mlp_typed: row j of cloud i (b x n rows) is concat(interpolate(points2[i] at the 3-NN of xyz1[i,j] in xyz2[i]),
 * points1[i,j]), the first c2 inputs bit-identical to what pn2_fp_interpolate_concat_ragged_typed writes.  xyz1 (b,n,3)
 * f32, lengths1 (b,) device int32 or NULL (rows j >= lengths1[i], clamped to [1, n], are padding), xyz2 (b,m,3) f32,
 * points1 (b,n,c1) in `dtype` or NULL (c1 is then taken as 0), points2 (b,m,c2) in `dtype`, c2 >= 1, c2 + c1 <= 1536,
 * b <= 65535.  The 3-NN indices and weights go through `workspace`, pn2_fp_mlp_workspace_bytes(b, n) bytes (256-byte
 * aligned); two launches.
 * pn2_mlp_rows_typed: row r is x[r] (rows, c) in `dtype`, 1 <= c <= 1536; mask (rows,) bytes, nonzero on the real rows,
 * or NULL (every row is real).  One launch. */
size_t pn2_fp_mlp_workspace_bytes(int b, int n);
int pn2_fp_mlp_typed(int dtype, int b, int n, int m, int c2, int c1, const float* xyz1, const int* lengths1, const float* xyz2,
                     const void* points1, const void* points2, int nlayers, const int* widths, const float* const* weight,
                     const float* const* bias, const float* const* bn_weight, const float* const* bn_bias,
                     const float* const* bn_mean, const float* const* bn_var, const float* bn_eps, const int* relu, void* out,
                     long long out_row_stride, void* workspace, size_t workspace_bytes, void* stream);
int pn2_mlp_rows_typed(int dtype, long long rows, int c, const void* x, const unsigned char* mask, int nlayers,
                       const int* widths, const float* const* weight, const float* const* bias, const float* const* bn_weight,
                       const float* const* bn_bias, const float* const* bn_mean, const float* const* bn_var,
                       const float* bn_eps, const int* relu, void* out, long long out_row_stride, void* stream);

/* ---- the sampling+grouping half of a set-abstraction layer, device-resident ------------------ */

/* query_ball_point + group_point(xyz) in ONE launch (tf_grouping_g.cu:3-57 back to back, as
 * sample_and_group issues them, utils/pointnet_util.py:44-46): idx (b,m,nsample), pts_cnt (b,m) exactly as
 * pn2_query_ball_point writes them, and grouped_xyz (b,m,nsample,3) = xyz1 gathered at idx (NULL to
 * skip), minus the query when center != 0 (the tile+sub of :46, one rounding per coordinate).
 * Each cloud is binned into a uniform grid held in shared memory (or kept in index order when its
 * balls are dense), so it applies when pn2_ball_group_fits(n) != 0 (n <= 9700); otherwise
 * cudaErrorInvalidValue — use pn2_query_ball_point_ws + pn2_group_point. */
int pn2_ball_group_fits(int n);
int pn2_ball_group(int b, int n, int m, float radius, int nsample, const float* xyz1, const float* xyz2,
                   int* idx, int* pts_cnt, float* grouped_xyz, int center, void* stream);

/* farthest_point_sample + gather_point + query_ball_point + group_point(xyz)
 * (utils/pointnet_util.py:40-46) on DEVICE buffers, results bit-identical to the four separate
 * calls: fps_idx (b,m) i32 (the sampling indices; required, it is also the channel between the two
 * kernels), new_xyz (b,m,3), idx (b,m,nsample), pts_cnt (b,m), grouped_xyz (b,m,nsample,3) or NULL,
 * centred on new_xyz when center != 0.
 * When sampling runs one CTA per cloud (n <= 8192) and the cloud fits the shared-memory grid, the
 * ball query + grouping run as a programmatically dependent grid on the SMs the sampling chain
 * leaves idle and consume centroids while they are being produced; the layer then costs the sampling
 * time plus about a microsecond.  Otherwise the four kernels run back to back, using `workspace`
 * (pn2_sa_layer_device_workspace_bytes bytes, may be NULL when that is 0) for the sampling scratch
 * and the ball-query grid.  Independent batches may be issued on different streams: one layer
 * occupies 2*b SMs. */
size_t pn2_sa_layer_device_workspace_bytes(int b, int n, int m, int nsample);
/* The multi-scale form (pointnet_sa_module_msg, utils/pointnet_util.py:156-196: ONE farthest_point_sample +
 * gather_point, then query_ball_point + group_point(xyz) per scale): radii / nsamples / idx / pts_cnt /
 * grouped_xyz are HOST arrays of nscales (<= 16) entries (grouped_xyz, or any entry of it, may be NULL).
 * On the overlapped path every scale's grouping grid runs while the sampling chain is still going. */
int pn2_sa_layer_msg_device(int b, int n, int m, int nscales, const float* radii, const int* nsamples,
                            const float* xyz, int* fps_idx, float* new_xyz, int* const* idx,
                            int* const* pts_cnt, float* const* grouped_xyz, int center, void* workspace,
                            size_t workspace_bytes, void* stream);
/* tuning: grouping CTAs per cloud and scale on the overlapped path (0 = automatic: one) */
void pn2_set_sa_consumer_ctas(int ctas_per_cloud);
int pn2_sa_layer_device(int b, int n, int m, float radius, int nsample, const float* xyz, int* fps_idx,
                        float* new_xyz, int* idx, int* pts_cnt, float* grouped_xyz, int center,
                        void* workspace, size_t workspace_bytes, void* stream);
/* The two layer calls on ragged clouds (see pn2_fps_gather_ragged): `lengths` (b,) device int32 after xyz,
 * otherwise the arguments, paths and workspace of the calls above.  Both the overlapped path and the sequential
 * one honour the lengths; every output index is < lengths[i], so the grouping and any later layer need none. */
int pn2_sa_layer_device_ragged(int b, int n, int m, float radius, int nsample, const float* xyz,
                               const int* lengths, int* fps_idx, float* new_xyz, int* idx, int* pts_cnt,
                               float* grouped_xyz, int center, void* workspace, size_t workspace_bytes,
                               void* stream);
int pn2_sa_layer_msg_device_ragged(int b, int n, int m, int nscales, const float* radii, const int* nsamples,
                                   const float* xyz, const int* lengths, int* fps_idx, float* new_xyz,
                                   int* const* idx, int* const* pts_cnt, float* const* grouped_xyz, int center,
                                   void* workspace, size_t workspace_bytes, void* stream);

/* farthest_point_sample + gather_point + knn_point + group_point(xyz) (sample_and_group(..., knn=True),
 * utils/pointnet_util.py:40-46) on DEVICE buffers, results bit-identical to pn2_fps_gather, pn2_knn_point and
 * group_point(xyz, idx) [- new_xyz] called one after the other: fps_idx (b,m) i32 (required: it is also the channel
 * between the two kernels), new_xyz (b,m,3), idx (b,m,k) i32, dist (b,m,k) f32 = knn_point's val or NULL,
 * grouped_xyz (b,m,k,3) or NULL, centred on new_xyz when center != 0 (one rounding per coordinate).
 * 1 <= k <= min(n, 128), as for pn2_knn_point; otherwise cudaErrorInvalidValue, as for NULL xyz / fps_idx /
 * new_xyz / idx, before any device is touched.
 * The kNN grouping can run as a programmatically dependent grid on the SMs the sampling chain leaves idle (each
 * consumer CTA holds the cloud in shared memory and serves centroids as they are picked) when sampling runs one CTA
 * per cloud (n <= 8192), pn2_sa_knn_layer_fits(n, k) and b < SMs / 2.  It does when a cost comparison from
 * (b, n, m, k) and the SM count says the consumers beat the sequential ops (DESIGN.md §6.2.1: at N 4096 -> 1024 on
 * 132 SMs, b <= 33 at k = 32 and b <= 26 at k = 64).  Otherwise the kernels run back to back, using `workspace`
 * (pn2_sa_knn_layer_workspace_bytes bytes) for the sampling scratch and, when dist is NULL, knn_point's distances.
 * The workspace size follows the same choice: 0 when the call will overlap; on the sequential path it includes the
 * distances, so it is an upper bound when dist is given.  Ask for it on the device, and under the
 * pn2_set_sa_knn_path / pn2_set_sa_consumer_ctas settings, of the call; a workspace that turns out too small is
 * refused with cudaErrorInvalidValue.  Asynchronous; capturable in a CUDA graph after the first call on a device.
 * pn2_set_sa_consumer_ctas also sets the kNN consumer CTAs per cloud (0 = automatic: every SM the sampling
 * leaves per cloud).
 * pn2_sa_knn_layer_fits(n, k) only says that the consumer's shared memory holds the cloud and its W buffers
 * (1 <= k <= min(n, 64)); the overlapped path also needs the conditions above. */
int pn2_sa_knn_layer_fits(int n, int k);
size_t pn2_sa_knn_layer_workspace_bytes(int b, int n, int m, int k);
int pn2_sa_knn_layer_device(int b, int n, int m, int k, const float* xyz, int* fps_idx, float* new_xyz, int* idx,
                            float* dist, float* grouped_xyz, int center, void* workspace, size_t workspace_bytes,
                            void* stream);
/* pn2_sa_knn_layer_device on ragged clouds (see pn2_fps_gather_ragged): `lengths` (b,) device int32 after xyz,
 * otherwise the arguments, paths (still chosen from (b, n, m, k)) and workspace of pn2_sa_knn_layer_device.  Cloud i's
 * fps_idx and new_xyz are pn2_fps_gather_ragged's; idx, dist and grouped_xyz are pn2_knn_point_ragged's (lengths1 =
 * lengths, no query lengths) and their gather, including the column-0 filler of a cloud shorter than k.  Every index
 * is < lengths[i], so the grouping and any later layer need no lengths. */
int pn2_sa_knn_layer_device_ragged(int b, int n, int m, int k, const float* xyz, const int* lengths, int* fps_idx,
                                   float* new_xyz, int* idx, float* dist, float* grouped_xyz, int center,
                                   void* workspace, size_t workspace_bytes, void* stream);
/* measurement switch for pn2_sa_knn_layer_device: 0 = the cost rule (default), 1 = overlapped wherever it can run
 * (fits, one sampling CTA per cloud, an idle SM per cloud), 2 = always sequential.  The outputs do not depend on it. */
void pn2_set_sa_knn_path(int mode);

/* ---- whole-scene segmentation (scannet/scannet_dataset.py:83-118, scannet/train.py:326-427; DESIGN.md §6.9) --------
 * A scene xyz (p,3) f32 (finite) is cut into nx x ny xy blocks, i-major: block (i,j) spans bmin = (lo_x + i*stride,
 * lo_y + j*stride), bmax = bmin + block_size.  Every test is in double on the float32 coordinate, each operation rounded:
 * context member: bmin - padding <= x,y <= bmax + padding; core member: a context member with
 * bmin - 0.001 <= x,y <= bmax + 0.001.  z is not tested.  The caller plans the grid (lo = the scene's minimum, nx the
 * smallest k >= 1 with lo_x + (k-1)*stride + block_size >= the maximum; ny alike), needs 0 < stride <= block_size,
 * padding >= 0 and nx * ny <= 16384.
 *
 * Two calls on one workspace of pn2_scene_blocks_workspace_bytes(p, nx, ny) bytes (256-byte aligned; 0 = invalid grid):
 *   pn2_scene_blocks_count: counts (2*nx*ny) int32 receives the context member count of every block, then the core
 *     member count of every block.  The caller reads them back and plans the batch: a block without core members is
 *     dropped, a block of c members becomes k = ceil(c / max_points) sub-blocks, and sub_begin / sub_count (nx*ny) int32
 *     give each block's first sub-block and k (0 = dropped).
 *   pn2_scene_blocks_fill: writes the padded (b, n) batch.  Member r (in ascending scene index) of a block goes to
 *     sub-block sub_begin + r mod k, row r div k: out_xyz (b,n,3) its coordinates, point_idx (b,n) its scene index,
 *     core (b,n) 1 for a core member; padding rows are 0 / -1 / 0.  occ_off (p+1) and occ_row (occ_off[p] entries) are
 *     the CSR of every point's core rows b*n_row + row, ascending.  b*n*3 < 2^31.
 * Results are the same bits on every run (no atomic order reaches them).  Invalid arguments return cudaErrorInvalidValue
 * without a launch. */
size_t pn2_scene_blocks_workspace_bytes(int p, int nx, int ny);
int pn2_scene_blocks_count(int p, const float* xyz, double lo_x, double lo_y, double block_size, double stride, double padding,
                           int nx, int ny, int* counts, void* workspace, size_t workspace_bytes, void* stream);
int pn2_scene_blocks_fill(int p, const float* xyz, double lo_x, double lo_y, double block_size, double stride, double padding,
                          int nx, int ny, const int* sub_begin, const int* sub_count, int b, int n, float* out_xyz,
                          int* point_idx, unsigned char* core, int* occ_off, int* occ_row, void* workspace,
                          size_t workspace_bytes, void* stream);
/* Ordered merge of block logits: logits (row_end - row_begin, c) in `dtype` hold the rows [row_begin, row_end) of the
 * (b, n) batch pn2_scene_blocks_fill wrote (point_idx, core, occ_off, occ_row as it wrote them).  For every point, its
 * core rows inside the range are added one at a time, in ascending row order, onto accum (p,c) float32:
 * accum = accum + logit, each add rounded.  Merging a batch chunk by chunk gives the bits of one merge over all of it.
 * No atomics, no read-back. */
int pn2_scene_merge_typed(int dtype, int p, int c, int b, int n, int row_begin, int row_end, const void* logits,
                          const int* point_idx, const unsigned char* core, const int* occ_off, const int* occ_row,
                          float* accum, void* stream);

/* ---- training crops (scannet/scannet_dataset.py:27-60, scannet/train.py:181-197, utils/provider.py:52-70; DESIGN.md
 * §6.10) ----------------------------------------------------------------------------------------------------------
 * A scene set: s scenes packed into xyz (p,3) f32 (finite), label (p) int32 in [0, num_class), offsets (s+1) int64
 * (scene k holds rows offsets[k] .. offsets[k+1]-1, none empty; max_scene = the largest scene), lo / hi (s,3) f32 the
 * per-scene extrema (hi_z > lo_z), label_weights (num_class) f32.  Crop i of b is drawn from scene crop_scene[i]
 * (int64, device) with the counter-based draws of DESIGN.md §6.10 keyed by the seed (*seed_dev when seed_dev is not
 * NULL, read on the device, else `seed`): ten attempted columns, the first valid one taken (else the last), its m =
 * min(c, npoints) context members of smallest (hash key, scene-local index) in that order, rows r >= 1 dropped with
 * probability u * max_dropout, x/y rotated about the origin by a random angle when `rotate`.  Outputs (b, npoints):
 * out_xyz (x3) f32, out_label int64, out_weight f32 (label_weights[label] on core rows), point_idx int32 (row of the
 * scene set, -1 on padding), core u8; per crop lengths int32 (>= 1), attempt int32, valid u8.  Padding rows are 0 / -1.
 * A crop_scene value outside [0, s) gives lengths 0 and attempt -1.  npoints <= 16384, b <= 65535, b*npoints*3 < 2^31,
 * 0 <= max_dropout <= 1.  The workspace is pn2_scene_crops_workspace_bytes(b, npoints) bytes, 256-byte aligned
 * (0 = invalid shape).  Same bits on every run; nothing is read back, so the call can be captured in a CUDA graph.
 * Invalid arguments return cudaErrorInvalidValue without a launch. */
size_t pn2_scene_crops_workspace_bytes(int b, int npoints);
int pn2_scene_crops(int s, int p, int max_scene, const float* xyz, const int* label, const long long* offsets, const float* lo,
                    const float* hi, int num_class, const float* label_weights, int b, const long long* crop_scene,
                    long long seed, const long long* seed_dev, int npoints, double max_dropout, int rotate, float* out_xyz,
                    long long* out_label, float* out_weight, int* lengths, int* point_idx, unsigned char* core, int* attempt,
                    unsigned char* valid, void* workspace, size_t workspace_bytes, void* stream);

/* ---- shape batches (modelnet_dataset.py:60-84, modelnet_h5_dataset.py:72-114, utils/provider.py:40-234,
 * part_seg/part_dataset_all_normal.py:83-112, evaluate.py:117-158; DESIGN.md §6.11) -------------------------------
 * A shape set: s shapes packed into xyz (p,3) f32, normals (p,3) f32 or NULL, part (p) int32 or NULL, label (s) int32,
 * offsets (s+1) int64 (shape k holds rows offsets[k] .. offsets[k+1]-1, none empty; max_shape = the largest shape,
 * <= 16384).  Entry e is drawn from shape shape_idx[e] (int64, device; b entries) with the counter-based draws of
 * DESIGN.md §6.11 keyed by the seed (*seed_dev when seed_dev is not NULL, read on the device, else `seed`): the m
 * smallest (hash key, row) pairs of its pool (rows 0 .. min(P, npoints)-1, or all P rows when subset_random), rows
 * r >= 1 dropped with probability u * max_dropout, then xyz' = (p M) s + t + j and n' = n M in double, rounded once:
 * M = Ry(theta) Rp (rotate, perturb), s in [scale_lo, scale_hi) (scale_on), t in [-shift, shift), j = clip(jitter_sigma
 * N(0,1), +-jitter_clip) per coordinate (jitter_on); a step that is off is the identity.  votes > 0: b * votes entries,
 * entry e = v*b + i the vote v of shape_idx[i], rotated by v / votes of a turn about y, its first npoints rows in a
 * seeded order; every other step must then be off.  Outputs (E, npoints), E the entries: out_points (x3, or x6 with
 * with_normals) f32, out_part int64 (NULL: not written; needs part), point_idx int32 (row of the set, -1 on padding);
 * per entry out_label int64, lengths int32.  Padding rows are 0 / -1.  A shape_idx value outside [0, s) gives lengths 0.
 * npoints <= 16384, E * npoints * channels < 2^31, 0 <= max_dropout <= 1, shift >= 0, jitter_clip > 0.  No workspace.
 * Same bits on every run; nothing is read back, so the call can be captured in a CUDA graph.  Invalid arguments return
 * cudaErrorInvalidValue without a launch. */
int pn2_shape_batch(int s, int p, int max_shape, const float* xyz, const float* normals, const int* label, const int* part,
                    const long long* offsets, int b, const long long* shape_idx, long long seed, const long long* seed_dev,
                    int votes, int npoints, int subset_random, int rotate, int perturb, int scale_on, double scale_lo,
                    double scale_hi, double shift, int jitter_on, double jitter_sigma, double jitter_clip,
                    double max_dropout, int with_normals, float* out_points, long long* out_label, long long* out_part,
                    int* lengths, int* point_idx, void* stream);

/* ---- virtual scans (scannet/scene_util.py virtual_scan, scannet/scannet_dataset.py:122-166; DESIGN.md §6.12) -------
 * A scene set as for pn2_scene_crops, plus mean (s,3) f64, each scene's mean in float64.  Entry i of b scans scene
 * scan_scene[i] (int64, device) from the view scan_mode[i] (int64, device): -1 a random view from the counter-based
 * draws of DESIGN.md §6.12 keyed by the seed (*seed_dev when seed_dev is not NULL, read on the device, else `seed`),
 * any other m the fixed view at azimuth pi/4 m.  200 x 150 rays; a point is near when its nearest ray in (azimuth,
 * elevation) is within 0.01 (ties: the lower ray), and visible when it is near, at least 100 points are near, and its
 * range is the minimum over the near points of its ray.  The rows are the m = min(visible, npoints) visible points of
 * smallest (hash key, scene-local index), in that order.  Outputs (b, npoints): out_xyz (x3) f32 (the scene's own
 * coordinates), out_label int64, out_weight f32 (label_weights[label], 0 on every row of an invalid entry), point_idx
 * int32 (row of the scene set, -1 on padding); per entry lengths int32 (m), visible int32 (the visible points; 0 when
 * fewer than 100 are near; -1 for a scan_scene value outside [0, s), with lengths 0), valid u8 (visible >= min_points).
 * Padding rows are 0 / -1.  npoints <= 16384, b <= 4096, b*npoints*3 < 2^31, min_points >= 0.  The workspace is
 * pn2_virtual_scans_workspace_bytes(b, max_scene, npoints) bytes, 256-byte aligned (0 = invalid shape); it holds
 * per-entry ray tables, cell offsets and z-buffers and a bitmap of max_scene bits per entry.  Same bits on every run;
 * nothing is read back, so the call can be captured in a CUDA graph.  Invalid arguments return cudaErrorInvalidValue
 * without a launch. */
size_t pn2_virtual_scans_workspace_bytes(int b, int max_scene, int npoints);
int pn2_virtual_scans(int s, int p, int max_scene, const float* xyz, const int* label, const long long* offsets,
                      const double* mean, int num_class, const float* label_weights, int b, const long long* scan_scene,
                      const long long* scan_mode, long long seed, const long long* seed_dev, int npoints, int min_points,
                      float* out_xyz, long long* out_label, float* out_weight, int* lengths, int* point_idx, int* visible,
                      unsigned char* valid, void* workspace, size_t workspace_bytes, void* stream);

/* ---- dataset text (modelnet_dataset.py:84, part_seg/part_dataset_all_normal.py:88; DESIGN.md §6.18) --------------
 * F files, concatenated: text (nbytes) u8 on the device, file f at bytes file_off[f] .. file_off[f+1]-1 (file_off
 * (F+1) int64, device; offsets are clamped to [0, nbytes]).  A file is parsed on the device when every line of it is
 * exactly ncol fields and a terminator ("\n", "\r\n", or none on the last line); fields are separated by one ','
 * (PN2_DELIM_COMMA) or by runs of ' ' / '\t' that may also lead and trail the line (PN2_DELIM_WHITESPACE), and a field
 * is [+-]? (digits [. digits]? | . digits) ([eE] [+-]? digits)? whose significant digits M (leading zeros stripped)
 * and decimal exponent E satisfy M <= 2^53 and |E| <= 22.  Its rows then hold exactly
 * np.loadtxt(file, delimiter=...).astype(np.float32) (one row stays a row).  Any other file gets the reason code of
 * its first line outside that grammar and is the caller's to parse.
 *
 * pn2_text_rows_scan: rows (F) int64, the file's lines; status (F) int32, PN2_TEXT_OK or a reason code.
 * pn2_text_rows_parse: for every file whose status (the scan's, device) is PN2_TEXT_OK, its first min(rows, keep)
 * rows as float32 to out (out_rows, ncol) from row row_off[f] (int64, device) on; rows past out_rows are not written.
 * 1 <= ncol <= 64, keep >= 0.  Nothing is allocated or read back.  Invalid arguments return cudaErrorInvalidValue
 * without a launch. */
#define PN2_DELIM_WHITESPACE 0
#define PN2_DELIM_COMMA 1
#define PN2_TEXT_OK 0
#define PN2_TEXT_SYNTAX 1   /* a byte or a field outside the grammar ("nan", "inf", "1_0", "1.", ", " ...) */
#define PN2_TEXT_FIELDS 2   /* a line of other than ncol fields */
#define PN2_TEXT_BLANK 3    /* an empty or all-blank line */
#define PN2_TEXT_CR 4       /* a '\r' that does not end a "\r\n" */
#define PN2_TEXT_COMMENT 5  /* a '#' */
#define PN2_TEXT_INEXACT 6  /* a value outside the exact conversion: M > 2^53 or |E| > 22 */
int pn2_text_rows_scan(int num_files, const unsigned char* text, const long long* file_off, long long nbytes, int ncol,
                       int delim, long long* rows, int* status, void* stream);
int pn2_text_rows_parse(int num_files, const unsigned char* text, const long long* file_off, long long nbytes, int ncol,
                        int delim, const int* status, long long keep, const long long* row_off, float* out,
                        long long out_rows, void* stream);

/* ---- point-cloud rendering (utils/render_balls_so.cpp render_ball, utils/show3d_balls.py; DESIGN.md §6.16) --------
 * Image i of b (out (b, h, w, 3) u8) is what render_ball(h, w, show, len_i, xyz_i, c0, c1, c2, r) writes for cloud i
 * alone on a canvas filled with background[0..2] (a host array of 3 bytes): xyz (b, n, 3) int32 (x the row, y the
 * column), colors (b, n, 3) f32 holding c0, c1, c2 per point (NULL: 255 everywhere), lengths (b,) int32 on the device
 * (NULL: n), clamped to [0, n]; padding rows are never read and a cloud of length 0 renders as background.  r < 1 is
 * taken as 1; r <= 4096.  Every coordinate of a real point must satisfy |x|, |y|, |z| <= 2^30 (not checked).  Bit for
 * bit: the pixel goes to the largest key (z2 + 2^31) << 32 | ~i over the (point, pattern entry) pairs on the canvas
 * with z2 > -2100000000, and its colour is recomputed in render_ball's arithmetic order.  b <= 65535, h * w < 2^31,
 * n < 2^30 / 3.  The workspace is pn2_render_balls_workspace_bytes(b, h, w) bytes, 256-byte aligned (0 = invalid
 * shape): 8 bytes per pixel per image and 8 per image.  Nothing is read back, so the call can be captured in a CUDA
 * graph.  b = 0 does nothing; invalid arguments return cudaErrorInvalidValue without a launch. */
size_t pn2_render_balls_workspace_bytes(int b, int h, int w);
int pn2_render_balls(int b, int n, int h, int w, const int* xyz, const float* colors, const int* lengths, int r,
                     const unsigned char* background, void* workspace, size_t workspace_bytes, unsigned char* out,
                     void* stream);
/* pn2_render_balls, and counters (2 u64 on the device, added to) += the pixel atomics issued and the ones skipped
 * because the pixel already held a key at least as large: for measurement. */
int pn2_render_balls_counted(int b, int n, int h, int w, const int* xyz, const float* colors, const int* lengths, int r,
                             const unsigned char* background, void* workspace, size_t workspace_bytes,
                             unsigned char* out, unsigned long long* counters, void* stream);
/* showpoints' view transform of b clouds xyz (b, n, 3) f64 with lengths as above, for v views: p' = (p - mean) /
 * ((radius * 2.2) / size) over the cloud's real points in float64 (mean in a fixed order, so a cloud's result does not
 * depend on the rest of the batch; a cloud whose points coincide maps to 0), then p' R_v + (size/2, size/2, 0) with
 * rotations (v, 3, 3) f64 on the host (row-major, R_v = Rx Ry zoom), clamped to +-2^30 and truncated toward zero into
 * out (b, v, n, 3) int32; padding rows are 0.  The workspace holds 32 * b bytes, 8-byte aligned.  b <= 65535,
 * n < 2^30 / 3, v >= 1, size >= 1. */
int pn2_project_points(int b, int n, int v, const double* xyz, const int* lengths, const double* rotations, int size,
                       void* workspace, size_t workspace_bytes, int* out, void* stream);

/* ---- host-buffer entry point (the reference feeds numpy through feed_dict) ----------------- */

/* One SSG set-abstraction sampling+grouping layer (farthest_point_sample + gather_point +
 * query_ball_point + group_point(xyz), utils/pointnet_util.py:40-45) on HOST buffers:
 * copies h_xyz (b,n,3) to the device, runs the four ops, copies new_xyz (b,m,3), idx (b,m,nsample),
 * pts_cnt (b,m) and grouped_xyz (b,m,nsample,3; NOT centred) back — through pn2_sa_layer_device.
 * Any of the four output pointers may be NULL: that result is neither copied back nor, for
 * grouped_xyz, computed (a caller that regroups on the host saves 3/4 of the device-to-host bytes).
 * Host buffers should be pinned for the copies to be asynchronous.  `workspace` is a device buffer of at least
 * pn2_sa_layer_workspace_bytes(b,n,m,nsample) bytes supplied by the caller.  Asynchronous on
 * `stream`: synchronise the stream before reading the outputs. */
size_t pn2_sa_layer_workspace_bytes(int b, int n, int m, int nsample);
int pn2_sa_layer_host(int b, int n, int m, float radius, int nsample, const float* h_xyz,
                      float* h_new_xyz, int* h_idx, int* h_pts_cnt, float* h_grouped_xyz,
                      void* workspace, size_t workspace_bytes, void* stream);
/* The same layer on a batch of variable-size clouds, packed on the host (DESIGN.md §6.8).
 * h_xyz is PACKED: cloud i is rows [off_i, off_i + h_lengths[i]) of a (sum of lengths, 3) float32 host array, off
 * the exclusive prefix sum of the lengths, no padding.  n is the capacity: every length must satisfy
 * 1 <= h_lengths[i] <= n, otherwise cudaErrorInvalidValue before anything is enqueued (no clamping).  The outputs
 * and their NULL rules are pn2_sa_layer_host's; cloud i's are bit for bit what pn2_sa_layer_host returns for that
 * cloud alone with n = h_lengths[i].
 * h_lengths is read synchronously during the call (validation, copy size and row stride) and again by the
 * asynchronous copy that carries it to the device; h_xyz is read only by the asynchronous copy.  Keep both
 * unchanged until the stream has passed the copies.
 * Enqueued on `stream`: one copy of the b lengths, one copy of the 12 * sum(lengths) packed bytes, one kernel that
 * writes the real rows into a padded (b, n_run, 3) device batch, n_run = max(lengths) (padding rows are neither
 * written nor read), pn2_sa_layer_device_ragged(b, n_run, ...), then the copies back.  The sampling plan and the
 * ball-query path are therefore chosen for the longest cloud of the batch, not for the capacity.  Nothing is
 * synchronised.  `workspace`: a 256-byte-aligned device buffer of at least
 * pn2_sa_layer_host_ragged_workspace_bytes(b,n,m,nsample) bytes (cudaErrorInvalidValue when smaller,
 * cudaErrorMisalignedAddress when misaligned). */
size_t pn2_sa_layer_host_ragged_workspace_bytes(int b, int n, int m, int nsample);
int pn2_sa_layer_host_ragged(int b, int n, int m, float radius, int nsample, const float* h_xyz,
                             const int* h_lengths, float* h_new_xyz, int* h_idx, int* h_pts_cnt,
                             float* h_grouped_xyz, void* workspace, size_t workspace_bytes, void* stream);
/* The multi-scale layer (pointnet_sa_module_msg, utils/pointnet_util.py:156-196) on HOST buffers (DESIGN.md §6.8):
 * ONE farthest_point_sample + gather_point for every scale, then query_ball_point + group_point(xyz) per scale,
 * through pn2_sa_layer_msg_device.  radii, nsamples, h_idx, h_pts_cnt and h_grouped_xyz are HOST arrays of nscales
 * (1..16) entries, as for pn2_sa_layer_msg_device: h_new_xyz (b,m,3), every h_idx[k] (b,m,nsamples[k]) and
 * h_pts_cnt[k] (b,m) are required; h_grouped_xyz, or any entry of it, may be NULL, and such a scale's grouped_xyz
 * (b,m,nsamples[k],3; NOT centred) is neither computed nor copied back.  Scale k's outputs are bit for bit those of
 * pn2_sa_layer_host with (radii[k], nsamples[k]) alone: the sampling is shared.
 * Enqueued on `stream`: one copy of the 12*b*n input bytes, pn2_sa_layer_msg_device(center = 0), then the copies
 * back: new_xyz, then each scale's idx, pts_cnt and (when wanted) grouped_xyz.  Nothing is synchronised.
 * A bad count or shape, nscales outside 1..16, a radius that is not positive (or NaN), a non-positive nsample, a NULL
 * required pointer or a workspace smaller than pn2_sa_layer_msg_host_workspace_bytes(b,n,m,nscales,nsamples) returns
 * cudaErrorInvalidValue, a workspace not 256-byte aligned cudaErrorMisalignedAddress, before any device call.  The
 * workspace size is 0 for invalid arguments. */
size_t pn2_sa_layer_msg_host_workspace_bytes(int b, int n, int m, int nscales, const int* nsamples);
int pn2_sa_layer_msg_host(int b, int n, int m, int nscales, const float* radii, const int* nsamples,
                          const float* h_xyz, float* h_new_xyz, int* const* h_idx, int* const* h_pts_cnt,
                          float* const* h_grouped_xyz, void* workspace, size_t workspace_bytes, void* stream);
/* The multi-scale layer on packed variable-size clouds: h_xyz and h_lengths as for pn2_sa_layer_host_ragged (every
 * length checked on the host, 1 <= h_lengths[i] <= n, before anything is enqueued), everything else as for
 * pn2_sa_layer_msg_host.  Enqueued: the lengths copy, one copy of the 12 * sum(lengths) packed bytes, the unpack
 * kernel at the row stride n_run = max(lengths), pn2_sa_layer_msg_device_ragged(b, n_run, ...), then the copies back.
 * Cloud i's outputs are bit for bit what pn2_sa_layer_msg_host returns for that cloud alone with n = h_lengths[i]. */
size_t pn2_sa_layer_msg_host_ragged_workspace_bytes(int b, int n, int m, int nscales, const int* nsamples);
int pn2_sa_layer_msg_host_ragged(int b, int n, int m, int nscales, const float* radii, const int* nsamples,
                                 const float* h_xyz, const int* h_lengths, float* h_new_xyz, int* const* h_idx,
                                 int* const* h_pts_cnt, float* const* h_grouped_xyz, void* workspace,
                                 size_t workspace_bytes, void* stream);

/* ---- introspection ------------------------------------------------------------------------- */
int pn2_api_version(void);
const char* pn2_error_string(int code);
/* number of kernel launches (not memcpys) this library has issued in this process */
unsigned long long pn2_launch_count(void);
/* the exact d2-domain threshold the ball query uses for `radius`
 * (largest float t with max(sqrtf(t),1e-20f) < radius; negative if no t qualifies) */
float pn2_ball_threshold(float radius);
/* tuning override for experiments: threads, points/thread, cluster size of the FPS kernel
 * (cluster 0 = global-scratch fallback); threads = 0 restores the built-in plan.
 * The per-step update exists in two bit-identical forms — the plain scalar chain and the packed FP32x2 /
 * value-only chain that is the built-in choice wherever it is instantiated (environment: PN2_FPS_PACKED=0/1 for
 * one CTA per cloud, PN2_FPS_PACKED_CLUSTER=0/1 for clusters).  An override can name the chain: cluster = -1 /
 * -2 = one CTA per cloud with the plain / packed chain; for cluster plans the two low bits of `threads`
 * (threads is a multiple of 128): +1 = packed, +2 = plain. */
void pn2_set_fps_config(int threads, int points_per_thread, int cluster);
/* the kernel variant pn2_fps would launch for (b, n): threads per CTA, points per thread and
 * cluster size (1 = one CTA per cloud, >= 2 = thread-block cluster per cloud, 0 = global-scratch
 * fallback) */
int pn2_fps_plan(int b, int n, int* threads, int* points_per_thread, int* cluster);
/* how many thread-block clusters of the FPS cluster kernel (threads, points/thread, cluster size) the
 * current device can hold at once (cudaOccupancyMaxActiveClusters); 0 = no such kernel / cannot launch.
 * The planner uses it to keep every cloud's cluster co-resident. */
int pn2_fps_cluster_capacity(int threads, int points_per_thread, int cluster);
/* tuning override: lanes cooperating on one ball query (1,2,4,..,32); 0 restores the heuristic */
void pn2_set_bq_group(int lanes_per_query);
/* tuning override for pn2_query_ball_point_ws: 0 = automatic, 1 = brute force only, 2 = the workspace
 * (global-memory) grid path even where the shared-memory grid kernel would apply */
void pn2_set_bq_mode(int mode);

#ifdef __cplusplus
}
#endif
#endif /* PN2_API_H_ */

/*
 * delora_b200 — C ABI of the H100-native (sm_90a) DeLORA hot path.
 *
 * The reference (leggedrobotics/delora) is pure Python with no FFI layer of its own; its
 * operator surface for this path is the set of Python methods cited on each entry point
 * below (paths relative to the reference root).  Every function here is what a ctypes
 * binding of that method calls; `delora_b200/_lib.py` is that binding and INTEGRATION.md
 * shows the stub a maintainer of the reference would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller (torch allocates), unless the
 *     parameter name starts with `h_`;
 *   - `stream` is a `cudaStream_t` passed as `void*` (NULL = legacy default stream); all
 *     work is enqueued on it and nothing synchronises the device;
 *   - return value: 0 = ok, non-zero = error; `delora_last_error()` returns a thread-local,
 *     NUL-terminated description of the last failure on the calling thread;
 *   - no global mutable state: scratch memory is passed in by the caller.  Functions are
 *     re-entrant per stream.
 *   - batches: `B` independent scans / scan pairs per call, one launch per operator for the
 *     whole batch.  Variable-length lists are padded to a stride with a device-side count.
 */
#ifndef DELORA_B200_H_
#define DELORA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DELORA_B200_ABI_VERSION 3

/* float4-packed list element: (x, y, z, tag).  `tag` is an int32 bit pattern or a float flag,
 * as documented per array. */
typedef struct { float x, y, z, w; } delora_f4;

/* loss switches (config/hyperparameters.yaml:14-19) */
#define DELORA_LOSS_PO2PO        1u   /* point_to_point_loss                 */
#define DELORA_LOSS_PO2PL        2u   /* point_to_plane_loss                 */
#define DELORA_LOSS_PL2PL        4u   /* plane_to_plane_loss                 */
#define DELORA_NORMAL_LINEAR     8u   /* normal_loss: "linear" (default "squared") */
#define DELORA_ICP_STATS       256u  /* diagnostic: count the work of the NN search (delora_icp_stats) */
#define DELORA_LOSS_IDENTITY_FIT 512u /* delora_odometry_train_step only: the identity pre-training objective
                                         (unsupervised_at_start: False, src/deploy/deployer.py:324-327) */
#define DELORA_TRAIN_NORMALIZATION_SCALING 1024u /* delora_odometry_train_step only: the model is trained with
                                                    normalization_scaling (see _train_step; needs w_pre > 0) */
#define DELORA_TRAIN_DROPOUT 2048u /* delora_odometry_train_step only: the model is trained with use_dropout (the
                                      three dropouts of the reference's encoder; see _train_step) */
#define DELORA_LOSS_PO2PO_ALONE 4096u /* po2po_alone (src/losses/icp_losses.py:36-46), read by the odometry training,
                                         streams and adapting entry points: every surviving point of scan_2 is paired
                                         with its nearest surviving point of scan_1 and no normal plays a part.  Needs
                                         DELORA_LOSS_PO2PO; refuses DELORA_LOSS_PO2PL, _PL2PL and DELORA_NORMAL_LINEAR.
                                         The outputs are the bits of the same call with DELORA_LOSS_PO2PO alone on
                                         all-zero normal grids; no normal is estimated (delora_project_points_fwd). */

/* number of floats in one row of the `losses` output of delora_icp_fwd_bwd */
#define DELORA_LOSS_ROW 8   /* [po2po, po2pl, pl2pl, M_pairs, M_po2po, 0, 0, 0] */
/* number of floats per block-partial row in the icp workspace */
#define DELORA_ICP_PARTIAL 40
/* number of floats in one row of the `info` output of delora_icp_dense_information:
 * [0, 36) H row-major, [36, 42) its eigenvalues ascending, [42, 78) the unit eigenvector of eigenvalue k at 42 + 6 k,
 * 78 M_pairs, 79 M_po2po.  Equal eigenvalues keep the order of the eigen-solve's columns (the lower column first): on a
 * diagonal H the eigenvectors of a repeated eigenvalue are the unit axes in increasing index. */
#define DELORA_INFO_ROW 80

int         delora_abi_version(void);
const char* delora_last_error(void);

/* ---------------------------------------------------------------------------------------
 * Spherical projection.
 * Replaces utility.projection.ImageProjectionLayer.project_to_img
 *   (src/utility/projection.py:48-106; (u,v): :21-31; dedupe: :34-43).
 *
 * points     [B, C, n_stride] fp32 channels-first (x, y, z, extra channels...)
 * n_points   [B] int32 (device): valid points of each scan (<= n_stride)
 * keys       [B, H*W] uint64 scratch.  MUST be all-ones (0xFF bytes) on entry; it is all-ones
 *            again on exit (the resolve pass resets it), so one memset at allocation suffices.
 * image      [B, C+1, H, W] fp32 out: channels of the closest point per pixel + its range;
 *            empty pixels are 0.
 * index_map  [B, H, W] int32 out: index (into the scan) of the point kept in the pixel, -1 if empty.
 * hfov/vfov  radians, as the reference's bin scripts hand them over (bin/run_training.py:62-67).
 * div_mode   0: (a - f0) / span   (torch CPU op sequence, the golden vectors)
 *            1: (a - f0) * (1/span)  (torch CUDA's scalar-divide kernel) — see DESIGN.md.
 * Tie rule: equal fp32 range in one pixel -> lowest point index wins.
 */
int delora_project_fwd(const float* points, const int32_t* n_points, int B, int C, int n_stride,
                       int H, int W, double hfov0, double hfov1, double vfov0, double vfov1,
                       int div_mode, uint64_t* keys, float* image, int32_t* index_map, void* stream);

/* (u, v) of every point, un-rounded, in the ORIGINAL point order (the reference returns them
 * permuted by its range sort; see delora_sort_by_range).  src/utility/projection.py:21-31.
 * u, v: [B, n_stride] fp32 out; range: [B, n_stride] fp32 out (may be NULL). */
int delora_project_uv(const float* points, const int32_t* n_points, int B, int C, int n_stride,
                      int H, int W, double hfov0, double hfov1, double vfov0, double vfov1,
                      int div_mode, float* u, float* v, float* range, void* stream);

/* Stable ascending sort of each scan's points by fp32 range (ties: lower index first):
 * the order `torch.argsort(range)` imposes in src/utility/projection.py:63-67, made
 * deterministic.  LSD radix sort, 4 passes of 8 bits, one launch set for the batch.
 * range      [B, n_stride] fp32, any values: ordered as torch.argsort(stable=True) orders them
 *            (-0 equals +0, every NaN sorts last in index order)
 * order      [B, n_stride] int32 out: point indices in ascending (range, index) order
 * scratch    bytes >= delora_sort_scratch_bytes(B, n_stride)
 */
int64_t delora_sort_scratch_bytes(int B, int n_stride);
int delora_sort_by_range(const float* range, const int32_t* n_points, int B, int n_stride,
                         int32_t* order, void* scratch, void* stream);

/* ---------------------------------------------------------------------------------------
 * Per-pixel normals.
 * Replaces preprocessing.normal_computation.NormalsComputer.compute_normal_vectors
 *   (src/preprocessing/normal_computation.py:89-122, :53-87) and utility.linalg.cov
 *   (src/utility/linalg.py:33-56).
 *
 * image      [B, C_img, H, W] fp32 (first three channels are x, y, z)
 * nb_h, nb_w neighbourhood side lengths (7, 11); patch = (2*(nb_h/2)+1) x (2*(nb_w/2)+1), edge-clamped
 * normals    [B, 3, H, W] fp32 out (may be NULL); 0 where the pixel is not valid (x!=0 & y!=0 & z!=0)
 *            or has fewer than max(`min_neighbors`, 2) range-gated neighbours (the pixel itself included): a set of
 *            one point has no covariance, so min_neighbors 0 and 1 act as 2 (the reference's eigen-solve raises there).
 * epsilon_range  the range gate |(|q| - |c|)| <= epsilon_range; NaN, infinite or negative is refused (the same rule as
 *            delora_odometry_train_params and delora_odometry_residual_params).
 * pts_grid   [B, H*W] float4 out or NULL: (x, y, z, bits(pixel id)) of valid pixels, (+inf,+inf,+inf,-1) else
 * nrm_grid   [B, H*W] float4 out or NULL: (nx, ny, nz, has_normal ? 1 : 0)   (both or neither)
 *            -- the dense layout delora_icp_dense_fwd_bwd consumes (one point per spherical cell).
 */
int delora_normals_fwd(const float* image, int B, int C_img, int H, int W, int nb_h, int nb_w,
                       float epsilon_range, int min_neighbors, float* normals,
                       delora_f4* pts_grid, delora_f4* nrm_grid, void* stream);

/* Projection followed by the normals' dense grids, in one call: the same arguments and outputs as delora_project_fwd
 * (keys all-ones on entry and on exit) followed by delora_normals_fwd(image, B, C+1, H, W, nb_h, nb_w, epsilon_range,
 * min_neighbors, NULL, pts_grid, nrm_grid), bit-identical to those two calls.  For C = 3 or 4 and the 7x11
 * neighbourhood the normals kernel resolves the projection's depth keys itself (no separate resolve pass, the image
 * is written but not read back); other C or neighbourhoods run the two calls.
 * pts_grid, nrm_grid  [B, H*W] float4 out, as delora_normals_fwd writes them (both required); epsilon_range and
 *                     min_neighbors as there (a NaN, infinite or negative epsilon_range refused, fewer than 2 neighbours: no normal)
 * split_event         cudaEvent_t or NULL: recorded on `stream` after the projection's scatter pass (or after the whole
 *                     projection on the two-call path) and before the normals kernel, for per-kernel timing.
 */
int delora_project_normals_fwd(const float* points, const int32_t* n_points, int B, int C, int n_stride,
                               int H, int W, double hfov0, double hfov1, double vfov0, double vfov1,
                               int div_mode, uint64_t* keys, float* image, int32_t* index_map, int nb_h, int nb_w,
                               float epsilon_range, int min_neighbors, delora_f4* pts_grid, delora_f4* nrm_grid,
                               void* split_event, void* stream);

/* The points-only front end of DELORA_LOSS_PO2PO_ALONE: delora_project_normals_fwd without the normals.  The same
 * depth keys and resolve pass, so image, index_map and pts_grid are bit-identical to that call's (for any
 * neighbourhood); nrm_grid [B, H*W] float4 is written all zeros.  No neighbourhood is staged, no tap accumulated and no
 * eigen-solve run.  Keys all-ones on entry and on exit.  C must be 3 or 4. */
int delora_project_points_fwd(const float* points, const int32_t* n_points, int B, int C, int n_stride, int H, int W,
                              double hfov0, double hfov1, double vfov0, double vfov1, int div_mode, uint64_t* keys,
                              float* image, int32_t* index_map, delora_f4* pts_grid, delora_f4* nrm_grid, void* stream);

/* ---------------------------------------------------------------------------------------
 * Image -> lists (row-major order of the valid pixels), the layout the reference stores and
 * trains on (src/preprocessing/normal_computation.py:30-41, :84-87;
 * src/preprocessing/preprocesser.py:64-68), plus the cell index used by the NN search.
 *
 * pts4       [B, H*W] out: (x, y, z, bits(pixel id))    for the P_b valid pixels, in order
 * nrm4       [B, H*W] out: (nx, ny, nz, has_normal ? 1 : 0)
 * cell_start [B, H*W + 1] int32 out: exclusive prefix of the valid flags (CSR over pixels)
 * counts     [B] int32 out: P_b
 * scratch    int32 [B * delora_scan_blocks(H*W)]
 */
int delora_scan_blocks(int n_cells);
int delora_lists_from_images(const float* image, const float* normals, int B, int C_img, int H, int W,
                             delora_f4* pts4, delora_f4* nrm4, int32_t* cell_start, int32_t* counts,
                             int32_t* scratch, void* stream);

/* Bin arbitrary point lists (the reference's [1,3,N] tensors) into the spherical cell grid:
 * counting sort by cell.  Needed by losses.icp_losses.ICPLosses.forward for lists that did
 * not come from delora_lists_from_images (src/losses/icp_losses.py:34 builds a cKDTree here).
 * Points outside the field of view go to the border cells (the search stays exact): rows clamp, and an azimuth in
 * the horizontal gap goes to the border column (0 or W-1) it is nearer to around the circle.
 *
 * pts, nrm   [B, 3, n_stride] fp32 channels-first;  n [B] int32
 * pts4/nrm4  [B, n_stride] out, sorted by cell; pts4.w = bits(original list index)
 * cell_start [B, H*W+1] int32 out
 * cursor     [B, H*W] int32 scratch (any contents), scratch int32 [B*delora_scan_blocks(H*W)]
 */
int delora_grid_build(const float* pts, const float* nrm, const int32_t* n, int B, int n_stride,
                      int H, int W, double hfov0, double hfov1, double vfov0, double vfov1,
                      delora_f4* pts4, delora_f4* nrm4, int32_t* cell_start, int32_t* cursor,
                      int32_t* scratch, void* stream);

/* Dense grids for the training step: the scan's points and its per-point (precomputed) normals,
 * gathered through the projection's pixel -> point index map (src/deploy/deployer.py:258-261).
 * points [B,C,n_stride], normal_lists [B,3,n_stride], index_map [B,H,W] ->
 * pts_grid/nrm_grid [B,H*W] float4 as delora_icp_dense_fwd_bwd expects them. */
int delora_grids_from_projection(const float* points, const float* normal_lists, const int32_t* index_map,
                                 int B, int C, int n_stride, int H, int W,
                                 delora_f4* pts_grid, delora_f4* nrm_grid, void* stream);

/* The reference's two-resolution training data in one call: the dense grids of S scans projected at H x Wp, as
 * delora_normals_fwd / delora_project_normals_fwd write them, re-projected at H x W.  This is the preprocessing stage
 * (src/preprocessing/preprocesser.py: projection and normals at horizontal_cells_preprocessing, the valid pixels stored
 * in row-major order) followed by the training stage's projection of those stored points at the model width
 * (src/deploy/deployer.py:252-261).  The result is bit-identical to
 *   delora_lists_from_images -> channels-first lists -> delora_project_fwd at H x W with C = 3 ->
 *   delora_grids_from_projection,
 * without building the lists: a valid cell's pixel id grows with its list index, so equal ranges in one model pixel
 * go to the same point ("lowest point index wins").
 * pts_grid_pre, nrm_grid_pre  [S, H*Wp] float4: valid cells (x, y, z, bits(pixel id)), empty (+inf, +inf, +inf, -1)
 * keys       [S, H*W] uint64 scratch, all-ones on entry and on exit (as for delora_project_fwd)
 * image      [S, 4, H, W] fp32 out: x, y, z of the kept point and its range; empty pixels are 0
 * index_map  [S, H, W] int32 out or NULL: the H x Wp cell of the kept point, -1 if empty
 * pts_grid, nrm_grid  [S, H*W] float4 out, as delora_grids_from_projection writes them: w = bits(model pixel id),
 *            has-normal = normal non-zero
 * hfov/vfov, div_mode as for delora_project_fwd. */
int delora_project_grids_fwd(const delora_f4* pts_grid_pre, const delora_f4* nrm_grid_pre, int S, int H, int Wp, int W,
                             double hfov0, double hfov1, double vfov0, double vfov1, int div_mode, uint64_t* keys,
                             float* image, int32_t* index_map, delora_f4* pts_grid, delora_f4* nrm_grid, void* stream);

/* Pack channels-first lists to float4 (no sorting): pts4.w = bits(list index), nrm4.w = has_normal. */
int delora_pack_lists(const float* pts, const float* nrm, const int32_t* n, int B, int n_stride,
                      delora_f4* pts4, delora_f4* nrm4, void* stream);

/* ---------------------------------------------------------------------------------------
 * Fused SE(3) transform + exact nearest neighbour + ICP losses, forward and backward.
 * Replaces, per scan pair:
 *   deploy.deployer.Deployer.{transform,rotate}_point_cloud_transformation_matrix  (src/deploy/deployer.py:181-189)
 *   losses.icp_losses.ICPLosses.forward          (src/losses/icp_losses.py:28-158; cKDTree :34, query :24-26)
 *   KDPointToPlaneLoss / KDPlaneToPlaneLoss / KDPointToPointLoss   (:196-206, :224-240, :168-179)
 *   and autograd's backward of those down to the 3x4 transform (SURVEY.md §3.4).
 *
 * src_pts4/src_nrm4 [B, src_stride]: source points / normals BEFORE the transform (nrm4.w ignored;
 *                   has-normal is decided on the rotated normal as the reference does, :48-50)
 * n_src             [B] int32
 * T                 [B, 12] fp32 row-major 3x4 (R | t); NULL = identity (inputs already transformed)
 * tgt_pts4/tgt_nrm4 [B, tgt_stride] sorted by cell (from delora_lists_from_images / delora_grid_build)
 * cell_start        [B, H*W+1]
 * lambda_po2pl      weight of the po2pl term in the gradient (deployer.py:310)
 * flags             DELORA_LOSS_* bits
 * losses            [B, DELORA_LOSS_ROW] out (unweighted means, as ICPLosses returns them)
 * grad_T            [B, 12] out: d(po2po + lambda*po2pl + pl2pl)/d(R|t), row-major 3x4
 * nn_index          [B, src_stride] int32 out or NULL: tag (tgt_pts4.w bits) of the NN of every source point
 * point_dir         [B, src_stride] float4 out or NULL: unscaled d(loss)/d(source point): r*n_t with w = 1 for a
 *                   kept (normal, normal) pair; (s - t) with w = 2 for a po2po pair; w = 0 otherwise
 * normal_dir        [B, src_stride] float4 out or NULL: unscaled d(pl2pl)/d(source normal)
 *                   (delora_icp_point_grads turns the two into the reference-shaped gradients)
 * scratch           fp32 [delora_icp_scratch_floats(B, src_stride)]: per-warp partial rows and their column sums, the
 *                   dense path's work list (an int4 item per warp, a float4 entry and an int32 result per source point,
 *                   an int32 count per warp) and range extents (float2 per 4 x 16-cell block and per pixel row), and
 *                   int32 counters.  Zero it ONCE after allocation; every call leaves the counters at zero again.  The
 *                   place and size of every section follow from (B, src_stride) alone: a buffer that is reused with a
 *                   different batch size or image size must be zeroed again first.
 * The NN is the exact float64 Euclidean nearest neighbour (lowest tag on exact ties).
 */
int     delora_icp_partial_rows(int src_stride);
int64_t delora_icp_scratch_floats(int B, int src_stride);
int delora_icp_fwd_bwd(const delora_f4* src_pts4, const delora_f4* src_nrm4, const int32_t* n_src,
                       int src_stride, const float* T,
                       const delora_f4* tgt_pts4, const delora_f4* tgt_nrm4, const int32_t* cell_start,
                       int tgt_stride, int B, int H, int W,
                       double hfov0, double hfov1, double vfov0, double vfov1,
                       float lambda_po2pl, uint32_t flags,
                       float* losses, float* grad_T, int32_t* nn_index,
                       delora_f4* point_dir, delora_f4* normal_dir,
                       float* scratch, void* stream);

/* The same operator on dense range-image grids (the layout delora_normals_fwd writes): source =
 * the valid pixels of `src_grid`, target = `tgt_grid`, at most one point per cell, so neither
 * list compaction nor a CSR index is needed.  This is the training-step fast path
 * (src/deploy/deployer.py:252-261 keeps exactly one point per pixel of both scans).
 * src_grid/src_ngrid, tgt_grid/tgt_ngrid: [B, H*W] float4;  T: [B, 12];
 * scratch: fp32 [delora_icp_scratch_floats(B, H*W)], zeroed once (see above).  Its range-pyramid section holds
 * H*W/16 + 4096 blocks per pair; a grid that needs more, ceil(H/4) * ceil(W/16) (very tall and narrow grids such as
 * W = 1 with H > 21844), is refused before any launch.
 * Launches target_extents_kernel (range extents of the target grids), icp_dense_kernel (window search, at most 32
 * growing steps per warp; the environment variable DELORA_ICP_MAX_STRIPS overrides the limit for profiling),
 * icp_dense_pending_kernel (range-pruned block search of the lanes still open) and icp_finalize_kernel; results do
 * not depend on the limit. */
int delora_icp_dense_fwd_bwd(const delora_f4* src_grid, const delora_f4* src_ngrid, const float* T,
                             const delora_f4* tgt_grid, const delora_f4* tgt_ngrid, int B, int H, int W,
                             double hfov0, double hfov1, double vfov0, double vfov1,
                             float lambda_po2pl, uint32_t flags, float* losses, float* grad_T,
                             float* scratch, void* stream);

/* How well each pair constrains its transform: the Gauss-Newton information of the ICP objective at T, beside the
 * losses.  LiDAR odometry fails in degenerate scenes (a corridor or tunnel, a flat field, a single wall) where the
 * residual is low and yet some direction of the pose is unobservable; H says which.  It needs no ground truth, uses
 * the exact correspondences of the losses and leaves T unchanged.
 *
 * Per pair: source point p and normal m (before the transform), T = (R | t), s = R p + t; q, n_t: the matched target
 * point and normal (the exact NN, with the masks of the losses).  T is perturbed on the right, in the source frame:
 * T(xi) = T Exp(xi), xi = (rho, phi) = (x, y, z, rot x, rot y, rot z), ROS's covariance order; to first order
 * s(xi) = s + R rho - R [p]x phi.  With u = R^T n_t and R_k the rows of R, the Jacobians per kept pair are
 *   po2pl (a normal on both sides, DELORA_LOSS_PO2PL)   r = n_t.(s - q)          J = [u, p x u]            (1 x 6)
 *   pl2pl squared (both sides, DELORA_LOSS_PL2PL)       e = R m - n_t            J = [0, -R [m]x]          (3 x 6)
 *   pl2pl linear (with DELORA_NORMAL_LINEAR)            o = 1 - n_t.(R m)        J = [0, u x m]            (1 x 6)
 *   po2po (a normal on neither side, DELORA_LOSS_PO2PO) d = s - q                J = [R, -R [p]x]          (3 x 6)
 * and, over the enabled terms only,
 *   H = 2 (lambda_po2pl / M  sum_po2pl J^T J  +  1 / M  sum_pl2pl J^T J  +  1 / (3 M')  sum_po2po J^T J),
 * the Gauss-Newton approximation of the Hessian in xi of po2po + lambda_po2pl po2pl + pl2pl with the losses' own means
 * (po2pl and pl2pl over the M pairs with a normal on both sides, po2po over the 3 M' coordinates of the M' pairs
 * with a normal on neither); a term whose count is 0 contributes nothing.  Its eigenvalues say how well the pair
 * constrains the pose, its eigenvectors in which directions: a near-zero eigenvalue is a direction the frame does not
 * determine.  No covariance is returned, because any covariance needs a noise model and that is the host's choice;
 * sigma^2 H^-1 (sigma^2 the variance of one residual, over the directions whose eigenvalue is not near zero) is one way
 * to build one, e.g. for the 6 x 6 covariance of a ROS nav_msgs/Odometry.
 *
 * info [B, DELORA_INFO_ROW] out (layout above): H from fp32 per-pair J^T J and fp32 sums over each warp of 32 source
 * pixels, then float64 sums over the warps in a fixed order, the weights in float64, stored as fp32; the eigenvalues
 * and eigenvectors by a float64 cyclic Jacobi solve of that float64 H; each eigenvector's largest-magnitude component
 * (the first of equals) is positive.  Bit-identical from run to run; a pair's row does not depend on B or on the other
 * pairs.  losses and grad_T: bit-identical to delora_icp_dense_fwd_bwd on the same inputs (the same search kernels,
 * instantiated to also write the NN ids; the scratch layout is the same).
 * info_scratch: fp32 [delora_icp_information_scratch_floats(B, H, W)], no initialisation needed; after the call its
 * first B * H * W int32 are the id of every source pixel's kept nearest neighbour (-1 where the losses keep no pair).
 * Refused: what delora_icp_dense_fwd_bwd refuses, null info / info_scratch, DELORA_ICP_STATS in flags.
 * Cost beside delora_icp_dense_fwd_bwd: two launches, icp_info_rows_kernel and icp_info_finalize_kernel (measured
 * below, with delora_odometry_streams_push_info). */
int64_t delora_icp_information_scratch_floats(int B, int H, int W);     /* host only, -1 for a bad shape */
int delora_icp_dense_information(const delora_f4* src_grid, const delora_f4* src_ngrid, const float* T,
                                 const delora_f4* tgt_grid, const delora_f4* tgt_ngrid, int B, int H, int W,
                                 double hfov0, double hfov1, double vfov0, double vfov1,
                                 float lambda_po2pl, uint32_t flags, float* losses, float* grad_T,
                                 float* scratch, float* info, float* info_scratch, void* stream);
/* The information in metres for pairs whose clouds were divided by a factor (a model trained with
 * normalization_scaling runs its ICP on the pair divided by the pair's factor f).  The arguments of
 * delora_icp_dense_information plus factor [B] fp32 (device, every factor > 0; not checked on the host), the factor
 * each pair's grids were divided by.  The operator's H is then taken in xi = (rho / f, phi) with rho in metres; since
 * T(xi) = T Exp(xi) and a normalised translation of rho / f is rho metres, the information in the metres and radians
 * of the T the model serves is H_m = D H D, D = diag(1/f, 1/f, 1/f, 1, 1, 1).  D is applied in float64 to the float64
 * H before it is stored and solved, so the eigenvalues and eigenvectors are those of H_m.  The losses row stays in the
 * model's units (the objective has no single rescale: pl2pl is unit-free), and losses, grad_T and the NN ids are
 * delora_icp_dense_information's bits.  With every factor = 1 the output is delora_icp_dense_information's, bit for bit
 * (each float64 product is by 1.0).  Refused: what delora_icp_dense_information refuses, a null factor. */
int delora_icp_dense_information_scaled(const delora_f4* src_grid, const delora_f4* src_ngrid, const float* T,
                                        const delora_f4* tgt_grid, const delora_f4* tgt_ngrid, int B, int H, int W,
                                        double hfov0, double hfov1, double vfov0, double vfov1,
                                        float lambda_po2pl, uint32_t flags, float* losses, float* grad_T,
                                        float* scratch, float* info, float* info_scratch, const float* factor,
                                        void* stream);

/* Diagnostic for delora_icp_dense_fwd_bwd calls made with DELORA_ICP_STATS in `flags`: copies the 32 device
 * counters to the HOST array out32 (may be NULL) and optionally zeroes them.  [0] warps, [1] window-growing steps,
 * [2] cells evaluated per lane (both summed per warp), [3] warps that entered the range-pruned block search,
 * [4] lanes searched there, [5] blocks bounded, [6] blocks scanned, [7] max blocks scanned for one lane,
 * [8] float64 tie re-rankings, [9] max blocks bounded for one lane, [10] lanes with > 256 blocks, [11] lanes that
 * reached the block search without any candidate, [16..23] warps by number of steps {0, 1-2, 3-5, 6-10, 11-20, 21-40, 41-63, limit},
 * [24..31] cells per lane summed over the warps of the same bucket.  Synchronises the device. */
int delora_icp_stats(uint32_t* out32, int reset);

/* Backward of ICPLosses.forward w.r.t. its two differentiable inputs, for callers that hand in
 * already-transformed clouds and let autograd continue (src/deploy/deployer.py:294-307 -> :341):
 * upstream [B,3] = d(total)/d(loss_po2po, loss_po2pl, loss_pl2pl);  losses = the row written by
 * delora_icp_fwd_bwd;  grad_pts, grad_nrm: [B, 3, src_stride] channels-first out. */
int delora_icp_point_grads(const delora_f4* point_dir, const delora_f4* normal_dir, const int32_t* n_src,
                           int src_stride, int B, const float* losses, const float* upstream,
                           float* grad_pts, float* grad_nrm, void* stream);

/* ---------------------------------------------------------------------------------------
 * Encoder convolution, forward, on the Hopper tensor cores (wgmma; bf16 in, fp32 accumulate, bf16 out).
 * Replaces the cuDNN call behind torch.nn.Conv2d in the reference's encoder
 *   (src/models/resnet_modified.py:40 stem, :126-134 conv3x3 / conv1x1; used at :95-120, :159-177)
 *   including the circular width padding (:97, :162, :167), the zero height padding, the
 *   activation and the residual add of BasicBlock.forward (:174-175).
 * x        [B, Hin+2, Win+2, Cin]  bf16 NHWC with materialised padding (rows 0/Hin+1 zero, column 0 =
 *          column Win, column Win+1 = column 1)
 * w        [Cout, ksize*ksize, Cin] bf16 (tap-major K: torch weight.permute(0,2,3,1))
 * residual [B, Hout+2, Wout+2, Cout] bf16 or NULL, added before the activation
 * y        [B, Hout+2, Wout+2, Cout] bf16 out (interior + circular halo columns are written; the
 *          zero halo rows must have been zeroed once by the caller)
 * saved    [B, Hout+2, Wout+2, Cout] bf16 or NULL: forward activation output for the backward modes
 * ksize 3 (pad 1 in H, wrap in W) or 1 (no padding); stride_h/w in {1,2};
 * act: 0 none, 1 relu, 2 tanh (forward);  3 / 4: multiply (acc + residual) by tanh'(saved) = 1 - saved^2 /
 *      relu'(saved) -- the data-gradient pass: dgrad of a stride-1 conv is this same kernel run on the output
 *      gradient with the flipped, transposed filter (strided convs: on the zero-upsampled gradient).
 * Cin, Cout multiples of 64 (the 8-channel stem input is channel-padded by delora_images_to_nhwc_bf16). */
int delora_conv2d_fprop_bf16(const void* x, const void* w, const void* residual, const void* saved, void* y, int B,
                             int Hin, int Win, int Cin, int Cout, int ksize, int stride_h, int stride_w, int act,
                             void* stream);
/* Data gradient of a 3x3 convolution of stride (stride_h, stride_w) in {1,2}^2 -- autograd's backward of the same
 * nn.Conv2d layers (src/models/resnet_modified.py:126-134) w.r.t. their input -- by PHASE DECOMPOSITION: every
 * output phase (h % stride_h, w % stride_w) is a small convolution of the (un-upsampled) output gradient with the
 * subset of flipped taps that hits non-zero positions; no zero-upsampled tensor is materialised.
 * dz [B,Hout+2,Wout+2,Cout] (Hout = (Hin-1)/stride_h + 1 ...), w_flip [Cin, 9, Cout] (delora_conv_weight_prep_bf16),
 * residual / saved / dx [B,Hin+2,Win+2,Cin]; act as in delora_conv2d_fprop_bf16 (3 / 4 = multiply by act'(saved)).
 * residual_strided = 1: `residual` is [B,Hout+2,Wout+2,Cin] instead and is added at the input pixels
 * (stride_h * h, stride_w * w) only -- the data gradient of the block's 1x1 strided downsample (:134), which never
 * reaches the other pixels (replaces a zero-upsampled copy of it).
 * Takes the layers delora_conv2d_dgrad_eligible accepts; for the others use delora_zero_upsample_nhwc_bf16 +
 * delora_conv2d_fprop_bf16. */
int delora_conv2d_dgrad_bf16(const void* dz, const void* w_flip, const void* residual, const void* saved, void* dx,
                             int B, int Hin, int Win, int Cin, int Cout, int stride_h, int stride_w, int act,
                             int residual_strided, void* stream);
/* 1 if delora_conv2d_dgrad_bf16 takes the data gradient of this 3x3 layer (Cin, Cout of the FORWARD convolution, Win its
 * input width), 0 if not: strides in {1,2}, Cout % 64 == 0, Cin % 128 == 0 or Cin = 64 with >= 128 columns per phase
 * (ceil(Win / stride_w)), and an even Win for stride_w = 2 (an odd circular width mixes the phases at the seam).
 * Host only: needs no device and launches nothing. */
int delora_conv2d_dgrad_eligible(int Cin, int Cout, int Win, int stride_h, int stride_w);
/* Weight gradient of the same convolution on wgmma (split-K over pixels, deterministic reduction):
 * x [B,Hin+2,Win+2,Cin] padded NHWC bf16 (the layer input), dz [B,Hout+2,Wout+2,Cout] padded NHWC bf16
 * (gradient w.r.t. the pre-activation output) -> dw [Cout, Cin_true, k, k] fp32 (torch layout; Cin_true <= Cin
 * for the channel-padded stem).  scratch: fp32 [delora_conv2d_wgrad_scratch_floats(...)].
 * Any Hin, Win >= 1: Hout = (Hin-1)/stride_h + 1, Wout = (Win-1)/stride_w + 1; ragged tiles are zero-filled. */
int64_t delora_conv2d_wgrad_scratch_floats(int B, int Hout, int Wout, int Cin, int Cout, int ksize);
int delora_conv2d_wgrad_bf16(const void* x, const void* dz, float* dw, float* scratch, int B, int Hin, int Win,
                             int Cin, int Cin_true, int Cout, int ksize, int stride_h, int stride_w, void* stream);
/* y[h*sh, w*sw] = x[h, w], zero elsewhere (padded NHWC bf16 in and out): input of the dgrad of strided convs.
 * y is [B,Hout+2,Wout+2,C] with (Hout, Wout) the INPUT size of the strided convolution
 * ((Hout-1)/sh+1 == H, (Wout-1)/sw+1 == W: 45 -> 23 -> 45 for the odd widths of 64x720 images). */
int delora_zero_upsample_nhwc_bf16(const void* x, int B, int H, int W, int C, int sh, int sw, int Hout, int Wout,
                                   void* y, void* stream);

/* torch filter w [Cout,Cin,k,k] fp32 -> w_fwd [Cout,k*k,Cin_pad] bf16 (the `w` operand of delora_conv2d_fprop_bf16;
 * channels >= Cin zero) and, unless NULL, w_flip [Cin,k*k,Cout] bf16 (spatially flipped, in/out swapped: the filter
 * of the data-gradient pass).  One launch per layer and step replaces autograd's permute / flip / cast chain. */
int delora_conv_weight_prep_bf16(const float* w, int Cout, int Cin, int ksize, int Cin_pad, void* w_fwd, void* w_flip,
                                 void* stream);

/* All encoder filters in one launch (replaces 20 delora_conv_weight_prep_bf16 calls per training step).
 * table: device array of n_layers x 8 int64 = {fp32 weight ptr, w_fwd ptr, w_flip ptr or 0, Cout, Cin, k, Cin_pad, kind};
 * kind 0 = the layouts of delora_conv_weight_prep_bf16, kind 1 = the stem layout of delora_stem_weight_prep_bf16. */
int delora_conv_weight_prep_multi(const void* table, int n_layers, void* stream);

/* ---- Encoder stem (src/models/resnet_modified.py:40 conv1: 3x3, stride (1,2), 8 -> 64 channels, + activation :99) on a
 * 16-channel input layout; replaces the channel-padded (8 -> 64) route through delora_conv2d_fprop/wgrad_bf16.
 * x16    [B, H+2, W+2, 16] bf16: channels 0..7 = cat(image_1, image_2) (src/models/model.py:98), 8..15 zero, padding
 *        materialised as everywhere (delora_images_to_nhwc16_bf16 writes it)
 * w_stem [3, 64, 64] bf16: [filter row][output channel][k = q * 16 + c] (delora_stem_weight_prep_bf16)
 * y      [B, H+2, W/2+2, 64] bf16 out (fp16 bit patterns when out_f16 = 1);  dz same shape;  dw [64, Cin_true, 3, 3]
 *        fp32.  W must be even. */
int delora_images_to_nhwc16_bf16(const float* image_1, const float* image_2, int B, int H, int W, void* x16, void* stream);
int delora_stem_weight_prep_bf16(const float* w, int Cin, void* w_stem, void* stream);
int delora_stem_fprop_bf16(const void* x16, const void* w_stem, void* y, int B, int H, int W, int act, int out_f16,
                           void* stream);
int64_t delora_stem_wgrad_scratch_floats(int B, int H, int W);
int delora_stem_wgrad_bf16(const void* x16, const void* dz, float* dw, float* scratch, int B, int H, int W, int Cin_true,
                           void* stream);

/* cat(image_1, image_2) ([B,4,H,W] fp32 each, src/models/model.py:98) -> [B,H+2,W+2,Cpad] bf16 padded NHWC */
int delora_images_to_nhwc_bf16(const float* image_1, const float* image_2, int B, int H, int W, int Cpad,
                               void* x, void* stream);
/* MaxPool2d(3, stride (1,2), padding (1,0)) on the W-wrapped input (src/models/resnet_modified.py:46,:100-101) */
int delora_maxpool_w_nhwc_bf16(const void* x, int B, int H, int W, int C, void* y, void* stream);
/* training variants of the pools: forward with argmax (idx: uint8 [B,H,W/2,C]); backward of the max-pool
 * fused with act'(a) of the stem activation a; backward of the global average pool fused with act'(a) of
 * the last block (g: [B,C] fp32).  act: 0 none, 1 relu, 2 tanh.  All tensors padded NHWC bf16.
 * Pre-activation form (what the training path uses for the stem): the forward pool takes the stem's PRE-activation
 * z and applies `act` to the maximum (max act(z) = act(max z) for the monotonic tanh / relu); the backward then gets
 * `a` = z and act = 5 (relu'(z)) or 6 (tanh'(z) = 4 e^{-2|z|} / (1 + e^{-2|z|})^2): 1 - a^2 evaluated on a bf16-rounded,
 * saturated tanh output has no correct digit, the metre-valued inputs saturate the stem heavily.
 * x_f16 / a_f16 = 1: that tensor holds fp16 instead of bf16 values (delora_stem_fprop_bf16 with out_f16 = 1): three more
 * mantissa bits keep the pool's argmax on the fp32 winner when two window entries nearly tie. */
int delora_maxpool_w_idx_nhwc_bf16(const void* x, int B, int H, int W, int C, void* y, void* idx, int act, int x_f16,
                                   void* stream);
int delora_maxpool_w_bwd_nhwc_bf16(const void* dy, const void* idx, const void* a, int B, int H, int W, int C, int act,
                                   void* dz, int a_f16, void* stream);
int delora_avgpool_bwd_nhwc_bf16(const float* g, const void* a, int B, int H, int W, int C, int act, void* dz,
                                 void* stream);
/* AdaptiveAvgPool2d((1,1)) (src/models/resnet_modified.py:111): padded NHWC bf16 [B,H+2,W+2,C] -> y [B,C] fp32
 * (fp32 sums in a fixed order; C a multiple of 64) */
int delora_avgpool_nhwc_bf16(const void* x, int B, int H, int W, int C, float* y, void* stream);
/* padded NHWC bf16 -> NCHW fp32 (interior), the reference's feature-map layout */
int delora_nhwc_to_nchw_f32(const void* x, int B, int H, int W, int C, float* y, void* stream);

/* quaternion (x, y, z, w) + translation -> 4x4, and its backward.
 * Replaces models.model_parts.GeometryHandler.get_transformation_matrix_quaternion
 *   (src/models/model_parts.py:37-44 -> kornia 0.3.0 quaternion_to_rotation_matrix).
 * quaternion [B,4], translation [B,3] -> T [B,16].  grad variant: gT [B,16] -> gq [B,4], gt [B,3]. */
int delora_quat_to_T(const float* quaternion, const float* translation, int B, float* T, void* stream);
int delora_quat_to_T_bwd(const float* quaternion, const float* grad_T, int B,
                         float* grad_quaternion, float* grad_translation, void* stream);

/* ---------------------------------------------------------------------------------------
 * Encoder trunk: ResNetModified (src/models/resnet_modified.py:95-120) from the two range images to the average-pooled
 * features, the kernels above in one fixed sequence -- the sequence the odometry entry points below run as well.
 * layers[4]: BasicBlocks per stage (1 .. 64 each).  H >= 1, W >= 2 with (W - 1) / 2 + 1 even (the max-pool halves it).
 * act: 1 relu, 2 tanh.  The stem takes the 16-channel layout when W is even, the channel-padded one otherwise, so the
 * weight section depends on W's parity.
 *
 * Weight section: delora_trunk_weight_bytes(layers, W) device bytes, written by delora_trunk_prep_weights from the
 * fp32 filters: filters is a HOST array of device pointers, one per convolution in state_dict order (resnet.conv1,
 * then per block conv1, conv2 and the downsample's conv if it has one).  The bf16 forward and flipped filters; prep
 * copies its table from host memory and launches one kernel.
 * Activation workspace: delora_trunk_activation_bytes(layers, B, H, W, saving) device bytes for batches of exactly B
 * pairs, zeroed once after allocation (the zero halo rows).  saving = 0: rotating inference buffers; saving = 1: every
 * activation the backward reads, its gradient buffers and the split-K scratch.  A size query returns -1 on bad
 * arguments.
 * forward: img1, img2 [B, 4, H, W] fp32 -> pooled [B, 512] fp32.  stage_out NULL or void*[4]: receives the addresses
 * (in acts) of x1..x4, [B, h+2, w+2, C] padded NHWC bf16 with C = 64, 128, 256, 512.
 * backward (after a saving forward of the same arguments, weights unchanged): call it for stage = 3, 2, 1, 0 in that
 * order.  Stage 3 starts from g_pooled [B, 512] fp32 (read by stage 3 only); stage 0 ends with the max-pool and the
 * stem.  Each call writes the weight gradient of every convolution of its stage (stage 0: and the stem) to
 * conv_dw[c] (fp32 [Cout, Cin, k, k], c in the order of `filters`; a HOST array of device pointers), so that the
 * gradients of a stage can be used once its call is enqueued.
 * _dropout variants: the input and stage-3 dropouts of a DELORA_TRAIN_DROPOUT training step (see _train_step), with
 * their masks at the step and seed of dropout_ctr, a device int64[3] in the training workspace's counter-slot layout:
 * [0] the step, [2] the seed ([1] is not read).  Pass the same counter to the forward and to the four backward calls;
 * the backward overwrites x3d, so each backward with a counter follows its own forward.
 * x1 .. x4 (stage_out) are the stage outputs before the stage-3 dropout, as the step keeps them; `pooled` and the weight
 * gradients are the step's.  dropout_ctr NULL: exactly delora_trunk_forward / delora_trunk_backward.  A counter needs
 * saving = 1 (x3d lives in a backward buffer); refused before any launch otherwise.  The fc dropout is not the trunk's.
 */
int64_t delora_trunk_weight_bytes(const int* layers, int W);
int delora_trunk_prep_weights(const int* layers, int W, const float* const* filters, void* weights, void* stream);
int64_t delora_trunk_activation_bytes(const int* layers, int B, int H, int W, int saving);
int delora_trunk_forward(const int* layers, int B, int H, int W, int act, int saving, const float* img1,
                         const float* img2, const void* weights, void* acts, float* pooled, void** stage_out,
                         void* stream);
int delora_trunk_backward(const int* layers, int B, int H, int W, int act, const void* weights, void* acts,
                          const float* g_pooled, float* const* conv_dw, int stage, void* stream);
int delora_trunk_forward_dropout(const int* layers, int B, int H, int W, int act, int saving, const float* img1,
                                 const float* img2, const void* weights, void* acts, float* pooled, void** stage_out,
                                 const int64_t* dropout_ctr, void* stream);
int delora_trunk_backward_dropout(const int* layers, int B, int H, int W, int act, const void* weights, void* acts,
                                  const float* g_pooled, float* const* conv_dw, int stage, const int64_t* dropout_ctr,
                                  void* stream);

/* ---------------------------------------------------------------------------------------
 * Odometry inference: raw scans -> relative transforms, the whole model behind one call.
 * Replaces, for inference, deploy.tester.Tester.test_dataset's per-frame path
 *   (src/deploy/tester.py:38-107 -> src/deploy/deployer.py:237-281): the projection of both scans,
 *   models.model.OdometryModel.forward (src/models/model.py:96-116: encoder trunk, resnet.fc, the two MLP
 *   heads or the single MLP, quaternion / norm of the whole [B,4] block) and GeometryHandler's quaternion -> T.
 *
 * The trunk is the one of delora_trunk_forward (the projected images are bit-identical to delora_project_fwd's, the
 * pooled features to the Python trunk's, which runs delora_trunk_forward); the fully connected tail is one
 * fp32 launch per layer (odometry_linear_kernel) plus one launch for the last layer, the norm and quaternion -> T
 * (odometry_out_kernel), with a fixed summation order.  Not representable: pre_feature_extraction,
 * factor_fewer_resnet_channels != 1; dropout is the identity at inference.
 *
 * Models trained with normalization_scaling run through delora_odometry_pairs_normalized (below), not _pairs / _push.
 *
 * Workspace: one caller-owned device buffer of delora_odometry_workspace_bytes(d) bytes holds every activation,
 * the bf16 filters, the fp32 tail weights and the stream's cached range image.  Its layout is a function of the
 * descriptor only.  Use: _init once, _load_weights, then any number of _pairs / _push calls.  One workspace serves
 * one stream of calls at a time.
 */
typedef struct {
    int H, W;                            /* range image of the model (vertical_cells, horizontal_cells);
                                            (W - 1) / 2 + 1 must be even (the stem's max-pool halves it) */
    double hfov0, hfov1, vfov0, vfov1;   /* radians, as the bin scripts pass them */
    int n_stride;                        /* max points per scan: the point stride of `points` */
    int max_batch;                       /* max pairs per delora_odometry_pairs call (1 .. 1024) */
    int act;                             /* 1 relu, 2 tanh */
    int layers[4];                       /* BasicBlocks per stage, e.g. {2,2,2,2} (1 .. 64 each) */
    int resnet_outputs;                  /* fc width, 1000 in the shipped config */
    int single_mlp;                      /* use_single_mlp_at_output (0 / 1) */
    int w_pre;                           /* horizontal_cells_preprocessing, the width the normals are estimated at.
                                            Read and validated by the delora_odometry_train_* entry points (0: at W;
                                            else >= 2 with H * w_pre < 2^27) and by delora_odometry_streams_pre_* and
                                            _streams_push_pre (>= 2 with H * w_pre < 2^27; 0 is refused) alone.
                                            Training callers must zero it (or copy the descriptor from a .dlw header);
                                            other inference and streams callers may leave it uninitialised. */
} delora_odometry_desc;

/* Weight file (.dlw, written by delora_b200/deploy/export.py), little-endian, readable with fread alone:
 *   bytes   0..127  delora_odometry_file_header below (explicit offsets: magic 0, abi_version 8, header_bytes 12,
 *                   desc 16: H 16, W 20, hfov0 24, hfov1 32, vfov0 40, vfov1 48, n_stride 56, max_batch 60, act 64,
 *                   layers 68..83, resnet_outputs 84, single_mlp 88, w_pre 92; blob_floats 96; model_flags 104;
 *                   objective_flags 108; lambda_po2pl 112; zero 116..127; exporters before w_pre wrote zeros at 92,
 *                   i.e. w_pre = 0, exporters before model_flags wrote zeros at 104, i.e. no flag, and exporters
 *                   before the objective wrote zeros at 108..115, i.e. the shipped objective)
 *   bytes 128..     float32[blob_floats]: the tensors of OdometryModel.state_dict() concatenated in state_dict order,
 *                   each tensor row-major (the blob delora_odometry_load_weights takes). */
#define DELORA_ODOMETRY_FILE_MAGIC "DELORAW"     /* 7 characters + NUL = the 8 magic bytes */
/* model_flags bits: how the model expects its input, beyond the descriptor */
#define DELORA_MODEL_NORMALIZATION_SCALING 1u    /* trained with normalization_scaling: run it through
                                                    delora_odometry_pairs_normalized */
#define DELORA_MODEL_DROPOUT 2u                  /* configured with use_dropout: train it with DELORA_TRAIN_DROPOUT;
                                                    inference and streams ignore the bit (dropout is the identity) */
typedef struct {
    char magic[8];
    int32_t abi_version;                 /* DELORA_B200_ABI_VERSION of the exporter */
    int32_t header_bytes;                /* 128 */
    delora_odometry_desc desc;
    int64_t blob_floats;                 /* == delora_odometry_weight_floats(&desc) */
    uint32_t model_flags;                /* DELORA_MODEL_* bits (byte 104) */
    uint32_t objective_flags;            /* byte 108: the ICP objective the model is configured with, the loss_flags
                                            bits DELORA_LOSS_PO2PO / _PO2PL / _PL2PL, DELORA_NORMAL_LINEAR and
                                            DELORA_LOSS_PO2PO_ALONE (at least one ICP loss bit); 0: written before
                                            the field, the shipped objective (see delora_odometry_file_objective) */
    float lambda_po2pl;                  /* byte 112: the objective's lambda_po2pl (ignored when objective_flags = 0) */
    uint8_t reserved[12];
} delora_odometry_file_header;

/* Host only (no GPU needed): the objective a .dlw / .dlt header records, as the loss_flags ICP bits and lambda_po2pl
 * of delora_odometry_train_params / delora_odometry_residual_params.  objective_flags = 0 gives the shipped objective,
 * DELORA_LOSS_PO2PL | DELORA_LOSS_PL2PL with lambda_po2pl 1.  Refused (non-zero, delora_last_error() naming the field):
 * a null pointer, objective_flags with a bit outside the five above or without an ICP loss bit, DELORA_LOSS_PO2PO_ALONE
 * without DELORA_LOSS_PO2PO or with _PO2PL, _PL2PL or DELORA_NORMAL_LINEAR, and a lambda_po2pl that is not finite. */
int delora_odometry_file_objective(const delora_odometry_file_header* h, uint32_t* loss_flags, float* lambda_po2pl);

/* Host only (no GPU needed): validate the descriptor (non-zero + delora_last_error() if it is invalid; the size
 * functions then return -1) and size the weight blob / the workspace. */
int64_t delora_odometry_weight_floats(const delora_odometry_desc* d);
int64_t delora_odometry_workspace_bytes(const delora_odometry_desc* d);
/* Zero the workspace (every activation buffer's zero halo rows) and set the projection key buffer to all ones.
 * Once after allocation; later calls never write those regions except as the kernels above do. */
int delora_odometry_init(const delora_odometry_desc* d, void* workspace, void* stream);
/* weights: DEVICE fp32[delora_odometry_weight_floats(d)], the .dlw blob.  Converts the convolution filters to the bf16
 * layouts (delora_conv_weight_prep_multi) and copies the fc / head tensors into the workspace; every weight region is
 * rewritten, so loading a second blob replaces the first completely.  `weights` must stay valid until the stream has
 * run the call.  The prep table is copied from host memory (the call may wait for the stream to reach it). */
int delora_odometry_load_weights(const delora_odometry_desc* d, const float* weights, void* workspace, void* stream);
/* B pairs (1 <= B <= max_batch): points [2B, 3, n_stride] fp32 (scan_1 of pair 0..B-1, then scan_2 of pair 0..B-1),
 * n_points [2B] int32 (device).  T [B, 16] out (row-major 4x4: scan_2 -> scan_1 frame); pooled [B, 512] fp32 out
 * (the average-pooled encoder features) or NULL.  The quaternion is divided by the norm of the whole [B, 4] block
 * (src/models/model.py:114), so a row's T can differ in the last bits with the batch it was computed in.
 * Device counts above n_stride are clamped to n_stride on the device (a host-side check would need a synchronise).
 * Only launches: no allocation, no synchronisation, no host decision on device data. */
int delora_odometry_pairs(const delora_odometry_desc* d, const float* points, const int32_t* n_points, int B,
                          void* workspace, float* T, float* pooled, void* stream);

/* Models trained with normalization_scaling (config/hyperparameters.yaml:23; the file's model_flags has
 * DELORA_MODEL_NORMALIZATION_SCALING).  Such a model saw each pair divided by a factor and predicts its translation in
 * those units: Deployer.normalize_input (src/deploy/deployer.py:222-235) and the rescale at :344-346 / :371-373.
 *
 * delora_normalization_factors: the factor of B pairs, the operator that replaces normalize_input's mean.
 *   points [2B, 3, n_stride] fp32 (scan_1 of pair 0..B-1, then scan_2 of pair 0..B-1), n_points [2B] int32 (device,
 *   clamped to [0, n_stride] on the device) -> factor [B] fp32 out (device).  Per scan, m = the mean of its points'
 *   ranges: each range is sqrt((x*x + y*y) + z*z) of the fp32 coordinates, correctly rounded (the projection's range
 *   channel), the ranges are summed in float64 in a fixed order that depends on neither B nor the launch, divided by
 *   the count and rounded to fp32.  factor = (m_1 + m_2) / 2 in fp32.  Bit-identical from run to run; within a few
 *   ulp of torch's mean, whose CUDA reduction order is not reproducible.  A scan without points is outside the
 *   contract: its mean is NaN (0 / 0), as torch.mean of an empty tensor in the reference.  The reference's ROS node
 *   (src/ros_utils/odometry_publisher.py:102-111) pools the ranges of both scans into one mean instead; that variant
 *   is not provided.  Refused before any launch, naming the argument: null points / n_points / factor, B outside
 *   [1, 65535], n_stride < 1.
 *
 * delora_odometry_pairs_normalized: delora_odometry_pairs with the factor applied, as the Tester runs such a model.
 *   Both scans of pair b are divided by factor[b] (x / f correctly rounded, before any other use), projected and run
 *   through the model; then T[:3, 3] of row b is multiplied by factor[b] in fp32.  The images and pooled features are
 *   bit-identical to delora_odometry_pairs on a copy of the points divided by the factor.  Same workspace and arguments
 *   as delora_odometry_pairs, plus factor [B] fp32, a required caller-owned device output that also carries the factor
 *   between the kernels.  Only launches, so one call can be captured into a CUDA graph.  Refused before any launch,
 *   naming the argument: an invalid descriptor, null points / n_points / workspace / T / factor, B outside
 *   [1, max_batch].
 *
 * Streaming a normalised model: the _push and _streams_push workspaces cache the previous frame's projected image,
 * which depends on the factor of the NEXT pair, so they cannot serve normalised models.  Stream one sensor through
 * delora_odometry_pairs_normalized with B = 1 on (previous scan, this scan), as the reference's ROS node does
 * (examples/odometry_stream.c does so for flagged files); serve several through delora_odometry_streams_push_normalized
 * (below), which keeps each stream's previous SCAN instead.  Train one with DELORA_TRAIN_NORMALIZATION_SCALING in
 * delora_odometry_train_params.loss_flags (see delora_odometry_train_step). */
int delora_normalization_factors(const float* points, const int32_t* n_points, int B, int n_stride, float* factor,
                                 void* stream);
int delora_odometry_pairs_normalized(const delora_odometry_desc* d, const float* points, const int32_t* n_points, int B,
                                     void* workspace, float* T, float* pooled, float* factor, void* stream);
/* Streaming, batch 1: project the frame points [1, 3, n_stride] (n_points [1], device), run the model on (cached
 * previous image, this image), write T [16], then cache this image.  T == NULL: only project and cache (the first
 * frame of a stream).  Bit-identical to delora_odometry_pairs with B = 1 on (previous scan, this scan).  With T
 * non-NULL the launch sequence is fixed, so one call can be captured into a CUDA graph and replayed per frame. */
int delora_odometry_push(const delora_odometry_desc* d, const float* points, const int32_t* n_points,
                         void* workspace, float* T, void* stream);

/* Several streams in one workspace: S = d->max_batch independent sensors (or vehicles) that share the descriptor, i.e.
 * the image geometry and the model.  One call per tick projects the S new frames and runs the model once at batch S.
 * Each quaternion is divided by the norm of its own row, so row s of T is bit-identical to what a delora_odometry_push
 * workspace returns when fed only stream s's active frames (after a reset: as if that stream had just started).
 * The workspace (its own layout, delora_odometry_streams_workspace_bytes) holds each stream's previous frame and whether
 * it has one; both live on the device.  _streams_push only enqueues work (no allocation, no synchronisation, no host
 * decision on device data) and its launch sequence depends on neither `active` nor the stream state, so one captured
 * call can be replayed every tick whatever the activity pattern.  Refused before any launch, with the field or pointer
 * named: an invalid descriptor, and null points / n_points / workspace / T / valid. */
int64_t delora_odometry_streams_workspace_bytes(const delora_odometry_desc* d);     /* host only, -1 if invalid */
/* Zero the workspace (no stream has a previous frame) and arm the projection keys.  Once after allocation. */
int delora_odometry_streams_init(const delora_odometry_desc* d, void* workspace, void* stream);
/* The .dlw blob of delora_odometry_load_weights (DEVICE fp32[weight_floats]), same conversion and same rules. */
int delora_odometry_streams_load_weights(const delora_odometry_desc* d, const float* weights, void* workspace,
                                         void* stream);
/* points [S, 3, n_stride], n_points [S] (device, clamped to [0, n_stride] on the device), active [S] int32 (device;
 * NULL = all active).  For every active stream: project its frame; if the stream has a previous frame, write T[s]
 * (row-major 4x4, this frame -> previous frame, as _push) and valid[s] = 1; then this frame becomes the stream's
 * previous frame.  Inactive streams: T row untouched, valid[s] = 0, cached frame untouched.  T [S, 16] fp32 and
 * valid [S] int32 are device outputs; valid[s] is written for every stream. */
int delora_odometry_streams_push(const delora_odometry_desc* d, const float* points, const int32_t* n_points,
                                 const int32_t* active, void* workspace, float* T, int32_t* valid, void* stream);
/* Forget the previous frame of every stream with mask[s] != 0 (device int32 [S]); the next push of such a stream only
 * caches its frame.  Refused: an invalid descriptor, null mask / workspace. */
int delora_odometry_streams_reset(const delora_odometry_desc* d, const int32_t* mask, void* workspace, void* stream);

/* A per-frame ICP residual beside every streamed transform: the model's own training objective (the point-to-plane /
 * plane-to-plane / point-to-point residual of this frame moved by T against the stream's previous frame, with the
 * matched-pair counts) as a quality signal that needs no ground truth.  Replaces, per streamed frame, the loss branch
 * of the reference's Tester (inference_only: False; src/deploy/tester.py:61-65 -> src/deploy/deployer.py:280-369)
 * without its visible_pixels and log images.  The call reports numbers only; what is a good frame is the host's policy.
 *
 * The residual workspace is the streams workspace with sections appended: no offset of the streams layout moves, so
 * delora_odometry_streams_load_weights and delora_odometry_streams_reset work on it unchanged (_residual_init replaces
 * _streams_init).  Appended, each 256-byte aligned, for S = max_batch streams of H x W cells: the point and normal grids
 * (float4 per cell) of the S new frames and of the S previous frames (64 bytes per cell and stream), the S x 12
 * transforms the ICP reads, its losses and dL/dT (computed, not returned) and its scratch for B = S
 * (delora_icp_scratch_floats(S, H * W)); the index map of the new frames is the one the streams layout already has.
 * Sizes from the host-only query (layers {2,2,2,2}, resnet_outputs 1000, two heads, n_stride 131072), streams ->
 * residual workspace: 64 x 2048: S = 1 86.0 -> 99.3 MiB, S = 4 271.8 -> 325.0 MiB, S = 16 1015.1 -> 1227.9 MiB;
 * 64 x 720: S = 1 46.2 -> 50.9 MiB, S = 4 112.8 -> 131.6 MiB, S = 16 379.1 -> 454.3 MiB.
 *
 * delora_odometry_streams_push_residual: T [S, 16] and valid [S] are what delora_odometry_streams_push writes for the
 * same history, byte for byte: the new frames go through delora_project_normals_fwd, whose image is bit-identical to
 * delora_project_fwd's, so the trunk input does not change.  The normals are estimated at the model's H x W on the raw
 * frame with rp's neighbourhood: a serving-time signal on the images the model sees, not the training recipe's w_pre
 * normals.  losses [S, DELORA_LOSS_ROW] (device, required): for every stream with valid[s] = 1 the row
 * delora_icp_dense_fwd_bwd writes for source = this frame's grids moved by T[s], target = the previous frame's grids
 * (the training step's orientation, scan_2 -> scan_1), bit-identical to that operator run alone at B = 1 on the two
 * frames; rows with valid[s] = 0 are zeros.  The 3x4 part of T reaches the ICP on the device.
 * The launch sequence depends on neither `active` nor the stream state (one captured call serves every tick), so the
 * ICP runs at B = S every tick.  Streams without a transform cost it no search: a stream without a frame has empty
 * grids from the projection, and a stream on its first frame since the start or a reset has its grids cached and then
 * emptied before the ICP (odometry_streams_grids_kernel<0>), so no source pixel ever searches a stale or empty target;
 * the valid streams' grids are cached after the ICP (<1>).  Each stream's grids are thus copied once per tick (64 bytes
 * per cell read and written) and only when it has a frame; a separate staging grid for the ICP's sources would have
 * copied every stream's grids twice and cost another 32 bytes per cell and stream.
 * Measured on one H100 80GB HBM3 at a 700 W power limit (max SM clock 1980 MHz), graph-replayed ticks, all streams
 * active, near-identity heads on consecutive synthetic frames, medians of alternating samples, _streams_push ->
 * _streams_push_residual per tick: 64 x 2048: S = 1 1.20 -> 1.28 ms, S = 4 2.15 -> 2.30 ms,
 * S = 16 8.22 -> 8.70 ms; 64 x 720: S = 1 1.13 -> 1.18 ms, S = 4 1.33 -> 1.40 ms, S = 16 4.97 -> 5.12 ms
 * (scripts/gpu_odometry_eval.py, profiles/odometry_eval_h100_700w.json).
 * Refused before any launch, naming the field or pointer: an invalid descriptor; null residual_params; a loss_flags
 * without an ICP loss bit or with any bit other than DELORA_LOSS_PO2PO / _PO2PL / _PL2PL / DELORA_NORMAL_LINEAR; nb_h or
 * nb_w not odd and positive; epsilon_range < 0; min_neighbors < 0; null points / n_points / workspace / T / valid /
 * losses.  Models flagged DELORA_MODEL_NORMALIZATION_SCALING cannot be streamed here: the residual's grids would need a
 * definition of their units and of the projection they come from. */
typedef struct {
    float lambda_po2pl;                  /* weight of po2pl in dL/dT only; the loss rows are unweighted */
    uint32_t loss_flags;                 /* DELORA_LOSS_PO2PO / _PO2PL / _PL2PL (at least one), DELORA_NORMAL_LINEAR */
    int nb_h, nb_w;                      /* neighborhood_side_length (7, 11): odd and positive */
    float epsilon_range;                 /* 0.5 */
    int min_neighbors;                   /* min_num_points_in_neighborhood_to_determine_point_class, 10 */
} delora_odometry_residual_params;
int64_t delora_odometry_streams_residual_workspace_bytes(const delora_odometry_desc* d);   /* host only, -1 if invalid */
/* Zero the workspace (no stream has a previous frame, the ICP scratch is armed for B = S), arm the projection keys and
 * empty the cached grids.  Once after allocation, instead of delora_odometry_streams_init. */
int delora_odometry_streams_residual_init(const delora_odometry_desc* d, void* workspace, void* stream);
int delora_odometry_streams_push_residual(const delora_odometry_desc* d, const delora_odometry_residual_params* rp,
                                          const float* points, const int32_t* n_points, const int32_t* active,
                                          void* workspace, float* T, int32_t* valid, float* losses, void* stream);

/* How well each streamed frame determines its transform, beside the residual: the Gauss-Newton information of the
 * residual's ICP objective at the served T (delora_icp_dense_information), so that a host can tell a frame of a
 * degenerate scene (corridor, open field, flat wall: low residual, an unobservable direction) from a good one, give a
 * fusion filter a covariance or flag the frame.  A diagnostic: T is what _streams_push_residual serves.
 *
 * The information workspace is the residual workspace with one section appended: no offset of the residual layout
 * moves, so delora_odometry_streams_load_weights and delora_odometry_streams_reset work on it unchanged (_info_init
 * replaces _residual_init).  Appended (256-byte aligned): the information rows of the S pairs and the operator's
 * info_scratch at B = S (delora_icp_information_scratch_floats(S, H, W): 4 bytes per cell and stream for the NN ids,
 * 8 bytes per cell and stream for the partial rows, a 64-float row per 32 cells), 12 bytes per cell and stream in all: at 64 x 2048,
 * 1.5 MiB per stream; at 64 x 720, 0.53 MiB per stream.
 *
 * delora_odometry_streams_push_info: the arguments of delora_odometry_streams_push_residual plus info
 * [S, DELORA_INFO_ROW] (device, required).  T, valid and losses are what _streams_push_residual writes for the same
 * history, byte for byte; info[s] is the row delora_icp_dense_information writes for that pair, bit-identical to the
 * operator run alone at B = 1 on the two frames, for every stream with valid[s] = 1; rows with valid[s] = 0 are zeros.
 * Graph-capturable like _streams_push_residual (the launch sequence depends on neither `active` nor the stream state).
 * Refused before any launch: everything _streams_push_residual refuses, and a null info.
 * Measured on one H100 80GB HBM3 at a 700 W power limit (max SM clock 1980 MHz), graph-replayed ticks, all streams
 * active, near-identity heads on consecutive synthetic frames, medians of alternating samples,
 * _streams_push_residual -> _streams_push_info per tick: 64 x 2048: S = 1 1.28 -> 1.34 ms, S = 4 2.31 -> 2.42 ms, S
 * = 16 8.71 -> 8.96 ms; 64 x 720: S = 1 1.18 -> 1.22 ms, S = 4 1.39 -> 1.43 ms, S = 16 5.12 -> 5.19 ms. Of that, per
 * tick (torch.profiler): icp_info_rows_kernel 4.3 / 16.4 / 60.0 us at 64 x 2048 (S = 1 / 4 / 16), 2.4 / 5.3 / 23.9
 * us at 64 x 720; icp_info_finalize_kernel 57 / 63 / 90 us and 32 / 33 / 41 us, almost all of it the float64 Jacobi
 * solve, which runs on one thread per pair (scripts/gpu_odometry_streams_info.py,
 * profiles/odometry_streams_info_h100_700w.json). */
int64_t delora_odometry_streams_info_workspace_bytes(const delora_odometry_desc* d);   /* host only, -1 if invalid */
/* Zero the workspace, arm the projection keys and empty the cached grids.  Once after allocation, instead of
 * delora_odometry_streams_residual_init. */
int delora_odometry_streams_info_init(const delora_odometry_desc* d, void* workspace, void* stream);
int delora_odometry_streams_push_info(const delora_odometry_desc* d, const delora_odometry_residual_params* rp,
                                      const float* points, const int32_t* n_points, const int32_t* active,
                                      void* workspace, float* T, int32_t* valid, float* losses, float* info,
                                      void* stream);

/* Several streams of a model flagged DELORA_MODEL_NORMALIZATION_SCALING in one workspace.  Such a model sees each pair
 * divided by the factor of that pair, so a stream's previous frame is projected anew every tick: the workspace keeps
 * each stream's previous SCAN, and one call per tick computes the S factors, projects both scans of every pair, runs
 * the model once at batch S and multiplies each translation back by its factor.
 *
 * The normalised streams workspace is the streams workspace with sections appended: no offset of the streams layout
 * moves, so delora_odometry_streams_load_weights and delora_odometry_streams_reset work on it unchanged
 * (_streams_normalized_init replaces _streams_init).  The streams layout's cached images become this tick's projection
 * of each previous frame, rewritten every tick; its S key buffers serve both projections.  Appended, each 256-byte
 * aligned, for S = max_batch streams: the point rows [2S, 3, n_stride] fp32 (each stream's previous frame, then its
 * last frame), their counts [2S] and the count of each stream's last frame [S] int32, and the factors [S] fp32.
 * Sizes from the host-only query (layers {2,2,2,2}, resnet_outputs 1000, two heads, n_stride 131072), streams ->
 * normalised streams workspace: 64 x 2048: S = 1 86.0 -> 89.0 MiB, S = 4 271.8 -> 283.8 MiB,
 * S = 16 1015.1 -> 1063.1 MiB; 64 x 720: S = 1 46.2 -> 49.2 MiB, S = 4 112.8 -> 124.8 MiB, S = 16 379.1 -> 427.1 MiB.
 *
 * delora_odometry_streams_push_normalized: the arguments of delora_odometry_streams_push, plus factor [S] fp32, a
 * required device output.  For every stream with valid[s] = 1, row s of T (its translation multiplied by the factor)
 * and factor[s] are bit-identical to delora_odometry_pairs_normalized with B = 1 on (that stream's previous active
 * frame, this frame), in an inference workspace with the same weights.  valid[s] follows _streams_push: 1 for an active
 * stream that has a previous frame.  factor[s] = 0 where valid[s] = 0.  Inactive streams leave their T row and their
 * cached frame untouched.  An empty active frame gives NaN for the pairs it belongs to (this one and, after it, the
 * next), as in delora_odometry_pairs_normalized; no other stream is affected.  Per tick: the masked count clamp fused
 * with the staging of the frames (odometry_streams_stage_kernel), delora_normalization_factors' kernel at B = S (each
 * factor is the B = 1 factor bit for bit: its per-scan float64 order does not depend on B), two scaled projections,
 * the pairs' trunk-input conversion, the trunk and the tail at B = S, and odometry_streams_out_kernel's rescaling
 * variant.
 * Measured on one H100 80GB HBM3 at a 700 W power limit (SM clock 1980 MHz), graph-replayed ticks, all streams active,
 * near-identity heads on consecutive synthetic frames, medians of alternating samples, ms per tick: _streams_push on
 * the same weights / _streams_push_normalized / S captured _pairs_normalized calls at B = 1:
 * 64 x 2048: S = 1 1.21 / 1.24 / 1.23, S = 4 2.18 / 2.22 / 5.00, S = 16 8.34 / 8.48 / 19.82;
 * 64 x 720: S = 1 1.14 / 1.17 / 1.17, S = 4 1.35 / 1.39 / 4.69, S = 16 5.02 / 5.09 / 18.91
 * (scripts/gpu_odometry_streams_normalized.py, profiles/odometry_streams_normalized_h100_700w.json).  At S = 16 a
 * stream costs 0.53 ms (64 x 2048) and 0.32 ms (64 x 720) instead of 1.24 and 1.18 ms; at S = 1 the staging costs what
 * the one pairs call does, within 0.01 ms.
 * Only launches, with a sequence that depends on neither `active` nor the stream state, so one captured call serves
 * every tick.  Counts above n_stride are clamped on the device.  Refused before any launch, naming the field or
 * pointer: an invalid descriptor, null points / n_points / workspace / T / valid / factor. */
int64_t delora_odometry_streams_normalized_workspace_bytes(const delora_odometry_desc* d); /* host only, -1 if invalid */
/* Zero the workspace (no stream has a previous frame) and arm the projection keys.  Once after allocation, instead of
 * delora_odometry_streams_init. */
int delora_odometry_streams_normalized_init(const delora_odometry_desc* d, void* workspace, void* stream);
int delora_odometry_streams_push_normalized(const delora_odometry_desc* d, const float* points, const int32_t* n_points,
                                            const int32_t* active, void* workspace, float* T, int32_t* valid,
                                            float* factor, void* stream);

/* Several streams served on the reference's two-resolution recipe: the images a model trained with w_pre > 0 saw in
 * training, and the reference's Tester feeds it (its dataset loads the preprocessed point lists, src/data/
 * dataset.py:115-122, and Deployer.step projects them at the model width, src/deploy/deployer.py:252-255), with the
 * training step's ICP residual beside every transform, for plain and normalization_scaling models alike.  The raw-scan
 * streams above feed the model the ROS node's input instead (each frame projected straight to H x W); the two images
 * differ wherever a w_pre pixel straddles two W pixels.  Per tick, for S = max_batch streams: the training step's stages
 * 1-3 at B = S (delora_odometry_train_step, w_pre > 0), each pair's first frame coming from the workspace: projection +
 * normals of the S new frames at H x w_pre (rp's neighbourhood); with DELORA_TRAIN_NORMALIZATION_SCALING in
 * rp->loss_flags the factor of each pair (cached frame, new frame) over their valid H x w_pre cells; both frames of
 * every pair projected again to H x W (delora_project_grids_fwd; divided by the pair's factor when flagged, normals
 * not); the trunk and tail at B = S, each quaternion divided by its own row's norm; the dense ICP at B = S, source =
 * this frame's H x W grids moved by the model's T, target = the previous frame's (the training orientation), in the
 * model's units (flagged models: normalised, as training); then each active stream's new H x w_pre grids become its
 * cached previous frame.  A cached frame is projected again every tick, so one layout serves both kinds of model.
 *
 * The recipe streams workspace is the residual workspace with sections appended: no offset of the streams layout
 * moves, so delora_odometry_streams_load_weights and delora_odometry_streams_reset work on it unchanged
 * (_streams_pre_init replaces _streams_init).  The residual sections hold this tick's H x W grids of both frames and
 * the ICP's inputs, outputs and scratch.  Appended, each 256-byte aligned, for S streams: the depth keys, image and
 * index map of the new frames at H x w_pre (S * H * w_pre * 28 bytes), the H x w_pre point and normal grids of each
 * stream's cached frame and of the new frames (S * H * w_pre * 64 bytes), T in the model's units [S, 16] and the pair
 * factors [S].  Sizes from the host-only query (layers {2,2,2,2}, resnet_outputs 1000, two heads, n_stride 131072,
 * w_pre 2250), streams -> residual -> recipe streams workspace:
 *   64 x 720:  S = 1 46.2 -> 50.9 -> 63.6 MiB, S = 4 112.8 -> 131.6 -> 182.1 MiB, S = 16 379.1 -> 454.3 -> 656.4 MiB;
 *   64 x 2048: S = 1 86.0 -> 99.3 -> 111.9 MiB, S = 4 271.8 -> 325.0 -> 375.5 MiB, S = 16 1015.1 -> 1227.9 -> 1430.0 MiB.
 *
 * delora_odometry_streams_push_pre: the arguments of delora_odometry_streams_push_residual, plus factor [S] fp32.
 * T [S, 16] and valid [S] follow _streams_push's rules (valid[s] = 1 for an active stream with a previous frame; T rows
 * of the others are not written).  For a plain model row s of T is bit-identical to delora_odometry_pairs at B = 1 on
 * (previous frame, this frame) given as their preprocessed point lists (the valid H x w_pre cells in row-major order,
 * what Preprocesser.preprocess_scans stores); for a flagged one T's translation is multiplied back by the factor, as
 * delora_odometry_pairs_normalized does.  losses [S, DELORA_LOSS_ROW] (device, required): the ICP row where valid[s] = 1,
 * bit-identical to delora_icp_dense_fwd_bwd at B = 1 on the two frames' grids and T's 3x4 in the model's units; zeros
 * elsewhere.  It is the number delora_odometry_train_eval reports for the pair, up to the trunk's rounding (the
 * training forward keeps the stem's pre-activation in fp16).  factor [S] (device): required with
 * DELORA_TRAIN_NORMALIZATION_SCALING in rp->loss_flags and NULL without it; factor[s] = the pair's factor where
 * valid[s] = 1 (eval's losses[b][6]), 0 elsewhere.  An empty active frame gives what delora_odometry_pairs_normalized
 * gives (NaN) for flagged models and what _streams_push gives otherwise; no other stream is affected.  A stream
 * without a transform this tick costs the ICP no search: its source grids are emptied first.  Inactive streams leave
 * their T row and cached frame untouched.
 * Cost per tick: the raw-scan path's projection, trunk and tail, plus the projection + normals at H x w_pre, a second
 * H x W projection per pair, the ICP at B = S and the cache write (64 bytes per H x w_pre cell of each active stream).
 * Measured on one H100 80GB HBM3 at a 700 W power limit (max SM clock 1980 MHz), graph-replayed ticks, all streams
 * active, near-identity heads on consecutive synthetic frames, w_pre 2250, medians of alternating samples, ms per tick
 * _streams_push / _streams_push_residual / _streams_push_pre on the same weights:
 * 64 x 720: S = 1 1.15 / 1.20 / 1.21, S = 4 1.34 / 1.41 / 1.47, S = 16 4.99 / 5.14 / 5.44;
 * 64 x 2048: S = 1 1.21 / 1.29 / 1.31, S = 4 2.17 / 2.31 / 2.38, S = 16 8.30 / 8.73 / 8.98
 * (scripts/gpu_odometry_streams_pre.py, profiles/odometry_streams_pre_h100_700w.json).  The recipe costs 0.02-0.30 ms
 * per tick over the raw-scan residual, which already pays for normals and the ICP; the re-projection of the cached
 * frames, the part a second layout caching plain models' images could save, is a share of that, so there is one
 * layout.  On those synthetic 64-ring scans, 2.2 % (64 x 720) and 7.3 % (64 x 2048) of the H x W pixels differ between
 * the raw-scan and the recipe image.
 * Only launches, with a sequence that depends on neither `active` nor the stream state, so one captured call serves
 * every tick.  Refused before any launch, naming the field or pointer: everything _streams_push_residual refuses,
 * w_pre < 2 (0 included) or H * w_pre >= 2^27, a loss_flags bit other than the ICP loss bits, DELORA_NORMAL_LINEAR and
 * DELORA_TRAIN_NORMALIZATION_SCALING, a null losses, and a factor that does not match the flag. */
int64_t delora_odometry_streams_pre_workspace_bytes(const delora_odometry_desc* d);   /* host only, -1 if invalid */
/* Zero the workspace (no stream has a previous frame, the ICP scratch is armed for B = S), arm the projection keys and
 * empty the cached grids.  Once after allocation, instead of delora_odometry_streams_init. */
int delora_odometry_streams_pre_init(const delora_odometry_desc* d, void* workspace, void* stream);
int delora_odometry_streams_push_pre(const delora_odometry_desc* d, const delora_odometry_residual_params* rp,
                                     const float* points, const int32_t* n_points, const int32_t* active,
                                     void* workspace, float* T, int32_t* valid, float* losses, float* factor,
                                     void* stream);

/* The recipe streams with the information of each frame's residual beside it (see delora_icp_dense_information and
 * _streams_push_info): the Gauss-Newton information of the recipe's ICP objective at the served T, so that a host
 * serving a model on the images it trained on, plain or normalization_scaling, can tell a frame of a degenerate scene
 * from a good one.  The recipe streams workspace with the information section of _streams_info appended (the rows of
 * the S pairs and delora_icp_information_scratch_floats(S, H, W) floats, each 256-byte aligned): no offset of the
 * recipe layout moves, so delora_odometry_streams_load_weights and delora_odometry_streams_reset work on it unchanged
 * (_pre_info_init replaces _pre_init).
 * delora_odometry_streams_push_pre_info: the arguments of delora_odometry_streams_push_pre plus info
 * [S, DELORA_INFO_ROW] (device, required).  T, valid, losses and factor are what _streams_push_pre writes for the same
 * history, byte for byte.  Where valid[s] = 1, info[s] is, bit for bit, the row of the operator run alone at B = 1 on
 * the pair's H x W grids and T's 3x4 in the model's units: delora_icp_dense_information for a plain model;
 * delora_icp_dense_information_scaled with the pair's factor for a flagged one, whose grids are divided by that
 * factor.  So H, its eigenvalues and eigenvectors are always in the metres and radians of the served T, xi = (x, y, z,
 * rot x, rot y, rot z) perturbing T on the right; the losses row and M, M' stay the model's.  Rows with valid[s] = 0
 * are zeros.  Graph-capturable like _streams_push_pre.  Refused before any launch: everything _streams_push_pre
 * refuses, and a null info.
 * Measured on one H100 80GB HBM3 at a 700 W power limit (max SM clock 1980 MHz), graph-replayed ticks, all streams
 * active, near-identity heads on consecutive synthetic frames, w_pre 2250, medians of alternating samples,
 * _streams_push_pre -> _streams_push_pre_info per tick: 64 x 2048: S = 1 1.30 -> 1.36 ms, S = 4 2.34 -> 2.46 ms,
 * S = 16 8.98 -> 9.21 ms; 64 x 720: S = 1 1.20 -> 1.23 ms, S = 4 1.46 -> 1.50 ms, S = 16 5.41 -> 5.52 ms
 * (scripts/gpu_odometry_streams_pre_adapt_info.py, profiles/odometry_streams_pre_adapt_info_h100_700w.json). */
int64_t delora_odometry_streams_pre_info_workspace_bytes(const delora_odometry_desc* d);   /* host only, -1 if invalid */
int delora_odometry_streams_pre_info_init(const delora_odometry_desc* d, void* workspace, void* stream);
int delora_odometry_streams_push_pre_info(const delora_odometry_desc* d, const delora_odometry_residual_params* rp,
                                          const float* points, const int32_t* n_points, const int32_t* active,
                                          void* workspace, float* T, int32_t* valid, float* losses, float* factor,
                                          float* info, void* stream);

/* ---------------------------------------------------------------------------------------
 * Odometry training: raw scan pairs -> updated weights, one call per step.
 * Replaces, for the self-supervised step, deploy.deployer.Deployer.step + Trainer's Adam
 *   (src/deploy/deployer.py:237-342, src/deploy/trainer.py:23-24) as delora_b200/train_step.py's SyntheticTrainStep
 *   runs it: projection and normals of both scans, OdometryModel.forward, the dense ICP losses (source = scan_2 moved
 *   by the predicted T, target = scan_1), objective = mean over the pairs of po2po + lambda_po2pl * po2pl + pl2pl,
 *   the backward through the heads, resnet.fc and the encoder trunk (the kernels and order of the Python training
 *   encoder), one Adam update (no weight decay) of the fp32 master weights and one re-prep of the bf16 filters.
 * Same descriptor and .dlw blob as inference; the same models are not representable.
 *
 * Normals (d->w_pre).  0: the normals are estimated on the model's H x W image (SyntheticTrainStep's shortcut).
 * > 0: the reference's recipe -- its offline stage (src/preprocessing/preprocesser.py) projects each scan at
 * horizontal_cells_preprocessing and estimates the normals there, its training stage (src/deploy/deployer.py:252-261)
 * projects the stored points at the model width.  Each step runs delora_project_normals_fwd of the 2B scans at
 * H x w_pre (nb_h, nb_w, epsilon_range, min_neighbors of the step), then delora_project_grids_fwd to H x W; the trunk
 * onward is unchanged.  The workspace gains, after every other section, the image, index map and both grids at
 * H x w_pre for 2 * max_batch scans (2 * max_batch * H * w_pre * 52 bytes, each buffer 256-byte aligned), and its
 * one depth-key buffer grows to max(W, w_pre) columns; nothing moves at w_pre = 0.  At 64 x 720, n_stride 131072,
 * w_pre 0 -> 2250: 325.2 -> 341.0 MiB (max_batch 1), 521.3 -> 584.4 MiB (4), 1305.9 -> 1558.3 MiB (16).  Measured
 * step cost on one H100 80GB HBM3 at a 700 W power limit (graph-replayed steps, paired differences): within the
 * noise (< 0.02 ms) at B = 1, +0.10 ms at B = 4, +0.38 ms at B = 16 (14.35 -> 14.70 ms).
 *
 * Workspace: one caller-owned device buffer of delora_odometry_train_workspace_bytes(d) bytes holds the fp32 master
 * weights, their gradient, Adam's m, v and step count, the bf16 filters, every saved activation and backward buffer
 * for max_batch pairs and the ICP scratch.  Its layout is a function of the descriptor (the split-K scratch of the
 * weight gradients is sized for the current device's SM count; 132, an H100 SXM, without a device).  It holds device
 * pointers into itself: do not move or copy it to another address.  Use: _train_init once, then any number of
 * _train_step calls, _train_weights to read the weights out.  Every step is launches only (no allocation, no
 * synchronisation, no host decision on device data), so a step can be captured into a CUDA graph and replayed;
 * B may change from one step to the next.  Results are bit-identical from run to run. */
typedef struct {
    float lr, beta1, beta2, eps;         /* Adam (torch defaults 0.9, 0.999, 1e-8); lr >= 0, betas in [0, 1), eps > 0 */
    float lambda_po2pl;                  /* config lambda_po2pl */
    uint32_t loss_flags;                 /* DELORA_LOSS_* / DELORA_NORMAL_LINEAR bits, at least one ICP loss bit
                                            (PO2PO, PO2PL, PL2PL), plus DELORA_LOSS_IDENTITY_FIT,
                                            DELORA_TRAIN_NORMALIZATION_SCALING and DELORA_TRAIN_DROPOUT (see
                                            _train_step) */
    int nb_h, nb_w;                      /* neighborhood_side_length (7, 11): odd and positive */
    float epsilon_range;                 /* 0.5 */
    int min_neighbors;                   /* min_num_points_in_neighborhood_to_determine_point_class, 10 */
} delora_odometry_train_params;

/* Host only (no GPU needed): -1 (and delora_last_error()) for an invalid descriptor, w_pre included.  The four
 * training entry points refuse a w_pre other than 0 or >= 2 with H * w_pre < 2^27, naming the field. */
int64_t delora_odometry_train_workspace_bytes(const delora_odometry_desc* d);
/* Zero the workspace, set the projection key buffer to all ones, copy `weights` (DEVICE fp32, the .dlw blob) into the
 * master weights, zero Adam's m, v and step count and prep the bf16 filters (fprop and flipped layouts).  The prep
 * table is copied from host memory (the call may wait for the stream to reach it). */
int delora_odometry_train_init(const delora_odometry_desc* d, const float* weights, void* workspace, void* stream);
/* One training step on B pairs (1 <= B <= max_batch): points [2B, 3, n_stride] and n_points [2B] as for
 * delora_odometry_pairs.  Outputs, each DEVICE and each may be NULL: losses [B, DELORA_LOSS_ROW] as the ICP operator
 * writes them; T [B, 16] of the weights BEFORE the update; pooled [B, 512]; grads [weight_floats] the gradient of the
 * objective in blob order.  Refused before any launch: an invalid descriptor or hyperparameter (the message names the
 * field), null points / n_points / workspace, B outside [1, max_batch].
 * Identity pre-training: with DELORA_LOSS_IDENTITY_FIT in hp->loss_flags the objective is the reference's first phase
 * (unsupervised_at_start: False; src/deploy/deployer.py:324-327, :334-336), MSELoss(T_{B-1}, I) / B: only the LAST
 * pair's 4x4 transform counts (the reference overwrites its loss inside the pair loop), the mean runs over its 16
 * entries.  dL/dT is 2 (T - I) / (16 B) on the 3x4 part of row B-1 and zero elsewhere; the backward from there on is
 * the ICP objective's (the norm of the whole [B, 4] quaternion block still gives every pair's head outputs a
 * gradient).  The ICP losses are still computed and written to `losses` (the reference logs them in this phase); the
 * identity objective goes to losses[B-1][5] (column 5 is 0 in the other rows and in steps without the bit).  At least
 * one ICP loss bit is still required.
 * Normalised models: with DELORA_TRAIN_NORMALIZATION_SCALING in hp->loss_flags the step trains a model that uses
 * normalization_scaling as the reference's Deployer.step does (src/deploy/deployer.py:222-235, :252-261, :344-346).  It
 * needs the reference's recipe, d->w_pre > 0 (refused before any launch otherwise, the message names w_pre): the normals
 * come from the unscaled points at H x w_pre; the factor of each pair is the mean of its two scans' mean ranges over
 * the valid H x w_pre cells (the points the preprocessing stored; the definition of delora_normalization_factors, the
 * same float64 order), and those points are divided by it (correctly rounded) before the H x W projection.  The ICP
 * losses are in normalised units, as in the reference; the identity fit uses the unscaled T; the T output is rescaled
 * (T[:3, 3] *= factor in fp32); losses[b][6] is the factor (0 in steps without the bit).  No workspace size changes:
 * the factor is kept in the H x w_pre image, which nothing reads after the preprocessing projection.
 * Dropout: with DELORA_TRAIN_DROPOUT in hp->loss_flags the step applies the three dropouts (p = 0.2) of a model
 * configured with use_dropout (src/models/resnet_modified.py:33-38, :96, :110, :117; the reference's Trainer never
 * calls model.eval(), so they are active in every training step, the identity fit included).  It combines with
 * DELORA_LOSS_IDENTITY_FIT and DELORA_TRAIN_NORMALIZATION_SCALING.  The masks follow the contract below, with s = the
 * workspace's Adam step count at the start of the step (the int64 of _train_get_state) and the workspace's seed
 * (delora_odometry_train_set_dropout_seed, 0 after _train_init); they are drawn on the device, so a graph replay draws
 * fresh masks every step and a run resumed through _train_set_state + _train_set_dropout_seed draws the masks the
 * uninterrupted run would have.  The masks are regenerated in the backward; nothing is stored but x3d below, and no
 * workspace size changes.
 *   - input (tensor 0): every element of cat(image_1, image_2) is multiplied by keep * 1.25f in fp32 inside the trunk
 *     input conversion, before the bf16 (+ bf16 residual) rounding: the stem sees the bits of pre-multiplied images.
 *   - stage-3 channels (tensor 1, Dropout2d): layer4's first block (its conv1, its downsample and both weight
 *     gradients) reads x3d = bf16_rn(float(x3) * 1.25f) for kept (pair, channel) and 0 for dropped ones, x3 = layer3's
 *     output, which stays as it was for the act' epilogues.  The backward multiplies the data gradient of x3, after
 *     act'(x3), by keep * 1.25 and rounds it to bf16 once more.  x3d lives in a stage-3 backward buffer that nothing
 *     writes before layer3's own backward.
 *   - fc output (tensor 2): fc_out = act(keep * 1.25f * (W pooled + b)) in fp32; the heads' backward multiplies the
 *     gradient of fc_out by keep * 1.25 after act'.
 * Without the bit every launch is the one of a step without dropout; inference and streams never apply dropout. */
int delora_odometry_train_step(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                               const float* points, const int32_t* n_points, int B, void* workspace,
                               float* losses, float* T, float* pooled, float* grads, void* stream);
/* Evaluation on a training workspace: the ICP losses of the current weights on B pairs, nothing updated.  Replaces the
 * loss branch of the reference's Tester (inference_only: False; src/deploy/tester.py:61-65 ->
 * src/deploy/deployer.py:280-369) for a host that trains through delora_odometry_train_step and scores held-out
 * sequences (training_identifiers / testing_identifiers) on the same workspace.  Same descriptor, hyperparameters,
 * inputs and losses / T / pooled outputs as the step; it runs the step's projection + normals (at w_pre when set),
 * forward and ICP losses (one function serves both) and stops: from the same workspace state and inputs its outputs are
 * bit-identical to the step's (T of the weights before the update), and the master weights, the gradient, Adam's m, v
 * and step count, the dropout seed and the bf16 filters are byte-for-byte unchanged.  Steps interleaved with evals of
 * any B end in the state the steps alone reach, bit for bit (the eval records its batch size for the ICP scratch's
 * re-arm).  Dropout is the identity, as at inference: DELORA_TRAIN_DROPOUT is accepted and ignored, so a host can pass
 * the parameters it trains with, and the outputs are those of a step without the bit.  DELORA_LOSS_IDENTITY_FIT is
 * accepted and ignored too: the identity objective belongs to the step's backward, column 5 of `losses` stays 0.
 * DELORA_TRAIN_NORMALIZATION_SCALING acts as in the step (T in metres, the factor in column 6).  lr, betas and eps are
 * validated and not used.  Launches only, capturable into a CUDA graph; the step's refusals, naming the argument.
 * Measured on the H100 above (w_pre 0, lr 0, graph-replayed, medians of alternating samples), _train_step ->
 * _train_eval: 64 x 720: B = 1 3.53 -> 1.19 ms, B = 4 4.43 -> 1.40 ms, B = 16 14.32 -> 5.20 ms; 64 x 2048: B = 1
 * 3.73 -> 1.28 ms, B = 4 6.68 -> 2.34 ms, B = 16 22.97 -> 8.83 ms. */
int delora_odometry_train_eval(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                               const float* points, const int32_t* n_points, int B, void* workspace,
                               float* losses, float* T, float* pooled, void* stream);
/* Copy the current fp32 master weights to `weights` (DEVICE fp32[weight_floats]): a .dlw blob, loadable by
 * delora_odometry_load_weights and delora_odometry_train_init. */
int delora_odometry_train_weights(const delora_odometry_desc* d, const void* workspace, float* weights, void* stream);
/* The optimizer state, for checkpoints that resume a run exactly (src/deploy/trainer.py:26-36 loads, :153-173 saves
 * model_state_dict + optimizer_state_dict).  weights, exp_avg (Adam's m), exp_avg_sq (v): DEVICE fp32[weight_floats]
 * each, in blob order; step: DEVICE int64, the number of Adam updates so far (torch's state["step"]).
 * _get_state copies them out of a training workspace; every output may be NULL (skipped).  Launches copies only, no
 * synchronisation: capturable into a CUDA graph.
 * _set_state, after _train_init: overwrites the master weights, m, v and the step count and re-preps the bf16 filters
 * (fprop and flipped layouts) from the new weights; the next step continues as the workspace the state came from
 * would have (bit-identical), whatever batch size that one last ran.  All four inputs are required (a fresh Adam is
 * _train_init's).  Both refuse before any launch, naming the argument: an invalid descriptor, a null input, a null
 * workspace. */
int delora_odometry_train_get_state(const delora_odometry_desc* d, const void* workspace, float* weights, float* exp_avg,
                                    float* exp_avg_sq, int64_t* step, void* stream);
int delora_odometry_train_set_state(const delora_odometry_desc* d, const float* weights, const float* exp_avg,
                                    const float* exp_avg_sq, const int64_t* step, void* workspace, void* stream);

/* ---- Adapting streams: serve S = max_batch streams and take the training step on the pairs just served, one call per
 * tick.  The model keeps learning on the frames it serves (a new environment, a new sensor mount, a model trained on
 * another dataset) without a second workspace, a host copy of each stream's previous scan, a second projection and
 * forward of every pair, or a weight hand-off (_train_weights -> _streams_load_weights) after every update.
 *
 * Workspace: the training workspace of d (max_batch = S; delora_odometry_train_workspace_bytes(d) bytes, its layout
 * unchanged) followed by the stream section, each buffer 256-byte aligned:
 *   w_pre = 0: each stream's cached previous frame as its H x W image (S * H * W * 16 bytes) and its H x W point and
 *              normal grids (2 * S * H * W * 16 bytes);
 *   w_pre > 0: each stream's cached H x w_pre point and normal grids (2 * S * H * w_pre * 16 bytes);
 *   then has_prev [S] int32 and the device count of valid pairs (one int32).
 * So every delora_odometry_train_* entry point called with d works on it unchanged and leaves the stream section alone:
 * _train_weights, _train_get_state / _set_state (the .dlt checkpoint), _train_set_dropout_seed, _train_eval.  Sizes from
 * the host-only query (layers {2,2,2,2}, resnet_outputs 1000, two heads, n_stride 131072), training -> adapting streams
 * workspace:
 *   64 x 720, w_pre 0:    S = 1 325.2 -> 327.3 MiB, S = 4 521.3 -> 529.8 MiB, S = 16 1305.9 -> 1339.7 MiB;
 *   64 x 720, w_pre 2250: S = 1 341.0 -> 345.4 MiB, S = 4 584.4 -> 602.0 MiB, S = 16 1558.3 -> 1628.7 MiB;
 *   64 x 2048, w_pre 0:   S = 1 425.5 -> 431.5 MiB, S = 4 922.5 -> 946.5 MiB, S = 16 2910.6 -> 3006.6 MiB.
 *
 * delora_odometry_streams_adapt_init: _train_init on the whole workspace (the stream section zeroed: no stream has a
 * previous frame), then the cached grids emptied.  delora_odometry_streams_adapt_reset: forget the previous frame of
 * every stream with mask[s] != 0 (device int32 [S]); only launches.
 *
 * delora_odometry_streams_push_adapt, one tick: points [S, 3, n_stride], n_points [S], active [S] or NULL (all active),
 * T [S, 16] and valid [S] as for delora_odometry_streams_push; losses [S, DELORA_LOSS_ROW] as for _streams_push_pre.
 *   1. The training step's stages 1-3 at B = S: scan_1 of pair s is stream s's cached frame, scan_2 this tick's frame.
 *      Only this tick's frames are projected (with normals; at w_pre > 0 at H x w_pre, then both frames of every pair
 *      re-projected at H x W, divided by the pair factor with DELORA_TRAIN_NORMALIZATION_SCALING).
 *   2. The quaternion of each row is divided by its own row's norm, not by that of the [S, 4] block, so a stream's T
 *      does not depend on the other streams (the reference's training at batch_size 1 does the same).  The sum has the
 *      block norm's fmaf order, so at S = 1 the bits are those of _train_step at B = 1 on (previous frame, this frame).
 *   3. valid[s] = active[s] && stream s has a previous frame.  T (the weights before this tick's update; in metres for
 *      normalised models) and the loss row are written for valid streams (losses[s][6] = the factor for normalised
 *      models, as in the step); the T rows of the others are not written, their loss rows are zeros, and their ICP
 *      sources are emptied, so they cost the ICP no search.
 *   4. update = 1 only: the backward and one Adam update of the objective mean over the valid pairs of po2po +
 *      lambda_po2pl * po2pl + pl2pl, i.e. the mean of the valid streams' B = 1 gradients.  1 / n_valid is read on the
 *      device; invalid rows get dL/dT = 0 and add exact zeros to every sum.  With no valid pair the step count does not
 *      advance and Adam does not run (the gradient section is still written).  The bf16 filters are re-prepped after
 *      Adam, so the next tick serves the updated model.  update = 0 serves and scores only, so a host can adapt on its
 *      own cadence (for instance when the residual rises).
 *   5. Every active stream's stage-1 output of this tick becomes its cached frame; inactive streams keep theirs.
 * Only launches, with a sequence that depends on neither `active`, the stream state nor n_valid: one captured graph per
 * value of `update` serves every tick.  Refused before any launch, naming the field or pointer: everything _train_step
 * refuses at B = S, update not 0 or 1, a null points / n_points / workspace / T / valid / losses,
 * DELORA_LOSS_IDENTITY_FIT (a pre-training phase, not adaptation) and DELORA_TRAIN_DROPOUT (the served T is
 * dropout-free, and one forward cannot be both).  Out of scope: dropout while adapting and any policy for when to
 * adapt; several GPUs adapting one model: delora_odometry_streams_push_adapt_group below; streams of several sensor
 * geometries adapting one model: delora_odometry_streams_push_adapt_geometries below.
 * Cost, measured on one H100 80GB HBM3 at a 700 W power limit (max SM clock 1980 MHz), graph-replayed ticks, all
 * streams active, near-identity heads, lr 0, medians of alternating samples, ms per tick at S = 1 / 4 / 16,
 * update = 0 | update = 1 | _train_step at B = S alone | the two-workspace composition a host needs without this call
 * (a _streams_push_residual tick, or _streams_push_pre at w_pre > 0, + _train_step at B = S + _train_weights +
 * _streams_load_weights):
 *   64 x 720, w_pre 0:    1.20 / 1.41 / 5.12 | 3.51 / 4.43 / 14.20 | 3.50 / 4.42 / 14.23 | 4.82 / 5.95 / 19.54;
 *   64 x 720, w_pre 2250: 1.23 / 1.47 / 5.45 | 3.58 / 4.50 / 14.46 | 3.56 / 4.51 / 14.52 | 4.92 / 6.11 / 20.12;
 *   64 x 2048, w_pre 0:   1.31 / 2.33 / 8.78 | 3.79 / 6.67 / 22.89 | 3.76 / 6.66 / 22.91 | 5.20 / 9.13 / 31.83
 * (scripts/gpu_odometry_streams_adapt.py, profiles/odometry_streams_adapt_h100_700w.json).  An update = 1 tick costs
 * one _train_step at B = S (within 0.06 ms) and saves the streams tick and the weight hand-off: 1.3-1.6 ms at S = 1,
 * 5.3-8.9 ms at S = 16.  An update = 0 tick costs what _streams_push_residual / _streams_push_pre cost. */
int64_t delora_odometry_streams_adapt_workspace_bytes(const delora_odometry_desc* d);   /* host only, -1 if invalid */
int delora_odometry_streams_adapt_init(const delora_odometry_desc* d, const float* weights, void* workspace,
                                       void* stream);
int delora_odometry_streams_push_adapt(const delora_odometry_desc* d, const delora_odometry_train_params* hp, int update,
                                       const float* points, const int32_t* n_points, const int32_t* active,
                                       void* workspace, float* T, int32_t* valid, float* losses, void* stream);
int delora_odometry_streams_adapt_reset(const delora_odometry_desc* d, const int32_t* mask, void* workspace,
                                        void* stream);

/* ---- Dropout masks of the training step (DELORA_TRAIN_DROPOUT), exactly enough to re-implement them elsewhere:
 * Philox4x32-10 (multipliers 0xD2511F53, 0xCD9E8D57; Weyl constants 0x9E3779B9, 0xBB67AE85; curand's philox4x32_10),
 *   key = (low 32 bits of seed, high 32 bits of seed).  Element i of tensor t at step s: counter = (low 32 bits of
 *   i >> 2, t, low 32 bits of s, high 32 bits of s), the word is output word i & 3.  The element is kept iff
 *   (word >> 8) < 13421773, i.e. u < 0.8f with u = (word >> 8) * 2^-24 (0.8f is exactly 13421773 * 2^-24); a kept
 *   value is multiplied by 1.25f (1 / (1 - p), exact in fp32), a dropped one becomes 0.
 * Tensor ids and element indices, per pair b (independent of B and max_batch):
 *   t = 0  input:               ((b * 8 + c) * H + h) * W + w over cat(image_1, image_2) (channels 0..3 image_1)
 *   t = 1  stage-3 channels:    b * C3 + c, C3 = layer3's channel count (256)
 *   t = 2  fc output:           b * resnet_outputs + j
 * delora_odometry_train_set_dropout_seed: store `seed` in the training workspace (launches one kernel, capturable).
 *   Refused before any launch, naming the argument: an invalid descriptor, a null workspace.
 * delora_dropout_keep_mask: keep [n] uint8 (device) = 1 for the kept elements 0 .. n-1 of tensor `tensor` at
 *   (seed, step), else 0, with the device function the step runs.  Refused before any launch, naming the argument:
 *   null keep, n < 0, tensor outside 0..2. */
int delora_odometry_train_set_dropout_seed(const delora_odometry_desc* d, uint64_t seed, void* workspace, void* stream);
int delora_dropout_keep_mask(uint64_t seed, int64_t step, int tensor, int64_t n, uint8_t* keep, void* stream);

/* Training checkpoint (.dlt, written by delora_b200/deploy/export.py and examples/odometry_train.c), little-endian,
 * readable with fread alone:
 *   bytes   0..127  a delora_odometry_file_header (the .dlw layout above) with magic "DELORAT" and header_bytes 256
 *   bytes 128..135  step (int64): Adam updates so far
 *   bytes 136..139  epoch (int32): epochs completed (the reference checkpoint's `epoch` + 1)
 *   bytes 140..143  unsupervised (int32): 0 = still in the identity pre-training phase, 1 = ICP objective
 *   bytes 144..159  lr, beta1, beta2, eps (float32 each): Adam's hyperparameters
 *   bytes 160..163  loss (float32): the mean objective of the last epoch
 *   bytes 164..171  dropout_seed (uint64): the seed of delora_odometry_train_set_dropout_seed (files written before the
 *                   field have zeros there, i.e. seed 0)
 *   bytes 172..255  zero
 *   bytes 256..     float32[blob_floats] weights, then float32[blob_floats] exp_avg, then float32[blob_floats]
 *                   exp_avg_sq, each in blob order (the three arrays of delora_odometry_train_set_state). */
#define DELORA_TRAINING_FILE_MAGIC "DELORAT"     /* 7 characters + NUL = the 8 magic bytes */
typedef struct {
    delora_odometry_file_header base;    /* magic DELORA_TRAINING_FILE_MAGIC, header_bytes 256 */
    int64_t step;
    int32_t epoch;
    int32_t unsupervised;
    float lr, beta1, beta2, eps;
    float loss;
    uint32_t dropout_seed[2];            /* bytes 164..171: the uint64 seed as (low word, high word), which keeps the
                                            struct's layout (a uint64_t member would be aligned to byte 168) */
    uint8_t reserved[84];
} delora_odometry_train_file_header;

/* ---- Data-parallel training step: average of the weight gradients over the ranks (SURVEY.md 8(e); the reference
 * steps one optimizer on one device, src/deploy/trainer.py:23-24, on `loss / batch_size`, src/deploy/deployer.py:329-342
 * -- equal per-rank batches + the mean over ranks reproduce it over the global batch).
 * One all-reduce of elements [offset, offset + count) of a flat fp32 buffer that is SYMMETRIC memory: allocated with
 * the same size on every rank of the node and mapped into every peer (CUDA VMM / torch symmetric memory).
 * peer_bufs[q] / peer_flags[q]: HOST arrays of `world` device addresses -- where rank q's flat buffer / flag words are
 *   mapped in THIS process (index `rank` = the local ones).  Flag words: delora_grad_allreduce_flag_words() uint32,
 *   zeroed once before the first call.
 * multicast_ptr: address of the flat buffer's NVSwitch multicast mapping, or 0 (then peers are read / written one by
 *   one in rank order).  seq: a counter that increases by one with every call, identical on all ranks.
 * scale: applied to the sum (1 / world for the average).  status: device int32, set non-zero if a peer did not arrive
 *   within 20 s (the kernel then carries on; it never hangs).  The kernel needs no shared memory and few registers so
 *   that its n_ctas CTAs are resident NEXT TO the persistent convolution CTAs and the reduction overlaps the backward.
 * n_ctas CTAs (<= 160) of n_threads threads (32 .. 128).
 * Every rank must call it with the same offset / count / seq / n_ctas / n_threads. */
int delora_grad_allreduce_flag_words(void);
int delora_grad_allreduce_f32(const uint64_t* peer_bufs, const uint64_t* peer_flags, uint64_t multicast_ptr, int rank,
                              int world, long long offset, long long count, float scale, uint32_t seq, int n_ctas,
                              int n_threads, int32_t* status, void* stream);

/* ---- Data-parallel training through the C ABI: delora_odometry_train_step on several GPUs, the gradient averaged
 * over the ranks inside the step (the C route of the Python Trainer's bucketed all-reduce, parallel_grad.py).
 *
 * Every rank owns one training workspace (same descriptor, same weights, same Adam state and step count) and calls
 * delora_odometry_train_step_group once per step on its own B pairs.  The step is _train_step with one change: Adam
 * consumes the MEAN over the ranks of the gradient (scale 1 / world on the sum over ranks q = 0 .. world-1 in that
 * order, as BucketedGradAllReduce; every rank ends with bit-identical weights, m and v).  Each rank's objective is its
 * own mean over its B pairs (its quaternion block normalised over its own B), so with equal B on every rank the
 * average reproduces the reference's `loss / batch_size` over the global batch (src/deploy/deployer.py:329-342);
 * unequal B gives an unweighted mean of the ranks' means.  losses, T and pooled stay local to the rank; grads, if
 * non-NULL, receives the averaged gradient.
 *
 * Overlap: the gradient is produced in DELORA_TRAIN_GROUP_BUCKETS buckets, in the backward's order over the blob (the
 * blob is in state_dict order: stem, layer1 .. layer4, fc, heads): [0] heads + fc after the tail backward, [1] layer4
 * after stage 3, [2] layer3, [3] layer2, [4] stem + layer1 after stage 0.  Each bucket is all-reduced
 * (delora_grad_allreduce_f32's kernel, in place in every rank's gradient section) on side_stream as soon as its stage
 * is done, while the next stage's backward runs on `stream`; `stream` joins side_stream before Adam.  Bucket
 * boundaries are stage boundaries rounded UP to a multiple of 4 floats (the kernel moves float4s), so a bucket holds
 * at most 3 floats of the section after it, which the backward produced earlier, and never one it has not produced
 * yet; the last bucket ends at most 3 floats past the blob, inside the gradient section's padding.
 * delora_odometry_train_group_buckets gives the table, delora_odometry_train_grad_offset where the gradient section
 * starts, so a host that brings its own collective (NCCL, MPI) can reproduce the schedule.
 *
 * Sequence numbers come from the device: bucket k of the step that takes the Adam step count to s uses
 * seq = s * DELORA_TRAIN_GROUP_BUCKETS + k, read from the workspace by the kernel, so one captured step replays
 * correctly.  The flag words must be zeroed on every rank before the first group step, must serve no other all-reduce,
 * and must be zeroed again on every rank (with no step in flight) whenever delora_odometry_train_set_state changes the
 * step count, which all ranks must always share.
 *
 * Memory: peer_ws[q] is where rank q's training workspace is mapped in this process (peer_ws[rank] = `workspace`).
 * In one process: device pointers with cudaDeviceEnablePeerAccess both ways (examples/odometry_train.c --gpus N).  In
 * several processes: allocate each workspace with cuMemCreate (a shareable handle type), export and exchange the
 * handles, and cuMemMap + cuMemSetAccess every peer's into each process; a multicast object bound to all workspaces
 * (cuMulticastCreate / cuMulticastBindMem) gives `multicast`, the address of the workspace's multicast mapping.
 * The step allocates nothing and creates no stream or event: side_stream, fork_events and join_event are the
 * caller's (with world == 1 they are not used and may be NULL).  Only launches and event records / waits, so one
 * rank's step can be captured into a CUDA graph on `stream` (side_stream joins the capture through fork_events).
 * With world == 1 the call launches exactly what delora_odometry_train_step launches: the same bits, no collective.
 * Refused before any launch, naming the field: everything _train_step refuses; a null group; world outside
 * [1, DELORA_GRAD_ALLREDUCE_MAX_WORLD], rank outside [0, world); a null or unaligned (16 bytes) peer_ws[q], peer_ws[rank]
 * other than `workspace`, a null or unaligned (4 bytes) peer_flags[q]; an unaligned multicast; a null status; n_ctas
 * outside [1, 160]; n_threads not 32, 64, 96 or 128; with world > 1, a null fork_events[k] or join_event.
 * status: set non-zero by the kernel when a peer did not arrive within 20 s (see delora_grad_allreduce_f32).
 * Measured on one H100 80GB HBM3 at a 700 W power limit (max SM clock 1980 MHz), B = 16, graph-replayed steps,
 * medians of paired differences, world = 1 group step - _train_step: 64 x 720 -0.019 ms (14.26 ms), 64 x 2048
 * -0.000 ms (22.97 ms), i.e. within the noise (scripts/gpu_train_group.py, profiles/train_group_h100_700w.json).
 * Multi-GPU scaling and the all-reduce time left exposed on an 8-GPU NVLink node are not measured yet
 * (scripts/gpu_train_group.py --gpus N measures them). */
#define DELORA_GRAD_ALLREDUCE_MAX_WORLD 16
#define DELORA_TRAIN_GROUP_BUCKETS 5
typedef struct {
    int32_t rank, world;
    uint64_t peer_ws[DELORA_GRAD_ALLREDUCE_MAX_WORLD];     /* rank q's training workspace, mapped in this process */
    uint64_t peer_flags[DELORA_GRAD_ALLREDUCE_MAX_WORLD];  /* rank q's delora_grad_allreduce_flag_words() uint32 */
    uint64_t multicast;                  /* multicast address of the workspaces, or 0 (unicast, rank by rank) */
    int32_t n_ctas, n_threads;           /* the all-reduce kernel's grid: 1 .. 160 CTAs of 32 .. 128 threads */
    int32_t* status;                     /* device int32, 0 while every peer arrives */
    void* side_stream;                   /* cudaStream_t the buckets are all-reduced on */
    void* fork_events[DELORA_TRAIN_GROUP_BUCKETS];  /* cudaEvent_t, recorded on `stream` when bucket k is complete */
    void* join_event;                    /* cudaEvent_t, recorded on side_stream after the last bucket */
} delora_odometry_train_group;
int delora_odometry_train_step_group(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                                     const delora_odometry_train_group* g, const float* points, const int32_t* n_points,
                                     int B, void* workspace, float* losses, float* T, float* pooled, float* grads,
                                     void* stream);
/* Host only (no GPU needed): the byte offset of the gradient section (fp32[weight_floats], blob order) in a training
 * workspace; -1 (and delora_last_error()) for an invalid descriptor. */
int64_t delora_odometry_train_grad_offset(const delora_odometry_desc* d);
/* Host only: the all-reduce schedule of the group step, DELORA_TRAIN_GROUP_BUCKETS entries each, in launch order:
 * bucket k covers gradient floats [offsets[k], offsets[k] + counts[k]) (multiples of 4).  Non-zero for an invalid
 * descriptor or a null output. */
int delora_odometry_train_group_buckets(const delora_odometry_desc* d, int64_t* offsets, int64_t* counts);

/* ---- Adapting streams on several GPUs: one model adapted from the streams every rank serves.  Each rank owns one
 * adapting-streams group workspace (same descriptor, so the same S; a rank with fewer sensors marks the rest inactive;
 * same weights and Adam state) and calls delora_odometry_streams_push_adapt_group once per tick on its own S streams.
 * The update of a tick with update = 1 is one Adam step on the mean over the valid pairs of the WHOLE group, whatever
 * their number on each rank, and every rank ends it with bit-identical weights, m, v and step count.
 *
 * Workspace: the adapting-streams layout of d (delora_odometry_streams_adapt_workspace_bytes(d) bytes, unchanged)
 * followed by a 256-byte group section: a tick counter (int64, the group's update = 1 ticks so far), the fleet-wide
 * count of valid pairs of the last such tick (int32) and the count exchange's slots.  So _streams_adapt_reset,
 * _train_weights, _train_get_state / _set_state and _train_eval work on it unchanged.
 * delora_odometry_streams_adapt_group_init: _streams_adapt_init over the group size; the group section starts at zero.
 * It also loads the collective kernels on the current device: under lazy module loading a kernel's first launch waits
 * for the device's running kernels.  Ranks that share one device and one host thread should also take one
 * _push_adapt tick with update = 1 at the same descriptor first (or run with CUDA_MODULE_LOADING=EAGER), so that no
 * first launch waits behind a rank that spins in the count exchange for a peer not yet enqueued.
 *
 * One tick, update = 1, world > 1 (`g` as for delora_odometry_train_step_group, peer_ws[q] = rank q's group workspace):
 *   1. _push_adapt's stages 1-3: T, valid, the loss rows and the cache write, the same bits.
 *   2. The valid-count exchange on `stream` (collective k = 0): one CTA meets the peers through the flag words and
 *      sums every rank's count in rank order into the fleet-wide count N; the tick counter advances.  On every such
 *      tick, N = 0 included.
 *   3. The tail backward divides by N (so a rank without a valid pair contributes exact zeros), then the trunk
 *      backward, with the DELORA_TRAIN_GROUP_BUCKETS buckets SUMMED over the ranks (scale 1: every rank has already
 *      divided by N) on side_stream as in _train_step_group.
 *   4. `stream` joins side_stream; Adam runs on every rank iff N > 0, and the step count advances iff N > 0.
 * Sequence numbers come from the tick counter: seq = tick * (DELORA_TRAIN_GROUP_BUCKETS + 1) + k, the count exchange
 * k = 0 and the buckets k = 1 .. DELORA_TRAIN_GROUP_BUCKETS, read on the device, so a captured tick replays correctly
 * and a tick without a valid pair still takes new numbers.
 * update = 0 is exactly _push_adapt(update = 0): no collective, the counter stays, so ranks may take different numbers
 * of serve-only ticks between updates.  world = 1 launches exactly what _push_adapt launches: the same bits.
 * Contract: every rank makes the same number of update = 1 calls; the flag words are zeroed on every rank before the
 * first group tick and again after every _adapt_group_init; they serve no other collective (in particular not
 * _train_step_group on the same workspaces).  status: as for _train_step_group (20 s per meet, then carries on).
 * Refused before any launch, naming the field: everything _push_adapt refuses and everything _train_step_group
 * refuses about g.  Out of scope: unequal S per rank, mixed geometries in one tick, dropout or the identity fit while
 * adapting, more than one node, any policy for when to adapt.
 * Measured on one H100 80GB HBM3 at a 700 W power limit (max SM clock 1980 MHz), 64 x 720, w_pre 0, graph-replayed
 * update = 1 ticks, lr 0, medians of paired differences, world = 1 group tick - _push_adapt: -0.002 / -0.003 /
 * -0.021 ms on 3.54 / 4.40 / 14.21 ms ticks at S = 1 / 4 / 16, i.e. within the noise
 * (scripts/gpu_odometry_streams_adapt_group.py, profiles/odometry_streams_adapt_group_h100_700w.json).  The count
 * exchange's cost on a multi-GPU node is not measured yet (the script's --gpus N measures it). */
int64_t delora_odometry_streams_adapt_group_workspace_bytes(const delora_odometry_desc* d);   /* host only */
int delora_odometry_streams_adapt_group_init(const delora_odometry_desc* d, const float* weights, void* workspace,
                                             void* stream);
int delora_odometry_streams_push_adapt_group(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                                             const delora_odometry_train_group* g, int update,
                                             const float* points, const int32_t* n_points, const int32_t* active,
                                             void* workspace, float* T, int32_t* valid, float* losses, void* stream);

/* ---- Adapting streams with the information of each frame's residual: the Gauss-Newton information of the tick's ICP
 * objective at the served T (before the tick's update), beside the losses, so that a fleet adapting its model while it
 * drives can tell when a frame comes from a degenerate scene (see delora_icp_dense_information).
 * Workspace: the group layout of the adapting streams (delora_odometry_streams_adapt_group_workspace_bytes(d) bytes,
 * unchanged) followed by the information section: the rows of the S pairs and delora_icp_information_scratch_floats(S,
 * H, W) floats, each 256-byte aligned.  One workspace serves both pushes below; _streams_adapt_reset, _train_weights,
 * _train_get_state / _set_state and _train_eval work on it unchanged.  delora_odometry_streams_adapt_info_init:
 * _streams_adapt_group_init over this size (the collective kernels preloaded too).
 * delora_odometry_streams_push_adapt_info: the arguments of _push_adapt plus info [S, DELORA_INFO_ROW] (device,
 * required); delora_odometry_streams_push_adapt_group_info: those of _push_adapt_group plus info.  The tick's ICP is
 * the information operator in place of delora_icp_dense_fwd_bwd; its losses and dL/dT are that operator's bits, so T,
 * valid, the loss rows and the updated model (weights, Adam state) are _push_adapt's (_push_adapt_group's) bytes over
 * the same ticks.  Where valid[s] = 1, info[s] is bit for bit the row of the operator run alone at B = 1 on the tick's
 * H x W grids and T's 3x4 in the model's units: delora_icp_dense_information for a plain model,
 * delora_icp_dense_information_scaled with the pair's factor for a DELORA_TRAIN_NORMALIZATION_SCALING one, so H is in
 * the metres and radians of the served T.  Rows with valid[s] = 0 are zeros.  Refused before any launch: what
 * _push_adapt (_push_adapt_group) refuses, and a null info.  The information of the adapting streams of several
 * geometries: delora_odometry_streams_push_adapt_geometries_info below.
 * Measured on one H100 80GB HBM3 at a 700 W power limit (max SM clock 1980 MHz), graph-replayed update = 1 ticks,
 * lr 0, w_pre 0, all streams active, medians of alternating samples, _push_adapt -> _push_adapt_info per tick:
 * 64 x 2048: S = 1 3.73 -> 3.79 ms, S = 4 6.69 -> 6.77 ms, S = 16 23.05 -> 23.19 ms; 64 x 720: S = 1 3.54 -> 3.57 ms,
 * S = 4 4.44 -> 4.48 ms, S = 16 14.23 -> 14.30 ms (scripts/gpu_odometry_streams_pre_adapt_info.py,
 * profiles/odometry_streams_pre_adapt_info_h100_700w.json).  The group push's cost across several GPUs is not
 * measured. */
int64_t delora_odometry_streams_adapt_info_workspace_bytes(const delora_odometry_desc* d);   /* host only */
int delora_odometry_streams_adapt_info_init(const delora_odometry_desc* d, const float* weights, void* workspace,
                                            void* stream);
int delora_odometry_streams_push_adapt_info(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                                            int update, const float* points, const int32_t* n_points,
                                            const int32_t* active, void* workspace, float* T, int32_t* valid,
                                            float* losses, float* info, void* stream);
int delora_odometry_streams_push_adapt_group_info(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                                                  const delora_odometry_train_group* g, int update,
                                                  const float* points, const int32_t* n_points, const int32_t* active,
                                                  void* workspace, float* T, int32_t* valid, float* losses, float* info,
                                                  void* stream);

/* ---- Training on several sensor geometries from one workspace (the reference's `datasets` list,
 * config/deployment_options.yaml:3: its Trainer shuffles over the concatenated datasets, src/deploy/trainer.py:95-101,
 * and each step projects at the geometry of its batch's dataset, src/deploy/deployer.py:240-255).
 *
 * A training workspace has two sections.  The MODEL section comes first: master weights, gradient, Adam's m and v,
 * the counters (Adam's step count, the ICP scratch's batch marker, the dropout seed) and the bf16 filters.  Its layout
 * depends only on act, layers, resnet_outputs, single_mlp and the parity of W (which selects the stem's filter
 * layout).  The GEOMETRY section follows it: frames, grids, ICP scratch, trunk activations, tail buffers and the w_pre
 * buffers.  So descriptors d[0 .. n-1] that agree in those model fields and in W's parity share one model section,
 * and one workspace of the model section plus the largest geometry section serves all of them.  H, W, the fields of
 * view, n_stride, max_batch and w_pre may differ between them.
 *
 * delora_odometry_train_geometries_workspace_bytes: host only; that size, which is the largest
 *   delora_odometry_train_workspace_bytes(&d[g]).  -1 (and delora_last_error()) when the set is refused.
 * delora_odometry_train_geometries_init: _train_init on the shared size, armed for d[0].
 * delora_odometry_train_use_geometry: re-arm the geometry section for d[g] exactly as _train_init arms it (zeros, the
 *   all-ones depth keys, the zeroed ICP scratch with its batch marker).  The model section keeps its weights,
 *   gradient, m, v, step count, dropout seed and bf16 filters.  Launches only (memsets), capturable into a CUDA graph.
 *   Afterwards every training entry point called with &d[g] on the workspace (_train_step, _train_eval,
 *   _train_weights, _train_get_state, _train_set_state, _train_set_dropout_seed, _train_step_group,
 *   _train_grad_offset) acts exactly as on a single-geometry workspace of d[g] holding the same state: the same bits.
 *   Call it whenever the next call's geometry differs from the last one's; the host keeps track of which is armed.
 * Refused before any launch, naming the index and the field: a null d, n < 1, a descriptor _train_workspace_bytes
 * refuses, a model field (act, layers, resnet_outputs, single_mlp) other than d[0]'s, a W of another parity than
 * d[0]'s (a different model-section layout); _use_geometry also refuses g outside [0, n) and a null workspace.
 * Not covered: one step that mixes geometries (the reference cannot either, config/hyperparameters.yaml:3); mixing W
 * parities; inference and streams.  A model trained this way is served per sensor by the inference and streams
 * workspaces from the same .dlw blob, one descriptor per sensor, and adapted from a mixed fleet by
 * delora_odometry_streams_push_adapt_geometries below.
 * Memory, n_stride 131072, max_batch 16: 64 x 2048 with 64 x 720 (w_pre 2250) share 2911 MiB where two
 * single-geometry workspaces take 2911 + 1558 MiB.
 * Cost: the re-arm zeroes d[g]'s whole geometry section, which max_batch sizes, whatever B the next step takes.  So
 * set max_batch to the B you train at.  Measured on one H100 80GB HBM3 at a 700 W power limit, graph-replayed, median
 * paired difference of a step right after a switch against a steady step:
 *   max_batch = B = 1:    64 x 2048 +0.075 ms (3.69 ms step), 64 x 720 (w_pre 2250) +0.044 ms (3.49 ms);
 *   max_batch = B = 16:   64 x 2048 +0.91 ms (23.00 ms), 64 x 720 (w_pre 2250) +0.48 ms (14.53 ms);
 *   max_batch 16, B = 1:  64 x 2048 +0.88 ms (3.71 ms, 24 %), 64 x 720 (w_pre 2250) +0.44 ms (3.51 ms, 13 %).
 * (scripts/gpu_train_geometries.py, profiles/train_geometries_h100_700w.json) */
int64_t delora_odometry_train_geometries_workspace_bytes(const delora_odometry_desc* d, int n);
int delora_odometry_train_geometries_init(const delora_odometry_desc* d, int n, const float* weights, void* workspace,
                                          void* stream);
int delora_odometry_train_use_geometry(const delora_odometry_desc* d, int n, int g, void* workspace, void* stream);

/* ---- Adapting streams of several sensor geometries in one workspace: one model, one call per tick, one Adam step on
 * the mean over every geometry's valid pairs (a fleet that carries, say, a 64 x 720 and a 64 x 512 sensor adapting
 * the model both were trained on through delora_odometry_train_geometries_*).
 *
 * d[0 .. n-1], 1 <= n <= 16: the set delora_odometry_train_geometries_* accepts (the same act, layers,
 * resnet_outputs, single_mlp and W parity), each one a descriptor _push_adapt accepts.  Geometry g serves
 * S_g = d[g].max_batch streams; streams are numbered in geometry order, S_total = S_0 + ... + S_{n-1}, and T
 * [S_total, 16], valid [S_total], losses [S_total, DELORA_LOSS_ROW], active [S_total] (or NULL: all active) and the
 * reset mask [S_total] use that order.  points and n_points are HOST arrays of n device pointers: points[g]
 * [S_g, 3, d[g].n_stride], n_points[g] [S_g].
 *
 * Workspace, each buffer 256-byte aligned:
 *   1. the adapting-streams workspace of d[0], unchanged: the model section, d[0]'s geometry section, its stream
 *      section;
 *   2. for g = 1 .. n-1 in order: d[g]'s training geometry section (at max_batch S_g), its stream section (as
 *      _push_adapt's: the cache, has_prev, the count of valid pairs) and one gradient slice (fp32[weight_floats], blob
 *      order);
 *   3. n > 1 only: a fleet section of 8 + 24 (n - 1) bytes, the count of valid pairs over every geometry (int32) and
 *      each geometry g >= 1's counters (the batch marker of its ICP scratch).
 * So with n = 1 the workspace IS _push_adapt's, and every delora_odometry_train_* call with &d[0] works on it
 * unchanged (_train_weights, _train_get_state / _set_state and the .dlt round trip, _train_grad_offset), as does
 * _push_adapt(&d[0]), which drives geometry 0 alone.  A geometry section cannot be shared: the zero halo rows of the
 * activations sit at other places for another H x W.  Sizes from the host-only query (layers {2,2,2,2},
 * resnet_outputs 1000, two heads, n_stride 131072), 64 x 720 (w_pre 2250) + 64 x 512 (w_pre 512) at S_g = 1 / 4 / 16
 * each: 475.6 / 879.2 / 2493.3 MiB, where two _push_adapt workspaces take 345.4 + 308.8 / 602.0 + 455.6 /
 * 1628.7 + 1043.2 MiB (the second workspace's weights, Adam's m and v and bf16 filters are not repeated; of its
 * 4 x 45.3 MiB fp32 blobs only the gradient slice remains).
 *
 * delora_odometry_streams_adapt_geometries_init: _train_init of d[0] on the whole workspace (every other section
 * zeroed), every geometry's depth keys armed and cached grids emptied.  delora_odometry_streams_adapt_geometries_reset:
 * forget the previous frame of every stream with mask[s] != 0; only launches.
 *
 * delora_odometry_streams_push_adapt_geometries, one tick:
 *   1. For each g: _push_adapt's stages 1-3 of d[g] at B = S_g on its own geometry and stream sections, into rows
 *      S_0 + ... + S_{g-1} onwards: T, valid, the loss rows (the factor in losses[s][6] with
 *      DELORA_TRAIN_NORMALIZATION_SCALING) and the cache write, the bits a _push_adapt workspace of d[g] holding the
 *      same weights writes.  update = 0 stops there (each geometry's ICP batch marker recorded as _push_adapt does).
 *   2. update = 1: one kernel sums the geometries' counts of valid pairs in geometry order into the fleet count N.
 *      Each geometry's backward divides by N (invalid rows add exact zeros); geometry 0 writes the model's gradient
 *      section, geometry g >= 1 its slice.  Adam reads the n gradients, sums them per float in geometry order, writes
 *      the sum to the gradient section (so _train_grad_offset holds the fleet's mean gradient after the tick) and
 *      updates iff N > 0; with N = 0 the step count stays and the weights are not touched.  Then one bf16 re-prep.
 * With n = 1 the tick launches exactly what _push_adapt launches: the same bits.  Only launches, with a sequence that
 * depends on neither `active`, the stream state nor the counts: one captured graph per value of `update` serves every
 * tick.  Refused before any launch, naming the index and the field: n outside [1, 16], every refusal of
 * delora_odometry_train_geometries_*, everything _push_adapt refuses for any d[g] (DELORA_LOSS_IDENTITY_FIT and
 * DELORA_TRAIN_DROPOUT included), a null points / n_points array, a null points[g] or n_points[g], and
 * DELORA_TRAIN_NORMALIZATION_SCALING with any d[g].w_pre = 0.  Out of scope: mixed geometries across GPUs, mixed W
 * parities, dropout or the identity fit while adapting, one trunk launch over unlike image sizes (each geometry's
 * trunk runs at its own B).
 * Cost, measured on one H100 80GB HBM3 at a 700 W power limit (max SM clock 1980 MHz), graph-replayed ticks, all
 * streams active, near-identity heads, lr 0, medians of alternating samples, 64 x 720 (w_pre 2250) + 64 x 512
 * (w_pre 512), ms per tick at S_g = 1 / 4, this call | a _push_adapt tick of each geometry's own workspace:
 *   update = 0: 2.38 / 2.73 | 2.39 / 2.73 (paired difference -0.002 ms);
 *   update = 1: 6.71 / 8.23 | 6.86 / 8.40 (paired difference -0.16 ms: one Adam step and one bf16 re-prep instead of
 *               two, against one extra read of the gradient slice)
 * (scripts/gpu_odometry_streams_adapt_geometries.py, profiles/odometry_streams_adapt_geometries_h100_700w.json). */
int64_t delora_odometry_streams_adapt_geometries_workspace_bytes(const delora_odometry_desc* d, int n);   /* host only */
int delora_odometry_streams_adapt_geometries_init(const delora_odometry_desc* d, int n, const float* weights,
                                                  void* workspace, void* stream);
int delora_odometry_streams_push_adapt_geometries(const delora_odometry_desc* d, int n,
                                                  const delora_odometry_train_params* hp, int update,
                                                  const float* const* points, const int32_t* const* n_points,
                                                  const int32_t* active, void* workspace, float* T, int32_t* valid,
                                                  float* losses, void* stream);
int delora_odometry_streams_adapt_geometries_reset(const delora_odometry_desc* d, int n, const int32_t* mask,
                                                   void* workspace, void* stream);

/* ---- The same adapting streams of several geometries with the information of each frame's residual: the
 * Gauss-Newton information of the tick's ICP objective at the served T, as _push_adapt_info serves it for one geometry.
 *
 * Workspace: the _adapt_geometries workspace of (d, n), unchanged, followed by one information section: the rows of
 * all S_total pairs in fleet stream order, then one info_scratch of max_g delora_icp_information_scratch_floats(S_g,
 * H_g, W_g) floats, each 256-byte aligned.  The geometries' ICPs run one after another on one stream, so they share
 * that scratch.  No other offset moves: delora_odometry_streams_adapt_geometries_init (which leaves the information
 * section as it was: every row is written before it is read, and the scratch needs no initialisation) and _reset,
 * _push_adapt_geometries itself and the delora_odometry_train_* calls listed above work on it unchanged.
 * delora_odometry_streams_adapt_geometries_info_workspace_bytes: host only; -1 (and delora_last_error()) for every set
 * _adapt_geometries_workspace_bytes refuses, with the same message.
 *
 * delora_odometry_streams_push_adapt_geometries_info: the arguments of _push_adapt_geometries plus info [S_total,
 * DELORA_INFO_ROW] (device, required), in fleet stream order.  Each geometry's ICP is the information operator in place
 * of delora_icp_dense_fwd_bwd (delora_icp_dense_information, or delora_icp_dense_information_scaled with the pair's
 * factor for DELORA_TRAIN_NORMALIZATION_SCALING), whose losses and dL/dT are the same bits.  So:
 *   - T, valid, the loss rows and the model after the tick (weights, Adam's m, v and step count, the gradient section)
 *     are _push_adapt_geometries's bytes over the same ticks;
 *   - where valid[s] = 1, info[s] is bit for bit the row a _push_adapt_info workspace of d[g] holding the same weights
 *     writes: the operator's row at B = 1, in the metres and radians of the served T, before the tick's update;
 *   - rows with valid[s] = 0 are zeros;
 *   - with n = 1 every output is _push_adapt_info's bytes.
 * Only launches, with a sequence that depends on neither `active`, the stream state nor the counts: one captured graph
 * per value of `update` serves every tick.  Refused before any launch: everything _push_adapt_geometries refuses, and a
 * null info.  Out of scope: geometries across several GPUs.
 * Cost, measured on one H100 80GB HBM3 at a 700 W power limit (max SM clock 1980 MHz), graph-replayed ticks, all
 * streams active, near-identity heads, lr 0, medians of 7 alternating samples, 64 x 720 (w_pre 2250) + 64 x 512
 * (w_pre 512), _push_adapt_geometries -> _push_adapt_geometries_info per tick:
 *   S_g = 1: update = 0 2.39 -> 2.46 ms (paired difference +0.066 ms), update = 1 6.75 -> 6.82 ms (+0.067 ms);
 *   S_g = 4: update = 0 2.71 -> 2.79 ms (+0.073 ms), update = 1 8.14 -> 8.21 ms (+0.073 ms);
 * the workspace grows by 0.5 / 2.1 MiB (scripts/gpu_odometry_streams_adapt_geometries_info.py,
 * profiles/odometry_streams_adapt_geometries_info_h100_700w.json). */
int64_t delora_odometry_streams_adapt_geometries_info_workspace_bytes(const delora_odometry_desc* d, int n);   /* host only */
int delora_odometry_streams_push_adapt_geometries_info(const delora_odometry_desc* d, int n,
                                                       const delora_odometry_train_params* hp, int update,
                                                       const float* const* points, const int32_t* const* n_points,
                                                       const int32_t* active, void* workspace, float* T, int32_t* valid,
                                                       float* losses, float* info, void* stream);

/* ---- The section map of an odometry workspace: where each buffer the entry points of a workspace kind read or write
 * lies, for tests and tools that check a layout (disjoint sections, which calls write where).  Host only, launches
 * nothing; the layout is the one the kind's entry points plan, built by the same plan functions.
 *
 * kind, and the entry points whose workspace it is:
 *   DELORA_WS_PAIRS                     delora_odometry_init / _load_weights / _pairs / _pairs_normalized / _push
 *   DELORA_WS_STREAMS                   delora_odometry_streams_init / _load_weights / _push / _reset
 *   DELORA_WS_STREAMS_RESIDUAL          _streams_residual_init, _streams_push_residual
 *   DELORA_WS_STREAMS_INFO              _streams_info_init, _streams_push_info
 *   DELORA_WS_STREAMS_NORMALIZED        _streams_normalized_init, _streams_push_normalized
 *   DELORA_WS_STREAMS_PRE               _streams_pre_init, _streams_push_pre (w_pre >= 2)
 *   DELORA_WS_STREAMS_PRE_INFO          _streams_pre_info_init, _streams_push_pre_info (w_pre >= 2)
 *   DELORA_WS_TRAIN                     delora_odometry_train_* of one geometry: _init, _step, _step_group, _eval, the
 *                                       state calls and the dropout seed (w_pre > 0 adds the preprocessing sections)
 *   DELORA_WS_TRAIN_GEOMETRIES          _train_geometries_init, _train_use_geometry and the calls above on geometry g
 *   DELORA_WS_ADAPT                     _streams_adapt_init, _streams_push_adapt, _streams_adapt_reset
 *   DELORA_WS_ADAPT_GROUP               _streams_adapt_group_init, _streams_push_adapt_group
 *   DELORA_WS_ADAPT_INFO                _streams_adapt_info_init, _streams_push_adapt_info, _streams_push_adapt_group_info
 *   DELORA_WS_ADAPT_GEOMETRIES          _streams_adapt_geometries_init / _push_adapt_geometries / _reset
 *   DELORA_WS_ADAPT_GEOMETRIES_INFO     the same and _streams_push_adapt_geometries_info
 * n: the number of descriptors in d; 1 for every kind but the three geometries kinds.
 *
 * Each record: the byte offset and size of one section (the bytes asked for, without the padding to the next 256-byte
 * boundary), its role and name, the geometry whose entry points read it (0 for kinds of one geometry) and flags:
 *   DELORA_WS_SUBRANGE  the section lies inside a larger 256-byte aligned allocation and need not itself be aligned;
 *   DELORA_WS_SHARED    geometries kinds: the model section every geometry reads, listed once per geometry at the
 *                       same offset (its weights, and the information scratch the geometries' ICPs share).
 * Roles: DELORA_WS_WEIGHTS (written only by init, load_weights, set_state and Adam), DELORA_WS_STATE (carried from one
 * call to the next: a stream's cached frame, Adam's moments and step count), DELORA_WS_SCRATCH (written and read
 * within a call), DELORA_WS_OUTPUT (a result the call copies to the caller's arrays, or the gradient section
 * delora_odometry_train_grad_offset names).  Every record but DELORA_WS_TRAIN_GEOMETRIES's lies inside the kind's
 * *_workspace_bytes and no two overlap, the DELORA_WS_SHARED copies aside; DELORA_WS_TRAIN_GEOMETRIES's geometries each
 * have their geometry section over the same bytes (one geometry trains at a time).  No section is empty.  The smaller
 * kind's records appear unchanged in the larger one: STREAMS in RESIDUAL in INFO, TRAIN in ADAPT in ADAPT_GROUP in
 * ADAPT_INFO, ADAPT_GEOMETRIES in ADAPT_GEOMETRIES_INFO.
 *
 * Returns the number of sections, and writes the first min(that, cap) of them to out (out may be NULL with cap = 0);
 * -1 (and delora_last_error()) for a bad kind, n or cap and for every descriptor the kind's *_workspace_bytes
 * refuses. */
#define DELORA_WS_PAIRS                  0
#define DELORA_WS_STREAMS                1
#define DELORA_WS_STREAMS_RESIDUAL       2
#define DELORA_WS_STREAMS_INFO           3
#define DELORA_WS_STREAMS_NORMALIZED     4
#define DELORA_WS_STREAMS_PRE            5
#define DELORA_WS_STREAMS_PRE_INFO       6
#define DELORA_WS_TRAIN                  7
#define DELORA_WS_TRAIN_GEOMETRIES       8
#define DELORA_WS_ADAPT                  9
#define DELORA_WS_ADAPT_GROUP           10
#define DELORA_WS_ADAPT_INFO            11
#define DELORA_WS_ADAPT_GEOMETRIES      12
#define DELORA_WS_ADAPT_GEOMETRIES_INFO 13
#define DELORA_WS_KINDS                 14

#define DELORA_WS_WEIGHTS 0
#define DELORA_WS_STATE   1
#define DELORA_WS_SCRATCH 2
#define DELORA_WS_OUTPUT  3

#define DELORA_WS_SUBRANGE 1
#define DELORA_WS_SHARED   2

typedef struct {
    int64_t offset;
    int64_t bytes;
    int32_t role;
    int32_t geometry;
    int32_t flags;
    char name[44];         /* NUL-terminated, e.g. "cache_pts", "trunk.fwd[3]", "trunk.acts[12]" */
} delora_ws_section;
int delora_odometry_workspace_sections(int kind, const delora_odometry_desc* d, int n, delora_ws_section* out,
                                       int cap);   /* host only */

#ifdef __cplusplus
}
#endif
#endif /* DELORA_B200_H_ */

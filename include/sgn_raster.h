/*
 * sgn_raster.h -- C ABI of libsgn_raster.so, the H100-native (sm_90a) Gaussian rasterizer hot path
 * that replaces the gsplat 0.1.x calls made by street-gaussians-ns.
 *
 * Every entry point below names the reference interface it stands in for (paths relative to
 * /root/reference/street_gaussians_ns/).  gsplat itself is an un-vendored pip dependency of the
 * reference; its semantics are restated in SURVEY.md Appendix A.
 *
 * Conventions
 *   - all data pointers are DEVICE pointers owned by the caller (e.g. torch allocations), fp32 /
 *     int32, row-major contiguous, 16-byte aligned;  `stream` is a cudaStream_t passed as void*.
 *   - structs (sgn_camera, sgn_segment, ...) are plain host structs passed by pointer; segment
 *     tables are staged to a caller-provided device buffer with sgn_upload().
 *   - every function returns 0 on success, a negative sgn_status otherwise; the message is
 *     available from sgn_last_error() (thread local).  No exceptions cross the ABI, no allocation
 *     inside the library: scratch sizes are queried, buffers are passed in.  The only process-wide state is a launch
 *     counter and one lazily created auxiliary stream per device, onto which sgn_blend_fwd / sgn_blend_bwd fork the
 *     object-class pass (event fork / join around it: calls from several host threads on different streams stay
 *     correctly ordered, they merely share that side stream).
 *   - there is NO CPU fallback: a missing device or a failed launch is an error.
 */
#ifndef SGN_RASTER_H_
#define SGN_RASTER_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SGN_ABI_VERSION 2
#define SGN_MAX_FOURIER 8
#define SGN_RECORD_FLOATS 12 /* per-Gaussian projected record, see below */

typedef enum sgn_status {
    SGN_OK = 0,
    SGN_ERR_INVALID = -1,   /* bad argument (shape, alignment, block width ...) */
    SGN_ERR_CUDA = -2,      /* a CUDA runtime call or launch failed */
    SGN_ERR_WORKSPACE = -3, /* scratch buffer too small */
    SGN_ERR_OVERFLOW = -4   /* intersection count exceeds the provided capacity */
} sgn_status;

/* Per-Gaussian projected record (12 floats, 48 B, 16-byte aligned):
 *   [0] x  [1] y            pixel centre            == gsplat project_gaussians `xys`
 *   [2] a  [3] b  [4] c     conic (inverse cov2d)   == `conics`
 *   [5] opacity             sigmoid(logit)          (sgn_splatfacto.py:946-949)
 *                           antialiased mode: sigmoid(logit) * comp
 *                           with a 3D filter (sgn_camera.filter_3d): sigmoid(logit) * coef [* comp]
 *   [6] r  [7] g  [8] b     clamp(SH+0.5, min 0)    (sgn_splatfacto.py:939-940)
 *   [9] depth               view-space z            == `depths`
 *   [10] aux (int bits)     bits 0-2: colour clamp pass mask, bit 3: object class, bit 4: visible
 *   [11] comp               antialiased mode: sqrt(max(0, det(cov2d) / det(cov2d + 0.3 I))) of a visible row (cov2d before
 *                           the blur), 0 otherwise; classic mode: 0
 * xys / conics / depths handed back to Python are strided views of this array. */

/* One visible sub-model of the scene graph for one frame (sgn_splatfacto_scene_graph.py:332-360).
 * Rows [row0, row0+count) of the concatenated index space; concatenation order is the reference's:
 * background first, then actors in annotation order. */
typedef struct sgn_segment {
    int32_t row0;
    int32_t count;
    int32_t F;        /* fourier_features_dim of features_dc (1..8)            (:239-247) */
    int32_t cls;      /* 0 background, 1 object                                 (:364-366) */
    int32_t has_pose; /* apply R,t,q  (object2world_gs, :404-417)                          */
    int32_t chunk0;   /* index of this segment's first 128-row chunk: sum over earlier segments of ceil(count/128) */
    float R[9];       /* object->world rotation, row-major (Box.rot cast to fp32, :411)    */
    float t[3];       /* Box.center cast to fp32 (:410)                                    */
    float q[4];       /* quaternion_from_matrix(rot), wxyz (:413)                          */
    float idft[SGN_MAX_FOURIER]; /* IDFT(t, F) basis (:420-433); [1,0,..] when F == 1      */
    const float* means;         /* [count,3]          gauss_params (sgn_splatfacto.py:291-300) */
    const float* scales;        /* [count,3] log                                            */
    const float* quats;         /* [count,4] wxyz, un-normalised                            */
    const float* features_dc;   /* [count,F,3]                                              */
    const float* features_rest; /* [count,(sh_degree+1)^2-1,3]                              */
    const float* opacities;     /* [count,1] logit                                          */
} sgn_segment;

/* Gradient destinations, one per segment, same shapes as the parameters (dense: rows the
 * rasterizer never touched receive zeros, as autograd of the reference produces). */
typedef struct sgn_segment_grads {
    float* means;
    float* scales;
    float* quats;
    float* features_dc;
    float* features_rest;
    float* opacities;
} sgn_segment_grads;

/* Camera + render settings (sgn_splatfacto.py:822-841, 860-873, 934-938). */
typedef struct sgn_camera {
    float viewmat[12]; /* world->camera 3x4 row-major (viewmat[:3,:], :831-836) */
    float fx, fy, cx, cy;
    int32_t width, height;
    float cam_pos[3];  /* camera_to_worlds[:3,3] for SH view directions (:934) */
    float limx, limy;  /* 1.3*tan(fov/2), float32 as gsplat computes it */
    float clip_thresh; /* 0.01 */
    int32_t block_width;      /* config.block_width; binning semantics (tile AABB) */
    int32_t sh_degree;        /* coefficients stored */
    int32_t sh_degree_to_use; /* min(step//interval, sh_degree) train, sh_degree eval (:936-938) */
    int32_t antialiased;      /* rasterize_mode (sgn_splatfacto.py:214-223): 0 "classic", 1 "antialiased" -- the record's
                                 opacity is scaled by the blur compensation, forward and backward (gsplat's antialiased
                                 mode; the reference leaves the multiply commented out, :946-949) */
    const float* const* filter_3d; /* NULL: off.  Otherwise a DEVICE array of nseg pointers, one per segment of the table the
                                      call is given, each to that segment's count per-row 3D filter sizes sigma (Mip-Splatting's
                                      3D smoothing filter, sgn_filter3d): the projection uses s' = sqrt(s^2 + sigma^2) and scales
                                      the opacity by coef = prod_k sqrt(s_k^2 / (s_k^2 + sigma^2)), forward and backward */
} sgn_camera;

/* Blend settings. */
typedef struct sgn_blend_opts {
    float alpha_clamp_fwd; /* 0.999  gsplat rasterize_forward  */
    float alpha_clamp_bwd; /* 0.99   gsplat rasterize_backward */
    int32_t class_streams; /* also produce objects-only / background-only accumulation
                              (get_submodel_output, sgn_splatfacto_scene_graph.py:364-366) */
    int32_t has_sky;       /* rgb = rgb*alpha + sky*(1-alpha) (sgn_splatfacto.py:971-972) */
    int32_t eval_clamp;    /* not training: rgb.clamp(0,1) (:974-975) */
    /* tuning (0 = default): list length / traversal depth up to which one warp renders a whole tile;
     * each doubling splits the tile into 2/4/8 row strips rendered by independent warps */
    int32_t split_fwd_main, split_fwd_acc, split_bwd_main, split_bwd_acc;
    /* raw mode (gsplat rasterize_gaussians semantics, Level-1 shim): no post-ops; the four blended
     * channels come back as out = sum(c*alpha*T) + T_final*background[c] in rgb[...,0:3] and depth */
    int32_t raw_mode;
    float background[4];
    int32_t tuning; /* SGN_TUNE_* bits: execution variants with identical results up to fp32 rounding */
} sgn_blend_opts;

/* main forward skips row pairs an entry cannot reach / that have fully terminated (exact no-op) */
#define SGN_TUNE_FWD_ROW_SKIP 1
/* paired row-slot (two fp32 pixel rows per instruction pair) slot bodies in the main forward / backward kernels */
#define SGN_TUNE_FWD_PACKED 4
#define SGN_TUNE_BWD_PACKED 8
/* the accumulation-only (object / background) kernels do NOT skip unreachable row pairs */
#define SGN_TUNE_ACC_NO_ROW_SKIP 16
/* experiment: the main forward reads its lists as materialised 48-byte staged entries moved by cp.async.bulk + mbarrier
 * (sgn_blend_fwd_out.staged must then point to 48 * M bytes of scratch) instead of gathering records per lane */
#define SGN_TUNE_FWD_TMA 32

const char* sgn_last_error(void);
int sgn_abi_version(void);
/* number of kernel launches this library has issued in this process (a CUB device-wide call counts as 1) */
long long sgn_launch_count(void);
size_t sgn_sizeof_segment(void);
size_t sgn_sizeof_segment_grads(void);
size_t sgn_sizeof_camera(void);

/* Async H2D copy of a small host table (segment / grads table) into caller-provided device memory. */
int sgn_upload(const void* host, size_t bytes, void* dev, void* stream);

/* ---- fused compose + project + SH + sigmoid -------------------------------------------------
 * Replaces, in ONE launch over all segments: get_fourier_features + object2world_gs + the six
 * torch.cat (sgn_splatfacto_scene_graph.py:332-360), exp(scales) / cat(dc,rest) / quat normalise
 * (sgn_splatfacto.py:857-858,864), gsplat project_gaussians (:860-873), view directions +
 * spherical_harmonics + clamp (:934-940) and sigmoid(opacities) (:946-949).
 * Outputs: records[N,12] (layout above), radii[N] i32, num_tiles_hit[N] i32, tile_bbox[N] (4 x u16:
 * xmin,ymin,xmax,ymax in tiles), tiles_touched[N] i32 = number of AABB tiles the Gaussian can really
 * reach (exact test, see sgn_bin_count), touch_mask[N] u32 = one bit per AABB tile when the AABB has at
 * most 32 tiles.  Work is split into 128-row chunks that never straddle segments:
 * num_chunks = sum over segments of ceil(count/128), sgn_segment.chunk0 = the segment's first chunk.
 * cam->antialiased: record [5] is sigmoid(logit) * comp and [11] is comp (layout above), and the touch test uses that
 * opacity, tau = ln(255 o comp), so a row with comp == 0 reaches no tile.  The backward (every form below, with the same
 * camera) then sends the opacity cotangent to the logit as v * comp * s (1 - s) and, through comp, to cov2d and from
 * there to means, scales, quats and the pose / view partials.
 * cam->filter_3d (non-NULL): every row i of segment k is projected with the scales s' = sqrt(s^2 + sigma^2), sigma =
 * cam->filter_3d[k][i], and its opacity is multiplied by coef = prod_k sqrt(r_k), r_k = s_k^2 / (s_k^2 + sigma^2) (then by comp
 * in the antialiased mode, computed from the filtered covariance).  sigma is a constant: the backward sends the scales' cotangent
 * through d log s' / d log s = r and d coef / d log s_k = coef (1 - r_k), with coef recomputed from the parameters and sigma, and
 * the opacity cotangent to the logit as v * coef [* comp] * s (1 - s).  NULL: the outputs are those of a camera without the field. */
int sgn_project_fwd(const sgn_segment* segs_dev, int nseg, int N, int num_chunks, const sgn_camera* cam,
                    float* records, int32_t* radii, int32_t* num_tiles_hit, uint16_t* tile_bbox,
                    int32_t* tiles_touched, uint32_t* touch_mask, void* stream);

/* Backward of the above.  v_records[N,12] holds the per-Gaussian cotangents in record layout
 * ([0:2] v_xy, [2:5] v_conic, [5] v_opacity, [6:9] v_rgb, [9] v_depth), as accumulated by
 * sgn_blend_bwd.  Writes dense parameter gradients for every segment.
 * Replaces gsplat project_gaussians backward + compute_sh_backward + autograd of the glue. */
int sgn_project_bwd(const sgn_segment* segs_dev, const sgn_segment_grads* grads_dev, int nseg, int N, int num_chunks,
                    const sgn_camera* cam, const float* records, const int32_t* radii,
                    const float* v_records, void* stream);
/* The same backward over the chunks [chunk_begin, chunk_end) only (rows of the concatenated row space in 128-row chunks):
 * the data-parallel step produces the gradient arena range by range so that the exchange of a finished range
 * (sgn_allreduce_sym) overlaps the production of the next one. */
int sgn_project_bwd_range(const sgn_segment* segs_dev, const sgn_segment_grads* grads_dev, int nseg, int N, int num_chunks,
                          const sgn_camera* cam, const float* records, const int32_t* radii, const float* v_records,
                          int chunk_begin, int chunk_end, void* stream);

/* The range backward that ALSO yields the cotangents of the segments' object->world poses: every 128-row chunk of a
 * segment with has_pose stores the sums over its rows of (v_R[9] row-major, v_t[3], v_q[4]) -- means_w = R m + t gives
 * v_t = sum vmw and v_R[r][c] = sum vmw[r] m[c]; q_w = q_box (x) q gives v_q = sum vqr (x) conj(q), q un-normalised -- to
 * pose_partials[num_chunks, SGN_POSE_FLOATS] (chunks of other segments are not written).  The parameter gradients are
 * bit-identical to sgn_project_bwd_range's.  sgn_pose_grad_reduce, called after the last range, sums a segment's chunks
 * into v_pose[nseg, SGN_POSE_FLOATS] (zero rows for segments without a pose).  Neither stage uses atomics: v_pose is the
 * same bits on every run over the same v_records. */
#define SGN_POSE_FLOATS 16
int sgn_project_bwd_pose(const sgn_segment* segs_dev, const sgn_segment_grads* grads_dev, int nseg, int N, int num_chunks,
                         const sgn_camera* cam, const float* records, const int32_t* radii, const float* v_records,
                         int chunk_begin, int chunk_end, float* pose_partials, void* stream);
int sgn_pose_grad_reduce(const sgn_segment* segs_dev, int nseg, int num_chunks, const float* pose_partials, float* v_pose,
                         void* stream);

/* ---- the view on the device (camera pose optimisation) ------------------------------------------------------------------
 * `view` is a DEVICE array of SGN_VIEW_FLOATS + 3 floats: viewmat[12] (world->camera 3x4, row-major), then cam_pos[3]; it
 * replaces cam->viewmat / cam->cam_pos (every other field of `cam` is used as given).  A view computed on the device --
 * sgn_camera_adjust_fwd -- thus reaches the projection without a host read-back.
 * sgn_project_fwd_view: sgn_project_fwd (its direct form) with that view; with the camera's own view the outputs are the
 * same bits.  sgn_project_bwd_view: sgn_project_bwd_range with that view that also stores, per 128-row chunk of
 * [chunk_begin, chunk_end), the sums over its rows of the cotangent of viewmat[12] (v_W = sum v_pc p_w^T + 2 G W S_w,
 * v_c = sum v_pc; p_c = W p_w + c and S_c = W S_w W^T the camera-space mean and covariance, v_pc and G their cotangents) to
 * view_partials[num_chunks, SGN_VIEW_FLOATS]; cam_pos only orients the SH colour, whose view direction is treated as
 * constant, so it gets no cotangent.  With pose_partials non-NULL it also yields the pose sums of sgn_project_bwd_pose.
 * The parameter gradients are bit-identical to sgn_project_bwd_range's.  sgn_view_grad_reduce, after the last range,
 * sums all chunks into v_view[SGN_VIEW_FLOATS] in a fixed order: no atomics, the same bits on every run. */
#define SGN_VIEW_FLOATS 12
int sgn_project_fwd_view(const sgn_segment* segs_dev, int nseg, int N, int num_chunks, const sgn_camera* cam, const float* view,
                         float* records, int32_t* radii, int32_t* num_tiles_hit, uint16_t* tile_bbox, int32_t* tiles_touched,
                         uint32_t* touch_mask, void* stream);
int sgn_project_bwd_view(const sgn_segment* segs_dev, const sgn_segment_grads* grads_dev, int nseg, int N, int num_chunks,
                         const sgn_camera* cam, const float* view, const float* records, const int32_t* radii,
                         const float* v_records, int chunk_begin, int chunk_end, float* pose_partials /* or NULL */,
                         float* view_partials, void* stream);
int sgn_view_grad_reduce(int num_chunks, const float* view_partials, float* v_view, void* stream);

/* nerfstudio's CameraOptimizer, mode "SO3xR3" (cameras/camera_optimizers.py, lie_groups.py), one launch each way.
 * pose_adjustment: device, float32 [num_cameras, 6] (translation 0:3, axis-angle 3:6).
 * Forward: reg[1] (device) = mean_rows |x[:, 0:3]| w_t + mean_rows |x[:, 3:6]| w_r (the regulariser), norms[2] (device) =
 * {|x[:, 0:3]|, |x[:, 3:6]|} (Frobenius norms); sums in a fixed order.  With cam_idx >= 0 also the corrected view of that camera:
 * x = pose_adjustment[cam_idx], theta = sqrt(max(|w|^2, 1e-4)), R_a = I + sin(theta)/theta K + (1 - cos(theta))/theta^2 K^2
 * (K = skew(w)), t_a = x[0:3];  c2w' = c2w [R_a t_a; 0 1];  view = (viewmat of c2w' as Camera._viewmat builds it, then
 * cam_pos = c2w'[:3, 3]), float32.  c2w: 12 HOST floats (3x4 row-major), ignored (may be NULL) when cam_idx == -1.
 * Backward: writes EVERY row of v_pose_adjustment: the regulariser's gradient for the cotangent g_reg[0] (device scalar; a
 * row with a zero norm gets zero from that norm, as torch gives) plus, in row cam_idx, the chain from v_view[SGN_VIEW_FLOATS]
 * (cam_pos has no cotangent, see above).  g_reg / v_view NULL: that share is zero. */
int sgn_camera_adjust_fwd(const float* pose_adjustment, int num_cameras, int cam_idx, const float* c2w, float w_t, float w_r,
                          float* view, float* reg, float* norms, void* stream);
int sgn_camera_adjust_bwd(const float* pose_adjustment, int num_cameras, int cam_idx, const float* c2w, float w_t, float w_r,
                          const float* v_view, const float* g_reg, float* v_pose_adjustment, void* stream);

/* ---- Level-1: gsplat 0.1.x function API on plain tensors (sgn_splatfacto.py:11-14) -------------------
 * gsplat.project_gaussians(means3d, scales, glob_scale, quats, viewmat, fx, fy, cx, cy, H, W, block_width,
 * clip_thresh) -> xys[N,2], depths[N], radii[N] i32, conics[N,3], compensation[N], num_tiles_hit[N] i32,
 * cov3d[N,6]   (call site sgn_splatfacto.py:860-873), and its backward (cotangent pointers may be NULL). */
int sgn_l1_project_fwd(int N, const float* means, const float* scales, float glob_scale, const float* quats,
                       const sgn_camera* cam, float* xys, float* depths, int32_t* radii, float* conics,
                       float* compensation, int32_t* num_tiles_hit, float* cov3d, void* stream);
int sgn_l1_project_bwd(int N, const float* means, const float* scales, float glob_scale, const float* quats,
                       const sgn_camera* cam, const int32_t* radii, const float* v_xys, const float* v_depths,
                       const float* v_conics, float* v_means, float* v_scales, float* v_quats, void* stream);
/* The same backward with a cotangent of `compensation` too (v_compensation may be NULL: then the outputs are
 * sgn_l1_project_bwd's).  comp = sqrt(max(0, det(cov2d) / det(cov2d + 0.3 I))) reaches means, scales and quats through
 * cov2d; a row whose comp is 0 (the clamp) passes no cotangent through it. */
int sgn_l1_project_bwd_comp(int N, const float* means, const float* scales, float glob_scale, const float* quats,
                            const sgn_camera* cam, const int32_t* radii, const float* v_xys, const float* v_depths,
                            const float* v_conics, const float* v_compensation, float* v_means, float* v_scales,
                            float* v_quats, void* stream);
/* gsplat.spherical_harmonics(degrees_to_use, viewdirs[N,3], coeffs[N,K,3]) (call site :939): forward when
 * `colors` is non-NULL, backward (v_coeffs = Y_k * v_colors) when `v_coeffs` is non-NULL. */
int sgn_l1_sh(int N, int K, int degree, const float* viewdirs, const float* coeffs, const float* v_colors,
              float* colors, float* v_coeffs, void* stream);

/* ---- binning: cumulative intersects, key emit, radix sort, tile bin edges ---------------------
 * Replaces the inside of gsplat rasterize_gaussians: compute_cumulative_intersects,
 * map_gaussian_to_intersects, torch.sort, get_tile_bin_edges (SURVEY.md 3.3 / Appendix A.5). */
/* step 0 (only when the records do not come from sgn_project_fwd, e.g. the Level-1 rasterize path):
 * per-Gaussian count of the AABB tiles it can actually reach.  Exact, conservative ellipse-vs-tile test:
 * a tile where no pixel centre can have alpha >= 1/255 is a no-op for every stream and is dropped;
 * gsplat's num_tiles_hit is NOT changed. */
int sgn_bin_count(int N, const sgn_camera* cam, const float* records, const int32_t* radii,
                  const uint16_t* tile_bbox, int32_t* tiles_touched, uint32_t* touch_mask, void* stream);
/* step 1: stable depth order of the N rows (invisible rows last) and the inclusive scan of tiles_touched IN THAT
 * ORDER (cum[rank]); order[rank] = the entry payload of the row at that depth rank (row | object class << 31, the
 * sorted_ids layout below), so the run of entries of rank r is [cum[r-1], cum[r]) with that payload; the total M is
 * also written to *total_dev (int64). */
size_t sgn_bin_scan_scratch_bytes(int N);
int sgn_bin_scan(int N, const float* records, const int32_t* radii, const int32_t* tiles_touched,
                 int32_t* order, int32_t* cum, int64_t* total_dev, void* scratch, size_t scratch_bytes, void* stream);
/* step 2: emit (in depth order) + stable sort by tile id + bin edges for M = total intersections. */
size_t sgn_bin_sort_scratch_bytes(int64_t M);
int sgn_bin_sort(int N, int64_t M, const sgn_camera* cam, const float* records, const int32_t* radii,
                 const uint16_t* tile_bbox, const uint32_t* touch_mask, const int32_t* order, const int32_t* cum,
                 int32_t* sorted_ids /*[M]*/, int32_t* tile_bins /*[tiles,2]*/, void* scratch, size_t scratch_bytes,
                 void* stream);
/* The same step without the host knowing M: `capacity` bounds the buffers (sorted_ids[capacity], scratch of
 * sgn_bin_sort_scratch_bytes(capacity)) and the launches, the real count is read from *total_dev on the device.  gsplat reads
 * the count back every frame (`cum_tiles_hit[-1].item()`); without that read-back the host can run ahead of the GPU.  Unused
 * slots are padded with a key behind every tile (the sort runs over `capacity` items).  If *total_dev > capacity the lists
 * are truncated and *overflow_dev is set to 1 (never cleared here): the caller checks it later and grows the capacity. */
int sgn_bin_sort_capped(int N, int64_t capacity, const int64_t* total_dev, int32_t* overflow_dev, const sgn_camera* cam,
                        const float* records, const int32_t* radii, const uint16_t* tile_bbox, const uint32_t* touch_mask,
                        const int32_t* order, const int32_t* cum, int32_t* sorted_ids, int32_t* tile_bins, void* scratch,
                        size_t scratch_bytes, void* stream);
/* EXPERIMENTAL alternative to steps 1 + 2 (csrc/binning_local.cu; same lists, same order, same payload): tile histogram +
 * unordered scatter + a shared-memory sort inside every tile instead of the two device-wide radix sorts.
 *   sgn_bin_local_count: tile_count[tiles], tile_start[tiles] (exclusive scan), info_dev = {M, longest list} (int64[2]);
 *   the caller reads info_dev, and when the longest list exceeds sgn_bin_local_cap() uses steps 1 + 2 for this frame;
 *   sgn_bin_local_sort: sorted_ids[M], tile_bins[tiles,2].  Scratch: sgn_bin_local_scratch_bytes(M, tiles) (M = 0 for count). */
int sgn_bin_local_cap(void);
size_t sgn_bin_local_scratch_bytes(int64_t M, int tiles);
int sgn_bin_local_count(int N, const sgn_camera* cam, const float* records, const int32_t* radii, const uint16_t* tile_bbox,
                        const uint32_t* touch_mask, int32_t* tile_count, int32_t* tile_start, int64_t* info_dev, void* scratch,
                        size_t scratch_bytes, void* stream);
int sgn_bin_local_sort(int N, int64_t M, int longest_list, const sgn_camera* cam, const float* records, const int32_t* radii,
                       const uint16_t* tile_bbox, const uint32_t* touch_mask, const int32_t* tile_count, const int32_t* tile_start,
                       int32_t* sorted_ids, int32_t* tile_bins, int32_t* cls_ids /*[2,M] or NULL*/,
                       int32_t* cls_bins /*[2,tiles,2] or NULL: the class sub-lists of step 3, built in the same pass*/,
                       void* scratch, size_t scratch_bytes, void* stream);
/* sorted_ids payload: bits 0-30 = Gaussian row (concatenated index space), bit 31 = object class.
 * step 3 (only for the class renders): per-tile class sub-lists, a stable partition of every tile's
 * list into background entries (class 0) and object entries (class 1) -- what the reference's
 * objects-only / background-only re-renders sort and traverse (sgn_splatfacto_scene_graph.py:
 * 255-303,364-366).  cls_ids is [2,M] (class c at cls_ids + c*M), cls_bins is [2,tiles,2]. */
size_t sgn_bin_class_scratch_bytes(int tiles);
int sgn_bin_class_lists(const sgn_camera* cam, int64_t M, const int32_t* sorted_ids, const int32_t* tile_bins,
                        int32_t* cls_ids, int32_t* cls_bins, void* scratch, size_t scratch_bytes, void* stream);

/* ---- alpha blending ------------------------------------------------------------------------------
 * Forward: gsplat rasterize_forward for rgb AND the depth pass in one traversal
 * (sgn_splatfacto.py:954-996), optionally the two accumulation-only re-renders
 * (sgn_splatfacto_scene_graph.py:364-366), with the reference's post-ops fused in the epilogue
 * (:968-975, :995).  Saves raw[H,W,4] (premultiplied rgb + depth), final_T / final_idx per stream. */
typedef struct sgn_blend_fwd_out {
    float* rgb;            /* [H,W,3] final */
    float* accumulation;   /* [H,W]   1 - T */
    float* depth;          /* [H,W]   where(alpha>1e-3, d/alpha, 10) */
    float* object_acc;     /* [H,W] or NULL */
    float* background_acc; /* [H,W] or NULL */
    float* raw;            /* [H,W,4] saved for backward */
    float* final_T;        /* [3,H,W] planar: slot 0 main, 1 object, 2 background */
    int32_t* final_idx;    /* [3,H,W] */
    int32_t* tile_depth;   /* [3,tiles] entries traversed per tile: main; object entries walked past the main traversal;
                              background pass.  Sizes the backward */
    int32_t* sched;        /* scratch of sgn_blend_sched_ints(tiles) int32, or NULL: heavy-first work lists (longest tile
                              lists are scheduled first; without it CTAs take the tiles in raster order) */
    float* staged;         /* scratch of 12 * M floats (16-byte aligned) for SGN_TUNE_FWD_TMA, or NULL */
} sgn_blend_fwd_out;

size_t sgn_blend_sched_ints(int tiles);
int sgn_blend_fwd(const sgn_camera* cam, const sgn_blend_opts* opts, const float* records,
                  const int32_t* sorted_ids, const int32_t* tile_bins, int64_t M,
                  const int32_t* cls_ids /*[2,M] or NULL*/, const int32_t* cls_bins /*[2,tiles,2] or NULL*/,
                  const float* sky /*[H,W,3] or NULL*/, const sgn_blend_fwd_out* out, void* stream);

typedef struct sgn_blend_bwd_in {
    const float* v_rgb;            /* [H,W,3] or NULL */
    const float* v_accumulation;   /* [H,W]   or NULL */
    const float* v_depth;          /* [H,W]   or NULL */
    const float* v_object_acc;     /* [H,W]   or NULL */
    const float* v_background_acc; /* [H,W]   or NULL */
    const float* raw;
    const float* final_T;
    const int32_t* final_idx;
    const int32_t* tile_depth;     /* [3,tiles] from the forward */
    int32_t* sched;                /* scratch of sgn_blend_sched_ints(tiles) int32 (may be the forward's), or NULL */
    const float* sky;              /* [H,W,3] or NULL */
    float* v_sky;                  /* [H,W,3] or NULL: gradient to the sky colour */
    /* Deterministic mode (NULL = off): the per-Gaussian gradients are accumulated in 64-bit fixed point (one rounding per
     * addend, integer adds: bit-identical totals whatever the execution order) instead of with float atomics, then written
     * to v_records.  v_fixed: [num_gaussians,12] int64, ZERO on entry; fixed_scale: one float of device scratch. */
    int64_t* v_fixed;
    float* fixed_scale;
    int64_t num_gaussians;
} sgn_blend_bwd_in;

/* Backward: gsplat rasterize_backward for all streams in one traversal.  v_records[N,12] must be
 * zero on entry; it is accumulated into (record layout, see sgn_project_bwd). */
int sgn_blend_bwd(const sgn_camera* cam, const sgn_blend_opts* opts, const float* records,
                  const int32_t* sorted_ids, const int32_t* tile_bins, int64_t M,
                  const int32_t* cls_ids /*[2,M] or NULL*/, const int32_t* cls_bins /*[2,tiles,2] or NULL*/,
                  const sgn_blend_bwd_in* in, float* v_records, void* stream);

/* Generic per-Gaussian channels (the north-star's per-Gaussian semantic logits; the reference's dormant consumer:
 * scripts/render.py:188,231-236): extra[N,C] is composited with the weights of the main render -- out[p,c] = sum_k
 * extra[k,c] alpha_k T_k over the entries the main pass blended (final_T / final_idx slot 0 of sgn_blend_fwd) -- 8 channels per
 * traversal.  What the reference would obtain from one more gsplat rasterize_gaussians(colors = logits) call.  The backward
 * ACCUMULATES into v_extra[N,C] (zero it first) and into v_records[N,12] (geometry part: call it between sgn_blend_bwd and
 * sgn_project_bwd). */
int sgn_blend_extra_fwd(const sgn_camera* cam, const sgn_blend_opts* opts, const float* records, const int32_t* sorted_ids,
                        const int32_t* tile_bins, const float* final_T, const int32_t* final_idx, const float* extra, int C,
                        float* out /*[H,W,C]*/, void* stream);
int sgn_blend_extra_bwd(const sgn_camera* cam, const sgn_blend_opts* opts, const float* records, const int32_t* sorted_ids,
                        const int32_t* tile_bins, const float* final_T, const int32_t* final_idx, const float* extra, int C,
                        const float* v_out /*[H,W,C]*/, float* v_extra /*[N,C]*/, float* v_records /*[N,12]*/, void* stream);
/* Deterministic form of sgn_blend_extra_bwd (the extra channels under sgn_blend_bwd_in.v_fixed): the per-Gaussian sums are
 * accumulated in 64-bit fixed point (one rounding per addend, integer adds: bit-identical totals whatever the execution
 * order), converted, and then ADDED to v_extra and to the geometry part of v_records, as the float form adds.
 * fixed_geom [num_gaussians,6] and fixed_extra [num_gaussians,C] int64, ZERO on entry; fixed_scale: two floats of device
 * scratch. */
int sgn_blend_extra_bwd_det(const sgn_camera* cam, const sgn_blend_opts* opts, const float* records, const int32_t* sorted_ids,
                            const int32_t* tile_bins, const float* final_T, const int32_t* final_idx, const float* extra, int C,
                            int64_t num_gaussians, const float* v_out /*[H,W,C]*/, float* v_extra /*[N,C]*/,
                            float* v_records /*[N,12]*/, int64_t* fixed_geom, int64_t* fixed_extra, float* fixed_scale,
                            void* stream);

/* ---- loss epilogue (SURVEY.md 8f rank 2) ------------------------------------------------------------------
 * The image-space loss terms of the reference that re-read the rasterizer's outputs right after the render, and
 * their cotangents: L1 = w_l1 * mean|gt - rgb| (sgn_splatfacto.py:1079-1084; with mask: both sides times mask,
 * :1073-1076), sky = w_sky * mean(sky_mask * accumulation) (:1090-1093), entropy = w_entropy * mean(-(oa log oa +
 * (1-oa) log(1-oa))) with oa = clamp(object_acc, 1e-5, 1-1e-5) (sgn_splatfacto_scene_graph.py:386-389).
 * A term whose inputs are NULL is 0 / gets no cotangent.  gt is the float image or the uint8 one (gt = u8 / 255). */
typedef struct sgn_loss_in {
    const float* rgb;           /* [H,W,3] or NULL */
    const uint8_t* gt_u8;       /* [H,W,3] exactly one of gt_u8 / gt_f32 when rgb is given */
    const float* gt_f32;
    const float* mask;          /* [H,W,1] or NULL */
    const float* accumulation;  /* [H,W,1] or NULL */
    const uint8_t* sky_mask;    /* [H,W] 1 = sky (semantic == SKY) or NULL */
    const float* object_acc;    /* [H,W,1] or NULL */
    float w_l1, w_sky, w_entropy;
} sgn_loss_in;
size_t sgn_loss_scratch_bytes(void);
/* losses[3] (device) = {L1, sky, entropy} terms, already weighted */
int sgn_loss_fwd(int H, int W, const sgn_loss_in* in, float* losses, void* scratch, size_t scratch_bytes, void* stream);
/* cotangents of the outputs for incoming gradients grad_losses[3] (device scalars; NULL = all ones); each output may be NULL */
int sgn_loss_bwd(int H, int W, const sgn_loss_in* in, const float* grad_losses, float* v_rgb, float* v_accumulation,
                 float* v_object_acc, void* stream);

/* SSIM term (sgn_splatfacto.py:1085-1087): weight * (1 - SSIM(gt*mask, rgb*mask)) with pytorch_msssim.SSIM(data_range=1,
 * size_average=True, channel=3): 11-tap Gaussian window (sigma 1.5), valid padding, mean of the (H-10) x (W-10) x 3 map.
 * The forward stores three derivative maps (36 B per valid pixel) in the caller's workspace for the backward.  H or W < 11,
 * a null rgb / gt, both gt pointers, or a short workspace return an error and launch nothing. */
size_t sgn_ssim_workspace_bytes(int H, int W);
/* *loss (device) = weight * (1 - SSIM(gt*mask, rgb*mask)); uses in->rgb, in->gt_u8 | in->gt_f32, in->mask only */
int sgn_ssim_fwd(int H, int W, const sgn_loss_in* in, float weight, float* loss, void* workspace, size_t workspace_bytes, void* stream);
/* v_rgb [H,W,3] = d(grad_loss * loss)/d rgb, from the workspace sgn_ssim_fwd filled (grad_loss: device scalar; NULL = 1) */
int sgn_ssim_bwd(int H, int W, const sgn_loss_in* in, float weight, const float* grad_loss, const void* workspace, float* v_rgb,
                 void* stream);

/* ---- per-step metrics (get_metrics_dict, sgn_splatfacto.py:1015-1040; eval psnr of :1109-1187) ---------------
 * One HBM-bound pass over the image and the frame's parameters, through the device segment table of sgn_project_fwd (no copy):
 *   out[0] psnr            = 10 log10(1 / mean((gt*mask - rgb*mask)^2)) over H*W*3 (torchmetrics PeakSignalNoiseRatio,
 *                            data_range 1); +inf for equal images.  Uses image->rgb, image->gt_u8 | image->gt_f32, image->mask;
 *                            image == NULL or image->rgb == NULL: no psnr (NaN).
 *   out[1] scale_mean      = mean(exp(scales)) over the N rows of the table x 3
 *   out[2] log_scale_mean  = mean(scales)
 *   out[3] sigmoid_opacity = mean(sigmoid(opacities))   (table_dev == NULL: out[1..3] are NaN)
 *   out[4] radii_mean      = mean(radii[0..N))          (radii == NULL: NaN)
 * Sums in fp64 in a fixed order (bit-identical run to run), results rounded once to fp32; means over zero rows are NaN.  No
 * host synchronisation.  A null table with nseg > 0, both or neither gt pointer with rgb, a null out / scratch (SGN_ERR_INVALID)
 * or a short scratch (SGN_ERR_WORKSPACE) launch nothing. */
size_t sgn_metrics_scratch_bytes(void);
int sgn_metrics(int H, int W, const sgn_loss_in* image, const sgn_segment* table_dev, int nseg, int N, int num_chunks,
                const int32_t* radii, float* out, void* scratch, size_t scratch_bytes, void* stream);

/* ---- sky cube map (EnvLight, sgn_splatfacto.py:109-150; use_sky_sphere = True) ------------------------------
 * nvdiffrast dr.texture(tex[None], l, filter_mode='linear', boundary_mode='cube') on a learnable [6,R,R,3] map, and its
 * gradient for the map (the gradient for the directions: the _uv / _rot entry points below).  The camera path generates the reference's per-pixel world
 * directions itself: d = normalize(((x - cx + ju) / fx, (y - cy + jv) / fy, 1)), rotated by c2w[:3,:3] (recovered from
 * cam->viewmat), then l = (d.x, d.z, -d.y); ju = jv = 0.5 in eval (jitter pointers NULL), two [H,W] uniform draws in
 * training.  The backward recomputes the directions from the same jitter.  v_tex is ACCUMULATED into (zero it first); it
 * uses float atomics, so it is not bit-reproducible (the _det entry points below are).  R < 1, a null required pointer, a
 * single jitter array or sizes beyond 32-bit indexing return SGN_ERR_INVALID and launch nothing. */
/* sky[H,W,3]; dirs[H,W,3] (the lookup directions l) or NULL */
int sgn_sky_fwd(const sgn_camera* cam, const float* jitter_u, const float* jitter_v, const float* tex, int R, float* sky, float* dirs,
                void* stream);
int sgn_sky_bwd(const sgn_camera* cam, const float* jitter_u, const float* jitter_v, int R, const float* v_sky, float* v_tex,
                void* stream);
/* The same sampler on given directions uv[P,3]: out[P,3]; backward accumulates into v_tex. */
int sgn_cube_texture_fwd(int P, const float* uv, const float* tex, int R, float* out, void* stream);
int sgn_cube_texture_bwd(int P, const float* uv, int R, const float* v_out, float* v_tex, void* stream);
/* Deterministic backward: the same arguments and the same accumulation into v_tex, bit-identical from run to run and
 * whatever the order of the lookups.  Every addend is rounded once to 64-bit fixed point (2^32 units per unit of
 * max|v_out|, a power of two) and added as an integer; the sums are then converted and added to v_tex.  scratch: at least
 * sgn_sky_det_scratch_bytes(R) bytes of device memory, 8-byte aligned (int64 [6,R,R,3] and the grid scale); the library
 * zeroes it on the stream itself.  A null, misaligned or too small scratch returns SGN_ERR_INVALID and launches nothing. */
size_t sgn_sky_det_scratch_bytes(int R); /* 0 for an invalid R */
int sgn_sky_bwd_det(const sgn_camera* cam, const float* jitter_u, const float* jitter_v, int R, const float* v_sky, float* v_tex,
                    void* scratch, size_t scratch_bytes, void* stream);
int sgn_cube_texture_bwd_det(int P, const float* uv, int R, const float* v_out, float* v_tex, void* scratch, size_t scratch_bytes,
                             void* stream);
/* The three camera-path sky entry points with c2w[:3,:3] recovered from a DEVICE view (viewmat[12], cam_pos[3]; see
 * sgn_project_fwd_view) instead of cam->viewmat, by the same exact transpose and negation.  No cotangent for the view (the
 * _rot forms below give one). */
int sgn_sky_fwd_view(const sgn_camera* cam, const float* view, const float* jitter_u, const float* jitter_v, const float* tex, int R,
                     float* sky, float* dirs, void* stream);
int sgn_sky_bwd_view(const sgn_camera* cam, const float* view, const float* jitter_u, const float* jitter_v, int R, const float* v_sky,
                     float* v_tex, void* stream);
int sgn_sky_bwd_det_view(const sgn_camera* cam, const float* view, const float* jitter_u, const float* jitter_v, int R,
                         const float* v_sky, float* v_tex, void* scratch, size_t scratch_bytes, void* stream);
/* Gradient for the lookup direction (nvdiffrast's TextureGradKernelCubeLinear with indexCubeMapGrad, texture.cu:123-148 and
 * :1005-1046, filter_mode='linear', boundary_mode='cube'): per lookup g_s = sum_ch v ((a10 - a00) + fv (a11 + a00 - a10 -
 * a01)) R, g_t likewise with fu and a01, the four taps as the forward reads them (wrapped taps; at a cube corner the
 * missing tap is the mean of the other three), mapped to the 3-vector through s = <l,U> / (2|<l,N>|) + 1/2 on the RAW
 * direction (the [0,1] clamp of s, t is straight-through, as in nvdiffrast).  A zero cotangent, an invalid direction or a
 * non-finite result gives 0.  Each lookup reads tex; nothing is reordered, so the direction gradient is bit-reproducible.
 * The texture gradient beside it is that of the entry points above, bit for bit in the _det forms (the same kernel body);
 * v_tex may be NULL to skip it (then scratch is not read).
 * sgn_cube_texture_bwd_uv[_det]: nvdiffrast's gradTex + gradUV on given directions; v_uv[P,3] is WRITTEN.
 * sgn_sky_bwd_view_rot / sgn_sky_bwd_det_view_rot: the _view backward that also reduces the direction gradient to the
 * view's rotation (EnvLight.forward, sgn_splatfacto.py:140-147: l = to_opengl(c2w[:3,:3] u), u the normalised jittered
 * camera-space direction, independent of the rotation): v_d = (v_l.x, -v_l.z, v_l.y), v_R[i][j] = sum_pixels v_d[i] u[j],
 * v_view[4j+i] = s_j v_R[i][j] with s = (1, -1, -1) (the inverse of the view -> c2w mapping), v_view[3], [7], [11] = 0.
 * Per 32 x 32 tile the nine sums go to rot_partials (device, 4-byte aligned, sgn_sky_rot_scratch_bytes(W, H) bytes); one
 * more launch adds them in a fixed order and WRITES v_view[SGN_VIEW_FLOATS] (device).  No atomics: v_view is the same bits
 * on every run, in both forms. */
int sgn_cube_texture_bwd_uv(int P, const float* uv, const float* tex, int R, const float* v_out, float* v_tex /* or NULL */, float* v_uv,
                            void* stream);
int sgn_cube_texture_bwd_uv_det(int P, const float* uv, const float* tex, int R, const float* v_out, float* v_tex /* or NULL */,
                                float* v_uv, void* scratch, size_t scratch_bytes, void* stream);
size_t sgn_sky_rot_scratch_bytes(int width, int height); /* 0 for an empty image */
int sgn_sky_bwd_view_rot(const sgn_camera* cam, const float* view, const float* jitter_u, const float* jitter_v, const float* tex, int R,
                         const float* v_sky, float* v_tex /* or NULL */, float* rot_partials, size_t partials_bytes, float* v_view,
                         void* stream);
int sgn_sky_bwd_det_view_rot(const sgn_camera* cam, const float* view, const float* jitter_u, const float* jitter_v, const float* tex,
                             int R, const float* v_sky, float* v_tex /* or NULL */, void* scratch, size_t scratch_bytes,
                             float* rot_partials, size_t partials_bytes, float* v_view, void* stream);

/* ---- densification statistics (SURVEY.md 8f rank 3) -------------------------------------------------------
 * What each sub-model's `after_train` accumulates after backward (sgn_splatfacto.py:513-541), for all visible
 * sub-models of the frame in one launch: grads = ||v_records[:,0:2]||; on a sub-model's first call
 * xys_grad_norm = grads, vis_counts = 1, max_2Dsize = 0 (then the max below); afterwards, for rows with
 * radii > 0: xys_grad_norm += grads, vis_counts += 1; max_2Dsize = max(max_2Dsize, radii / max(H, W)). */
typedef struct sgn_densify_segment {
    int32_t row0, count;  /* rows of this sub-model in the frame's row space */
    int32_t first;        /* 1: the sub-model's statistics are being created by this call */
    int32_t pad;
    float* xys_grad_norm; /* [count] */
    float* vis_counts;    /* [count] */
    float* max_2Dsize;    /* [count] */
} sgn_densify_segment;
size_t sgn_sizeof_densify_segment(void);
int sgn_densify_stats(const sgn_densify_segment* table_dev, int nseg, int N, const float* v_records /*[N,12]*/,
                      const int32_t* radii /*[N]*/, int height, int width, void* stream);

/* ---- fused multi-tensor Adam (SURVEY.md 8f rank 1) ------------------------------------------------------
 * torch.optim.Adam semantics (betas, eps, no weight decay, no amsgrad) for every Gaussian parameter tensor in
 * ONE launch; replaces the nine nerfstudio Adam optimizers over ~200 tensors (sgn_config.py:71-108).
 * Gradients / exp_avg / exp_avg_sq are flat arenas of 16-byte aligned slices (offsets in floats, multiples of 4):
 * the gradient arena has the layout sgn_project_bwd wrote for the frame, the moment arenas cover every tensor of
 * the model; parameters are updated in place.  The table lists the tensors that have a gradient this step.  The host fills, per tensor and
 * per step, step_size = lr / (1 - beta1^t) and sqrt_bc2 = sqrt(1 - beta2^t), both evaluated in double. */
typedef struct sgn_adam_tensor {
    float* param;
    int64_t arena_offset; /* of the tensor's moments in exp_avg / exp_avg_sq */
    int64_t grad_offset;  /* of its gradient in grad_arena: the arena of a frame only holds the sub-models visible in that
                             frame (torch.optim.Adam skips parameters whose .grad is None: no decay, no step count) */
    int64_t numel;
    int32_t chunk0; /* first block of this tensor: sum over earlier tensors of ceil(numel / sgn_adam_chunk_elems()) */
    float beta1, beta2, eps, step_size, sqrt_bc2;
    float one_minus_beta1, one_minus_beta2; /* rounded from double on the host, as torch passes them (1 - 0.999f != 0.001f) */
} sgn_adam_tensor;
size_t sgn_sizeof_adam_tensor(void);
int sgn_adam_chunk_elems(void);
int sgn_adam_step(const sgn_adam_tensor* table_dev, int ntensors, int num_chunks, const float* grad_arena,
                  float* exp_avg, float* exp_avg_sq, void* stream);

/* ---- gradient exchange of the camera-sharded data-parallel step (SURVEY.md 8e) ---------------------------------
 * The reference has no distributed code; SURVEY 8e defines the exchange: SUM (or mean) of the flat per-Gaussian gradient
 * arena over the replicas.  sgn_allreduce_sym is that exchange as ONE kernel of this library over peer-mapped
 * ("symmetric") memory -- what a training loop would otherwise hand to ncclAllReduce: rank r reduces the r-th part of
 * every listed slice (multimem.ld_reduce through `multicast`, i.e. inside the NVSwitch; or, with multicast == NULL, loads
 * from every peer pointer in rank order), multiplies by `scale` and pushes the result to all replicas (multimem.st / one
 * store per peer), in place.  `local` is this rank's arena, `peer_ptrs_dev` a DEVICE array of `world` arena base pointers
 * (this rank's own included).  Slice offsets / lengths are in floats, multiples of 4.  The caller orders the call between
 * two cross-GPU barriers on the same stream (all replicas written; all parts pushed).  Bit-identical results on all ranks. */
#define SGN_AR_MAX_SLICES 48
/* Row skipping (optional, NULL = exchange everything): a slice with slice_widths[s] > 0 holds slice_rows[s] rows of that many
 * floats, row j of the slice is entry slice_row0[s] + j of `visible_union` (uint8, 1 = some replica saw the Gaussian).  Rows
 * nobody saw carry an all-zero gradient on every replica (sgn_project_bwd writes zeros there): their sum is already in place,
 * so they are neither pulled nor pushed.  sgn_visible_flags writes this rank's flags (radii > 0) -- into symmetric memory --
 * and sgn_visible_union ORs the peers' flags (peer base + flags_byte_offset) into a local array. */
int sgn_allreduce_sym(void* local, void* multicast, const uint64_t* peer_ptrs_dev, int rank, int world, int nslices,
                      const int64_t* slice_offsets, const int64_t* slice_lengths, const int32_t* slice_widths,
                      const int64_t* slice_row0, const int64_t* slice_rows, const uint8_t* visible_union, float scale, int max_ctas,
                      void* stream);
int sgn_visible_flags(const int32_t* radii, int64_t n, uint8_t* flags, void* stream);
int sgn_visible_union(const uint64_t* peer_ptrs_dev, int64_t flags_byte_offset, int world, int64_t n, uint8_t* out, void* stream);

/* ---- refinement: split / duplicate / cull (SURVEY.md 8f rank 3) ---------------------------------------------
 * What `SplatfactoModel.refinement_after` does to ONE sub-model every `refine_every` steps
 * (sgn_splatfacto.py:550-646 with cull_gaussians :648-672, split_gaussians :674-710, dup_gaussians :712-720 and the
 * optimizer surgery dup_in_optim / remove_from_optim :459-511), as two launches instead of ~120 torch statements
 * with eight host syncs per sub-model:
 *   sgn_refine_decide: per row, from the running statistics of sgn_densify_stats, the log-scales and the opacity
 *     logit -> flags (SGN_RF_* bits, csrc/sgn_refine_rules.cuh) and four 0/1 marks the caller prefix-sums;
 *   sgn_refine_apply: rebuilds the six parameter tensors and their Adam moments in the reference's row order
 *     [surviving old rows | split samples, sample-major | duplicates]: a split sample's mean is
 *     mean + R(q) (exp(scale) * z), split rows shrink by 1/1.6 in log space, new rows start with zero moments.
 * Both are HBM-bound streaming passes (decide: 32 B read per row; apply: 3 x 4 B read + written per element). */
typedef struct sgn_refine_config {
    int32_t densify;         /* 1: split + duplicate + cull (do_densification, :563-619); 0: cull only (:620-621) */
    int32_t n_split_samples; /* config.n_split_samples (2) */
    int32_t use_screen_size; /* step < stop_screen_size_at (:575, :662) */
    int32_t cull_big;        /* step > refine_every * reset_alpha_every (:659) */
    float max_size;          /* (float)max(last_size) (:570) */
    float densify_grad_thresh, densify_size_thresh, split_screen_size;
    float cull_alpha_thresh, cull_scale_thresh, cull_screen_size;
    float inv_size_fac;      /* fp32 reciprocal of size_fac = 1.6 (:694-695) */
} sgn_refine_config;

/* Source / destination of the rebuild: the six parameter tensors in gradient-arena order (means, scales, quats,
 * features_dc, features_rest, opacities) and, when an Adam state exists, exp_avg (m) and exp_avg_sq (v) per tensor
 * (all NULL = no optimizer state).  width[k] = floats per row of tensor k (3, 3, 4, 3F, 3(K-1), 1). */
typedef struct sgn_refine_tensors {
    const float* src[6];
    float* dst[6];
    const float* src_m[6];
    float* dst_m[6];
    const float* src_v[6];
    float* dst_v[6];
    int32_t width[6];
} sgn_refine_tensors;
size_t sgn_sizeof_refine_config(void);
size_t sgn_sizeof_refine_tensors(void);
/* flags[n] u8; marks[4,n] i32 = {survives, split samples survive, duplicate survives, is split} per row.
 * xys_grad_norm / vis_counts may be NULL when !cfg->densify, max_2Dsize when !cfg->use_screen_size. */
int sgn_refine_decide(int n, const sgn_refine_config* cfg, const float* scales /*[n,3]*/, const float* opacities /*[n,1]*/,
                      const float* xys_grad_norm, const float* vis_counts, const float* max_2Dsize, uint8_t* flags,
                      int32_t* marks, void* stream);
/* scan[4,n] = inclusive prefix sums of marks along the rows; totals[4] (HOST) = their last column; samples =
 * [n_split_samples * totals[3], 3] standard-normal draws (torch.randn, :680), NULL when totals[3] == 0.
 * Destinations hold totals[0] + n_split_samples * totals[1] + totals[2] rows. */
int sgn_refine_apply(int n, const sgn_refine_config* cfg, const sgn_refine_tensors* tensors, const uint8_t* flags,
                     const int32_t* scan, const int32_t* totals, const float* samples, void* stream);

/* ---- exact k-nearest-neighbour search (model initialisation, lidar chamfer distance) -------------------------
 * The initial scales of SplatfactoModel.populate_modules (sgn_splatfacto.py:260-264: log of the mean distance to the 3 nearest
 * other seed points, from sklearn's NearestNeighbors on the CPU, :439-457) and the nearest distances of calc_chamfer_distance
 * (data/utils/geometric_metric.py:59-69).  points [n,3] fp32; query [m,3] fp32 or NULL.  For every query row: its k nearest
 * points (1 <= k <= 16), ascending by fp32 distance, a tie going to the smaller row.  With query == NULL the queries are the
 * points themselves (m is ignored, n >= k + 1) and row i is never its own neighbour, while an exact duplicate of it is one at
 * distance 0; with a query set n >= k.  Exact: no cap on how far a search looks.  Deterministic: the same bytes every run.
 * Outputs, any of which may be NULL (not all three): dist [m,k] fp32 Euclidean distances, idx [m,k] int32 rows of `points`,
 * log_scales [m,3] = logf(mean of the k distances) broadcast (the scales tensor of populate_modules; -inf when they are all 0).
 * Inputs must be finite.  n, m < 2^31 - 1. */
size_t sgn_knn_scratch_bytes(int64_t n, int64_t m /* 0 without a query set */);
int sgn_knn(const float* points, int64_t n, const float* query, int64_t m, int k, float* dist, int32_t* idx, float* log_scales,
            void* scratch, size_t scratch_bytes, void* stream);

/* ---- lidar depth supervision (Street Gaussians' depth term; the reference's batch["depth_image"], sgn_datamanager.py:360-361,
 * and the depth_result its eval calls, sgn_splatfacto.py:1160-1168) ------------------------------------------------------------
 * sgn_lidar_depth_map: points [M,3] fp32 (device) into depth_map [H,W] fp32 (device; H, W = cam->height, cam->width) for the
 * camera the render uses.  to_world: NULL (the points are in the world frame) or a HOST 3x4 row-major sweep-to-world matrix,
 * composed with cam->viewmat in fp64 and rounded once to fp32.  A point's camera-space position pv, its depth z = pv.z and its
 * pixel centre u = (pv.x * rw) * fx + cx, v = (pv.y * rw) * fy + cy with rw = 1 / (z + 1e-6) are the projection's own
 * individually rounded arithmetic.  A point with z <= clip_thresh, or with u or v outside [0, W) x [0, H), is dropped; any
 * other goes to pixel (floor(u), floor(v)), where the nearest return wins.  Pixels without a return are 0.  The map is the same
 * bits every run; M = 0 is valid (an all-zero map).  cam->clip_thresh must be >= 0.  No host synchronisation.
 *
 * Loss over the valid pixels (target > 0 and, with a mask [H,W], mask != 0): *loss = weight * sum |depth - target| / n_valid,
 * exactly 0 when n_valid = 0; *n_valid (device int32) is what the backward divides by.  The backward writes all of v_depth:
 * grad_loss * weight * sign(depth - target) / n_valid on the valid pixels, 0 elsewhere (grad_loss: device scalar, NULL = 1).
 *
 * Metrics over the same valid pixels, with d = max(depth, 1e-3f), t = target: out[8] (device fp32) = {abs_rel = mean |d-t|/t,
 * sq_rel = mean (d-t)^2/t, rmse = sqrt(mean (d-t)^2), rmse_log = sqrt(mean (log d - log t)^2), a1, a2, a3 = fraction with
 * max(d/t, t/d) < 1.25^k, n_valid}; NaN means when n_valid = 0.
 * Loss and metrics sum in fp64 in a fixed order (bit-identical run to run).  Null inputs, an empty image, a null output
 * (SGN_ERR_INVALID) or a short scratch (SGN_ERR_WORKSPACE) launch nothing. */
int sgn_lidar_depth_map(const float* points, int64_t M, const sgn_camera* cam, const float* to_world, float* depth_map, void* stream);
size_t sgn_depth_scratch_bytes(void);
int sgn_depth_loss_fwd(int H, int W, const float* depth, const float* target, const float* mask, float weight, float* loss,
                       int32_t* n_valid, void* scratch, size_t scratch_bytes, void* stream);
int sgn_depth_loss_bwd(int H, int W, const float* depth, const float* target, const float* mask, float weight, const int32_t* n_valid,
                       const float* grad_loss, float* v_depth, void* stream);
int sgn_depth_metrics(int H, int W, const float* depth, const float* target, const float* mask, float* out, void* scratch,
                      size_t scratch_bytes, void* stream);

/* ---- per-Gaussian semantic logits (Street Gaussians' semantic term; the reference's batch["semantic"], data/sgn_dataset.py:125)
 * logits [H,W,C] fp32 (the semantic map sgn_blend_extra_fwd composites from extra[N,C]), labels [H,W] int64, mask [H,W] fp32 or
 * NULL; 1 <= C <= 64.  A pixel is valid when 0 <= label < C and (mask is NULL or mask != 0): any other label (e.g. 255) is ignored.
 *
 * Loss: *loss = weight * sum_valid CE(p) / n_valid with CE(p) = logsumexp(S[p,:]) - S[p,label], logsumexp in fp32 with the max
 * subtracted; exactly 0 when n_valid = 0.  *n_valid (device int32) is what the backward divides by.  The backward writes all of
 * v_logits: grad_loss * weight / n_valid * (softmax(S[p]) - onehot(label)) on the valid pixels, 0 elsewhere (grad_loss: device
 * scalar, NULL = 1).  Sums in fp64 per-block partials added in a fixed order (bit-identical run to run).
 *
 * Metrics: confusion [C,C] (device int64, overwritten) = counts of (label, argmax S) over the valid pixels, a tie going to the
 * lowest class index; integer atomics, so the counts are the same every run.
 *
 * Refinement carry: one further per-row tensor src [n,width] (1 <= width <= 64) and, optionally, its Adam moments rebuilt with
 * the row map of sgn_refine_apply for the same flags / scan / totals: [survivors | split samples, sample-major, each a copy of
 * its parent | duplicates]; survivors keep their moments, new rows get zero moments.  This is exactly what sgn_refine_apply
 * does to features_dc.  dst [totals[0] + n_split_samples * totals[1] + totals[2], width].
 * Null inputs, C or width out of range (SGN_ERR_INVALID) or a short scratch (SGN_ERR_WORKSPACE) launch nothing. */
size_t sgn_semantic_scratch_bytes(void);
int sgn_semantic_loss_fwd(int H, int W, int C, const float* logits, const int64_t* labels, const float* mask, float weight, float* loss,
                          int32_t* n_valid, void* scratch, size_t scratch_bytes, void* stream);
int sgn_semantic_loss_bwd(int H, int W, int C, const float* logits, const int64_t* labels, const float* mask, float weight,
                          const int32_t* n_valid, const float* grad_loss, float* v_logits, void* stream);
int sgn_semantic_metrics(int H, int W, int C, const float* logits, const int64_t* labels, const float* mask, int64_t* confusion,
                         void* stream);
int sgn_refine_carry(int n, const sgn_refine_config* cfg, const uint8_t* flags, const int32_t* scan, const int32_t* totals,
                     const float* src, float* dst, int width, const float* src_m, const float* src_v, float* dst_m, float* dst_v,
                     void* stream);

/* ---- scale regularisation (nerfstudio's use_scale_regularization, which the reference's config sets, sgn_splatfacto.py:206-211)
 * Over the N rows of the segment table (read in place, 128-row chunks as sgn_project_fwd), with s = exp(scales):
 *   *out = 0.1 * mean_rows(max(amax(s) / amin(s), max_ratio) - max_ratio)
 * expf / division / max in fp32 per row, sums in fp64 per block added in a fixed order (bit-identical run to run), the mean rounded
 * once to fp32, then * 0.1f.  N = 0 gives NaN, as torch's mean of nothing.  No host synchronisation.
 * The backward ADDS d out / d scales * (*v_out) into grads_dev[k].scales (v_out: device scalar), following torch autograd of the
 * expression in fp32: the gradient is halved at amax / amin == max_ratio (torch.maximum's tie) and split evenly between tied
 * elements of the max and of the min.  Rows with amax / amin < max_ratio are not written.  Elementwise: deterministic.
 * A null table with nseg > 0, a null out / scratch / v_out, chunks without segments (SGN_ERR_INVALID) or a short scratch
 * (SGN_ERR_WORKSPACE) launch nothing. */
size_t sgn_scale_reg_scratch_bytes(void);
int sgn_scale_reg_fwd(const sgn_segment* table_dev, int nseg, int N, int num_chunks, float max_ratio, float* out, void* scratch,
                      size_t scratch_bytes, void* stream);
int sgn_scale_reg_bwd(const sgn_segment* table_dev, const sgn_segment_grads* grads_dev, int nseg, int N, int num_chunks, float max_ratio,
                      const float* v_out, void* stream);

/* ---- 3D smoothing filter sizes (Mip-Splatting, Yu et al. 2024, eq. 7: compute_3D_filter)
 * For every row i of sub-model m (nsub sub-models; subs_dev[m] = its means [count,3], its output sigma [count], its count and
 * its first 128-row chunk, chunk0 = sum over earlier sub-models of ceil(count/128); num_chunks the total):
 *   nu_i = max over views v with xforms[v * nsub + m].present of max(fx, fy) / z, over the views where
 *          p = M[0:3,0:3] mu_i + M[:,3] (M = xforms[v * nsub + m].M, row-major 3x4, object -> camera) has z > near and
 *          u = fx x / z + cx in [-0.15 W, 1.15 W], w = fy y / z + cy in [-0.15 H, 1.15 H] (bounds inclusive);
 *   sigma_i = sqrt(variance) / nu_i.
 * Rows no view samples get the largest sigma of the sampled rows; with none sampled, every sigma is 0.  The transform and tests
 * are evaluated in fp64.  stats (device, 2 x int32, overwritten): [0] the number of sampled rows, [1] the bits of the largest
 * sampled sigma.  No float atomics, no host synchronisation: two launches and one memset. */
typedef struct sgn_filter_view {
    float fx, fy, cx, cy;
    int32_t width, height;
} sgn_filter_view;
typedef struct sgn_filter_xform {
    double M[12];    /* object -> camera: the view matrix composed with the sub-model's object -> world pose at the view's time */
    int32_t present; /* 0: the sub-model is not in this view (an actor without a box at the view's timestamp) */
    int32_t pad;
} sgn_filter_xform;
typedef struct sgn_filter_sub {
    const float* means; /* [count,3] */
    float* out;         /* [count] sigma */
    int32_t count;
    int32_t chunk0;
} sgn_filter_sub;
size_t sgn_sizeof_filter_xform(void);
int sgn_filter3d(const sgn_filter_sub* subs_dev, int nsub, int num_chunks, const sgn_filter_view* views_dev, int V,
                 const sgn_filter_xform* xforms_dev, double variance, double near, int32_t* stats, void* stream);

/* ---- per-image bilateral grids (Wang et al., SIGGRAPH 2024; gsplat's use_bilateral_grid): appearance correction
 * A grid is [12, L, Hg, Wg] float32 (a 3x4 affine per node, row-major over output channels r, g, b by inputs r, g, b, 1).
 * Slice of one H x W image rgb [H,W,3] with one grid: pixel (i, j) samples the grid trilinearly (corners clamped) at
 *   gx = (j + 0.5) / W * (Wg - 1), gy = (i + 0.5) / H * (Hg - 1), gz = clamp(0.299 r + 0.587 g + 0.114 b, 0, 1) * (L - 1)
 * giving M = [A | t]; out = A c + t (F.grid_sample(align_corners=True, padding_mode="border") followed by the affine).
 * sgn_bilagrid_slice_bwd writes d_rgb [H,W,3] (A^T d_out plus the guidance term where the gray is strictly inside (0, 1)) and
 * overwrites d_grid [12,L,Hg,Wg] with the trilinear scatter of d_out (x) (c, 1).  No float atomics: two runs give the same
 * bits.  L <= 32 in the backward.  scratch: sgn_bilagrid_slice_bwd_scratch_bytes (per-block partials).
 * Total variation over N grids [N,12,L,Hg,Wg]: tv = (1/N) sum over the axes L, Hg, Wg of mean((forward difference)^2), each
 * mean over every image and coefficient, an axis of size 1 adding 0; out is a device float, summed in fp64 in a fixed order
 * (scratch: sgn_bilagrid_tv_scratch_bytes).  sgn_bilagrid_tv_bwd overwrites d_grids with v_out[0] * d tv / d grids. */
int sgn_bilagrid_slice_fwd(const float* grid, int L, int Hg, int Wg, const float* rgb, int H, int W, float* out, void* stream);
size_t sgn_bilagrid_slice_bwd_scratch_bytes(int L, int Hg, int Wg, int H, int W);
int sgn_bilagrid_slice_bwd(const float* grid, int L, int Hg, int Wg, const float* rgb, const float* d_out, int H, int W, float* d_rgb,
                           float* d_grid, void* scratch, size_t scratch_bytes, void* stream);
size_t sgn_bilagrid_tv_scratch_bytes(void);
int sgn_bilagrid_tv_fwd(const float* grids, int N, int L, int Hg, int Wg, float* out, void* scratch, size_t scratch_bytes, void* stream);
int sgn_bilagrid_tv_bwd(const float* grids, int N, int L, int Hg, int Wg, const float* v_out, float* d_grids, void* stream);

/* ---- densification by MCMC (Kheradmand et al., NeurIPS 2024; gsplat's MCMCStrategy)
 * Throughout o = sigmoid(logit) and s = exp(log_scale) in fp32.  Random draws come from Philox4x32-10 with key = seed and counter
 * (index, step, sub, purpose) -- purpose SGN_MCMC_NOISE / _RELOCATE / _ADD, index the row or the draw -- so a call gives the same
 * bits on every run and for every launch shape.
 *
 * sgn_mcmc_noise: for every row of every sub-model (subs_dev[k]: rows [0, count), first 128-row chunk chunk0, first row row0 of
 * the concatenated index space, Philox sub index, its noise_lr), with eps ~ N(0, I3) from Philox (or normals[row0 + row] when
 * normals != NULL) and lr the means' learning rate:
 *   gate = 1 / (1 + exp(-100 ((1 - o) - 0.995))),  Sigma = R(q/|q|) diag(s^2) R^T,  means += Sigma (eps * gate * (lr * noise_lr)).
 *
 * sgn_mcmc_sample: weights w_i = o_i (0 for rows with o_i <= min_opacity when exclude_dead), their fp64 inclusive prefix sum P
 * (summed in a fixed order), then draw j takes the first row with P_i > u_j * P_{n-1}, u_j from Philox (or uniforms[j], in
 * [0, 1)).  The number of draws is *num_draws_dev when given (device), else max_draws.  counts [n] is overwritten with the
 * number of draws of each row (integer atomics).  With a zero total no row is drawn and draws[j] = -1.  dead_rows / num_dead
 * (optional, device): the rows with o_i <= min_opacity in ascending order and their number.  total (optional, device double):
 * P_{n-1}.  scratch: sgn_mcmc_sample_scratch_bytes(n).  Nothing is read back.
 *
 * sgn_mcmc_relocate: for every row i with c = counts[i] > 0 and N = min(c + 1, 51), in fp64, rounded once:
 *   o' = 1 - (1 - o)^(1/N),  denom = sum_{k=1..N} (-1)^(k-1) C(N,k) o'^k / sqrt(k),
 *   log_scale = log((o / denom) s),  logit = logit(clamp(o', min_opacity, 1 - 2^-23)),
 * and zeroes row i of every tensor of `zero` (the Adam moments) when zero != NULL.
 *
 * sgn_mcmc_copy_rows: row dst_j <- row src_j in every tensor of `t`, for j < (*num_rows_dev or max_rows), dst_j = dst_rows[j] or
 * dst_row0 + j, skipping src_j < 0.  Sources and destinations must not overlap.
 *
 * sgn_mcmc_reg_fwd / _bwd: over the N rows of the segment table (128-row chunks), out[0] = w_o * mean_i o_i and
 * out[1] = w_s * mean_{i,k} s_ik (fp64 sums in a fixed order, each mean rounded once to fp32, times w in fp32; bit-identical
 * run to run).  The backward ADDS v_out[0] * d out[0] + v_out[1] * d out[1] into grads_dev[k].opacities / .scales (v_out:
 * two device floats, either pointer may be NULL = no cotangent).  Elementwise: deterministic. */
#define SGN_MCMC_NOISE 0
#define SGN_MCMC_RELOCATE 1
#define SGN_MCMC_ADD 2
#define SGN_MCMC_MAX_TENSORS 16
typedef struct sgn_mcmc_sub {
    float* means;             /* [count,3], updated in place */
    const float* scales;      /* [count,3] log */
    const float* quats;       /* [count,4] wxyz, un-normalised */
    const float* opacities;   /* [count,1] logit */
    int32_t count;
    int32_t chunk0;
    int32_t row0;
    int32_t index;            /* the sub-model's index: part of the Philox counter */
    float noise_lr;
    int32_t pad;
} sgn_mcmc_sub;
typedef struct sgn_mcmc_tensors {
    float* data[SGN_MCMC_MAX_TENSORS]; /* row-major [rows, width] */
    int32_t width[SGN_MCMC_MAX_TENSORS];
    int32_t count;
    int32_t pad;
} sgn_mcmc_tensors;
size_t sgn_sizeof_mcmc_sub(void);
size_t sgn_sizeof_mcmc_tensors(void);
int sgn_mcmc_noise(const sgn_mcmc_sub* subs_dev, int nsub, int num_chunks, float lr, uint64_t seed, int step, const float* normals,
                   void* stream);
size_t sgn_mcmc_sample_scratch_bytes(int n);
int sgn_mcmc_sample(const float* opacities, int n, float min_opacity, int exclude_dead, int max_draws, const int32_t* num_draws_dev,
                    uint64_t seed, int step, int sub, int purpose, const double* uniforms, int32_t* draws, int32_t* counts,
                    int32_t* dead_rows, int32_t* num_dead, double* total, void* scratch, size_t scratch_bytes, void* stream);
int sgn_mcmc_relocate(float* opacities, float* scales, int n, const int32_t* counts, float min_opacity, const sgn_mcmc_tensors* zero,
                      void* stream);
int sgn_mcmc_copy_rows(const sgn_mcmc_tensors* t, const int32_t* dst_rows, int dst_row0, const int32_t* src_rows, int max_rows,
                       const int32_t* num_rows_dev, void* stream);
size_t sgn_mcmc_reg_scratch_bytes(void);
int sgn_mcmc_reg_fwd(const sgn_segment* table_dev, int nseg, int N, int num_chunks, float w_opacity, float w_scale, float* out,
                     void* scratch, size_t scratch_bytes, void* stream);
int sgn_mcmc_reg_bwd(const sgn_segment* table_dev, const sgn_segment_grads* grads_dev, int nseg, int N, int num_chunks, float w_opacity,
                     float w_scale, const float* v_opacity, const float* v_scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SGN_RASTER_H_ */

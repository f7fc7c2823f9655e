/*
 * rgs_b200.h -- C ABI of the H100-native (sm_90a) differentiable Gaussian-splat rasterizer.
 *
 * This is the drop-in boundary of the hot path.  The reference binds the same path through a pybind11
 * torch extension (`diff_gaussian_rasterization._C`, reference: submodules/diff-gaussian-rasterization/
 * ext.cpp:15-20, rasterize_points.h:18-81) whose C++ core is CudaRasterizer::Rasterizer
 * (cuda_rasterizer/rasterizer.h:25-149).  The entry points below are what that core exposes, restated
 * as a plain C ABI: raw device pointers, sizes and a cudaStream_t, no torch types.  The torch glue in
 * rade-gs_b200/csrc/torch_glue.cpp is the only caller in the product and rebuilds the reference's four
 * pybind symbols on top of it.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless stated otherwise; optional inputs are NULL when absent
 *     (the reference passes empty tensors whose data pointer is null, rasterize_points.cu:104-112);
 *   - matrices are 16 floats in the memory order torch hands over (`world_view_transform`, i.e.
 *     column-major of the maths matrix, cuda_rasterizer/auxiliary.h:74-93);
 *   - scratch memory is obtained through caller-supplied resize callbacks, exactly like the reference's
 *     std::function<char*(size_t)> geometry/binning/image buffers (cuda_rasterizer/rasterizer.h:31-35);
 *     their CONTENT is private to this library, the caller only keeps them alive between forward and
 *     backward and hands the same bytes back;
 *   - functions return >= 0 on success (rgs_forward: num_rendered) and a negative rgs_status on error;
 *     rgs_last_error() gives the message of the last failure on the calling thread.
 *   - there is no CPU fallback: without a CUDA device every compute entry point fails with RGS_E_CUDA.
 */
#ifndef RGS_B200_H_INCLUDED
#define RGS_B200_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RGS_ABI_VERSION 4

typedef enum rgs_status {
	RGS_OK = 0,
	RGS_E_INVALID = -1,      /* bad argument (shape/flag combination the reference rejects)            */
	RGS_E_CUDA = -2,         /* CUDA runtime error (message in rgs_last_error)                         */
	RGS_E_UNSUPPORTED = -3,  /* e.g. prefiltered=true (mis-wired in the reference, SURVEY app. A-15)    */
	RGS_E_ALLOC = -4,        /* a resize callback returned NULL                                        */
	RGS_E_CAPACITY = -5      /* rgs_tsdf_touch: the frame-local hash is full; grow it and call again     */
} rgs_status;

/* Resize callback: make the buffer at least `bytes` long and return its device address.
 * Mirrors cuda_rasterizer/rasterizer.h:31-33 / rasterize_points.cu:27-33 (resizeFunctional). */
typedef char* (*rgs_resize_fn)(void* user, size_t bytes);

/* Camera + raster settings shared by forward and backward
 * (GaussianRasterizationSettings, diff_gaussian_rasterization/__init__.py:171-186). */
typedef struct rgs_camera {
	int32_t width, height;
	float tan_fovx, tan_fovy;
	float kernel_size;       /* 2D mip filter added to the cov2D diagonal (forward.cu:116-118)       */
	float scale_modifier;
	const float* viewmatrix; /* [16] */
	const float* projmatrix; /* [16] */
	const float* cam_pos;    /* [3]  */
	const float* background; /* [3]  */
	int32_t sh_degree;       /* active degree D                                                        */
	int32_t sh_coeffs;       /* M = coefficients stored per Gaussian (0 when shs == NULL)              */
	int32_t require_coord, require_depth, prefiltered, debug;
	/* Tile-row slab rendered by this call: tile rows [tile_row_begin, tile_row_end).  (0, -1) = whole
	 * image.  Multi-GPU row sharding (DESIGN.md "Multi-GPU"); the reference has no equivalent.       */
	int32_t tile_row_begin, tile_row_end;
	/* ABI 3: compact_slab != 0 -> every [C,H,W] map of this call (forward outputs; backward's upstream gradients, alpha and
	 * normal maps) holds ONLY the pixel rows of the slab, i.e. is [C, Hs, W] with Hs = min(tile_row_end*16, H) - tile_row_begin*16.
	 * Per-rank image memory, its zero-fill and the image-side scratch then scale with 1/ranks.  0 = full-size maps whose rows
	 * outside the slab the library does not touch. */
	int32_t compact_slab;
} rgs_camera;

/* Per-Gaussian model inputs (rasterize_points.h:18-41). */
typedef struct rgs_gaussians {
	int32_t P;
	const float* means3D;        /* [P,3]                       */
	const float* opacities;      /* [P]                         */
	const float* shs;            /* [P,M,3] or NULL             */
	const float* colors_precomp; /* [P,3]   or NULL             */
	const float* scales;         /* [P,3]   or NULL             */
	const float* rotations;      /* [P,4]   or NULL (r,x,y,z)   */
	const float* cov3D_precomp;  /* [P,6]   or NULL             */
	/* ABI 2, opt-in (SURVEY.md 8f-1): SH coefficients left in the two tensors the model stores them in
	 * (GaussianModel._features_dc / _features_rest, scene/gaussian_model.py:133-136), sparing the per-iteration
	 * torch.cat copy.  When shs_rest != NULL, `shs` is [P,1,3] (coefficient 0) and shs_rest [P,M-1,3]. */
	const float* shs_rest;
} rgs_gaussians;

/* Forward outputs (rasterize_points.cu:71-78); maps of a variant that is switched off are zero-filled. */
typedef struct rgs_forward_out {
	float* out_color;  /* [3,H,W] */
	float* out_coord;  /* [3,H,W] */
	float* out_mcoord; /* [3,H,W] */
	float* out_alpha;  /* [1,H,W] */
	float* out_normal; /* [3,H,W] */
	float* out_depth;  /* [1,H,W] */
	float* out_mdepth; /* [1,H,W] */
	int32_t* radii;    /* [P]     */
} rgs_forward_out;

typedef struct rgs_buffers {
	rgs_resize_fn geom;    void* geom_user;
	rgs_resize_fn binning; void* binning_user;
	rgs_resize_fn image;   void* image_user;
} rgs_buffers;

/* Replaces CudaRasterizer::Rasterizer::forward (rasterizer.h:25-66, rasterizer_impl.cu:254-425).
 * Returns num_rendered (>= 0) or a negative rgs_status.  One stream synchronisation inside (the
 * reference has the same blocking read of num_rendered, rasterizer_impl.cu:354). */
int64_t rgs_forward(const rgs_camera* cam, const rgs_gaussians* g, const rgs_forward_out* out,
                    const rgs_buffers* bufs, void* cuda_stream);

/* ---- rgs_forward without the host read, for CUDA-graph capture (DESIGN.md §9 item 3) ----
 * The binning buffer and the per-tile sort are sized from the caller's capacities instead of the frame's instance count and
 * longest tile list, so the call makes no device-to-host copy, no synchronisation and no host allocation (buffers grow only
 * through the resize callbacks).  Same kernels as rgs_forward; for a frame that fits, the maps, radii, sorted ids and keys are
 * bit-identical to rgs_forward's.  Returns preset->instances: the num_rendered to give the backward (it fixes the binning
 * layout).  `status` is DEVICE memory, 4 words, accumulated over calls until the caller clears it:
 *   [0] overflow bits OR-ed in (1: the frame has more instances than `instances`, 2: a longer tile list than `longest_list`),
 *   [1] the largest instance count seen, [2] the longest tile list seen, [3] reserved.
 * A frame that overflows writes nothing outside the carved buffers: its maps are the background and its radii as computed;
 * the caller discards the result and calls again with larger capacities.  Whole image only: a tile-row slab, compact_slab,
 * debug (it synchronises) and prefiltered are rejected.  The first call on a device must be made outside stream capture (it
 * opts the sort kernels in to their shared memory). */
typedef struct rgs_preset {
	int64_t instances;      /* the binning buffer is carved for this many instances                          */
	int32_t longest_list;   /* tile-sort shared memory / long-list passes are sized for this list length     */
	uint32_t* status;       /* DEVICE, 4 words (above)                                                        */
} rgs_preset;
int64_t rgs_forward_preset(const rgs_camera* cam, const rgs_gaussians* g, const rgs_forward_out* out,
                           const rgs_buffers* bufs, const rgs_preset* preset, void* cuda_stream);

/* ---- balanced row sharding: each frame's slabs cut from that frame's instance counts (DESIGN.md "Multi-GPU") ----
 * Partition rule, integer-only, the same on every rank because preprocess and the tile counts are:
 *   - I_y = instances (splat-tile pairs) in tile row y, over the whole image; grid_x tiles per row;
 *   - row weight w_y = I_y + RGS_BALANCE_TILE_COST * grid_x: the blend kernels pay per instance and, per tile, a fixed cost
 *     (CTA start, per-pixel set-up, the seven map writes, backward's per-pixel reads) worth RGS_BALANCE_TILE_COST instances;
 *   - every slab holds at least one tile row (grid_y < world_size is RGS_E_INVALID);
 *   - B* = the least possible largest slab weight over all such partitions into world_size contiguous slabs;
 *   - cut greedily: ranks in order, each takes rows while its weight stays <= B* and enough rows remain for one per later
 *     rank; the last rank takes the rest (its weight is <= B* too).
 * row_cuts (host, world_size + 1 entries) receives the slab boundaries: rank r owns tile rows [row_cuts[r], row_cuts[r+1]).
 * row_instances is a host array of grid_y counts.  Host-only, no GPU needed. */
#define RGS_BALANCE_TILE_COST 2048
int32_t rgs_balance_partition(int32_t grid_y, int32_t grid_x, int32_t world_size, const uint32_t* row_instances, int32_t* row_cuts);

/* Maps callback of rgs_forward_balanced: the slab is known only after the frame's tile counts are read, so the caller allocates
 * the forward maps then.  Receives the chosen tile rows [tile_row_begin, tile_row_end) and the maps' height (the slab's pixel rows
 * with cam->compact_slab, else the image height); sets out's seven map pointers ([C, height, W] each; with full-size maps the rows
 * outside the slab are the caller's to fill, as for rgs_forward).  Returns 0, or non-zero when it could not allocate. */
typedef int32_t (*rgs_maps_fn)(void* user, int32_t tile_row_begin, int32_t tile_row_end, int32_t height, rgs_forward_out* out);

/* rgs_forward for rank `rank` of `world_size` with the slab chosen from this frame:
 *   preprocess over the whole image's tile rows -> tile counts -> per-row I_y and L_y (longest tile list of the row) -> ONE
 *   host read (it replaces rgs_forward's read of num_rendered; still the only synchronisation) -> rgs_balance_partition ->
 *   the tile ranges, chunk offsets, totals and per-splat tile counts restricted to this rank's slab -> `maps` -> binning,
 *   sort and blend of the slab.
 * Binning, sort, blend and the buffers left for backward are exactly those of rgs_forward with cam->tile_row_begin/end set to
 * the chosen slab, so backward is rgs_backward_render / rgs_backward_render_exchange with those rows.  cam->tile_row_begin /
 * tile_row_end are ignored.  out->radii is used as given, out's map pointers are set by `maps`.  row_cuts (host, world_size + 1)
 * receives the whole partition; row_stats (host, 2 * grid_y, may be NULL) receives I_y then L_y.  Returns num_rendered of the
 * slab or a negative rgs_status. */
int64_t rgs_forward_balanced(const rgs_camera* cam, const rgs_gaussians* g, int32_t world_size, int32_t rank, rgs_forward_out* out,
                             rgs_maps_fn maps, void* maps_user, const rgs_buffers* bufs, int32_t* row_cuts, uint32_t* row_stats,
                             void* cuda_stream);

/* ---- opacity integration at query points (SURVEY.md 8f-3) ----
 * Replaces CudaRasterizer::Rasterizer::integrate (rasterizer.h:68-108, rasterizer_impl.cu:573-844; binding
 * rasterize_points.cu:269-388).  All outputs are fully written by the call (untouched points get the reference's fill values
 * 1 / 0 / 0 / -1000; out_color channel 5 is zero, channel 8 counts the points per pixel).  cam->kernel_size is used as
 * given (the reference's Python wrapper passes 0.0); require_coord / require_depth / tile rows are ignored. */
typedef struct rgs_integrate_io {
	int32_t PN;
	const float* points3D;        /* [PN,3] query points (world space)                         */
	float* out_color;             /* [9,H,W] rgb, expected depth, median depth, 0, max depth, alpha, points per pixel */
	float* out_alpha_integrated;  /* [PN]                                                      */
	float* out_color_integrated;  /* [PN,3]                                                    */
	float* out_coordinate2d;      /* [PN,2] pixel coordinates of the projected points          */
	float* out_sdf;               /* [PN]   median-splat depth along the ray minus point depth */
	int32_t* radii;               /* [P]                                                       */
} rgs_integrate_io;

/* Returns num_rendered or a negative rgs_status.  point_buffer is a fourth resizable scratch buffer (the reference's
 * pointBuffer / point_binningBuffer).  overflowed_pixels (may be NULL; non-NULL costs one more stream synchronisation)
 * receives the number of pixels that collected 2048 contributing splats and stopped there, as in the reference. */
int64_t rgs_integrate(const rgs_camera* cam, const rgs_gaussians* g, const rgs_integrate_io* io, const rgs_buffers* bufs,
                      rgs_resize_fn point_buffer, void* point_buffer_user, int32_t* overflowed_pixels, void* cuda_stream);

/* Upstream gradients of the seven maps (rasterize_points.h:57-63) + forward results read by backward. */
typedef struct rgs_backward_in {
	const float* dL_dout_color;  /* [3,H,W] */
	const float* dL_dout_coord;  /* [3,H,W] */
	const float* dL_dout_mcoord; /* [3,H,W] */
	const float* dL_dout_depth;  /* [1,H,W] */
	const float* dL_dout_mdepth; /* [1,H,W] */
	const float* dL_dout_alpha;  /* [1,H,W] */
	const float* dL_dout_normal; /* [3,H,W] */
	const float* out_alpha;      /* forward's alpha map  [1,H,W] */
	const float* out_normal;     /* forward's normal map [3,H,W] */
	const int32_t* radii;        /* [P] */
	const char* geom_buffer;     /* bytes written by rgs_forward */
	const char* binning_buffer;
	const char* image_buffer;
	int64_t num_rendered;
} rgs_backward_in;

/* Final gradients (rasterize_points.cu:180-193,245).  All are fully written (zeros for Gaussians that
 * were not rendered); the caller does not need to clear them. */
typedef struct rgs_backward_out {
	float* dL_dmeans2D;   /* [P,3] (x, y, |.| channel, backward.cu:1002-1006) */
	float* dL_dcolors;    /* [P,3] */
	float* dL_dopacity;   /* [P]   */
	float* dL_dmeans3D;   /* [P,3] */
	float* dL_dcov3D;     /* [P,6] */
	float* dL_dsh;        /* [P,M,3] or NULL when M == 0 */
	float* dL_dscales;    /* [P,3] */
	float* dL_drotations; /* [P,4] */
	float* dL_dsh_rest;   /* ABI 2: [P,M-1,3] when the forward call passed shs_rest (then dL_dsh is [P,1,3]); else NULL */
} rgs_backward_out;

/* Floats per Gaussian of the screen-space gradient accumulator for a variant (16 or 32). */
int32_t rgs_grad_stride(int32_t require_coord, int32_t require_depth);

/* Stage 1 of backward: replaces BACKWARD::render (backward.cu:631-1016).  Zero-fills and accumulates
 * grad_accum[P * rgs_grad_stride] with the per-Gaussian screen-space gradients of this call's tile slab.
 * The accumulator is a plain sum over pixels, hence additive across slabs/ranks: multi-GPU callers
 * all-reduce it between stage 1 and stage 2. */
int32_t rgs_backward_render(const rgs_camera* cam, const rgs_gaussians* g, const rgs_backward_in* in,
                            float* grad_accum, void* cuda_stream);

/* Stage 2: replaces BACKWARD::preprocess (backward.cu:145-628): grad_accum -> parameter gradients. */
int32_t rgs_backward_preprocess(const rgs_camera* cam, const rgs_gaussians* g, const rgs_backward_in* in,
                                const float* grad_accum, const rgs_backward_out* out, void* cuda_stream);

/* Replaces CudaRasterizer::Rasterizer::backward (rasterizer.h:110-148, rasterizer_impl.cu:429-571):
 * stage 1 + stage 2 with an internally allocated accumulator (scratch through `grad_scratch`). */
int32_t rgs_backward(const rgs_camera* cam, const rgs_gaussians* g, const rgs_backward_in* in,
                     const rgs_backward_out* out, rgs_resize_fn grad_scratch, void* grad_scratch_user,
                     void* cuda_stream);

/* ---- multi-GPU: device-side exchange of the accumulator rows over peer memory (ABI 3; DESIGN.md "Multi-GPU") ----
 * One process per GPU, rank r renders the tile rows of its slab (rgs_camera.tile_row_begin/end).  The north star's
 * "all-reduce of the per-Gaussian gradients after backward" is done by the library itself over NVLink instead of by a
 * host-driven collective: each rank creates one exchange object (a device allocation exported with cudaIpcGetMemHandle),
 * the caller gathers the 64-byte handles of all ranks with whatever transport it has (torch.distributed in the product)
 * and connects; after that
 *     rgs_backward_render_exchange  = stage 1 into a persistent local accumulator + push of the touched rows to their
 *                                     owner rank (vector reductions into peer memory) + barrier + spread of the summed
 *                                     rows to every rank + barrier (all on the given stream, no host synchronisation)
 *     rgs_exchange_result           = the summed rows [capacity, row_floats] to hand to rgs_backward_preprocess
 * All ranks must make the same sequence of calls with the same P.  The result is bit-identical on every rank.
 * The reference is single-GPU and has no equivalent; the sum reproduced is backward.cu:878-1013's atomic accumulation. */
typedef struct rgs_exchange rgs_exchange;
#define RGS_IPC_HANDLE_BYTES 64
int32_t rgs_exchange_create(int32_t rank, int32_t world, int64_t capacity_rows, int32_t row_floats, rgs_exchange** out,
                            void* ipc_handle /* host, RGS_IPC_HANDLE_BYTES */);
int32_t rgs_exchange_connect(rgs_exchange* ex, const void* all_handles /* host, world * RGS_IPC_HANDLE_BYTES, rank-major */);
int32_t rgs_exchange_destroy(rgs_exchange* ex);
float* rgs_exchange_accumulator(rgs_exchange* ex);     /* persistent local accumulator (all-zero between steps) */
const float* rgs_exchange_result(rgs_exchange* ex);    /* summed rows, valid after rgs_backward_render_exchange on the same stream */
/* push + barrier + spread + barrier for an accumulator already filled by stage 1 (tiles_touched: this call's per-splat tile
 * counts inside the slab, radii: forward's radii) */
int32_t rgs_exchange_rows(rgs_exchange* ex, int32_t P, const uint32_t* tiles_touched, const int32_t* radii, void* cuda_stream);
int32_t rgs_backward_render_exchange(const rgs_camera* cam, const rgs_gaussians* g, const rgs_backward_in* in, rgs_exchange* ex,
                                     void* cuda_stream);
/* Synchronises the stream and returns 0 when every barrier so far completed, 1 + p when one gave up (after ~10 s) waiting for
 * rank p -- the rows of that step are then meaningless; callers fall back to a host-driven collective. */
int32_t rgs_exchange_status(rgs_exchange* ex, void* cuda_stream);

/* Replaces CudaRasterizer::Rasterizer::markVisible (rasterizer.h:18-23, rasterizer_impl.cu:176-188). */
int32_t rgs_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                         uint8_t* present, void* cuda_stream);

/* ---- next row of the path (SURVEY.md 8f-1), opt-in: the per-Gaussian arithmetic directly around the rasterizer call ----
 * rgs_activate_*: fused GaussianModel.get_scaling_n_opacity_with_3D_filter + get_rotation (reference
 * scene/gaussian_model.py:156-166, 125-126): raw parameters -> (scales [P,3], opacity [P], unit rotations [P,4]) and back.
 * rgs_densification_stats: train.py:187-188 + GaussianModel.add_densification_stats (scene/gaussian_model.py:743-747) in one
 * pass over the Gaussians with radii > 0; max_radii2D may be NULL. */
int32_t rgs_activate_forward(int32_t P, const float* raw_scaling, const float* raw_opacity, const float* raw_rotation,
                             const float* filter_3D, float* scales, float* opacity, float* rotations, void* cuda_stream);
int32_t rgs_activate_backward(int32_t P, const float* raw_scaling, const float* raw_opacity, const float* raw_rotation,
                              const float* filter_3D, const float* g_scales, const float* g_opacity, const float* g_rotations,
                              float* d_raw_scaling, float* d_raw_opacity, float* d_raw_rotation, void* cuda_stream);
int32_t rgs_densification_stats(int32_t P, const float* means2D_grad, const int32_t* radii, float* grad_accum,
                                float* grad_accum_abs, float* grad_accum_abs_max, float* denom, float* max_radii2D,
                                void* cuda_stream);

/* rgs_compute_3d_filter: GaussianModel.compute_3D_filter (scene/gaussian_model.py:179-232) as two kernels instead of a Python
 * loop over cameras.  cams: DEVICE table [n_cams,16] = R (3x3 row-major, Camera.R), T (3), focal_x, focal_y, width, height;
 * focal_length = max focal_x over the cameras (host).  filter_3D [P] receives distance / focal_length * sqrt(0.2);
 * max_distance (device scalar) receives the largest distance among points seen by a camera, 0 if none was seen (the
 * reference raises in that case). */
int32_t rgs_compute_3d_filter(int32_t P, const float* xyz, int32_t n_cams, const float* cams, float focal_length,
                              float* filter_3D, float* max_distance, void* cuda_stream);

/* ---- image-side consumers of the maps (SURVEY.md 8f-2), opt-in ----
 * rgs_ssim_l1_forward: utils/loss_utils.py:17-18 and :35-63 over `planes` [H,W] fp32 planes.  sums[0] = sum of the SSIM map,
 *   sums[1] = sum |img - gt| (the call zeroes them; divide by planes*H*W for the means).  dmaps ([3,planes,H,W], may be NULL
 *   for evaluation) receives the partial derivatives of the SSIM map that rgs_ssim_l1_backward needs.
 * rgs_ssim_l1_backward: d_img = upstream * (w_ssim * d(sum SSIM map)/d img + w_l1 * sign(img - gt)); upstream is a DEVICE
 *   scalar or NULL (1.0).  For train.py:163's loss: w_ssim = -lambda_dssim / n, w_l1 = (1 - lambda_dssim) / n.
 * rgs_normal_consistency: train.py:143-156 with utils/graphics_utils.py:97-126.  from_depth != 0: the two maps are [1,H,W]
 *   depth maps, back-projected with rays ((x+0.5)*inv_fx + cx, (y+0.5)*inv_fy + cy, 1); else they are [3,H,W] point maps.
 *   loss_sum = sum over pixels of w_expected*(1 - <normal, n_expected>) + w_median*(1 - <normal, n_median>) (zeroed by the call);
 *   d_normal [3,H,W], d_expected / d_median (shaped like the maps) are fully written. */
int32_t rgs_ssim_l1_forward(int32_t planes, int32_t H, int32_t W, const float* img, const float* gt, float* dmaps, double* sums,
                            void* cuda_stream);
int32_t rgs_ssim_l1_backward(int32_t planes, int32_t H, int32_t W, const float* img, const float* gt, const float* dmaps,
                             float w_ssim, float w_l1, const float* upstream, float* d_img, void* cuda_stream);
/* Row-sharded form (multi-GPU, ABI 3): only SSIM-map / L1 rows [row_lo, row_hi) are counted; `img` must also hold the 5 halo rows
 * either side of that range (the neighbouring ranks' pixels; zero padding applies at the true image border only).  Backward writes
 * d_img for the block rows covering [row_lo - 5, row_hi + 5): the halo rows receive this rank's contribution to its neighbours'
 * pixels; rows outside stay untouched (the caller zero-fills). */
int32_t rgs_ssim_l1_forward_rows(int32_t planes, int32_t H, int32_t W, int32_t row_lo, int32_t row_hi, const float* img, const float* gt,
                                 float* dmaps, double* sums, void* cuda_stream);
int32_t rgs_ssim_l1_backward_rows(int32_t planes, int32_t H, int32_t W, int32_t row_lo, int32_t row_hi, const float* img, const float* gt,
                                  const float* dmaps, float w_ssim, float w_l1, const float* upstream, float* d_img, void* cuda_stream);
int32_t rgs_normal_consistency(int32_t H, int32_t W, int32_t from_depth, float inv_fx, float inv_fy, float cx, float cy,
                               const float* rendered_normal, const float* map_expected, const float* map_median,
                               float w_expected, float w_median, double* loss_sum, float* d_normal, float* d_expected,
                               float* d_median, void* cuda_stream);
/* Row-sharded form (multi-GPU, ABI 3): rgs_normal_consistency for loss rows [row_lo, row_hi) of an H x W image, 0 <= row_lo <=
 * row_hi <= H.  Every buffer is a window of whole rows, planar [C, rows, W]:
 *   map_expected, map_median  rows [max(0, row_lo - 2), min(H, row_hi + 2))   (the stencils of the range and one row beyond)
 *   rendered_normal           rows [max(0, row_lo - 1), min(H, row_hi + 1))
 *   d_normal, d_expected, d_median                                             rows [row_lo, row_hi), fully written
 * Rays, the image border (the outermost pixels keep a zero normal: error 1) and every stencil use the GLOBAL row index.  A pixel's
 * gradient is complete: the stencils one row outside the range that read it are evaluated here too (their loss is not counted),
 * so no gradient crosses a slab boundary.  Every per-pixel output is bit-identical to the whole-image call's value at that pixel;
 * loss_sum (zeroed by the call) sums the range's rows and differs from the whole image's rows' sum in summation order only.
 * row_lo == row_hi launches nothing and leaves loss_sum = 0. */
int32_t rgs_normal_consistency_rows(int32_t H, int32_t W, int32_t row_lo, int32_t row_hi, int32_t from_depth, float inv_fx, float inv_fy,
                                    float cx, float cy, const float* rendered_normal, const float* map_expected, const float* map_median,
                                    float w_expected, float w_median, double* loss_sum, float* d_normal, float* d_expected,
                                    float* d_median, void* cuda_stream);

/* ---- decoupled-appearance L1 loss (train.py:37-58 with GOF's AppearanceNetwork, scene/appearance_network.py) ----
 * The image is planar fp32 [3, H0, W0], H0, W0 >= 32.  The crop is H = H0 / 32 * 32 rows by W = W0 / 32 * 32 columns at
 * top = H0 / 2 - H / 2, left = W0 / 2 - W / 2.  The network's head (conv1, up1..up4) is rgs_appearance_head_* below; these
 * functions run the rest.  up4 is the head's output [16, H/2, W/2].  w2 [16,16,3,3], b2 [16], w3 [3,16,3,3], b3 [3] are conv2 and conv3.  All
 * arithmetic is fp32 (FFMA, no tensor cores); sums are fixed-order, so every output is bit-reproducible from run to run.
 *
 * rgs_appearance_downsample: down [3, H/32, W/32] = bilinear, align_corners=True, of the crop.  Source index = s * dst in fp32
 *   with s = (in - 1) / (out - 1) in fp32, or 0 when out == 1 (torch's rule); taps i0 = (int)src and i0 + 1 (i0 itself at
 *   the last input row), weights 1 - l and l with l = src - i0.
 * rgs_appearance_downsample_backward: d_image += the transpose of that map applied to d_down (read-modify-write: the taps of
 *   different samples are disjoint).  No host synchronisation.
 * rgs_appearance_l1_forward: X = up4 upsampled x2 (bilinear, align_corners=True, same index rule) to [16, H, W];
 *   A = relu(conv2(X) + b2); M = sigmoid(conv3(A) + b3) = 1 / (1 + exp(-s)); both convolutions 3x3 with zero padding at the
 *   crop's border.  loss[0] = mean over the 3 H W crop elements of |M * crop(image) - crop(gt)|, summed per CTA in fp32 per
 *   tile, across tiles and CTAs in fp64, in a fixed order.  act [16, H, W] (NULL when no backward follows) receives A;
 *   transformed [3, H, W] (may be NULL) receives M * crop(image).  partials: RGS_APPEARANCE_CTAS doubles of scratch.
 * rgs_appearance_l1_backward: the gradients of upstream * loss, upstream a DEVICE scalar (NULL: 1).  d_image [3, H0, W0] is fully
 *   written: sgn(t - gt) * (upstream / (3 H W)) * M inside the crop (sgn(0) = 0), zero outside; the downsample's share is added
 *   afterwards by rgs_appearance_downsample_backward.  d_up4 [16, H/2, W/2] goes through sigmoid' = M (1 - M), conv3^T, the ReLU
 *   mask (A > 0), conv2^T and the upsample's transpose as a gather.  d_w2, d_b2, d_w3, d_b3 are the weight and bias gradients:
 *   each of RGS_APPEARANCE_CTAS CTAs owns a fixed set of tiles and writes one fp64 row of RGS_APPEARANCE_GRAD_FLOATS partial sums
 *   into partials; the rows are summed in row order.  act is forward's output.  d_x: [16, H, W] floats of scratch. */
#define RGS_APPEARANCE_CTAS 264
#define RGS_APPEARANCE_GRAD_FLOATS 2755
int32_t rgs_appearance_downsample(int32_t H0, int32_t W0, const float* image, float* down, void* cuda_stream);
int32_t rgs_appearance_downsample_backward(int32_t H0, int32_t W0, const float* d_down, float* d_image, void* cuda_stream);
int32_t rgs_appearance_l1_forward(int32_t H0, int32_t W0, const float* image, const float* gt, const float* up4, const float* w2, const float* b2,
                                  const float* w3, const float* b3, float* act, float* transformed, double* partials, float* loss, void* cuda_stream);
int32_t rgs_appearance_l1_backward(int32_t H0, int32_t W0, const float* image, const float* gt, const float* up4, const float* act, const float* w2,
                                   const float* w3, const float* b3, const float* upstream, float* d_image, float* d_up4, float* d_w2, float* d_b2,
                                   float* d_w3, float* d_b3, double* partials, float* d_x, void* cuda_stream);
/* Row-sharded forms (multi-GPU; added functions, ABI 4).  A slab holds IMAGE rows [row_lo, row_hi), 0 <= row_lo <= row_hi <= H0;
 * its crop rows are [c0, c1) = clamp([row_lo - top, row_hi - top), 0, H).  Every buffer is a window of whole rows, planar.  The
 * whole-image functions above are these over [0, H0): the same kernels, tiles and CTAs, hence the same bits.
 * Ownership partitions the rows of the maps the head exchanges (a slab may own none):
 *   low-res row oy   the slab whose crop rows hold its upper tap (int)(s * oy) (the downsample's fp32 rule above)
 *   up4 row u        the slab whose crop rows hold 2u
 * Halos, from the x2 upsample's tap rule: sy = (H/2 - 1) / (H - 1) < 1/2, so crop row y taps up4 rows within [(y - 2) / 2,
 * (y + 2) / 2]; the gather of up4 row u reads d_x rows [2u - 2, 2u + 2].  With the owned u's, d_x is needed on crop rows
 * [c0 - 2, c1 + 2), d(conv2) on [c0 - 3, c1 + 3), the loss derivative (image, gt) on [c0 - 4, c1 + 4) and act on [c0 - 5, c1 + 5),
 * each clipped to the crop, and each empty when c0 == c1.
 *
 * rgs_appearance_row_windows: windows[RGS_APPEARANCE_WINDOWS] = {c0, c1, oy_lo, oy_hi, u_lo, u_hi, act_lo, act_hi, dx_lo, dx_hi,
 *   img_lo, img_hi}: the counted crop rows, the owned low-res and up4 rows, and the crop rows of act, d_x and of the image / gt
 *   rows backward reads.  Host only.
 * rgs_appearance_downsample_rows: down [3, oy_hi - oy_lo, w] = the owned low-res rows, each bit-identical to the whole map's.
 *   image holds image rows [image_lo, image_lo + image_rows) of the render, inside the image and holding crop rows
 *   [c0, min(c1 + 1, H)) (the taps reach at most one row below the slab).
 * rgs_appearance_l1_forward_rows: image and gt are windows of the same rows [image_lo, image_lo + image_rows), holding crop rows
 *   [c0, c1).  up4 is the whole head output.  act [16, act_hi - act_lo, W] receives A on crop rows [act_lo, act_hi).  loss_sum[0]
 *   (fp64, not divided) = the sum of |M * crop - gt| over crop rows [c0, c1), in the whole call's order (fp32 per tile, fp64
 *   over the tiles of each of RGS_APPEARANCE_CTAS CTAs, then over the CTAs); partials: RGS_APPEARANCE_CTAS doubles of scratch.
 *   The loss of the whole image is (float)(sum over slabs of loss_sum / (3 H W)).
 * rgs_appearance_l1_backward_rows: image and gt windows as in forward, holding crop rows [img_lo, img_hi); act is forward's.
 *   d_image [3, row_hi - row_lo, W0], fully written: the slab's rows of the whole call's d_image (zero outside the crop),
 *   bit-identical.  d_up4 [16, u_hi - u_lo, W/2] = the owned up4 rows of the whole call's d_up4, bit-identical: d_x is computed
 *   completely on crop rows [dx_lo, dx_hi), which evaluates the loss derivative also at halo pixels whose loss a neighbour
 *   counts.  grad_row [RGS_APPEARANCE_GRAD_FLOATS] (fp64, not cast): dW2 [16,16,3,3], db2 [16], dW3 [3,16,3,3], db3 [3] over
 *   crop rows [c0, c1), summed per CTA over its tiles and then over the CTAs in order.  partials: RGS_APPEARANCE_CTAS x
 *   RGS_APPEARANCE_GRAD_FLOATS doubles, d_x: 16 x (dx_hi - dx_lo) x W floats, both scratch.
 * rgs_appearance_downsample_backward_rows: d_image [3, row_hi - row_lo, W0] += the taps of the whole d_down [3, h, w] that
 *   land in rows [row_lo, row_hi), in the whole call's order: each element gets the whole call's bits.
 * A slab without crop rows launches no kernel: loss_sum = 0, grad_row = 0, d_image = 0. */
#define RGS_APPEARANCE_WINDOWS 12
int32_t rgs_appearance_row_windows(int32_t H0, int32_t W0, int32_t row_lo, int32_t row_hi, int32_t* windows);
int32_t rgs_appearance_downsample_rows(int32_t H0, int32_t W0, int32_t row_lo, int32_t row_hi, const float* image, int32_t image_lo, int32_t image_rows,
                                       float* down, void* cuda_stream);
int32_t rgs_appearance_downsample_backward_rows(int32_t H0, int32_t W0, int32_t row_lo, int32_t row_hi, const float* d_down, float* d_image,
                                                void* cuda_stream);
int32_t rgs_appearance_l1_forward_rows(int32_t H0, int32_t W0, int32_t row_lo, int32_t row_hi, const float* image, const float* gt, int32_t image_lo,
                                       int32_t image_rows, const float* up4, const float* w2, const float* b2, const float* w3, const float* b3, float* act,
                                       double* partials, double* loss_sum, void* cuda_stream);
int32_t rgs_appearance_l1_backward_rows(int32_t H0, int32_t W0, int32_t row_lo, int32_t row_hi, const float* image, const float* gt, int32_t image_lo,
                                        int32_t image_rows, const float* up4, const float* act, const float* w2, const float* w3, const float* b3,
                                        const float* upstream, float* d_image, float* d_up4, double* grad_row, double* partials, float* d_x,
                                        void* cuda_stream);
/* The network's head (added functions, ABI 4): conv1 (67 -> 256) + ReLU, then up1..up4, each PixelShuffle(2) (torch's rule
 * out[c][2y+i][2x+j] = in[4c+2i+j][y][x]), a 3x3 convolution (64 -> 128, 32 -> 64, 16 -> 32, 8 -> 16) and a ReLU, every
 * convolution with zero padding at its own map's border.  h = H/32, w = W/32 >= 1 (h w <= 2^18).  conv1's input is down
 * [3, h, w] (rgs_appearance_downsample's output) followed by the 64-float embedding row on every pixel, zero in the padding ring
 * as in the concatenated input; neither it nor any shuffled map is materialised.  The ten parameters have torch's layouts:
 * w1 [256,67,3,3], b1 [256], wu1 [128,64,3,3], bu1 [128], wu2 [64,32,3,3], bu2 [64], wu3 [32,16,3,3], bu3 [32], wu4 [16,8,3,3],
 * bu4 [16].  All arithmetic is fp32 FFMA (no tensor cores, no TF32), every sum has a fixed order and there are no float atomics:
 * every output is bit-reproducible from run to run, whatever torch's cuDNN and TF32 settings.
 *
 * rgs_appearance_head_forward: act [RGS_APPEARANCE_HEAD_ACT_PER_HW h w] receives the post-ReLU outputs of conv1 [256, h, w],
 *   up1 [128, 2h, 2w], up2 [64, 4h, 4w] and up3 [32, 8h, 8w], back to back; up4 [16, 16h, 16w] the head's output.
 * rgs_appearance_head_backward: from d_up4 [16, 16h, 16w] (rgs_appearance_l1_backward's) and forward's act and up4: each layer's
 *   ReLU mask (output > 0), the data gradient (the flipped-weight convolution, then the inverse shuffle) and the weight and
 *   bias gradients.  d_down [3, h, w] is conv1's input gradient on the image channels (for rgs_appearance_downsample_backward);
 *   d_emb [64] is its sum over every pixel on channels 3..66: fp32 over pixels t, t + 256, ... for each of 256 partial sums,
 *   which are added in order in fp64, one cast.  d_w*, d_b* have the parameters' layouts: each layer's map is cut into tiles of
 *   4 x 32 pixels (up4: 8 x 32) and the tiles, in row-major order, into bands; within a band each weight's and each bias's sum
 *   runs in fp32 over the tiles in order, within a tile over rows g, g + G, ... for each of G pixel groups (G = 1 for conv1..up2,
 *   2 for up3, 8 for up4) and over the columns in order, the groups added in group order; the bands are added in band order in
 *   fp64, one cast.  scratch: rgs_appearance_head_scratch_bytes.
 * rgs_appearance_head_scratch_bytes: the backward's scratch for an h x w head input (host only): the fp64 band rows (at most
 *   16 MB) plus 3072 h w floats, 37.6 MB at h, w = 37, 50 (1600 x 1200). */
#define RGS_APPEARANCE_HEAD_ACT_PER_HW 3840
int32_t rgs_appearance_head_scratch_bytes(int32_t h, int32_t w, size_t* bytes);
int32_t rgs_appearance_head_forward(int32_t h, int32_t w, const float* down, const float* emb, const float* w1, const float* b1, const float* wu1,
                                    const float* bu1, const float* wu2, const float* bu2, const float* wu3, const float* bu3, const float* wu4,
                                    const float* bu4, float* act, float* up4, void* cuda_stream);
int32_t rgs_appearance_head_backward(int32_t h, int32_t w, const float* down, const float* emb, const float* w1, const float* wu1, const float* wu2,
                                     const float* wu3, const float* wu4, const float* act, const float* up4, const float* d_up4, float* d_down,
                                     float* d_emb, float* d_w1, float* d_b1, float* d_wu1, float* d_bu1, float* d_wu2, float* d_bu2, float* d_wu3,
                                     float* d_bu3, float* d_wu4, float* d_bu4, void* scratch, void* cuda_stream);

/* ---- initial Gaussian scales: simple_knn's distCUDA2 (reference scene/gaussian_model.py:20, :315-316) ----
 * points [P,3] (device, fp32) -> mean_dist2 [P] (device): the mean of the squared Euclidean distances from point i to its 3 nearest
 * OTHER points, where "other" is decided by index (an exact duplicate of i is a neighbour at distance 0).  Exact in fp32: every pair
 * distance is (dx*dx + dy*dy) + dz*dz with dx = p.x - q.x etc., each operation separately rounded (no FMA contraction), and the
 * result is ((d0 + d1) + d2) / 3.0f with IEEE division over the three smallest values d0 <= d1 <= d2.  The result is therefore a pure
 * function of the multiset of neighbour distances: independent of input order, traversal order and thread count.
 * Fewer than 4 points: the mean over the P - 1 others (ascending sum / (P - 1)); a lone point gets 1.0.
 * A point with a NaN or infinite coordinate is nobody's neighbour and gets NaN; the other rows are computed as if it were absent
 * (including the small-cloud rule when fewer than 4 finite points remain).
 * Scratch memory comes through `scratch` (about 60 bytes per point).  One stream synchronisation inside.  P == 0 returns 0 without
 * any CUDA call; P < 0 or a NULL pointer with P > 0 returns RGS_E_INVALID. */
int32_t rgs_knn_mean_dist2(int32_t P, const float* points, float* mean_dist2, rgs_resize_fn scratch, void* scratch_user, void* cuda_stream);

/* ---- TSDF fusion and marching cubes on a sparse voxel-block grid (reference mesh_extract.py:66-105, there Open3D's
 * VoxelBlockGrid on the CPU) ----
 * Every value the functions below store is fixed bit for bit by this contract; every arithmetic step is one IEEE fp32
 * operation rounded on its own (no FMA contraction), in the order written.  Open3D's own rules (pixel rounding, image-border
 * test, touch shape, triangle table) are not known here: where this contract chooses, it says so; bit parity with Open3D is
 * not a goal.
 *
 * Grid.  Voxels form blocks of 16^3 (RGS_TSDF_BLOCK_RES; no other resolution).  Grid point g = 16 * block + local (integer
 * vectors, 0 <= local < 16) sits at the world point (float)g_k * voxel_size per component k.  Inside a block the voxels are
 * stored x fastest: v = x + 16 y + 256 z, so a pool seen as [capacity, 16, 16, 16, C] is indexed [block, z, y, x, c].
 * A block key packs the block coordinate with 21 bits per axis: key = (bx + 2^20) << 42 | (by + 2^20) << 21 | (bz + 2^20),
 * -2^20 <= b < 2^20, so ascending keys are ascending (bx, by, bz).  The hash is open addressing with linear probing over
 * `hash_slots` (a power of two); a free slot holds key RGS_TSDF_EMPTY_KEY and value -1.  Blocks are never freed.
 *
 * Camera (rgs_tsdf_camera).  The caller converts its parameters to fp32 once: fx, fy, cx, cy and the world->camera
 * extrinsic [R | t] (R row-major).  trunc = trunc_voxel_multiplier * voxel_size (one fp32 product).  A call whose camera
 * centre c = -R^T t (evaluated in double) has some c_k +- (depth_max + trunc) outside the key range (blocks
 * [-2^20 + 1, 2^20 - 2]) returns RGS_E_INVALID; a pixel whose touched blocks would still leave the range (very wide fields
 * of view) touches nothing, so keys never wrap and every grid point is an exact fp32 integer times voxel_size.
 *
 * Touch (rgs_tsdf_touch; Open3D compute_unique_block_coordinates).  Pixel (i, j) (column, row) is valid when
 * 0 < d <= depth_max, d = depth[j, i] / depth_scale.  Its ray through the pixel centre: xn = ((i + 0.5) - cx) / fx,
 * yn = ((j + 0.5) - cy) / fy; for z in {d - trunc, d + trunc} the camera point is (xn * z, yn * z, z), q = p_c - t and
 * p_w,k = (R_0k q.x + R_1k q.y) + R_2k q.z; its block coordinate is floor(p_w,k / (16 * voxel_size)).  Every block of the
 * axis-aligned box spanned by the two block coordinates is touched (a box, not a DDA walk; with the default multiplier 8 at
 * most 2 x 2 x 2).  The result is the set of touched blocks in ascending key order.
 *
 * Integrate (rgs_tsdf_integrate; Open3D integrate).  The given blocks are inserted first (a new block's voxels are the
 * zeros the caller filled the pools with).  Then each voxel of those blocks, at p = g * voxel_size, is updated by exactly
 * one thread, so the grid does not depend on scheduling, block order or duplicate coordinates:
 *   x_c = ((R_00 p.x + R_01 p.y) + R_02 p.z) + t_0 (likewise y_c, z_c);  u = (fx * x_c) / z_c + cx,  v = (fy * y_c) / z_c + cy;
 *   pixel (floor u, floor v), accepted iff it lies in [0, W) x [0, H) (chosen: the pixel whose square contains (u, v));
 *   skipped when z_c <= 0, the pixel is not accepted, d <= 0, d > depth_max or sdf = d - z_c < -trunc;
 *   otherwise obs = min(sdf, trunc) / trunc, tsdf <- (w * tsdf + obs) / (w + 1), each colour channel
 *   col <- (w * col + c) / (w + 1) with c the float colour as given, then w <- w + 1.
 *
 * Extract (rgs_tsdf_extract; Open3D extract_triangle_mesh).  A voxel is valid when it is allocated and w >= weight_threshold;
 * it is inside when tsdf < 0 (0 is outside).  The cell at g (corners g + {0,1}^3, corner c = cx + 2 cy + 4 cz, case bit c set
 * when corner c is inside) emits triangles iff its 8 corners are valid.  Edge e of a cell runs along axis a = e / 4 from the
 * corner offset by (e & 1, e >> 1 & 1) on the other two axes in ascending axis order; its vertex belongs to grid point
 * g + offset, and the vertex of (g, a) sits at g * voxel_size with component a advanced: g_a * vs + t * vs,
 * t = f0 / (f0 - f1), colour c0 + t * (c1 - c0) (0: g, 1: g + e_a).  A vertex exists iff an emitted triangle uses it.
 * Triangle table, derived by rule (rgs_tsdf.cu, constexpr): on each cube face the sign-change edges are joined by segments
 * (on a face whose diagonal corners share a sign, each inside corner is cut off by its own segment); every segment is
 * directed so that direction x (outward face normal) points to the inside corner of its first edge; the directed segments
 * form closed loops; each loop is walked from its lowest-numbered edge e0 -> e1 -> ... and fanned as (e0, e_k, e_k+1).  The
 * right-hand normal of every triangle then points toward increasing tsdf, and two cells agree on their shared face, so the
 * mesh over fully valid cells is watertight.  Order: active blocks by key; vertices by (block, voxel, axis); triangles by
 * (block, voxel, table order).  The mesh is therefore the same bits for every run and every grid capacity.
 *
 * Normals (rgs_tsdf_vertex_normals; Open3D compute_vertex_normals).  n_f = (v1 - v0) x (v2 - v0), each component
 * a.y * b.z - a.z * b.y etc. rounded per operation; each vertex sums n_f over its triangles in ascending triangle index from
 * (0, 0, 0), then n / sqrtf((n.x n.x + n.y n.y) + n.z n.z) (IEEE sqrt and division); a zero length gives (0, 0, 0).
 *
 * Memory.  The library allocates nothing persistent: the caller owns every array of rgs_tsdf_grid and grows it on the host.
 * counters[0] = allocated blocks, counters[1] = blocks of the last touch, counters[2] = RGS_TSDF_* flags (sticky).  Growth:
 * allocate pools of twice the capacity (old contents copied to the front, the rest zero), a new hash (all free), call
 * rgs_tsdf_rehash, keep the counters.  rgs_tsdf_touch's read of the counters (the one host read per view) returns the
 * allocated count: a caller that keeps allocated + blocks passed to integrate <= capacity never overflows.  A block that
 * finds no slot is skipped and sets RGS_TSDF_OVERFLOW, which every later call that reads the counters reports. */
#define RGS_TSDF_BLOCK_RES 16
#define RGS_TSDF_EMPTY_KEY 0xffffffffffffffffull
#define RGS_TSDF_OVERFLOW 1          /* counters[2]: a block found no pool slot (grid state incomplete) */
#define RGS_TSDF_BAD_COORD 2         /* counters[2]: integrate got a block coordinate outside the key range */
typedef struct rgs_tsdf_grid {
	float voxel_size;
	int64_t capacity;           /* blocks the pools hold                                                              */
	int64_t hash_slots;         /* power of two, >= 2 * capacity                                                      */
	uint64_t* hash_keys;        /* [hash_slots]                                                                       */
	int32_t* hash_values;       /* [hash_slots] pool index of the block                                               */
	float* tsdf;                /* [capacity * 4096]                                                                  */
	float* weight;              /* [capacity * 4096]                                                                  */
	float* color;               /* [capacity * 4096 * 3]                                                              */
	int32_t* stamps;            /* [capacity] last integrate call that claimed the block (start at 0)                 */
	int64_t frame_slots;        /* power of two: touch's frame-local hash                                             */
	uint64_t* frame_keys;       /* [frame_slots]                                                                      */
	uint64_t* frame_list;       /* [frame_slots / 2]                                                                  */
	int32_t* counters;          /* [4] see above                                                                      */
} rgs_tsdf_grid;

typedef struct rgs_tsdf_camera {
	int32_t width, height;
	float fx, fy, cx, cy;
	float R[9];                 /* world -> camera rotation, row-major */
	float t[3];
	float depth_scale, depth_max, trunc_voxel_multiplier;
} rgs_tsdf_camera;

/* depth [H, W] fp32.  Writes the touched blocks in ascending key order to block_coords (int32 [frame_slots / 2, 3]) and
 * returns their count, or RGS_E_CAPACITY / another negative status.  allocated (host, may be NULL) receives counters[0].
 * Scratch through `scratch`.  One stream synchronisation inside. */
int64_t rgs_tsdf_touch(const rgs_tsdf_grid* grid, const rgs_tsdf_camera* cam, const float* depth, int32_t* block_coords, int64_t* allocated,
                       rgs_resize_fn scratch, void* scratch_user, void* cuda_stream);
/* block_coords int32 [n, 3] (device), depth [H, W], color [H, W, 3] fp32.  call_id > 0, different for every call on the
 * grid.  Scratch through `scratch`.  No host synchronisation. */
int32_t rgs_tsdf_integrate(const rgs_tsdf_grid* grid, const rgs_tsdf_camera* cam, int64_t n, const int32_t* block_coords, const float* depth,
                           const float* color, int32_t call_id, rgs_resize_fn scratch, void* scratch_user, void* cuda_stream);
/* Inserts every allocated block of the old hash into grid's (empty) hash with its pool index. */
int32_t rgs_tsdf_rehash(const rgs_tsdf_grid* grid, const uint64_t* old_keys, const int32_t* old_values, int64_t old_slots, void* cuda_stream);
/* Active blocks in ascending key order: keys and pool indices (capacity entries each).  Returns the count.  One stream
 * synchronisation inside. */
int64_t rgs_tsdf_active_blocks(const rgs_tsdf_grid* grid, uint64_t* keys, int32_t* pool_index, rgs_resize_fn scratch, void* scratch_user,
                               void* cuda_stream);
/* Marching cubes.  The outputs come through `resize` with these user pointers: vertices fp32 [V, 3], colors fp32 [V, 3],
 * triangles int32 [F, 3]; V and F are written to num_vertices / num_triangles (host).  Two stream synchronisations inside. */
typedef struct rgs_tsdf_mesh_out {
	void* vertices_user;
	void* colors_user;
	void* triangles_user;
	int64_t num_vertices, num_triangles;
} rgs_tsdf_mesh_out;
int32_t rgs_tsdf_extract(const rgs_tsdf_grid* grid, float weight_threshold, rgs_resize_fn resize, rgs_tsdf_mesh_out* out, void* scratch_user,
                         void* cuda_stream);
/* normals fp32 [V, 3] of any mesh (triangle indices must lie in [0, V)).  Scratch through `scratch`. */
int32_t rgs_tsdf_vertex_normals(int64_t V, const float* vertices, int64_t F, const int32_t* triangles, float* normals, rgs_resize_fn scratch,
                                void* scratch_user, void* cuda_stream);

/* ---- bounded TSDF of the 2DGS-derived extractor (reference utils/mesh_utils.py:118-160 extract_mesh_bounded, there
 *      Open3D's legacy ScalableTSDFVolume with RGB8 colour on the CPU; :272-285 export_image) ----
 * The volume is an rgs_tsdf_grid (16^3 voxel units = the grid's blocks, same keys, hash, pools, growth and counters as
 * above); the functions below replace touch and integrate, and rgs_tsdf_extract is reused.  Every stored value is fixed
 * bit for bit; fp32 operations are rounded one by one in the order written (no FMA contraction).  Open3D is not a
 * reference here: where its rule is not known, the rule below is chosen, and bit parity with Open3D is not a goal.
 *
 * RGBD (rgs_scalable_rgbd; create_from_color_and_depth(depth_scale=1, depth_trunc, convert_rgb_to_intensity=False) of the
 * reference's np.asarray(rgb * 255, dtype=np.uint8) and its masked depth).  rgb fp32 [3, H, W] -> color uint8 [H, W, 3]:
 *   byte = B(rgb * 255.0f) (one fp32 product), B(x) = the low 8 bits of the int32 truncation of x when -2^31 < x < 2^31,
 *   else 0 (NaN included): numpy's float32 -> uint8 cast on x86-64 (cvttss2si), so 1.01 -> 1, -0.01 -> 254, NaN -> 0.
 *   depth fp32 [H, W] -> depth_out: d = 0 where mask (fp32 [H, W], may be NULL) < 0.5; then d = 0 where (double)d >=
 *   depth_trunc (chosen: >=).  NaN depth stays NaN and is skipped below, as every d <= 0.
 * Touch (rgs_scalable_touch; the legacy volume's unit allocation).  Pixels (u, v) with u, v = 0 mod 4 and d = depth[v, u]
 *   > 0: x = ((u - cx) d) / fx, y = ((v - cy) d) / fy (integer pixel coordinates), q = (x, y, d) - t, p_k = (R_0k q.x +
 *   R_1k q.y) + R_2k q.z (chosen: fp32 R^T (p - t), not a double inverse); lo_k = floor((p_k - sdf_trunc) / (16 voxel_size)),
 *   hi_k = floor((p_k + sdf_trunc) / (16 voxel_size)); every unit of the box [lo, hi] is touched (a pixel whose box leaves
 *   the key range touches nothing).  Units come back in ascending key order, with rgs_tsdf_touch's frame hash, counters and
 *   RGS_E_CAPACITY protocol.  The camera's depth_scale, depth_max and trunc_voxel_multiplier are not read; sdf_trunc is the
 *   absolute truncation (positive, finite).
 * Integrate (rgs_scalable_integrate).  The units are inserted and claimed as in rgs_tsdf_integrate; then every voxel of
 *   them, one thread each, at its centre p = ((float)g + 0.5f) voxel_size (g the integer grid point; the sum is exact for
 *   |g| < 2^23):  x_c = ((R_00 p.x + R_01 p.y) + R_02 p.z) + t_0 (likewise y_c, z_c); skipped unless z_c > 0;
 *   u = floor(((x_c / z_c) fx + cx) + 0.5), v likewise (the rounded projection), accepted iff in [0, W) x [0, H);
 *   skipped unless d = depth[v, u] > 0; xn = (u - cx) / fx, yn = (v - cy) / fy, sdf = (d - z_c) sqrtf((1 + xn xn) + yn yn)
 *   (IEEE sqrt); skipped unless sdf > -sdf_trunc; then tsdf_obs = min(1, sdf / sdf_trunc), tsdf <- (w tsdf + tsdf_obs) /
 *   (w + 1), each colour channel col <- (w col + (float)byte) / (w + 1) (fp32 on 0..255; chosen), w <- w + 1.
 *   The principal point is used as given: the reference's cx = W / 2 is half a pixel from the rasterizer's pixel centres.
 * Extract: rgs_tsdf_extract with weight_threshold = 1 (weights are whole counts, so a corner of weight 0 is invalid); the
 *   caller then adds 0.5f voxel_size to every vertex component (one fp32 addition: vertices sit on voxel centres) and
 *   divides every colour by 255.0f (one fp32 division).
 * Image export (rgs_scalable_image_u8; save_img_u8): image fp32 [3, H, W] -> out uint8 [H, W, 3],
 *   y = x scale + offset (two roundings), 0 if NaN, clipped to [0, 1], byte = (int)(y * 255.0f) (truncation).
 * No host synchronisation except rgs_scalable_touch's one counter read. */
int32_t rgs_scalable_rgbd(int32_t H, int32_t W, const float* rgb, const float* depth, const float* mask, double depth_trunc, uint8_t* color,
                          float* depth_out, void* cuda_stream);
int32_t rgs_scalable_image_u8(int32_t H, int32_t W, const float* image, float scale, float offset, uint8_t* out, void* cuda_stream);
/* depth fp32 [H, W].  unit_coords int32 [frame_slots / 2, 3]; returns the count, RGS_E_CAPACITY or another negative status. */
int64_t rgs_scalable_touch(const rgs_tsdf_grid* grid, const rgs_tsdf_camera* cam, float sdf_trunc, const float* depth, int32_t* unit_coords,
                           int64_t* allocated, rgs_resize_fn scratch, void* scratch_user, void* cuda_stream);
/* unit_coords int32 [n, 3], depth fp32 [H, W], color uint8 [H, W, 3]; call_id as rgs_tsdf_integrate. */
int32_t rgs_scalable_integrate(const rgs_tsdf_grid* grid, const rgs_tsdf_camera* cam, float sdf_trunc, int64_t n, const int32_t* unit_coords,
                               const float* depth, const uint8_t* color, int32_t call_id, rgs_resize_fn scratch, void* scratch_user, void* cuda_stream);

/* ---- DTU evaluation: the chamfer distances of dtu_eval/eval.py and the mask culling of evaluate_dtu_mesh.py:82-138 ----
 * All arithmetic is IEEE fp64 with every operation rounded on its own (no FMA contraction), in the order written; a - b is
 * one rounded subtraction.  Points are fp64 [N, 3] on the device, row-major.  The squared pair distance is
 * d2(p, q) = (dx*dx + dy*dy) + dz*dz with dx = p.x - q.x etc., and a distance is sqrt(d2) (IEEE sqrt); this is the value
 * scikit-learn's kd-tree reports for the same pair.  Point counts are at most 2^31 - 1.  A non-finite coordinate in a cloud
 * handed to rgs_dtu_radius_downsample or rgs_dtu_nearest returns RGS_E_INVALID (scikit-learn's fit rejects it too). */

/* Surface sampling (eval.py:54-71, sample_single_tri).  faces int32 [F, 3] index vertices fp64 [V, 3].  Per triangle, with
 * e1 = v1 - v0, e2 = v2 - v0: l1 = sqrt((e1.x^2 + e1.y^2) + e1.z^2) (likewise l2); the cross product c = e1 x e2 with
 * c.x = e1.y*e2.z - e1.z*e2.y, c.y = e1.z*e2.x - e1.x*e2.z, c.z = e1.x*e2.y - e1.y*e2.x; area2 = |c| as for l1.  A triangle
 * is sampled iff area2 > 0 (a NaN area is not).  thr = density * sqrt((l1 * l2) / area2), n1 = floor(l1 / thr),
 * n2 = floor(l2 / thr); for i = 0..n1 (outer), j = 0..n2 (inner), c0 = (i + 0.5) / max(n1, 1e-7), c1 = (j + 0.5) /
 * max(n2, 1e-7), the point q = (e1 * c0 + e2 * c1) + v0 (per component) is emitted iff c0 + c1 < 1.  The output is the V
 * vertices in order followed by the samples in triangle order: fp64 [V + S, 3] through resize(out->points_user, bytes).
 * Scratch comes through resize(out->scratch_user) (about 32 bytes per face) and resize(out->rows_user) (16 bytes per sampled
 * row).  One host read (the totals) before anything is sized by the totals; V + S > 2^31 - 1, a face index outside [0, V)
 * or a non-finite n1 / n2 returns RGS_E_INVALID before the output is requested.  num_points receives V + S.  A triangle is
 * counted by one thread in O(rows + columns) steps; the points themselves are written one thread each. */
typedef struct rgs_dtu_samples_out {
	void* points_user;
	void* scratch_user;
	void* rows_user;
	int64_t num_points;
} rgs_dtu_samples_out;
int32_t rgs_dtu_sample_mesh(int64_t V, const double* vertices, int64_t F, const int32_t* faces, double density, rgs_resize_fn resize,
                            rgs_dtu_samples_out* out, void* cuda_stream);

/* Radius downsample (eval.py:80-94).  points fp64 [N, 3] in their processing order (the reference's shuffled order).
 * kept[i] (uint8) = 1 iff point i lies within `radius` (d2 <= radius * radius, the product rounded once) of no kept point
 * j < i: the greedy, lexicographically first maximal independent set in index order, which is what the reference's loop
 * over radius_neighbors computes.  The result does not depend on thread count or scheduling.  radius must be positive and
 * finite.  Scratch through `scratch` (about 200 bytes per point).  One host read per round; rounds (host, may be NULL)
 * receives their number: at most the length of the longest chain of neighbours with increasing index, polylogarithmic in N
 * for a random order. */
int32_t rgs_dtu_radius_downsample(int64_t N, const double* points, double radius, uint8_t* kept, int32_t* rounds, rgs_resize_fn scratch,
                                  void* scratch_user, void* cuda_stream);

/* Exact 1-NN distances (eval.py:118-134, kneighbors(n_neighbors=1)).  For each query q: dist = sqrt(min_p d2(q, p)) over
 * the M reference points, and index = the index of a reference point attaining it (which one among ties is unspecified).
 * M >= 1 (an empty reference set returns RGS_E_INVALID); N may be 0.  Scratch through `scratch` (about 90 bytes per
 * reference point and 24 per query).  One host read (the bounds). */
int32_t rgs_dtu_nearest(int64_t M, const double* reference, int64_t N, const double* query, double* dist, int64_t* index, rgs_resize_fn scratch,
                        void* scratch_user, void* cuda_stream);

/* Mask dilation (evaluate_dtu_mesh.py:120-122, skimage binary_dilation(mask, disk(6))).  masks uint8 [n_views, H, W]
 * (nonzero = set) -> dilated uint8 [n_views, H, W]: 1 iff a set pixel lies at (dx, dy) with dx^2 + dy^2 <= 36 (113 pixels);
 * pixels outside the image are unset.  No host synchronisation. */
int32_t rgs_dtu_dilate_masks(int32_t n_views, int32_t H, int32_t W, const uint8_t* masks, uint8_t* dilated, void* cuda_stream);

/* Vertex culling (evaluate_dtu_mesh.py:82-133).  proj fp64 [n_views, 3, 4] holds rows 0..2 of K @ w2c per view, with K the
 * reference's 4x4 intrinsic (fx, fy, W / 2, H / 2) and w2c its world_view_transform.T.  Per vertex and view:
 * c_r = ((P_r0 x + P_r1 y) + P_r2 z) + P_r3; u = (c_0 / (c_2 + 1e-6)) / (W - 1), v likewise with H - 1; gx = (u - 0.5) * 2,
 * gy = (v - 0.5) * 2.  The view is passed when not (-1 < gx < 1 and -1 < gy < 1); otherwise the dilated mask is read at
 * column rint(((gx + 1) / 2) * (W - 1)), row rint(((gy + 1) / 2) * (H - 1)) (grid_sample nearest with align_corners, ties
 * to even) and the view is passed iff it is set.  keep uint8 [V] = 1 iff every view is passed.  No host synchronisation. */
int32_t rgs_dtu_cull_vertices(int64_t V, const double* vertices, int32_t n_views, int32_t H, int32_t W, const double* proj, const uint8_t* dilated,
                              uint8_t* keep, void* cuda_stream);

/* ---- Tanks and Temples evaluation: eval_tnt/run.py, registration.py and evaluation.py without Open3D ----
 * The DTU block's arithmetic rules hold: IEEE fp64, every operation rounded on its own in the order written (no FMA
 * contraction), points fp64 [N, 3] on the device, counts at most 2^31 - 1, and a non-finite input returns RGS_E_INVALID.
 * Correspondences and distances come from rgs_dtu_nearest.
 *
 * A transform is a HOST pointer to 16 doubles, the 4x4 matrix row-major; its last row must be exactly (0 0 0 1) and every
 * entry finite, else RGS_E_INVALID.  It maps p to p' with p'_r = ((T_r0 * x + T_r1 * y) + T_r2 * z) + T_r3 (no division by
 * the homogeneous coordinate, which is 1).  NULL means no transform: the points are copied unchanged. */

/* Polygon crop volume (Open3D's SelectionPolygonVolume): orthogonal_axis 0 / 1 / 2 for X / Y / Z; the polygon's two
 * coordinates (u, v) are the remaining axes in increasing order ((y, z), (x, z), (x, y)).  polygon is DEVICE fp64 [K, 2],
 * 3 <= K <= 2048, vertex k joined to vertex (k + 1) mod K.  A point w = p[orthogonal_axis] is kept iff
 * axis_min <= w <= axis_max (inclusive at both ends) and (u, v) passes the crossing-number test: for each edge (a, b) with
 * a.v < v <= b.v or b.v < v <= a.v (half-open, so a horizontal edge never counts and a vertex is counted once), the
 * crossing x = a.u + ((v - a.v) * (b.u - a.u)) / (b.v - a.v) is counted iff x < u; the point is inside iff the count is
 * odd.  Open3D's own boundary rule was not available to confirm this one: points exactly on an edge or a vertex may be
 * decided differently there. */
typedef struct rgs_tnt_crop_volume {
	int32_t orthogonal_axis;
	int32_t num_vertices;
	double axis_min, axis_max;
	const double* polygon;
} rgs_tnt_crop_volume;

/* Transform, then crop (registration.py:113-131, evaluation.py:75-89).  points fp64 [N, 3]; transform host [16] or NULL;
 * volume (host struct) or NULL for no crop (every point kept).  kept uint8 [N] receives the mask over the transformed
 * points; cropped fp64 [N, 3] receives the kept transformed points compacted in input order, *num_kept (host) their count.
 * One thread per point with the polygon in shared memory, then CUB's stable DeviceSelect; one host read.  Scratch through
 * `scratch` (about 40 bytes per point). */
int32_t rgs_tnt_crop(int64_t N, const double* points, const double* transform, const rgs_tnt_crop_volume* volume, uint8_t* kept, double* cropped,
                     int64_t* num_kept, rgs_resize_fn scratch, void* scratch_user, void* cuda_stream);

/* In-place transform (Open3D's PointCloud::Transform, applied by the ICP after every update).  points fp64 [N, 3] are
 * overwritten with T p as above.  No host synchronisation and no finiteness check of the points. */
int32_t rgs_tnt_transform(int64_t N, double* points, const double* transform, void* cuda_stream);

/* Voxel downsample (Open3D's VoxelDownSample).  origin = min_bound - voxel * 0.5 per axis (min_bound over all points);
 * a point's voxel index per axis is floor((p - origin) / voxel), and the key (ix << 42) | (iy << 21) | iz.  When an axis
 * needs more than 2^21 cells (floor((max_bound - origin) / voxel) >= 2^21) the call returns RGS_E_INVALID after one bounds
 * pass, before any output or the sort scratch is requested.  Each voxel's mean is its sum ((0 + p_0) + p_1) + ... over its
 * points in input order, divided by the count: the same sum Open3D's AccumulatedPoint forms, so each value matches it bit
 * for bit.  Output in ascending key order (Open3D's is its hash map's): means fp64 [V, 3] through
 * resize(out->means_user), counts int64 [V] through resize(out->counts_user); out->num_voxels receives V.  voxel must be
 * positive and finite.  Scratch through resize(out->scratch_user): first 64 bytes (the bounds), then about 48 bytes per
 * point.  Two host reads (the bounds, the voxel count).  One warp per voxel adds its points in order, so a voxel of 10^5
 * points occupies one warp and not the launch. */
typedef struct rgs_tnt_voxel_out {
	void* means_user;
	void* counts_user;
	void* scratch_user;
	int64_t num_voxels;
} rgs_tnt_voxel_out;
int32_t rgs_tnt_voxel_downsample(int64_t N, const double* points, double voxel, rgs_resize_fn resize, rgs_tnt_voxel_out* out, void* cuda_stream);

/* Moments of the scaled point-to-point ICP (Open3D's TransformationEstimationPointToPoint(true), Eigen's umeyama).
 * source fp64 [N, 3] (already transformed), target fp64 [M, 3], dist fp64 [N] and index int64 [N] from
 * rgs_dtu_nearest(target, source).  Source point i corresponds to target point index[i] iff dist[i] < threshold (strict,
 * as nanoflann's radius search; Open3D was not available to confirm it).  moments (HOST fp64 [19]) receives
 *   [0] n, the correspondence count;  [1] the sum of d2(s_i, t_index[i]) over correspondences (d2 as rgs_dtu_nearest);
 *   [2..4] ms = S_s * (1 / n);  [5..7] mt = S_t * (1 / n), with S the sums of the corresponding points;
 *   [8..16] sigma = (1 / n) * sum (t - mt)(s - ms)^T, row-major;  [17] var_s = (1 / n) * sum ((sx^2 + sy^2) + sz^2) with s
 *   the centred source point;  [18] 0 (the count of non-finite inputs: nonzero returns RGS_E_INVALID).
 * Two passes (means, then centred sums), each reduced in a fixed tree: block b sums points [1024 b, 1024 b + 1024), thread
 * t its points 1024 b + t + 256 k for k = 0..3 in that order from 0.0, then a halving tree over the 256 threads (slot t
 * += slot t + s for s = 128, 64, .., 1); one block then sums the block results the same way (thread t: results t,
 * t + 256, .. in order).  The shape depends on N only, so repeated calls return identical bits; no floating-point
 * atomics.  With n = 0 every entry is 0.  Scratch through `scratch` (about 0.1 byte per point).  One host read. */
int32_t rgs_tnt_icp_moments(int64_t N, const double* source, int64_t M, const double* target, const double* dist, const int64_t* index, double threshold,
                            double* moments, rgs_resize_fn scratch, void* scratch_user, void* cuda_stream);

/* ---- Tanks and Temples mesh cull (reference eval_tnt/cull_mesh.py: extract_depth_from_mesh, Mesher.point_masks) ----
 * Every operation below is one IEEE fp32 operation rounded to nearest on its own, in the order written (no contraction);
 * so every output bit is fixed.  w2c (host, fp32 [12]) is rows 0..2 of the world-to-camera matrix, row-major; the Python
 * layer (rade_gs_b200.tnt_cull) forms it as the fp64 inverse of the fp32-rounded 4x4 pose, rounded to fp32.  A point p
 * maps to camera coordinates X_r = ((m_r0 x + m_r1 y) + m_r2 z) + m_r3.  The camera looks down +Z (OpenCV): pixel column
 * u = fx X / Z + cx, row v = fy Y / Z + cy, the model of pyrender's IntrinsicsCamera.
 *
 * rgs_tnt_mesh_depth: vertices fp32 [V, 3] and faces int32 [F, 3] on the device; depth fp32 [H, W] (device) receives the
 *   camera-space Z of the nearest surface at each pixel centre, 0 where nothing is drawn.  Homogeneous rasterization, with
 *   no back-face culling and no clip:
 *   - A, B, C: the face's vertices in camera coordinates.  The face draws nothing when a coordinate is not finite, when
 *     every Z < znear, when every Z > zfar, or when num = ((n_x A_x + n_y A_y) + n_z A_z) is 0 (zero-area or edge-on
 *     faces), with n = (B - A) x (C - A) and a x b = (a_y b_z - a_z b_y, a_z b_x - a_x b_z, a_x b_y - a_y b_x).
 *   - Bounding box, of the face clipped at Z = znear: for each edge (P, Q) in the order (A, B), (B, C), (C, A), the point
 *     P when P_z >= znear, then, when exactly one of P_z, Q_z is < znear, the crossing point P + s (Q - P) with
 *     s = (znear - P_z) / (Q_z - P_z), each coordinate P_i + (s (Q_i - P_i)).  Each point gives u = ((fx X) / Z) + cx and
 *     v = ((fy Y) / Z) + cy; umin..vmax their extremes clamped with fmin(fmax(., -1), W) (H for v); the box is columns
 *     max(floor(umin - 0.5), 0) .. min(ceil(umax - 0.5), W - 1), rows likewise; an empty box draws nothing.  The box only
 *     limits the pixels tested: coverage is decided by the edge functions alone.
 *   - Edge vectors, for (P, Q) = (A, B), (B, C), (C, A): c = (P + Q) x (Q - P), negated when num < 0.  Swapping P and Q
 *     negates c exactly, so two faces sharing an edge evaluate exactly opposite edge functions on it.
 *   - Pixel (x, y) of the box: dx = ((x + 0.5) - cx) / fx, dy = ((y + 0.5) - cy) / fy, e(c) = ((c_x dx) + (c_y dy)) + c_z.
 *     It is inside when for every edge e > 0, or e == 0 and c is lexicographically positive (c_x > 0, or c_x == 0 and
 *     c_y > 0, or c_x == c_y == 0 and c_z > 0): a pixel centre on a shared edge is drawn by exactly one of the two faces.
 *   - Its depth is Z = num / e(n), the ray's hit on the face's plane (perspective-correct); kept when znear <= Z <= zfar.
 *     The smallest kept Z per pixel wins (atomicMin on the bits of the positive float), so the result does not depend on
 *     launch order, thread count or the work split, and two calls give identical bits.
 *   Work split (no effect on the result): a box of at most 16 pixels is drawn by the face's own thread, one of at most
 *   4096 by one CTA, larger ones by stripes of the whole grid.
 *   Errors (RGS_E_INVALID with a message): V or F outside [0, 2^31), H or W outside [1, 32768], not 0 < znear < zfar,
 *   non-finite intrinsics or fx, fy == 0, and a face index outside [0, V) (a device flag, read after drawing: one host read
 *   per call when F > 0).  Scratch through `scratch` (8 bytes per face plus a few).
 *
 * rgs_tnt_visibility_count: points fp32 [N, 3], depth fp32 [H, W] (device, H, W >= 2), counts int32 [N] (device, added
 *   to).  Mesher.point_masks for one view, eps the occlusion margin (0.005 in the reference):
 *   - (X, Y, Z) as above; z = Z + 1e-8f; u = ((fx X) + (cx Z)) / z; v = ((fy Y) + (cy Z)) / z  (K @ cam with the zero
 *     terms dropped; torch's matmul may fuse or reorder these products, which moves u, v, z by an ulp);
 *   - in_frustum = u >= 0 and u <= W - 1 and v >= 0 and v <= H - 1 and z > 0; outside it the point is not counted;
 *   - the grid: g_x = ((u * r_w) * 2) - 1 with r_w = 1.0f / (float)(W - 1) (torch on CUDA multiplies by the fp32
 *     reciprocal of a host-scalar divisor; on the CPU it divides), g_y likewise;
 *   - grid_sample(bilinear, padding_mode='border', align_corners=True): ix = ((g_x + 1) / 2) * (W - 1), clipped to
 *     min(W - 1, max(ix, 0)), iy likewise; x0 = floor(ix), y0 = floor(iy), x1 = x0 + 1, y1 = y0 + 1; weights
 *     nw = (x1 - ix)(y1 - iy), ne = (ix - x0)(y1 - iy), sw = (x1 - ix)(iy - y0), se = (ix - x0)(iy - y0); the sample is
 *     s = 0, then s = s + D[y][x] * w for nw, ne, sw, se in that order, each corner skipped when x1 = W or y1 = H;
 *   - seen = in_frustum and (s > 0 ? z < s + eps : true); counts[n] += seen. */
int32_t rgs_tnt_mesh_depth(int64_t V, const float* vertices, int64_t F, const int32_t* faces, const float* w2c, float fx, float fy, float cx, float cy,
                           int32_t H, int32_t W, float znear, float zfar, float* depth, rgs_resize_fn scratch, void* scratch_user, void* cuda_stream);
int32_t rgs_tnt_visibility_count(int64_t N, const float* points, const float* depth, const float* w2c, float fx, float fy, float cx, float cy, int32_t H,
                                 int32_t W, float eps, int32_t* counts, void* cuda_stream);

/* ---- Tetrahedra mesh extraction: mesh_extract_tetrahedra.py, utils/tetmesh.py and GaussianModel.get_tetra_points ----
 * Arrays are fp32 / int32 / int64 on the device, row-major.  Stages 2-5 are fixed bit for bit: every fp32 operation below is
 * one IEEE operation rounded to nearest on its own (no FMA contraction unless an fma is written), in the order written;
 * x * 0.5 is exact. */

/* Tetra points (gaussian_model.py:400-429).  xyz [P, 3], scaling [P, 3] (get_scaling_with_3D_filter), rotation [P, 4] raw
 * (w, x, y, z), normalised here: n = sqrt(((w^2 + x^2) + y^2) + z^2), q = rotation / n, R as build_rotation.  s3 = scaling * 3.
 * points [9P, 3]: row 8 g + k (k = 0..7) is R (c_k * s3) + xyz_g with c_k = (2 bx - 1, 2 by - 1, 2 bz - 1), k = 4 bx + 2 by + bz
 * (trimesh.creation.box()'s vertex order, doubled); rows 8P + g are the centres xyz_g.  scales [9P] (the reference's [9P, 1]):
 * max(s3) of the Gaussian (NaN if any is NaN) at the same rows; these are exact.  The rotated corners are not bit-fixed (the
 * reference uses a batched matrix product): R c + xyz is evaluated in fp32 with contraction allowed. */
int32_t rgs_tetra_points(int64_t P, const float* xyz, const float* scaling, const float* rotation, float* points, float* scales, void* cuda_stream);

/* Cull SDF, one view (mesh_extract_tetrahedra.py:32-56, evaluage_cull_alpha).  alpha [N] and coord [N, 2] (pixel x, y) are
 * integrate()'s alpha_integrated and point_coordinate; render7 [H, W] its render[7]; gt_mask [H, W] or NULL.  Inputs are not
 * modified.  Per point:
 *   gx = (((x * 2) + 1) / (W - 1)) - 1, gy likewise with y and H;
 *   ix = (((gx + 1) * W) - 1) * 0.5, iy likewise with H (grid_sample, align_corners=False);
 *   x0 = floor(ix), y0 = floor(iy), x1 = x0 + 1, y1 = y0 + 1, wx = ix - x0, ex = 1 - wx, wy = iy - y0, ey = 1 - wy;
 *   m(x, y) = render7[y, x] * gt_mask[y, x] (render7[y, x] without a mask) when 0 <= x <= W - 1 and 0 <= y <= H - 1, else 0;
 *   v = (((ey * ex) * m(x0, y0) + (ey * wx) * m(x1, y0)) + (wy * ex) * m(x0, y1)) + (wy * wx) * m(x1, y1);
 *   if v > 0.5: final = NaN if alpha or final is NaN, else (final < alpha ? final : alpha); weight += 1.
 * final [N] (start: 1) and weight int32 [N] (start: 0) are the caller's accumulators.  No host synchronisation. */
int32_t rgs_tetra_cull_add(int64_t N, const float* alpha, const float* coord, int32_t H, int32_t W, const float* render7, const float* gt_mask,
                           float* final_alpha, int32_t* weight, void* cuda_stream);
/* sdf [N] = 0.5 - final where weight > 0, else -100.  No host synchronisation. */
int32_t rgs_tetra_cull_finish(int64_t N, const float* final_alpha, const int32_t* weight, float* sdf, void* cuda_stream);

/* Marching tetrahedra (utils/tetmesh.py, _unbatched_marching_tetrahedra).  points [N, 3], sdf [N], scales [N], tets int64
 * [T, 4].  A vertex is occupied when sdf > 0; a tet is valid when 1 to 3 of its vertices are.  Every tet index must lie in
 * [0, N): otherwise RGS_E_INVALID (found by a device flag, before any output is requested).  The edges (0,1), (0,2), (0,3),
 * (1,2), (1,3), (2,3) of the valid tets, as (min, max) pairs, are made unique; output vertex m is the m-th edge in ascending
 * (a, b) order whose endpoints differ in occupancy.  Outputs through resize: interp int64 [M, 2] = (a, b); ends [M, 2, 3] =
 * (points[a], points[b]); end_sdf [M, 2]; end_scales [M, 2].  faces int64 [F, 3] come from triangle_table[code] (code = sum of
 * 2^k over the occupied vertices k) on the tet's edge vertices: for chunk c of torch.chunk(tets, T // 2^25 + 1) when
 * T > 2^25 (one chunk otherwise), first every 1-triangle tet of the chunk in tet order (3 entries), then every 2-triangle tet
 * (6 entries, two faces).  This is the reference's order, chunk loop included.  N, T < 2^31 and 6 x (valid tets) < 2^31 - 256,
 * else RGS_E_INVALID.  Scratch through resize(out->scratch_user) (about 6 bytes per tet) and resize(out->sort_user) (about
 * 240 bytes per valid tet).  Two host reads (the valid-tet count with the index flag; M and F). */
typedef struct rgs_tetra_march_out {
	void* interp_user;
	void* ends_user;
	void* end_sdf_user;
	void* end_scales_user;
	void* faces_user;
	void* scratch_user;
	void* sort_user;
	int64_t num_vertices, num_faces;
} rgs_tetra_march_out;
int32_t rgs_tetra_marching(int64_t N, const float* points, const float* sdf, const float* scales, int64_t T, const int64_t* tets, rgs_resize_fn resize,
                           rgs_tetra_march_out* out, void* cuda_stream);

/* Bisection step (mesh_extract_tetrahedra.py:92-102).  left, right [M, 3], left_sdf, right_sdf [M] are updated in place; mid
 * [M, 3] receives the next midpoints.  With c = (l + r) * 0.5 per component: when mid_sdf [M] is given,
 * low = (mid_sdf < 0 and left_sdf < 0) or (mid_sdf > 0 and left_sdf > 0) (so 0 and NaN go right); low: left = c,
 * left_sdf = mid_sdf, else right = c, right_sdf = mid_sdf.  Then mid = (left + right) * 0.5.  mid_sdf NULL: only mid is
 * written (the first midpoints).  No host synchronisation. */
int32_t rgs_tetra_bisect(int64_t M, const float* mid_sdf, float* left, float* right, float* left_sdf, float* right_sdf, float* mid, void* cuda_stream);

/* Distance / scale filter and compaction (mesh_extract_tetrahedra.py:105-112, trimesh update_vertices then update_faces).
 * points [M, 3] (the final midpoints); ends [M, 2, 3] and end_scales [M, 2] from rgs_tetra_marching (the original edge
 * endpoints); faces int64 [F, 3] with entries in [0, M): an entry outside it returns RGS_E_INVALID (a device flag, read with
 * the counts).  With d = end0 - end1: vertex m is kept iff sqrt(fma(dz, dz, fma(dy, dy, dx*dx))) <= s0 + s1 (the fused
 * multiply-adds round once each: torch.norm's order on the CPU, which decides the ties below).  Adjacent box corners along a
 * Gaussian's longest axis are exactly s0 + s1 apart, so ties occur; torch.norm on a GPU may round them differently.  Kept vertices stay in order (also those no
 * face uses); a face is kept iff its 3 vertices are, its entries renumbered to ranks among the kept vertices, in order.
 * vertices fp32 [V', 3] and faces int64 [F', 3] through resize; counts in out.  Scratch through resize(out->scratch_user)
 * (about 16 bytes per vertex and 25 per face).  One host read. */
typedef struct rgs_tetra_filter_out {
	void* vertices_user;
	void* faces_user;
	void* scratch_user;
	int64_t num_vertices, num_faces;
} rgs_tetra_filter_out;
int32_t rgs_tetra_filter(int64_t M, const float* points, const float* ends, const float* end_scales, int64_t F, const int64_t* faces, rgs_resize_fn resize,
                         rgs_tetra_filter_out* out, void* cuda_stream);

/* ---- Delaunay tetrahedralization of the tetra points (mesh_extract_tetrahedra.py:63, cpp.triangulate) ----
 *
 * rgs_delaunay: points fp32 [N, 3] on the device -> int32 cells [T, 4] through resize(out->cells_user), the Delaunay
 * tetrahedralization of the distinct points.
 *
 * Predicates (exact on the fp64 values of the fp32 inputs).
 *   orient3d(a, b, c, d) = sign det[b - a, c - a, d - a]; a cell is positive when it is > 0.
 *   insphere(a, b, c, d, e) = -sign D5, D5 = det of the rows (x, y, z, x^2 + y^2 + z^2, 1) of a, b, c, d, e: for a
 *   positive a, b, c, d it is > 0 exactly when e lies strictly inside their circumsphere ("in conflict").
 *   Both run Shewchuk's stage-A floating-point filter first (bound (7 + 56 eps) eps, resp. (16 + 224 eps) eps, times the
 *   permanent, plus 2^-600 for underflowed products; eps = 2^-53; the file is compiled without FMA contraction).  When the
 *   filter cannot decide, the determinant is summed exactly over its monomials as a fixed-point integer: any finite fp32
 *   coordinates are in range there, and the filter neither overflows nor underflows beyond its slack for coordinates up
 *   to 2^128.  rgs_delaunay's own limit is |coordinate| <= 2^90, so that the ghosts below stay finite fp32 values.
 *   Perturbed insphere (Devillers & Teillaud 2011, the scheme of CGAL's Delaunay_triangulation_3): when insphere is 0, the
 *   five points are ranked by lexicographic (x, y, z) order and, from the largest down, the first non-zero
 *   -(-1)^i orient3d(the four points other than point i, in order) is the sign (i = 0..4 the position in (a, b, c, d, e)).
 *   The ranking depends on the coordinates only, so the cells depend on the point set, not on the input order.
 * Duplicates.  Numerically equal points (-0.0 == 0.0) count as one, represented by their smallest index; the other copies
 *   appear in no cell.
 * Ghosts.  With lo, hi the bounding box of the input, c = (lo + hi) / 2, R the smallest power of two >= max(hi - lo)
 *   (at least 2^-100) and S = D R, D = 2^30, four ghost vertices g = fl32(c + S s) for s = (1,1,1), (1,-1,-1), (-1,1,-1),
 *   (-1,-1,1) bound the points and take part in the perturbation like any point (they rank by their coordinates).  The
 *   output is every cell of Del(P u G) without a ghost vertex; each is a Delaunay cell of P.  The one difference from
 *   Del(P): a hull cell of P whose circumsphere contains a ghost is missing (only near-flat hull slivers have such spheres).
 * Output.  Every cell is positive; each row is rotated by an even permutation so that its smallest index comes first and
 *   the smallest of the other three second; rows are sorted lexicographically.  The bits do not depend on scheduling.
 *   Fewer than 4 distinct points, or coplanar points, give T = 0 (scipy raises instead).
 * Limits.  0 <= N <= RGS_DELAUNAY_MAX_POINTS; more than 2^29 cells (a face is referenced as cell << 2 | face in an int32)
 *   return RGS_E_CAPACITY.  A coordinate that is not finite or exceeds 2^90 in magnitude returns RGS_E_INVALID.  A new cell
 *   that is not positive, or a point that finds no cell, is a predicate bug: RGS_E_CUDA with a message, never a cell.
 * Memory (through resize, one user pointer each): points_user about 64 bytes per point plus the sorts' workspace;
 *   mesh_user[0] and [1] (the mesh, 56 bytes per cell, starting at 8 N + 64 cells and doubling into the other buffer when
 *   full); slab_user about 2.8 KB per nominee slot, K = min(N, 2^19) slots of 64 cells and 128 faces.  The cavities that
 *   overflow a round's slot are inserted right after it through the same claims in max(1, K / 16) slots 16 times as
 *   large; one larger still is inserted alone with the whole slab area, doubled until it fits.  sort_user about 40 bytes
 *   per cell.  Host reads: 3, plus one per round, one per large-slot pass and two per lone cavity.  Statistics: rounds;
 *   the largest cavity inserted through a slot; overflowed = the round slots that overflowed, summed over rounds (a point
 *   counts once per round it overflows in); alone = the cavities inserted alone; the mesh growths.  Building a star
 *   links its cells in O(b^2) steps of one thread for b boundary faces. */
#define RGS_DELAUNAY_MAX_POINTS (1 << 26)
typedef struct rgs_delaunay_out {
	void* cells_user;
	void* points_user;
	void* mesh_user[2];
	void* slab_user;
	void* sort_user;
	int64_t num_cells;
	int32_t rounds, max_cavity, overflowed, alone, mesh_growths;
} rgs_delaunay_out;
int32_t rgs_delaunay(int64_t N, const float* points, rgs_resize_fn resize, rgs_delaunay_out* out, void* cuda_stream);
/* The predicates above, by the same device code, on M index tuples [M, 5] (a, b, c, d, e) into points fp32 [N, 3]:
 * signs int8 [M, 3] = (orient3d(a, b, c, d), insphere(a, b, c, d, e), perturbed insphere).  An index outside [0, N) or a
 * coordinate that is not finite returns RGS_E_INVALID.  4 bytes of scratch through resize; one host read. */
int32_t rgs_delaunay_predicates(int64_t N, const float* points, int64_t M, const int32_t* tuples, int8_t* signs, rgs_resize_fn resize,
                                void* scratch_user, void* cuda_stream);

/* ---- LPIPS v0.1 with the VGG16 trunk (metric.py:74, lpipsPyTorch's LPIPS('vgg')) ----
 *
 * The two images of one pair go through together: every activation is fp32 NHWC [2, H, W, C], image x first.  The
 * stages, in the order a caller runs them: input conv, then per block its 3x3 convs, the distance of the block's last
 * ReLU (relu1_2, relu2_2, relu3_3, relu4_3, relu5_3) and, except after block 5, the max-pool.
 *
 * rgs_lpips_input_conv (conv1_1, fp32 SIMT): x, y fp32 CHW [3, H, W], H >= 16 and W >= 16 (the reference fails below 16
 *   inside its fourth pool), H * W <= 2^28.  z = (v - mean_c) / std_c in fp32 with mean = (-.030, -.088, -.188) and
 *   std = (.458, .448, .450) as fp32 constants, applied to the [0, 1] values as given (lpipsPyTorch does not rescale to
 *   [-1, 1]); zero padding of z; weight fp32 [64][3][3][3] (torch's layout), bias [64]; per output
 *   acc = fma chain over (c, ky, kx) in that order from 0, then relu(acc + bias) rounded to TF32 -> out [2, H, W, 64].
 * rgs_lpips_conv3x3 (TF32 tensor cores): in [2, H, W, C_in], weight [C_out][3][3][C_in] (torch's [C_out][C_in][3][3]
 *   repacked), bias [C_out], C_in % 32 == 0, C_out % 64 == 0, both <= 512 -> out [2, H, W, C_out] = relu(conv + bias)
 *   rounded to TF32 with cvt.rna (nearest, ties away from zero).  The products run on wgmma.mma_async .tf32, which reads
 *   the top 19 bits of each operand and ignores the low 13: operands that are not TF32 values are truncated.  Every
 *   activation this file writes is a TF32 value, and rade_gs_b200.metrics rounds the weights with cvt.rna's rule when it
 *   loads them, so in the full trunk no operand bit is dropped; the error is the fp32 accumulation of K = 9 C_in
 *   products in the tensor cores' order, the bias addition and the output rounding (2^-11 relative).
 * rgs_lpips_maxpool: 2x2, stride 2, floor: in [2, H, W, C] -> out [2, H / 2, W / 2, C], C % 4 == 0; torch.max_pool2d's
 *   rule (window scanned row by row, a value replaces the maximum when greater or NaN), so results are bit-equal to it.
 * rgs_lpips_distance: feats [2, H, W, C], C in {64, 128, 256, 512}, lin fp32 [C] (the layer's 1x1 head).  Per pixel,
 *   fp32: n = sqrt(sum_c f^2) + 1e-10 for each image, map = sum_c lin_c (fx / nx - fy / ny)^2 -> map [H, W].  mean (one
 *   fp64 on the device) = (sum of map) / (H W), summed in fp64 in a fixed order: 16 pixels per warp in pixel order, 8 warps
 *   per CTA in warp order, the CTA sums in a fixed 512-thread tree.  Scratch through resize: 8 bytes per 128 pixels.
 *   The LPIPS value is the sum of the five layer means.
 * Every stage is deterministic: the same inputs give the same bits on every run and on every H100.  No stage reads
 * memory it did not write except its inputs.  An output must not overlap an input. */
int32_t rgs_lpips_input_conv(int32_t H, int32_t W, const float* x, const float* y, const float* weight, const float* bias, float* out, void* cuda_stream);
int32_t rgs_lpips_conv3x3(int32_t H, int32_t W, int32_t C_in, int32_t C_out, const float* in, const float* weight, const float* bias, float* out,
                          void* cuda_stream);
int32_t rgs_lpips_maxpool(int32_t H, int32_t W, int32_t C, const float* in, float* out, void* cuda_stream);
int32_t rgs_lpips_distance(int32_t H, int32_t W, int32_t C, const float* feats, const float* lin, float* map, double* mean, rgs_resize_fn resize,
                           void* scratch_user, void* cuda_stream);

/* ---- contracted-space TSDF mesh of unbounded scenes (utils/mesh_utils.py:163-271 extract_mesh_unbounded, :23-44
 *      post_process_mesh; utils/mcube_utils.py:17-95 marching_cubes_with_contraction) ----
 * Every fp32 value below is one IEEE operation rounded on its own, in the order written (no FMA contraction); |x| is
 * sqrtf((x.x x.x + x.y x.y) + x.z x.z).  Points are fp32 [N, 3] on the device, row-major.  Every output is the same bits on
 * every run; no stage reads memory it did not write except its inputs.
 *
 * Normalisation (host, rade_gs_b200.unbounded, with the reference's numpy expressions): c2w = numpy's inv of the fp32
 * world_view_transform^T (an fp32 result), poses = c2w[:3] @ diag(1, -1, -1, 1) in float64, center = the point nearest
 * to the optical axes, radius = min |c2w[:3, 3] - center|, voxel_size = 2 radius / resolution (float64).  Where the
 * reference combines these float64 scalars with fp32 tensors the tensor keeps fp32 and the scalar is rounded to fp32;
 * the kernels take c = fp32(center), r = fp32(radius), trunc0 = fp32(5 voxel_size) and compute (x - c) / r as one
 * division (the reference on CUDA multiplies by fp32(1 / r) instead, torch's division by a scalar: within one rounding).
 * R = min(quantile_0.95(|contract((x - c) / r)|) + 0.01, 1.9): numpy's quantile and sum over the fp32 norms that
 * rgs_unbounded_contract returns (no 2^24 limit), in numpy's dtype (float32 under numpy >= 2, float64 under numpy 1), as the
 * reference computes it; the crop bounds and samples are numpy's linspace of that R, rounded to fp32.
 *
 * rgs_unbounded_contract: inverse = 0: q = (p - c) / r, m = |q|, out = q if m < 1 else (2 - 1 / m) * (q / m); norms (may be
 *   NULL) = |out|.  inverse = 1 (inv_contraction and the clip): m = |p|, u = p if m < 1 else (1 / (2 - m)) * (p / m),
 *   out = clip(u r + c, -max_range, max_range) (NaN stays NaN); norms = |out|.  With c = 0, r = 1 the two are the
 *   reference's contract and uncontract exactly.
 * rgs_unbounded_sdf (the hot path): sample (i, j, k) of an n^3 crop, stored at (i n + j) n + k, is s = (xs[i], ys[j], zs[k])
 *   (the caller passes numpy's linspace rounded to fp32).  p = uncontract(s) r + c (as above, no clip).  trunc =
 *   trunc0, times 1 / (2 - min(|p|, 1.9f)) when |p| > 1 (the world-space norm, as the reference writes it; NaN stays NaN).
 *   Per view v in order: h_j = ((p.x M[0][j] + p.y M[1][j]) + p.z M[2][j]) + M[3][j] with M the row-major 4x4
 *   full_proj_transform; u = h_0 / h_3, v = h_1 / h_3; the view counts iff -1 < u < 1, -1 < v < 1 and h_3 > 0.  Depth is
 *   grid_sample(bilinear, border, align_corners=True): ix = ((u + 1) / 2) (W - 1) clamped to [0, W - 1] (likewise iy),
 *   x0 = floor(ix), x1 = x0 + 1, weights nw = (x1 - ix)(y1 - iy), ne = (ix - x0)(y1 - iy), sw = (x1 - ix)(iy - y0),
 *   se = (ix - x0)(iy - y0), d = 0 + nw D + ne D + sw D + se D in that order, skipping corners outside the image.
 *   sdf = d - h_3; the view is kept iff sdf > -trunc; then t <- (t w + clamp(sdf / trunc, -1, 1)) / (w + 1), w <- w + 1,
 *   from t = 1, w = 1.  The output is t.  depth fp32 [V, H, W], full_proj fp32 [V, 4, 4], 1 <= n <= 640.
 * rgs_unbounded_colors: the same projection, masks and bilinear weights at each point p (no contraction) with trunc = trunc0;
 *   each kept view updates col_k <- (col_k w + rgb_k) / (w + 1), w <- w + 1, from col = 0, w = 1.  rgb fp32 [V, 3, H, W].
 * rgs_unbounded_mcubes: an n^3 crop (layout as rgs_unbounded_sdf, 2 <= n <= 640) with lattice point (i, j, k) at
 *   lo + (i, j, k) sp, with the spacing sp given (the reference's (x_max - x_min) / (n - 1), computed by the caller in
 *   numpy's dtype: float32 under numpy >= 2).  A point is inside iff its value < 0 (0 and NaN are outside).  The
 *   cell at (i, j, k) < n - 1 uses the triangle table of rgs_tsdf_extract (corner c = x + 2y + 4z, edge e along axis e / 4):
 *   every triangle's right-hand normal points toward increasing values (free space).  The vertex of a sign-change lattice
 *   edge from g along axis a is owned by g: component a is (g_a + t) sp_a + lo_a, the others g_k sp_k + lo_k, with
 *   t = f(g) / (f(g) - f(g + e_a)), all fp64 with each operation rounded.  Vertices fp64 [V, 3] in (point, axis) order,
 *   triangles int32 [F, 3] in (cell, table order).  A crop without a sign change gives an empty mesh (the reference's skip
 *   of crops with min > 0 or max < 0 gives the same).  One stream synchronisation inside.
 * rgs_unbounded_merge (trimesh merge_vertices(digits_vertex=6), restated as this rule): key = (rint(x 1e6), rint(y 1e6),
 *   rint(z 1e6)) (fp64 product, ties to even), each in [-2^21, 2^21) or the call fails.  Vertices with equal keys merge
 *   into the first of them in input order, which keeps its unrounded coordinates, rounded to fp32 (.float()).  Survivors
 *   keep their input order.  Triangles are renumbered and kept, also when they become degenerate.  One synchronisation.
 * rgs_unbounded_clusters (Open3D cluster_connected_triangles + the removals of post_process_mesh): two triangles are
 *   connected iff they share an edge as an unordered vertex pair (a vertex contact does not connect; a repeated index
 *   forms the edge (a, a)).  threshold = max(sizes_ascending[C - k], 50) for 1 <= k <= C, max(smallest size, 50) for k = 0,
 *   and 50 when k > C (the reference raises IndexError there).  Triangles of clusters smaller than the threshold go, then
 *   vertices no remaining triangle uses (order kept), then triangles with a repeated index.  The outputs are the old
 *   indices of the kept vertices (int32, ascending) and the kept triangles renumbered (int32 [F', 3], order kept).  Two
 *   stream synchronisations inside.
 * Triangle indices must lie in [0, V): the merge and the clusters return RGS_E_INVALID otherwise. */
#define RGS_UNBOUNDED_MAX_CROP 640
typedef struct rgs_unbounded_mesh_out {
	void* vertices_user;        /* fp64 [V, 3] through resize */
	void* triangles_user;       /* int32 [F, 3] through resize */
	int64_t num_vertices, num_triangles;
} rgs_unbounded_mesh_out;
typedef struct rgs_unbounded_clusters_out {
	void* vertex_index_user;    /* int32 [V'] through resize */
	void* triangles_user;       /* int32 [F', 3] through resize */
	int64_t num_vertices, num_triangles, num_clusters, threshold;
} rgs_unbounded_clusters_out;
/* center (host) fp32 [3], radius > 0, max_range > 0 (inverse only; +inf for none).  out fp32 [n, 3], norms fp32 [n] or NULL. */
int32_t rgs_unbounded_contract(int64_t n, const float* points, const float center[3], float radius, int32_t inverse, float max_range, float* out, float* norms,
                               void* cuda_stream);
int32_t rgs_unbounded_sdf(int32_t n, const float* xs, const float* ys, const float* zs, int32_t V, int32_t H, int32_t W, const float* full_proj,
                          const float* depth, const float center[3], float radius, float trunc, float* sdf, void* cuda_stream);
int32_t rgs_unbounded_colors(int64_t N, const float* points, int32_t V, int32_t H, int32_t W, const float* full_proj, const float* depth, const float* rgb,
                             float trunc, float* colors, void* cuda_stream);
/* lo, spacing: host fp64 [3]. */
int32_t rgs_unbounded_mcubes(int32_t n, const float* sdf, const double lo[3], const double spacing[3], rgs_resize_fn resize, rgs_unbounded_mesh_out* out,
                             void* scratch_user, void* cuda_stream);
/* vertices fp64 [V, 3], triangles int32 [F, 3] -> triangles_out int32 [F, 3] (caller-allocated), merged vertices fp32 [U, 3]
 * through resize(vertices_user), U in *num_merged (host). */
int32_t rgs_unbounded_merge(int64_t V, const double* vertices, int64_t F, const int32_t* triangles, int32_t* triangles_out, rgs_resize_fn resize,
                            void* vertices_user, int64_t* num_merged, void* scratch_user, void* cuda_stream);
int32_t rgs_unbounded_clusters(int64_t V, int64_t F, const int32_t* triangles, int64_t cluster_to_keep, rgs_resize_fn resize, rgs_unbounded_clusters_out* out,
                               void* scratch_user, void* cuda_stream);

/* ---- densify-and-prune and opacity reset (reference scene/gaussian_model.py:495-513 reset_opacity, :662-741 densify_and_prune) ----
 * Inputs per Gaussian (fp32, device): grad_accum, grad_accum_abs, denom [P] (the [P,1] statistics), raw scaling [P,3], raw
 * opacity [P], rotation [P,4], xyz [P,3]; 0 < P < 2^31.
 *
 * Floating-point contract.
 *   - Selections, counts, row order and every copied float are bit-exact against the reference run on CUDA.
 *   - exp, log and sigmoid = 1 / (1 + exp(-x)) are the accurate libdevice functions (no fast-math), as torch's CUDA kernels
 *     compute them.  Every other operation is one IEEE fp32 operation rounded on its own, in the order written below.
 *   - g = accum / denom and g_abs = accum_abs / denom; NaN (0/0, NaN inputs) becomes 0, x/0 for x > 0 stays +inf.
 *   - |g| for the clone and ratio tests is torch.norm of a one-element row on CUDA: sqrt(g * g) in fp32.
 *   - ratio = (float)count * (1.0f / (float)P), count = #{|g| >= max_grad}, as ATen's CUDA mean (a sum times the fp32
 *     reciprocal; torch on the CPU divides instead).  Exact while count <= 2^24.
 *   - Q = torch.quantile(g_abs, 1 - ratio), linear: q = 1 - ratio, rank = q * (float)(P - 1), lo = (int64)rank,
 *     hi = ceil(rank), w = rank - lo, a = sorted[lo], b = sorted[hi] (indices clamped to P - 1, which only binds above 2^24
 *     rows), d = b - a, Q = |w| < 0.5 ? fma(w, d, a) : fma(-d, 1 - w, b) (torch.lerp as built for CUDA).  The order statistics
 *     come from a full radix sort of g_abs, so Q is exact for any P; there is no 2^24 limit.
 *   - clone = (|g| >= max_grad or |g_abs| >= Q) and max_k exp(s_k) <= dense; split = (g >= max_grad or g_abs >= Q) and
 *     max_k exp(s_k) > dense, over the original rows.  A clone carries its parent's raw scaling bit for bit, so the same
 *     max exp(s) <= dense that made it a clone keeps it from being split.
 *   - New rows: q = r / sqrt(((r0 r0 + r1 r1) + r2 r2) + r3 r3); R as build_rotation (utils/general_utils.py:80-101), each
 *     product, sum and difference rounded (2 * t and 1 - t as written); xyz_new_i = ((R_i0 s0 + R_i1 s1) + R_i2 s2) + xyz_i,
 *     every product and sum rounded, left to right.  This is the order of torch.bmm on the CPU; cuBLAS's torch.bmm on CUDA
 *     may order or fuse the three products differently, which moves xyz_new_i by at most
 *     2^-21 * (|R_i0 s0| + |R_i1 s1| + |R_i2 s2| + |xyz_i|).  The same bound covers torch on the CPU, whose vectorised sqrt
 *     (the quaternion norm) is not correctly rounded; CUDA's sqrtf, used here, is.
 *   - Split children: scaling log(exp(s) * (1.0f / 1.6f)) (torch on CUDA multiplies by the fp32 reciprocal of a Python
 *     scalar divisor; on the CPU it divides: the two differ by at most one rounding of the quotient).
 *   - Prune: sigmoid(o) < min_opacity, or, when prune_large: 0 > max_screen_size (max_radii2D is all zeros by then) or
 *     max_k exp(s_k) > world.  Python thresholds are rounded to fp32 first (max_grad, dense = percent_dense * extent,
 *     min_opacity, max_screen_size, world = 0.1 * extent), as torch compares a float32 tensor with a Python scalar.
 *   - reset_opacity: coef = sqrt(((sq0 sq1) sq2) / ((a0 a1) a2)), sq_k = exp(s_k)^2, a_k = sq_k + f^2; o = sigmoid(x) * coef;
 *     x' = min(o, 0.01f) / coef; result log(x' / (1 - x')).
 *
 * Output rows, in order: the original rows not split, the clones, the first child of every split row, the second child of
 * every split row, each in index order and each without the rows the final prune drops.
 *
 * rgs_densify_select: flags [P] (one byte per Gaussian), block_offsets [5 * rgs_densify_blocks(P) + 5] (per-CTA offsets, then
 *   the totals), ratio_q [2] (device:
 *   ratio, Q) and counts_host [5] (host: C clones, S split rows, surviving originals K0, surviving clones K1, surviving
 *   children per copy K2; the result has K0 + K1 + 2 K2 rows).  Scratch through the resize callback (about 8 bytes per
 *   Gaussian plus the sort's workspace).  One stream synchronisation (the counts).
 * rgs_densify_plan: src, draw [K0 + K1 + 2 K2] (source row and draw index of every output row, draw -1 on original rows,
 *   draw < C a clone's row of the clone draws, draw >= C row draw - C of the split draws) and the exp(scaling) rows packed
 *   as the std of the draws: std_clone [C,3], std_split [2S,3] (stds.repeat(2, 1)).
 * rgs_densify_gather: xyz_out and scaling_out [N,3] of every output row from the caller's draws sample_clone [C,3] and
 *   sample_split [2S,3]; every other column through cols: out[j] = in[src[j]] (width floats per row), zeros on new rows
 *   when zero_new_rows.
 * rgs_reset_opacity: out [P] as above. */
#define RGS_DENSIFY_MAX_COLUMNS 18
typedef struct rgs_densify_thresholds {
	float max_grad, dense, min_opacity, max_screen_size, world;
	float inv_split;       /* 1.0f / (float)(0.8 * N), N = 2 */
	int32_t prune_large;   /* max_screen_size is truthy */
} rgs_densify_thresholds;
typedef struct rgs_densify_column {
	const float* in;       /* [P, width] */
	float* out;            /* [N, width] */
	int64_t width;
	int32_t zero_new_rows;
} rgs_densify_column;
int32_t rgs_densify_blocks(int32_t P);
int32_t rgs_densify_select(int32_t P, const float* grad_accum, const float* grad_accum_abs, const float* denom, const float* scaling, const float* opacity,
                           const rgs_densify_thresholds* thresholds, uint8_t* flags, int32_t* block_offsets, float* ratio_q, int32_t* counts_host,
                           rgs_resize_fn scratch, void* scratch_user, void* cuda_stream);
int32_t rgs_densify_plan(int32_t P, const uint8_t* flags, const int32_t* block_offsets, const int32_t* counts_host, const float* scaling, int32_t* src,
                         int32_t* draw, float* std_clone, float* std_split, void* cuda_stream);
int32_t rgs_densify_gather(int32_t N, const int32_t* src, const int32_t* draw, int32_t C, const float* xyz, const float* rotation, const float* scaling,
                           const float* sample_clone, const float* sample_split, float inv_split, float* xyz_out, float* scaling_out, int32_t n_cols,
                           const rgs_densify_column* cols, void* cuda_stream);
int32_t rgs_reset_opacity(int32_t P, const float* scaling, const float* opacity, const float* filter_3D, float* out, void* cuda_stream);

/* Introspection for parity tests: views into the private buffers written by rgs_forward
 * (the reference keeps the same data at BinningState::point_list / ImageState::ranges,
 * rasterizer_impl.cu:237-250,224-235).  Pointers are device addresses inside the given buffers. */
typedef struct rgs_debug_views {
	const uint32_t* point_list;      /* [num_rendered] sorted Gaussian ids                 */
	const uint64_t* point_list_keys; /* [num_rendered] sorted (tile<<32 | depth bits) keys */
	const uint32_t* tile_ranges;     /* [tiles][2]  start,end                              */
	const uint32_t* n_contrib;       /* [2,H,W] last contributor, median contributor       */
	const uint32_t* tiles_touched;   /* [P]                                                */
	const float* records;            /* [P, record_floats] packed render records           */
	int32_t record_floats;
	const float* depths;             /* [P] view-space z                                   */
} rgs_debug_views;
int32_t rgs_debug_get_views(const rgs_camera* cam, int32_t P, int64_t num_rendered, const char* geom_buffer,
                            const char* binning_buffer, const char* image_buffer, rgs_debug_views* views);

/* Optional per-stage device timing for benchmarking: while enabled, every stage launch is bracketed by CUDA
 * events on the launching stream.  rgs_stage_times synchronises on them and returns, per stage, the summed
 * duration and the number of launches since timing was switched on (names are static strings). */
void rgs_stage_timing(int32_t enable);
int32_t rgs_stage_times(const char** names, double* total_ms, int64_t* launches, int32_t capacity);

const char* rgs_last_error(void);
int32_t rgs_abi_version(void);
/* Number of kernel launches issued by this library since process start (bench.py's gpu_launches). */
int64_t rgs_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* RGS_B200_H_INCLUDED */

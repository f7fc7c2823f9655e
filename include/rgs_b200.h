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

#define RGS_ABI_VERSION 3

typedef enum rgs_status {
	RGS_OK = 0,
	RGS_E_INVALID = -1,      /* bad argument (shape/flag combination the reference rejects)            */
	RGS_E_CUDA = -2,         /* CUDA runtime error (message in rgs_last_error)                         */
	RGS_E_UNSUPPORTED = -3,  /* e.g. prefiltered=true (mis-wired in the reference, SURVEY app. A-15)    */
	RGS_E_ALLOC = -4         /* a resize callback returned NULL                                        */
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
/* Alternative to create + connect: the caller provides the windows (e.g. torch symmetric memory: cuMem VMM allocations mapped on every
 * rank, plus an NVLS multicast mapping).  window_ptrs[p] = this process's mapping of rank p's window, each rgs_exchange_window_bytes
 * long and zero-filled; multicast_ptr = multicast mapping of all windows or 0.  With a multicast mapping the spread phase issues ONE
 * store per 16 bytes and the NVSwitch replicates it (outbound traffic / world). */
size_t rgs_exchange_window_bytes(int32_t world, int64_t capacity_rows, int32_t row_floats);
int32_t rgs_exchange_attach(int32_t rank, int32_t world, int64_t capacity_rows, int32_t row_floats, const uint64_t* window_ptrs,
                            uint64_t multicast_ptr, rgs_exchange** out);
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
const char* rgs_exchange_last_error(void);

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

// rgs_api.cu -- the C ABI (include/rgs_b200.h): buffer carving, orchestration, error handling.
//
// Replaces CudaRasterizer::Rasterizer::{forward,backward,markVisible} and the GeometryState /
// BinningState / ImageState chunk allocator (reference: cuda_rasterizer/rasterizer_impl.cu:190-250,
// 254-425, 429-571, 176-188; cuda_rasterizer/rasterizer_impl.h:22-94).
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "rgs_common.cuh"

namespace rgs {

static std::atomic<int64_t> g_launches{0};
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

static thread_local std::string t_error;

// ---- optional per-stage device timing (bench.py's roofline leg): cudaEvents recorded on the launching stream
// around each stage, read back by rgs_stage_times() after a synchronize.  Off by default: zero overhead.
enum Stage { ST_PREPROCESS, ST_SCAN, ST_BINNING, ST_RENDER_FWD, ST_RENDER_BWD, ST_PREPROCESS_BWD, ST_EXCHANGE, ST_COUNT };
static const char* kStageNames[ST_COUNT] = {"preprocess_forward", "scan", "binning_sort", "render_forward", "render_backward", "preprocess_backward", "gradient_exchange"};
struct StageRec { int stage; cudaEvent_t a, b; };
static std::mutex g_stage_mu;
static std::vector<StageRec> g_stage_pending;
static double g_stage_ms[ST_COUNT];
static int64_t g_stage_n[ST_COUNT];
static std::atomic<int> g_stage_on{0};

struct StageScope {
	cudaStream_t s; int stage; cudaEvent_t a = nullptr, b = nullptr; bool on;
	StageScope(int st, cudaStream_t stream) : s(stream), stage(st), on(g_stage_on.load() != 0) {
		if (on) { cudaEventCreate(&a); cudaEventCreate(&b); cudaEventRecord(a, s); }
	}
	~StageScope() {
		if (on) { cudaEventRecord(b, s); std::lock_guard<std::mutex> lk(g_stage_mu); g_stage_pending.push_back({stage, a, b}); }
	}
};
static void stage_collect() {
	std::lock_guard<std::mutex> lk(g_stage_mu);
	for (auto& r : g_stage_pending) {
		cudaEventSynchronize(r.b);
		float ms = 0.f;
		if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) { g_stage_ms[r.stage] += ms; g_stage_n[r.stage]++; }
		cudaEventDestroy(r.a); cudaEventDestroy(r.b);
	}
	g_stage_pending.clear();
}

static int fail(int code, const std::string& msg) {
	t_error = msg;
	return code;
}

#define RGS_CUDA_TRY(expr)                                                                                   \
	do {                                                                                                     \
		cudaError_t _e = (expr);                                                                             \
		if (_e != cudaSuccess) return fail(RGS_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
	} while (0)

// A launcher's result as a status of entry `what`.  The DTU and TNT launchers report a non-finite input point as
// cudaErrorInvalidValue; they pass `invalid`, the message that turns it into RGS_E_INVALID.
static int cuda_status(cudaError_t e, const char* what, const char* invalid = nullptr) {
	if (e == cudaSuccess) return RGS_OK;
	if (invalid && e == cudaErrorInvalidValue) return fail(RGS_E_INVALID, std::string(what) + ": " + invalid);
	return fail(RGS_E_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

static const char* const kNonFinitePoint = "a point has a NaN or infinite coordinate";

// `bytes` from the caller's resize callback into `buf`.  NULL is a failure only when bytes were asked for: an empty
// output may come back as NULL.
static int grow(rgs_resize_fn fn, void* user, size_t bytes, char*& buf, const char* what) {
	buf = fn(user, bytes);
	return buf || bytes == 0 ? (int)RGS_OK : fail(RGS_E_ALLOC, std::string(what) + " callback returned NULL");
}

// After each stage in debug mode: synchronise and surface the error, like CHECK_CUDA (auxiliary.h:404-411).
static int debug_sync(const rgs_camera* cam, cudaStream_t s, const char* stage) {
	cudaError_t e = cudaGetLastError();
	if (e == cudaSuccess && cam->debug) e = cudaStreamSynchronize(s);
	if (e != cudaSuccess) return fail(RGS_E_CUDA, std::string("[CUDA ERROR] in ") + stage + ": " + cudaGetErrorString(e));
	return RGS_OK;
}

static GeomView carve_geom(char* base, int P, bool coord, size_t* total) {
	Carver c(base);
	GeomView g;
	g.records = c.take<float>((size_t)P * rec_floats(coord));
	g.depths = c.take<float>(P);
	g.tiles_touched = c.take<uint32_t>(P);
	g.bwd_rows = c.take<uint32_t>(P);
	g.clamped = c.take<uint8_t>(P);
	g.sigma_inv = c.take<float>((size_t)P * SIGMA_INV_FLOATS);
	g.bwd_row_count = c.take<uint32_t>(1);
	if (total) *total = c.size();
	return g;
}

static BinView carve_bin(char* base, size_t R, int tiles, size_t* total) {
	Carver c(base);
	BinView b;
	b.point_list = c.take<uint32_t>(R);
	b.keys_sorted = c.take<uint64_t>(R);
	b.hitmask = c.take<uint32_t>(hitmask_words(R, tiles));
	b.keys_unsorted = c.take<uint64_t>(R);
	if (total) *total = c.size();
	return b;
}

static ImgView carve_img(char* base, int grid_x, int grid_y, size_t N, bool coord, bool depth, size_t* total) {
	const int tiles = grid_x * grid_y;
	Carver c(base);
	ImgView v;
	v.ranges = c.take<uint2>(tiles);
	v.tile_count = c.take<uint32_t>(tiles);
	v.totals = c.take<uint32_t>(2);
	v.chunk_base = c.take<uint32_t>(tiles);
	v.n_contrib = c.take<uint32_t>(2 * N);
	v.accum_depth = c.take<float>(depth ? N : 0);
	v.normal_length = c.take<float>((coord || depth) ? N : 0);
	v.accum_coord = c.take<float>(coord ? 3 * N : 0);
	v.tile_diff = c.take<int>((size_t)(grid_x + 1) * (grid_y + 1));
	if (total) *total = c.size();
	return v;
}

// Height of the [C,Hs,W] maps: the whole image, or with compact_slab only the pixel rows of tile rows [row_begin, row_end).
static int slab_height(const rgs_camera* cam, int row_begin, int row_end) {
	if (!cam->compact_slab) return cam->height;
	const int hs = (row_end * TILE_Y < cam->height ? row_end * TILE_Y : cam->height) - row_begin * TILE_Y;
	return hs > 0 ? hs : 0;
}

static int make_params(const rgs_camera* cam, const rgs_gaussians* g, FwdParams& p) {
	if (!cam || !g) return fail(RGS_E_INVALID, "null camera / gaussians");
	if (cam->width <= 0 || cam->height <= 0) return fail(RGS_E_INVALID, "image size must be positive");
	if (g->P < 0) return fail(RGS_E_INVALID, "negative Gaussian count");
	if (cam->prefiltered)
		return fail(RGS_E_UNSUPPORTED,
		            "prefiltered=True is mis-wired in the reference (rasterizer_impl.cu:343-345 feeds it to the `integrate` switch) and is not supported");
	const bool has_sh = g->shs != nullptr, has_col = g->colors_precomp != nullptr;
	if (has_sh == has_col && g->P > 0) return fail(RGS_E_INVALID, "Please provide excatly one of either SHs or precomputed colors!");
	const bool has_sr = g->scales != nullptr && g->rotations != nullptr, has_cov = g->cov3D_precomp != nullptr;
	if (has_sr == has_cov && g->P > 0)
		return fail(RGS_E_INVALID, "Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
	if (has_sh && (cam->sh_degree < 0 || cam->sh_degree > 3 || (cam->sh_degree + 1) * (cam->sh_degree + 1) > cam->sh_coeffs))
		return fail(RGS_E_INVALID, "sh_degree does not fit the stored SH coefficients");
	if (has_sh && cam->sh_coeffs > 16)
		return fail(RGS_E_INVALID, "at most 16 SH coefficients per Gaussian (degree 3) are supported");  // the SH kernels stage rows of <= 16 x 3 floats
	p.P = g->P;
	p.D = cam->sh_degree;
	p.M = has_sh ? cam->sh_coeffs : 0;
	p.W = cam->width;
	p.H = cam->height;
	p.grid_x = (cam->width + TILE_X - 1) / TILE_X;
	p.grid_y = (cam->height + TILE_Y - 1) / TILE_Y;
	p.row_begin = cam->tile_row_begin;
	p.row_end = cam->tile_row_end < 0 ? p.grid_y : cam->tile_row_end;
	if (p.row_begin < 0 || p.row_end > p.grid_y || p.row_begin > p.row_end) return fail(RGS_E_INVALID, "tile row slab out of range");
	p.py_off = cam->compact_slab ? p.row_begin * TILE_Y : 0;
	p.Hs = slab_height(cam, p.row_begin, p.row_end);
	p.tan_fovx = cam->tan_fovx;
	p.tan_fovy = cam->tan_fovy;
	// focal lengths computed on the host in float, as the reference does (rasterizer_impl.cu:288-289)
	p.focal_y = cam->height / (2.0f * cam->tan_fovy);
	p.focal_x = cam->width / (2.0f * cam->tan_fovx);
	p.kernel_size = cam->kernel_size;
	p.scale_modifier = cam->scale_modifier;
	p.coord = cam->require_coord != 0;
	p.depth = cam->require_depth != 0;
	p.means3D = g->means3D;
	p.opacities = g->opacities;
	p.shs = g->shs;
	p.shs_rest = has_sh ? g->shs_rest : nullptr;
	if (p.shs_rest != nullptr && p.M < 2) return fail(RGS_E_INVALID, "shs_rest given but sh_coeffs < 2");
	p.colors_precomp = g->colors_precomp;
	p.scales = g->scales;
	p.rotations = g->rotations;
	p.cov3D_precomp = g->cov3D_precomp;
	p.viewmatrix = cam->viewmatrix;
	p.projmatrix = cam->projmatrix;
	p.cam_pos = cam->cam_pos;
	p.background = cam->background;
	return RGS_OK;
}

// pinned 4-byte mailbox per thread for the num_rendered read-back
static uint32_t* pinned_mailbox() {
	static thread_local uint32_t* box = nullptr;
	if (!box) {
		if (cudaHostAlloc((void**)&box, 64, cudaHostAllocDefault) != cudaSuccess) box = nullptr;
	}
	return box;
}

}  // namespace rgs

using namespace rgs;

extern "C" {

const char* rgs_last_error(void) { return t_error.c_str(); }
int32_t rgs_abi_version(void) { return RGS_ABI_VERSION; }
int64_t rgs_launch_count(void) { return g_launches.load(); }
void rgs_stage_timing(int32_t enable) {
	stage_collect();
	if (enable) { std::lock_guard<std::mutex> lk(g_stage_mu); for (int i = 0; i < ST_COUNT; i++) { g_stage_ms[i] = 0; g_stage_n[i] = 0; } }
	g_stage_on.store(enable ? 1 : 0);
}
int32_t rgs_stage_times(const char** names, double* total_ms, int64_t* launches, int32_t capacity) {
	stage_collect();
	int n = capacity < ST_COUNT ? capacity : ST_COUNT;
	for (int i = 0; i < n; i++) { names[i] = kStageNames[i]; total_ms[i] = g_stage_ms[i]; launches[i] = g_stage_n[i]; }
	return n;
}
int32_t rgs_grad_stride(int32_t require_coord, int32_t /*require_depth*/) { return grad_floats(require_coord != 0); }

// preprocess -> tile counts -> (one host sync for the instance count) -> binning / sort: everything before blending.
// Shared by rgs_forward and rgs_integrate.  Returns num_rendered or a negative status.
static int64_t forward_to_binning(const rgs_camera* cam, const FwdParams& p, int* radii, const rgs_buffers* bufs, cudaStream_t s, GeomView& g,
                                  BinView& b, ImgView& img) {
	int rc;
	const int P = p.P;
	const size_t N = (size_t)p.W * p.Hs;
	const int tiles = p.grid_x * p.grid_y;

	// image-side scratch first: needed even when there is nothing to draw (background fill)
	size_t img_bytes = 0;
	carve_img(nullptr, p.grid_x, p.grid_y, N, p.coord, p.depth, &img_bytes);
	char* img_ptr;
	if ((rc = grow(bufs->image, bufs->image_user, img_bytes, img_ptr, "image buffer")) != RGS_OK) return rc;
	img = carve_img(img_ptr, p.grid_x, p.grid_y, N, p.coord, p.depth, nullptr);

	size_t geom_bytes = 0;
	carve_geom(nullptr, P, p.coord, &geom_bytes);
	char* geom_ptr;
	if ((rc = grow(bufs->geom, bufs->geom_user, geom_bytes, geom_ptr, "geometry buffer")) != RGS_OK) return rc;
	g = carve_geom(geom_ptr, P, p.coord, nullptr);

	int64_t R = 0;
	uint32_t max_list = 0;
	if (P > 0) {
		RGS_CUDA_TRY(cudaMemsetAsync(img.tile_diff, 0, (size_t)(p.grid_x + 1) * (p.grid_y + 1) * sizeof(int), s));
		{ StageScope sc(ST_PREPROCESS, s); launch_preprocess_forward(p, g, radii, img.tile_diff, s); }
		if ((rc = debug_sync(cam, s, "preprocess")) != RGS_OK) return rc;
		{ StageScope sc(ST_SCAN, s); launch_tile_scan(p, img, s); }
		// the one host sync of the forward pass: the instance count sizes the binning buffers and is returned to the
		// caller (reference: blocking cudaMemcpy, rasterizer_impl.cu:354); the longest tile list picks the sort path
		uint32_t* box = pinned_mailbox();
		if (!box) return fail(RGS_E_CUDA, "cudaHostAlloc failed for the num_rendered mailbox");
		RGS_CUDA_TRY(cudaMemcpyAsync(box, img.totals, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
		RGS_CUDA_TRY(cudaStreamSynchronize(s));
		R = (int64_t)box[0];
		max_list = box[1];
	}
	size_t bin_bytes = 0;
	carve_bin(nullptr, (size_t)R, tiles, &bin_bytes);
	char* bin_ptr;
	if ((rc = grow(bufs->binning, bufs->binning_user, bin_bytes, bin_ptr, "binning buffer")) != RGS_OK) return rc;
	b = carve_bin(bin_ptr, (size_t)R, tiles, nullptr);
	// forward-render writes a ballot word only for the chunks a warp actually tested; backward masks every position at or
	// behind the warp's last contributor, so the unwritten words never matter -- zero them anyway (<= R bytes) so that no
	// consumer (debug views, initcheck) ever sees memory the library did not write
	if (R > 0) RGS_CUDA_TRY(cudaMemsetAsync(b.hitmask, 0, hitmask_words((size_t)R, tiles) * sizeof(uint32_t), s));

	if (P == 0) {
		RGS_CUDA_TRY(cudaMemsetAsync(img.ranges, 0, (size_t)tiles * sizeof(uint2), s));
	} else {
		// lists longer than the shared-memory sort take the multi-CTA path inside launch_tile_binning
		StageScope sc(ST_BINNING, s);
		launch_tile_binning(p, g, b, img, radii, R, max_list, s);
	}
	if ((rc = debug_sync(cam, s, "binning")) != RGS_OK) return rc;
	return R;
}

int64_t rgs_forward(const rgs_camera* cam, const rgs_gaussians* gs, const rgs_forward_out* out, const rgs_buffers* bufs, void* cuda_stream) {
	FwdParams p;
	int rc = make_params(cam, gs, p);
	if (rc != RGS_OK) return rc;
	if (!out || !bufs || !bufs->geom || !bufs->binning || !bufs->image) return fail(RGS_E_INVALID, "null outputs / buffer callbacks");
	cudaStream_t s = (cudaStream_t)cuda_stream;
	GeomView g;
	BinView b;
	ImgView img;
	const int64_t R = forward_to_binning(cam, p, out->radii, bufs, s, g, b, img);
	if (R < 0) return R;
	RenderOut ro{out->out_color, out->out_coord, out->out_mcoord, out->out_alpha, out->out_normal, out->out_depth, out->out_mdepth};
	{ StageScope sc(ST_RENDER_FWD, s); launch_render_forward(p, g, b, img, ro, s); }
	if ((rc = debug_sync(cam, s, "render")) != RGS_OK) return rc;
	return R;
}

// Replaces CudaRasterizer::Rasterizer::integrate (rasterizer.h:68-108, rasterizer_impl.cu:573-844).
int64_t rgs_integrate(const rgs_camera* cam, const rgs_gaussians* gs, const rgs_integrate_io* io, const rgs_buffers* bufs, rgs_resize_fn point_buffer,
                      void* point_buffer_user, int32_t* overflowed_pixels, void* cuda_stream) {
	if (!cam) return fail(RGS_E_INVALID, "null camera / gaussians");
	rgs_camera c = *cam;
	c.require_depth = 1;  // the integrate path always carries the ray-space planes (rasterizer_impl.cu:634-668)
	c.require_coord = 0;
	c.tile_row_begin = 0;
	c.tile_row_end = -1;
	c.compact_slab = 0;
	FwdParams p;
	int rc = make_params(&c, gs, p);
	if (rc != RGS_OK) return rc;
	if (!io || !bufs || !bufs->geom || !bufs->binning || !bufs->image || !point_buffer) return fail(RGS_E_INVALID, "null outputs / buffer callbacks");
	if (io->PN <= 0 || p.P <= 0) return fail(RGS_E_INVALID, "integrate needs at least one Gaussian and one point (the reference returns its fill values)");
	if (!io->points3D || !io->out_color || !io->out_alpha_integrated || !io->out_color_integrated || !io->out_coordinate2d || !io->out_sdf || !io->radii)
		return fail(RGS_E_INVALID, "null integrate inputs / outputs");
	cudaStream_t s = (cudaStream_t)cuda_stream;
	GeomView g;
	BinView b;
	ImgView img;
	const int64_t R = forward_to_binning(&c, p, io->radii, bufs, s, g, b, img);
	if (R < 0) return R;
	const int tiles = p.grid_x * p.grid_y;
	const size_t N = (size_t)p.W * p.H;
	const int PN = io->PN;
	IntegrateView v;
	size_t bytes = 0;
	for (int pass = 0; pass < 2; pass++) {
		char* base = nullptr;
		if (pass == 1 && (rc = grow(point_buffer, point_buffer_user, bytes, base, "point buffer")) != RGS_OK) return rc;
		Carver cv(base);
		v.PN = PN;
		v.points3D = io->points3D;
		v.invray = cv.take<float>((size_t)p.P * 8);
		v.masks = cv.take<uint32_t>(integrate_mask_words(R, tiles));
		v.aux = cv.take<float4>(2 * N);
		v.overflow = cv.take<int>(1);
		v.key_in = cv.take<uint32_t>(PN);
		v.key_out = cv.take<uint32_t>(PN);
		v.pid_in = cv.take<uint32_t>(PN);
		v.pid_out = cv.take<uint32_t>(PN);
		v.pxy = cv.take<float2>(PN);
		v.pdepth = cv.take<float>(PN);
		v.sort_temp_bytes = integrate_sort_temp_bytes(PN);
		v.sort_temp = cv.take<char>(v.sort_temp_bytes);
		bytes = cv.size();
	}
	IntegrateOut out{io->out_color, io->out_alpha_integrated, io->out_color_integrated, io->out_coordinate2d, io->out_sdf};
	launch_integrate(p, g, b, img, io->radii, v, out, s);
	if ((rc = debug_sync(&c, s, "integrate")) != RGS_OK) return rc;
	if (overflowed_pixels) {
		// rare diagnostic (the reference printf's from the kernel): one more small blocking read
		int host = 0;
		RGS_CUDA_TRY(cudaMemcpyAsync(&host, v.overflow, sizeof(int), cudaMemcpyDeviceToHost, s));
		RGS_CUDA_TRY(cudaStreamSynchronize(s));
		*overflowed_pixels = host;
	}
	return R;
}

static int backward_views(const rgs_camera* cam, const rgs_gaussians* gs, const rgs_backward_in* in, FwdParams& p, GeomView& g, BinView& b, ImgView& img) {
	int rc = make_params(cam, gs, p);
	if (rc != RGS_OK) return rc;
	if (!in || !in->geom_buffer || !in->image_buffer) return fail(RGS_E_INVALID, "null backward inputs / buffers");
	const size_t N = (size_t)p.W * p.Hs;
	g = carve_geom(const_cast<char*>(in->geom_buffer), p.P, p.coord, nullptr);
	b = carve_bin(const_cast<char*>(in->binning_buffer), (size_t)in->num_rendered, p.grid_x * p.grid_y, nullptr);
	img = carve_img(const_cast<char*>(in->image_buffer), p.grid_x, p.grid_y, N, p.coord, p.depth, nullptr);
	return RGS_OK;
}

int32_t rgs_backward_render(const rgs_camera* cam, const rgs_gaussians* gs, const rgs_backward_in* in, float* grad_accum, void* cuda_stream) {
	FwdParams p;
	GeomView g;
	BinView b;
	ImgView img;
	int rc = backward_views(cam, gs, in, p, g, b, img);
	if (rc != RGS_OK) return rc;
	if (p.P == 0) return RGS_OK;
	if (!grad_accum) return fail(RGS_E_INVALID, "null gradient accumulator");
	cudaStream_t s = (cudaStream_t)cuda_stream;
	RenderGradIn gin{in->dL_dout_color, in->dL_dout_coord, in->dL_dout_mcoord, in->dL_dout_depth, in->dL_dout_mdepth,
	                 in->dL_dout_alpha, in->dL_dout_normal, in->out_alpha, in->out_normal};
	{ StageScope sc(ST_RENDER_BWD, s); launch_render_backward(p, g, b, img, gin, grad_accum, s); }
	return debug_sync(cam, s, "backward render");
}

int32_t rgs_backward_render_exchange(const rgs_camera* cam, const rgs_gaussians* gs, const rgs_backward_in* in, rgs_exchange* ex, void* cuda_stream) {
	FwdParams p;
	GeomView g;
	BinView b;
	ImgView img;
	int rc = backward_views(cam, gs, in, p, g, b, img);
	if (rc != RGS_OK) return rc;
	if (p.P == 0) return RGS_OK;
	float* acc = rgs_exchange_accumulator(ex);
	if (!acc) return fail(RGS_E_INVALID, "null exchange");
	cudaStream_t s = (cudaStream_t)cuda_stream;
	RenderGradIn gin{in->dL_dout_color, in->dL_dout_coord, in->dL_dout_mcoord, in->dL_dout_depth, in->dL_dout_mdepth,
	                 in->dL_dout_alpha, in->dL_dout_normal, in->out_alpha, in->out_normal};
	{ StageScope sc(ST_RENDER_BWD, s); launch_render_backward(p, g, b, img, gin, acc, s, /*zero_first=*/false); }
	if ((rc = debug_sync(cam, s, "backward render")) != RGS_OK) return rc;
	{
		StageScope sc(ST_EXCHANGE, s);
		rc = rgs_exchange_rows(ex, p.P, g.tiles_touched, in->radii, cuda_stream);
	}
	if (rc != RGS_OK) return fail(rc, rgs_exchange_last_error());
	return debug_sync(cam, s, "gradient exchange");
}

static int32_t backward_preprocess_impl(const rgs_camera* cam, const rgs_gaussians* gs, const rgs_backward_in* in, const float* grad_accum,
                                        const rgs_backward_out* out, void* cuda_stream, bool prefilled) {
	FwdParams p;
	GeomView g;
	BinView b;
	ImgView img;
	int rc = backward_views(cam, gs, in, p, g, b, img);
	if (rc != RGS_OK) return rc;
	if (p.P == 0) return RGS_OK;
	if (!grad_accum || !out) return fail(RGS_E_INVALID, "null gradient accumulator / outputs");
	cudaStream_t s = (cudaStream_t)cuda_stream;
	ParamGradOut po{out->dL_dmeans2D, out->dL_dcolors, out->dL_dopacity, out->dL_dmeans3D, out->dL_dcov3D, out->dL_dsh, out->dL_dscales, out->dL_drotations, out->dL_dsh_rest};
	if ((p.shs_rest != nullptr) != (po.d_sh_rest != nullptr) && po.d_sh != nullptr)
		return fail(RGS_E_INVALID, "dL_dsh_rest must be given exactly when shs_rest is");
	{ StageScope sc(ST_PREPROCESS_BWD, s); launch_preprocess_backward(p, g, in->radii, grad_accum, po, s, prefilled); }
	return debug_sync(cam, s, "backward preprocess");
}

int32_t rgs_backward_preprocess(const rgs_camera* cam, const rgs_gaussians* gs, const rgs_backward_in* in, const float* grad_accum,
                                const rgs_backward_out* out, void* cuda_stream) {
	return backward_preprocess_impl(cam, gs, in, grad_accum, out, cuda_stream, false);
}

// per-device side stream + events for work that may run underneath the main stream's kernels
struct SideStream {
	cudaStream_t stream = nullptr;
	cudaEvent_t fork = nullptr, join = nullptr;
};
static SideStream* side_stream() {
	static thread_local SideStream per_dev[64];
	int dev = 0;
	if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
	SideStream& ss = per_dev[dev & 63];
	if (!ss.stream) {
		if (cudaStreamCreateWithFlags(&ss.stream, cudaStreamNonBlocking) != cudaSuccess) return nullptr;
		if (cudaEventCreateWithFlags(&ss.fork, cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&ss.join, cudaEventDisableTiming) != cudaSuccess)
			return nullptr;
	}
	return &ss;
}

int32_t rgs_backward(const rgs_camera* cam, const rgs_gaussians* gs, const rgs_backward_in* in, const rgs_backward_out* out,
                     rgs_resize_fn grad_scratch, void* grad_scratch_user, void* cuda_stream) {
	if (!gs || !cam) return fail(RGS_E_INVALID, "null camera / gaussians");
	if (gs->P == 0) return RGS_OK;
	if (!grad_scratch) return fail(RGS_E_INVALID, "null scratch callback");
	if (!out) return fail(RGS_E_INVALID, "null gradient accumulator / outputs");
	const size_t bytes = (size_t)gs->P * grad_floats(cam->require_coord != 0) * sizeof(float);
	char* acc_bytes;
	if (const int rc = grow(grad_scratch, grad_scratch_user, bytes, acc_bytes, "gradient scratch")) return rc;
	float* acc = reinterpret_cast<float*>(acc_bytes);
	cudaStream_t s = (cudaStream_t)cuda_stream;
	// The zero-fill of the dense gradient tensors (pure HBM writes, ~280 MB at 1 M Gaussians) runs on a side stream underneath the
	// issue-bound backward blend; everything queued on `s` before this call is ordered before it (the tensors may be recycled memory).
	bool prefilled = false;
	SideStream* ss = !cam->debug ? side_stream() : nullptr;
	if (ss) {
		FwdParams p;
		int rc0 = make_params(cam, gs, p);
		if (rc0 != RGS_OK) return rc0;
		ParamGradOut po{out->dL_dmeans2D, out->dL_dcolors, out->dL_dopacity, out->dL_dmeans3D, out->dL_dcov3D, out->dL_dsh, out->dL_dscales, out->dL_drotations, out->dL_dsh_rest};
		if (cudaEventRecord(ss->fork, s) == cudaSuccess && cudaStreamWaitEvent(ss->stream, ss->fork, 0) == cudaSuccess) {
			launch_backward_zero_fill(p, po, ss->stream);
			prefilled = cudaEventRecord(ss->join, ss->stream) == cudaSuccess;
		}
	}
	int rc = rgs_backward_render(cam, gs, in, acc, cuda_stream);
	if (prefilled && cudaStreamWaitEvent(s, ss->join, 0) != cudaSuccess) return fail(RGS_E_CUDA, "cudaStreamWaitEvent failed");
	if (rc != RGS_OK) return rc;
	return backward_preprocess_impl(cam, gs, in, acc, out, cuda_stream, prefilled);
}

int32_t rgs_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* /*projmatrix*/, uint8_t* present, void* cuda_stream) {
	if (P < 0) return fail(RGS_E_INVALID, "negative Gaussian count");
	if (P == 0) return RGS_OK;
	if (!means3D || !viewmatrix || !present) return fail(RGS_E_INVALID, "null pointer");
	launch_mark_visible(P, means3D, viewmatrix, present, (cudaStream_t)cuda_stream);
	return cuda_status(cudaGetLastError(), "mark visible");
}

int32_t rgs_activate_forward(int32_t P, const float* raw_scaling, const float* raw_opacity, const float* raw_rotation, const float* filter_3D,
                             float* scales, float* opacity, float* rotations, void* cuda_stream) {
	if (P < 0) return fail(RGS_E_INVALID, "negative Gaussian count");
	if (P == 0) return RGS_OK;
	if (!raw_scaling || !raw_opacity || !raw_rotation || !filter_3D || !scales || !opacity || !rotations) return fail(RGS_E_INVALID, "null pointer");
	launch_activate_forward(P, raw_scaling, raw_opacity, raw_rotation, filter_3D, scales, opacity, rotations, (cudaStream_t)cuda_stream);
	return cuda_status(cudaGetLastError(), "activate forward");
}

int32_t rgs_activate_backward(int32_t P, const float* raw_scaling, const float* raw_opacity, const float* raw_rotation, const float* filter_3D,
                              const float* g_scales, const float* g_opacity, const float* g_rotations, float* d_raw_scaling, float* d_raw_opacity,
                              float* d_raw_rotation, void* cuda_stream) {
	if (P < 0) return fail(RGS_E_INVALID, "negative Gaussian count");
	if (P == 0) return RGS_OK;
	if (!raw_scaling || !raw_opacity || !raw_rotation || !filter_3D || !g_scales || !g_opacity || !g_rotations || !d_raw_scaling || !d_raw_opacity ||
	    !d_raw_rotation)
		return fail(RGS_E_INVALID, "null pointer");
	launch_activate_backward(P, raw_scaling, raw_opacity, raw_rotation, filter_3D, g_scales, g_opacity, g_rotations, d_raw_scaling, d_raw_opacity,
	                         d_raw_rotation, (cudaStream_t)cuda_stream);
	return cuda_status(cudaGetLastError(), "activate backward");
}

int32_t rgs_densification_stats(int32_t P, const float* means2D_grad, const int32_t* radii, float* grad_accum, float* grad_accum_abs,
                                float* grad_accum_abs_max, float* denom, float* max_radii2D, void* cuda_stream) {
	if (P < 0) return fail(RGS_E_INVALID, "negative Gaussian count");
	if (P == 0) return RGS_OK;
	if (!means2D_grad || !radii || !grad_accum || !grad_accum_abs || !grad_accum_abs_max || !denom) return fail(RGS_E_INVALID, "null pointer");
	launch_densification_stats(P, means2D_grad, radii, grad_accum, grad_accum_abs, grad_accum_abs_max, denom, max_radii2D, (cudaStream_t)cuda_stream);
	return cuda_status(cudaGetLastError(), "densification stats");
}

int32_t rgs_compute_3d_filter(int32_t P, const float* xyz, int32_t n_cams, const float* cams, float focal_length, float* filter_3D,
                              float* max_distance, void* cuda_stream) {
	if (P < 0 || n_cams < 0) return fail(RGS_E_INVALID, "negative count");
	if (P == 0) return RGS_OK;
	if (!xyz || !filter_3D || !max_distance || (n_cams > 0 && !cams)) return fail(RGS_E_INVALID, "null pointer");
	if (!(focal_length > 0.0f)) return fail(RGS_E_INVALID, "focal_length must be positive");
	launch_compute_3d_filter(P, xyz, n_cams, cams, focal_length, filter_3D, max_distance, (cudaStream_t)cuda_stream);
	return cuda_status(cudaGetLastError(), "compute 3d filter");
}

int32_t rgs_knn_mean_dist2(int32_t P, const float* points, float* mean_dist2, rgs_resize_fn scratch, void* scratch_user, void* cuda_stream) {
	if (P < 0) return fail(RGS_E_INVALID, "negative point count");
	if (P == 0) return RGS_OK;
	if (!points || !mean_dist2 || !scratch) return fail(RGS_E_INVALID, "null pointer");
	char* buf;
	if (const int rc = grow(scratch, scratch_user, knn_scratch_bytes(P), buf, "knn scratch")) return rc;
	return cuda_status(launch_knn_mean_dist2(P, points, mean_dist2, buf, (cudaStream_t)cuda_stream), "knn");
}

// ---- TSDF grid (rgs_tsdf.cu) ----

static bool pow2(int64_t n) { return n > 0 && (n & (n - 1)) == 0; }
static bool finite_pos(float x) { return std::isfinite(x) && x > 0.0f; }

static int tsdf_grid_check(const rgs_tsdf_grid* g) {
	if (!g) return fail(RGS_E_INVALID, "null grid");
	if (!finite_pos(g->voxel_size)) return fail(RGS_E_INVALID, "voxel_size must be positive and finite");
	if (g->capacity <= 0 || g->capacity > (INT32_MAX / (RGS_TSDF_BLOCK_RES * RGS_TSDF_BLOCK_RES * RGS_TSDF_BLOCK_RES)))
		return fail(RGS_E_INVALID, "grid capacity must be in [1, 524287] blocks");
	if (!pow2(g->hash_slots) || g->hash_slots < 2 * g->capacity) return fail(RGS_E_INVALID, "hash_slots must be a power of two >= 2 * capacity");
	if (!pow2(g->frame_slots) || g->frame_slots < 2 || g->frame_slots > ((int64_t)1 << 31))
		return fail(RGS_E_INVALID, "frame_slots must be a power of two in [2, 2^31]");
	if (!g->hash_keys || !g->hash_values || !g->tsdf || !g->weight || !g->color || !g->stamps || !g->frame_keys || !g->frame_list || !g->counters)
		return fail(RGS_E_INVALID, "null grid array");
	return RGS_OK;
}

static int tsdf_camera_check(const rgs_tsdf_grid* g, const rgs_tsdf_camera* c) {
	if (!c) return fail(RGS_E_INVALID, "null camera");
	if (c->width <= 0 || c->height <= 0) return fail(RGS_E_INVALID, "image size must be positive");
	if (!std::isfinite(c->fx) || !std::isfinite(c->fy) || c->fx == 0.0f || c->fy == 0.0f || !std::isfinite(c->cx) || !std::isfinite(c->cy))
		return fail(RGS_E_INVALID, "intrinsics must be finite with nonzero focal lengths");
	for (int i = 0; i < 9; i++)
		if (!std::isfinite(c->R[i])) return fail(RGS_E_INVALID, "extrinsic must be finite");
	for (int i = 0; i < 3; i++)
		if (!std::isfinite(c->t[i])) return fail(RGS_E_INVALID, "extrinsic must be finite");
	if (!finite_pos(c->depth_scale) || !finite_pos(c->depth_max) || !finite_pos(c->trunc_voxel_multiplier))
		return fail(RGS_E_INVALID, "depth_scale, depth_max and trunc_voxel_multiplier must be positive and finite");
	// camera centre +- (depth_max + trunc) must stay inside the block-key range (the keys must never wrap)
	const double reach = (double)c->depth_max + (double)c->trunc_voxel_multiplier * (double)g->voxel_size;
	const double bs = (double)g->voxel_size * RGS_TSDF_BLOCK_RES;
	for (int k = 0; k < 3; k++) {
		const double ck = -((double)c->R[k] * c->t[0] + (double)c->R[3 + k] * c->t[1] + (double)c->R[6 + k] * c->t[2]);
		const double lo = std::floor((ck - reach) / bs), hi = std::floor((ck + reach) / bs);
		if (!(lo >= -(1 << 20) + 1 && hi <= (1 << 20) - 2))
			return fail(RGS_E_INVALID, "camera out of the grid's key range: centre +- (depth_max + trunc) must lie within 2^20 - 2 blocks of the origin");
	}
	return RGS_OK;
}

// counters[0..3] to the host; fails when an earlier call left the grid incomplete
static int tsdf_read_counters(const rgs_tsdf_grid* g, int32_t* cnt, cudaStream_t s) {
	cudaError_t e = cudaMemcpyAsync(cnt, g->counters, 4 * sizeof(int32_t), cudaMemcpyDeviceToHost, s);
	if (e == cudaSuccess) e = cudaStreamSynchronize(s);
	return cuda_status(e, "tsdf");
}

static int tsdf_flags_check(const int32_t* cnt) {
	if (cnt[2] & RGS_TSDF_BAD_COORD) return fail(RGS_E_INVALID, "tsdf: an integrate call was given a block coordinate outside [-2^20, 2^20)");
	if (cnt[2] & RGS_TSDF_OVERFLOW) return fail(RGS_E_INVALID, "tsdf: an integrate call found no free block slot; the grid is incomplete");
	return RGS_OK;
}

int64_t rgs_tsdf_touch(const rgs_tsdf_grid* grid, const rgs_tsdf_camera* cam, const float* depth, int32_t* block_coords, int64_t* allocated,
                       rgs_resize_fn scratch, void* scratch_user, void* cuda_stream) {
	int rc = tsdf_grid_check(grid);
	if (rc == RGS_OK) rc = tsdf_camera_check(grid, cam);
	if (rc != RGS_OK) return rc;
	if (!depth || !block_coords || !scratch) return fail(RGS_E_INVALID, "null pointer");
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	int32_t cnt[4];
	if ((rc = cuda_status(launch_tsdf_touch(*grid, *cam, depth, cnt, s), "tsdf touch")) != RGS_OK) return rc;
	if ((rc = tsdf_flags_check(cnt)) != RGS_OK) return rc;
	if (allocated) *allocated = cnt[0];
	if (cnt[3] || cnt[1] > grid->frame_slots / 2) return fail(RGS_E_CAPACITY, "tsdf touch: more blocks than the frame-local hash holds");
	const int64_t n = cnt[1];
	if (n == 0) return 0;
	char* buf;
	if ((rc = grow(scratch, scratch_user, tsdf_touch_scratch_bytes(n), buf, "tsdf scratch")) != RGS_OK) return rc;
	if ((rc = cuda_status(launch_tsdf_touch_sort(*grid, n, block_coords, buf, s), "tsdf touch")) != RGS_OK) return rc;
	return n;
}

int32_t rgs_tsdf_integrate(const rgs_tsdf_grid* grid, const rgs_tsdf_camera* cam, int64_t n, const int32_t* block_coords, const float* depth,
                           const float* color, int32_t call_id, rgs_resize_fn scratch, void* scratch_user, void* cuda_stream) {
	int rc = tsdf_grid_check(grid);
	if (rc == RGS_OK) rc = tsdf_camera_check(grid, cam);
	if (rc != RGS_OK) return rc;
	if (n < 0 || n > INT32_MAX) return fail(RGS_E_INVALID, "block count out of range");
	if (call_id <= 0) return fail(RGS_E_INVALID, "call_id must be positive");
	if (n == 0) return RGS_OK;
	if (!block_coords || !depth || !color || !scratch) return fail(RGS_E_INVALID, "null pointer");
	char* buf;
	if ((rc = grow(scratch, scratch_user, (size_t)n * sizeof(int32_t), buf, "tsdf scratch")) != RGS_OK) return rc;
	return cuda_status(launch_tsdf_integrate(*grid, *cam, n, block_coords, depth, color, call_id, reinterpret_cast<int32_t*>(buf), (cudaStream_t)cuda_stream),
	                 "tsdf integrate");
}

int32_t rgs_tsdf_rehash(const rgs_tsdf_grid* grid, const uint64_t* old_keys, const int32_t* old_values, int64_t old_slots, void* cuda_stream) {
	const int rc = tsdf_grid_check(grid);
	if (rc != RGS_OK) return rc;
	if (old_slots < 0) return fail(RGS_E_INVALID, "negative slot count");
	if (old_slots == 0) return RGS_OK;
	if (!old_keys || !old_values) return fail(RGS_E_INVALID, "null pointer");
	return cuda_status(launch_tsdf_rehash(*grid, old_keys, old_values, old_slots, (cudaStream_t)cuda_stream), "tsdf rehash");
}

int64_t rgs_tsdf_active_blocks(const rgs_tsdf_grid* grid, uint64_t* keys, int32_t* pool_index, rgs_resize_fn scratch, void* scratch_user, void* cuda_stream) {
	int rc = tsdf_grid_check(grid);
	if (rc != RGS_OK) return rc;
	if (!keys || !pool_index || !scratch) return fail(RGS_E_INVALID, "null pointer");
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	int32_t cnt[4];
	if ((rc = tsdf_read_counters(grid, cnt, s)) != RGS_OK || (rc = tsdf_flags_check(cnt)) != RGS_OK) return rc;
	const int N = cnt[0];
	if (N == 0) return 0;
	char* buf;
	if ((rc = grow(scratch, scratch_user, tsdf_active_scratch_bytes(N), buf, "tsdf scratch")) != RGS_OK) return rc;
	if ((rc = cuda_status(launch_tsdf_active(*grid, N, keys, pool_index, buf, s), "tsdf active blocks")) != RGS_OK) return rc;
	return N;
}

int32_t rgs_tsdf_extract(const rgs_tsdf_grid* grid, float weight_threshold, rgs_resize_fn resize, rgs_tsdf_mesh_out* out, void* scratch_user,
                         void* cuda_stream) {
	int rc = tsdf_grid_check(grid);
	if (rc != RGS_OK) return rc;
	if (!resize || !out) return fail(RGS_E_INVALID, "null pointer");
	if (std::isnan(weight_threshold)) return fail(RGS_E_INVALID, "weight_threshold is NaN");
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	int32_t cnt[4];
	if ((rc = tsdf_read_counters(grid, cnt, s)) != RGS_OK || (rc = tsdf_flags_check(cnt)) != RGS_OK) return rc;
	const int N = cnt[0];
	int64_t totals[2] = {0, 0};
	char* buf = nullptr;
	if (N > 0) {
		if ((rc = grow(resize, scratch_user, tsdf_extract_scratch_bytes(*grid, N), buf, "tsdf scratch")) != RGS_OK) return rc;
		if ((rc = cuda_status(launch_tsdf_extract_count(*grid, N, weight_threshold, buf, totals, s), "tsdf extract")) != RGS_OK) return rc;
	}
	out->num_vertices = totals[0];
	out->num_triangles = totals[1];
	char *v, *c, *t;
	if ((rc = grow(resize, out->vertices_user, (size_t)totals[0] * 3 * sizeof(float), v, "tsdf mesh")) != RGS_OK ||
	    (rc = grow(resize, out->colors_user, (size_t)totals[0] * 3 * sizeof(float), c, "tsdf mesh")) != RGS_OK ||
	    (rc = grow(resize, out->triangles_user, (size_t)totals[1] * 3 * sizeof(int32_t), t, "tsdf mesh")) != RGS_OK)
		return rc;
	if (N == 0) return RGS_OK;
	return cuda_status(launch_tsdf_extract_emit(*grid, N, buf, reinterpret_cast<float*>(v), reinterpret_cast<float*>(c), reinterpret_cast<int32_t*>(t), s),
	                 "tsdf extract");
}

int32_t rgs_tsdf_vertex_normals(int64_t V, const float* vertices, int64_t F, const int32_t* triangles, float* normals, rgs_resize_fn scratch,
                                void* scratch_user, void* cuda_stream) {
	if (V < 0 || F < 0 || V > INT32_MAX || 3 * F > INT32_MAX) return fail(RGS_E_INVALID, "vertex / triangle count out of range");
	if (V == 0) return F == 0 ? (int32_t)RGS_OK : fail(RGS_E_INVALID, "triangles without vertices");
	if (!vertices || !normals || !scratch || (F > 0 && !triangles)) return fail(RGS_E_INVALID, "null pointer");
	char* buf;
	if (const int rc = grow(scratch, scratch_user, tsdf_normals_scratch_bytes(V, F), buf, "tsdf scratch")) return rc;
	return cuda_status(launch_tsdf_normals(V, vertices, F, triangles, normals, buf, (cudaStream_t)cuda_stream), "tsdf vertex normals");
}

// ---- DTU evaluation (rgs_dtu_eval.cu) ----

int32_t rgs_dtu_sample_mesh(int64_t V, const double* vertices, int64_t F, const int32_t* faces, double density, rgs_resize_fn resize,
                            rgs_dtu_samples_out* out, void* cuda_stream) {
	if (V < 0 || F < 0 || V > INT32_MAX || F > INT32_MAX - 1) return fail(RGS_E_INVALID, "dtu sample: vertex / face count out of range");
	if (!resize || !out || (V > 0 && !vertices) || (F > 0 && !faces)) return fail(RGS_E_INVALID, "null pointer");
	if (!(std::isfinite(density) && density > 0.0)) return fail(RGS_E_INVALID, "dtu sample: density must be positive and finite");
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	int rc;
	int64_t totals[2] = {0, 0};   // samples, rows
	char* buf = nullptr;
	if (F > 0) {
		if (V == 0) return fail(RGS_E_INVALID, "dtu sample: faces without vertices");
		if ((rc = grow(resize, out->scratch_user, dtu_sample_scratch_bytes(F), buf, "dtu sample scratch")) != RGS_OK ||
		    (rc = cuda_status(launch_dtu_sample_count(V, vertices, F, faces, density, buf, totals, s), "dtu sample")) != RGS_OK)
			return rc;
		if (V + totals[0] > INT32_MAX)
			return fail(RGS_E_INVALID, "dtu sample: more than 2^31 - 1 points (or a face index outside [0, V), or a triangle whose sample count is not finite)");
	}
	out->num_points = V + totals[0];
	char *rows = nullptr, *pts;
	if ((totals[0] > 0 && (rc = grow(resize, out->rows_user, dtu_sample_rows_bytes(totals[1]), rows, "dtu sample")) != RGS_OK) ||
	    (rc = grow(resize, out->points_user, (size_t)out->num_points * 3 * sizeof(double), pts, "dtu sample")) != RGS_OK)
		return rc;
	if (out->num_points == 0) return RGS_OK;
	return cuda_status(launch_dtu_sample_emit(V, vertices, F, faces, density, buf, totals[0], totals[1], rows, reinterpret_cast<double*>(pts), s), "dtu sample", kNonFinitePoint);
}

int32_t rgs_dtu_radius_downsample(int64_t N, const double* points, double radius, uint8_t* kept, int32_t* rounds, rgs_resize_fn scratch,
                                  void* scratch_user, void* cuda_stream) {
	if (rounds) *rounds = 0;
	if (N < 0 || N > INT32_MAX) return fail(RGS_E_INVALID, "dtu downsample: point count out of range");
	if (!(std::isfinite(radius) && radius > 0.0)) return fail(RGS_E_INVALID, "dtu downsample: radius must be positive and finite");
	if (N == 0) return RGS_OK;
	if (!points || !kept || !scratch) return fail(RGS_E_INVALID, "null pointer");
	char* buf;
	if (const int rc = grow(scratch, scratch_user, dtu_downsample_scratch_bytes((int)N), buf, "dtu downsample scratch")) return rc;
	return cuda_status(launch_dtu_downsample((int)N, points, radius, kept, buf, rounds, (cudaStream_t)cuda_stream), "dtu downsample", kNonFinitePoint);
}

int32_t rgs_dtu_nearest(int64_t M, const double* reference, int64_t N, const double* query, double* dist, int64_t* index, rgs_resize_fn scratch,
                        void* scratch_user, void* cuda_stream) {
	if (M < 0 || N < 0 || M > INT32_MAX || N > INT32_MAX) return fail(RGS_E_INVALID, "dtu nearest: point count out of range");
	if (M == 0) return fail(RGS_E_INVALID, "dtu nearest: the reference set is empty");
	if (!reference || !scratch || (N > 0 && (!query || !dist || !index))) return fail(RGS_E_INVALID, "null pointer");
	char* buf;
	if (const int rc = grow(scratch, scratch_user, dtu_nearest_scratch_bytes((int)M, (int)N), buf, "dtu nearest scratch")) return rc;
	return cuda_status(launch_dtu_nearest((int)M, reference, (int)N, query, dist, index, buf, (cudaStream_t)cuda_stream), "dtu nearest", kNonFinitePoint);
}

int32_t rgs_dtu_dilate_masks(int32_t n_views, int32_t H, int32_t W, const uint8_t* masks, uint8_t* dilated, void* cuda_stream) {
	if (n_views < 0 || H <= 0 || W <= 0) return fail(RGS_E_INVALID, "dtu dilate: image size must be positive");
	if (n_views > 0 && (!masks || !dilated)) return fail(RGS_E_INVALID, "null pointer");
	return cuda_status(launch_dtu_dilate(n_views, H, W, masks, dilated, (cudaStream_t)cuda_stream), "dtu dilate", kNonFinitePoint);
}

int32_t rgs_dtu_cull_vertices(int64_t V, const double* vertices, int32_t n_views, int32_t H, int32_t W, const double* proj, const uint8_t* dilated,
                              uint8_t* keep, void* cuda_stream) {
	if (V < 0 || n_views < 0 || H <= 0 || W <= 0) return fail(RGS_E_INVALID, "dtu cull: negative count or empty image");
	if (V > 0 && (!vertices || !keep || (n_views > 0 && (!proj || !dilated)))) return fail(RGS_E_INVALID, "null pointer");
	return cuda_status(launch_dtu_cull(V, vertices, n_views, H, W, proj, dilated, keep, (cudaStream_t)cuda_stream), "dtu cull", kNonFinitePoint);
}

// ---- TNT evaluation (rgs_tnt_eval.cu) ----

static int tnt_check_transform(const double* T, const char* what) {
	if (!T) return RGS_OK;
	for (int k = 0; k < 16; k++)
		if (!std::isfinite(T[k])) return fail(RGS_E_INVALID, std::string(what) + ": the transform has a NaN or infinite entry");
	if (T[12] != 0.0 || T[13] != 0.0 || T[14] != 0.0 || T[15] != 1.0) return fail(RGS_E_INVALID, std::string(what) + ": the transform's last row must be (0 0 0 1)");
	return RGS_OK;
}

int32_t rgs_tnt_crop(int64_t N, const double* points, const double* transform, const rgs_tnt_crop_volume* volume, uint8_t* kept, double* cropped,
                     int64_t* num_kept, rgs_resize_fn scratch, void* scratch_user, void* cuda_stream) {
	if (N < 0 || N > INT32_MAX) return fail(RGS_E_INVALID, "tnt crop: point count out of range");
	if (!num_kept) return fail(RGS_E_INVALID, "null pointer");
	*num_kept = 0;
	if (const int rc = tnt_check_transform(transform, "tnt crop")) return rc;
	if (volume) {
		if (volume->orthogonal_axis < 0 || volume->orthogonal_axis > 2) return fail(RGS_E_INVALID, "tnt crop: orthogonal_axis must be 0, 1 or 2");
		if (volume->num_vertices < 3 || volume->num_vertices > 2048) return fail(RGS_E_INVALID, "tnt crop: the polygon needs 3 to 2048 vertices");
		if (!volume->polygon) return fail(RGS_E_INVALID, "null pointer");
		if (std::isnan(volume->axis_min) || std::isnan(volume->axis_max)) return fail(RGS_E_INVALID, "tnt crop: axis_min / axis_max is NaN");
	}
	if (N == 0) return RGS_OK;
	if (!points || !kept || !cropped || !scratch) return fail(RGS_E_INVALID, "null pointer");
	char* buf;
	if (const int rc = grow(scratch, scratch_user, tnt_crop_scratch_bytes((int)N), buf, "tnt crop scratch")) return rc;
	const cudaError_t e = launch_tnt_crop((int)N, points, transform, volume ? volume->orthogonal_axis : 0, volume ? volume->axis_min : 0.0,
	                                      volume ? volume->axis_max : 0.0, volume ? volume->num_vertices : 0, volume ? volume->polygon : nullptr, kept,
	                                      cropped, num_kept, buf, (cudaStream_t)cuda_stream);
	return cuda_status(e, "tnt crop", kNonFinitePoint);
}

int32_t rgs_tnt_transform(int64_t N, double* points, const double* transform, void* cuda_stream) {
	if (N < 0 || N > INT32_MAX) return fail(RGS_E_INVALID, "tnt transform: point count out of range");
	if (!transform) return fail(RGS_E_INVALID, "null pointer");
	if (const int rc = tnt_check_transform(transform, "tnt transform")) return rc;
	if (N > 0 && !points) return fail(RGS_E_INVALID, "null pointer");
	return cuda_status(launch_tnt_transform(N, points, transform, (cudaStream_t)cuda_stream), "tnt transform", kNonFinitePoint);
}

int32_t rgs_tnt_voxel_downsample(int64_t N, const double* points, double voxel, rgs_resize_fn resize, rgs_tnt_voxel_out* out, void* cuda_stream) {
	if (!resize || !out) return fail(RGS_E_INVALID, "null pointer");
	out->num_voxels = 0;
	if (N < 0 || N > INT32_MAX) return fail(RGS_E_INVALID, "tnt voxel: point count out of range");
	if (!(std::isfinite(voxel) && voxel > 0.0)) return fail(RGS_E_INVALID, "tnt voxel: voxel size must be positive and finite");
	if (N > 0 && !points) return fail(RGS_E_INVALID, "null pointer");
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	int rc;
	double lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0}, origin[3] = {0, 0, 0};
	if (N > 0) {
		char* bbuf;
		int64_t bad = 0;
		if ((rc = grow(resize, out->scratch_user, tnt_bounds_scratch_bytes(), bbuf, "tnt voxel scratch")) != RGS_OK ||
		    (rc = cuda_status(launch_tnt_bounds((int)N, points, bbuf, lo, hi, &bad, s), "tnt voxel")) != RGS_OK)
			return rc;
		if (bad) return fail(RGS_E_INVALID, "tnt voxel: a point has a NaN or infinite coordinate");
		for (int a = 0; a < 3; a++) {
			origin[a] = lo[a] - voxel * 0.5;
			const double top = std::floor((hi[a] - origin[a]) / voxel);
			if (!(top < 2097152.0)) return fail(RGS_E_INVALID, "tnt voxel: more than 2^21 voxels along an axis");
		}
	}
	char* buf = nullptr;
	int32_t V = 0;
	if (N > 0 && ((rc = grow(resize, out->scratch_user, tnt_voxel_scratch_bytes((int)N), buf, "tnt voxel scratch")) != RGS_OK ||
	              (rc = cuda_status(launch_tnt_voxel_sort((int)N, points, origin, voxel, buf, &V, s), "tnt voxel")) != RGS_OK))
		return rc;
	out->num_voxels = V;
	char *means, *counts;
	if ((rc = grow(resize, out->means_user, (size_t)V * 3 * sizeof(double), means, "tnt voxel")) != RGS_OK ||
	    (rc = grow(resize, out->counts_user, (size_t)V * sizeof(int64_t), counts, "tnt voxel")) != RGS_OK)
		return rc;
	if (V == 0) return RGS_OK;
	return cuda_status(launch_tnt_voxel_mean((int)N, points, V, buf, reinterpret_cast<double*>(means), reinterpret_cast<int64_t*>(counts), s), "tnt voxel", kNonFinitePoint);
}

int32_t rgs_tnt_icp_moments(int64_t N, const double* source, int64_t M, const double* target, const double* dist, const int64_t* index, double threshold,
                            double* moments, rgs_resize_fn scratch, void* scratch_user, void* cuda_stream) {
	if (N < 0 || M < 0 || N > INT32_MAX || M > INT32_MAX) return fail(RGS_E_INVALID, "tnt moments: point count out of range");
	if (std::isnan(threshold)) return fail(RGS_E_INVALID, "tnt moments: the threshold is NaN");
	if (!moments || !scratch || (N > 0 && (!source || !dist || !index)) || (M > 0 && !target)) return fail(RGS_E_INVALID, "null pointer");
	char* buf;
	if (const int rc = grow(scratch, scratch_user, tnt_moments_scratch_bytes(N), buf, "tnt moments scratch")) return rc;
	return cuda_status(launch_tnt_moments(N, source, M, target, dist, index, threshold, buf, moments, (cudaStream_t)cuda_stream), "tnt moments",
	                   "a point or a distance is NaN or infinite");
}

// ---- tetrahedra mesh extraction (rgs_tetra.cu) ----

int32_t rgs_tetra_points(int64_t P, const float* xyz, const float* scaling, const float* rotation, float* points, float* scales, void* cuda_stream) {
	if (P < 0 || 9 * P > INT32_MAX) return fail(RGS_E_INVALID, "tetra points: Gaussian count out of range");
	if (P == 0) return RGS_OK;
	if (!xyz || !scaling || !rotation || !points || !scales) return fail(RGS_E_INVALID, "null pointer");
	return cuda_status(launch_tetra_points((int)P, xyz, scaling, rotation, points, scales, (cudaStream_t)cuda_stream), "tetra points");
}

int32_t rgs_tetra_cull_add(int64_t N, const float* alpha, const float* coord, int32_t H, int32_t W, const float* render7, const float* gt_mask,
                           float* final_alpha, int32_t* weight, void* cuda_stream) {
	if (N < 0 || H <= 0 || W <= 0) return fail(RGS_E_INVALID, "tetra cull: negative point count or empty image");
	if (N == 0) return RGS_OK;
	if (!alpha || !coord || !render7 || !final_alpha || !weight) return fail(RGS_E_INVALID, "null pointer");
	return cuda_status(launch_tetra_cull_add(N, alpha, coord, H, W, render7, gt_mask, final_alpha, weight, (cudaStream_t)cuda_stream), "tetra cull");
}

int32_t rgs_tetra_cull_finish(int64_t N, const float* final_alpha, const int32_t* weight, float* sdf, void* cuda_stream) {
	if (N < 0) return fail(RGS_E_INVALID, "tetra cull: negative point count");
	if (N == 0) return RGS_OK;
	if (!final_alpha || !weight || !sdf) return fail(RGS_E_INVALID, "null pointer");
	return cuda_status(launch_tetra_cull_finish(N, final_alpha, weight, sdf, (cudaStream_t)cuda_stream), "tetra cull finish");
}

int32_t rgs_tetra_marching(int64_t N, const float* points, const float* sdf, const float* scales, int64_t T, const int64_t* tets, rgs_resize_fn resize,
                           rgs_tetra_march_out* out, void* cuda_stream) {
	if (!resize || !out) return fail(RGS_E_INVALID, "null pointer");
	out->num_vertices = out->num_faces = 0;
	if (N < 0 || N > INT32_MAX || T < 0 || T > INT32_MAX) return fail(RGS_E_INVALID, "tetra marching: point or tet count out of range");
	if ((N > 0 && (!points || !sdf || !scales)) || (T > 0 && !tets)) return fail(RGS_E_INVALID, "null pointer");
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	int rc;
	int32_t V = 0, M = 0, F = 0;
	char* s1 = nullptr;
	if (T > 0) {
		int32_t bad = 0;
		if ((rc = grow(resize, out->scratch_user, tetra_march_scratch1_bytes(T), s1, "tetra marching scratch")) != RGS_OK ||
		    (rc = cuda_status(launch_tetra_march_valid(T, N, tets, sdf, s1, &bad, &V, s), "tetra marching")) != RGS_OK)
			return rc;
		if (bad) return fail(RGS_E_INVALID, "tetra marching: a tet index lies outside [0, N)");
		if (V > (INT32_MAX - 255) / 6) return fail(RGS_E_INVALID, "tetra marching: too many valid tets (6 x valid must stay below 2^31)");
	}
	char* s2 = nullptr;
	if (V > 0) {
		if ((rc = grow(resize, out->sort_user, tetra_march_scratch2_bytes(V), s2, "tetra marching scratch")) != RGS_OK ||
		    (rc = cuda_status(launch_tetra_march_sort(T, N, tets, sdf, V, s1, s2, &M, &F, s), "tetra marching")) != RGS_OK)
			return rc;
	}
	char *interp, *ends, *end_sdf, *end_scl, *faces;
	if ((rc = grow(resize, out->interp_user, (size_t)M * 2 * sizeof(int64_t), interp, "tetra marching")) != RGS_OK ||
	    (rc = grow(resize, out->ends_user, (size_t)M * 6 * sizeof(float), ends, "tetra marching")) != RGS_OK ||
	    (rc = grow(resize, out->end_sdf_user, (size_t)M * 2 * sizeof(float), end_sdf, "tetra marching")) != RGS_OK ||
	    (rc = grow(resize, out->end_scales_user, (size_t)M * 2 * sizeof(float), end_scl, "tetra marching")) != RGS_OK ||
	    (rc = grow(resize, out->faces_user, (size_t)F * 3 * sizeof(int64_t), faces, "tetra marching")) != RGS_OK)
		return rc;
	out->num_vertices = M;
	out->num_faces = F;
	if (V == 0) return RGS_OK;
	return cuda_status(launch_tetra_march_emit(T, points, sdf, scales, V, s1, s2, N, reinterpret_cast<int64_t*>(interp), reinterpret_cast<float*>(ends),
	                                          reinterpret_cast<float*>(end_sdf), reinterpret_cast<float*>(end_scl), reinterpret_cast<int64_t*>(faces), s),
	                  "tetra marching");
}

int32_t rgs_tetra_bisect(int64_t M, const float* mid_sdf, float* left, float* right, float* left_sdf, float* right_sdf, float* mid, void* cuda_stream) {
	if (M < 0) return fail(RGS_E_INVALID, "tetra bisect: negative vertex count");
	if (M == 0) return RGS_OK;
	if (!left || !right || !mid || (mid_sdf && (!left_sdf || !right_sdf))) return fail(RGS_E_INVALID, "null pointer");
	return cuda_status(launch_tetra_bisect(M, mid_sdf, left, right, left_sdf, right_sdf, mid, (cudaStream_t)cuda_stream), "tetra bisect");
}

int32_t rgs_tetra_filter(int64_t M, const float* points, const float* ends, const float* end_scales, int64_t F, const int64_t* faces, rgs_resize_fn resize,
                         rgs_tetra_filter_out* out, void* cuda_stream) {
	if (!resize || !out) return fail(RGS_E_INVALID, "null pointer");
	out->num_vertices = out->num_faces = 0;
	if (M < 0 || M > INT32_MAX || F < 0 || F > INT32_MAX) return fail(RGS_E_INVALID, "tetra filter: vertex or face count out of range");
	if ((M > 0 && (!points || !ends || !end_scales)) || (F > 0 && !faces)) return fail(RGS_E_INVALID, "null pointer");
	if (M == 0 && F > 0) return fail(RGS_E_INVALID, "tetra filter: faces without vertices");
	char *verts, *fout, *buf;
	int rc;
	if ((rc = grow(resize, out->vertices_user, (size_t)M * 3 * sizeof(float), verts, "tetra filter")) != RGS_OK ||
	    (rc = grow(resize, out->faces_user, (size_t)F * 3 * sizeof(int64_t), fout, "tetra filter")) != RGS_OK)
		return rc;
	if (M == 0) return RGS_OK;
	int64_t nv = 0, nf = 0;
	int32_t bad = 0;
	if ((rc = grow(resize, out->scratch_user, tetra_filter_scratch_bytes((int)M, F), buf, "tetra filter scratch")) != RGS_OK ||
	    (rc = cuda_status(launch_tetra_filter((int)M, points, ends, end_scales, F, faces, buf, reinterpret_cast<float*>(verts),
	                                          reinterpret_cast<int64_t*>(fout), &nv, &nf, &bad, (cudaStream_t)cuda_stream),
	                      "tetra filter")) != RGS_OK)
		return rc;
	if (bad) return fail(RGS_E_INVALID, "tetra filter: a face index lies outside [0, M)");
	out->num_vertices = nv;
	out->num_faces = nf;
	return RGS_OK;
}

// ---- Delaunay tetrahedralization (rgs_delaunay.cu) ----

int32_t rgs_delaunay(int64_t N, const float* points, rgs_resize_fn resize, rgs_delaunay_out* out, void* cuda_stream) {
	if (!resize || !out) return fail(RGS_E_INVALID, "null pointer");
	out->num_cells = 0;
	out->rounds = out->max_cavity = out->overflowed = out->alone = out->mesh_growths = 0;
	if (N < 0 || N > RGS_DELAUNAY_MAX_POINTS) return fail(RGS_E_INVALID, "delaunay: point count out of range (at most 2^26)");
	if (N > 0 && !points) return fail(RGS_E_INVALID, "null pointer");
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	constexpr int64_t MAX_CELLS = (int64_t)1 << 29;
	int rc;
	char* cells_out = nullptr;
	if (N == 0) return grow(resize, out->cells_user, 0, cells_out, "delaunay");

	size_t bytes = 0;
	char* pbuf = nullptr;
	carve_dt_points(nullptr, (int)N, &bytes);
	if ((rc = grow(resize, out->points_user, bytes, pbuf, "delaunay scratch")) != RGS_OK) return rc;
	const DtPointsView v = carve_dt_points(pbuf, (int)N, nullptr);
	DtCounters h;
	if ((rc = cuda_status(launch_dt_prepare((int)N, points, v, &h, s), "delaunay")) != RGS_OK) return rc;
	if (h.bad) return fail(RGS_E_INVALID, "delaunay: a coordinate is not finite or exceeds 2^90 in magnitude");
	const int n = (int)h.unique;
	if (n < 4) return grow(resize, out->cells_user, 0, cells_out, "delaunay");

	int cur = 0;
	int64_t cap = std::min<int64_t>(8 * (int64_t)n + 64, MAX_CELLS);
	char* mbuf = nullptr;
	carve_dt_mesh(nullptr, cap, &bytes);
	if ((rc = grow(resize, out->mesh_user[0], bytes, mbuf, "delaunay mesh")) != RGS_OK) return rc;
	DtMesh m = carve_dt_mesh(mbuf, cap, nullptr);
	if ((rc = cuda_status(launch_dt_init((int)N, points, n, v, h, m, cap, s), "delaunay")) != RGS_OK) return rc;

	const int K = std::min(DT_MAX_SLOTS, n);
	int64_t cc_total = (int64_t)K * DT_SLOT_CELLS, cb_total = (int64_t)K * DT_SLOT_FACES;
	DtSlots sl;
	auto slabs = [&]() -> int {
		char* buf = nullptr;
		carve_dt_slots(nullptr, K, cc_total, cb_total, &bytes);
		const int r = grow(resize, out->slab_user, bytes, buf, "delaunay slabs");
		sl = carve_dt_slots(buf, K, cc_total, cb_total, nullptr);
		return r;
	};
	// the mesh moves into the other buffer at (at least) twice the size; dead rows fill the new tail
	auto grow_mesh = [&](int64_t want) -> int {
		const int64_t nc = std::min(std::max(2 * cap, want), MAX_CELLS);
		if (nc < want || nc <= cap) return fail(RGS_E_CAPACITY, "delaunay: the mesh needs more than 2^29 cells");
		char* buf = nullptr;
		carve_dt_mesh(nullptr, nc, &bytes);
		if (const int r = grow(resize, out->mesh_user[1 - cur], bytes, buf, "delaunay mesh")) return r;
		const DtMesh nm = carve_dt_mesh(buf, nc, nullptr);
		if (const int r = cuda_status(launch_dt_grow_mesh(m, cap, nm, nc, s), "delaunay")) return r;
		m = nm;
		cap = nc;
		cur = 1 - cur;
		out->mesh_growths++;
		return RGS_OK;
	};
	auto checked = [&](const DtCounters& c) -> int {
		return c.violation ? fail(RGS_E_CUDA, "delaunay: a new cell is not positively oriented or a point found no cell (predicate bug)") : RGS_OK;
	};
	if ((rc = slabs()) != RGS_OK) return rc;

	// Every pass can leave the device's cell counter above the capacity (a winner that found no room has added its cells
	// already); the mesh then grows to at least twice that count, so `cells`, the extent the next pass initialises and
	// scans, is the device's count.
	int epoch = 0, cells = 1;
	auto after_pass = [&]() -> int {
		if (const int r = checked(h)) return r;
		if (h.full)
			if (const int r = grow_mesh(2 * (int64_t)h.cells)) return r;
		cells = (int)std::min<int64_t>(h.cells, cap);
		return RGS_OK;
	};
	// the cavities too large for a round's slot go in right after it, several at once, in slots 16 times as large
	const int KL = std::max(1, K / 16);
	while ((int)h.inserted < n) {
		out->rounds++;
		if ((rc = cuda_status(launch_dt_round(n, v, m, sl, K, DT_SLOT_CELLS, DT_SLOT_FACES, ++epoch, cap, cells, s), "delaunay")) != RGS_OK ||
		    (rc = cuda_status(launch_dt_read(v, &h, s), "delaunay")) != RGS_OK || (rc = after_pass()) != RGS_OK)
			return rc;
		if (h.overflowed == 0) continue;
		out->overflowed += h.overflowed;
		if ((rc = cuda_status(launch_dt_large(n, v, m, sl, KL, (int)(cc_total / KL), (int)(cb_total / KL), ++epoch, cap, cells, s), "delaunay")) != RGS_OK ||
		    (rc = cuda_status(launch_dt_read(v, &h, s), "delaunay")) != RGS_OK || (rc = after_pass()) != RGS_OK)
			return rc;
		// one still larger: the smallest such point goes in alone, with the whole slab area (grown as needed)
		while (h.overflowed > 0) {
			if ((rc = cuda_status(launch_dt_single_cavity(v, m, sl, cc_total, cb_total, cells, s), "delaunay")) != RGS_OK ||
			    (rc = cuda_status(launch_dt_read(v, &h, s), "delaunay")) != RGS_OK)
				return rc;
			if (h.overflowed) {
				cc_total *= 2;
				cb_total *= 2;
				if (cc_total > MAX_CELLS) return fail(RGS_E_CAPACITY, "delaunay: a cavity exceeds 2^29 cells");
				if ((rc = slabs()) != RGS_OK) return rc;
				continue;
			}
			if ((rc = cuda_status(launch_dt_single_star(n, v, m, sl, cc_total, cb_total, ++epoch, cap, s), "delaunay")) != RGS_OK ||
			    (rc = cuda_status(launch_dt_read(v, &h, s), "delaunay")) != RGS_OK || (rc = after_pass()) != RGS_OK)
				return rc;
			if (!h.full) {
				out->alone++;
				break;
			}
			h.overflowed = 1;
		}
	}
	out->max_cavity = h.max_cavity;

	char* sbuf = nullptr;
	int T = 0;
	if ((rc = grow(resize, out->sort_user, dt_sort_bytes(cells), sbuf, "delaunay sort")) != RGS_OK ||
	    (rc = cuda_status(launch_dt_emit(n, v, m, sbuf, cells, &T, s), "delaunay")) != RGS_OK ||
	    (rc = grow(resize, out->cells_user, (size_t)T * 4 * sizeof(int32_t), cells_out, "delaunay")) != RGS_OK ||
	    (rc = cuda_status(launch_dt_sort(sbuf, cells, T, reinterpret_cast<int4*>(cells_out), s), "delaunay")) != RGS_OK)
		return rc;
	out->num_cells = T;
	return RGS_OK;
}

int32_t rgs_delaunay_predicates(int64_t N, const float* points, int64_t M, const int32_t* tuples, int8_t* signs, rgs_resize_fn resize,
                                void* scratch_user, void* cuda_stream) {
	if (N < 0 || N > INT32_MAX || M < 0 || M > INT32_MAX) return fail(RGS_E_INVALID, "delaunay predicates: count out of range");
	if (M == 0) return RGS_OK;
	if (!resize || !points || !tuples || !signs) return fail(RGS_E_INVALID, "null pointer");
	char* buf = nullptr;
	int bad = 0;
	int rc;
	if ((rc = grow(resize, scratch_user, sizeof(int), buf, "delaunay predicates scratch")) != RGS_OK ||
	    (rc = cuda_status(launch_dt_predicates((int)N, points, (int)M, tuples, signs, reinterpret_cast<int*>(buf), &bad, (cudaStream_t)cuda_stream),
	                      "delaunay predicates")) != RGS_OK)
		return rc;
	if (bad == 1) return fail(RGS_E_INVALID, "delaunay predicates: an index lies outside [0, N)");
	if (bad) return fail(RGS_E_INVALID, "delaunay predicates: a coordinate is not finite");
	return RGS_OK;
}

// the activation sizes every LPIPS stage accepts: [2, H, W, C] with 2 H W C < 2^31 elements
static int lpips_size(int32_t H, int32_t W, int64_t C, int32_t min_side, const char* what) {
	if (H < min_side || W < min_side)
		return fail(RGS_E_INVALID, std::string(what) + ": the image must be at least " + std::to_string(min_side) + " x " + std::to_string(min_side) +
		                               " pixels, got " + std::to_string(H) + " x " + std::to_string(W));
	if ((int64_t)H * W * C * 2 > INT32_MAX) return fail(RGS_E_INVALID, std::string(what) + ": the activations exceed 2^31 elements");
	return RGS_OK;
}

int32_t rgs_lpips_input_conv(int32_t H, int32_t W, const float* x, const float* y, const float* weight, const float* bias, float* out, void* cuda_stream) {
	if (const int rc = lpips_size(H, W, 64, 16, "lpips input conv")) return rc;
	if (!x || !y || !weight || !bias || !out) return fail(RGS_E_INVALID, "null pointer");
	return cuda_status(launch_lpips_input_conv(H, W, x, y, weight, bias, out, (cudaStream_t)cuda_stream), "lpips input conv");
}

int32_t rgs_lpips_conv3x3(int32_t H, int32_t W, int32_t C_in, int32_t C_out, const float* in, const float* weight, const float* bias, float* out,
                          void* cuda_stream) {
	if (C_in <= 0 || C_in % 32 || C_in > 512 || C_out <= 0 || C_out % 64 || C_out > 512)
		return fail(RGS_E_INVALID, "lpips conv3x3: C_in must be a multiple of 32 and C_out of 64, both at most 512");
	if (const int rc = lpips_size(H, W, std::max(C_in, C_out), 1, "lpips conv3x3")) return rc;
	if (!in || !weight || !bias || !out) return fail(RGS_E_INVALID, "null pointer");
	return cuda_status(launch_lpips_conv3x3(H, W, C_in, C_out, in, weight, bias, out, (cudaStream_t)cuda_stream), "lpips conv3x3");
}

int32_t rgs_lpips_maxpool(int32_t H, int32_t W, int32_t C, const float* in, float* out, void* cuda_stream) {
	if (C <= 0 || C % 4) return fail(RGS_E_INVALID, "lpips maxpool: C must be a positive multiple of 4");
	if (const int rc = lpips_size(H, W, C, 2, "lpips maxpool")) return rc;
	if (!in || !out) return fail(RGS_E_INVALID, "null pointer");
	return cuda_status(launch_lpips_maxpool(H, W, C, in, out, (cudaStream_t)cuda_stream), "lpips maxpool");
}

int32_t rgs_lpips_distance(int32_t H, int32_t W, int32_t C, const float* feats, const float* lin, float* map, double* mean, rgs_resize_fn resize,
                           void* scratch_user, void* cuda_stream) {
	if (C != 64 && C != 128 && C != 256 && C != 512) return fail(RGS_E_INVALID, "lpips distance: C must be 64, 128, 256 or 512");
	if (const int rc = lpips_size(H, W, C, 1, "lpips distance")) return rc;
	if (!feats || !lin || !map || !mean || !resize) return fail(RGS_E_INVALID, "null pointer");
	char* buf = nullptr;
	if (const int rc = grow(resize, scratch_user, sizeof(double) * lpips_distance_blocks(H * W), buf, "lpips distance scratch")) return rc;
	return cuda_status(launch_lpips_distance(H * W, C, feats, lin, map, reinterpret_cast<double*>(buf), mean, (cudaStream_t)cuda_stream),
	                   "lpips distance");
}

int32_t rgs_ssim_l1_forward_rows(int32_t planes, int32_t H, int32_t W, int32_t row_lo, int32_t row_hi, const float* img, const float* gt, float* dmaps,
                                 double* sums, void* cuda_stream) {
	if (planes < 0 || H <= 0 || W <= 0) return fail(RGS_E_INVALID, "image size must be positive");
	if (row_lo < 0 || row_hi > H || row_lo > row_hi) return fail(RGS_E_INVALID, "row range out of the image");
	if (!img || !gt || !sums) return fail(RGS_E_INVALID, "null pointer");
	if (planes > 65535) return fail(RGS_E_INVALID, "too many image planes");
	launch_ssim_l1_forward(planes, H, W, row_lo, row_hi, img, gt, dmaps, sums, (cudaStream_t)cuda_stream);
	return cuda_status(cudaGetLastError(), "ssim l1 forward");
}

int32_t rgs_ssim_l1_backward_rows(int32_t planes, int32_t H, int32_t W, int32_t row_lo, int32_t row_hi, const float* img, const float* gt,
                                  const float* dmaps, float w_ssim, float w_l1, const float* upstream, float* d_img, void* cuda_stream) {
	if (planes < 0 || H <= 0 || W <= 0) return fail(RGS_E_INVALID, "image size must be positive");
	if (row_lo < 0 || row_hi > H || row_lo > row_hi) return fail(RGS_E_INVALID, "row range out of the image");
	if (!img || !gt || !dmaps || !d_img) return fail(RGS_E_INVALID, "null pointer");
	if (planes > 65535) return fail(RGS_E_INVALID, "too many image planes");
	launch_ssim_l1_backward(planes, H, W, row_lo, row_hi, img, gt, dmaps, w_ssim, w_l1, upstream, d_img, (cudaStream_t)cuda_stream);
	return cuda_status(cudaGetLastError(), "ssim l1 backward");
}

int32_t rgs_ssim_l1_forward(int32_t planes, int32_t H, int32_t W, const float* img, const float* gt, float* dmaps, double* sums, void* cuda_stream) {
	return rgs_ssim_l1_forward_rows(planes, H, W, 0, H, img, gt, dmaps, sums, cuda_stream);
}

int32_t rgs_ssim_l1_backward(int32_t planes, int32_t H, int32_t W, const float* img, const float* gt, const float* dmaps, float w_ssim, float w_l1,
                             const float* upstream, float* d_img, void* cuda_stream) {
	return rgs_ssim_l1_backward_rows(planes, H, W, 0, H, img, gt, dmaps, w_ssim, w_l1, upstream, d_img, cuda_stream);
}

int32_t rgs_normal_consistency(int32_t H, int32_t W, int32_t from_depth, float inv_fx, float inv_fy, float cx, float cy, const float* rendered_normal,
                               const float* map_expected, const float* map_median, float w_expected, float w_median, double* loss_sum,
                               float* d_normal, float* d_expected, float* d_median, void* cuda_stream) {
	if (H <= 0 || W <= 0) return fail(RGS_E_INVALID, "image size must be positive");
	if (!rendered_normal || !map_expected || !map_median || !loss_sum || !d_normal || !d_expected || !d_median) return fail(RGS_E_INVALID, "null pointer");
	launch_normal_consistency(H, W, from_depth != 0, inv_fx, inv_fy, cx, cy, rendered_normal, map_expected, map_median, w_expected, w_median, loss_sum,
	                          d_normal, d_expected, d_median, (cudaStream_t)cuda_stream);
	return cuda_status(cudaGetLastError(), "normal consistency");
}

static int32_t appearance_size(int32_t H0, int32_t W0) {
	if (H0 < 32 || W0 < 32) return fail(RGS_E_INVALID, "appearance loss: the image must be at least 32 x 32");
	if ((int64_t)H0 * W0 > (int64_t)1 << 28) return fail(RGS_E_INVALID, "appearance loss: image too large");
	return RGS_OK;
}

int32_t rgs_appearance_downsample(int32_t H0, int32_t W0, const float* image, float* down, void* cuda_stream) {
	if (const int32_t rc = appearance_size(H0, W0)) return rc;
	if (!image || !down) return fail(RGS_E_INVALID, "null pointer");
	return cuda_status(launch_appearance_downsample(H0, W0, image, down, (cudaStream_t)cuda_stream), "appearance downsample");
}

int32_t rgs_appearance_downsample_backward(int32_t H0, int32_t W0, const float* d_down, float* d_image, void* cuda_stream) {
	if (const int32_t rc = appearance_size(H0, W0)) return rc;
	if (!d_down || !d_image) return fail(RGS_E_INVALID, "null pointer");
	return cuda_status(launch_appearance_downsample_backward(H0, W0, d_down, d_image, (cudaStream_t)cuda_stream), "appearance downsample backward");
}

int32_t rgs_appearance_l1_forward(int32_t H0, int32_t W0, const float* image, const float* gt, const float* up4, const float* w2, const float* b2,
                                  const float* w3, const float* b3, float* act, float* transformed, double* partials, float* loss, void* cuda_stream) {
	if (const int32_t rc = appearance_size(H0, W0)) return rc;
	if (!image || !gt || !up4 || !w2 || !b2 || !w3 || !b3 || !partials || !loss) return fail(RGS_E_INVALID, "null pointer");
	return cuda_status(launch_appearance_l1_forward(H0, W0, image, gt, up4, w2, b2, w3, b3, act, transformed, partials, loss, (cudaStream_t)cuda_stream),
	                   "appearance l1 forward");
}

int32_t rgs_appearance_l1_backward(int32_t H0, int32_t W0, const float* image, const float* gt, const float* up4, const float* act, const float* w2,
                                   const float* w3, const float* b3, const float* upstream, float* d_image, float* d_up4, float* d_w2, float* d_b2,
                                   float* d_w3, float* d_b3, double* partials, float* d_x, void* cuda_stream) {
	if (const int32_t rc = appearance_size(H0, W0)) return rc;
	if (!image || !gt || !up4 || !act || !w2 || !w3 || !b3 || !d_image || !d_up4 || !d_w2 || !d_b2 || !d_w3 || !d_b3 || !partials || !d_x)
		return fail(RGS_E_INVALID, "null pointer");
	return cuda_status(launch_appearance_l1_backward(H0, W0, image, gt, up4, act, w2, w3, b3, upstream, d_image, d_up4, d_w2, d_b2, d_w3, d_b3, partials,
	                                                 d_x, (cudaStream_t)cuda_stream),
	                   "appearance l1 backward");
}

int32_t rgs_densify_blocks(int32_t P) { return P > 0 ? densify_blocks(P) : 0; }

int32_t rgs_densify_select(int32_t P, const float* grad_accum, const float* grad_accum_abs, const float* denom, const float* scaling, const float* opacity,
                           const rgs_densify_thresholds* thresholds, uint8_t* flags, int32_t* block_offsets, float* ratio_q, int32_t* counts_host,
                           rgs_resize_fn scratch, void* scratch_user, void* cuda_stream) {
	if (P <= 0) return fail(RGS_E_INVALID, "densify: the model has no Gaussians");
	if (!grad_accum || !grad_accum_abs || !denom || !scaling || !opacity || !thresholds || !flags || !block_offsets || !ratio_q || !counts_host || !scratch)
		return fail(RGS_E_INVALID, "null pointer");
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	char* buf = nullptr;
	if (const int rc = grow(scratch, scratch_user, densify_select_scratch_bytes(P), buf, "densify scratch")) return rc;
	// the five totals follow the per-CTA offsets in the scratch's tail: one copy brings them to the host
	int32_t* totals = block_offsets + 5 * (size_t)densify_blocks(P);
	cudaError_t e = launch_densify_select(P, grad_accum, grad_accum_abs, denom, scaling, opacity, *thresholds, flags, block_offsets, ratio_q, totals, buf, s);
	if (e == cudaSuccess) e = cudaMemcpyAsync(counts_host, totals, 5 * sizeof(int32_t), cudaMemcpyDeviceToHost, s);
	if (e == cudaSuccess) e = cudaStreamSynchronize(s);
	return cuda_status(e, "densify select");
}

int32_t rgs_densify_plan(int32_t P, const uint8_t* flags, const int32_t* block_offsets, const int32_t* counts_host, const float* scaling, int32_t* src,
                         int32_t* draw, float* std_clone, float* std_split, void* cuda_stream) {
	if (P <= 0) return fail(RGS_E_INVALID, "densify: the model has no Gaussians");
	if (!flags || !block_offsets || !counts_host || !scaling) return fail(RGS_E_INVALID, "null pointer");
	const int32_t* c = counts_host;
	for (int k = 0; k < 5; k++)
		if (c[k] < 0 || c[k] > P) return fail(RGS_E_INVALID, "densify plan: counts out of range");
	if ((c[0] && !std_clone) || (c[1] && !std_split) || ((c[2] || c[3] || c[4]) && (!src || !draw))) return fail(RGS_E_INVALID, "null pointer");
	return cuda_status(launch_densify_plan(P, flags, block_offsets, counts_host, scaling, src, draw, std_clone, std_split, (cudaStream_t)cuda_stream),
	                   "densify plan");
}

int32_t rgs_densify_gather(int32_t N, const int32_t* src, const int32_t* draw, int32_t C, const float* xyz, const float* rotation, const float* scaling,
                           const float* sample_clone, const float* sample_split, float inv_split, float* xyz_out, float* scaling_out, int32_t n_cols,
                           const rgs_densify_column* cols, void* cuda_stream) {
	if (N < 0 || C < 0 || n_cols < 0 || n_cols > RGS_DENSIFY_MAX_COLUMNS) return fail(RGS_E_INVALID, "densify gather: bad sizes");
	if (N == 0) return RGS_OK;
	if (!src || !draw || !xyz || !rotation || !scaling || !xyz_out || !scaling_out || (n_cols && !cols)) return fail(RGS_E_INVALID, "null pointer");
	for (int k = 0; k < n_cols; k++)
		if (!cols[k].in || !cols[k].out || cols[k].width <= 0) return fail(RGS_E_INVALID, "densify gather: bad column");
	return cuda_status(launch_densify_gather(N, src, draw, C, xyz, rotation, scaling, sample_clone, sample_split, inv_split, xyz_out, scaling_out, n_cols,
	                                         cols, (cudaStream_t)cuda_stream),
	                   "densify gather");
}

int32_t rgs_reset_opacity(int32_t P, const float* scaling, const float* opacity, const float* filter_3D, float* out, void* cuda_stream) {
	if (P < 0) return fail(RGS_E_INVALID, "negative Gaussian count");
	if (P == 0) return RGS_OK;
	if (!scaling || !opacity || !filter_3D || !out) return fail(RGS_E_INVALID, "null pointer");
	return cuda_status(launch_reset_opacity(P, scaling, opacity, filter_3D, out, (cudaStream_t)cuda_stream), "reset opacity");
}

int32_t rgs_debug_get_views(const rgs_camera* cam, int32_t P, int64_t num_rendered, const char* geom_buffer, const char* binning_buffer,
                            const char* image_buffer, rgs_debug_views* views) {
	if (!cam || !views) return fail(RGS_E_INVALID, "null pointer");
	const bool coord = cam->require_coord != 0, depth = cam->require_depth != 0;
	const int grid_x = (cam->width + TILE_X - 1) / TILE_X, grid_y = (cam->height + TILE_Y - 1) / TILE_Y;
	const size_t N = (size_t)cam->width * slab_height(cam, cam->tile_row_begin, cam->tile_row_end < 0 ? grid_y : cam->tile_row_end);
	GeomView g = carve_geom(const_cast<char*>(geom_buffer), P, coord, nullptr);
	BinView b = carve_bin(const_cast<char*>(binning_buffer), (size_t)num_rendered, grid_x * grid_y, nullptr);
	ImgView img = carve_img(const_cast<char*>(image_buffer), grid_x, grid_y, N, coord, depth, nullptr);
	views->point_list = b.point_list;
	views->point_list_keys = b.keys_sorted;
	views->tile_ranges = reinterpret_cast<const uint32_t*>(img.ranges);
	views->n_contrib = img.n_contrib;
	views->tiles_touched = g.tiles_touched;
	views->records = g.records;
	views->record_floats = rec_floats(coord);
	views->depths = g.depths;
	return RGS_OK;
}

}  // extern "C"

// rgs_api.cu -- the rasterizer's C-ABI entry points (include/rgs_b200.h): buffer carving and orchestration across the
// rasterizer's kernel files, plus the error buffer, launch counter and stage timing that every entry point shares.  The
// other subsystems' entry points sit beside their kernels.
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

static bool capturing(cudaStream_t s) {
	cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
	return cudaStreamIsCapturing(s, &st) == cudaSuccess && st != cudaStreamCaptureStatusNone;
}

// Records nothing while the stream is being captured into a CUDA graph: the events would be graph nodes, read back never.
struct StageScope {
	cudaStream_t s; int stage; cudaEvent_t a = nullptr, b = nullptr; bool on;
	StageScope(int st, cudaStream_t stream) : s(stream), stage(st), on(g_stage_on.load() != 0 && !capturing(stream)) {
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

int fail(int code, const std::string& msg) {
	t_error = msg;
	return code;
}

int cuda_status(cudaError_t e, const char* what, const char* invalid) {
	if (e == cudaSuccess) return RGS_OK;
	if (invalid && e == cudaErrorInvalidValue) return fail(RGS_E_INVALID, std::string(what) + ": " + invalid);
	return fail(RGS_E_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

const char* const kNonFinitePoint = "a point has a NaN or infinite coordinate";

int grow(rgs_resize_fn fn, void* user, size_t bytes, char*& buf, const char* what) {
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

// The whole image's tile counts of a balanced forward before its slab is chosen: the scan's per-tile arrays, its difference grid
// and the per-row statistics (3 words per tile row, rgs_balance.cu's row_stats_kernel).
static ImgView carve_counts(char* base, int grid_x, int grid_y, uint32_t*& stats, size_t* total) {
	const int tiles = grid_x * grid_y;
	Carver c(base);
	ImgView v{};
	v.ranges = c.take<uint2>(tiles);
	v.tile_count = c.take<uint32_t>(tiles);
	v.totals = c.take<uint32_t>(2);
	v.chunk_base = c.take<uint32_t>(tiles);
	v.tile_diff = c.take<int>((size_t)(grid_x + 1) * (grid_y + 1));
	stats = c.take<uint32_t>((size_t)3 * grid_y);
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

// pinned per-thread mailbox of the balanced forward's per-row read-back, grown on demand
static uint32_t* pinned_row_stats(size_t words) {
	static thread_local uint32_t* box = nullptr;
	static thread_local size_t capacity = 0;
	if (words > capacity) {
		if (box) cudaFreeHost(box);
		capacity = 0;
		if (cudaHostAlloc((void**)&box, words * sizeof(uint32_t), cudaHostAllocDefault) != cudaSuccess) return box = nullptr;
		capacity = words;
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

static int carve_geom_buffer(const FwdParams& p, const rgs_buffers* bufs, GeomView& g) {
	size_t geom_bytes = 0;
	carve_geom(nullptr, p.P, p.coord, &geom_bytes);
	char* geom_ptr;
	const int rc = grow(bufs->geom, bufs->geom_user, geom_bytes, geom_ptr, "geometry buffer");
	if (rc == RGS_OK) g = carve_geom(geom_ptr, p.P, p.coord, nullptr);
	return rc;
}

// image-side scratch, carved for p's maps ([C, Hs, W])
static int carve_img_buffer(const FwdParams& p, const rgs_buffers* bufs, ImgView& img) {
	const size_t N = (size_t)p.W * p.Hs;
	size_t img_bytes = 0;
	carve_img(nullptr, p.grid_x, p.grid_y, N, p.coord, p.depth, &img_bytes);
	char* img_ptr;
	const int rc = grow(bufs->image, bufs->image_user, img_bytes, img_ptr, "image buffer");
	if (rc == RGS_OK) img = carve_img(img_ptr, p.grid_x, p.grid_y, N, p.coord, p.depth, nullptr);
	return rc;
}

// preprocess -> per-tile counts, ranges and totals of p's tile rows (P > 0)
static int preprocess_and_scan(const rgs_camera* cam, const FwdParams& p, int* radii, GeomView g, ImgView img, cudaStream_t s) {
	int rc;
	RGS_CUDA_TRY(cudaMemsetAsync(img.tile_diff, 0, (size_t)(p.grid_x + 1) * (p.grid_y + 1) * sizeof(int), s));
	{ StageScope sc(ST_PREPROCESS, s); launch_preprocess_forward(p, g, radii, img.tile_diff, s); }
	if ((rc = debug_sync(cam, s, "preprocess")) != RGS_OK) return rc;
	{ StageScope sc(ST_SCAN, s); launch_tile_scan(p, img, s); }
	return RGS_OK;
}

// binning buffer for R instances -> scatter and per-tile sort of p's tile rows (with preset_status: R and max_list are capacities)
static int64_t bin_tiles(const rgs_camera* cam, const FwdParams& p, int* radii, const rgs_buffers* bufs, cudaStream_t s, GeomView g, BinView& b,
                         ImgView img, int64_t R, uint32_t max_list, uint32_t* preset_status = nullptr) {
	int rc;
	const int P = p.P;
	const int tiles = p.grid_x * p.grid_y;
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
		launch_tile_binning(p, g, b, img, radii, R, max_list, s, preset_status);
	}
	if ((rc = debug_sync(cam, s, "binning")) != RGS_OK) return rc;
	return R;
}

// preprocess -> tile counts -> (one host sync for the instance count) -> binning / sort: everything before blending.
// Shared by rgs_forward and rgs_integrate.  Returns num_rendered or a negative status.
static int64_t forward_to_binning(const rgs_camera* cam, const FwdParams& p, int* radii, const rgs_buffers* bufs, cudaStream_t s, GeomView& g,
                                  BinView& b, ImgView& img) {
	int rc;
	// image-side scratch first: needed even when there is nothing to draw (background fill)
	if ((rc = carve_img_buffer(p, bufs, img)) != RGS_OK || (rc = carve_geom_buffer(p, bufs, g)) != RGS_OK) return rc;

	int64_t R = 0;
	uint32_t max_list = 0;
	if (p.P > 0) {
		if ((rc = preprocess_and_scan(cam, p, radii, g, img, s)) != RGS_OK) return rc;
		// the one host sync of the forward pass: the instance count sizes the binning buffers and is returned to the
		// caller (reference: blocking cudaMemcpy, rasterizer_impl.cu:354); the longest tile list picks the sort path
		uint32_t* box = pinned_mailbox();
		if (!box) return fail(RGS_E_CUDA, "cudaHostAlloc failed for the num_rendered mailbox");
		RGS_CUDA_TRY(cudaMemcpyAsync(box, img.totals, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
		RGS_CUDA_TRY(cudaStreamSynchronize(s));
		R = (int64_t)box[0];
		max_list = box[1];
	}
	return bin_tiles(cam, p, radii, bufs, s, g, b, img, R, max_list);
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

// The sort kernels' shared-memory opt-in, once per device: rgs_forward_preset does it outside stream capture and refuses a capture on
// a device that has not had it.
static bool g_graph_ready[64];

int64_t rgs_forward_preset(const rgs_camera* cam, const rgs_gaussians* gs, const rgs_forward_out* out, const rgs_buffers* bufs, const rgs_preset* preset,
                           void* cuda_stream) {
	FwdParams p;
	int rc = make_params(cam, gs, p);
	if (rc != RGS_OK) return rc;
	if (!out || !bufs || !bufs->geom || !bufs->binning || !bufs->image) return fail(RGS_E_INVALID, "null outputs / buffer callbacks");
	if (!preset || !preset->status) return fail(RGS_E_INVALID, "rgs_forward_preset: null preset / status");
	if (preset->instances < 0 || preset->longest_list < 0) return fail(RGS_E_INVALID, "rgs_forward_preset: negative capacity");
	if (cam->debug) return fail(RGS_E_UNSUPPORTED, "rgs_forward_preset: debug mode synchronizes after every stage; use rgs_forward");
	if (cam->tile_row_begin != 0 || cam->tile_row_end != -1 || cam->compact_slab)
		return fail(RGS_E_UNSUPPORTED, "rgs_forward_preset renders the whole image only: no tile-row slab, no compact_slab");
	cudaStream_t s = (cudaStream_t)cuda_stream;
	int dev = 0;
	RGS_CUDA_TRY(cudaGetDevice(&dev));
	if (!capturing(s)) {
		prepare_tile_binning();
		g_graph_ready[dev & 63] = true;
	} else if (!g_graph_ready[dev & 63]) {
		return fail(RGS_E_INVALID, "rgs_forward_preset: make one call outside stream capture on this device first (one-time set-up)");
	}
	GeomView g;
	BinView b;
	ImgView img;
	if ((rc = carve_img_buffer(p, bufs, img)) != RGS_OK || (rc = carve_geom_buffer(p, bufs, g)) != RGS_OK) return rc;
	if (p.P > 0 && (rc = preprocess_and_scan(cam, p, out->radii, g, img, s)) != RGS_OK) return rc;
	const int64_t R = bin_tiles(cam, p, out->radii, bufs, s, g, b, img, preset->instances, (uint32_t)preset->longest_list, p.P > 0 ? preset->status : nullptr);
	if (R < 0) return R;
	RenderOut ro{out->out_color, out->out_coord, out->out_mcoord, out->out_alpha, out->out_normal, out->out_depth, out->out_mdepth};
	{ StageScope sc(ST_RENDER_FWD, s); launch_render_forward(p, g, b, img, ro, s); }
	if ((rc = debug_sync(cam, s, "render")) != RGS_OK) return rc;
	return R;
}

int64_t rgs_forward_balanced(const rgs_camera* cam, const rgs_gaussians* gs, int32_t world_size, int32_t rank, rgs_forward_out* out, rgs_maps_fn maps,
                             void* maps_user, const rgs_buffers* bufs, int32_t* row_cuts, uint32_t* row_stats, void* cuda_stream) {
	if (!cam) return fail(RGS_E_INVALID, "null camera / gaussians");
	rgs_camera whole = *cam;
	whole.tile_row_begin = 0;
	whole.tile_row_end = -1;
	FwdParams p;
	int rc = make_params(&whole, gs, p);
	if (rc != RGS_OK) return rc;
	if (!out || !maps || !row_cuts || !bufs || !bufs->geom || !bufs->binning || !bufs->image)
		return fail(RGS_E_INVALID, "null outputs / callbacks / row_cuts");
	if (world_size <= 0 || rank < 0 || rank >= world_size) return fail(RGS_E_INVALID, "balanced forward: rank / world_size out of range");
	cudaStream_t s = (cudaStream_t)cuda_stream;
	const int gy = p.grid_y;
	GeomView g;
	if ((rc = carve_geom_buffer(p, bufs, g)) != RGS_OK) return rc;
	// the whole image's tile counts live in the binning buffer until the slab is known: the image buffer is then carved for the
	// slab's maps only, as a fixed-slab call carves it, and the binning buffer is grown for the slab's instances after the
	// restriction has read them
	size_t count_bytes = 0;
	uint32_t* d_stats = nullptr;
	carve_counts(nullptr, p.grid_x, gy, d_stats, &count_bytes);
	char* count_ptr;
	if ((rc = grow(bufs->binning, bufs->binning_user, count_bytes, count_ptr, "binning buffer")) != RGS_OK) return rc;
	const ImgView counts = carve_counts(count_ptr, p.grid_x, gy, d_stats, nullptr);
	std::vector<uint32_t> stats((size_t)3 * gy, 0u);  // I_y, L_y, 32-instance chunks per row
	if (p.P > 0) {
		if ((rc = preprocess_and_scan(&whole, p, out->radii, g, counts, s)) != RGS_OK) return rc;
		{ StageScope sc(ST_SCAN, s); launch_row_stats(p, counts, d_stats, s); }
		// the one host sync of the balanced forward: the per-row counts choose the slab, size its binning buffers and give num_rendered
		uint32_t* box = pinned_row_stats(stats.size());
		if (!box) return fail(RGS_E_CUDA, "cudaHostAlloc failed for the row-stats mailbox");
		RGS_CUDA_TRY(cudaMemcpyAsync(box, d_stats, stats.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
		RGS_CUDA_TRY(cudaStreamSynchronize(s));
		std::memcpy(stats.data(), box, stats.size() * sizeof(uint32_t));
	}
	if ((rc = rgs_balance_partition(gy, p.grid_x, world_size, stats.data(), row_cuts)) != RGS_OK) return rc;
	if (row_stats) std::memcpy(row_stats, stats.data(), (size_t)2 * gy * sizeof(uint32_t));

	rgs_camera slab = *cam;
	slab.tile_row_begin = row_cuts[rank];
	slab.tile_row_end = row_cuts[rank + 1];
	FwdParams ps;
	if ((rc = make_params(&slab, gs, ps)) != RGS_OK) return rc;
	SlabShift sh{0u, 0u, 0u, 0u, 0u};
	for (int y = 0; y < gy; y++) {
		if (y < ps.row_begin) {
			sh.range_off += stats[y];
			sh.chunk_off += stats[2 * gy + y];
		} else if (y < ps.row_end) {
			sh.rendered += stats[y];
			sh.longest = stats[gy + y] > sh.longest ? stats[gy + y] : sh.longest;
			sh.chunk_total += stats[2 * gy + y];
		}
	}
	ImgView img;
	if ((rc = carve_img_buffer(ps, bufs, img)) != RGS_OK) return rc;
	if (p.P > 0) {
		StageScope sc(ST_SCAN, s);
		launch_slab_restrict(ps, g, counts, img, out->radii, sh, s);
	}
	if (maps(maps_user, ps.row_begin, ps.row_end, ps.Hs, out) != 0) return fail(RGS_E_ALLOC, "maps callback failed");
	BinView b;
	const int64_t R = bin_tiles(&slab, ps, out->radii, bufs, s, g, b, img, (int64_t)sh.rendered, sh.longest);
	if (R < 0) return R;
	RenderOut ro{out->out_color, out->out_coord, out->out_mcoord, out->out_alpha, out->out_normal, out->out_depth, out->out_mdepth};
	{ StageScope sc(ST_RENDER_FWD, s); launch_render_forward(ps, g, b, img, ro, s); }
	if ((rc = debug_sync(&slab, s, "render")) != RGS_OK) return rc;
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

// Stage 1 into the accumulator rows `acc` (`missing`: the error when there are none), zero-filled first with `zero_first`.  Leaves
// p and g for the caller's next step.
static int backward_render(const rgs_camera* cam, const rgs_gaussians* gs, const rgs_backward_in* in, float* acc, const char* missing,
                           bool zero_first, cudaStream_t s, FwdParams& p, GeomView& g) {
	BinView b;
	ImgView img;
	int rc = backward_views(cam, gs, in, p, g, b, img);
	if (rc != RGS_OK || p.P == 0) return rc;
	if (!acc) return fail(RGS_E_INVALID, missing);
	RenderGradIn gin{in->dL_dout_color, in->dL_dout_coord, in->dL_dout_mcoord, in->dL_dout_depth, in->dL_dout_mdepth,
	                 in->dL_dout_alpha, in->dL_dout_normal, in->out_alpha, in->out_normal};
	{ StageScope sc(ST_RENDER_BWD, s); launch_render_backward(p, g, b, img, gin, acc, s, zero_first); }
	return debug_sync(cam, s, "backward render");
}

int32_t rgs_backward_render(const rgs_camera* cam, const rgs_gaussians* gs, const rgs_backward_in* in, float* grad_accum, void* cuda_stream) {
	FwdParams p;
	GeomView g;
	return backward_render(cam, gs, in, grad_accum, "null gradient accumulator", true, (cudaStream_t)cuda_stream, p, g);
}

int32_t rgs_backward_render_exchange(const rgs_camera* cam, const rgs_gaussians* gs, const rgs_backward_in* in, rgs_exchange* ex, void* cuda_stream) {
	FwdParams p;
	GeomView g;
	cudaStream_t s = (cudaStream_t)cuda_stream;
	int rc = backward_render(cam, gs, in, rgs_exchange_accumulator(ex), "null exchange", false, s, p, g);
	if (rc != RGS_OK || p.P == 0) return rc;
	{
		StageScope sc(ST_EXCHANGE, s);
		rc = rgs_exchange_rows(ex, p.P, g.tiles_touched, in->radii, cuda_stream);
	}
	if (rc != RGS_OK) return rc;
	return debug_sync(cam, s, "gradient exchange");
}

static ParamGradOut param_grads(const rgs_backward_out* o) {
	return {o->dL_dmeans2D, o->dL_dcolors, o->dL_dopacity, o->dL_dmeans3D, o->dL_dcov3D, o->dL_dsh, o->dL_dscales, o->dL_drotations, o->dL_dsh_rest};
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
	const ParamGradOut po = param_grads(out);
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
// for work ordered after `s`.  Not created while `s` is being captured (none: the caller runs the work on `s`).
static SideStream* side_stream(cudaStream_t s) {
	static thread_local SideStream per_dev[64];
	int dev = 0;
	if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
	SideStream& ss = per_dev[dev & 63];
	if (!ss.stream) {
		if (capturing(s)) return nullptr;
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
	SideStream* ss = !cam->debug ? side_stream(s) : nullptr;
	if (ss) {
		FwdParams p;
		int rc0 = make_params(cam, gs, p);
		if (rc0 != RGS_OK) return rc0;
		const ParamGradOut po = param_grads(out);
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

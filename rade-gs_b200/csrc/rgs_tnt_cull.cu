// rgs_tnt_cull.cu -- the Tanks and Temples mesh cull (reference eval_tnt/cull_mesh.py) on the GPU: a depth-only triangle
// rasterizer (pyrender's DEPTH_ONLY | SKIP_CULL_FACES pass) and the multi-view visibility count of Mesher.point_masks.
//
// The contract (include/rgs_b200.h, rgs_tnt_mesh_depth / rgs_tnt_visibility_count) fixes every stored bit: each arithmetic
// step is one intrinsic rounded on its own (__fadd_rn / __fmul_rn / __fdiv_rn), so nvcc contracts nothing and the numpy
// model tests/tnt_cull_model.py reproduces the depth maps and the counts.
//   depth    homogeneous rasterization in camera space: a pixel centre's ray d = ((px - cx) / fx, (py - cy) / fy, 1) is inside
//            a triangle when its three edge functions (P + Q) x (Q - P) . d carry the triangle's orientation; the surface depth
//            is the ray's hit on the triangle's plane.  A shared edge gives the two triangles edge functions of exactly
//            opposite value, and a fixed tie rule hands a pixel centre on the edge to exactly one of them.  No projection
//            through the camera is needed, so triangles that cross the near plane or reach far off screen need no clip.
//            The nearest fragment wins by atomicMin on the bits of the positive depth.
//   split    the triangle kernel (one thread per face) transforms, rejects and bounds each face; a bounding box of at most
//            SMALL_AREA pixels is rasterized there, larger ones are queued: boxes up to MEDIUM_AREA pixels get one CTA each,
//            larger ones are spread over the whole grid.  A face that crosses the near plane is bounded by its clipped polygon.
//   count    one thread per point: the reference's projection, frustum test, grid_sample(bilinear, border, align_corners)
//            and the occlusion test, each operation rounded on its own in the order written.
//
// This file also holds the C-ABI entry points rgs_tnt_mesh_depth and rgs_tnt_visibility_count.
#include "rgs_common.cuh"

namespace rgs {

namespace {

constexpr int SMALL_AREA = 16;      // pixels a single thread tests
constexpr int MEDIUM_AREA = 4096;   // pixels one CTA walks; above this every CTA of the grid takes a stripe
constexpr unsigned EMPTY_BITS = 0xffffffffu;   // depth buffer sentinel while drawing: above every positive float's bits

struct View {
	float m[12];   // w2c rows 0..2, row-major
	float fx, fy, cx, cy, znear, zfar;
	int H, W;
};

__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }

// ((m0 x + m1 y) + m2 z) + m3 per row
__device__ __forceinline__ float3 to_camera(const View& v, float x, float y, float z) {
	float o[3];
#pragma unroll
	for (int r = 0; r < 3; r++) o[r] = fadd(fadd(fadd(fmul(v.m[4 * r], x), fmul(v.m[4 * r + 1], y)), fmul(v.m[4 * r + 2], z)), v.m[4 * r + 3]);
	return make_float3(o[0], o[1], o[2]);
}

__device__ __forceinline__ float3 sub3(float3 a, float3 b) { return make_float3(fsub(a.x, b.x), fsub(a.y, b.y), fsub(a.z, b.z)); }
__device__ __forceinline__ float3 add3(float3 a, float3 b) { return make_float3(fadd(a.x, b.x), fadd(a.y, b.y), fadd(a.z, b.z)); }
__device__ __forceinline__ float3 cross3(float3 a, float3 b) {
	return make_float3(fsub(fmul(a.y, b.z), fmul(a.z, b.y)), fsub(fmul(a.z, b.x), fmul(a.x, b.z)), fsub(fmul(a.x, b.y), fmul(a.y, b.x)));
}
__device__ __forceinline__ float3 neg3(float3 a) { return make_float3(-a.x, -a.y, -a.z); }

// the tie rule: a pixel centre with edge function exactly 0 belongs to the triangle whose (oriented) edge vector is
// lexicographically positive; the neighbour across the edge holds its negation
__device__ __forceinline__ bool tie_owner(float3 c) { return c.x > 0.f || (c.x == 0.f && (c.y > 0.f || (c.y == 0.f && c.z > 0.f))); }

struct Tri {
	float3 c[3];   // oriented edge vectors
	float3 n;      // plane normal (B - A) x (C - A)
	float num;     // n . A
	int x0, y0, x1, y1;   // pixel bounding box, inclusive
};

// Transforms face f and decides whether it can draw.  false: nothing to draw (non-finite vertex, every vertex in front
// of znear or beyond zfar, zero orientation, empty box).  bad: an index outside [0, V).
__device__ bool setup_tri(const View& v, int64_t V, const float* __restrict__ verts, const int32_t* __restrict__ faces, int64_t f, Tri& t, bool& bad) {
	float3 P[3];
#pragma unroll
	for (int k = 0; k < 3; k++) {
		const int32_t i = faces[3 * f + k];
		if (i < 0 || i >= V) {
			bad = true;
			return false;
		}
		P[k] = to_camera(v, verts[3 * (int64_t)i], verts[3 * (int64_t)i + 1], verts[3 * (int64_t)i + 2]);
	}
	bool finite = true, all_near = true, all_far = true, crosses = false;
#pragma unroll
	for (int k = 0; k < 3; k++) {
		finite = finite && isfinite(P[k].x) && isfinite(P[k].y) && isfinite(P[k].z);
		all_near = all_near && P[k].z < v.znear;
		all_far = all_far && P[k].z > v.zfar;
		crosses = crosses || P[k].z < v.znear;
	}
	if (!finite || all_near || all_far) return false;
	// the box of the face clipped at Z = znear: the vertices in front of it and the crossing points of the edges that
	// cross it (a face that crosses is still drawn by its edge functions, not by these points)
	float umin = INFINITY, umax = -INFINITY, vmin = INFINITY, vmax = -INFINITY;
	auto extend = [&](float X, float Y, float Z) {
		const float u = fadd(__fdiv_rn(fmul(v.fx, X), Z), v.cx), w = fadd(__fdiv_rn(fmul(v.fy, Y), Z), v.cy);
		umin = fminf(umin, u), umax = fmaxf(umax, u), vmin = fminf(vmin, w), vmax = fmaxf(vmax, w);
	};
#pragma unroll
	for (int k = 0; k < 3; k++) {
		const float3 a = P[k], b = P[k == 2 ? 0 : k + 1];
		if (!(a.z < v.znear)) extend(a.x, a.y, a.z);
		if (crosses && ((a.z < v.znear) != (b.z < v.znear))) {
			const float s = __fdiv_rn(fsub(v.znear, a.z), fsub(b.z, a.z));
			extend(fadd(a.x, fmul(s, fsub(b.x, a.x))), fadd(a.y, fmul(s, fsub(b.y, a.y))), fadd(a.z, fmul(s, fsub(b.z, a.z))));
		}
	}
	const float Wf = (float)v.W, Hf = (float)v.H;
	umin = fminf(fmaxf(umin, -1.f), Wf), umax = fminf(fmaxf(umax, -1.f), Wf);
	vmin = fminf(fmaxf(vmin, -1.f), Hf), vmax = fminf(fmaxf(vmax, -1.f), Hf);
	t.x0 = max((int)floorf(fsub(umin, 0.5f)), 0), t.x1 = min((int)ceilf(fsub(umax, 0.5f)), v.W - 1);
	t.y0 = max((int)floorf(fsub(vmin, 0.5f)), 0), t.y1 = min((int)ceilf(fsub(vmax, 0.5f)), v.H - 1);
	if (t.x0 > t.x1 || t.y0 > t.y1) return false;
	t.n = cross3(sub3(P[1], P[0]), sub3(P[2], P[0]));
	t.num = fadd(fadd(fmul(t.n.x, P[0].x), fmul(t.n.y, P[0].y)), fmul(t.n.z, P[0].z));
	if (!(t.num != 0.f)) return false;
	const bool flip = t.num < 0.f;
#pragma unroll
	for (int k = 0; k < 3; k++) {
		const float3 a = P[k], b = P[k == 2 ? 0 : k + 1];
		const float3 c = cross3(add3(a, b), sub3(b, a));
		t.c[k] = flip ? neg3(c) : c;
	}
	return true;
}

__device__ __forceinline__ float edge(float3 c, float dx, float dy) { return fadd(fadd(fmul(c.x, dx), fmul(c.y, dy)), c.z); }

__device__ __forceinline__ void shade(const View& v, const Tri& t, int x, int y, unsigned* __restrict__ depth) {
	const float dx = __fdiv_rn(fsub(fadd((float)x, 0.5f), v.cx), v.fx), dy = __fdiv_rn(fsub(fadd((float)y, 0.5f), v.cy), v.fy);
#pragma unroll
	for (int k = 0; k < 3; k++) {
		const float e = edge(t.c[k], dx, dy);
		if (!(e > 0.f || (e == 0.f && tie_owner(t.c[k])))) return;
	}
	const float z = __fdiv_rn(t.num, edge(t.n, dx, dy));
	if (z >= v.znear && z <= v.zfar) atomicMin(depth + (int64_t)y * v.W + x, __float_as_uint(z));
}

// counters: [0] medium queue length, [1] large queue length, [2] bad index flag
__global__ void __launch_bounds__(256) tnt_raster_kernel(View v, int64_t V, const float* __restrict__ verts, int64_t F, const int32_t* __restrict__ faces,
                                                         unsigned* __restrict__ depth, int32_t* __restrict__ medium, int32_t* __restrict__ large,
                                                         int32_t* __restrict__ counters) {
	const int64_t f = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
	if (f >= F) return;
	Tri t;
	bool bad = false;
	if (!setup_tri(v, V, verts, faces, f, t, bad)) {
		if (bad) counters[2] = 1;
		return;
	}
	const int bw = t.x1 - t.x0 + 1, area = bw * (t.y1 - t.y0 + 1);
	if (area <= SMALL_AREA) {
		for (int p = 0; p < area; p++) shade(v, t, t.x0 + p % bw, t.y0 + p / bw, depth);
	} else if (area <= MEDIUM_AREA) {
		medium[atomicAdd(counters, 1)] = (int32_t)f;
	} else {
		large[atomicAdd(counters + 1, 1)] = (int32_t)f;
	}
}

// one CTA per queued face
__global__ void __launch_bounds__(256) tnt_raster_medium_kernel(View v, int64_t V, const float* __restrict__ verts, const int32_t* __restrict__ faces,
                                                                unsigned* __restrict__ depth, const int32_t* __restrict__ medium, const int32_t* __restrict__ counters) {
	const int n = counters[0];
	for (int q = blockIdx.x; q < n; q += gridDim.x) {
		Tri t;
		bool bad = false;
		setup_tri(v, V, verts, faces, medium[q], t, bad);   // true for every queued face
		const int bw = t.x1 - t.x0 + 1, area = bw * (t.y1 - t.y0 + 1);
		for (int p = threadIdx.x; p < area; p += blockDim.x) shade(v, t, t.x0 + p % bw, t.y0 + p / bw, depth);
	}
}

// every CTA takes a stripe of every queued face
__global__ void __launch_bounds__(256) tnt_raster_large_kernel(View v, int64_t V, const float* __restrict__ verts, const int32_t* __restrict__ faces,
                                                               unsigned* __restrict__ depth, const int32_t* __restrict__ large, const int32_t* __restrict__ counters) {
	const int n = counters[1];
	const int64_t stride = (int64_t)gridDim.x * blockDim.x;
	for (int q = 0; q < n; q++) {
		Tri t;
		bool bad = false;
		setup_tri(v, V, verts, faces, large[q], t, bad);
		const int bw = t.x1 - t.x0 + 1;
		const int64_t area = (int64_t)bw * (t.y1 - t.y0 + 1);
		for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < area; p += stride) shade(v, t, t.x0 + (int)(p % bw), t.y0 + (int)(p / bw), depth);
	}
}

// sentinel -> 0 (nothing drawn)
__global__ void __launch_bounds__(256) tnt_depth_finish_kernel(int64_t n, unsigned* __restrict__ depth) {
	const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
	if (i < n && depth[i] == EMPTY_BITS) depth[i] = 0u;
}

// ---- visibility count (cull_mesh.py:126-175) ---------------------------------------------------------------------------

struct CountParams {
	float m[12];
	float fx, fy, cx, cy, eps, inv_w1, inv_h1;   // inv_* = 1.0f / (float)(W - 1), 1.0f / (float)(H - 1)
	int H, W;
};

__global__ void __launch_bounds__(256) tnt_visibility_kernel(int64_t N, const float* __restrict__ points, const float* __restrict__ depth, CountParams c,
                                                             int32_t* __restrict__ counts) {
	const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
	if (i >= N) return;
	const float x = points[3 * i], y = points[3 * i + 1], zz = points[3 * i + 2];
	float cam[3];
#pragma unroll
	for (int r = 0; r < 3; r++) cam[r] = fadd(fadd(fadd(fmul(c.m[4 * r], x), fmul(c.m[4 * r + 1], y)), fmul(c.m[4 * r + 2], zz)), c.m[4 * r + 3]);
	const float z = fadd(cam[2], 1e-8f);
	const float u = __fdiv_rn(fadd(fmul(c.fx, cam[0]), fmul(c.cx, cam[2])), z);
	const float w = __fdiv_rn(fadd(fmul(c.fy, cam[1]), fmul(c.cy, cam[2])), z);
	const float Wm1 = (float)(c.W - 1), Hm1 = (float)(c.H - 1);
	if (!(u >= 0.f && u <= Wm1 && w >= 0.f && w <= Hm1 && z > 0.f)) return;
	// grid = u / (W - 1) * 2 - 1 (torch on CUDA: times the fp32 reciprocal), then grid_sample's ((g + 1) / 2) * (W - 1)
	const float gx = fsub(fmul(fmul(u, c.inv_w1), 2.f), 1.f), gy = fsub(fmul(fmul(w, c.inv_h1), 2.f), 1.f);
	const float ix = fminf(Wm1, fmaxf(fmul(__fdiv_rn(fadd(gx, 1.f), 2.f), Wm1), 0.f));
	const float iy = fminf(Hm1, fmaxf(fmul(__fdiv_rn(fadd(gy, 1.f), 2.f), Hm1), 0.f));
	const float fx0 = floorf(ix), fy0 = floorf(iy), fx1 = fadd(fx0, 1.f), fy1 = fadd(fy0, 1.f);
	const int x0 = (int)fx0, y0 = (int)fy0;
	const float wnw = fmul(fsub(fx1, ix), fsub(fy1, iy)), wne = fmul(fsub(ix, fx0), fsub(fy1, iy));
	const float wsw = fmul(fsub(fx1, ix), fsub(iy, fy0)), wse = fmul(fsub(ix, fx0), fsub(iy, fy0));
	const bool xr = x0 + 1 < c.W, yb = y0 + 1 < c.H;
	const float* row = depth + (int64_t)y0 * c.W;
	float s = 0.f;
	s = fadd(s, fmul(row[x0], wnw));
	if (xr) s = fadd(s, fmul(row[x0 + 1], wne));
	if (yb) s = fadd(s, fmul(row[c.W + x0], wsw));
	if (xr && yb) s = fadd(s, fmul(row[c.W + x0 + 1], wse));
	if (s > 0.f && !(z < fadd(s, c.eps))) return;
	counts[i] += 1;
}

template <typename T>
void fill_matrix(T& p, const float* w2c) {
	for (int k = 0; k < 12; k++) p.m[k] = w2c[k];
}

}  // namespace
}  // namespace rgs

using namespace rgs;

extern "C" {

int32_t rgs_tnt_mesh_depth(int64_t V, const float* vertices, int64_t F, const int32_t* faces, const float* w2c, float fx, float fy, float cx, float cy,
                           int32_t H, int32_t W, float znear, float zfar, float* depth, rgs_resize_fn scratch, void* scratch_user, void* cuda_stream) {
	if (V < 0 || V > INT32_MAX || F < 0 || F > INT32_MAX) return fail(RGS_E_INVALID, "tnt mesh depth: vertex or face count out of range");
	if (H <= 0 || W <= 0 || H > 32768 || W > 32768) return fail(RGS_E_INVALID, "tnt mesh depth: H and W must lie in [1, 32768]");
	if (!(znear > 0.f) || !(zfar > znear)) return fail(RGS_E_INVALID, "tnt mesh depth: need 0 < znear < zfar");
	if (!(fx != 0.f) || !(fy != 0.f) || !isfinite(fx) || !isfinite(fy) || !isfinite(cx) || !isfinite(cy))
		return fail(RGS_E_INVALID, "tnt mesh depth: intrinsics must be finite with nonzero fx and fy");
	if (!w2c || !depth || !scratch || (V > 0 && !vertices) || (F > 0 && !faces)) return fail(RGS_E_INVALID, "null pointer");
	if (V == 0 && F > 0) return fail(RGS_E_INVALID, "tnt mesh depth: a face index lies outside [0, V)");
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	const int64_t n = (int64_t)H * W;
	View v;
	fill_matrix(v, w2c);
	v.fx = fx, v.fy = fy, v.cx = cx, v.cy = cy, v.znear = znear, v.zfar = zfar, v.H = H, v.W = W;
	Carver c(nullptr);
	c.take<int32_t>(4);
	c.take<int32_t>((size_t)F);
	c.take<int32_t>((size_t)F);
	char* buf = nullptr;
	int rc;
	if ((rc = grow(scratch, scratch_user, c.size(), buf, "tnt mesh depth scratch")) != RGS_OK) return rc;
	Carver k(buf);
	int32_t* counters = k.take<int32_t>(4);
	int32_t* medium = k.take<int32_t>((size_t)F);
	int32_t* large = k.take<int32_t>((size_t)F);
	unsigned* d = reinterpret_cast<unsigned*>(depth);
	RGS_CUDA_TRY(cudaMemsetAsync(counters, 0, 4 * sizeof(int32_t), s));
	RGS_CUDA_TRY(cudaMemsetAsync(d, 0xff, (size_t)n * sizeof(float), s));
	if (F > 0) {
		tnt_raster_kernel<<<(unsigned)((F + 255) / 256), 256, 0, s>>>(v, V, vertices, F, faces, d, medium, large, counters);
		tnt_raster_medium_kernel<<<8 * sm_count(), 256, 0, s>>>(v, V, vertices, faces, d, medium, counters);
		tnt_raster_large_kernel<<<4 * sm_count(), 256, 0, s>>>(v, V, vertices, faces, d, large, counters);
		count_launch(3);
	}
	tnt_depth_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(n, d);
	count_launch();
	if (F > 0) {
		int32_t bad = 0;
		RGS_CUDA_TRY(cudaMemcpyAsync(&bad, counters + 2, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
		RGS_CUDA_TRY(cudaStreamSynchronize(s));
		if (bad) return fail(RGS_E_INVALID, "tnt mesh depth: a face index lies outside [0, V)");
	}
	return cuda_status(cudaGetLastError(), "tnt mesh depth");
}

int32_t rgs_tnt_visibility_count(int64_t N, const float* points, const float* depth, const float* w2c, float fx, float fy, float cx, float cy, int32_t H,
                                 int32_t W, float eps, int32_t* counts, void* cuda_stream) {
	if (N < 0) return fail(RGS_E_INVALID, "tnt visibility count: negative point count");
	if (H < 2 || W < 2 || H > 32768 || W > 32768) return fail(RGS_E_INVALID, "tnt visibility count: H and W must lie in [2, 32768]");
	if (!w2c || !depth || (N > 0 && (!points || !counts))) return fail(RGS_E_INVALID, "null pointer");
	if (N == 0) return RGS_OK;
	CountParams c;
	fill_matrix(c, w2c);
	c.fx = fx, c.fy = fy, c.cx = cx, c.cy = cy, c.eps = eps, c.H = H, c.W = W;
	c.inv_w1 = 1.0f / (float)(W - 1);
	c.inv_h1 = 1.0f / (float)(H - 1);
	tnt_visibility_kernel<<<(unsigned)((N + 255) / 256), 256, 0, (cudaStream_t)cuda_stream>>>(N, points, depth, c, counts);
	count_launch();
	return cuda_status(cudaGetLastError(), "tnt visibility count");
}

}  // extern "C"

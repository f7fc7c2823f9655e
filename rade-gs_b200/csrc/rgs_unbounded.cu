// rgs_unbounded.cu -- the contracted-space TSDF mesh of unbounded scenes: the reference's GaussianExtractor path
// (utils/mesh_utils.py:163-271, utils/mcube_utils.py:17-95, there eager torch, scikit-image and trimesh).  Runs once per
// trained model, off the rasterizer path.
//
// The contract (include/rgs_b200.h, rgs_unbounded_*) fixes every stored bit: each arithmetic step is one intrinsic rounded
// on its own (__fmul_rn / __fadd_rn / __fsub_rn / __fdiv_rn, IEEE sqrt, the fp64 ones for vertex positions), so nvcc
// cannot contract to FMA and a numpy restatement reproduces every output.
//   contract  one thread per point: normalise + contract (or uncontract + unnormalise + clip) and the norm.
//   sdf       one thread per crop sample, voxel-outer: the running (tsdf, weight) pair stays in registers while the thread
//             folds the views in order; the projection matrices are staged through shared memory in chunks, the depth
//             maps are gathered through L1/L2.  The result therefore cannot depend on how the grid is split.
//   colors    the same projection per vertex with a constant truncation and a running RGB average.
//   mcubes    per lattice point: case and owned sign-change edges -> two CUB exclusive scans -> emit (vertices by
//             (point, axis), triangles by (cell, table order)), so the crop mesh does not depend on scheduling.
//   merge     rint(x * 10^6) keys, two stable radix sorts (44 low bits, then 22 high bits), a max-scan of group heads:
//             each group keeps its first emitted vertex.
//   clusters  edge keys radix-sorted, union-find hooked to the smaller root (atomicCAS, roots only ever decrease), pointer
//             jumping, integer atomics for the sizes, one radix sort of the sizes for the k-th largest.
//
// This file also holds the C-ABI entry points rgs_unbounded_* (include/rgs_b200.h).
#include <cub/cub.cuh>

#include <cmath>

#include "rgs_common.cuh"
#include "rgs_mcubes.cuh"

namespace rgs {

namespace {

unsigned blocks_for(int64_t n) { return (unsigned)((n + 255) / 256); }

__device__ inline float norm3(float x, float y, float z) {
	return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
}

// torch.clamp(max=hi): NaN stays NaN
__device__ inline float clamp_max(float x, float hi) { return x > hi ? hi : x; }

struct Affine {
	float c[3], r, max_range;
};

// ---- contraction ------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(256) unb_contract_kernel(int64_t n, const float* __restrict__ in, Affine a, int inverse, float* __restrict__ out,
                                                           float* __restrict__ norms) {
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	float p[3] = {in[3 * i], in[3 * i + 1], in[3 * i + 2]};
	if (!inverse) {
		for (int k = 0; k < 3; k++) p[k] = __fdiv_rn(__fsub_rn(p[k], a.c[k]), a.r);
		const float m = norm3(p[0], p[1], p[2]);
		if (!(m < 1.0f)) {
			const float s = __fsub_rn(2.0f, __fdiv_rn(1.0f, m));
			for (int k = 0; k < 3; k++) p[k] = __fmul_rn(s, __fdiv_rn(p[k], m));
		}
	} else {
		const float m = norm3(p[0], p[1], p[2]);
		if (!(m < 1.0f)) {
			const float s = __fdiv_rn(1.0f, __fsub_rn(2.0f, m));
			for (int k = 0; k < 3; k++) p[k] = __fmul_rn(s, __fdiv_rn(p[k], m));
		}
		for (int k = 0; k < 3; k++) {
			const float w = __fadd_rn(__fmul_rn(p[k], a.r), a.c[k]);
			p[k] = w > a.max_range ? a.max_range : (w < -a.max_range ? -a.max_range : w);  // np.clip: NaN stays NaN
		}
	}
	for (int k = 0; k < 3; k++) out[3 * i + k] = p[k];
	if (norms) norms[i] = norm3(p[0], p[1], p[2]);
}

// ---- projection and bilinear sampling ---------------------------------------------------------------------------------

struct Views {
	int V, H, W;
	const float* proj;   // [V][16], the row-major 4x4 full_proj_transform: [x y z 1] @ M
	const float* depth;  // [V][H][W]
	const float* rgb;    // [V][3][H][W]
};

// [p 1] @ M; in view iff -1 < x/w < 1, -1 < y/w < 1 and w > 0
__device__ inline bool project(const float* M, float px, float py, float pz, float& u, float& v, float& w) {
	float c[4];
#pragma unroll
	for (int j = 0; j < 4; j++) c[j] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(px, M[j]), __fmul_rn(py, M[4 + j])), __fmul_rn(pz, M[8 + j])), M[12 + j]);
	w = c[3];
	u = __fdiv_rn(c[0], w);
	v = __fdiv_rn(c[1], w);
	return u > -1.0f && u < 1.0f && v > -1.0f && v < 1.0f && w > 0.0f;
}

// grid_sample(mode='bilinear', padding_mode='border', align_corners=True) of one channel at normalised (u, v)
struct Bilinear {
	int64_t o[4];
	float wt[4];
	bool in[4];
};

__device__ inline Bilinear bilinear(float u, float v, int W, int H) {
	float ix = __fmul_rn(__fdiv_rn(__fadd_rn(u, 1.0f), 2.0f), (float)(W - 1));
	float iy = __fmul_rn(__fdiv_rn(__fadd_rn(v, 1.0f), 2.0f), (float)(H - 1));
	ix = fminf((float)(W - 1), fmaxf(ix, 0.0f));
	iy = fminf((float)(H - 1), fmaxf(iy, 0.0f));
	const float x0 = floorf(ix), y0 = floorf(iy), x1 = __fadd_rn(x0, 1.0f), y1 = __fadd_rn(y0, 1.0f);
	Bilinear b;
	b.wt[0] = __fmul_rn(__fsub_rn(x1, ix), __fsub_rn(y1, iy));  // nw
	b.wt[1] = __fmul_rn(__fsub_rn(ix, x0), __fsub_rn(y1, iy));  // ne
	b.wt[2] = __fmul_rn(__fsub_rn(x1, ix), __fsub_rn(iy, y0));  // sw
	b.wt[3] = __fmul_rn(__fsub_rn(ix, x0), __fsub_rn(iy, y0));  // se
	const int xi = (int)x0, yi = (int)y0;
#pragma unroll
	for (int q = 0; q < 4; q++) {
		const int x = xi + (q & 1), y = yi + (q >> 1);
		b.in[q] = x < W && y < H;
		b.o[q] = (int64_t)y * W + x;
	}
	return b;
}

__device__ inline float sample(const float* __restrict__ img, const Bilinear& b) {
	float acc = 0.0f;
#pragma unroll
	for (int q = 0; q < 4; q++)
		if (b.in[q]) acc = __fadd_rn(acc, __fmul_rn(__ldg(img + b.o[q]), b.wt[q]));
	return acc;
}

// ---- SDF of one crop --------------------------------------------------------------------------------------------------

constexpr int SDF_THREADS = 256;
constexpr int PROJ_CHUNK = 64;  // views whose matrices sit in shared memory at a time

__global__ void __launch_bounds__(SDF_THREADS) unb_sdf_kernel(int n, const float* __restrict__ xs, const float* __restrict__ ys, const float* __restrict__ zs,
                                                              Views vw, Affine a, float trunc0, float* __restrict__ sdf) {
	__shared__ float sM[PROJ_CHUNK * 16];
	const int64_t N = (int64_t)n * n * n;
	const int64_t g = (int64_t)blockIdx.x * SDF_THREADS + threadIdx.x;
	const bool live = g < N;
	float p[3] = {0.0f, 0.0f, 0.0f}, trunc = trunc0;
	if (live) {
		const int k = (int)(g % n), j = (int)(g / n % n), i = (int)(g / ((int64_t)n * n));
		float s[3] = {xs[i], ys[j], zs[k]};
		const float m = norm3(s[0], s[1], s[2]);
		if (!(m < 1.0f)) {
			const float f = __fdiv_rn(1.0f, __fsub_rn(2.0f, m));
			for (int q = 0; q < 3; q++) s[q] = __fmul_rn(f, __fdiv_rn(s[q], m));
		}
		for (int q = 0; q < 3; q++) p[q] = __fadd_rn(__fmul_rn(s[q], a.r), a.c[q]);
		// adaptive truncation on the world-space norm (the reference's expression)
		const float pm = norm3(p[0], p[1], p[2]);
		if (pm > 1.0f) trunc = __fmul_rn(trunc0, __fdiv_rn(1.0f, __fsub_rn(2.0f, clamp_max(pm, 1.9f))));
	}
	const int64_t HW = (int64_t)vw.H * vw.W;
	float t = 1.0f, wt = 1.0f;
	for (int v0 = 0; v0 < vw.V; v0 += PROJ_CHUNK) {
		const int nv = min(PROJ_CHUNK, vw.V - v0);
		__syncthreads();
		for (int q = threadIdx.x; q < nv * 16; q += SDF_THREADS) sM[q] = vw.proj[(int64_t)v0 * 16 + q];
		__syncthreads();
		if (!live) continue;
		for (int v = 0; v < nv; v++) {
			float u, vv, w;
			if (!project(sM + 16 * v, p[0], p[1], p[2], u, vv, w)) continue;
			const float d = sample(vw.depth + (int64_t)(v0 + v) * HW, bilinear(u, vv, vw.W, vw.H));
			const float s = __fsub_rn(d, w);
			if (!(s > -trunc)) continue;
			const float c = fminf(fmaxf(__fdiv_rn(s, trunc), -1.0f), 1.0f);
			t = __fdiv_rn(__fadd_rn(__fmul_rn(t, wt), c), __fadd_rn(wt, 1.0f));
			wt = __fadd_rn(wt, 1.0f);
		}
	}
	if (live) sdf[g] = t;
}

// ---- vertex colours ---------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(256) unb_colors_kernel(int64_t N, const float* __restrict__ pts, Views vw, float trunc, float* __restrict__ out) {
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= N) return;
	const float px = pts[3 * i], py = pts[3 * i + 1], pz = pts[3 * i + 2];
	const int64_t HW = (int64_t)vw.H * vw.W;
	float col[3] = {0.0f, 0.0f, 0.0f}, wt = 1.0f;
	for (int v = 0; v < vw.V; v++) {
		float u, vv, w;
		if (!project(vw.proj + 16 * v, px, py, pz, u, vv, w)) continue;
		const Bilinear b = bilinear(u, vv, vw.W, vw.H);
		const float s = __fsub_rn(sample(vw.depth + (int64_t)v * HW, b), w);
		if (!(s > -trunc)) continue;
		const float wp = __fadd_rn(wt, 1.0f);
		for (int k = 0; k < 3; k++) col[k] = __fdiv_rn(__fadd_rn(__fmul_rn(col[k], wt), sample(vw.rgb + ((int64_t)v * 3 + k) * HW, b)), wp);
		wt = wp;
	}
	for (int k = 0; k < 3; k++) out[3 * i + k] = col[k];
}

// ---- marching cubes on a dense crop -----------------------------------------------------------------------------------

// per lattice point g = (i n + j) n + k: info bits 0..7 = case of the cell at g (0 when g has no cell), bits 8..10 = the
// owned edges (g, a) that change sign; cnt[g] = owned vertices, cnt[M + 1 + g] = triangles (cnt[M] = cnt[2M + 1] = 0)
__global__ void __launch_bounds__(256) unb_mc_count_kernel(int n, const float* __restrict__ f, uint16_t* __restrict__ info, int32_t* __restrict__ cnt) {
	const int64_t M = (int64_t)n * n * n;
	const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (g > M) return;
	if (g == M) {
		cnt[M] = 0;
		cnt[2 * M + 1] = 0;
		return;
	}
	const int64_t st[3] = {(int64_t)n * n, n, 1};
	const int p[3] = {(int)(g / st[0]), (int)(g / n % n), (int)(g % n)};
	const bool in0 = f[g] < 0.0f;
	int m = 0;
#pragma unroll
	for (int a = 0; a < 3; a++)
		if (p[a] + 1 < n && (f[g + st[a]] < 0.0f) != in0) m |= 1 << a;
	int cs = 0;
	if (p[0] + 1 < n && p[1] + 1 < n && p[2] + 1 < n) {
#pragma unroll
		for (int c = 0; c < 8; c++) cs |= (f[g + (c & 1) * st[0] + (c >> 1 & 1) * st[1] + (c >> 2 & 1) * st[2]] < 0.0f) << c;
	}
	info[g] = (uint16_t)(cs | m << 8);
	cnt[g] = __popc(m);
	cnt[M + 1 + g] = c_tri.n[cs];
}

struct Crop {
	double lo[3], sp[3];
};

// lattice step along axis a
__device__ inline int64_t stride(int a, int n) { return a == 0 ? (int64_t)n * n : (a == 1 ? n : 1); }

__global__ void __launch_bounds__(256) unb_mc_emit_kernel(int n, const float* __restrict__ f, Crop cr, const uint16_t* __restrict__ info,
                                                          const int32_t* __restrict__ voff, const int32_t* __restrict__ toff, double* __restrict__ verts,
                                                          int32_t* __restrict__ tris) {
	const int64_t M = (int64_t)n * n * n;
	const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= M) return;
	const int p[3] = {(int)(g / ((int64_t)n * n)), (int)(g / n % n), (int)(g % n)};
	const int m = info[g] >> 8, cs = info[g] & 0xff;
	int r = voff[g];
	for (int a = 0; a < 3; a++) {
		if (!(m >> a & 1)) continue;
		const double f0 = f[g], f1 = f[g + stride(a, n)];
		const double t = __ddiv_rn(f0, __dsub_rn(f0, f1));
		for (int k = 0; k < 3; k++) {
			const double x = k == a ? __dadd_rn((double)p[k], t) : (double)p[k];
			verts[3 * (int64_t)r + k] = __dadd_rn(__dmul_rn(x, cr.sp[k]), cr.lo[k]);
		}
		r++;
	}
	const int nt = c_tri.n[cs];
	int32_t* tri = tris + 3 * (int64_t)toff[g];
	for (int q = 0; q < 3 * nt; q++) {
		const int e = c_tri.e[cs][q], a = e / 4, o = e % 4;
		const int64_t h = g + (o & 1) * stride(other_axis(a, 0), n) + (o >> 1) * stride(other_axis(a, 1), n);
		tri[q] = voff[h] + __popc((info[h] >> 8) & ((1 << a) - 1));
	}
}

// ---- vertex merge -----------------------------------------------------------------------------------------------------

constexpr int MERGE_BITS = 22;                  // per axis: rint(x * 1e6) + 2^21 in [0, 2^22)
constexpr int64_t MERGE_BIAS = 1 << (MERGE_BITS - 1);

__global__ void __launch_bounds__(256) unb_merge_keys_kernel(int64_t V, const double* __restrict__ v, uint64_t* __restrict__ lo, uint32_t* __restrict__ hi,
                                                             int32_t* __restrict__ idx, int32_t* __restrict__ flag) {
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= V) return;
	uint64_t k[3];
	for (int a = 0; a < 3; a++) {
		const double r = rint(__dmul_rn(v[3 * i + a], 1e6));
		if (!(r >= -(double)MERGE_BIAS && r < (double)MERGE_BIAS)) {  // also NaN
			atomicOr(flag, 1);
			k[a] = 0;
		} else {
			k[a] = (uint64_t)((int64_t)r + MERGE_BIAS);
		}
	}
	lo[i] = k[1] << MERGE_BITS | k[2];
	hi[i] = (uint32_t)k[0];
	idx[i] = (int32_t)i;
}

__global__ void __launch_bounds__(256) unb_gather_hi_kernel(int64_t V, const uint32_t* __restrict__ hi, const int32_t* __restrict__ idx, uint32_t* __restrict__ out) {
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i < V) out[i] = hi[idx[i]];
}

// position of the group head (first of equal keys in sorted order) at or before each sorted position
__global__ void __launch_bounds__(256) unb_heads_kernel(int64_t V, const int32_t* __restrict__ sidx, const uint64_t* __restrict__ lo,
                                                        const uint32_t* __restrict__ hi, int32_t* __restrict__ head) {
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= V) return;
	bool h = i == 0;
	if (!h) {
		const int32_t a = sidx[i], b = sidx[i - 1];
		h = lo[a] != lo[b] || hi[a] != hi[b];
	}
	head[i] = h ? (int32_t)i : 0;
}

struct MaxOp {
	__device__ int32_t operator()(int32_t a, int32_t b) const { return a > b ? a : b; }
};

// rep[v] = the first emitted vertex of v's group; surv[v] = (rep[v] == v), surv[V] = 0
__global__ void __launch_bounds__(256) unb_rep_kernel(int64_t V, const int32_t* __restrict__ sidx, const int32_t* __restrict__ hpos, int32_t* __restrict__ rep) {
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i < V) rep[sidx[i]] = sidx[hpos[i]];
}

__global__ void __launch_bounds__(256) unb_survivors_kernel(int64_t V, const int32_t* __restrict__ rep, int32_t* __restrict__ surv) {
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i < V) surv[i] = rep[i] == (int32_t)i;
	else if (i == V) surv[V] = 0;
}

__global__ void __launch_bounds__(256) unb_merge_emit_kernel(int64_t V, const double* __restrict__ v, const int32_t* __restrict__ rep,
                                                             const int32_t* __restrict__ newid, float* __restrict__ out) {
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= V || rep[i] != (int32_t)i) return;
	const int64_t r = newid[i];
	for (int k = 0; k < 3; k++) out[3 * r + k] = (float)v[3 * i + k];  // round to nearest, as .float()
}

__global__ void __launch_bounds__(256) unb_check_tris_kernel(int64_t F3, const int32_t* __restrict__ tris, int64_t V, int32_t* __restrict__ flag) {
	const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (m < F3 && !(tris[m] >= 0 && tris[m] < V)) atomicOr(flag, 2);
}

__global__ void __launch_bounds__(256) unb_renumber_kernel(int64_t F3, const int32_t* __restrict__ tris, const int32_t* __restrict__ rep,
                                                           const int32_t* __restrict__ newid, int32_t* __restrict__ out) {
	const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (m < F3) out[m] = newid[rep[tris[m]]];
}

// ---- connected triangle clusters --------------------------------------------------------------------------------------

__global__ void __launch_bounds__(256) unb_edges_kernel(int64_t F, const int32_t* __restrict__ tris, uint64_t* __restrict__ keys, int32_t* __restrict__ tid,
                                                        int32_t* __restrict__ parent) {
	const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= F) return;
	for (int e = 0; e < 3; e++) {
		const uint32_t a = (uint32_t)tris[3 * t + e], b = (uint32_t)tris[3 * t + (e + 1) % 3];
		keys[3 * t + e] = (uint64_t)min(a, b) << 32 | max(a, b);
		tid[3 * t + e] = (int32_t)t;
	}
	parent[t] = (int32_t)t;
}

// representative of x; halves paths on the way (parents only ever decrease, within one component)
__device__ inline int32_t find_root(int32_t* parent, int32_t x) {
	int32_t p = *(volatile int32_t*)&parent[x];
	while (p != x) {
		const int32_t gp = *(volatile int32_t*)&parent[p];
		if (gp != p) *(volatile int32_t*)&parent[x] = gp;
		x = p;
		p = gp;
	}
	return x;
}

// triangles of one edge key are consecutive in sorted order: each is united with its predecessor; the larger root is hooked
// under the smaller, so every cluster's root ends as its smallest triangle id
__global__ void __launch_bounds__(256) unb_union_kernel(int64_t E, const uint64_t* __restrict__ keys, const int32_t* __restrict__ tid, int32_t* parent) {
	const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (m == 0 || m >= E || keys[m] != keys[m - 1]) return;
	int32_t a = find_root(parent, tid[m - 1]), b = find_root(parent, tid[m]);
	while (a != b) {
		if (a < b) {
			const int32_t t = a;
			a = b;
			b = t;
		}
		const int32_t old = atomicCAS(&parent[a], a, b);
		if (old == a) break;
		a = find_root(parent, old);
		b = find_root(parent, b);
	}
}

__global__ void __launch_bounds__(256) unb_flatten_kernel(int64_t F, int32_t* parent, int32_t* __restrict__ size) {
	const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= F) return;
	const int32_t r = find_root(parent, (int32_t)t);
	atomicAdd(&size[r], 1);
}

// after every root is final: root[t] (into tid, reused), the cluster sizes (0 for non-roots) and the cluster count
__global__ void __launch_bounds__(256) unb_roots_kernel(int64_t F, const int32_t* __restrict__ parent, const int32_t* __restrict__ size, int32_t* __restrict__ root,
                                                        uint32_t* __restrict__ csize, int32_t* __restrict__ nclusters) {
	const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= F) return;
	int32_t r = (int32_t)t;
	while (parent[r] != r) r = parent[r];
	root[t] = r;
	const bool is_root = r == (int32_t)t;
	csize[t] = is_root ? (uint32_t)size[t] : 0u;
	if (is_root) atomicAdd(nclusters, 1);
}

// thr = max(sorted_sizes[-k], 50) over the C cluster sizes (ascending at the end of `sorted`, which holds F entries); with
// fewer than k clusters every cluster of at least 50 triangles stays
__global__ void unb_threshold_kernel(int64_t F, const uint32_t* __restrict__ sorted, const int32_t* __restrict__ nclusters, int64_t k, int32_t* __restrict__ thr) {
	const int64_t C = *nclusters;
	int64_t s = 0;
	if (k == 0 && C > 0) s = sorted[F - C];
	else if (k > 0 && k <= C) s = sorted[F - k];
	*thr = (int32_t)(s > 50 ? s : 50);
}

// keep[t] (cluster large enough), vref[v] = 1 for the vertices of kept triangles (vref zeroed before), tkeep[t] = kept and
// not degenerate; tkeep[F] = 0
__global__ void __launch_bounds__(256) unb_keep_kernel(int64_t F, const int32_t* __restrict__ tris, const int32_t* __restrict__ root,
                                                       const int32_t* __restrict__ size, const int32_t* __restrict__ thr, int32_t* __restrict__ vref,
                                                       int32_t* __restrict__ tkeep) {
	const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (t > F) return;
	if (t == F) {
		tkeep[F] = 0;
		return;
	}
	const bool keep = size[root[t]] >= *thr;
	const int32_t a = tris[3 * t], b = tris[3 * t + 1], c = tris[3 * t + 2];
	if (keep) {
		vref[a] = 1;
		vref[b] = 1;
		vref[c] = 1;
	}
	tkeep[t] = keep && a != b && b != c && a != c;
}

__global__ void __launch_bounds__(256) unb_clean_emit_kernel(int64_t V, int64_t F, const int32_t* __restrict__ tris, const int32_t* __restrict__ voff,
                                                             const int32_t* __restrict__ toff, int32_t* __restrict__ vidx, int32_t* __restrict__ tout) {
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i < V && voff[i + 1] != voff[i]) vidx[voff[i]] = (int32_t)i;
	if (i < F && toff[i + 1] != toff[i])
		for (int k = 0; k < 3; k++) tout[3 * (int64_t)toff[i] + k] = voff[tris[3 * i + k]];
}

// ---- host helpers -----------------------------------------------------------------------------------------------------

size_t exclusive_sum_bytes(int64_t n) {
	size_t b = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, b, (const int32_t*)nullptr, (int32_t*)nullptr, n);
	return b;
}

// in place: cnt[0..n) -> exclusive offsets
cudaError_t exclusive_sum(int32_t* cnt, int64_t n, char* temp, size_t bytes, cudaStream_t s) {
	size_t b = bytes;
	count_launch();
	return cub::DeviceScan::ExclusiveSum(temp, b, cnt, cnt, n, s);
}

struct McScratch {
	uint16_t* info;
	int32_t* cnt;  // [2 (M + 1)]: vertex counts then triangle counts, scanned in place
	char* temp;
	size_t temp_bytes;
};

McScratch carve_mc(char* base, int64_t M, size_t* total) {
	Carver cv(base);
	McScratch x;
	x.temp_bytes = exclusive_sum_bytes(M + 1);
	x.info = cv.take<uint16_t>(M);
	x.cnt = cv.take<int32_t>(2 * (M + 1));
	x.temp = cv.take<char>(x.temp_bytes);
	if (total) *total = cv.size();
	return x;
}

struct MergeScratch {
	uint64_t *lo, *lo_s;
	uint32_t *hi, *hi_g, *hi_s;
	int32_t *idx, *idx1, *idx2, *hpos, *rep, *newid, *flag;
	char* temp;
	size_t temp_bytes;
};

MergeScratch carve_merge(char* base, int64_t V, size_t* total) {
	MergeScratch x;
	size_t a = 0, b = 0, c = 0, d = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, a, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr, (int)V, 0, 2 * MERGE_BITS);
	cub::DeviceRadixSort::SortPairs(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr, (int)V, 0, MERGE_BITS);
	cub::DeviceScan::InclusiveScan(nullptr, c, (const int32_t*)nullptr, (int32_t*)nullptr, MaxOp(), (int)V);
	d = exclusive_sum_bytes(V + 1);
	x.temp_bytes = std::max(std::max(a, b), std::max(c, d));
	Carver cv(base);
	x.lo = cv.take<uint64_t>(V);
	x.lo_s = cv.take<uint64_t>(V);
	x.hi = cv.take<uint32_t>(V);
	x.hi_g = cv.take<uint32_t>(V);
	x.hi_s = cv.take<uint32_t>(V);
	x.idx = cv.take<int32_t>(V);
	x.idx1 = cv.take<int32_t>(V);
	x.idx2 = cv.take<int32_t>(V);
	x.hpos = cv.take<int32_t>(V);
	x.rep = cv.take<int32_t>(V);
	x.newid = cv.take<int32_t>(V + 1);
	x.flag = cv.take<int32_t>(1);
	x.temp = cv.take<char>(x.temp_bytes);
	if (total) *total = cv.size();
	return x;
}

struct ClusterScratch {
	uint64_t *keys, *keys_s;
	int32_t *tid, *tid_s, *parent, *size, *root, *vref, *tkeep, *nclusters, *thr, *flag;
	uint32_t *csize, *csize_s;
	char* temp;
	size_t temp_bytes;
};

ClusterScratch carve_clusters(char* base, int64_t V, int64_t F, size_t* total) {
	ClusterScratch x;
	size_t a = 0, b = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, a, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(3 * F));
	cub::DeviceRadixSort::SortKeys(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)F);
	x.temp_bytes = std::max(std::max(a, b), std::max(exclusive_sum_bytes(V + 1), exclusive_sum_bytes(F + 1)));
	Carver cv(base);
	x.keys = cv.take<uint64_t>(3 * F);
	x.keys_s = cv.take<uint64_t>(3 * F);
	x.tid = cv.take<int32_t>(3 * F);
	x.tid_s = cv.take<int32_t>(3 * F);
	x.parent = cv.take<int32_t>(F);
	x.size = cv.take<int32_t>(F);
	x.root = cv.take<int32_t>(F);
	x.csize = cv.take<uint32_t>(F);
	x.csize_s = cv.take<uint32_t>(F);
	x.vref = cv.take<int32_t>(V + 1);
	x.tkeep = cv.take<int32_t>(F + 1);
	x.nclusters = cv.take<int32_t>(1);
	x.thr = cv.take<int32_t>(1);
	x.flag = cv.take<int32_t>(1);
	x.temp = cv.take<char>(x.temp_bytes);
	if (total) *total = cv.size();
	return x;
}

}  // namespace
}  // namespace rgs

using namespace rgs;

extern "C" {

static int views_check(int32_t V, int32_t H, int32_t W, const float* proj, const float* depth) {
	if (V < 1) return fail(RGS_E_INVALID, "unbounded: at least one view is required");
	if (H < 1 || W < 1 || (int64_t)H * W > ((int64_t)1 << 31)) return fail(RGS_E_INVALID, "unbounded: view size out of range");
	if (!proj || !depth) return fail(RGS_E_INVALID, "null pointer");
	return RGS_OK;
}

static int affine_check(const float center[3], float radius) {
	if (!center) return fail(RGS_E_INVALID, "null pointer");
	for (int k = 0; k < 3; k++)
		if (!std::isfinite(center[k])) return fail(RGS_E_INVALID, "unbounded: center must be finite");
	if (!(std::isfinite(radius) && radius > 0.0f)) return fail(RGS_E_INVALID, "unbounded: radius must be positive and finite");
	return RGS_OK;
}

static Affine make_affine(const float center[3], float radius, float max_range) {
	Affine a;
	for (int k = 0; k < 3; k++) a.c[k] = center[k];
	a.r = radius;
	a.max_range = max_range;
	return a;
}

int32_t rgs_unbounded_contract(int64_t n, const float* points, const float center[3], float radius, int32_t inverse, float max_range, float* out, float* norms,
                               void* cuda_stream) {
	if (n < 0 || n > INT32_MAX) return fail(RGS_E_INVALID, "unbounded contract: point count out of range");
	if (int rc = affine_check(center, radius)) return rc;
	if (std::isnan(max_range) || !(max_range > 0.0f)) return fail(RGS_E_INVALID, "unbounded contract: max_range must be positive");
	if (n == 0) return RGS_OK;
	if (!points || !out) return fail(RGS_E_INVALID, "null pointer");
	unb_contract_kernel<<<blocks_for(n), 256, 0, (cudaStream_t)cuda_stream>>>(n, points, make_affine(center, radius, max_range), inverse != 0, out, norms);
	count_launch();
	return cuda_status(cudaGetLastError(), "unbounded contract");
}

int32_t rgs_unbounded_sdf(int32_t n, const float* xs, const float* ys, const float* zs, int32_t V, int32_t H, int32_t W, const float* full_proj,
                          const float* depth, const float center[3], float radius, float trunc, float* sdf, void* cuda_stream) {
	if (n < 1 || n > RGS_UNBOUNDED_MAX_CROP) return fail(RGS_E_INVALID, "unbounded sdf: crop size must be in [1, 640]");
	if (int rc = views_check(V, H, W, full_proj, depth)) return rc;
	if (int rc = affine_check(center, radius)) return rc;
	if (!(std::isfinite(trunc) && trunc > 0.0f)) return fail(RGS_E_INVALID, "unbounded sdf: trunc must be positive and finite");
	if (!xs || !ys || !zs || !sdf) return fail(RGS_E_INVALID, "null pointer");
	const int64_t N = (int64_t)n * n * n;
	unb_sdf_kernel<<<(unsigned)((N + SDF_THREADS - 1) / SDF_THREADS), SDF_THREADS, 0, (cudaStream_t)cuda_stream>>>(
	    n, xs, ys, zs, Views{V, H, W, full_proj, depth, nullptr}, make_affine(center, radius, 0.0f), trunc, sdf);
	count_launch();
	return cuda_status(cudaGetLastError(), "unbounded sdf");
}

int32_t rgs_unbounded_colors(int64_t N, const float* points, int32_t V, int32_t H, int32_t W, const float* full_proj, const float* depth, const float* rgb,
                             float trunc, float* colors, void* cuda_stream) {
	if (N < 0 || N > INT32_MAX) return fail(RGS_E_INVALID, "unbounded colors: point count out of range");
	if (int rc = views_check(V, H, W, full_proj, depth)) return rc;
	if (!(std::isfinite(trunc) && trunc > 0.0f)) return fail(RGS_E_INVALID, "unbounded colors: trunc must be positive and finite");
	if (N == 0) return RGS_OK;
	if (!points || !rgb || !colors) return fail(RGS_E_INVALID, "null pointer");
	unb_colors_kernel<<<blocks_for(N), 256, 0, (cudaStream_t)cuda_stream>>>(N, points, Views{V, H, W, full_proj, depth, rgb}, trunc, colors);
	count_launch();
	return cuda_status(cudaGetLastError(), "unbounded colors");
}

int32_t rgs_unbounded_mcubes(int32_t n, const float* sdf, const double lo[3], const double spacing[3], rgs_resize_fn resize, rgs_unbounded_mesh_out* out,
                             void* scratch_user, void* cuda_stream) {
	if (n < 2 || n > RGS_UNBOUNDED_MAX_CROP) return fail(RGS_E_INVALID, "unbounded mcubes: crop size must be in [2, 640]");
	if (!sdf || !lo || !spacing || !resize || !out) return fail(RGS_E_INVALID, "null pointer");
	Crop cr;
	for (int k = 0; k < 3; k++) {
		if (!std::isfinite(lo[k]) || !std::isfinite(spacing[k])) return fail(RGS_E_INVALID, "unbounded mcubes: crop origin and spacing must be finite");
		cr.lo[k] = lo[k];
		cr.sp[k] = spacing[k];
	}
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	const int64_t M = (int64_t)n * n * n;
	size_t bytes = 0;
	carve_mc(nullptr, M, &bytes);
	char* buf;
	int rc;
	if ((rc = grow(resize, scratch_user, bytes, buf, "unbounded scratch")) != RGS_OK) return rc;
	const McScratch x = carve_mc(buf, M, nullptr);
	unb_mc_count_kernel<<<blocks_for(M + 1), 256, 0, s>>>(n, sdf, x.info, x.cnt);
	count_launch();
	RGS_CUDA_TRY(cudaGetLastError());
	RGS_CUDA_TRY(exclusive_sum(x.cnt, M + 1, x.temp, x.temp_bytes, s));
	RGS_CUDA_TRY(exclusive_sum(x.cnt + M + 1, M + 1, x.temp, x.temp_bytes, s));
	int32_t tot[2];
	RGS_CUDA_TRY(cudaMemcpyAsync(tot, x.cnt + M, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	RGS_CUDA_TRY(cudaMemcpyAsync(tot + 1, x.cnt + 2 * M + 1, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	RGS_CUDA_TRY(cudaStreamSynchronize(s));
	out->num_vertices = tot[0];
	out->num_triangles = tot[1];
	char *v, *t;
	if ((rc = grow(resize, out->vertices_user, (size_t)tot[0] * 3 * sizeof(double), v, "unbounded mesh")) != RGS_OK ||
	    (rc = grow(resize, out->triangles_user, (size_t)tot[1] * 3 * sizeof(int32_t), t, "unbounded mesh")) != RGS_OK)
		return rc;
	if (tot[0] == 0 && tot[1] == 0) return RGS_OK;
	unb_mc_emit_kernel<<<blocks_for(M), 256, 0, s>>>(n, sdf, cr, x.info, x.cnt, x.cnt + M + 1, reinterpret_cast<double*>(v), reinterpret_cast<int32_t*>(t));
	count_launch();
	return cuda_status(cudaGetLastError(), "unbounded mcubes");
}

int32_t rgs_unbounded_merge(int64_t V, const double* vertices, int64_t F, const int32_t* triangles, int32_t* triangles_out, rgs_resize_fn resize,
                            void* vertices_user, int64_t* num_merged, void* scratch_user, void* cuda_stream) {
	if (V < 0 || V >= INT32_MAX || F < 0 || 3 * F > INT32_MAX) return fail(RGS_E_INVALID, "unbounded merge: vertex / triangle count out of range");
	if (!resize || !num_merged || (V > 0 && !vertices) || (F > 0 && (!triangles || !triangles_out))) return fail(RGS_E_INVALID, "null pointer");
	if (V == 0 && F > 0) return fail(RGS_E_INVALID, "unbounded merge: triangle index out of range");
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	char* vout;
	int rc;
	if (V == 0) {
		*num_merged = 0;
		return grow(resize, vertices_user, 0, vout, "unbounded mesh");
	}
	size_t bytes = 0;
	carve_merge(nullptr, V, &bytes);
	char* buf;
	if ((rc = grow(resize, scratch_user, bytes, buf, "unbounded scratch")) != RGS_OK) return rc;
	const MergeScratch x = carve_merge(buf, V, nullptr);
	RGS_CUDA_TRY(cudaMemsetAsync(x.flag, 0, sizeof(int32_t), s));
	unb_merge_keys_kernel<<<blocks_for(V), 256, 0, s>>>(V, vertices, x.lo, x.hi, x.idx, x.flag);
	if (F > 0) unb_check_tris_kernel<<<blocks_for(3 * F), 256, 0, s>>>(3 * F, triangles, V, x.flag);
	count_launch(2);
	size_t tb = x.temp_bytes;
	// stable LSD order: (y, z) first, then x; ties keep ascending vertex index
	RGS_CUDA_TRY(cub::DeviceRadixSort::SortPairs(x.temp, tb, x.lo, x.lo_s, x.idx, x.idx1, (int)V, 0, 2 * MERGE_BITS, s));
	unb_gather_hi_kernel<<<blocks_for(V), 256, 0, s>>>(V, x.hi, x.idx1, x.hi_g);
	tb = x.temp_bytes;
	RGS_CUDA_TRY(cub::DeviceRadixSort::SortPairs(x.temp, tb, x.hi_g, x.hi_s, x.idx1, x.idx2, (int)V, 0, MERGE_BITS, s));
	unb_heads_kernel<<<blocks_for(V), 256, 0, s>>>(V, x.idx2, x.lo, x.hi, x.hpos);
	tb = x.temp_bytes;
	RGS_CUDA_TRY(cub::DeviceScan::InclusiveScan(x.temp, tb, x.hpos, x.hpos, MaxOp(), (int)V, s));
	unb_rep_kernel<<<blocks_for(V), 256, 0, s>>>(V, x.idx2, x.hpos, x.rep);
	unb_survivors_kernel<<<blocks_for(V + 1), 256, 0, s>>>(V, x.rep, x.newid);
	count_launch(7);
	RGS_CUDA_TRY(cudaGetLastError());
	RGS_CUDA_TRY(exclusive_sum(x.newid, V + 1, x.temp, x.temp_bytes, s));
	int32_t h[2];
	RGS_CUDA_TRY(cudaMemcpyAsync(h, x.newid + V, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	RGS_CUDA_TRY(cudaMemcpyAsync(h + 1, x.flag, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	RGS_CUDA_TRY(cudaStreamSynchronize(s));
	if (h[1] & 2) return fail(RGS_E_INVALID, "unbounded merge: triangle index out of range");
	if (h[1] & 1) return fail(RGS_E_INVALID, "unbounded merge: a vertex coordinate is not finite or |x| * 1e6 rounds outside [-2^21, 2^21)");
	*num_merged = h[0];
	if ((rc = grow(resize, vertices_user, (size_t)h[0] * 3 * sizeof(float), vout, "unbounded mesh")) != RGS_OK) return rc;
	unb_merge_emit_kernel<<<blocks_for(V), 256, 0, s>>>(V, vertices, x.rep, x.newid, reinterpret_cast<float*>(vout));
	if (F > 0) unb_renumber_kernel<<<blocks_for(3 * F), 256, 0, s>>>(3 * F, triangles, x.rep, x.newid, triangles_out);
	count_launch(2);
	return cuda_status(cudaGetLastError(), "unbounded merge");
}

int32_t rgs_unbounded_clusters(int64_t V, int64_t F, const int32_t* triangles, int64_t cluster_to_keep, rgs_resize_fn resize, rgs_unbounded_clusters_out* out,
                               void* scratch_user, void* cuda_stream) {
	if (V < 0 || V >= INT32_MAX || F < 0 || 3 * F > INT32_MAX) return fail(RGS_E_INVALID, "unbounded clusters: vertex / triangle count out of range");
	if (cluster_to_keep < 0) return fail(RGS_E_INVALID, "unbounded clusters: cluster_to_keep must be >= 0");
	if (!resize || !out || (F > 0 && !triangles)) return fail(RGS_E_INVALID, "null pointer");
	if (V == 0 && F > 0) return fail(RGS_E_INVALID, "unbounded clusters: triangle index out of range");
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	char *vi, *to;
	int rc;
	if (F == 0) {  // no triangle: no cluster, and every vertex is unreferenced
		out->num_vertices = out->num_triangles = out->num_clusters = 0;
		out->threshold = 50;
		if ((rc = grow(resize, out->vertex_index_user, 0, vi, "unbounded mesh")) != RGS_OK) return rc;
		return grow(resize, out->triangles_user, 0, to, "unbounded mesh");
	}
	size_t bytes = 0;
	carve_clusters(nullptr, V, F, &bytes);
	char* buf;
	if ((rc = grow(resize, scratch_user, bytes, buf, "unbounded scratch")) != RGS_OK) return rc;
	const ClusterScratch x = carve_clusters(buf, V, F, nullptr);
	RGS_CUDA_TRY(cudaMemsetAsync(x.flag, 0, sizeof(int32_t), s));
	unb_check_tris_kernel<<<blocks_for(3 * F), 256, 0, s>>>(3 * F, triangles, V, x.flag);
	count_launch();
	int32_t flag = 0;
	RGS_CUDA_TRY(cudaMemcpyAsync(&flag, x.flag, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	RGS_CUDA_TRY(cudaStreamSynchronize(s));
	if (flag) return fail(RGS_E_INVALID, "unbounded clusters: triangle index out of range");
	RGS_CUDA_TRY(cudaMemsetAsync(x.size, 0, (size_t)F * sizeof(int32_t), s));
	RGS_CUDA_TRY(cudaMemsetAsync(x.vref, 0, (size_t)(V + 1) * sizeof(int32_t), s));
	RGS_CUDA_TRY(cudaMemsetAsync(x.nclusters, 0, sizeof(int32_t), s));
	unb_edges_kernel<<<blocks_for(F), 256, 0, s>>>(F, triangles, x.keys, x.tid, x.parent);
	size_t tb = x.temp_bytes;
	RGS_CUDA_TRY(cub::DeviceRadixSort::SortPairs(x.temp, tb, x.keys, x.keys_s, x.tid, x.tid_s, (int)(3 * F), 0, 64, s));
	unb_union_kernel<<<blocks_for(3 * F), 256, 0, s>>>(3 * F, x.keys_s, x.tid_s, x.parent);
	unb_flatten_kernel<<<blocks_for(F), 256, 0, s>>>(F, x.parent, x.size);
	unb_roots_kernel<<<blocks_for(F), 256, 0, s>>>(F, x.parent, x.size, x.root, x.csize, x.nclusters);
	tb = x.temp_bytes;
	RGS_CUDA_TRY(cub::DeviceRadixSort::SortKeys(x.temp, tb, x.csize, x.csize_s, (int)F, 0, 32, s));
	unb_threshold_kernel<<<1, 1, 0, s>>>(F, x.csize_s, x.nclusters, cluster_to_keep, x.thr);
	unb_keep_kernel<<<blocks_for(F + 1), 256, 0, s>>>(F, triangles, x.root, x.size, x.thr, x.vref, x.tkeep);
	count_launch(8);
	RGS_CUDA_TRY(cudaGetLastError());
	RGS_CUDA_TRY(exclusive_sum(x.vref, V + 1, x.temp, x.temp_bytes, s));
	RGS_CUDA_TRY(exclusive_sum(x.tkeep, F + 1, x.temp, x.temp_bytes, s));
	int32_t h[4];
	RGS_CUDA_TRY(cudaMemcpyAsync(h, x.vref + V, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	RGS_CUDA_TRY(cudaMemcpyAsync(h + 1, x.tkeep + F, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	RGS_CUDA_TRY(cudaMemcpyAsync(h + 2, x.nclusters, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	RGS_CUDA_TRY(cudaMemcpyAsync(h + 3, x.thr, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	RGS_CUDA_TRY(cudaStreamSynchronize(s));
	out->num_vertices = h[0];
	out->num_triangles = h[1];
	out->num_clusters = h[2];
	out->threshold = h[3];
	if ((rc = grow(resize, out->vertex_index_user, (size_t)h[0] * sizeof(int32_t), vi, "unbounded mesh")) != RGS_OK ||
	    (rc = grow(resize, out->triangles_user, (size_t)h[1] * 3 * sizeof(int32_t), to, "unbounded mesh")) != RGS_OK)
		return rc;
	unb_clean_emit_kernel<<<blocks_for(std::max(V, F)), 256, 0, s>>>(V, F, triangles, x.vref, x.tkeep, reinterpret_cast<int32_t*>(vi), reinterpret_cast<int32_t*>(to));
	count_launch();
	return cuda_status(cudaGetLastError(), "unbounded clusters");
}

}  // extern "C"

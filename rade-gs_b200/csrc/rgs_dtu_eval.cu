// rgs_dtu_eval.cu -- the DTU chamfer evaluation (reference dtu_eval/eval.py) and its mesh culling
// (evaluate_dtu_mesh.py:82-138), on the GPU in fp64.  Runs once per trained model, off the rasterizer path.
//
// The contract (include/rgs_b200.h, rgs_dtu_*) fixes every stored bit: each arithmetic step is one intrinsic rounded on
// its own (__dadd_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn; a - b is __dadd_rn(a, -b), which is the same rounding), so nvcc
// contracts nothing and a numpy fp64 restatement reproduces the samples, the kept set and the distances.
//   sample     count (one thread per triangle: rows and points, walking the rows with a falling column bound), two CUB
//              exclusive scans, one host read, rows (one thread per triangle writes the first point of each of its rows),
//              emit (one thread per output point, binary search over the row starts), so a triangle with 10^6 samples
//              costs the same per point as one with 1.
//   downsample uniform grid of cell edge slightly above r, (cell, rank) radix sort, a 27-cell neighbour table per occupied
//              cell, then rounds over the undecided points until none is left (one host read per round).
//   nearest    an fp64 copy of rgs_knn.cu's design: Morton-sorted 32-point leaves of the reference set under an implicit
//              box tree, one warp per 32 Morton-sorted queries, nearer child first, stack one entry per lane.
//   cull       disk(6) dilation of each view's mask, then one thread per vertex over all views.
//
// This file also holds the C-ABI entry points rgs_dtu_* (include/rgs_b200.h).
#include <cub/cub.cuh>

#include "rgs_common.cuh"

namespace rgs {

namespace {

constexpr int64_t SAMPLE_SATURATED = (int64_t)1 << 31;   // a triangle whose count alone exceeds the limit (or cannot be counted)
constexpr double WALK_LIMIT = 4294967296.0;               // 2^32 rows or columns: more than 2^31 samples when the other side is >= 1

__device__ __forceinline__ double dsub(double a, double b) { return __dadd_rn(a, -b); }
__device__ __forceinline__ double dnorm3(double x, double y, double z) {
	return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
}
// the contract's squared pair distance: (dx*dx + dy*dy) + dz*dz, each operation rounded on its own
__device__ __forceinline__ double ddist2(double ax, double ay, double az, double bx, double by, double bz) {
	const double dx = dsub(ax, bx), dy = dsub(ay, by), dz = dsub(az, bz);
	return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}
__device__ __forceinline__ bool finite3d(double x, double y, double z) { return isfinite(x) && isfinite(y) && isfinite(z); }

// order-preserving double <-> uint64 map for atomicMin / atomicMax
__device__ __forceinline__ unsigned long long d2ord(double d) {
	const unsigned long long u = (unsigned long long)__double_as_longlong(d);
	return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__host__ __device__ __forceinline__ double ord2d(unsigned long long u) {
	const unsigned long long b = (u >> 63) ? (u & 0x7fffffffffffffffull) : ~u;
	double d;
	memcpy(&d, &b, sizeof(d));
	return d;
}

// bits[0..6] = ordered min x,y,z | max x,y,z | non-finite count
__global__ void __launch_bounds__(256) dtu_bounds_kernel(int64_t N, const double* __restrict__ p, unsigned long long* __restrict__ bits) {
	double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
	unsigned long long bad = 0;
	for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x) {
		const double x = p[3 * i], y = p[3 * i + 1], z = p[3 * i + 2];
		if (!finite3d(x, y, z)) { bad++; continue; }
		lo[0] = fmin(lo[0], x); lo[1] = fmin(lo[1], y); lo[2] = fmin(lo[2], z);
		hi[0] = fmax(hi[0], x); hi[1] = fmax(hi[1], y); hi[2] = fmax(hi[2], z);
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
		for (int k = 0; k < 3; k++) {
			lo[k] = fmin(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o));
			hi[k] = fmax(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o));
		}
		bad += __shfl_xor_sync(0xffffffffu, bad, o);
	}
	if ((threadIdx.x & 31) == 0) {
#pragma unroll
		for (int k = 0; k < 3; k++) {
			if (lo[k] <= hi[k]) {
				atomicMin(bits + k, d2ord(lo[k]));
				atomicMax(bits + 3 + k, d2ord(hi[k]));
			}
		}
		if (bad) atomicAdd(bits + 6, bad);
	}
}

struct Bounds {
	double lo[3], hi[3];
	unsigned long long nonfinite;
};

// nsets consecutive groups of 8 words: min words start at the largest ordered value, max words and the count at zero
cudaError_t reset_bounds(unsigned long long* bits, int nsets, cudaStream_t s) {
	for (int k = 0; k < nsets; k++) {
		cudaError_t e = cudaMemsetAsync(bits + 8 * k, 0xff, 3 * sizeof(unsigned long long), s);
		if (e == cudaSuccess) e = cudaMemsetAsync(bits + 8 * k + 3, 0, 5 * sizeof(unsigned long long), s);
		if (e != cudaSuccess) return e;
	}
	return cudaSuccess;
}

cudaError_t fetch_bounds(unsigned long long* bits, Bounds* out, int nsets, cudaStream_t s) {
	unsigned long long h[16];
	cudaError_t e = cudaMemcpyAsync(h, bits, 8 * nsets * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s);
	if (e == cudaSuccess) e = cudaStreamSynchronize(s);
	if (e != cudaSuccess) return e;
	for (int k = 0; k < nsets; k++) {
		for (int a = 0; a < 3; a++) {
			out[k].lo[a] = ord2d(h[8 * k + a]);
			out[k].hi[a] = ord2d(h[8 * k + 3 + a]);
		}
		out[k].nonfinite = h[8 * k + 6];
	}
	return cudaSuccess;
}

void launch_bounds(int64_t N, const double* p, unsigned long long* bits, cudaStream_t s) {
	if (N <= 0) return;
	const int blocks = (int)std::min<int64_t>((N + 255) / 256, 4 * sm_count());
	dtu_bounds_kernel<<<blocks, 256, 0, s>>>(N, p, bits);
	count_launch();
}

// ---- surface sampling (eval.py:54-71) ---------------------------------------------------------------------------------

struct Tri {
	double v0[3], e1[3], e2[3];
	double n1, n2, m1, m2;   // rows n1 + 1, columns n2 + 1; c = (k + 0.5) / m
	bool sampled;            // area2 > 0 and all three indices in range
	bool bad;                // an index out of range, or n1 / n2 not finite
};

__device__ Tri tri_setup(int64_t V, const double* __restrict__ verts, const int32_t* __restrict__ faces, int64_t t, double density) {
	Tri T;
	T.sampled = false;
	T.bad = false;
	T.n1 = T.n2 = 0.0;
	T.m1 = T.m2 = 1e-7;
	const int32_t a = faces[3 * t], b = faces[3 * t + 1], c = faces[3 * t + 2];
	if (a < 0 || b < 0 || c < 0 || a >= V || b >= V || c >= V) {
		T.bad = true;
		return T;
	}
	for (int k = 0; k < 3; k++) {
		T.v0[k] = verts[3 * (int64_t)a + k];
		T.e1[k] = dsub(verts[3 * (int64_t)b + k], T.v0[k]);
		T.e2[k] = dsub(verts[3 * (int64_t)c + k], T.v0[k]);
	}
	const double l1 = dnorm3(T.e1[0], T.e1[1], T.e1[2]), l2 = dnorm3(T.e2[0], T.e2[1], T.e2[2]);
	// np.cross: each component one product minus another, rounded separately
	const double cx = dsub(__dmul_rn(T.e1[1], T.e2[2]), __dmul_rn(T.e1[2], T.e2[1]));
	const double cy = dsub(__dmul_rn(T.e1[2], T.e2[0]), __dmul_rn(T.e1[0], T.e2[2]));
	const double cz = dsub(__dmul_rn(T.e1[0], T.e2[1]), __dmul_rn(T.e1[1], T.e2[0]));
	const double area2 = dnorm3(cx, cy, cz);
	if (!(area2 > 0.0)) return T;   // zero or NaN area: dropped
	const double thr = __dmul_rn(density, __dsqrt_rn(__ddiv_rn(__dmul_rn(l1, l2), area2)));
	T.n1 = floor(__ddiv_rn(l1, thr));
	T.n2 = floor(__ddiv_rn(l2, thr));
	T.m1 = fmax(T.n1, 1e-7);
	T.m2 = fmax(T.n2, 1e-7);
	T.sampled = true;
	T.bad = !(isfinite(T.n1) && isfinite(T.n2));
	return T;
}

__device__ __forceinline__ double coef(double k, double m) { return __ddiv_rn(__dadd_rn(k, 0.5), m); }
__device__ __forceinline__ bool inside(double c0, double c1) { return __dadd_rn(c0, c1) < 1.0; }

// Rows i = 0, 1, ... of the triangle; row i holds columns j < cols(i), where cols is non-increasing because c0 grows with
// i and rounding is monotone.  visit(i, prefix, cols) is called for every non-empty row.  Returns the point count, or
// SAMPLE_SATURATED once it exceeds 2^31 - 1.
template <typename Visit>
__device__ int64_t walk_rows(const Tri& T, int64_t& rows, Visit visit) {
	rows = 0;
	if (!T.sampled || T.n1 == 0.0 || T.n2 == 0.0) return 0;   // c = 0.5 / 1e-7 on an empty side: nothing passes c0 + c1 < 1
	if (T.n1 > WALK_LIMIT || T.n2 > WALK_LIMIT) return SAMPLE_SATURATED;  // > 2^31 rows (or columns of row 0) with >= 1 point
	int64_t j = (int64_t)T.n2 + 1, pts = 0;
	for (int64_t i = 0; i <= (int64_t)T.n1; i++) {
		const double c0 = coef((double)i, T.m1);
		while (j > 0 && !inside(c0, coef((double)(j - 1), T.m2))) j--;
		if (j == 0) break;
		visit(rows, i, pts);
		rows++;
		pts += j;
		if (pts > INT32_MAX) return SAMPLE_SATURATED;
	}
	return pts;
}

// counts [F + 1] points and rows per triangle (the trailing entry 0, so the exclusive scan's last entry is the total)
__global__ void __launch_bounds__(128) sample_count_kernel(int64_t V, const double* __restrict__ verts, int64_t F, const int32_t* __restrict__ faces,
                                                           double density, int64_t* __restrict__ pts, int64_t* __restrict__ rows) {
	const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
	if (t > F) return;
	if (t == F) {
		pts[t] = 0;
		rows[t] = 0;
		return;
	}
	const Tri T = tri_setup(V, verts, faces, t, density);
	int64_t r = 0, n = SAMPLE_SATURATED;
	if (!T.bad) n = walk_rows(T, r, [](int64_t, int64_t, int64_t) {});
	pts[t] = n;
	rows[t] = n == SAMPLE_SATURATED ? 0 : r;
}

__global__ void __launch_bounds__(128) sample_rows_kernel(int64_t V, const double* __restrict__ verts, int64_t F, const int32_t* __restrict__ faces,
                                                          double density, const int64_t* __restrict__ pts_off, const int64_t* __restrict__ rows_off,
                                                          int64_t* __restrict__ row_first, int32_t* __restrict__ row_tri, int32_t* __restrict__ row_i) {
	const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
	if (t >= F) return;
	const Tri T = tri_setup(V, verts, faces, t, density);
	const int64_t p0 = pts_off[t], r0 = rows_off[t];
	int64_t r = 0;
	walk_rows(T, r, [&](int64_t row, int64_t i, int64_t prefix) {
		row_first[r0 + row] = p0 + prefix;
		row_tri[r0 + row] = (int32_t)t;
		row_i[r0 + row] = (int32_t)i;
	});
}

// one thread per sample: q = (e1 * c0 + e2 * c1) + v0, written after the V vertices
__global__ void __launch_bounds__(128) sample_emit_kernel(int64_t V, const double* __restrict__ verts, const int32_t* __restrict__ faces, double density,
                                                          int64_t S, int64_t R, const int64_t* __restrict__ row_first, const int32_t* __restrict__ row_tri,
                                                          const int32_t* __restrict__ row_i, double* __restrict__ out) {
	const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
	if (s >= S) return;
	int64_t lo = 0, hi = R - 1;   // last row with row_first <= s
	while (lo < hi) {
		const int64_t mid = (lo + hi + 1) >> 1;
		if (row_first[mid] <= s) lo = mid;
		else hi = mid - 1;
	}
	const Tri T = tri_setup(V, verts, faces, row_tri[lo], density);
	const double c0 = coef((double)row_i[lo], T.m1), c1 = coef((double)(s - row_first[lo]), T.m2);
	double* o = out + 3 * (V + s);
#pragma unroll
	for (int k = 0; k < 3; k++) o[k] = __dadd_rn(__dadd_rn(__dmul_rn(T.e1[k], c0), __dmul_rn(T.e2[k], c1)), T.v0[k]);
}

// ---- radius downsample (eval.py:80-94) --------------------------------------------------------------------------------

constexpr uint8_t UNDECIDED = 0, KEPT = 1, REMOVED = 2;
constexpr int CELL_BITS = 21;
constexpr double CELL_MAX = (double)((1 << CELL_BITS) - 2);

struct Grid {
	double lo[3];
	double h;
};

__device__ __forceinline__ uint64_t cell_of(double x, double lo, double h) {
	const double t = floor(__ddiv_rn(dsub(x, lo), h));
	return t <= 0.0 ? 0ull : (t >= CELL_MAX + 1.0 ? (uint64_t)(CELL_MAX + 1.0) : (uint64_t)t);
}

__global__ void __launch_bounds__(256) ds_key_kernel(int N, const double* __restrict__ p, Grid g, uint64_t* __restrict__ keys, int32_t* __restrict__ ids) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= N) return;
	keys[i] = cell_of(p[3 * (int64_t)i], g.lo[0], g.h) << 42 | cell_of(p[3 * (int64_t)i + 1], g.lo[1], g.h) << 21 | cell_of(p[3 * (int64_t)i + 2], g.lo[2], g.h);
	ids[i] = i;
}

// sorted points packed, cell heads flagged
__global__ void __launch_bounds__(256) ds_pack_kernel(int N, const double* __restrict__ p, const uint64_t* __restrict__ keys, const int32_t* __restrict__ ids,
                                                      double4* __restrict__ packed, int32_t* __restrict__ head) {
	const int j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= N) return;
	const int64_t i = ids[j];
	packed[j] = make_double4(p[3 * i], p[3 * i + 1], p[3 * i + 2], 0.0);
	head[j] = (j == 0 || keys[j] != keys[j - 1]) ? 1 : 0;
}

// cell index of every sorted point (inclusive scan of the head flags minus 1); heads record the cell's key and start
__global__ void __launch_bounds__(256) ds_cells_kernel(int N, const uint64_t* __restrict__ keys, const int32_t* __restrict__ head, const int32_t* __restrict__ cell_incl,
                                                       int32_t* __restrict__ cell_of_pt, uint64_t* __restrict__ cell_key, int32_t* __restrict__ cell_start,
                                                       int32_t* __restrict__ num_cells) {
	const int j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= N) return;
	const int c = cell_incl[j] - 1;
	cell_of_pt[j] = c;
	if (head[j]) {
		cell_key[c] = keys[j];
		cell_start[c] = j;
	}
	if (j == N - 1) {
		cell_start[c + 1] = N;
		*num_cells = c + 1;
	}
}

// 27 neighbour cells of every occupied cell (-1: empty), by binary search over the sorted cell keys
__global__ void __launch_bounds__(256) ds_neighbours_kernel(const int32_t* __restrict__ num_cells, const uint64_t* __restrict__ cell_key, int32_t* __restrict__ nbr) {
	const int c = blockIdx.x * blockDim.x + threadIdx.x;
	const int C = *num_cells;
	if (c >= C) return;
	const uint64_t k = cell_key[c];
	const int64_t cx = (int64_t)(k >> 42), cy = (int64_t)(k >> 21 & 0x1fffff), cz = (int64_t)(k & 0x1fffff);
	int slot = 0;
	for (int dx = -1; dx <= 1; dx++)
		for (int dy = -1; dy <= 1; dy++)
			for (int dz = -1; dz <= 1; dz++, slot++) {
				const int64_t x = cx + dx, y = cy + dy, z = cz + dz;
				int found = -1;
				if (x >= 0 && y >= 0 && z >= 0 && x < (1 << CELL_BITS) && y < (1 << CELL_BITS) && z < (1 << CELL_BITS)) {
					const uint64_t want = (uint64_t)x << 42 | (uint64_t)y << 21 | (uint64_t)z;
					int lo = 0, hi = C;
					while (lo < hi) {
						const int mid = (lo + hi) >> 1;
						if (cell_key[mid] < want) lo = mid + 1;
						else hi = mid;
					}
					if (lo < C && cell_key[lo] == want) found = lo;
				}
				nbr[27 * (int64_t)c + slot] = found;
			}
}

__global__ void __launch_bounds__(256) ds_iota_kernel(int N, int32_t* __restrict__ list, uint8_t* __restrict__ state) {
	const int j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= N) return;
	list[j] = j;
	state[j] = UNDECIDED;
}

// One round.  Every listed (undecided) point scans its lower-ranked neighbours (d^2 <= r*r) cell by cell in rank order and
// stops at the first that is kept (-> removed) or still undecided (-> stays undecided); with none, it is kept.  States
// only ever go from undecided to final, and a final state is the greedy result, so reading a neighbour's state before or
// after another thread of this round wrote it gives a correct decision either way.
__global__ void __launch_bounds__(256) ds_round_kernel(int n, const int32_t* __restrict__ list, const double4* __restrict__ packed,
                                                       const int32_t* __restrict__ rank, const int32_t* __restrict__ cell_of_pt,
                                                       const int32_t* __restrict__ cell_start, const int32_t* __restrict__ nbr, double r2,
                                                       volatile uint8_t* state, int32_t* __restrict__ next, int32_t* __restrict__ next_count) {
	const int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= n) return;
	const int j = list[t];
	const double4 q = packed[j];
	const int rj = rank[j];
	const int c = cell_of_pt[j];
	uint8_t verdict = KEPT;
	for (int s = 0; s < 27 && verdict == KEPT; s++) {
		const int nc = nbr[27 * (int64_t)c + s];
		if (nc < 0) continue;
		const int e = cell_start[nc + 1];
		for (int k = cell_start[nc]; k < e; k++) {
			if (rank[k] >= rj) break;   // cells are sorted by rank: the rest rank higher
			const uint8_t st = state[k];
			if (st == REMOVED) continue;
			const double4 p = packed[k];
			if (ddist2(q.x, q.y, q.z, p.x, p.y, p.z) <= r2) {
				verdict = st == KEPT ? REMOVED : UNDECIDED;
				break;
			}
		}
	}
	if (verdict == UNDECIDED) {
		next[atomicAdd(next_count, 1)] = j;
	} else {
		state[j] = verdict;
	}
}

__global__ void __launch_bounds__(256) ds_scatter_kernel(int N, const int32_t* __restrict__ rank, const uint8_t* __restrict__ state, uint8_t* __restrict__ kept) {
	const int j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= N) return;
	kept[rank[j]] = state[j] == KEPT ? 1 : 0;
}

// ---- exact 1-NN, one set against another (eval.py:118-134) -----------------------------------------------------------

constexpr int NN_LEAF = 32;
constexpr int NN_WARPS = 4;

__device__ __forceinline__ uint64_t spread21(uint64_t v) {
	v &= 0x1fffffull;
	v = (v | (v << 32)) & 0x1f00000000ffffull;
	v = (v | (v << 16)) & 0x1f0000ff0000ffull;
	v = (v | (v << 8)) & 0x100f00f00f00f00full;
	v = (v | (v << 4)) & 0x10c30c30c30c30c3ull;
	v = (v | (v << 2)) & 0x1249249249249249ull;
	return v;
}

__device__ __forceinline__ uint64_t cell21(double x, double lo, double hi) {
	const double ext = hi - lo;
	if (!(ext > 0.0)) return 0;
	const double t = (x - lo) / ext * 2097152.0;
	return t >= 2097151.0 ? 2097151ull : (t > 0.0 ? (uint64_t)t : 0ull);
}

__global__ void __launch_bounds__(256) nn_morton_kernel(int N, const double* __restrict__ p, const unsigned long long* __restrict__ bits, uint64_t* __restrict__ keys,
                                                        int32_t* __restrict__ ids) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= N) return;
	const double x = p[3 * (int64_t)i], y = p[3 * (int64_t)i + 1], z = p[3 * (int64_t)i + 2];
	keys[i] = (spread21(cell21(x, ord2d(bits[0]), ord2d(bits[3]))) << 2) | (spread21(cell21(y, ord2d(bits[1]), ord2d(bits[4]))) << 1) |
	          spread21(cell21(z, ord2d(bits[2]), ord2d(bits[5])));
	ids[i] = i;
}

__global__ void __launch_bounds__(256) nn_leaf_kernel(int M, int L, int Lp, const double* __restrict__ p, const int32_t* __restrict__ order, double4* __restrict__ packed,
                                                      double4* __restrict__ node_lo, double4* __restrict__ node_hi) {
	const int leaf = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int lane = threadIdx.x & 31;
	if (leaf >= Lp) return;
	const int j = leaf * NN_LEAF + lane;
	double4 lo = make_double4(INFINITY, INFINITY, INFINITY, 0.0), hi = make_double4(-INFINITY, -INFINITY, -INFINITY, 0.0);
	if (leaf < L && j < M) {
		const int64_t i = order[j];
		const double4 q = make_double4(p[3 * i], p[3 * i + 1], p[3 * i + 2], 0.0);
		packed[j] = q;
		lo = q;
		hi = q;
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
		lo.x = fmin(lo.x, __shfl_xor_sync(0xffffffffu, lo.x, o));
		lo.y = fmin(lo.y, __shfl_xor_sync(0xffffffffu, lo.y, o));
		lo.z = fmin(lo.z, __shfl_xor_sync(0xffffffffu, lo.z, o));
		hi.x = fmax(hi.x, __shfl_xor_sync(0xffffffffu, hi.x, o));
		hi.y = fmax(hi.y, __shfl_xor_sync(0xffffffffu, hi.y, o));
		hi.z = fmax(hi.z, __shfl_xor_sync(0xffffffffu, hi.z, o));
	}
	if (lane == 0) {
		node_lo[Lp + leaf] = lo;
		node_hi[Lp + leaf] = hi;
	}
}

__global__ void __launch_bounds__(256) nn_level_kernel(int first, double4* __restrict__ node_lo, double4* __restrict__ node_hi) {
	const int n = first + blockIdx.x * blockDim.x + threadIdx.x;
	if (n >= 2 * first) return;
	const double4 a = node_lo[2 * n], b = node_lo[2 * n + 1], c = node_hi[2 * n], d = node_hi[2 * n + 1];
	node_lo[n] = make_double4(fmin(a.x, b.x), fmin(a.y, b.y), fmin(a.z, b.z), 0.0);
	node_hi[n] = make_double4(fmax(c.x, d.x), fmax(c.y, d.y), fmax(c.z, d.z), 0.0);
}

// Squared distance from q to the box [lo, hi], a lower bound of ddist2 in fp64 rounding: per axis the gap
// max(lo - q, q - hi, 0) is at most |p - q| for every p in the box, and the same rounded expression shape as ddist2 is
// monotone in each gap.  An empty box (lo = +inf, hi = -inf) is at +inf.
__device__ __forceinline__ double box_dist2(double4 q, double4 lo, double4 hi) {
	const double gx = fmax(fmax(dsub(lo.x, q.x), dsub(q.x, hi.x)), 0.0);
	const double gy = fmax(fmax(dsub(lo.y, q.y), dsub(q.y, hi.y)), 0.0);
	const double gz = fmax(fmax(dsub(lo.z, q.z), dsub(q.z, hi.z)), 0.0);
	return __dadd_rn(__dadd_rn(__dmul_rn(gx, gx), __dmul_rn(gy, gy)), __dmul_rn(gz, gz));
}

__device__ __forceinline__ bool warp_needs(bool active, double4 q, double best, const double4* __restrict__ node_lo, const double4* __restrict__ node_hi, int n,
                                           double& dist) {
	dist = active ? box_dist2(q, node_lo[n], node_hi[n]) : INFINITY;
	return __any_sync(0xffffffffu, active && dist < best);
}

__global__ void __launch_bounds__(NN_WARPS * 32) nn_query_kernel(int N, const double* __restrict__ query, const int32_t* __restrict__ qorder, int M, int Lp,
                                                                 const double4* __restrict__ packed, const int32_t* __restrict__ order,
                                                                 const double4* __restrict__ node_lo, const double4* __restrict__ node_hi,
                                                                 double* __restrict__ dist, int64_t* __restrict__ index) {
	const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int lane = threadIdx.x & 31;
	if (w * 32 >= N) return;   // warp-uniform
	const int j = w * 32 + lane;
	const bool active = j < N;
	const int64_t qi = active ? qorder[j] : 0;
	const double4 q = active ? make_double4(query[3 * qi], query[3 * qi + 1], query[3 * qi + 2], 0.0) : make_double4(0.0, 0.0, 0.0, 0.0);
	double best = INFINITY;
	int besti = -1;
	// Pruning: a node is entered when some lane's box distance is below its best so far.  box_dist2 is a lower bound in fp64,
	// so a skipped box holds no strictly nearer point; ties are skipped (which nearest point is reported is unspecified).
	int stack = 0, sp = 0, node = 1;
	double dn;
	bool have = warp_needs(active, q, best, node_lo, node_hi, node, dn);
	while (true) {
		if (have) {
			if (node >= Lp) {
				const int l = node - Lp;
				const int k0 = l * NN_LEAF + lane;
				const double4 p = k0 < M ? packed[k0] : make_double4(INFINITY, INFINITY, INFINITY, 0.0);
				const int pid = k0 < M ? order[k0] : -1;
#pragma unroll 4
				for (int k = 0; k < NN_LEAF; k++) {
					const double x = __shfl_sync(0xffffffffu, p.x, k), y = __shfl_sync(0xffffffffu, p.y, k), z = __shfl_sync(0xffffffffu, p.z, k);
					const int id = __shfl_sync(0xffffffffu, pid, k);
					const double d = ddist2(q.x, q.y, q.z, x, y, z);
					if (active && d < best) {
						best = d;
						besti = id;
					}
				}
				have = false;
			} else {
				double d0, d1;
				const bool n0 = warp_needs(active, q, best, node_lo, node_hi, 2 * node, d0);
				const bool n1 = warp_needs(active, q, best, node_lo, node_hi, 2 * node + 1, d1);
				if (n0 && n1) {
					double m0 = active ? d0 : INFINITY, m1 = active ? d1 : INFINITY;
#pragma unroll
					for (int o = 16; o > 0; o >>= 1) {
						m0 = fmin(m0, __shfl_xor_sync(0xffffffffu, m0, o));
						m1 = fmin(m1, __shfl_xor_sync(0xffffffffu, m1, o));
					}
					const int nearer = m1 < m0 ? 2 * node + 1 : 2 * node;
					if (lane == sp) stack = nearer ^ 1;
					sp++;
					node = nearer;
				} else if (n0 || n1) {
					node = n0 ? 2 * node : 2 * node + 1;
				} else {
					have = false;
				}
			}
		}
		if (!have) {
			if (sp == 0) break;
			sp--;
			node = __shfl_sync(0xffffffffu, stack, sp);
			have = warp_needs(active, q, best, node_lo, node_hi, node, dn);
		}
	}
	if (!active) return;
	dist[qi] = __dsqrt_rn(best);
	index[qi] = besti;
}

// ---- mask culling (evaluate_dtu_mesh.py:82-138) -----------------------------------------------------------------------

constexpr int DISK_R = 6;

// skimage binary_dilation(mask, disk(6)): any set pixel at x^2 + y^2 <= 36; pixels outside the image are unset
__global__ void __launch_bounds__(256) dilate_kernel(int n_views, int H, int W, const uint8_t* __restrict__ in, uint8_t* __restrict__ out) {
	const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
	const int64_t HW = (int64_t)H * W;
	if (i >= n_views * HW) return;
	const int64_t v = i / HW;
	const int y = (int)((i - v * HW) / W), x = (int)(i - v * HW - (int64_t)y * W);
	const uint8_t* m = in + v * HW;
	uint8_t hit = 0;
	for (int dy = -DISK_R; dy <= DISK_R && !hit; dy++) {
		const int yy = y + dy;
		if (yy < 0 || yy >= H) continue;
		for (int dx = -DISK_R; dx <= DISK_R; dx++) {
			const int xx = x + dx;
			if (dx * dx + dy * dy > DISK_R * DISK_R || xx < 0 || xx >= W) continue;
			if (m[(int64_t)yy * W + xx]) {
				hit = 1;
				break;
			}
		}
	}
	out[i] = hit;
}

__global__ void __launch_bounds__(256) cull_kernel(int64_t V, const double* __restrict__ verts, int n_views, int H, int W, const double* __restrict__ proj,
                                                   const uint8_t* __restrict__ masks, uint8_t* __restrict__ keep) {
	const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
	if (i >= V) return;
	const double x = verts[3 * i], y = verts[3 * i + 1], z = verts[3 * i + 2];
	const double w1 = (double)(W - 1), h1 = (double)(H - 1);
	uint8_t ok = 1;
	for (int v = 0; v < n_views && ok; v++) {
		const double* M = proj + 12 * v;
		double c[3];
#pragma unroll
		for (int r = 0; r < 3; r++)
			c[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(M[4 * r], x), __dmul_rn(M[4 * r + 1], y)), __dmul_rn(M[4 * r + 2], z)), M[4 * r + 3]);
		const double zz = __dadd_rn(c[2], 1e-6);
		const double px = __dmul_rn(dsub(__ddiv_rn(__ddiv_rn(c[0], zz), w1), 0.5), 2.0);
		const double py = __dmul_rn(dsub(__ddiv_rn(__ddiv_rn(c[1], zz), h1), 0.5), 2.0);
		if (!(px > -1.0 && px < 1.0 && py > -1.0 && py < 1.0)) continue;   // outside the view: passes it
		// grid_sample(mode='nearest', align_corners=True): ((g + 1) / 2) * (size - 1), rounded half to even
		const int xi = (int)rint(__dmul_rn(__ddiv_rn(__dadd_rn(px, 1.0), 2.0), w1));
		const int yi = (int)rint(__dmul_rn(__ddiv_rn(__dadd_rn(py, 1.0), 2.0), h1));
		ok = masks[((int64_t)v * H + yi) * W + xi];
	}
	keep[i] = ok;
}

// ---- sampling ----

struct SampleScratch {
	int64_t *pts, *rows, *pts_off, *rows_off;
	char* temp;
	size_t temp_bytes;
};

static SampleScratch carve_sample(char* base, int64_t F, size_t* total) {
	size_t temp = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, temp, (const int64_t*)nullptr, (int64_t*)nullptr, (int)(F + 1));
	Carver c(base);
	SampleScratch s;
	s.pts = c.take<int64_t>(F + 1);
	s.rows = c.take<int64_t>(F + 1);
	s.pts_off = c.take<int64_t>(F + 1);
	s.rows_off = c.take<int64_t>(F + 1);
	s.temp = c.take<char>(temp);
	s.temp_bytes = temp;
	if (total) *total = c.size();
	return s;
}

size_t dtu_sample_scratch_bytes(int64_t F) {
	size_t t = 0;
	carve_sample(nullptr, F, &t);
	return t;
}

cudaError_t launch_dtu_sample_count(int64_t V, const double* verts, int64_t F, const int32_t* faces, double density, char* scratch, int64_t* totals_host,
                                    cudaStream_t s) {
	SampleScratch k = carve_sample(scratch, F, nullptr);
	sample_count_kernel<<<(unsigned)((F + 1 + 127) / 128), 128, 0, s>>>(V, verts, F, faces, density, k.pts, k.rows);
	count_launch();
	size_t temp = k.temp_bytes;
	RGS_TRY(cub::DeviceScan::ExclusiveSum(k.temp, temp, k.pts, k.pts_off, (int)(F + 1), s));
	temp = k.temp_bytes;
	RGS_TRY(cub::DeviceScan::ExclusiveSum(k.temp, temp, k.rows, k.rows_off, (int)(F + 1), s));
	count_launch(2);
	RGS_TRY(cudaMemcpyAsync(totals_host, k.pts_off + F, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaMemcpyAsync(totals_host + 1, k.rows_off + F, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaStreamSynchronize(s));
	return cudaGetLastError();
}

size_t dtu_sample_rows_bytes(int64_t R) {
	Carver c(nullptr);
	c.take<int64_t>(R);
	c.take<int32_t>(R);
	c.take<int32_t>(R);
	return c.size();
}

cudaError_t launch_dtu_sample_emit(int64_t V, const double* verts, int64_t F, const int32_t* faces, double density, char* scratch, int64_t S, int64_t R,
                                   char* rows_scratch, double* out, cudaStream_t s) {
	SampleScratch k = carve_sample(scratch, F, nullptr);
	if (V > 0) RGS_TRY(cudaMemcpyAsync(out, verts, (size_t)V * 3 * sizeof(double), cudaMemcpyDeviceToDevice, s));
	if (S == 0) return cudaGetLastError();
	Carver c(rows_scratch);
	int64_t* row_first = c.take<int64_t>(R);
	int32_t* row_tri = c.take<int32_t>(R);
	int32_t* row_i = c.take<int32_t>(R);
	sample_rows_kernel<<<(unsigned)((F + 127) / 128), 128, 0, s>>>(V, verts, F, faces, density, k.pts_off, k.rows_off, row_first, row_tri, row_i);
	sample_emit_kernel<<<(unsigned)((S + 127) / 128), 128, 0, s>>>(V, verts, faces, density, S, R, row_first, row_tri, row_i, out);
	count_launch(2);
	return cudaGetLastError();
}

// ---- downsample ----

struct DsScratch {
	unsigned long long* bits;
	uint64_t *keys_in, *keys_out, *cell_key;
	int32_t *ids_in, *ids_out, *head, *cell_incl, *cell_of_pt, *cell_start, *nbr, *list_a, *list_b, *counters;
	double4* packed;
	uint8_t* state;
	char* temp;
	size_t temp_bytes;
};

static DsScratch carve_ds(char* base, int N, size_t* total) {
	size_t sort_bytes = 0, scan_bytes = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr, N);
	cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (const int32_t*)nullptr, (int32_t*)nullptr, N);
	Carver c(base);
	DsScratch k;
	k.bits = c.take<unsigned long long>(8);
	k.keys_in = c.take<uint64_t>(N);
	k.keys_out = c.take<uint64_t>(N);
	k.cell_key = c.take<uint64_t>(N);
	k.ids_in = c.take<int32_t>(N);
	k.ids_out = c.take<int32_t>(N);
	k.head = c.take<int32_t>(N);
	k.cell_incl = c.take<int32_t>(N);
	k.cell_of_pt = c.take<int32_t>(N);
	k.cell_start = c.take<int32_t>((size_t)N + 1);
	k.nbr = c.take<int32_t>(27 * (size_t)N);
	k.list_a = c.take<int32_t>(N);
	k.list_b = c.take<int32_t>(N);
	k.counters = c.take<int32_t>(2);
	k.packed = c.take<double4>(N);
	k.state = c.take<uint8_t>(N);
	k.temp_bytes = std::max(sort_bytes, scan_bytes);
	k.temp = c.take<char>(k.temp_bytes);
	if (total) *total = c.size();
	return k;
}

size_t dtu_downsample_scratch_bytes(int N) {
	size_t t = 0;
	carve_ds(nullptr, N, &t);
	return t;
}

// returns cudaErrorInvalidValue when a point is not finite (checked on the host after the bounds pass)
cudaError_t launch_dtu_downsample(int N, const double* pts, double radius, uint8_t* kept, char* scratch, int32_t* rounds, cudaStream_t s) {
	DsScratch k = carve_ds(scratch, N, nullptr);
	RGS_TRY(reset_bounds(k.bits, 1, s));
	launch_bounds(N, pts, k.bits, s);
	Bounds b;
	RGS_TRY(fetch_bounds(k.bits, &b, 1, s));
	if (b.nonfinite) return cudaErrorInvalidValue;
	// cell edge slightly above r, so the 27-cell filter stays conservative under rounding; coarser when the cloud spans more
	// than 2^21 - 2 cells on an axis (larger cells only make the filter looser)
	Grid g;
	double ext = 0.0;
	for (int a = 0; a < 3; a++) {
		g.lo[a] = b.lo[a];
		ext = std::max(ext, b.hi[a] - b.lo[a]);
	}
	g.h = std::max(radius * (1.0 + 1.0 / 1048576.0), ext / CELL_MAX * (1.0 + 1.0 / 1048576.0));
	const unsigned blocks = (unsigned)((N + 255) / 256);
	ds_key_kernel<<<blocks, 256, 0, s>>>(N, pts, g, k.keys_in, k.ids_in);
	count_launch();
	size_t temp = k.temp_bytes;
	RGS_TRY(cub::DeviceRadixSort::SortPairs(k.temp, temp, k.keys_in, k.keys_out, k.ids_in, k.ids_out, N, 0, 63, s));
	ds_pack_kernel<<<blocks, 256, 0, s>>>(N, pts, k.keys_out, k.ids_out, k.packed, k.head);
	temp = k.temp_bytes;
	RGS_TRY(cub::DeviceScan::InclusiveSum(k.temp, temp, k.head, k.cell_incl, N, s));
	ds_cells_kernel<<<blocks, 256, 0, s>>>(N, k.keys_out, k.head, k.cell_incl, k.cell_of_pt, k.cell_key, k.cell_start, k.counters + 1);
	ds_neighbours_kernel<<<blocks, 256, 0, s>>>(k.counters + 1, k.cell_key, k.nbr);
	ds_iota_kernel<<<blocks, 256, 0, s>>>(N, k.list_a, k.state);
	count_launch(5);
	const double r2 = radius * radius;
	int n = N, r = 0;
	int32_t *cur = k.list_a, *nxt = k.list_b;
	while (n > 0) {
		RGS_TRY(cudaMemsetAsync(k.counters, 0, sizeof(int32_t), s));
		ds_round_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(n, cur, k.packed, k.ids_out, k.cell_of_pt, k.cell_start, k.nbr, r2, k.state, nxt,
		                                                            k.counters);
		count_launch();
		RGS_TRY(cudaMemcpyAsync(&n, k.counters, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
		RGS_TRY(cudaStreamSynchronize(s));
		std::swap(cur, nxt);
		r++;
	}
	ds_scatter_kernel<<<blocks, 256, 0, s>>>(N, k.ids_out, k.state, kept);
	count_launch();
	if (rounds) *rounds = r;
	return cudaGetLastError();
}

// ---- nearest ----

struct NnScratch {
	unsigned long long* bits;   // [16]: reference bounds, query bounds
	uint64_t *keys_in, *keys_out, *qkeys_in, *qkeys_out;
	int32_t *ids_in, *ids_out, *qids_in, *qids_out;
	double4 *packed, *node_lo, *node_hi;
	char* temp;
	size_t temp_bytes;
};

static NnScratch carve_nn(char* base, int M, int N, size_t* total) {
	const int Lp = pow2_at_least((M + NN_LEAF - 1) / NN_LEAF);
	size_t a = 0, b = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, a, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr, M);
	cub::DeviceRadixSort::SortPairs(nullptr, b, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr, N);
	Carver c(base);
	NnScratch k;
	k.bits = c.take<unsigned long long>(16);
	k.keys_in = c.take<uint64_t>(M);
	k.keys_out = c.take<uint64_t>(M);
	k.ids_in = c.take<int32_t>(M);
	k.ids_out = c.take<int32_t>(M);
	k.qkeys_in = c.take<uint64_t>(N);
	k.qkeys_out = c.take<uint64_t>(N);
	k.qids_in = c.take<int32_t>(N);
	k.qids_out = c.take<int32_t>(N);
	k.packed = c.take<double4>(M);
	k.node_lo = c.take<double4>(2 * (size_t)Lp);
	k.node_hi = c.take<double4>(2 * (size_t)Lp);
	k.temp_bytes = std::max(a, b);
	k.temp = c.take<char>(k.temp_bytes);
	if (total) *total = c.size();
	return k;
}

size_t dtu_nearest_scratch_bytes(int M, int N) {
	size_t t = 0;
	carve_nn(nullptr, M, N, &t);
	return t;
}

cudaError_t launch_dtu_nearest(int M, const double* ref, int N, const double* query, double* dist, int64_t* index, char* scratch, cudaStream_t s) {
	NnScratch k = carve_nn(scratch, M, N, nullptr);
	RGS_TRY(reset_bounds(k.bits, 2, s));
	launch_bounds(M, ref, k.bits, s);
	launch_bounds(N, query, k.bits + 8, s);
	Bounds b[2];
	RGS_TRY(fetch_bounds(k.bits, b, 2, s));
	if (b[0].nonfinite || b[1].nonfinite) return cudaErrorInvalidValue;

	nn_morton_kernel<<<(M + 255) / 256, 256, 0, s>>>(M, ref, k.bits, k.keys_in, k.ids_in);
	size_t temp = k.temp_bytes;
	RGS_TRY(cub::DeviceRadixSort::SortPairs(k.temp, temp, k.keys_in, k.keys_out, k.ids_in, k.ids_out, M, 0, 63, s));
	const int L = (M + NN_LEAF - 1) / NN_LEAF, Lp = pow2_at_least(L);
	nn_leaf_kernel<<<(Lp + 7) / 8, 256, 0, s>>>(M, L, Lp, ref, k.ids_out, k.packed, k.node_lo, k.node_hi);
	count_launch(3);
	for (int first = Lp / 2; first >= 1; first /= 2) {
		nn_level_kernel<<<(first + 255) / 256, 256, 0, s>>>(first, k.node_lo, k.node_hi);
		count_launch();
	}
	if (N == 0) return cudaGetLastError();
	nn_morton_kernel<<<(N + 255) / 256, 256, 0, s>>>(N, query, k.bits + 8, k.qkeys_in, k.qids_in);
	temp = k.temp_bytes;
	RGS_TRY(cub::DeviceRadixSort::SortPairs(k.temp, temp, k.qkeys_in, k.qkeys_out, k.qids_in, k.qids_out, N, 0, 63, s));
	const int warps = (N + 31) / 32;
	nn_query_kernel<<<(warps + NN_WARPS - 1) / NN_WARPS, NN_WARPS * 32, 0, s>>>(N, query, k.qids_out, M, Lp, k.packed, k.ids_out, k.node_lo, k.node_hi, dist,
	                                                                            index);
	count_launch(3);
	return cudaGetLastError();
}

}  // namespace
}  // namespace rgs

using namespace rgs;

extern "C" {

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
	const int64_t n = (int64_t)n_views * H * W;
	if (n == 0) return RGS_OK;
	dilate_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)cuda_stream>>>(n_views, H, W, masks, dilated);
	count_launch();
	return cuda_status(cudaGetLastError(), "dtu dilate", kNonFinitePoint);
}

int32_t rgs_dtu_cull_vertices(int64_t V, const double* vertices, int32_t n_views, int32_t H, int32_t W, const double* proj, const uint8_t* dilated,
                              uint8_t* keep, void* cuda_stream) {
	if (V < 0 || n_views < 0 || H <= 0 || W <= 0) return fail(RGS_E_INVALID, "dtu cull: negative count or empty image");
	if (V > 0 && (!vertices || !keep || (n_views > 0 && (!proj || !dilated)))) return fail(RGS_E_INVALID, "null pointer");
	if (V == 0) return RGS_OK;
	cull_kernel<<<(unsigned)((V + 255) / 256), 256, 0, (cudaStream_t)cuda_stream>>>(V, vertices, n_views, H, W, proj, dilated, keep);
	count_launch();
	return cuda_status(cudaGetLastError(), "dtu cull", kNonFinitePoint);
}

}  // extern "C"

// rgs_knn.cu -- mean squared distance to the 3 nearest other points (`simple_knn._C.distCUDA2`), the initial Gaussian
// scales of GaussianModel.create_from_pcd (reference scene/gaussian_model.py:315-316).  Runs once at initialisation.
//
// The result is exact under a fixed fp32 arithmetic (include/rgs_b200.h, rgs_knn_mean_dist2): every pair distance is
// (dx*dx + dy*dy) + dz*dz with each operation separately rounded, and the output is ((d0 + d1) + d2) / 3 over the three
// smallest values.  It is a function of the multiset of distances only, so traversal order and thread count do not
// change a bit.
//
// The clouds the reference feeds this (100 k uniform points, 1.2 M draws WITH replacement from mesh vertices, clustered
// COLMAP clouds with far outliers, up to 10 M points) defeat a uniform grid: a few cells take most of the points.  So:
//   1. bounding box of the finite points and their count (one host read: it sizes the tree);
//   2. 63-bit Morton codes over that box (non-finite points get ~0 and sort last), CUB radix sort of (code, index);
//   3. the sorted finite points packed as float4, cut into leaves of 32, one AABB per leaf;
//   4. an implicit balanced binary tree over the leaves in Morton order (heap numbering, leaves padded to a power of
//      two with empty boxes), built level by level with box unions;
//   5. one warp per leaf: the 32 lanes hold 32 spatially coherent queries, seed their top-3 from the other points of
//      the leaf, then traverse the tree TOGETHER, nearer child first, entering a node when any lane's box distance is
//      below that lane's third-best.  A visited leaf is loaded once (one point per lane) and broadcast with shuffles.
//      The traversal stack lives one entry per lane in a register (entry k in lane k), so it needs no local memory;
//      its depth is bounded by the tree height, at most 26 for P < 2^31.
//
// This file also holds the C-ABI entry points rgs_knn_mean_dist2 (include/rgs_b200.h).
#include <algorithm>

#include <cub/cub.cuh>

#include "rgs_common.cuh"

namespace rgs {

namespace {

constexpr int KNN_LEAF = 32;       // points per leaf = lanes per warp
constexpr int KNN_WARPS = 4;       // warps per query block
constexpr uint64_t KNN_NONFINITE_KEY = ~0ull;

__device__ __forceinline__ bool finite3(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }

// order-preserving float <-> uint32 map, so that atomicMin / atomicMax on the integers order the floats
__device__ __forceinline__ uint32_t f2ord(float f) {
	const uint32_t u = __float_as_uint(f);
	return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(uint32_t u) { return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u); }

// the contract's pair distance: (dx*dx + dy*dy) + dz*dz, every operation rounded on its own (no FMA contraction)
__device__ __forceinline__ float dist2(float4 a, float4 b) {
	const float dx = __fsub_rn(a.x, b.x), dy = __fsub_rn(a.y, b.y), dz = __fsub_rn(a.z, b.z);
	return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// Squared distance from q to the box [lo, hi].  Two properties make the search exact (see the pruning test in
// knn_query_kernel):
//  * it is a lower bound in fp32, not only in real arithmetic: the per-axis gap max(lo - q, q - hi, 0) is combined with
//    the same rounded expression shape as dist2.  For any point p in the box |p - q| >= gap on every axis, and
//    round-to-nearest subtraction, multiplication and addition are monotone, so the result never exceeds dist2(q, p).
//    A contracted (FMA) or reordered expression could exceed it in the last bit and prune a true neighbour.
//  * an empty box (lo = +inf, hi = -inf) is at +inf.
__device__ __forceinline__ float box_dist2(float4 q, float4 lo, float4 hi) {
	const float gx = fmaxf(fmaxf(__fsub_rn(lo.x, q.x), __fsub_rn(q.x, hi.x)), 0.0f);
	const float gy = fmaxf(fmaxf(__fsub_rn(lo.y, q.y), __fsub_rn(q.y, hi.y)), 0.0f);
	const float gz = fmaxf(fmaxf(__fsub_rn(lo.z, q.z), __fsub_rn(q.z, hi.z)), 0.0f);
	return __fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), __fmul_rn(gz, gz));
}

// keep the three smallest values b0 <= b1 <= b2; a value equal to b2 changes nothing, so it is not inserted
__device__ __forceinline__ void insert3(float d, float& b0, float& b1, float& b2) {
	if (d < b2) {
		if (d < b1) {
			b2 = b1;
			if (d < b0) { b1 = b0; b0 = d; } else { b1 = d; }
		} else {
			b2 = d;
		}
	}
}

// bits[0..6] = ordered min x,y,z | max x,y,z | finite count
__global__ void __launch_bounds__(256) knn_bounds_kernel(int P, const float* __restrict__ pts, uint32_t* __restrict__ bits) {
	float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
	uint32_t n = 0;
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) {
		const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
		if (!finite3(x, y, z)) continue;
		lo[0] = fminf(lo[0], x); lo[1] = fminf(lo[1], y); lo[2] = fminf(lo[2], z);
		hi[0] = fmaxf(hi[0], x); hi[1] = fmaxf(hi[1], y); hi[2] = fmaxf(hi[2], z);
		n++;
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
		for (int k = 0; k < 3; k++) {
			lo[k] = fminf(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o));
			hi[k] = fmaxf(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o));
		}
		n += __shfl_xor_sync(0xffffffffu, n, o);
	}
	if ((threadIdx.x & 31) == 0 && n > 0) {
#pragma unroll
		for (int k = 0; k < 3; k++) {
			atomicMin(bits + k, f2ord(lo[k]));
			atomicMax(bits + 3 + k, f2ord(hi[k]));
		}
		atomicAdd(bits + 6, n);
	}
}

// spread the low 21 bits of v to every third bit
__device__ __forceinline__ uint64_t spread21(uint64_t v) {
	v &= 0x1fffffull;
	v = (v | (v << 32)) & 0x1f00000000ffffull;
	v = (v | (v << 16)) & 0x1f0000ff0000ffull;
	v = (v | (v << 8)) & 0x100f00f00f00f00full;
	v = (v | (v << 4)) & 0x10c30c30c30c30c3ull;
	v = (v | (v << 2)) & 0x1249249249249249ull;
	return v;
}

// cell of x in [lo, hi] on a 2^21 grid, in double so that boxes spanning most of the float range still quantise
__device__ __forceinline__ uint64_t cell21(float x, float lo, float hi) {
	const double ext = (double)hi - (double)lo;
	if (!(ext > 0.0)) return 0;
	const double t = ((double)x - (double)lo) / ext * 2097152.0;
	return t >= 2097151.0 ? 2097151ull : (t > 0.0 ? (uint64_t)t : 0ull);
}

__global__ void __launch_bounds__(256) knn_morton_kernel(int P, const float* __restrict__ pts, const uint32_t* __restrict__ bits,
                                                         uint64_t* __restrict__ keys, uint32_t* __restrict__ ids) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
	uint64_t key = KNN_NONFINITE_KEY;
	if (finite3(x, y, z)) {
		const float lx = ord2f(bits[0]), ly = ord2f(bits[1]), lz = ord2f(bits[2]);
		const float hx = ord2f(bits[3]), hy = ord2f(bits[4]), hz = ord2f(bits[5]);
		key = (spread21(cell21(x, lx, hx)) << 2) | (spread21(cell21(y, ly, hy)) << 1) | spread21(cell21(z, lz, hz));  // < 2^63
	}
	keys[i] = key;
	ids[i] = (uint32_t)i;
}

// one warp per (padded) leaf: gather the leaf's sorted points into the packed array and write the leaf box
__global__ void __launch_bounds__(256) knn_leaf_kernel(int F, int L, int Lp, const float* __restrict__ pts, const uint32_t* __restrict__ order,
                                                       float4* __restrict__ packed, float4* __restrict__ node_lo, float4* __restrict__ node_hi) {
	const int leaf = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int lane = threadIdx.x & 31;
	if (leaf >= Lp) return;
	const int j = leaf * KNN_LEAF + lane;
	float4 lo = make_float4(INFINITY, INFINITY, INFINITY, 0.0f), hi = make_float4(-INFINITY, -INFINITY, -INFINITY, 0.0f);
	if (leaf < L && j < F) {
		const uint32_t i = order[j];
		const float4 p = make_float4(pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2], 0.0f);
		packed[j] = p;
		lo = p;
		hi = p;
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
		lo.x = fminf(lo.x, __shfl_xor_sync(0xffffffffu, lo.x, o));
		lo.y = fminf(lo.y, __shfl_xor_sync(0xffffffffu, lo.y, o));
		lo.z = fminf(lo.z, __shfl_xor_sync(0xffffffffu, lo.z, o));
		hi.x = fmaxf(hi.x, __shfl_xor_sync(0xffffffffu, hi.x, o));
		hi.y = fmaxf(hi.y, __shfl_xor_sync(0xffffffffu, hi.y, o));
		hi.z = fmaxf(hi.z, __shfl_xor_sync(0xffffffffu, hi.z, o));
	}
	if (lane == 0) {
		node_lo[Lp + leaf] = lo;
		node_hi[Lp + leaf] = hi;
	}
}

// internal nodes [first, 2*first): union of the two children
__global__ void __launch_bounds__(256) knn_level_kernel(int first, float4* __restrict__ node_lo, float4* __restrict__ node_hi) {
	const int n = first + blockIdx.x * blockDim.x + threadIdx.x;
	if (n >= 2 * first) return;
	const float4 a = node_lo[2 * n], b = node_lo[2 * n + 1], c = node_hi[2 * n], d = node_hi[2 * n + 1];
	node_lo[n] = make_float4(fminf(a.x, b.x), fminf(a.y, b.y), fminf(a.z, b.z), 0.0f);
	node_hi[n] = make_float4(fmaxf(c.x, d.x), fmaxf(c.y, d.y), fmaxf(c.z, d.z), 0.0f);
}

// any active lane whose box distance to node n is below its current third-best
__device__ __forceinline__ bool warp_needs(bool active, float4 q, float b2, const float4* __restrict__ node_lo, const float4* __restrict__ node_hi,
                                           int n, float& dist) {
	dist = active ? box_dist2(q, node_lo[n], node_hi[n]) : INFINITY;
	return __any_sync(0xffffffffu, active && dist < b2);
}

// Compare the query (lane) with the 32 points of leaf `leaf`, broadcast from the lane that loaded each one.  `self` is the
// lane whose point is the query itself (own leaf only; -1 elsewhere).
__device__ __forceinline__ void scan_leaf(int F, int leaf, int lane, int self, bool active, float4 q, const float4* __restrict__ packed, float& b0,
                                          float& b1, float& b2) {
	const int j = leaf * KNN_LEAF + lane;
	float4 p = j < F ? packed[j] : make_float4(INFINITY, INFINITY, INFINITY, 0.0f);  // padding: d = +inf, never inserted
#pragma unroll 8
	for (int k = 0; k < KNN_LEAF; k++) {
		float4 r;
		r.x = __shfl_sync(0xffffffffu, p.x, k);
		r.y = __shfl_sync(0xffffffffu, p.y, k);
		r.z = __shfl_sync(0xffffffffu, p.z, k);
		const float d = dist2(q, r);
		if (active && k != self) insert3(d, b0, b1, b2);
	}
}

__global__ void __launch_bounds__(KNN_WARPS * 32) knn_query_kernel(int P, int F, int Lp, const float4* __restrict__ packed, const uint32_t* __restrict__ order,
                                                                   const float4* __restrict__ node_lo, const float4* __restrict__ node_hi,
                                                                   float* __restrict__ out) {
	const int leaf = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int lane = threadIdx.x & 31;
	const int j = leaf * KNN_LEAF + lane;   // sorted position of this lane's query
	if (leaf * KNN_LEAF >= P) return;       // warp-uniform
	if (j >= F) {                           // non-finite points sort last: nobody's neighbour, NaN themselves
		if (j < P) out[order[j]] = __int_as_float(0x7fc00000);
		if (leaf * KNN_LEAF >= F) return;   // warp-uniform: no finite query in this warp
	}
	const bool active = j < F;
	const float4 q = active ? packed[j] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
	float b0 = INFINITY, b1 = INFINITY, b2 = INFINITY;
	scan_leaf(F, leaf, lane, lane, active, q, packed, b0, b1, b2);

	// Warp-cooperative depth-first traversal, nearer child first.  Stack entry k is held by lane k.
	//
	// Pruning: a node is skipped for a lane when its box distance is >= that lane's third-best (and the warp skips it
	// when that holds for every lane).  Two facts make this exact:
	//  * box_dist2 is a lower bound of dist2 in fp32 arithmetic, not only in real arithmetic (see box_dist2), so a
	//    pruned box cannot hold a point closer than the third-best;
	//  * ties are pruned (>=, not >): a point at exactly the third-best distance cannot lower any of the three values.
	//    Entering such boxes would make all-duplicate and lattice clouds, where almost every distance ties, visit
	//    every leaf -- a quadratic search (the reference's 1.2 M with-replacement cloud is exactly this case).
	// The query's own leaf was scanned above and is skipped here, so no point is counted twice.
	int stack = 0, sp = 0;
	float dn;
	int node = 1;
	bool have = warp_needs(active, q, b2, node_lo, node_hi, node, dn);
	while (true) {
		if (have) {
			if (node >= Lp) {
				const int l = node - Lp;
				if (l != leaf) scan_leaf(F, l, lane, -1, active, q, packed, b0, b1, b2);
				have = false;
			} else {
				float d0, d1;
				const bool n0 = warp_needs(active, q, b2, node_lo, node_hi, 2 * node, d0);
				const bool n1 = warp_needs(active, q, b2, node_lo, node_hi, 2 * node + 1, d1);
				if (n0 && n1) {
					float m0 = active ? d0 : INFINITY, m1 = active ? d1 : INFINITY;
#pragma unroll
					for (int o = 16; o > 0; o >>= 1) {
						m0 = fminf(m0, __shfl_xor_sync(0xffffffffu, m0, o));
						m1 = fminf(m1, __shfl_xor_sync(0xffffffffu, m1, o));
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
			have = warp_needs(active, q, b2, node_lo, node_hi, node, dn);  // the third-best may have dropped since the push
		}
	}
	if (!active) return;
	// ((d0 + d1) + d2) / 3; fewer than 4 finite points: the mean over the F - 1 others, and 1.0 for a lone point
	const int n = F - 1 < 3 ? F - 1 : 3;
	float r = 1.0f;
	if (n == 1) r = b0;
	else if (n == 2) r = __fdiv_rn(__fadd_rn(b0, b1), 2.0f);
	else if (n == 3) r = __fdiv_rn(__fadd_rn(__fadd_rn(b0, b1), b2), 3.0f);
	out[order[j]] = r;
}

int leaves_of(int F) { return (F + KNN_LEAF - 1) / KNN_LEAF; }
struct KnnScratch {
	uint32_t* bits;
	uint64_t *keys_in, *keys_out;
	uint32_t *ids_in, *ids_out;
	float4* packed;
	float4 *node_lo, *node_hi;
	char* sort_temp;
	size_t sort_temp_bytes;
};

// nodes are sized for P (an upper bound of the finite count, which is only known after the bounds pass)
KnnScratch carve_knn(char* base, int P, size_t* total) {
	const int Lp = pow2_at_least(leaves_of(P));
	size_t sort_bytes = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr, P);
	Carver c(base);
	KnnScratch k;
	k.bits = c.take<uint32_t>(8);
	k.keys_in = c.take<uint64_t>(P);
	k.keys_out = c.take<uint64_t>(P);
	k.ids_in = c.take<uint32_t>(P);
	k.ids_out = c.take<uint32_t>(P);
	k.packed = c.take<float4>(P);
	k.node_lo = c.take<float4>(2 * (size_t)Lp);
	k.node_hi = c.take<float4>(2 * (size_t)Lp);
	k.sort_temp = c.take<char>(sort_bytes);
	k.sort_temp_bytes = sort_bytes;
	if (total) *total = c.size();
	return k;
}

size_t knn_scratch_bytes(int P) {
	size_t total = 0;
	carve_knn(nullptr, P, &total);
	return total;
}

cudaError_t launch_knn_mean_dist2(int P, const float* points, float* out, char* scratch, cudaStream_t s) {
	KnnScratch k = carve_knn(scratch, P, nullptr);
	// bounds: min words start at the largest ordered value, max words and the count at zero
	RGS_TRY(cudaMemsetAsync(k.bits, 0xff, 3 * sizeof(uint32_t), s));
	RGS_TRY(cudaMemsetAsync(k.bits + 3, 0, 5 * sizeof(uint32_t), s));
	const int bounds_blocks = std::min((P + 255) / 256, 4 * sm_count());
	knn_bounds_kernel<<<bounds_blocks, 256, 0, s>>>(P, points, k.bits);
	count_launch();
	// the finite count sizes the tree: one blocking read
	uint32_t F = 0;
	RGS_TRY(cudaMemcpyAsync(&F, k.bits + 6, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaStreamSynchronize(s));

	knn_morton_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, points, k.bits, k.keys_in, k.ids_in);
	count_launch();
	size_t temp = k.sort_temp_bytes;
	RGS_TRY(cub::DeviceRadixSort::SortPairs(k.sort_temp, temp, k.keys_in, k.keys_out, k.ids_in, k.ids_out, P, 0, 64, s));
	count_launch();
	const int L = leaves_of((int)F), Lp = pow2_at_least(L > 0 ? L : 1);
	if (F > 0) {
		knn_leaf_kernel<<<(Lp + 7) / 8, 256, 0, s>>>((int)F, L, Lp, points, k.ids_out, k.packed, k.node_lo, k.node_hi);
		count_launch();
		for (int first = Lp / 2; first >= 1; first /= 2) {
			knn_level_kernel<<<(first + 255) / 256, 256, 0, s>>>(first, k.node_lo, k.node_hi);
			count_launch();
		}
	}
	const int warps = leaves_of(P);
	knn_query_kernel<<<(warps + KNN_WARPS - 1) / KNN_WARPS, KNN_WARPS * 32, 0, s>>>(P, (int)F, Lp, k.packed, k.ids_out, k.node_lo, k.node_hi, out);
	count_launch();
	return cudaGetLastError();
}

}  // namespace
}  // namespace rgs

using namespace rgs;

extern "C" {

int32_t rgs_knn_mean_dist2(int32_t P, const float* points, float* mean_dist2, rgs_resize_fn scratch, void* scratch_user, void* cuda_stream) {
	if (P < 0) return fail(RGS_E_INVALID, "negative point count");
	if (P == 0) return RGS_OK;
	if (!points || !mean_dist2 || !scratch) return fail(RGS_E_INVALID, "null pointer");
	char* buf;
	if (const int rc = grow(scratch, scratch_user, knn_scratch_bytes(P), buf, "knn scratch")) return rc;
	return cuda_status(launch_knn_mean_dist2(P, points, mean_dist2, buf, (cudaStream_t)cuda_stream), "knn");
}

}  // extern "C"

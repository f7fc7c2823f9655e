// rgs_delaunay.cu -- exact Delaunay tetrahedralization of fp32 points (contract at rgs_delaunay in include/rgs_b200.h).
//
// Predicates.  orient3d and insphere first run Shewchuk's stage-A floating-point filter on the fp64 values of the fp32
// inputs.  When it cannot decide, the determinant is expanded into its monomials over the raw coordinates and summed
// exactly: every fp32 value is m * 2^(E - 149) with an integer m < 2^24 and 0 <= E <= 253, so a degree-k monomial is an
// integer of at most 24k bits shifted by the sum of its E, and the sum of all monomials is an exact two's-complement
// fixed-point number in a few dozen 64-bit words (the common factor 2^(-149 k) does not change the sign).  This file is
// built with -fmad=false: a contracted a*b+c would break the filter's error bound.
//
// Ties of insphere are broken by the lifting perturbation of Devillers & Teillaud: the lifted coordinate of the point
// of lexicographic rank r gets eps^(2^-r)-style weight, so the sign of the first non-zero cofactor, taken over the five
// points from the largest (x, y, z) down, decides.
//
// Triangulation: parallel Bowyer-Watson in rounds over a mesh that starts as one ghost tetrahedron.  Per round every live
// cell holding uninserted points nominates the one of smallest (hash, index); each nominee collects its conflict region (cavity) by a
// breadth-first search from its located cell; it claims the cavity and the ring of cells just outside it with a 64-bit
// atomicMin of (hash priority, slot); a nominee holding every claim replaces its cavity by the star of its boundary faces;
// the points of the dead cells walk to the new cell that contains them.  The claimed ring keeps the winners' cavities
// apart, so each winner rewrites its neighbours' back-pointers alone.  The cavities larger than a round's slot go through
// the same claim protocol right after the round, in 16x larger slots; one still larger is inserted on its own, with the
// whole slab area as its capacity.
//
// This file also holds the C-ABI entry points rgs_delaunay and rgs_delaunay_predicates (include/rgs_b200.h).
#include <algorithm>
#include <cstring>
#include <cub/cub.cuh>

#include "rgs_common.cuh"

namespace rgs {
namespace {

constexpr int DT_BLOCK = 256;
constexpr uint64_t NO_NOMINEE = ~0ull;
constexpr uint64_t VISITED = ~1ull;   // a mark in nom[] for the single-cavity pass; point ids stay below 2^29

constexpr float DT_MAX_COORD = 0x1p90f;     // |coordinate| bound of rgs_delaunay's input
constexpr double DT_GHOST_SCALE = 0x1p30;   // D: ghost distance in units of the box's power-of-two extent
constexpr int DT_SLOT_CELLS = 64;           // per-nominee cavity capacity of a round ...
constexpr int DT_SLOT_FACES = 128;          // ... and its boundary-face capacity
constexpr int DT_MAX_SLOTS = 1 << 19;       // nominees per round

struct DtCounters {
	int bad;                 // points out of range or not finite
	uint32_t box[6];         // ordered-int bounding box (lo xyz, hi xyz)
	int cells;               // cells in use (dead ones included)
	int slots;               // nominees this round
	int full;                // a winner found no room to append: grow the mesh
	int overflowed;          // cavities larger than their slot in this pass
	int overflow_point;      // the smallest of their points
	int violation;           // a new cell was not positive, or a point found no cell: a predicate bug
	int inserted;            // points inserted so far
	int max_cavity;          // largest cavity inserted through a slot
	int out_cells;           // cells emitted
	uint32_t unique, spare;  // host side only: distinct points
};
struct DtPointsView {
	DtCounters* cnt;
	float4* verts;           // [n + 4] representatives in Morton order, then the ghosts
	uint32_t* rep;           // [n] original index of each vertex
	int32_t* loc;            // [n] located cell, -1 once inserted
	uint64_t* key64[2];
	uint32_t *key32[2], *ids[2], *first, *rank;   // first: after preparation, the round's overflowed points
	char* temp;
	size_t temp_bytes;
};
struct DtMesh {
	int4* tet;               // [cap] vertices, positive; -1 rows are dead
	int4* adj;               // [cap] neighbour across the face opposite vertex k: cell << 2 | face, -1 for none
	uint64_t* claim;         // [cap] (priority << 32 | slot) of the round
	uint64_t* nom;           // [cap] nominee of the round: (hash << 32 | point)
	int2* died;              // [cap] (pass, slot) that removed the cell
	int32_t* loc;            // the points' located cells (set by the launchers)
};
struct DtSlots {
	int *point, *cell, *k, *b, *base, *won;   // [K]
	int* cav;                // [K * DT_SLOT_CELLS] cavity cells
	int4* bnd;               // [K * DT_SLOT_FACES] the new cell of each boundary face
	int* bout;               // [K * DT_SLOT_FACES] the outside neighbour of each boundary face
};

// ---------------------------------------------------------------------------------------------------------------------
// exact predicates

struct Dec {                       // the three coordinates of a point as sign, integer mantissa, exponent (+149)
	uint32_t m[3];
	int e[3];
	uint32_t neg;                  // bit k: coordinate k is negative
};

__device__ __forceinline__ void decompose(float x, uint32_t& m, int& e, bool& neg) {
	const uint32_t u = __float_as_uint(x);
	neg = (u >> 31) != 0;
	const uint32_t eb = (u >> 23) & 0xffu, f = u & 0x7fffffu;
	m = eb ? (f | 0x800000u) : f;
	e = eb ? (int)eb - 1 : 0;
}

__device__ __forceinline__ Dec decompose(const float4& p) {
	Dec d;
	bool n0, n1, n2;
	decompose(p.x, d.m[0], d.e[0], n0);
	decompose(p.y, d.m[1], d.e[1], n1);
	decompose(p.z, d.m[2], d.e[2], n2);
	d.neg = (n0 ? 1u : 0u) | (n1 ? 2u : 0u) | (n2 ? 4u : 0u);
	return d;
}

// acc (W words, two's complement) += (neg ? -1 : 1) * M * 2^E
template <int W>
__device__ __forceinline__ void acc_add(uint64_t* acc, unsigned __int128 M, int E, bool neg) {
	const int q = E >> 6, b = E & 63;
	const uint64_t lo = (uint64_t)M, hi = (uint64_t)(M >> 64);
	uint64_t s[3];
	s[0] = lo << b;
	s[1] = b ? (hi << b) | (lo >> (64 - b)) : hi;
	s[2] = b ? hi >> (64 - b) : 0;
	uint64_t c = 0;
	if (!neg) {
		for (int k = 0; k < 3; k++) {
			const uint64_t a = acc[q + k], t = a + s[k], t2 = t + c;
			c = (uint64_t)(t < a) | (uint64_t)(t2 < t);
			acc[q + k] = t2;
		}
		for (int k = q + 3; c && k < W; k++) c = (++acc[k] == 0);
	} else {
		for (int k = 0; k < 3; k++) {
			const uint64_t a = acc[q + k], t = a - s[k], t2 = t - c;
			c = (uint64_t)(a < s[k]) | (uint64_t)(t < c);
			acc[q + k] = t2;
		}
		for (int k = q + 3; c && k < W; k++) c = (acc[k]-- == 0);
	}
}

template <int W>
__device__ __forceinline__ int acc_sign(const uint64_t* acc) {
	if ((int64_t)acc[W - 1] < 0) return -1;
	for (int k = 0; k < W; k++)
		if (acc[k]) return 1;
	return 0;
}

// the six terms of det3 over rows r0, r1, r2 (xyz), each multiplied by `sq` (the square of coordinate (sq_p, sq_k) when
// sq_p >= 0), with overall sign `neg`
template <int W>
__device__ __forceinline__ void add_det3(uint64_t* acc, const Dec* d, int r0, int r1, int r2, int sq_p, int sq_k, bool neg) {
	const int perm[6][3] = {{0, 1, 2}, {0, 2, 1}, {1, 0, 2}, {1, 2, 0}, {2, 0, 1}, {2, 1, 0}};
	const bool odd[6] = {false, true, true, false, false, true};
	unsigned __int128 f = 1;
	int fe = 0;
	if (sq_p >= 0) {
		const uint64_t m = d[sq_p].m[sq_k];
		if (!m) return;
		f = (unsigned __int128)(m * m);   // < 2^48
		fe = 2 * d[sq_p].e[sq_k];
	}
#pragma unroll
	for (int s = 0; s < 6; s++) {
		const int a = perm[s][0], b = perm[s][1], c = perm[s][2];
		const uint64_t m01 = (uint64_t)d[r0].m[a] * d[r1].m[b];
		const unsigned __int128 M3 = (unsigned __int128)m01 * d[r2].m[c];   // < 2^72; times f < 2^120
		if (!M3) continue;
		const bool n = neg ^ odd[s] ^ (((d[r0].neg >> a) ^ (d[r1].neg >> b) ^ (d[r2].neg >> c)) & 1u);
		acc_add<W>(acc, M3 * f, d[r0].e[a] + d[r1].e[b] + d[r2].e[c] + fe, n);
	}
}

// exact sign of det[b - a, c - a, d - a] = det3(b,c,d) - det3(a,c,d) + det3(a,b,d) - det3(a,b,c)
__device__ __noinline__ int orient3d_exact(const float4& a, const float4& b, const float4& c, const float4& e) {
	constexpr int W = 14;   // 3 * 247 + 72 + 5 + 1 bits, plus the two words a shifted monomial may span
	uint64_t acc[W];
	for (int k = 0; k < W; k++) acc[k] = 0;
	Dec d[4] = {decompose(a), decompose(b), decompose(c), decompose(e)};
	add_det3<W>(acc, d, 1, 2, 3, -1, 0, false);
	add_det3<W>(acc, d, 0, 2, 3, -1, 0, true);
	add_det3<W>(acc, d, 0, 1, 3, -1, 0, false);
	add_det3<W>(acc, d, 0, 1, 2, -1, 0, true);
	return acc_sign<W>(acc);
}

// exact sign of -D5, D5 = det of the rows (x, y, z, x^2 + y^2 + z^2, 1) of a, b, c, d, e: positive when e lies strictly
// inside the circumsphere of the positively oriented a, b, c, d
__device__ __noinline__ int insphere_exact(const float4* p) {
	constexpr int W = 22;   // 5 * 247 + 120 + 9 + 1 bits, plus the two words a shifted monomial may span
	uint64_t acc[W];
	for (int k = 0; k < W; k++) acc[k] = 0;
	Dec d[5];
	for (int i = 0; i < 5; i++) d[i] = decompose(p[i]);
	// D5 = sum_i (-1)^(i+5) det4_i(x, y, z, l), det4 = sum_t (-1)^(t+4) l_t det3(others): the term of (i, t) has sign
	// -(-1)^(i+t) in D5, so (-1)^(i+t) in -D5 (0-based i, t)
	for (int i = 0; i < 5; i++) {
		int r[4], n = 0;
		for (int j = 0; j < 5; j++)
			if (j != i) r[n++] = j;
		for (int t = 0; t < 4; t++) {
			int o[3], k = 0;
			for (int u = 0; u < 4; u++)
				if (u != t) o[k++] = r[u];
			const bool neg = ((i + t) & 1) != 0;
			for (int c = 0; c < 3; c++) add_det3<W>(acc, d, o[0], o[1], o[2], r[t], c, neg);
		}
	}
	return acc_sign<W>(acc);
}

// Shewchuk's stage-A filters; the absolute slack covers products that underflow (coordinates within 2^122 keep every
// intermediate below 2^615, so nothing overflows)
constexpr double EPS = 1.1102230246251565e-16;                 // 2^-53
constexpr double O3D_BOUND = (7.0 + 56.0 * EPS) * EPS;
constexpr double ISP_BOUND = (16.0 + 224.0 * EPS) * EPS;
constexpr double UNDERFLOW_SLACK = 0x1p-600;

__device__ int orient3d(const float4& pa, const float4& pb, const float4& pc, const float4& pd) {
	// Shewchuk's orient3d(pa, pb, pc, pd) is det[a - d, b - d, c - d] = -det[b - a, c - a, d - a]
	const double adx = (double)pa.x - pd.x, bdx = (double)pb.x - pd.x, cdx = (double)pc.x - pd.x;
	const double ady = (double)pa.y - pd.y, bdy = (double)pb.y - pd.y, cdy = (double)pc.y - pd.y;
	const double adz = (double)pa.z - pd.z, bdz = (double)pb.z - pd.z, cdz = (double)pc.z - pd.z;
	const double bdxcdy = bdx * cdy, cdxbdy = cdx * bdy, cdxady = cdx * ady, adxcdy = adx * cdy, adxbdy = adx * bdy, bdxady = bdx * ady;
	const double det = adz * (bdxcdy - cdxbdy) + bdz * (cdxady - adxcdy) + cdz * (adxbdy - bdxady);
	const double perm = (fabs(bdxcdy) + fabs(cdxbdy)) * fabs(adz) + (fabs(cdxady) + fabs(adxcdy)) * fabs(bdz) + (fabs(adxbdy) + fabs(bdxady)) * fabs(cdz);
	const double bound = O3D_BOUND * perm + UNDERFLOW_SLACK;
	if (det > bound) return -1;
	if (-det > bound) return 1;
	return orient3d_exact(pa, pb, pc, pd);
}

__device__ int insphere(const float4* p) {
	const float4 &pa = p[0], &pb = p[1], &pc = p[2], &pd = p[3], &pe = p[4];
	const double aex = (double)pa.x - pe.x, bex = (double)pb.x - pe.x, cex = (double)pc.x - pe.x, dex = (double)pd.x - pe.x;
	const double aey = (double)pa.y - pe.y, bey = (double)pb.y - pe.y, cey = (double)pc.y - pe.y, dey = (double)pd.y - pe.y;
	const double aez = (double)pa.z - pe.z, bez = (double)pb.z - pe.z, cez = (double)pc.z - pe.z, dez = (double)pd.z - pe.z;
	const double aexbey = aex * bey, bexaey = bex * aey, ab = aexbey - bexaey;
	const double bexcey = bex * cey, cexbey = cex * bey, bc = bexcey - cexbey;
	const double cexdey = cex * dey, dexcey = dex * cey, cd = cexdey - dexcey;
	const double dexaey = dex * aey, aexdey = aex * dey, da = dexaey - aexdey;
	const double aexcey = aex * cey, cexaey = cex * aey, ac = aexcey - cexaey;
	const double bexdey = bex * dey, dexbey = dex * bey, bd = bexdey - dexbey;
	const double abc = aez * bc - bez * ac + cez * ab;
	const double bcd = bez * cd - cez * bd + dez * bc;
	const double cda = cez * da + dez * ac + aez * cd;
	const double dab = dez * ab + aez * bd + bez * da;
	const double alift = aex * aex + aey * aey + aez * aez, blift = bex * bex + bey * bey + bez * bez;
	const double clift = cex * cex + cey * cey + cez * cez, dlift = dex * dex + dey * dey + dez * dez;
	const double det = (dlift * abc - clift * dab) + (blift * cda - alift * bcd);   // = D5
	const double aezp = fabs(aez), bezp = fabs(bez), cezp = fabs(cez), dezp = fabs(dez);
	const double aexbeyp = fabs(aexbey), bexaeyp = fabs(bexaey), bexceyp = fabs(bexcey), cexbeyp = fabs(cexbey);
	const double cexdeyp = fabs(cexdey), dexceyp = fabs(dexcey), dexaeyp = fabs(dexaey), aexdeyp = fabs(aexdey);
	const double aexceyp = fabs(aexcey), cexaeyp = fabs(cexaey), bexdeyp = fabs(bexdey), dexbeyp = fabs(dexbey);
	const double perm = ((cexdeyp + dexceyp) * bezp + (dexbeyp + bexdeyp) * cezp + (bexceyp + cexbeyp) * dezp) * alift +
	                    ((dexaeyp + aexdeyp) * cezp + (aexceyp + cexaeyp) * dezp + (cexdeyp + dexceyp) * aezp) * blift +
	                    ((aexbeyp + bexaeyp) * dezp + (bexdeyp + dexbeyp) * aezp + (dexaeyp + aexdeyp) * bezp) * clift +
	                    ((bexceyp + cexbeyp) * aezp + (cexaeyp + aexceyp) * bezp + (aexbeyp + bexaeyp) * cezp) * dlift;
	const double bound = ISP_BOUND * perm + UNDERFLOW_SLACK;
	if (det > bound) return -1;
	if (-det > bound) return 1;
	return insphere_exact(p);
}

__device__ __forceinline__ bool lex_less(const float4& a, const float4& b) {
	return a.x < b.x || (a.x == b.x && (a.y < b.y || (a.y == b.y && a.z < b.z)));
}

// insphere under the lifting perturbation: the lifted coordinate of point i gets eps_i > 0, eps of a lexicographically
// larger point infinitely larger; -D5 then gains -sum_i eps_i C_i with C_i = (-1)^i orient3d(the other four, in order)
__device__ int insphere_perturbed(const float4* p) {
	const int s = insphere(p);
	if (s) return s;
	int ord[5] = {0, 1, 2, 3, 4};
	for (int i = 1; i < 5; i++)   // descending lexicographic order
		for (int j = i; j > 0 && lex_less(p[ord[j - 1]], p[ord[j]]); j--) {
			const int t = ord[j];
			ord[j] = ord[j - 1];
			ord[j - 1] = t;
		}
	for (int k = 0; k < 5; k++) {
		const int i = ord[k];
		float4 q[4];
		int n = 0;
		for (int j = 0; j < 5; j++)
			if (j != i) q[n++] = p[j];
		const int o = orient3d(q[0], q[1], q[2], q[3]);
		if (o) return (i & 1) ? o : -o;
	}
	return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// preparation

__device__ __forceinline__ uint32_t f2ord(float f) {
	const uint32_t u = __float_as_uint(f);
	return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ uint32_t key_bits(float f) { return f == 0.0f ? 0u : __float_as_uint(f); }   // -0 == +0

__global__ void __launch_bounds__(DT_BLOCK) dt_check_kernel(int N, const float* __restrict__ pts, DtCounters* __restrict__ cnt,
                                                            uint64_t* __restrict__ key_yz, uint32_t* __restrict__ key_x, uint32_t* __restrict__ ids) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= N) return;
	const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
	const float lim = DT_MAX_COORD;
	if (!(fabsf(x) <= lim && fabsf(y) <= lim && fabsf(z) <= lim)) atomicAdd(&cnt->bad, 1);   // NaN fails too
	atomicMin(&cnt->box[0], f2ord(x));
	atomicMin(&cnt->box[1], f2ord(y));
	atomicMin(&cnt->box[2], f2ord(z));
	atomicMax(&cnt->box[3], f2ord(x));
	atomicMax(&cnt->box[4], f2ord(y));
	atomicMax(&cnt->box[5], f2ord(z));
	key_yz[i] = ((uint64_t)key_bits(y) << 32) | key_bits(z);
	key_x[i] = key_bits(x);
	ids[i] = (uint32_t)i;
}

__global__ void __launch_bounds__(DT_BLOCK) dt_gather_x_kernel(int N, const float* __restrict__ pts, const uint32_t* __restrict__ ids, uint32_t* __restrict__ key_x) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < N) key_x[i] = key_bits(pts[3 * (size_t)ids[i]]);
}

__device__ __forceinline__ bool same_point(const float* pts, uint32_t a, uint32_t b) {
	return pts[3 * (size_t)a] == pts[3 * (size_t)b] && pts[3 * (size_t)a + 1] == pts[3 * (size_t)b + 1] && pts[3 * (size_t)a + 2] == pts[3 * (size_t)b + 2];
}

// after the stable sorts, equal points are adjacent in ascending index order: the first of each run represents them
__global__ void __launch_bounds__(DT_BLOCK) dt_first_kernel(int N, const float* __restrict__ pts, const uint32_t* __restrict__ ids, uint32_t* __restrict__ first) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < N) first[i] = (i == 0 || !same_point(pts, ids[i], ids[i - 1])) ? 1u : 0u;
}

__device__ __forceinline__ uint64_t spread21(uint64_t v) {
	v &= 0x1fffffull;
	v = (v | (v << 32)) & 0x1f00000000ffffull;
	v = (v | (v << 16)) & 0x1f0000ff0000ffull;
	v = (v | (v << 8)) & 0x100f00f00f00f00full;
	v = (v | (v << 4)) & 0x10c30c30c30c30c3ull;
	v = (v | (v << 2)) & 0x1249249249249249ull;
	return v;
}
__device__ __forceinline__ uint64_t cell21(float x, double lo, double ext) {
	const double t = ext > 0.0 ? ((double)x - lo) / ext * 2097152.0 : 0.0;
	return t >= 2097151.0 ? 2097151ull : (t > 0.0 ? (uint64_t)t : 0ull);
}

// the representatives, compacted, with their Morton keys over the box
__global__ void __launch_bounds__(DT_BLOCK) dt_unique_kernel(int N, const float* __restrict__ pts, const uint32_t* __restrict__ ids,
                                                             const uint32_t* __restrict__ first, const uint32_t* __restrict__ rank, double3 lo, double ext,
                                                             uint64_t* __restrict__ mkey, uint32_t* __restrict__ rep, uint32_t* __restrict__ iota) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= N || !first[i]) return;
	const uint32_t id = ids[i], r = rank[i];
	const float x = pts[3 * (size_t)id], y = pts[3 * (size_t)id + 1], z = pts[3 * (size_t)id + 2];
	mkey[r] = (spread21(cell21(x, lo.x, ext)) << 2) | (spread21(cell21(y, lo.y, ext)) << 1) | spread21(cell21(z, lo.z, ext));
	rep[r] = id;
	iota[r] = r;
}

// vertices: the n representatives in Morton order, then the 4 ghosts; one cell (the ghost tetrahedron, made positive)
__global__ void __launch_bounds__(DT_BLOCK) dt_init_kernel(int n, const float* __restrict__ pts, const uint32_t* __restrict__ order,
                                                           const uint32_t* __restrict__ rep_in, uint32_t* __restrict__ rep, float4* __restrict__ verts,
                                                           int32_t* __restrict__ loc, float4 g0, float4 g1, float4 g2, float4 g3, DtMesh m) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) {
		const uint32_t id = rep_in[order[i]];
		rep[i] = id;
		verts[i] = make_float4(pts[3 * (size_t)id], pts[3 * (size_t)id + 1], pts[3 * (size_t)id + 2], 0.0f);
		loc[i] = 0;
	}
	if (i == 0) {
		verts[n] = g0;
		verts[n + 1] = g1;
		verts[n + 2] = g2;
		verts[n + 3] = g3;
		const bool pos = orient3d(g0, g1, g2, g3) > 0;
		m.tet[0] = pos ? make_int4(n, n + 1, n + 2, n + 3) : make_int4(n, n + 1, n + 3, n + 2);
		m.adj[0] = make_int4(-1, -1, -1, -1);
	}
}

// ---------------------------------------------------------------------------------------------------------------------
// rounds

__device__ __forceinline__ int geti(const int4& v, int k) { return k == 0 ? v.x : k == 1 ? v.y : k == 2 ? v.z : v.w; }
__device__ __forceinline__ void seti(int4& v, int k, int x) {
	if (k == 0) v.x = x;
	else if (k == 1) v.y = x;
	else if (k == 2) v.z = x;
	else v.w = x;
}

__device__ __forceinline__ uint32_t hash32(uint32_t x) {
	x ^= x >> 16;
	x *= 0x7feb352du;
	x ^= x >> 15;
	x *= 0x846ca68bu;
	x ^= x >> 16;
	return x;
}

__device__ __forceinline__ bool conflict(const float4* verts, const int4& t, int p) {
	float4 q[5] = {verts[t.x], verts[t.y], verts[t.z], verts[t.w], verts[p]};
	return insphere_perturbed(q) > 0;
}

// each cell nominates the point of smallest (hash, index): a random insertion order keeps cells fat and cavities small
// (the smallest index alone, in Morton order, grows slivers)
__global__ void __launch_bounds__(DT_BLOCK) dt_nominate_kernel(int n, const int32_t* __restrict__ loc, uint64_t* __restrict__ nom) {
	const int q = blockIdx.x * blockDim.x + threadIdx.x;
	if (q >= n) return;
	const int c = loc[q];
	if (c >= 0) atomicMin((unsigned long long*)nom + c, (unsigned long long)(((uint64_t)hash32((uint32_t)q ^ 0x9e3779b9u) << 32) | (uint32_t)q));
}

// cells: the host's count, the extent that the round's memsets initialised
__global__ void __launch_bounds__(DT_BLOCK) dt_collect_kernel(int cells, DtCounters* cnt, const uint64_t* __restrict__ nom, DtSlots sl, int K) {
	const int c = blockIdx.x * blockDim.x + threadIdx.x;
	if (c >= cells || nom[c] == NO_NOMINEE) return;
	const int slot = atomicAdd(&cnt->slots, 1);
	if (slot < K) {
		sl.point[slot] = (int)(uint32_t)nom[c];
		sl.cell[slot] = c;
	}
}

// breadth-first search of the cavity of slot's point; cavity cells into cav[slot * cc_cap ...], boundary faces (the new
// cell and the outside neighbour) into bnd / bout[slot * cb_cap ...].  mark: visited flags in nom[] (single-cavity pass).
// A cavity over the capacity is appended to `over_list` (a round's slots: the large-slot pass takes them all), or, in
// the large-slot pass (no list), recorded as overflow_point for the single-cavity pass.
__global__ void __launch_bounds__(DT_BLOCK) dt_cavity_kernel(int K, DtCounters* cnt, const float4* __restrict__ verts, DtMesh m, DtSlots sl,
                                                             int cc_cap, int cb_cap, int mark, uint32_t* __restrict__ over_list) {
	const int slot = blockIdx.x * blockDim.x + threadIdx.x;
	if (slot >= K || slot >= cnt->slots) return;
	const int p = sl.point[slot];
	int* cav = sl.cav + (size_t)slot * cc_cap;
	int4* bnd = sl.bnd + (size_t)slot * cb_cap;
	int* bout = sl.bout + (size_t)slot * cb_cap;
	int k = 1, b = 0;
	bool over = false;
	cav[0] = sl.cell[slot];
	if (mark) m.nom[cav[0]] = VISITED;
	for (int i = 0; i < k && !over; i++) {
		const int c = cav[i];
		const int4 t = m.tet[c], a = m.adj[c];
		for (int f = 0; f < 4; f++) {
			const int o = geti(a, f);
			if (o >= 0) {
				const int nc = o >> 2;
				bool seen = false;
				if (mark) seen = m.nom[nc] == VISITED;
				else
					for (int j = 0; j < k && !seen; j++) seen = cav[j] == nc;
				if (seen) continue;
				if (conflict(verts, m.tet[nc], p)) {
					if (k == cc_cap) { over = true; break; }
					if (mark) m.nom[nc] = VISITED;
					cav[k++] = nc;
					continue;
				}
			}
			if (b == cb_cap) { over = true; break; }
			int4 nt = t;
			seti(nt, f, p);
			bnd[b] = nt;
			bout[b] = o;
			b++;
		}
	}
	sl.k[slot] = over ? -1 : k;
	sl.b[slot] = b;
	if (over) {
		const int at = atomicAdd(&cnt->overflowed, 1);
		if (over_list) over_list[at] = (uint32_t)p;   // at most one entry per nominee: fits the n entries
		else atomicMin(&cnt->overflow_point, p);
	} else
		atomicMax(&cnt->max_cavity, k);
}

__device__ __forceinline__ uint64_t slot_key(int p, int slot) { return ((uint64_t)hash32((uint32_t)p) << 32) | (uint32_t)slot; }

__global__ void __launch_bounds__(DT_BLOCK) dt_claim_kernel(int K, const DtCounters* __restrict__ cnt, DtMesh m, DtSlots sl, int cc_cap, int cb_cap) {
	const int slot = blockIdx.x * blockDim.x + threadIdx.x;
	if (slot >= K || slot >= cnt->slots || sl.k[slot] < 0) return;
	const uint64_t key = slot_key(sl.point[slot], slot);
	const int k = sl.k[slot], b = sl.b[slot];
	for (int i = 0; i < k; i++) atomicMin((unsigned long long*)m.claim + sl.cav[(size_t)slot * cc_cap + i], (unsigned long long)key);
	for (int j = 0; j < b; j++) {
		const int o = sl.bout[(size_t)slot * cb_cap + j];
		if (o >= 0) atomicMin((unsigned long long*)m.claim + (o >> 2), (unsigned long long)key);
	}
}

// a winner (or the forced single cavity) replaces its k cavity cells by its b new cells: slots cav[0..min(k,b)) first,
// then b - k appended ones; leftover cavity slots die
__global__ void __launch_bounds__(DT_BLOCK) dt_star_kernel(int K, DtCounters* cnt, const float4* __restrict__ verts, DtMesh m, DtSlots sl, int cc_cap,
                                                           int cb_cap, int force, int epoch, int cap) {
	const int slot = blockIdx.x * blockDim.x + threadIdx.x;
	if (slot >= K || slot >= cnt->slots) return;
	const int k = sl.k[slot], b = sl.b[slot], p = sl.point[slot];
	sl.won[slot] = 0;
	if (k < 0) return;
	const int* cav = sl.cav + (size_t)slot * cc_cap;
	const int4* bnd = sl.bnd + (size_t)slot * cb_cap;
	const int* bout = sl.bout + (size_t)slot * cb_cap;
	if (!force) {
		const uint64_t key = slot_key(p, slot);
		for (int i = 0; i < k; i++)
			if (m.claim[cav[i]] != key) return;
		for (int j = 0; j < b; j++)
			if (bout[j] >= 0 && m.claim[bout[j] >> 2] != key) return;
	}
	int base = 0;
	if (b > k) {
		base = atomicAdd(&cnt->cells, b - k);
		if ((int64_t)base + (b - k) > cap) {   // the caller grows the mesh; this cavity waits for the next round
			atomicExch(&cnt->full, 1);
			return;
		}
	}
	sl.won[slot] = 1;
	sl.base[slot] = base;
	for (int i = 0; i < k; i++) m.died[cav[i]] = make_int2(epoch, slot);
	for (int j = 0; j < b; j++) {
		const int cell = j < k ? cav[j] : base + (j - k);
		const int4 t = bnd[j];
		if (orient3d(verts[t.x], verts[t.y], verts[t.z], verts[t.w]) <= 0) atomicExch(&cnt->violation, 1);
		int f = 0;
		while (geti(t, f) != p) f++;
		int4 a;
		seti(a, f, bout[j]);
		if (bout[j] >= 0) reinterpret_cast<int*>(m.adj + (bout[j] >> 2))[bout[j] & 3] = (cell << 2) | f;
		for (int s = 0; s < 4; s++) {
			if (s == f) continue;
			int e0 = -1, e1 = -1;   // the edge of the boundary face that the face opposite slot s shares with another new cell
			for (int u = 0; u < 4; u++)
				if (u != s && u != f) (e0 < 0 ? e0 : e1) = geti(t, u);
			int link = -1;
			for (int j2 = 0; j2 < b && link < 0; j2++) {
				if (j2 == j) continue;
				const int4 t2 = bnd[j2];
				int h0 = -1, h1 = -1, w = -1;
				for (int u = 0; u < 4; u++) {
					const int v = geti(t2, u);
					if (v == e0) h0 = u;
					else if (v == e1) h1 = u;
					else if (v != p) w = u;
				}
				if (h0 >= 0 && h1 >= 0) link = ((j2 < k ? cav[j2] : base + (j2 - k)) << 2) | w;
			}
			if (link < 0) atomicExch(&cnt->violation, 1);
			seti(a, s, link);
		}
		m.tet[cell] = t;
		m.adj[cell] = a;
	}
	for (int i = b; i < k; i++) m.tet[cav[i]] = make_int4(-1, -1, -1, -1);
	atomicAdd(&cnt->inserted, 1);
}

__device__ __forceinline__ bool in_closed(const float4* verts, const int4& t, const float4& q) {
	const float4 a = verts[t.x], b = verts[t.y], c = verts[t.z], d = verts[t.w];
	return orient3d(q, b, c, d) >= 0 && orient3d(a, q, c, d) >= 0 && orient3d(a, b, q, d) >= 0 && orient3d(a, b, c, q) >= 0;
}

// inserted points leave the pool; a point whose cell died finds the new cell of the same winner whose closure holds it
__global__ void __launch_bounds__(DT_BLOCK) dt_relocate_kernel(int n, DtCounters* cnt, const float4* __restrict__ verts, DtMesh m, DtSlots sl, int cc_cap,
                                                               int epoch) {
	const int q = blockIdx.x * blockDim.x + threadIdx.x;
	if (q >= n) return;
	const int c = m.loc[q];
	if (c < 0) return;
	const int2 dd = m.died[c];
	if (dd.x != epoch) return;
	const int slot = dd.y;
	if (sl.point[slot] == q) {
		m.loc[q] = -1;
		return;
	}
	const int k = sl.k[slot], b = sl.b[slot], base = sl.base[slot];
	const float4 pq = verts[q];
	for (int j = 0; j < b; j++) {
		const int cell = j < k ? sl.cav[(size_t)slot * cc_cap + j] : base + (j - k);
		if (in_closed(verts, m.tet[cell], pq)) {
			m.loc[q] = cell;
			return;
		}
	}
	atomicExch(&cnt->violation, 1);
}

// the large-slot pass: the points whose cavity overflowed a round's slot, up to K of them, each in a slot of the slab
// area divided K ways; they claim, star and relocate like a round's nominees
__global__ void __launch_bounds__(DT_BLOCK) dt_large_setup_kernel(int K, const DtCounters* __restrict__ cnt, const uint32_t* __restrict__ list,
                                                                  const int32_t* __restrict__ loc, DtSlots sl) {
	const int slot = blockIdx.x * blockDim.x + threadIdx.x;
	if (slot >= K || slot >= cnt->overflowed) return;
	const int p = (int)list[slot];
	sl.point[slot] = p;
	sl.cell[slot] = loc[p];
}

__global__ void dt_large_reset_kernel(DtCounters* cnt, int K) {
	cnt->slots = min(cnt->overflowed, K);
	cnt->overflowed = 0;
	cnt->overflow_point = 0x7fffffff;
	cnt->full = 0;
}

// the single-cavity pass: the overflowed point with the smallest index, alone in slot 0 (overflow_point stays set, so a
// retry after the slab or the mesh grew takes the same point)
__global__ void dt_single_kernel(DtCounters* cnt, DtMesh m, DtSlots sl) {
	const int p = cnt->overflow_point;
	sl.point[0] = p;
	sl.cell[0] = m.loc[p];
	cnt->slots = 1;
	cnt->overflowed = 0;
	cnt->full = 0;
}

__global__ void dt_round_reset_kernel(DtCounters* cnt, int cap) {
	cnt->cells = min(cnt->cells, cap);
	cnt->slots = 0;
	cnt->full = 0;
	cnt->overflowed = 0;
	cnt->overflow_point = 0x7fffffff;
}

// ---------------------------------------------------------------------------------------------------------------------
// output: the cells without a ghost, as representatives' indices, canonically rotated

__device__ __forceinline__ int4 canonical(int a, int b, int c, int d) {
	// an even permutation brings the smallest index first ...
	int4 r = make_int4(a, b, c, d);
	const int mn = min(min(a, b), min(c, d));
	if (b == mn) r = make_int4(b, a, d, c);
	else if (c == mn) r = make_int4(c, d, a, b);
	else if (d == mn) r = make_int4(d, c, b, a);
	// ... and a 3-cycle of the last three the smallest of them second
	if (r.z < r.y && r.z < r.w) r = make_int4(r.x, r.z, r.w, r.y);
	else if (r.w < r.y && r.w < r.z) r = make_int4(r.x, r.w, r.y, r.z);
	return r;
}

__global__ void __launch_bounds__(DT_BLOCK) dt_emit_kernel(int n, int cells, DtCounters* cnt, DtMesh m, const uint32_t* __restrict__ rep,
                                                           int4* __restrict__ rows) {
	const int c = blockIdx.x * blockDim.x + threadIdx.x;
	if (c >= cells) return;
	const int4 t = m.tet[c];
	if (t.x < 0 || t.x >= n || t.y >= n || t.z >= n || t.w >= n) return;
	const int r = atomicAdd(&cnt->out_cells, 1);
	rows[r] = canonical((int)rep[t.x], (int)rep[t.y], (int)rep[t.z], (int)rep[t.w]);
}

__global__ void __launch_bounds__(DT_BLOCK) dt_key_kernel(int T, const int4* __restrict__ rows, const uint32_t* __restrict__ ids, int hi,
                                                          uint64_t* __restrict__ keys, uint32_t* __restrict__ ids_out) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= T) return;
	const uint32_t id = ids ? ids[i] : (uint32_t)i;
	const int4 r = rows[id];
	keys[i] = hi ? ((uint64_t)(uint32_t)r.x << 32) | (uint32_t)r.y : ((uint64_t)(uint32_t)r.z << 32) | (uint32_t)r.w;
	ids_out[i] = id;
}

__global__ void __launch_bounds__(DT_BLOCK) dt_gather_rows_kernel(int T, const int4* __restrict__ rows, const uint32_t* __restrict__ ids, int4* __restrict__ out) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < T) out[i] = rows[ids[i]];
}

__global__ void __launch_bounds__(DT_BLOCK) dt_predicates_kernel(int M, int N, const float* __restrict__ pts, const int32_t* __restrict__ tuples,
                                                                 int8_t* __restrict__ signs, int* __restrict__ bad) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= M) return;
	float4 q[5];
	for (int k = 0; k < 5; k++) {
		const int id = tuples[5 * (size_t)i + k];
		if (id < 0 || id >= N) {
			atomicExch(bad, 1);
			return;
		}
		q[k] = make_float4(pts[3 * (size_t)id], pts[3 * (size_t)id + 1], pts[3 * (size_t)id + 2], 0.0f);
		if (!(isfinite(q[k].x) && isfinite(q[k].y) && isfinite(q[k].z))) {
			atomicExch(bad, 2);
			return;
		}
	}
	signs[3 * (size_t)i] = (int8_t)orient3d(q[0], q[1], q[2], q[3]);
	signs[3 * (size_t)i + 1] = (int8_t)insphere(q);
	signs[3 * (size_t)i + 2] = (int8_t)insphere_perturbed(q);
}

inline unsigned blocks(int64_t n) { return (unsigned)((n + DT_BLOCK - 1) / DT_BLOCK); }

// ---------------------------------------------------------------------------------------------------------------------
// host side

DtPointsView carve_dt_points(char* base, int N, size_t* total) {
	Carver c(base);
	DtPointsView v;
	v.cnt = c.take<DtCounters>(1);
	v.verts = c.take<float4>((size_t)N + 4);
	v.rep = c.take<uint32_t>(N);
	v.loc = c.take<int32_t>(N);
	v.key64[0] = c.take<uint64_t>(N);
	v.key64[1] = c.take<uint64_t>(N);
	v.key32[0] = c.take<uint32_t>(N);
	v.key32[1] = c.take<uint32_t>(N);
	v.ids[0] = c.take<uint32_t>(N);
	v.ids[1] = c.take<uint32_t>(N);
	v.first = c.take<uint32_t>(N);
	v.rank = c.take<uint32_t>(N);
	size_t t1 = 0, t2 = 0, t3 = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, t1, (uint64_t*)nullptr, (uint64_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, N, 0, 64);
	cub::DeviceRadixSort::SortPairs(nullptr, t2, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, N, 0, 32);
	cub::DeviceScan::ExclusiveSum(nullptr, t3, (uint32_t*)nullptr, (uint32_t*)nullptr, N);
	v.temp_bytes = std::max(t1, std::max(t2, t3));
	v.temp = c.take<char>(v.temp_bytes);
	if (total) *total = c.size();
	return v;
}

DtMesh carve_dt_mesh(char* base, int64_t cap, size_t* total) {
	Carver c(base);
	DtMesh m;
	m.tet = c.take<int4>(cap);
	m.adj = c.take<int4>(cap);
	m.claim = c.take<uint64_t>(cap);
	m.nom = c.take<uint64_t>(cap);
	m.died = c.take<int2>(cap);
	m.loc = nullptr;
	if (total) *total = c.size();
	return m;
}

DtSlots carve_dt_slots(char* base, int K, int64_t cc_total, int64_t cb_total, size_t* total) {
	Carver c(base);
	DtSlots s;
	s.point = c.take<int>(K);
	s.cell = c.take<int>(K);
	s.k = c.take<int>(K);
	s.b = c.take<int>(K);
	s.base = c.take<int>(K);
	s.won = c.take<int>(K);
	s.cav = c.take<int>(cc_total);
	s.bnd = c.take<int4>(cb_total);
	s.bout = c.take<int>(cb_total);
	if (total) *total = c.size();
	return s;
}

size_t dt_sort_bytes(int64_t cells) {
	size_t t = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, t, (uint64_t*)nullptr, (uint64_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)cells, 0, 64);
	Carver c(nullptr);
	c.take<int4>(cells);
	c.take<uint64_t>(cells);
	c.take<uint64_t>(cells);
	c.take<uint32_t>(cells);
	c.take<uint32_t>(cells);
	c.take<char>(t);
	return c.size();
}

cudaError_t launch_dt_prepare(int N, const float* pts, const DtPointsView& v, DtCounters* host, cudaStream_t s) {
	DtCounters init{};
	for (int k = 0; k < 3; k++) init.box[k] = 0xffffffffu;
	init.overflow_point = 0x7fffffff;
	RGS_TRY(cudaMemcpyAsync(v.cnt, &init, sizeof(init), cudaMemcpyHostToDevice, s));
	dt_check_kernel<<<blocks(N), DT_BLOCK, 0, s>>>(N, pts, v.cnt, v.key64[0], v.key32[0], v.ids[0]);
	count_launch();
	size_t tb = v.temp_bytes;
	RGS_TRY(cub::DeviceRadixSort::SortPairs(v.temp, tb, v.key64[0], v.key64[1], v.ids[0], v.ids[1], N, 0, 64, s));
	dt_gather_x_kernel<<<blocks(N), DT_BLOCK, 0, s>>>(N, pts, v.ids[1], v.key32[0]);
	count_launch();
	tb = v.temp_bytes;
	RGS_TRY(cub::DeviceRadixSort::SortPairs(v.temp, tb, v.key32[0], v.key32[1], v.ids[1], v.ids[0], N, 0, 32, s));
	dt_first_kernel<<<blocks(N), DT_BLOCK, 0, s>>>(N, pts, v.ids[0], v.first);
	count_launch();
	tb = v.temp_bytes;
	RGS_TRY(cub::DeviceScan::ExclusiveSum(v.temp, tb, v.first, v.rank, N, s));
	RGS_TRY(cudaMemcpyAsync(host, v.cnt, sizeof(DtCounters), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaMemcpyAsync(&host->unique, v.rank + (N - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaMemcpyAsync(&host->spare, v.first + (N - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaStreamSynchronize(s));
	host->unique += host->spare;
	return cudaGetLastError();
}

__host__ static float ord2f_host(uint32_t u) {
	const uint32_t b = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
	float f;
	memcpy(&f, &b, sizeof(f));
	return f;
}

cudaError_t launch_dt_init(int N, const float* pts, int n, const DtPointsView& v, const DtCounters& host, const DtMesh& m, int64_t cap, cudaStream_t s) {
	double lo[3], hi[3], ext = 0.0;
	for (int k = 0; k < 3; k++) {
		lo[k] = ord2f_host(host.box[k]);
		hi[k] = ord2f_host(host.box[3 + k]);
		ext = std::max(ext, hi[k] - lo[k]);
	}
	dt_unique_kernel<<<blocks(N), DT_BLOCK, 0, s>>>(N, pts, v.ids[0], v.first, v.rank, make_double3(lo[0], lo[1], lo[2]), ext, v.key64[0], v.key32[0],
	                                                v.key32[1]);
	count_launch();
	size_t tb = v.temp_bytes;
	RGS_TRY(cub::DeviceRadixSort::SortPairs(v.temp, tb, v.key64[0], v.key64[1], v.key32[1], v.ids[1], n, 0, 63, s));
	// ghosts: R = the smallest power of two >= the extent, S = 2^30 R, g_k = fl32(c + S * sign_k), c the box centre
	double R = 1.0;
	while (R < ext) R *= 2.0;
	while (R * 0.5 >= ext && R > 0x1p-100) R *= 0.5;
	const double S = DT_GHOST_SCALE * R;
	const double c[3] = {0.5 * (lo[0] + hi[0]), 0.5 * (lo[1] + hi[1]), 0.5 * (lo[2] + hi[2])};
	auto ghost = [&](double sx, double sy, double sz) {
		return make_float4((float)(c[0] + sx * S), (float)(c[1] + sy * S), (float)(c[2] + sz * S), 0.0f);
	};
	RGS_TRY(cudaMemsetAsync(m.tet, 0xff, (size_t)cap * sizeof(int4), s));
	RGS_TRY(cudaMemsetAsync(m.died, 0, (size_t)cap * sizeof(int2), s));
	dt_init_kernel<<<blocks(n), DT_BLOCK, 0, s>>>(n, pts, v.ids[1], v.key32[0], v.rep, v.verts, v.loc, ghost(1, 1, 1), ghost(1, -1, -1), ghost(-1, 1, -1),
	                                              ghost(-1, -1, 1), m);
	count_launch();
	DtCounters init{};
	init.cells = 1;
	init.overflow_point = 0x7fffffff;
	RGS_TRY(cudaMemcpyAsync(v.cnt, &init, sizeof(init), cudaMemcpyHostToDevice, s));
	return cudaGetLastError();
}

cudaError_t launch_dt_round(int n, const DtPointsView& v, const DtMesh& m, const DtSlots& sl, int K, int cc, int cb, int epoch, int64_t cap, int cells,
                            cudaStream_t s) {
	DtMesh mm = m;
	mm.loc = v.loc;
	dt_round_reset_kernel<<<1, 1, 0, s>>>(v.cnt, (int)cap);
	RGS_TRY(cudaMemsetAsync(m.nom, 0xff, (size_t)cells * sizeof(uint64_t), s));
	RGS_TRY(cudaMemsetAsync(m.claim, 0xff, (size_t)cells * sizeof(uint64_t), s));
	dt_nominate_kernel<<<blocks(n), DT_BLOCK, 0, s>>>(n, v.loc, m.nom);
	dt_collect_kernel<<<blocks(cells), DT_BLOCK, 0, s>>>(cells, v.cnt, m.nom, sl, K);
	dt_cavity_kernel<<<blocks(K), DT_BLOCK, 0, s>>>(K, v.cnt, v.verts, mm, sl, cc, cb, 0, v.first);
	dt_claim_kernel<<<blocks(K), DT_BLOCK, 0, s>>>(K, v.cnt, mm, sl, cc, cb);
	dt_star_kernel<<<blocks(K), DT_BLOCK, 0, s>>>(K, v.cnt, v.verts, mm, sl, cc, cb, 0, epoch, (int)cap);
	dt_relocate_kernel<<<blocks(n), DT_BLOCK, 0, s>>>(n, v.cnt, v.verts, mm, sl, cc, epoch);
	count_launch(7);
	return cudaGetLastError();
}

cudaError_t launch_dt_large(int n, const DtPointsView& v, const DtMesh& m, const DtSlots& sl, int K, int cc, int cb, int epoch, int64_t cap, int cells,
                            cudaStream_t s) {
	DtMesh mm = m;
	mm.loc = v.loc;
	dt_large_setup_kernel<<<blocks(K), DT_BLOCK, 0, s>>>(K, v.cnt, v.first, v.loc, sl);
	dt_large_reset_kernel<<<1, 1, 0, s>>>(v.cnt, K);
	RGS_TRY(cudaMemsetAsync(m.claim, 0xff, (size_t)cells * sizeof(uint64_t), s));
	dt_cavity_kernel<<<blocks(K), DT_BLOCK, 0, s>>>(K, v.cnt, v.verts, mm, sl, cc, cb, 0, nullptr);
	dt_claim_kernel<<<blocks(K), DT_BLOCK, 0, s>>>(K, v.cnt, mm, sl, cc, cb);
	dt_star_kernel<<<blocks(K), DT_BLOCK, 0, s>>>(K, v.cnt, v.verts, mm, sl, cc, cb, 0, epoch, (int)cap);
	dt_relocate_kernel<<<blocks(n), DT_BLOCK, 0, s>>>(n, v.cnt, v.verts, mm, sl, cc, epoch);
	count_launch(6);
	return cudaGetLastError();
}

cudaError_t launch_dt_single_cavity(const DtPointsView& v, const DtMesh& m, const DtSlots& sl, int64_t cc_total, int64_t cb_total, int cells, cudaStream_t s) {
	DtMesh mm = m;
	mm.loc = v.loc;
	dt_single_kernel<<<1, 1, 0, s>>>(v.cnt, mm, sl);
	RGS_TRY(cudaMemsetAsync(m.nom, 0xff, (size_t)cells * sizeof(uint64_t), s));
	dt_cavity_kernel<<<1, 1, 0, s>>>(1, v.cnt, v.verts, mm, sl, (int)cc_total, (int)cb_total, 1, nullptr);
	count_launch(2);
	return cudaGetLastError();
}

cudaError_t launch_dt_single_star(int n, const DtPointsView& v, const DtMesh& m, const DtSlots& sl, int64_t cc_total, int64_t cb_total, int epoch, int64_t cap,
                                  cudaStream_t s) {
	DtMesh mm = m;
	mm.loc = v.loc;
	dt_star_kernel<<<1, 1, 0, s>>>(1, v.cnt, v.verts, mm, sl, (int)cc_total, (int)cb_total, 1, epoch, (int)cap);
	dt_relocate_kernel<<<blocks(n), DT_BLOCK, 0, s>>>(n, v.cnt, v.verts, mm, sl, (int)cc_total, epoch);
	count_launch(2);
	return cudaGetLastError();
}

cudaError_t launch_dt_read(const DtPointsView& v, DtCounters* host, cudaStream_t s) {
	RGS_TRY(cudaMemcpyAsync(host, v.cnt, sizeof(DtCounters), cudaMemcpyDeviceToHost, s));
	return cudaStreamSynchronize(s);
}

cudaError_t launch_dt_grow_mesh(const DtMesh& from, int64_t from_cap, const DtMesh& to, int64_t to_cap, cudaStream_t s) {
	RGS_TRY(cudaMemcpyAsync(to.tet, from.tet, (size_t)from_cap * sizeof(int4), cudaMemcpyDeviceToDevice, s));
	RGS_TRY(cudaMemcpyAsync(to.adj, from.adj, (size_t)from_cap * sizeof(int4), cudaMemcpyDeviceToDevice, s));
	RGS_TRY(cudaMemcpyAsync(to.died, from.died, (size_t)from_cap * sizeof(int2), cudaMemcpyDeviceToDevice, s));
	RGS_TRY(cudaMemsetAsync(to.tet + from_cap, 0xff, (size_t)(to_cap - from_cap) * sizeof(int4), s));
	RGS_TRY(cudaMemsetAsync(to.died + from_cap, 0, (size_t)(to_cap - from_cap) * sizeof(int2), s));
	return cudaSuccess;
}

cudaError_t launch_dt_emit(int n, const DtPointsView& v, const DtMesh& m, char* sort, int64_t cells, int* T, cudaStream_t s) {
	Carver c(sort);
	int4* rows = c.take<int4>(cells);
	dt_emit_kernel<<<blocks(cells), DT_BLOCK, 0, s>>>(n, (int)cells, v.cnt, m, v.rep, rows);
	count_launch();
	DtCounters h;
	RGS_TRY(launch_dt_read(v, &h, s));
	*T = h.out_cells;
	return cudaSuccess;
}

cudaError_t launch_dt_sort(char* sort, int64_t cells, int T, int4* out, cudaStream_t s) {
	Carver c(sort);
	int4* rows = c.take<int4>(cells);
	uint64_t* k0 = c.take<uint64_t>(cells);
	uint64_t* k1 = c.take<uint64_t>(cells);
	uint32_t* i0 = c.take<uint32_t>(cells);
	uint32_t* i1 = c.take<uint32_t>(cells);
	size_t t = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, t, k0, k1, i0, i1, (int)cells, 0, 64);
	char* temp = c.take<char>(t);
	if (T == 0) return cudaSuccess;
	// two stable passes: (r2, r3), then (r0, r1)
	dt_key_kernel<<<blocks(T), DT_BLOCK, 0, s>>>(T, rows, nullptr, 0, k0, i0);
	size_t tb = t;
	RGS_TRY(cub::DeviceRadixSort::SortPairs(temp, tb, k0, k1, i0, i1, T, 0, 64, s));
	dt_key_kernel<<<blocks(T), DT_BLOCK, 0, s>>>(T, rows, i1, 1, k0, i0);
	tb = t;
	RGS_TRY(cub::DeviceRadixSort::SortPairs(temp, tb, k0, k1, i0, i1, T, 0, 64, s));
	dt_gather_rows_kernel<<<blocks(T), DT_BLOCK, 0, s>>>(T, rows, i1, out);
	count_launch(3);
	return cudaGetLastError();
}

cudaError_t launch_dt_predicates(int N, const float* pts, int M, const int32_t* tuples, int8_t* signs, int* bad_dev, int* bad_host, cudaStream_t s) {
	RGS_TRY(cudaMemsetAsync(bad_dev, 0, sizeof(int), s));
	dt_predicates_kernel<<<blocks(M), DT_BLOCK, 0, s>>>(M, N, pts, tuples, signs, bad_dev);
	count_launch();
	RGS_TRY(cudaMemcpyAsync(bad_host, bad_dev, sizeof(int), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaStreamSynchronize(s));
	return cudaGetLastError();
}

}  // namespace
}  // namespace rgs

using namespace rgs;

extern "C" {

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

}  // extern "C"

// rgs_tetra.cu -- tetrahedra mesh extraction (reference mesh_extract_tetrahedra.py, utils/tetmesh.py, gaussian_model.py:400-429)
// on the GPU: tetra points, the multi-view cull SDF, marching tetrahedra, the bisection step and the distance/scale filter.
// Runs once per trained model, off the rasterizer path.
//
// The contract (include/rgs_b200.h, rgs_tetra_*) fixes every stored bit of stages 2-5: each fp32 operation is one intrinsic
// rounded on its own (__fadd_rn / __fmul_rn / __fdiv_rn / __fsqrt_rn; the filter's two __fmaf_rn are written out), so nvcc contracts nothing and a numpy fp32 restatement
// reproduces the results.
//   points     one thread per Gaussian: normalised quaternion -> R, 8 box corners R (+-3s) + xyz, then the centres.
//   cull       one thread per point and view: pixel -> grid_sample coordinate, zero-padded bilinear sample of
//              render7 (* gt_mask), test > 0.5, running min and count; a finish pass writes the SDF.
//   marching   per tet: index check and occupancy code; CUB's stable select of the valid tets (one host read); 6 edge keys
//              (min, max) per valid tet, CUB radix sort, head flags and one scan over the crossing heads; a stable radix
//              sort of the valid tets by (chunk, two triangles) and a scan of their triangle counts (one host read); then
//              the vertices and the faces, one thread each.
//   bisect     one thread per vertex.
//   filter     one thread per vertex / face, a scan of the kept vertices and CUB's stable select of vertices and faces.
//
// This file also holds the C-ABI entry points rgs_tetra_* (include/rgs_b200.h).
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "rgs_common.cuh"

namespace rgs {

namespace {

// utils/tetmesh.py: triangle_table, num_triangles_table and base_tet_edges
__constant__ int8_t c_tri_table[16][6] = {
	{-1, -1, -1, -1, -1, -1}, {1, 0, 2, -1, -1, -1}, {4, 0, 3, -1, -1, -1}, {1, 4, 2, 1, 3, 4},
	{3, 1, 5, -1, -1, -1},    {2, 3, 0, 2, 5, 3},    {1, 4, 0, 1, 5, 4},    {4, 2, 5, -1, -1, -1},
	{4, 5, 2, -1, -1, -1},    {4, 1, 0, 4, 5, 1},    {3, 2, 0, 3, 5, 2},    {1, 3, 5, -1, -1, -1},
	{4, 1, 2, 4, 3, 1},       {3, 0, 4, -1, -1, -1}, {2, 0, 1, -1, -1, -1}, {-1, -1, -1, -1, -1, -1}};
// num_triangles_table as one nibble per occupancy code
__host__ __device__ __forceinline__ int num_triangles(int code) { return (int)((0x0112122112212110ull >> (4 * code)) & 0xf); }
__constant__ int8_t c_tet_edges[6][2] = {{0, 1}, {0, 2}, {0, 3}, {1, 2}, {1, 3}, {2, 3}};

constexpr int64_t CHUNK = 32ll * 1024 * 1024;   // utils/tetmesh.py chunk_size

// ---- tetra points (gaussian_model.py:400-429) ---------------------------------------------------------------------------

__global__ void __launch_bounds__(256) tetra_points_kernel(int P, const float* __restrict__ xyz, const float* __restrict__ s,
                                                           const float* __restrict__ rot, float* __restrict__ pts, float* __restrict__ scl) {
	const int g = blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= P) return;
	const int64_t G = g;
	const float r0 = rot[4 * G], r1 = rot[4 * G + 1], r2 = rot[4 * G + 2], r3 = rot[4 * G + 3];
	const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r0, r0), __fmul_rn(r1, r1)), __fmul_rn(r2, r2)), __fmul_rn(r3, r3)));
	const float r = __fdiv_rn(r0, nrm), x = __fdiv_rn(r1, nrm), y = __fdiv_rn(r2, nrm), z = __fdiv_rn(r3, nrm);
	float R[3][3];
	R[0][0] = 1.f - 2.f * (y * y + z * z);
	R[0][1] = 2.f * (x * y - r * z);
	R[0][2] = 2.f * (x * z + r * y);
	R[1][0] = 2.f * (x * y + r * z);
	R[1][1] = 1.f - 2.f * (x * x + z * z);
	R[1][2] = 2.f * (y * z - r * x);
	R[2][0] = 2.f * (x * z - r * y);
	R[2][1] = 2.f * (y * z + r * x);
	R[2][2] = 1.f - 2.f * (x * x + y * y);
	const float sx = __fmul_rn(s[3 * G], 3.f), sy = __fmul_rn(s[3 * G + 1], 3.f), sz = __fmul_rn(s[3 * G + 2], 3.f);
	const float px = xyz[3 * G], py = xyz[3 * G + 1], pz = xyz[3 * G + 2];
	// torch.max(dim) propagates NaN
	float m = sx;
	if (sy > m || isnan(sy)) m = isnan(m) ? m : sy;
	if (sz > m || isnan(sz)) m = isnan(m) ? m : sz;
#pragma unroll
	for (int k = 0; k < 8; k++) {   // trimesh.creation.box() corner order: k = 4 bx + 2 by + bz, coordinate 2 b - 1
		const float vx = (k & 4) ? sx : -sx, vy = (k & 2) ? sy : -sy, vz = (k & 1) ? sz : -sz;
		const int64_t o = 3 * (8 * G + k);
		pts[o] = R[0][0] * vx + R[0][1] * vy + R[0][2] * vz + px;
		pts[o + 1] = R[1][0] * vx + R[1][1] * vy + R[1][2] * vz + py;
		pts[o + 2] = R[2][0] * vx + R[2][1] * vy + R[2][2] * vz + pz;
		scl[8 * G + k] = m;
	}
	const int64_t c = 8 * (int64_t)P + G;
	pts[3 * c] = px;
	pts[3 * c + 1] = py;
	pts[3 * c + 2] = pz;
	scl[c] = m;
}

// ---- cull SDF (mesh_extract_tetrahedra.py:32-56) ------------------------------------------------------------------------

__device__ __forceinline__ float mask_at(const float* __restrict__ r7, const float* __restrict__ gt, int H, int W, float xf, float yf) {
	if (!(xf >= 0.f && xf <= (float)(W - 1) && yf >= 0.f && yf <= (float)(H - 1))) return 0.f;
	const int64_t o = (int64_t)yf * W + (int64_t)xf;
	return gt ? __fmul_rn(r7[o], gt[o]) : r7[o];
}

__global__ void __launch_bounds__(256) tetra_cull_add_kernel(int64_t N, const float* __restrict__ alpha, const float* __restrict__ coord, int H, int W,
                                                             const float* __restrict__ r7, const float* __restrict__ gt, float* __restrict__ fin,
                                                             int32_t* __restrict__ weight) {
	const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
	if (i >= N) return;
	const float gx = __fsub_rn(__fdiv_rn(__fadd_rn(__fmul_rn(coord[2 * i], 2.f), 1.f), (float)(W - 1)), 1.f);
	const float gy = __fsub_rn(__fdiv_rn(__fadd_rn(__fmul_rn(coord[2 * i + 1], 2.f), 1.f), (float)(H - 1)), 1.f);
	const float ix = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), (float)W), 1.f), 0.5f);
	const float iy = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), (float)H), 1.f), 0.5f);
	const float x0 = floorf(ix), y0 = floorf(iy);
	const float wx = __fsub_rn(ix, x0), ex = __fsub_rn(1.f, wx), wy = __fsub_rn(iy, y0), ey = __fsub_rn(1.f, wy);
	const float x1 = __fadd_rn(x0, 1.f), y1 = __fadd_rn(y0, 1.f);
	float v = __fmul_rn(__fmul_rn(ey, ex), mask_at(r7, gt, H, W, x0, y0));
	v = __fadd_rn(v, __fmul_rn(__fmul_rn(ey, wx), mask_at(r7, gt, H, W, x1, y0)));
	v = __fadd_rn(v, __fmul_rn(__fmul_rn(wy, ex), mask_at(r7, gt, H, W, x0, y1)));
	v = __fadd_rn(v, __fmul_rn(__fmul_rn(wy, wx), mask_at(r7, gt, H, W, x1, y1)));
	if (v > 0.5f) {
		const float a = alpha[i], f = fin[i];
		fin[i] = isnan(a) ? a : (isnan(f) ? f : (f < a ? f : a));
		weight[i] += 1;
	}
}

__global__ void __launch_bounds__(256) tetra_cull_finish_kernel(int64_t N, const float* __restrict__ fin, const int32_t* __restrict__ weight,
                                                                float* __restrict__ sdf) {
	const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
	if (i >= N) return;
	sdf[i] = weight[i] > 0 ? __fsub_rn(0.5f, fin[i]) : -100.f;
}

// ---- marching tetrahedra (utils/tetmesh.py) -----------------------------------------------------------------------------

// code[t] = occupancy bits (vertex k -> bit k) when 1..3 vertices have sdf > 0, else 0; valid[t] = code != 0
__global__ void __launch_bounds__(256) tetra_code_kernel(int64_t T, int64_t N, const int64_t* __restrict__ tets, const float* __restrict__ sdf,
                                                         uint8_t* __restrict__ code, uint8_t* __restrict__ valid, int32_t* __restrict__ bad) {
	const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
	if (t >= T) return;
	int c = 0;
	bool ok = true;
#pragma unroll
	for (int k = 0; k < 4; k++) {
		const int64_t v = tets[4 * t + k];
		if (v < 0 || v >= N) {
			ok = false;
			continue;
		}
		c |= (sdf[v] > 0.f) << k;
	}
	if (!ok) {
		atomicOr(bad, 1);
		c = 0;
	}
	if (c == 15) c = 0;
	code[t] = (uint8_t)c;
	valid[t] = c != 0;
}

__global__ void __launch_bounds__(256) tetra_edge_key_kernel(int V, const int32_t* __restrict__ ids, const int64_t* __restrict__ tets, int nb,
                                                             uint64_t* __restrict__ keys, int32_t* __restrict__ pos) {
	const int j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= 6 * V) return;
	const int v = j / 6, e = j - 6 * v;
	const int64_t t = ids[v];
	const uint64_t a = (uint64_t)tets[4 * t + c_tet_edges[e][0]], b = (uint64_t)tets[4 * t + c_tet_edges[e][1]];
	keys[j] = a < b ? (a << nb | b) : (b << nb | a);
	pos[j] = j;
}

// cross_head[j] = 1 iff sorted key j starts a run and its edge crosses (exactly one endpoint has sdf > 0)
__device__ __forceinline__ bool crosses(uint64_t key, int nb, const float* __restrict__ sdf) {
	const int64_t a = (int64_t)(key >> nb), b = (int64_t)(key & ((1ull << nb) - 1));
	return (sdf[a] > 0.f) != (sdf[b] > 0.f);
}

__global__ void __launch_bounds__(256) tetra_cross_head_kernel(int E, const uint64_t* __restrict__ keys, int nb, const float* __restrict__ sdf,
                                                               int32_t* __restrict__ head) {
	const int j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= E) return;
	head[j] = (j == 0 || keys[j] != keys[j - 1]) && crosses(keys[j], nb, sdf);
}

// idx_map[pos] = vertex of the edge (the rank of its crossing run), -1 for a non-crossing edge; the vertices from the heads
__global__ void __launch_bounds__(256) tetra_vertex_kernel(int E, const uint64_t* __restrict__ keys, const int32_t* __restrict__ pos, int nb,
                                                           const int32_t* __restrict__ head, const int32_t* __restrict__ incl, const float* __restrict__ pts,
                                                           const float* __restrict__ sdf, const float* __restrict__ scl, int32_t* __restrict__ idx_map,
                                                           int64_t* __restrict__ interp, float* __restrict__ ends, float* __restrict__ end_sdf,
                                                           float* __restrict__ end_scl) {
	const int j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= E) return;
	const uint64_t key = keys[j];
	idx_map[pos[j]] = crosses(key, nb, sdf) ? incl[j] - 1 : -1;
	if (!head[j]) return;
	const int64_t m = incl[j] - 1;
	const int64_t ab[2] = {(int64_t)(key >> nb), (int64_t)(key & ((1ull << nb) - 1))};
#pragma unroll
	for (int s = 0; s < 2; s++) {
		const int64_t a = ab[s];
		interp[2 * m + s] = a;
		ends[6 * m + 3 * s] = pts[3 * a];
		ends[6 * m + 3 * s + 1] = pts[3 * a + 1];
		ends[6 * m + 3 * s + 2] = pts[3 * a + 2];
		end_sdf[2 * m + s] = sdf[a];
		end_scl[2 * m + s] = scl[a];
	}
}

// face group of valid tet v: chunk * 2 + (two triangles); ntri[v] its triangle count
__global__ void __launch_bounds__(256) tetra_group_kernel(int V, const int32_t* __restrict__ ids, const uint8_t* __restrict__ code, int64_t chunk_len,
                                                          uint32_t* __restrict__ group, int32_t* __restrict__ vid) {
	const int v = blockIdx.x * blockDim.x + threadIdx.x;
	if (v >= V) return;
	const int64_t t = ids[v];
	group[v] = (uint32_t)(2 * (t / chunk_len) + (num_triangles(code[t]) == 2));
	vid[v] = v;
}

__global__ void __launch_bounds__(256) tetra_ntri_kernel(int V, const int32_t* __restrict__ vid_sorted, const int32_t* __restrict__ ids,
                                                         const uint8_t* __restrict__ code, int32_t* __restrict__ ntri) {
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= V) return;
	ntri[k] = num_triangles(code[ids[vid_sorted[k]]]);
}

__global__ void __launch_bounds__(256) tetra_face_kernel(int V, const int32_t* __restrict__ vid_sorted, const int32_t* __restrict__ ids,
                                                         const uint8_t* __restrict__ code, const int32_t* __restrict__ face_off,
                                                         const int32_t* __restrict__ idx_map, int64_t* __restrict__ faces) {
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= V) return;
	const int v = vid_sorted[k];
	const int c = code[ids[v]];
	const int n = 3 * num_triangles(c);
	const int64_t f = face_off[k];
	for (int q = 0; q < n; q++) faces[3 * f + q] = idx_map[6 * (int64_t)v + c_tri_table[c][q]];
}

// ---- bisection (mesh_extract_tetrahedra.py:90-102) ----------------------------------------------------------------------

__global__ void __launch_bounds__(256) tetra_bisect_kernel(int64_t M, const float* __restrict__ mid_sdf, float* __restrict__ left, float* __restrict__ right,
                                                           float* __restrict__ lsdf, float* __restrict__ rsdf, float* __restrict__ mid) {
	const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
	if (i >= M) return;
	float l[3], r[3];
#pragma unroll
	for (int a = 0; a < 3; a++) {
		l[a] = left[3 * i + a];
		r[a] = right[3 * i + a];
	}
	if (mid_sdf) {
		const float m = mid_sdf[i], ls = lsdf[i];
		const bool low = (m < 0.f && ls < 0.f) || (m > 0.f && ls > 0.f);
#pragma unroll
		for (int a = 0; a < 3; a++) {
			const float c = __fmul_rn(__fadd_rn(l[a], r[a]), 0.5f);
			if (low) l[a] = c;
			else r[a] = c;
		}
		if (low) {
			lsdf[i] = m;
#pragma unroll
			for (int a = 0; a < 3; a++) left[3 * i + a] = l[a];
		} else {
			rsdf[i] = m;
#pragma unroll
			for (int a = 0; a < 3; a++) right[3 * i + a] = r[a];
		}
	}
#pragma unroll
	for (int a = 0; a < 3; a++) mid[3 * i + a] = __fmul_rn(__fadd_rn(l[a], r[a]), 0.5f);
}

// ---- filter (mesh_extract_tetrahedra.py:105-112) ------------------------------------------------------------------------

__global__ void __launch_bounds__(256) tetra_keep_kernel(int M, const float* __restrict__ ends, const float* __restrict__ end_scl, int32_t* __restrict__ keep) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= M) return;
	const int64_t o = 6 * (int64_t)i;
	const float dx = __fsub_rn(ends[o], ends[o + 3]), dy = __fsub_rn(ends[o + 1], ends[o + 4]), dz = __fsub_rn(ends[o + 2], ends[o + 5]);
	const float d = __fsqrt_rn(__fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx))));   // torch.norm's order
	keep[i] = d <= __fadd_rn(end_scl[2 * (int64_t)i], end_scl[2 * (int64_t)i + 1]);
}

struct Tri {
	int64_t v[3];
};

__global__ void __launch_bounds__(256) tetra_face_keep_kernel(int64_t F, const int64_t* __restrict__ faces, const int32_t* __restrict__ keep,
                                                              const int32_t* __restrict__ excl, int M, Tri* __restrict__ remapped, uint8_t* __restrict__ fkeep,
                                                              int32_t* __restrict__ bad) {
	const int64_t f = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
	if (f >= F) return;
	Tri t;
	bool all = true;
#pragma unroll
	for (int q = 0; q < 3; q++) {
		const int64_t v = faces[3 * f + q];
		if (v < 0 || v >= M) {
			atomicOr(bad, 1);
			all = false;
			t.v[q] = -1;
			continue;
		}
		all = all && keep[v];
		t.v[q] = excl[v];
	}
	remapped[f] = t;
	fkeep[f] = all;
}

struct P3f {
	float x, y, z;
};

int bits_for(int64_t n) {   // bits to hold every value in [0, n)
	int b = 1;
	while (b < 63 && (1ll << b) < n) b++;
	return b;
}

// ---- launchers ----------------------------------------------------------------------------------------------------------

// Phase 1 (sized by T): codes, valid flags, the valid tet ids and the select's temp.
struct TetScratch1 {
	uint8_t* code;
	uint8_t* valid;
	int32_t* ids;
	int32_t* counters;   // [0] bad index flag, [1] valid tets
	void* temp;
	size_t temp_bytes;
};

static TetScratch1 carve1(Carver& c, int64_t T) {
	TetScratch1 k;
	k.code = c.take<uint8_t>(T);
	k.valid = c.take<uint8_t>(T);
	k.ids = c.take<int32_t>(T);
	k.counters = c.take<int32_t>(2);
	k.temp_bytes = 0;
	cub::DeviceSelect::Flagged(nullptr, k.temp_bytes, thrust::counting_iterator<int32_t>(0), (const uint8_t*)nullptr, (int32_t*)nullptr, (int32_t*)nullptr,
	                           (int)T);
	k.temp = c.take<char>(k.temp_bytes);
	return k;
}

size_t tetra_march_scratch1_bytes(int64_t T) {
	Carver c(nullptr);
	carve1(c, T);
	return c.size();
}

// Phase 2 (sized by the valid tets V): E = 6 V edge keys.
struct TetScratch2 {
	uint64_t *keys_in, *keys_out;
	int32_t *pos_in, *pos_out, *head, *incl, *idx_map;
	uint32_t *group_in, *group_out;
	int32_t *vid_in, *vid_out, *ntri, *face_off;
	void* temp;
	size_t temp_bytes;
};

static TetScratch2 carve2(Carver& c, int V) {
	const int E = 6 * V;
	size_t a = 0, b = 0, c2 = 0, d = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, a, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr, E);
	cub::DeviceScan::InclusiveSum(nullptr, b, (const int32_t*)nullptr, (int32_t*)nullptr, E);
	cub::DeviceRadixSort::SortPairs(nullptr, c2, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr, V);
	cub::DeviceScan::ExclusiveSum(nullptr, d, (const int32_t*)nullptr, (int32_t*)nullptr, V);
	TetScratch2 k;
	k.keys_in = c.take<uint64_t>(E);
	k.keys_out = c.take<uint64_t>(E);
	k.pos_in = c.take<int32_t>(E);
	k.pos_out = c.take<int32_t>(E);
	k.head = c.take<int32_t>(E);
	k.incl = c.take<int32_t>(E);
	k.idx_map = c.take<int32_t>(E);
	k.group_in = c.take<uint32_t>(V);
	k.group_out = c.take<uint32_t>(V);
	k.vid_in = c.take<int32_t>(V);
	k.vid_out = c.take<int32_t>(V);
	k.ntri = c.take<int32_t>(V);
	k.face_off = c.take<int32_t>(V);
	k.temp_bytes = std::max(std::max(a, b), std::max(c2, d));
	k.temp = c.take<char>(k.temp_bytes);
	return k;
}

size_t tetra_march_scratch2_bytes(int V) {
	Carver c(nullptr);
	carve2(c, V);
	return c.size();
}

cudaError_t launch_tetra_march_valid(int64_t T, int64_t N, const int64_t* tets, const float* sdf, char* scratch1, int32_t* bad, int32_t* num_valid,
                                     cudaStream_t s) {
	Carver c(scratch1);
	TetScratch1 k = carve1(c, T);
	RGS_TRY(cudaMemsetAsync(k.counters, 0, 2 * sizeof(int32_t), s));
	tetra_code_kernel<<<(unsigned)((T + 255) / 256), 256, 0, s>>>(T, N, tets, sdf, k.code, k.valid, k.counters);
	size_t temp = k.temp_bytes;
	RGS_TRY(cub::DeviceSelect::Flagged(k.temp, temp, thrust::counting_iterator<int32_t>(0), k.valid, k.ids, k.counters + 1, (int)T, s));
	count_launch(2);
	int32_t h[2];
	RGS_TRY(cudaMemcpyAsync(h, k.counters, sizeof(h), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaStreamSynchronize(s));
	*bad = h[0];
	*num_valid = h[1];
	return cudaGetLastError();
}

cudaError_t launch_tetra_march_sort(int64_t T, int64_t N, const int64_t* tets, const float* sdf, int V, const char* scratch1, char* scratch2,
                                    int32_t* num_vertices, int32_t* num_faces, cudaStream_t s) {
	Carver c1(const_cast<char*>(scratch1)), c2(scratch2);
	TetScratch1 k1 = carve1(c1, T);
	TetScratch2 k = carve2(c2, V);
	const int E = 6 * V, nb = bits_for(N);
	tetra_edge_key_kernel<<<(unsigned)((E + 255) / 256), 256, 0, s>>>(V, k1.ids, tets, nb, k.keys_in, k.pos_in);
	size_t temp = k.temp_bytes;
	RGS_TRY(cub::DeviceRadixSort::SortPairs(k.temp, temp, k.keys_in, k.keys_out, k.pos_in, k.pos_out, E, 0, 2 * nb, s));
	tetra_cross_head_kernel<<<(unsigned)((E + 255) / 256), 256, 0, s>>>(E, k.keys_out, nb, sdf, k.head);
	temp = k.temp_bytes;
	RGS_TRY(cub::DeviceScan::InclusiveSum(k.temp, temp, k.head, k.incl, E, s));
	// torch.chunk(tets, T // CHUNK + 1) when T > CHUNK: chunks of ceil(T / n) tets
	const int64_t n_chunks = T > CHUNK ? T / CHUNK + 1 : 1;
	const int64_t chunk_len = std::max<int64_t>(1, (T + n_chunks - 1) / n_chunks);
	const int64_t groups = 2 * ((T + chunk_len - 1) / chunk_len);
	tetra_group_kernel<<<(unsigned)((V + 255) / 256), 256, 0, s>>>(V, k1.ids, k1.code, chunk_len, k.group_in, k.vid_in);
	temp = k.temp_bytes;
	RGS_TRY(cub::DeviceRadixSort::SortPairs(k.temp, temp, k.group_in, k.group_out, k.vid_in, k.vid_out, V, 0, bits_for(groups), s));
	tetra_ntri_kernel<<<(unsigned)((V + 255) / 256), 256, 0, s>>>(V, k.vid_out, k1.ids, k1.code, k.ntri);
	temp = k.temp_bytes;
	RGS_TRY(cub::DeviceScan::ExclusiveSum(k.temp, temp, k.ntri, k.face_off, V, s));
	count_launch(7);
	int32_t h[3];
	RGS_TRY(cudaMemcpyAsync(h, k.incl + (E - 1), sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaMemcpyAsync(h + 1, k.face_off + (V - 1), sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaMemcpyAsync(h + 2, k.ntri + (V - 1), sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaStreamSynchronize(s));
	*num_vertices = h[0];
	*num_faces = h[1] + h[2];
	return cudaGetLastError();
}

cudaError_t launch_tetra_march_emit(int64_t T, const float* points, const float* sdf, const float* scales, int V, const char* scratch1, char* scratch2,
                                    int64_t N, int64_t* interp, float* ends, float* end_sdf, float* end_scl, int64_t* faces, cudaStream_t s) {
	Carver c1(const_cast<char*>(scratch1)), c2(scratch2);
	TetScratch1 k1 = carve1(c1, T);
	TetScratch2 k = carve2(c2, V);
	const int E = 6 * V, nb = bits_for(N);
	tetra_vertex_kernel<<<(unsigned)((E + 255) / 256), 256, 0, s>>>(E, k.keys_out, k.pos_out, nb, k.head, k.incl, points, sdf, scales, k.idx_map, interp,
	                                                                 ends, end_sdf, end_scl);
	tetra_face_kernel<<<(unsigned)((V + 255) / 256), 256, 0, s>>>(V, k.vid_out, k1.ids, k1.code, k.face_off, k.idx_map, faces);
	count_launch(2);
	return cudaGetLastError();
}

struct FilterScratch {
	int32_t *keep, *excl;
	uint8_t* fkeep;
	Tri* remapped;
	int32_t* count32;   // [0] kept vertices (written by the vertex select), [1] bad face index flag
	int64_t* count64;   // kept faces (written by the face select)
	void* temp;
	size_t temp_bytes;
};

static FilterScratch carve_filter(Carver& c, int M, int64_t F) {
	size_t a = 0, b = 0, c2 = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, a, (const int32_t*)nullptr, (int32_t*)nullptr, M);
	cub::DeviceSelect::Flagged(nullptr, b, (const P3f*)nullptr, (const int32_t*)nullptr, (P3f*)nullptr, (int32_t*)nullptr, M);
	cub::DeviceSelect::Flagged(nullptr, c2, (const Tri*)nullptr, (const uint8_t*)nullptr, (Tri*)nullptr, (int64_t*)nullptr, F);
	FilterScratch k;
	k.keep = c.take<int32_t>(M);
	k.excl = c.take<int32_t>(M);
	k.fkeep = c.take<uint8_t>(F);
	k.remapped = c.take<Tri>(F);
	k.count32 = c.take<int32_t>(2);
	k.count64 = c.take<int64_t>(1);
	k.temp_bytes = std::max(a, std::max(b, c2));
	k.temp = c.take<char>(k.temp_bytes);
	return k;
}

size_t tetra_filter_scratch_bytes(int M, int64_t F) {
	Carver c(nullptr);
	carve_filter(c, M, F);
	return c.size();
}

cudaError_t launch_tetra_filter(int M, const float* points, const float* ends, const float* end_scl, int64_t F, const int64_t* faces, char* scratch,
                                float* out_vertices, int64_t* out_faces, int64_t* num_vertices, int64_t* num_faces, int32_t* bad, cudaStream_t s) {
	Carver c(scratch);
	FilterScratch k = carve_filter(c, M, F);
	RGS_TRY(cudaMemsetAsync(k.count32, 0, 2 * sizeof(int32_t), s));
	tetra_keep_kernel<<<(unsigned)((M + 255) / 256), 256, 0, s>>>(M, ends, end_scl, k.keep);
	size_t temp = k.temp_bytes;
	RGS_TRY(cub::DeviceScan::ExclusiveSum(k.temp, temp, k.keep, k.excl, M, s));
	temp = k.temp_bytes;
	RGS_TRY(cub::DeviceSelect::Flagged(k.temp, temp, reinterpret_cast<const P3f*>(points), k.keep, reinterpret_cast<P3f*>(out_vertices), k.count32, M, s));
	int64_t h[2] = {0, 0};
	if (F > 0) {
		tetra_face_keep_kernel<<<(unsigned)((F + 255) / 256), 256, 0, s>>>(F, faces, k.keep, k.excl, M, k.remapped, k.fkeep, k.count32 + 1);
		temp = k.temp_bytes;
		RGS_TRY(cub::DeviceSelect::Flagged(k.temp, temp, k.remapped, k.fkeep, reinterpret_cast<Tri*>(out_faces), k.count64, F, s));
		count_launch(2);
		RGS_TRY(cudaMemcpyAsync(h + 1, k.count64, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
	}
	count_launch(3);
	int32_t h32[2];
	RGS_TRY(cudaMemcpyAsync(h32, k.count32, sizeof(h32), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaStreamSynchronize(s));
	*num_vertices = h32[0];
	*bad = h32[1];
	*num_faces = h[1];
	return cudaGetLastError();
}

}  // namespace
}  // namespace rgs

using namespace rgs;

extern "C" {

int32_t rgs_tetra_points(int64_t P, const float* xyz, const float* scaling, const float* rotation, float* points, float* scales, void* cuda_stream) {
	if (P < 0 || 9 * P > INT32_MAX) return fail(RGS_E_INVALID, "tetra points: Gaussian count out of range");
	if (P == 0) return RGS_OK;
	if (!xyz || !scaling || !rotation || !points || !scales) return fail(RGS_E_INVALID, "null pointer");
	tetra_points_kernel<<<(unsigned)((P + 255) / 256), 256, 0, (cudaStream_t)cuda_stream>>>((int)P, xyz, scaling, rotation, points, scales);
	count_launch();
	return cuda_status(cudaGetLastError(), "tetra points");
}

int32_t rgs_tetra_cull_add(int64_t N, const float* alpha, const float* coord, int32_t H, int32_t W, const float* render7, const float* gt_mask,
                           float* final_alpha, int32_t* weight, void* cuda_stream) {
	if (N < 0 || H <= 0 || W <= 0) return fail(RGS_E_INVALID, "tetra cull: negative point count or empty image");
	if (N == 0) return RGS_OK;
	if (!alpha || !coord || !render7 || !final_alpha || !weight) return fail(RGS_E_INVALID, "null pointer");
	tetra_cull_add_kernel<<<(unsigned)((N + 255) / 256), 256, 0, (cudaStream_t)cuda_stream>>>(N, alpha, coord, H, W, render7, gt_mask, final_alpha, weight);
	count_launch();
	return cuda_status(cudaGetLastError(), "tetra cull");
}

int32_t rgs_tetra_cull_finish(int64_t N, const float* final_alpha, const int32_t* weight, float* sdf, void* cuda_stream) {
	if (N < 0) return fail(RGS_E_INVALID, "tetra cull: negative point count");
	if (N == 0) return RGS_OK;
	if (!final_alpha || !weight || !sdf) return fail(RGS_E_INVALID, "null pointer");
	tetra_cull_finish_kernel<<<(unsigned)((N + 255) / 256), 256, 0, (cudaStream_t)cuda_stream>>>(N, final_alpha, weight, sdf);
	count_launch();
	return cuda_status(cudaGetLastError(), "tetra cull finish");
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
	tetra_bisect_kernel<<<(unsigned)((M + 255) / 256), 256, 0, (cudaStream_t)cuda_stream>>>(M, mid_sdf, left, right, left_sdf, right_sdf, mid);
	count_launch();
	return cuda_status(cudaGetLastError(), "tetra bisect");
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

}  // extern "C"

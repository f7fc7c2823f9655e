// rgs_tsdf.cu -- TSDF fusion and marching cubes on a sparse voxel-block grid: the mesh step of the reference's DTU path
// (mesh_extract.py:66-105, there Open3D's VoxelBlockGrid on the CPU).  Runs once per trained model, off the rasterizer path.
//
// The contract (include/rgs_b200.h, rgs_tsdf_*) fixes every stored bit: each arithmetic step is one intrinsic rounded on
// its own (__fmul_rn / __fadd_rn / __fsub_rn / __fdiv_rn, IEEE sqrt), so nvcc cannot contract to FMA and a numpy fp32
// restatement reproduces the grid and the mesh.
//   touch      one thread per pixel; the blocks of its truncation band go into a frame-local hash (open addressing,
//              atomicCAS), new keys are appended to a list; one host read of the counters; CUB radix sort of the list.
//   integrate  insert (one thread per coordinate, atomicCAS + a device allocation counter), claim (each block is updated by
//              the one coordinate that swapped in this call's id), then one CTA per block over its 16^3 voxels with SoA
//              pools, so a warp reads and writes 32 consecutive tsdf / weight values.
//   extract    active blocks gathered and radix-sorted by key, a 27-entry neighbour table per block, then per voxel:
//              state (valid, inside) -> cell (all 8 corners valid, case) -> counts (owned vertices, triangles) -> two CUB
//              exclusive scans -> emit.  Sorting and scanning in (block key, voxel) order makes the mesh independent of pool
//              order and grid capacity.
//   normals    (vertex, triangle) pairs stably radix-sorted by vertex, so every vertex sums its face normals in ascending
//              triangle order: no float atomics.
//   scalable   the bounded TSDF of the reference's GaussianExtractor (Open3D's legacy ScalableTSDFVolume, RGB8) on the same
//              grid: an RGBD kernel (numpy's uint8 wrap, mask, depth_trunc), a touch over every 4th pixel, and an integrate
//              kernel at voxel centres with the ray-distance SDF, after the same insert and claim; rgs_tsdf_extract as is.
//              Also the 8-bit conversion of the image export.
//
// This file also holds the C-ABI entry points rgs_tsdf_* (include/rgs_b200.h).
#include <cub/cub.cuh>

#include "rgs_common.cuh"
#include "rgs_mcubes.cuh"

namespace rgs {

namespace {

constexpr int RES = RGS_TSDF_BLOCK_RES;
constexpr int BV = RES * RES * RES;          // voxels per block
constexpr int BIAS = 1 << 20;                // 21 signed bits per axis
constexpr int KEY_LO = -BIAS + 1, KEY_HI = BIAS - 2;  // blocks a camera may reach (one block of margin either side)
constexpr uint64_t EMPTY = RGS_TSDF_EMPTY_KEY;

// ---- keys and the block hash -------------------------------------------------------------------------------------------

__host__ __device__ inline bool key_range(long long b) { return b >= -BIAS && b < BIAS; }
__host__ __device__ inline uint64_t pack_key(int bx, int by, int bz) {
	return (uint64_t)(bx + BIAS) << 42 | (uint64_t)(by + BIAS) << 21 | (uint64_t)(bz + BIAS);
}
__device__ inline int3 unpack_key(uint64_t k) {
	const int m = (1 << 21) - 1;
	return make_int3((int)(k >> 42 & m) - BIAS, (int)(k >> 21 & m) - BIAS, (int)(k & m) - BIAS);
}
__device__ inline uint64_t slot_of(uint64_t key, uint64_t mask) {
	uint64_t h = key * 0x9E3779B97F4A7C15ull;
	return (h ^ (h >> 31)) & mask;
}
// slot holding `key` after the call (fresh: this thread put it there), or -1 when every slot is taken
__device__ long long hash_insert(uint64_t* keys, uint64_t mask, uint64_t key, bool& fresh) {
	uint64_t s = slot_of(key, mask);
	for (uint64_t p = 0; p <= mask; p++, s = (s + 1) & mask) {
		const uint64_t prev = atomicCAS(reinterpret_cast<unsigned long long*>(keys + s), (unsigned long long)EMPTY, (unsigned long long)key);
		if (prev == EMPTY || prev == key) {
			fresh = prev == EMPTY;
			return (long long)s;
		}
	}
	return -1;
}
__device__ long long hash_find(const uint64_t* keys, uint64_t mask, uint64_t key) {
	uint64_t s = slot_of(key, mask);
	for (uint64_t p = 0; p <= mask; p++, s = (s + 1) & mask) {
		const uint64_t k = keys[s];
		if (k == key) return (long long)s;
		if (k == EMPTY) return -1;
	}
	return -1;
}

struct Cam {
	int W, H;
	float fx, fy, cx, cy, R[9], t[3], depth_scale, depth_max, trunc, vs, bs;
};

// ---- touch ------------------------------------------------------------------------------------------------------------

// the box of blocks [lo, hi] into the frame-local hash; new keys appended to the list
__device__ inline void touch_box(const float lo[3], const float hi[3], uint64_t* __restrict__ fkeys, uint64_t fmask, uint64_t* __restrict__ flist,
                                 int64_t fcap, int32_t* __restrict__ counters) {
	for (int k = 0; k < 3; k++)
		if (!(lo[k] >= (float)KEY_LO && hi[k] <= (float)KEY_HI)) return;  // also rejects NaN
	for (int bz = (int)lo[2]; bz <= (int)hi[2]; bz++)
		for (int by = (int)lo[1]; by <= (int)hi[1]; by++)
			for (int bx = (int)lo[0]; bx <= (int)hi[0]; bx++) {
				const uint64_t key = pack_key(bx, by, bz);
				bool fresh = false;
				if (hash_insert(fkeys, fmask, key, fresh) < 0) {
					atomicOr(counters + 3, 1);  // frame hash full
					return;
				}
				if (fresh) {
					const int n = atomicAdd(counters + 1, 1);
					if (n < fcap) flist[n] = key;
				}
			}
}

__global__ void __launch_bounds__(256) tsdf_touch_kernel(Cam c, const float* __restrict__ depth, uint64_t* __restrict__ fkeys, uint64_t fmask,
                                                         uint64_t* __restrict__ flist, int64_t fcap, int32_t* __restrict__ counters) {
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= (int64_t)c.W * c.H) return;
	const int px = (int)(i % c.W), py = (int)(i / c.W);
	const float d = __fdiv_rn(depth[i], c.depth_scale);
	if (!(d > 0.0f && d <= c.depth_max)) return;
	const float xn = __fdiv_rn(__fsub_rn(__fadd_rn((float)px, 0.5f), c.cx), c.fx);
	const float yn = __fdiv_rn(__fsub_rn(__fadd_rn((float)py, 0.5f), c.cy), c.fy);
	float lo[3], hi[3];
	for (int s = 0; s < 2; s++) {
		const float z = s ? __fadd_rn(d, c.trunc) : __fsub_rn(d, c.trunc);
		const float q0 = __fsub_rn(__fmul_rn(xn, z), c.t[0]), q1 = __fsub_rn(__fmul_rn(yn, z), c.t[1]), q2 = __fsub_rn(z, c.t[2]);
		for (int k = 0; k < 3; k++) {
			const float pw = __fadd_rn(__fadd_rn(__fmul_rn(c.R[k], q0), __fmul_rn(c.R[3 + k], q1)), __fmul_rn(c.R[6 + k], q2));
			const float b = floorf(__fdiv_rn(pw, c.bs));
			lo[k] = s ? fminf(lo[k], b) : b;
			hi[k] = s ? fmaxf(hi[k], b) : b;
		}
	}
	touch_box(lo, hi, fkeys, fmask, flist, fcap, counters);
}

// ---- scalable volume (Open3D's legacy ScalableTSDFVolume with RGB8 colour) ---------------------------------------------

// numpy's float32 -> uint8 cast on x86-64: truncation to int32 (cvttss2si, which gives INT_MIN for NaN and |x| >= 2^31),
// then the low byte.  A CUDA float-to-int conversion saturates instead, so the out-of-range cases are spelled out.
__device__ inline uint8_t numpy_u8(float x) { return (x > -2147483648.0f && x < 2147483648.0f) ? (uint8_t)(int32_t)x : (uint8_t)0; }

__global__ void __launch_bounds__(256) scalable_rgbd_kernel(int64_t P, const float* __restrict__ rgb, const float* __restrict__ depth,
                                                            const float* __restrict__ mask, double depth_trunc, uint8_t* __restrict__ color,
                                                            float* __restrict__ dout) {
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
#pragma unroll
	for (int k = 0; k < 3; k++) color[3 * i + k] = numpy_u8(__fmul_rn(rgb[k * P + i], 255.0f));
	float d = depth[i];
	if (mask && mask[i] < 0.5f) d = 0.0f;
	if ((double)d >= depth_trunc) d = 0.0f;
	dout[i] = d;
}

// save_img_u8: (clip(nan_to_num(x * scale + offset), 0, 1) * 255).astype(uint8), [3, H, W] -> [H, W, 3]
__global__ void __launch_bounds__(256) scalable_image_u8_kernel(int64_t P, const float* __restrict__ img, float scale, float offset,
                                                                uint8_t* __restrict__ out) {
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
#pragma unroll
	for (int k = 0; k < 3; k++) {
		const float x = __fadd_rn(__fmul_rn(img[k * P + i], scale), offset);
		const float y = isnan(x) ? 0.0f : fminf(fmaxf(x, 0.0f), 1.0f);
		out[3 * i + k] = (uint8_t)(int32_t)__fmul_rn(y, 255.0f);
	}
}

// every 4th pixel in both axes, unprojected at its integer coordinates; the units of the box around p +- sdf_trunc
__global__ void __launch_bounds__(256) scalable_touch_kernel(Cam c, const float* __restrict__ depth, uint64_t* __restrict__ fkeys, uint64_t fmask,
                                                             uint64_t* __restrict__ flist, int64_t fcap, int32_t* __restrict__ counters) {
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	const int sw = (c.W + 3) / 4, sh = (c.H + 3) / 4;
	if (i >= (int64_t)sw * sh) return;
	const int px = 4 * (int)(i % sw), py = 4 * (int)(i / sw);
	const float d = depth[(size_t)py * c.W + px];
	if (!(d > 0.0f)) return;
	const float q0 = __fsub_rn(__fdiv_rn(__fmul_rn(__fsub_rn((float)px, c.cx), d), c.fx), c.t[0]);
	const float q1 = __fsub_rn(__fdiv_rn(__fmul_rn(__fsub_rn((float)py, c.cy), d), c.fy), c.t[1]);
	const float q2 = __fsub_rn(d, c.t[2]);
	float lo[3], hi[3];
	for (int k = 0; k < 3; k++) {
		const float pw = __fadd_rn(__fadd_rn(__fmul_rn(c.R[k], q0), __fmul_rn(c.R[3 + k], q1)), __fmul_rn(c.R[6 + k], q2));
		lo[k] = floorf(__fdiv_rn(__fsub_rn(pw, c.trunc), c.bs));
		hi[k] = floorf(__fdiv_rn(__fadd_rn(pw, c.trunc), c.bs));
	}
	touch_box(lo, hi, fkeys, fmask, flist, fcap, counters);
}

__global__ void __launch_bounds__(256) tsdf_decode_kernel(int n, const uint64_t* __restrict__ keys, int32_t* __restrict__ out) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const int3 b = unpack_key(keys[i]);
	out[3 * (size_t)i] = b.x;
	out[3 * (size_t)i + 1] = b.y;
	out[3 * (size_t)i + 2] = b.z;
}

// ---- integrate --------------------------------------------------------------------------------------------------------

__device__ inline bool coord_key(const int32_t* bc, int64_t i, uint64_t& key) {
	const int bx = bc[3 * i], by = bc[3 * i + 1], bz = bc[3 * i + 2];
	if (!key_range(bx) || !key_range(by) || !key_range(bz)) return false;
	key = pack_key(bx, by, bz);
	return true;
}

__global__ void __launch_bounds__(256) tsdf_insert_kernel(rgs_tsdf_grid g, int64_t n, const int32_t* __restrict__ bc) {
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	uint64_t key;
	if (!coord_key(bc, i, key)) {
		atomicOr(g.counters + 2, RGS_TSDF_BAD_COORD);
		return;
	}
	bool fresh = false;
	const long long s = hash_insert(g.hash_keys, (uint64_t)g.hash_slots - 1, key, fresh);
	if (s < 0) {
		atomicOr(g.counters + 2, RGS_TSDF_OVERFLOW);
		return;
	}
	if (fresh) {
		const int idx = atomicAdd(g.counters, 1);
		if (idx < g.capacity) g.hash_values[s] = idx;
		else atomicOr(g.counters + 2, RGS_TSDF_OVERFLOW);
	}
}

// the coordinate that swaps this call's id into the block's stamp updates the block; duplicates get -1
__global__ void __launch_bounds__(256) tsdf_claim_kernel(rgs_tsdf_grid g, int64_t n, const int32_t* __restrict__ bc, int32_t call_id,
                                                         int32_t* __restrict__ slot) {
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	uint64_t key;
	int32_t idx = -1;
	if (coord_key(bc, i, key)) {
		const long long s = hash_find(g.hash_keys, (uint64_t)g.hash_slots - 1, key);
		if (s >= 0) idx = g.hash_values[s];
		if (idx >= 0 && atomicExch(g.stamps + idx, call_id) == call_id) idx = -1;
	}
	slot[i] = idx;
}

constexpr int INTEGRATE_THREADS = 256;

__global__ void __launch_bounds__(INTEGRATE_THREADS) tsdf_integrate_kernel(rgs_tsdf_grid g, Cam c, const int32_t* __restrict__ bc,
                                                                           const int32_t* __restrict__ slot, const float* __restrict__ depth,
                                                                           const float* __restrict__ color) {
	const int64_t b = blockIdx.x;
	const int32_t idx = slot[b];
	if (idx < 0) return;
	const int bx = bc[3 * b], by = bc[3 * b + 1], bz = bc[3 * b + 2];
	float* __restrict__ ts = g.tsdf + (size_t)idx * BV;
	float* __restrict__ ws = g.weight + (size_t)idx * BV;
	float* __restrict__ cs = g.color + (size_t)idx * BV * 3;
	for (int v = threadIdx.x; v < BV; v += INTEGRATE_THREADS) {
		const float px = __fmul_rn((float)(bx * RES + (v & 15)), c.vs);
		const float py = __fmul_rn((float)(by * RES + (v >> 4 & 15)), c.vs);
		const float pz = __fmul_rn((float)(bz * RES + (v >> 8)), c.vs);
		const float xc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(c.R[0], px), __fmul_rn(c.R[1], py)), __fmul_rn(c.R[2], pz)), c.t[0]);
		const float yc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(c.R[3], px), __fmul_rn(c.R[4], py)), __fmul_rn(c.R[5], pz)), c.t[1]);
		const float zc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(c.R[6], px), __fmul_rn(c.R[7], py)), __fmul_rn(c.R[8], pz)), c.t[2]);
		if (!(zc > 0.0f)) continue;
		const float u = floorf(__fadd_rn(__fdiv_rn(__fmul_rn(c.fx, xc), zc), c.cx));
		const float w = floorf(__fadd_rn(__fdiv_rn(__fmul_rn(c.fy, yc), zc), c.cy));
		if (!(u >= 0.0f && u < (float)c.W && w >= 0.0f && w < (float)c.H)) continue;
		const size_t pix = (size_t)w * c.W + (size_t)u;
		const float d = __fdiv_rn(depth[pix], c.depth_scale);
		if (!(d > 0.0f && d <= c.depth_max)) continue;
		const float sdf = __fsub_rn(d, zc);
		if (sdf < -c.trunc) continue;
		const float obs = __fdiv_rn(fminf(sdf, c.trunc), c.trunc);
		const float w0 = ws[v], w1 = __fadd_rn(w0, 1.0f);
		ts[v] = __fdiv_rn(__fadd_rn(__fmul_rn(w0, ts[v]), obs), w1);
#pragma unroll
		for (int k = 0; k < 3; k++) cs[3 * v + k] = __fdiv_rn(__fadd_rn(__fmul_rn(w0, cs[3 * v + k]), color[3 * pix + k]), w1);
		ws[v] = w1;
	}
}

// the scalable volume's update: samples at voxel centres, the rounded projection, the SDF as a distance along the ray
__global__ void __launch_bounds__(INTEGRATE_THREADS) scalable_integrate_kernel(rgs_tsdf_grid g, Cam c, const int32_t* __restrict__ bc,
                                                                               const int32_t* __restrict__ slot, const float* __restrict__ depth,
                                                                               const uint8_t* __restrict__ color) {
	const int64_t b = blockIdx.x;
	const int32_t idx = slot[b];
	if (idx < 0) return;
	const int bx = bc[3 * b], by = bc[3 * b + 1], bz = bc[3 * b + 2];
	float* __restrict__ ts = g.tsdf + (size_t)idx * BV;
	float* __restrict__ ws = g.weight + (size_t)idx * BV;
	float* __restrict__ cs = g.color + (size_t)idx * BV * 3;
	for (int v = threadIdx.x; v < BV; v += INTEGRATE_THREADS) {
		const float px = __fmul_rn(__fadd_rn((float)(bx * RES + (v & 15)), 0.5f), c.vs);
		const float py = __fmul_rn(__fadd_rn((float)(by * RES + (v >> 4 & 15)), 0.5f), c.vs);
		const float pz = __fmul_rn(__fadd_rn((float)(bz * RES + (v >> 8)), 0.5f), c.vs);
		const float xc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(c.R[0], px), __fmul_rn(c.R[1], py)), __fmul_rn(c.R[2], pz)), c.t[0]);
		const float yc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(c.R[3], px), __fmul_rn(c.R[4], py)), __fmul_rn(c.R[5], pz)), c.t[1]);
		const float zc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(c.R[6], px), __fmul_rn(c.R[7], py)), __fmul_rn(c.R[8], pz)), c.t[2]);
		if (!(zc > 0.0f)) continue;
		const float u = floorf(__fadd_rn(__fadd_rn(__fmul_rn(__fdiv_rn(xc, zc), c.fx), c.cx), 0.5f));
		const float w = floorf(__fadd_rn(__fadd_rn(__fmul_rn(__fdiv_rn(yc, zc), c.fy), c.cy), 0.5f));
		if (!(u >= 0.0f && u < (float)c.W && w >= 0.0f && w < (float)c.H)) continue;
		const size_t pix = (size_t)w * c.W + (size_t)u;
		const float d = depth[pix];
		if (!(d > 0.0f)) continue;
		const float xn = __fdiv_rn(__fsub_rn(u, c.cx), c.fx), yn = __fdiv_rn(__fsub_rn(w, c.cy), c.fy);
		const float sdf = __fmul_rn(__fsub_rn(d, zc), __fsqrt_rn(__fadd_rn(__fadd_rn(1.0f, __fmul_rn(xn, xn)), __fmul_rn(yn, yn))));
		if (!(sdf > -c.trunc)) continue;
		const float obs = fminf(1.0f, __fdiv_rn(sdf, c.trunc));
		const float w0 = ws[v], w1 = __fadd_rn(w0, 1.0f);
		ts[v] = __fdiv_rn(__fadd_rn(__fmul_rn(w0, ts[v]), obs), w1);
#pragma unroll
		for (int k = 0; k < 3; k++) cs[3 * v + k] = __fdiv_rn(__fadd_rn(__fmul_rn(w0, cs[3 * v + k]), (float)color[3 * pix + k]), w1);
		ws[v] = w1;
	}
}

__global__ void __launch_bounds__(256) tsdf_rehash_kernel(rgs_tsdf_grid g, const uint64_t* __restrict__ old_keys, const int32_t* __restrict__ old_vals,
                                                          int64_t old_slots) {
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= old_slots || old_keys[i] == EMPTY || old_vals[i] < 0) return;
	bool fresh = false;
	const long long s = hash_insert(g.hash_keys, (uint64_t)g.hash_slots - 1, old_keys[i], fresh);
	if (s < 0) atomicOr(g.counters + 2, RGS_TSDF_OVERFLOW);
	else g.hash_values[s] = old_vals[i];
}

// ---- active blocks ----------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(256) tsdf_gather_kernel(rgs_tsdf_grid g, uint64_t* __restrict__ keys, int32_t* __restrict__ vals, int32_t* __restrict__ count,
                                                          int32_t cap) {
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= g.hash_slots) return;
	const uint64_t k = g.hash_keys[i];
	const int32_t v = g.hash_values[i];
	if (k == EMPTY || v < 0) return;
	const int n = atomicAdd(count, 1);
	if (n < cap) {
		keys[n] = k;
		vals[n] = v;
	}
}

struct ActiveScratch {
	uint64_t *keys_in, *keys_out;
	int32_t *vals_in, *vals_out, *count;
	char* sort_temp;
	size_t sort_temp_bytes;
};

ActiveScratch carve_active(Carver& cv, int N) {
	ActiveScratch a;
	a.sort_temp_bytes = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, a.sort_temp_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr,
	                                N, 0, 63);
	a.keys_in = cv.take<uint64_t>(N);
	a.keys_out = cv.take<uint64_t>(N);
	a.vals_in = cv.take<int32_t>(N);
	a.vals_out = cv.take<int32_t>(N);
	a.count = cv.take<int32_t>(1);
	a.sort_temp = cv.take<char>(a.sort_temp_bytes);
	return a;
}

cudaError_t sort_active(const rgs_tsdf_grid& g, const ActiveScratch& a, int N, cudaStream_t s) {
	cudaError_t e = cudaMemsetAsync(a.count, 0, sizeof(int32_t), s);
	if (e != cudaSuccess) return e;
	tsdf_gather_kernel<<<(unsigned)((g.hash_slots + 255) / 256), 256, 0, s>>>(g, a.keys_in, a.vals_in, a.count, N);
	count_launch();
	size_t temp = a.sort_temp_bytes;
	e = cub::DeviceRadixSort::SortPairs(a.sort_temp, temp, a.keys_in, a.keys_out, a.vals_in, a.vals_out, N, 0, 63, s);
	count_launch();
	return e;
}

// ---- marching cubes ---------------------------------------------------------------------------------------------------

// flat index (sorted block * 4096 + voxel) of the voxel at local (x, y, z) in [-1, 16] of sorted block i, or -1
__device__ inline int64_t nb_voxel(const int32_t* __restrict__ nbr, int64_t i, int x, int y, int z) {
	const int k = ((x >> 4) + 1) + 3 * ((y >> 4) + 1) + 9 * ((z >> 4) + 1);   // >> 4 of -1 is -1 (arithmetic shift)
	const int32_t j = nbr[i * 27 + k];
	return j < 0 ? -1 : (int64_t)j * BV + ((x & 15) | (y & 15) << 4 | (z & 15) << 8);
}

__global__ void __launch_bounds__(256) tsdf_neighbours_kernel(rgs_tsdf_grid g, int N, const uint64_t* __restrict__ skeys, const int32_t* __restrict__ inv,
                                                              int32_t* __restrict__ nbr) {
	const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= (int64_t)N * 27) return;
	const int64_t i = t / 27;
	const int k = (int)(t % 27);
	const int3 b = unpack_key(skeys[i]);
	const int x = b.x + k % 3 - 1, y = b.y + k / 3 % 3 - 1, z = b.z + k / 9 - 1;
	int32_t j = -1;
	if (key_range(x) && key_range(y) && key_range(z)) {
		const long long s = hash_find(g.hash_keys, (uint64_t)g.hash_slots - 1, pack_key(x, y, z));
		if (s >= 0 && g.hash_values[s] >= 0) j = inv[g.hash_values[s]];
	}
	nbr[t] = j;
}

__global__ void __launch_bounds__(256) tsdf_inverse_kernel(int N, const int32_t* __restrict__ spool, int32_t* __restrict__ inv) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < N) inv[spool[i]] = i;
}

// bit 0 valid (w >= threshold), bit 1 inside (tsdf < 0)
__global__ void __launch_bounds__(256) tsdf_state_kernel(rgs_tsdf_grid g, int64_t M, const int32_t* __restrict__ spool, float thr, uint8_t* __restrict__ st) {
	const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= M) return;
	const size_t src = (size_t)spool[t / BV] * BV + (size_t)(t % BV);
	st[t] = (uint8_t)((g.weight[src] >= thr ? 1 : 0) | (g.tsdf[src] < 0.0f ? 2 : 0));
}

// cell at voxel g: bit 8 = all corners valid, bits 0..7 = case
__global__ void __launch_bounds__(256) tsdf_cell_kernel(int64_t M, const int32_t* __restrict__ nbr, const uint8_t* __restrict__ st, uint16_t* __restrict__ cell) {
	const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= M) return;
	const int64_t i = t / BV;
	const int v = (int)(t % BV), x = v & 15, y = v >> 4 & 15, z = v >> 8;
	int cs = 0;
	bool ok = true;
#pragma unroll
	for (int c = 0; c < 8; c++) {
		const int64_t q = nb_voxel(nbr, i, x + (c & 1), y + (c >> 1 & 1), z + (c >> 2 & 1));
		const uint8_t s = q < 0 ? 0 : st[q];
		ok = ok && (s & 1);
		cs |= (s >> 1 & 1) << c;
	}
	cell[t] = (uint16_t)(ok ? 0x100 | cs : 0);
}

// owned vertices (bit a: edge (g, a) has a vertex) and triangle count of the cell at g
__global__ void __launch_bounds__(256) tsdf_count_kernel(int64_t M, const int32_t* __restrict__ nbr, const uint8_t* __restrict__ st,
                                                         const uint16_t* __restrict__ cell, uint8_t* __restrict__ vmask, int32_t* __restrict__ vcnt,
                                                         int32_t* __restrict__ tcnt) {
	const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= M) return;
	const int64_t i = t / BV;
	const int v = (int)(t % BV), p[3] = {v & 15, v >> 4 & 15, v >> 8};
	const uint16_t own = cell[t];
	tcnt[t] = (own & 0x100) ? c_tri.n[own & 0xff] : 0;
	int m = 0;
#pragma unroll
	for (int a = 0; a < 3; a++) {
		int q[3] = {p[0], p[1], p[2]};
		q[a]++;
		const int64_t j = nb_voxel(nbr, i, q[0], q[1], q[2]);
		if (j < 0 || ((st[t] ^ st[j]) & 2) == 0) continue;
		// the four cells around the edge: g minus {0,1} on the two other axes
		bool near = false;
		const int b = other_axis(a, 0), c = other_axis(a, 1);
		for (int o = 0; o < 4 && !near; o++) {
			int r[3] = {p[0], p[1], p[2]};
			r[b] -= o & 1;
			r[c] -= o >> 1;
			const int64_t k = nb_voxel(nbr, i, r[0], r[1], r[2]);
			near = k >= 0 && (cell[k] & 0x100);
		}
		if (near) m |= 1 << a;
	}
	vmask[t] = (uint8_t)m;
	vcnt[t] = __popc(m);
}

struct MeshPtrs {
	float *verts, *colors;
	int32_t* tris;
};

__global__ void __launch_bounds__(256) tsdf_emit_kernel(rgs_tsdf_grid g, int64_t M, float vs, const uint64_t* __restrict__ skeys, const int32_t* __restrict__ spool,
                                                        const int32_t* __restrict__ nbr, const uint16_t* __restrict__ cell, const uint8_t* __restrict__ vmask,
                                                        const int32_t* __restrict__ voff, const int32_t* __restrict__ toff, MeshPtrs out) {
	const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= M) return;
	const int64_t i = t / BV;
	const int v = (int)(t % BV), p[3] = {v & 15, v >> 4 & 15, v >> 8};
	const int m = vmask[t];
	if (m) {
		const int3 b = unpack_key(skeys[i]);
		const int gp[3] = {b.x * RES + p[0], b.y * RES + p[1], b.z * RES + p[2]};
		const size_t s0 = (size_t)spool[i] * BV + v;
		int r = voff[t];
		for (int a = 0; a < 3; a++) {
			if (!(m >> a & 1)) continue;
			int q[3] = {p[0], p[1], p[2]};
			q[a]++;
			const int64_t j = nb_voxel(nbr, i, q[0], q[1], q[2]);
			const size_t s1 = (size_t)spool[j / BV] * BV + (size_t)(j % BV);
			const float f0 = g.tsdf[s0], f1 = g.tsdf[s1];
			const float tt = __fdiv_rn(f0, __fsub_rn(f0, f1));
			float pos[3];
			for (int k = 0; k < 3; k++) pos[k] = __fmul_rn((float)gp[k], vs);
			pos[a] = __fadd_rn(pos[a], __fmul_rn(tt, vs));
			for (int k = 0; k < 3; k++) {
				out.verts[3 * (size_t)r + k] = pos[k];
				const float c0 = g.color[3 * s0 + k], c1 = g.color[3 * s1 + k];
				out.colors[3 * (size_t)r + k] = __fadd_rn(c0, __fmul_rn(tt, __fsub_rn(c1, c0)));
			}
			r++;
		}
	}
	const uint16_t own = cell[t];
	if (!(own & 0x100)) return;
	const int cs = own & 0xff, nt = c_tri.n[cs];
	int32_t* tri = out.tris + 3 * (size_t)toff[t];
	for (int k = 0; k < 3 * nt; k++) {
		const int e = c_tri.e[cs][k], a = e / 4, o = e % 4;
		int q[3] = {p[0], p[1], p[2]};
		q[other_axis(a, 0)] += o & 1;
		q[other_axis(a, 1)] += o >> 1;
		const int64_t j = nb_voxel(nbr, i, q[0], q[1], q[2]);
		tri[k] = voff[j] + __popc(vmask[j] & ((1 << a) - 1));
	}
}

// ---- vertex normals ---------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(256) tsdf_pairs_kernel(int64_t F3, const int32_t* __restrict__ tris, uint32_t* __restrict__ vk, uint32_t* __restrict__ tv) {
	const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (m >= F3) return;
	vk[m] = (uint32_t)tris[m];
	tv[m] = (uint32_t)(m / 3);
}

__global__ void __launch_bounds__(256) tsdf_ranges_kernel(int64_t F3, const uint32_t* __restrict__ vk, int32_t* __restrict__ first, int32_t* __restrict__ last) {
	const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (m >= F3) return;
	const uint32_t k = vk[m];
	if (m == 0 || vk[m - 1] != k) first[k] = (int32_t)m;
	if (m == F3 - 1 || vk[m + 1] != k) last[k] = (int32_t)(m + 1);
}

__device__ inline float3 ld3(const float* p, int64_t i) { return make_float3(p[3 * i], p[3 * i + 1], p[3 * i + 2]); }

__global__ void __launch_bounds__(256) tsdf_normals_kernel(int64_t V, const float* __restrict__ verts, const int32_t* __restrict__ tris,
                                                           const uint32_t* __restrict__ tv, const int32_t* __restrict__ first,
                                                           const int32_t* __restrict__ last, float* __restrict__ normals) {
	const int64_t vi = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (vi >= V) return;
	float nx = 0.0f, ny = 0.0f, nz = 0.0f;
	for (int m = first[vi]; m < last[vi]; m++) {
		const int64_t f = tv[m];
		const float3 v0 = ld3(verts, tris[3 * f]), v1 = ld3(verts, tris[3 * f + 1]), v2 = ld3(verts, tris[3 * f + 2]);
		const float ax = __fsub_rn(v1.x, v0.x), ay = __fsub_rn(v1.y, v0.y), az = __fsub_rn(v1.z, v0.z);
		const float bx = __fsub_rn(v2.x, v0.x), by = __fsub_rn(v2.y, v0.y), bz = __fsub_rn(v2.z, v0.z);
		nx = __fadd_rn(nx, __fsub_rn(__fmul_rn(ay, bz), __fmul_rn(az, by)));
		ny = __fadd_rn(ny, __fsub_rn(__fmul_rn(az, bx), __fmul_rn(ax, bz)));
		nz = __fadd_rn(nz, __fsub_rn(__fmul_rn(ax, by), __fmul_rn(ay, bx)));
	}
	const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(ny, ny)), __fmul_rn(nz, nz)));
	const bool zero = len == 0.0f;
	normals[3 * vi] = zero ? 0.0f : __fdiv_rn(nx, len);
	normals[3 * vi + 1] = zero ? 0.0f : __fdiv_rn(ny, len);
	normals[3 * vi + 2] = zero ? 0.0f : __fdiv_rn(nz, len);
}

unsigned blocks_for(int64_t n) { return (unsigned)((n + 255) / 256); }

// ---- host launchers ----------------------------------------------------------------------------------------------------

Cam make_cam(const rgs_tsdf_grid& g, const rgs_tsdf_camera& c) {
	Cam k;
	k.W = c.width;
	k.H = c.height;
	k.fx = c.fx;
	k.fy = c.fy;
	k.cx = c.cx;
	k.cy = c.cy;
	for (int i = 0; i < 9; i++) k.R[i] = c.R[i];
	for (int i = 0; i < 3; i++) k.t[i] = c.t[i];
	k.depth_scale = c.depth_scale;
	k.depth_max = c.depth_max;
	k.trunc = c.trunc_voxel_multiplier * g.voxel_size;  // one fp32 product, as the contract states
	k.vs = g.voxel_size;
	k.bs = g.voxel_size * (float)RES;  // exact: a power-of-two scaling
	return k;
}

size_t tsdf_touch_scratch_bytes(int64_t n) {
	size_t temp = 0;
	cub::DeviceRadixSort::SortKeys(nullptr, temp, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)n, 0, 63);
	Carver cv(nullptr);
	cv.take<uint64_t>(n);
	cv.take<char>(temp);
	return cv.size();
}

// the scalable volume's camera: trunc is the absolute sdf_trunc
Cam make_scalable_cam(const rgs_tsdf_grid& g, const rgs_tsdf_camera& c, float sdf_trunc) {
	Cam k = make_cam(g, c);
	k.trunc = sdf_trunc;
	return k;
}

// phase 1: the frame-local hash and list; counters_host receives counters[0..3] (the one host read of a view)
cudaError_t launch_tsdf_touch(const rgs_tsdf_grid& g, const Cam& k, bool scalable, const float* depth, int32_t* counters_host, cudaStream_t s) {
	RGS_TRY(cudaMemsetAsync(g.frame_keys, 0xff, (size_t)g.frame_slots * sizeof(uint64_t), s));
	RGS_TRY(cudaMemsetAsync(g.counters + 1, 0, sizeof(int32_t), s));
	RGS_TRY(cudaMemsetAsync(g.counters + 3, 0, sizeof(int32_t), s));
	if (scalable) {
		const int64_t P = (int64_t)((k.W + 3) / 4) * ((k.H + 3) / 4);
		scalable_touch_kernel<<<blocks_for(P), 256, 0, s>>>(k, depth, g.frame_keys, (uint64_t)g.frame_slots - 1, g.frame_list, g.frame_slots / 2, g.counters);
	} else {
		const int64_t P = (int64_t)k.W * k.H;
		tsdf_touch_kernel<<<blocks_for(P), 256, 0, s>>>(k, depth, g.frame_keys, (uint64_t)g.frame_slots - 1, g.frame_list, g.frame_slots / 2, g.counters);
	}
	count_launch();
	RGS_TRY(cudaGetLastError());
	RGS_TRY(cudaMemcpyAsync(counters_host, g.counters, 4 * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	return cudaStreamSynchronize(s);
}

// phase 2: the n listed keys in ascending order, decoded into out [n, 3]
cudaError_t launch_tsdf_touch_sort(const rgs_tsdf_grid& g, int64_t n, int32_t* out, char* scratch, cudaStream_t s) {
	size_t temp = 0;
	cub::DeviceRadixSort::SortKeys(nullptr, temp, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)n, 0, 63);
	Carver cv(scratch);
	uint64_t* sorted = cv.take<uint64_t>(n);
	char* tmp = cv.take<char>(temp);
	RGS_TRY(cub::DeviceRadixSort::SortKeys(tmp, temp, g.frame_list, sorted, (int)n, 0, 63, s));
	count_launch();
	tsdf_decode_kernel<<<blocks_for(n), 256, 0, s>>>((int)n, sorted, out);
	count_launch();
	return cudaGetLastError();
}

// insert the n blocks, then give each to the one coordinate that claims it in this call (slot[i], -1 for the others)
void insert_and_claim(const rgs_tsdf_grid& g, int64_t n, const int32_t* bc, int32_t call_id, int32_t* slot, cudaStream_t s) {
	tsdf_insert_kernel<<<blocks_for(n), 256, 0, s>>>(g, n, bc);
	tsdf_claim_kernel<<<blocks_for(n), 256, 0, s>>>(g, n, bc, call_id, slot);
	count_launch(2);
}

cudaError_t launch_tsdf_integrate(const rgs_tsdf_grid& g, const rgs_tsdf_camera& c, int64_t n, const int32_t* bc, const float* depth, const float* color,
                                  int32_t call_id, int32_t* slot, cudaStream_t s) {
	const Cam k = make_cam(g, c);
	insert_and_claim(g, n, bc, call_id, slot, s);
	tsdf_integrate_kernel<<<(unsigned)n, INTEGRATE_THREADS, 0, s>>>(g, k, bc, slot, depth, color);
	count_launch();
	return cudaGetLastError();
}

cudaError_t launch_scalable_integrate(const rgs_tsdf_grid& g, const Cam& k, int64_t n, const int32_t* bc, const float* depth, const uint8_t* color,
                                      int32_t call_id, int32_t* slot, cudaStream_t s) {
	insert_and_claim(g, n, bc, call_id, slot, s);
	scalable_integrate_kernel<<<(unsigned)n, INTEGRATE_THREADS, 0, s>>>(g, k, bc, slot, depth, color);
	count_launch();
	return cudaGetLastError();
}

size_t tsdf_active_scratch_bytes(int N) {
	Carver cv(nullptr);
	carve_active(cv, N);
	return cv.size();
}

cudaError_t launch_tsdf_active(const rgs_tsdf_grid& g, int N, uint64_t* keys, int32_t* pools, char* scratch, cudaStream_t s) {
	Carver cv(scratch);
	const ActiveScratch a = carve_active(cv, N);
	RGS_TRY(sort_active(g, a, N, s));
	RGS_TRY(cudaMemcpyAsync(keys, a.keys_out, (size_t)N * sizeof(uint64_t), cudaMemcpyDeviceToDevice, s));
	RGS_TRY(cudaMemcpyAsync(pools, a.vals_out, (size_t)N * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
	return cudaSuccess;
}

struct ExtractScratch {
	ActiveScratch a;
	int32_t *inv, *nbr, *vcnt, *tcnt, *voff, *toff;
	uint8_t *st, *vmask;
	uint16_t* cell;
	char* scan_temp;
	size_t scan_temp_bytes;
};

ExtractScratch carve_extract(char* base, const rgs_tsdf_grid& g, int N, size_t* total) {
	const int64_t M = (int64_t)N * BV;
	Carver cv(base);
	ExtractScratch x;
	x.a = carve_active(cv, N);
	x.scan_temp_bytes = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, x.scan_temp_bytes, (const int32_t*)nullptr, (int32_t*)nullptr, M);
	x.inv = cv.take<int32_t>(g.capacity);
	x.nbr = cv.take<int32_t>((size_t)N * 27);
	x.st = cv.take<uint8_t>(M);
	x.cell = cv.take<uint16_t>(M);
	x.vmask = cv.take<uint8_t>(M);
	x.vcnt = cv.take<int32_t>(M);
	x.tcnt = cv.take<int32_t>(M);
	x.voff = cv.take<int32_t>(M);
	x.toff = cv.take<int32_t>(M);
	x.scan_temp = cv.take<char>(x.scan_temp_bytes);
	if (total) *total = cv.size();
	return x;
}

size_t tsdf_extract_scratch_bytes(const rgs_tsdf_grid& g, int N) {
	size_t total = 0;
	carve_extract(nullptr, g, N, &total);
	return total;
}

// phase 1: everything up to the scans; totals_host receives (V, F)
cudaError_t launch_tsdf_extract_count(const rgs_tsdf_grid& g, int N, float thr, char* scratch, int64_t* totals_host, cudaStream_t s) {
	const int64_t M = (int64_t)N * BV;
	ExtractScratch x = carve_extract(scratch, g, N, nullptr);
	RGS_TRY(sort_active(g, x.a, N, s));
	tsdf_inverse_kernel<<<blocks_for(N), 256, 0, s>>>(N, x.a.vals_out, x.inv);
	tsdf_neighbours_kernel<<<blocks_for((int64_t)N * 27), 256, 0, s>>>(g, N, x.a.keys_out, x.inv, x.nbr);
	tsdf_state_kernel<<<blocks_for(M), 256, 0, s>>>(g, M, x.a.vals_out, thr, x.st);
	tsdf_cell_kernel<<<blocks_for(M), 256, 0, s>>>(M, x.nbr, x.st, x.cell);
	tsdf_count_kernel<<<blocks_for(M), 256, 0, s>>>(M, x.nbr, x.st, x.cell, x.vmask, x.vcnt, x.tcnt);
	count_launch(5);
	RGS_TRY(cudaGetLastError());
	size_t temp = x.scan_temp_bytes;
	RGS_TRY(cub::DeviceScan::ExclusiveSum(x.scan_temp, temp, x.vcnt, x.voff, M, s));
	temp = x.scan_temp_bytes;
	RGS_TRY(cub::DeviceScan::ExclusiveSum(x.scan_temp, temp, x.tcnt, x.toff, M, s));
	count_launch(2);
	int32_t tail[4];
	RGS_TRY(cudaMemcpyAsync(tail, x.voff + M - 1, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaMemcpyAsync(tail + 1, x.vcnt + M - 1, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaMemcpyAsync(tail + 2, x.toff + M - 1, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaMemcpyAsync(tail + 3, x.tcnt + M - 1, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaStreamSynchronize(s));
	totals_host[0] = (int64_t)tail[0] + tail[1];
	totals_host[1] = (int64_t)tail[2] + tail[3];
	return cudaSuccess;
}

// phase 2 on the same scratch
cudaError_t launch_tsdf_extract_emit(const rgs_tsdf_grid& g, int N, char* scratch, float* verts, float* colors, int32_t* tris, cudaStream_t s) {
	const int64_t M = (int64_t)N * BV;
	ExtractScratch x = carve_extract(scratch, g, N, nullptr);
	tsdf_emit_kernel<<<blocks_for(M), 256, 0, s>>>(g, M, g.voxel_size, x.a.keys_out, x.a.vals_out, x.nbr, x.cell, x.vmask, x.voff, x.toff,
	                                               MeshPtrs{verts, colors, tris});
	count_launch();
	return cudaGetLastError();
}

struct NormalsScratch {
	int32_t *first, *last;
	uint32_t *vk_in, *vk_out, *tv_in, *tv_out;
	char* sort_temp;
	size_t sort_temp_bytes;
};

NormalsScratch carve_normals(char* base, int64_t V, int64_t F3, size_t* total) {
	NormalsScratch x;
	x.sort_temp_bytes = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, x.sort_temp_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr,
	                                (int)F3);
	Carver cv(base);
	x.first = cv.take<int32_t>(V);
	x.last = cv.take<int32_t>(V);
	x.vk_in = cv.take<uint32_t>(F3);
	x.vk_out = cv.take<uint32_t>(F3);
	x.tv_in = cv.take<uint32_t>(F3);
	x.tv_out = cv.take<uint32_t>(F3);
	x.sort_temp = cv.take<char>(x.sort_temp_bytes);
	if (total) *total = cv.size();
	return x;
}

size_t tsdf_normals_scratch_bytes(int64_t V, int64_t F) {
	size_t total = 0;
	carve_normals(nullptr, V, 3 * F, &total);
	return total;
}

cudaError_t launch_tsdf_normals(int64_t V, const float* verts, int64_t F, const int32_t* tris, float* normals, char* scratch, cudaStream_t s) {
	const int64_t F3 = 3 * F;
	NormalsScratch x = carve_normals(scratch, V, F3, nullptr);
	RGS_TRY(cudaMemsetAsync(x.first, 0, (size_t)V * sizeof(int32_t), s));
	RGS_TRY(cudaMemsetAsync(x.last, 0, (size_t)V * sizeof(int32_t), s));
	if (F3 > 0) {
		tsdf_pairs_kernel<<<blocks_for(F3), 256, 0, s>>>(F3, tris, x.vk_in, x.tv_in);
		count_launch();
		int bits = 1;
		while (bits < 32 && ((int64_t)1 << bits) < V) bits++;
		size_t temp = x.sort_temp_bytes;
		// radix sort is stable: each vertex's entries stay in ascending triangle order
		RGS_TRY(cub::DeviceRadixSort::SortPairs(x.sort_temp, temp, x.vk_in, x.vk_out, x.tv_in, x.tv_out, (int)F3, 0, bits, s));
		count_launch();
		tsdf_ranges_kernel<<<blocks_for(F3), 256, 0, s>>>(F3, x.vk_out, x.first, x.last);
		count_launch();
	}
	tsdf_normals_kernel<<<blocks_for(V), 256, 0, s>>>(V, verts, tris, x.tv_out, x.first, x.last, normals);
	count_launch();
	return cudaGetLastError();
}

}  // namespace
}  // namespace rgs

using namespace rgs;

extern "C" {

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

// image size, intrinsics and extrinsic (the checks both volumes share)
static int tsdf_pinhole_check(const rgs_tsdf_camera* c) {
	if (!c) return fail(RGS_E_INVALID, "null camera");
	if (c->width <= 0 || c->height <= 0) return fail(RGS_E_INVALID, "image size must be positive");
	if (!std::isfinite(c->fx) || !std::isfinite(c->fy) || c->fx == 0.0f || c->fy == 0.0f || !std::isfinite(c->cx) || !std::isfinite(c->cy))
		return fail(RGS_E_INVALID, "intrinsics must be finite with nonzero focal lengths");
	for (int i = 0; i < 9; i++)
		if (!std::isfinite(c->R[i])) return fail(RGS_E_INVALID, "extrinsic must be finite");
	for (int i = 0; i < 3; i++)
		if (!std::isfinite(c->t[i])) return fail(RGS_E_INVALID, "extrinsic must be finite");
	return RGS_OK;
}

static int tsdf_camera_check(const rgs_tsdf_grid* g, const rgs_tsdf_camera* c) {
	if (const int rc = tsdf_pinhole_check(c)) return rc;
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

// the touch of either volume after its argument checks: frame hash, counters, capacity protocol, sorted decode
static int64_t tsdf_touch_run(const rgs_tsdf_grid* grid, const Cam& k, bool scalable, const float* depth, int32_t* block_coords, int64_t* allocated,
                              rgs_resize_fn scratch, void* scratch_user, cudaStream_t s) {
	int rc;
	int32_t cnt[4];
	if ((rc = cuda_status(launch_tsdf_touch(*grid, k, scalable, depth, cnt, s), "tsdf touch")) != RGS_OK) return rc;
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

int64_t rgs_tsdf_touch(const rgs_tsdf_grid* grid, const rgs_tsdf_camera* cam, const float* depth, int32_t* block_coords, int64_t* allocated,
                       rgs_resize_fn scratch, void* scratch_user, void* cuda_stream) {
	int rc = tsdf_grid_check(grid);
	if (rc == RGS_OK) rc = tsdf_camera_check(grid, cam);
	if (rc != RGS_OK) return rc;
	if (!depth || !block_coords || !scratch) return fail(RGS_E_INVALID, "null pointer");
	return tsdf_touch_run(grid, make_cam(*grid, *cam), false, depth, block_coords, allocated, scratch, scratch_user, (cudaStream_t)cuda_stream);
}

int32_t rgs_scalable_rgbd(int32_t H, int32_t W, const float* rgb, const float* depth, const float* mask, double depth_trunc, uint8_t* color,
                          float* depth_out, void* cuda_stream) {
	if (H < 0 || W < 0) return fail(RGS_E_INVALID, "image size must not be negative");
	if (std::isnan(depth_trunc)) return fail(RGS_E_INVALID, "depth_trunc is NaN");
	const int64_t P = (int64_t)H * W;
	if (P == 0) return RGS_OK;
	if (!rgb || !depth || !color || !depth_out) return fail(RGS_E_INVALID, "null pointer");
	scalable_rgbd_kernel<<<blocks_for(P), 256, 0, (cudaStream_t)cuda_stream>>>(P, rgb, depth, mask, depth_trunc, color, depth_out);
	count_launch();
	return cuda_status(cudaGetLastError(), "scalable rgbd");
}

int32_t rgs_scalable_image_u8(int32_t H, int32_t W, const float* image, float scale, float offset, uint8_t* out, void* cuda_stream) {
	if (H < 0 || W < 0) return fail(RGS_E_INVALID, "image size must not be negative");
	const int64_t P = (int64_t)H * W;
	if (P == 0) return RGS_OK;
	if (!image || !out) return fail(RGS_E_INVALID, "null pointer");
	scalable_image_u8_kernel<<<blocks_for(P), 256, 0, (cudaStream_t)cuda_stream>>>(P, image, scale, offset, out);
	count_launch();
	return cuda_status(cudaGetLastError(), "scalable image_u8");
}

static int scalable_check(const rgs_tsdf_grid* grid, const rgs_tsdf_camera* cam, float sdf_trunc) {
	int rc = tsdf_grid_check(grid);
	if (rc == RGS_OK) rc = tsdf_pinhole_check(cam);
	if (rc == RGS_OK && !finite_pos(sdf_trunc)) rc = fail(RGS_E_INVALID, "sdf_trunc must be positive and finite");
	return rc;
}

int64_t rgs_scalable_touch(const rgs_tsdf_grid* grid, const rgs_tsdf_camera* cam, float sdf_trunc, const float* depth, int32_t* unit_coords,
                           int64_t* allocated, rgs_resize_fn scratch, void* scratch_user, void* cuda_stream) {
	if (const int rc = scalable_check(grid, cam, sdf_trunc)) return rc;
	if (!depth || !unit_coords || !scratch) return fail(RGS_E_INVALID, "null pointer");
	return tsdf_touch_run(grid, make_scalable_cam(*grid, *cam, sdf_trunc), true, depth, unit_coords, allocated, scratch, scratch_user,
	                      (cudaStream_t)cuda_stream);
}

int32_t rgs_scalable_integrate(const rgs_tsdf_grid* grid, const rgs_tsdf_camera* cam, float sdf_trunc, int64_t n, const int32_t* unit_coords,
                               const float* depth, const uint8_t* color, int32_t call_id, rgs_resize_fn scratch, void* scratch_user, void* cuda_stream) {
	int rc = scalable_check(grid, cam, sdf_trunc);
	if (rc != RGS_OK) return rc;
	if (n < 0 || n > INT32_MAX) return fail(RGS_E_INVALID, "block count out of range");
	if (call_id <= 0) return fail(RGS_E_INVALID, "call_id must be positive");
	if (n == 0) return RGS_OK;
	if (!unit_coords || !depth || !color || !scratch) return fail(RGS_E_INVALID, "null pointer");
	char* buf;
	if ((rc = grow(scratch, scratch_user, (size_t)n * sizeof(int32_t), buf, "tsdf scratch")) != RGS_OK) return rc;
	return cuda_status(launch_scalable_integrate(*grid, make_scalable_cam(*grid, *cam, sdf_trunc), n, unit_coords, depth, color, call_id,
	                                             reinterpret_cast<int32_t*>(buf), (cudaStream_t)cuda_stream),
	                   "scalable integrate");
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
	tsdf_rehash_kernel<<<blocks_for(old_slots), 256, 0, (cudaStream_t)cuda_stream>>>(*grid, old_keys, old_values, old_slots);
	count_launch();
	return cuda_status(cudaGetLastError(), "tsdf rehash");
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

}  // extern "C"

// rgs_tnt_eval.cu -- the Tanks and Temples scorer (reference eval_tnt/run.py, registration.py, evaluation.py) on the GPU in
// fp64: transform and polygon crop, voxel downsampling and the moments of the scaled point-to-point ICP.  Runs once per
// trained model, off the rasterizer path.  Nearest neighbours come from rgs_dtu_nearest.
//
// The contract (include/rgs_b200.h, rgs_tnt_*) fixes every stored bit: each arithmetic step is one intrinsic rounded on its
// own (__dadd_rn / __dmul_rn / __ddiv_rn), so nvcc contracts nothing and a numpy fp64 restatement reproduces the crop masks
// and the voxel means.
//   crop       one thread per point: optional 4x4 transform, axis range, crossing-number test against the polygon held in
//              shared memory; CUB's stable DeviceSelect compacts the kept points in input order (one host read).
//   voxel      bounds (one host read, the 2^21-cell check before anything else is requested), 63-bit keys, CUB's stable
//              radix sort of (key, input index), head flags and a scan (one host read: the voxel count), then one warp per
//              voxel: the lanes load 32 points at a time and every lane adds them in input order, so a voxel of 10^5 points
//              holds one warp and the launch keeps going around it.
//   moments    two passes (sums, then centred sums), each a fixed tree: 1024 points per block, 4 per thread in a fixed
//              order, a shared-memory halving tree, then one block over the partials.  The launch shape depends on N only.
//
// This file also holds the C-ABI entry points rgs_tnt_* (include/rgs_b200.h).
#include <cub/cub.cuh>

#include "rgs_common.cuh"

namespace rgs {

namespace {

__device__ __forceinline__ double dsub(double a, double b) { return __dadd_rn(a, -b); }
__device__ __forceinline__ bool finite3d(double x, double y, double z) { return isfinite(x) && isfinite(y) && isfinite(z); }

struct Xform {
	double m[12];   // rows 0..2 of the 4x4, row-major
};

// ((m0 x + m1 y) + m2 z) + m3 per row
__device__ __forceinline__ void apply_xform(const Xform& T, double& x, double& y, double& z) {
	double o[3];
#pragma unroll
	for (int r = 0; r < 3; r++)
		o[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T.m[4 * r], x), __dmul_rn(T.m[4 * r + 1], y)), __dmul_rn(T.m[4 * r + 2], z)), T.m[4 * r + 3]);
	x = o[0];
	y = o[1];
	z = o[2];
}

struct P3 {
	double x, y, z;
};

// ---- transform and crop (registration.py:113-131, evaluation.py:75-89) ------------------------------------------------

struct CropParams {
	int has_xform, has_volume, axis, K;
	double axis_min, axis_max;
};

__global__ void __launch_bounds__(256) tnt_xform_kernel(int64_t N, double* __restrict__ p, Xform T) {
	const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
	if (i >= N) return;
	double x = p[3 * i], y = p[3 * i + 1], z = p[3 * i + 2];
	apply_xform(T, x, y, z);
	p[3 * i] = x;
	p[3 * i + 1] = y;
	p[3 * i + 2] = z;
}

// polygon [K, 2] (u, v) staged in dynamic shared memory; out [N, 3] transformed points, kept [N]; bad counts non-finite inputs
__global__ void __launch_bounds__(256) tnt_crop_kernel(int64_t N, const double* __restrict__ p, Xform T, CropParams c, const double* __restrict__ poly,
                                                       P3* __restrict__ out, uint8_t* __restrict__ kept, unsigned long long* __restrict__ bad) {
	extern __shared__ double spoly[];
	if (c.has_volume)
		for (int k = threadIdx.x; k < 2 * c.K; k += blockDim.x) spoly[k] = poly[k];
	__syncthreads();
	const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
	if (i >= N) return;
	double x = p[3 * i], y = p[3 * i + 1], z = p[3 * i + 2];
	if (!finite3d(x, y, z)) atomicAdd(bad, 1ull);
	if (c.has_xform) apply_xform(T, x, y, z);
	out[i] = P3{x, y, z};
	uint8_t in = 1;
	if (c.has_volume) {
		const double w = c.axis == 0 ? x : (c.axis == 1 ? y : z);
		const double pu = c.axis == 0 ? y : x, pv = c.axis == 2 ? y : z;
		if (!(w >= c.axis_min && w <= c.axis_max)) {
			in = 0;
		} else {
			int crossings = 0;
			for (int k = 0; k < c.K; k++) {
				const int k1 = k + 1 == c.K ? 0 : k + 1;
				const double au = spoly[2 * k], av = spoly[2 * k + 1], bu = spoly[2 * k1], bv = spoly[2 * k1 + 1];
				if ((av < pv && pv <= bv) || (bv < pv && pv <= av)) {
					const double xu = __dadd_rn(au, __ddiv_rn(__dmul_rn(dsub(pv, av), dsub(bu, au)), dsub(bv, av)));
					if (xu < pu) crossings++;
				}
			}
			in = (uint8_t)(crossings & 1);
		}
	}
	kept[i] = in;
}

// ---- voxel downsample (Open3D VoxelDownSample) -------------------------------------------------------------------------

constexpr int VOXEL_BITS = 21;
constexpr double VOXEL_CELLS = 2097152.0;   // 2^21 cells per axis

// bits[0..6] = ordered min x,y,z | max x,y,z | non-finite count (the same encoding as rgs_dtu_eval.cu's bounds)
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

__global__ void __launch_bounds__(256) tnt_bounds_kernel(int64_t N, const double* __restrict__ p, unsigned long long* __restrict__ bits) {
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

struct VoxelGrid {
	double origin[3];
	double voxel;
};

__device__ __forceinline__ uint64_t voxel_index(double x, double origin, double voxel) {
	return (uint64_t)floor(__ddiv_rn(dsub(x, origin), voxel));   // >= 0: x >= min >= origin; < 2^21 checked on the host
}

__global__ void __launch_bounds__(256) tnt_voxel_key_kernel(int N, const double* __restrict__ p, VoxelGrid g, uint64_t* __restrict__ keys,
                                                            int32_t* __restrict__ ids) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= N) return;
	const int64_t j = i;
	keys[i] = voxel_index(p[3 * j], g.origin[0], g.voxel) << (2 * VOXEL_BITS) | voxel_index(p[3 * j + 1], g.origin[1], g.voxel) << VOXEL_BITS |
	          voxel_index(p[3 * j + 2], g.origin[2], g.voxel);
	ids[i] = i;
}

__global__ void __launch_bounds__(256) tnt_voxel_head_kernel(int N, const uint64_t* __restrict__ keys, int32_t* __restrict__ head) {
	const int j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= N) return;
	head[j] = (j == 0 || keys[j] != keys[j - 1]) ? 1 : 0;
}

// start[v] of every voxel (start[V] = N), from the inclusive scan of the head flags
__global__ void __launch_bounds__(256) tnt_voxel_start_kernel(int N, const int32_t* __restrict__ head, const int32_t* __restrict__ incl,
                                                              int32_t* __restrict__ start) {
	const int j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= N) return;
	if (head[j]) start[incl[j] - 1] = j;
	if (j == N - 1) start[incl[j]] = N;
}

// one warp per voxel: sum = ((0 + p_0) + p_1) + ... in input order, mean = sum / count
__global__ void __launch_bounds__(256) tnt_voxel_mean_kernel(int V, const double* __restrict__ p, const int32_t* __restrict__ ids,
                                                             const int32_t* __restrict__ start, double* __restrict__ means, int64_t* __restrict__ counts) {
	const int v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int lane = threadIdx.x & 31;
	if (v >= V) return;   // warp-uniform
	const int s = start[v], e = start[v + 1];
	double sx = 0.0, sy = 0.0, sz = 0.0;
	for (int c = s; c < e; c += 32) {
		const int j = c + lane;
		double x = 0.0, y = 0.0, z = 0.0;
		if (j < e) {
			const int64_t i = ids[j];
			x = p[3 * i];
			y = p[3 * i + 1];
			z = p[3 * i + 2];
		}
		const int n = min(32, e - c);
		for (int k = 0; k < n; k++) {
			sx = __dadd_rn(sx, __shfl_sync(0xffffffffu, x, k));
			sy = __dadd_rn(sy, __shfl_sync(0xffffffffu, y, k));
			sz = __dadd_rn(sz, __shfl_sync(0xffffffffu, z, k));
		}
	}
	if (lane == 0) {
		const double n = (double)(e - s);
		means[3 * (int64_t)v] = __ddiv_rn(sx, n);
		means[3 * (int64_t)v + 1] = __ddiv_rn(sy, n);
		means[3 * (int64_t)v + 2] = __ddiv_rn(sz, n);
		counts[v] = e - s;
	}
}

// ---- ICP moments (Open3D TransformationEstimationPointToPoint(True), Eigen::umeyama) -------------------------------------

constexpr int MOM_THREADS = 256;
constexpr int MOM_ITEMS = 4;
constexpr int MOM_CHUNK = MOM_THREADS * MOM_ITEMS;   // points per first-level block
constexpr int MOM_A = 9;                              // count, sum d2, sum s (3), sum t (3), non-finite count
constexpr int MOM_B = 10;                             // sum (t - mt)(s - ms)^T (9, row-major), sum |s - ms|^2

// halving tree over MOM_THREADS values per quantity; thread 0 ends with the block's sums
template <int Q>
__device__ __forceinline__ void block_tree(double (*sh)[MOM_THREADS], double (&v)[Q]) {
	const int t = threadIdx.x;
#pragma unroll
	for (int q = 0; q < Q; q++) sh[q][t] = v[q];
	__syncthreads();
	for (int s = MOM_THREADS / 2; s > 0; s >>= 1) {
		if (t < s) {
#pragma unroll
			for (int q = 0; q < Q; q++) sh[q][t] = __dadd_rn(sh[q][t], sh[q][t + s]);
		}
		__syncthreads();
	}
}

__device__ __forceinline__ bool is_corr(int64_t i, const double* __restrict__ dist, const int64_t* __restrict__ index, int64_t M, double thr) {
	const int64_t j = index[i];
	return dist[i] < thr && j >= 0 && j < M;
}

__global__ void __launch_bounds__(MOM_THREADS) tnt_mom_a_kernel(int64_t N, const double* __restrict__ src, int64_t M, const double* __restrict__ tgt,
                                                                const double* __restrict__ dist, const int64_t* __restrict__ index, double thr,
                                                                double* __restrict__ partial) {
	__shared__ double sh[MOM_A][MOM_THREADS];
	double v[MOM_A];
#pragma unroll
	for (int q = 0; q < MOM_A; q++) v[q] = 0.0;
	const int64_t base = blockIdx.x * (int64_t)MOM_CHUNK + threadIdx.x;
#pragma unroll
	for (int k = 0; k < MOM_ITEMS; k++) {
		const int64_t i = base + k * MOM_THREADS;
		if (i >= N) break;
		const double sx = src[3 * i], sy = src[3 * i + 1], sz = src[3 * i + 2];
		if (!finite3d(sx, sy, sz) || isnan(dist[i])) v[8] = __dadd_rn(v[8], 1.0);
		if (!is_corr(i, dist, index, M, thr)) continue;
		const int64_t j = index[i];
		const double tx = tgt[3 * j], ty = tgt[3 * j + 1], tz = tgt[3 * j + 2];
		if (!finite3d(tx, ty, tz)) v[8] = __dadd_rn(v[8], 1.0);
		const double dx = dsub(sx, tx), dy = dsub(sy, ty), dz = dsub(sz, tz);
		v[0] = __dadd_rn(v[0], 1.0);
		v[1] = __dadd_rn(v[1], __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
		v[2] = __dadd_rn(v[2], sx);
		v[3] = __dadd_rn(v[3], sy);
		v[4] = __dadd_rn(v[4], sz);
		v[5] = __dadd_rn(v[5], tx);
		v[6] = __dadd_rn(v[6], ty);
		v[7] = __dadd_rn(v[7], tz);
	}
	block_tree<MOM_A>(sh, v);
	if (threadIdx.x < MOM_A) partial[blockIdx.x * (int64_t)MOM_A + threadIdx.x] = sh[threadIdx.x][0];
}

// centred sums with the means of mom[2..7]
__global__ void __launch_bounds__(MOM_THREADS) tnt_mom_b_kernel(int64_t N, const double* __restrict__ src, int64_t M, const double* __restrict__ tgt,
                                                                const double* __restrict__ dist, const int64_t* __restrict__ index, double thr,
                                                                const double* __restrict__ mom, double* __restrict__ partial) {
	__shared__ double sh[MOM_B][MOM_THREADS];
	double v[MOM_B];
#pragma unroll
	for (int q = 0; q < MOM_B; q++) v[q] = 0.0;
	const double ms[3] = {mom[2], mom[3], mom[4]}, mt[3] = {mom[5], mom[6], mom[7]};
	const int64_t base = blockIdx.x * (int64_t)MOM_CHUNK + threadIdx.x;
#pragma unroll
	for (int k = 0; k < MOM_ITEMS; k++) {
		const int64_t i = base + k * MOM_THREADS;
		if (i >= N) break;
		if (!is_corr(i, dist, index, M, thr)) continue;
		const int64_t j = index[i];
		const double s[3] = {dsub(src[3 * i], ms[0]), dsub(src[3 * i + 1], ms[1]), dsub(src[3 * i + 2], ms[2])};
		const double t[3] = {dsub(tgt[3 * j], mt[0]), dsub(tgt[3 * j + 1], mt[1]), dsub(tgt[3 * j + 2], mt[2])};
#pragma unroll
		for (int r = 0; r < 3; r++)
#pragma unroll
			for (int c = 0; c < 3; c++) v[3 * r + c] = __dadd_rn(v[3 * r + c], __dmul_rn(t[r], s[c]));
		v[9] = __dadd_rn(v[9], __dadd_rn(__dadd_rn(__dmul_rn(s[0], s[0]), __dmul_rn(s[1], s[1])), __dmul_rn(s[2], s[2])));
	}
	block_tree<MOM_B>(sh, v);
	if (threadIdx.x < MOM_B) partial[blockIdx.x * (int64_t)MOM_B + threadIdx.x] = sh[threadIdx.x][0];
}

// one block: thread t adds partials t, t + 256, ... in order, then the halving tree.  Pass A writes mom[0..7] (the means
// as sum * (1 / n), Eigen's one_over_n) and mom[18] (non-finite count); pass B writes mom[8..17].  No correspondence: all 0.
template <int Q>
__global__ void __launch_bounds__(MOM_THREADS) tnt_mom_final_kernel(int64_t P, const double* __restrict__ partial, double* __restrict__ mom) {
	__shared__ double sh[Q][MOM_THREADS];
	double v[Q];
#pragma unroll
	for (int q = 0; q < Q; q++) v[q] = 0.0;
	for (int64_t b = threadIdx.x; b < P; b += MOM_THREADS)
#pragma unroll
		for (int q = 0; q < Q; q++) v[q] = __dadd_rn(v[q], partial[b * Q + q]);
	block_tree<Q>(sh, v);
	if (threadIdx.x != 0) return;
	if (Q == MOM_A) {
		const double n = sh[0][0];
		const double inv = n > 0.0 ? __ddiv_rn(1.0, n) : 0.0;
		mom[0] = n;
		mom[1] = n > 0.0 ? sh[1][0] : 0.0;
		for (int q = 2; q < 8; q++) mom[q] = __dmul_rn(sh[q][0], inv);
		mom[18] = sh[8][0];
	} else {
		const double n = mom[0];
		const double inv = n > 0.0 ? __ddiv_rn(1.0, n) : 0.0;
		for (int q = 0; q < 10; q++) mom[8 + q] = __dmul_rn(inv, sh[q][0]);
	}
}

static Xform make_xform(const double* T) {
	Xform x;
	for (int k = 0; k < 12; k++) x.m[k] = T ? T[k] : 0.0;
	return x;
}

// ---- crop ----

struct CropScratch {
	P3* moved;
	int64_t* num;
	unsigned long long* bad;
	char* temp;
	size_t temp_bytes;
};

static CropScratch carve_crop(char* base, int N, size_t* total) {
	size_t temp = 0;
	cub::DeviceSelect::Flagged(nullptr, temp, (const P3*)nullptr, (const uint8_t*)nullptr, (P3*)nullptr, (int64_t*)nullptr, N);
	Carver c(base);
	CropScratch k;
	k.moved = c.take<P3>(N);
	k.num = c.take<int64_t>(1);
	k.bad = c.take<unsigned long long>(1);
	k.temp = c.take<char>(temp);
	k.temp_bytes = temp;
	if (total) *total = c.size();
	return k;
}

size_t tnt_crop_scratch_bytes(int N) {
	size_t t = 0;
	carve_crop(nullptr, N, &t);
	return t;
}

cudaError_t launch_tnt_crop(int N, const double* pts, const double* xform, int axis, double axis_min, double axis_max, int K, const double* polygon,
                            uint8_t* kept, double* cropped, int64_t* num_kept, char* scratch, cudaStream_t s) {
	CropScratch k = carve_crop(scratch, N, nullptr);
	RGS_TRY(cudaMemsetAsync(k.bad, 0, sizeof(unsigned long long), s));
	CropParams c;
	c.has_xform = xform != nullptr;
	c.has_volume = polygon != nullptr;
	c.axis = axis;
	c.K = polygon ? K : 0;
	c.axis_min = axis_min;
	c.axis_max = axis_max;
	tnt_crop_kernel<<<(unsigned)((N + 255) / 256), 256, 2 * (size_t)c.K * sizeof(double), s>>>(N, pts, make_xform(xform), c, polygon, k.moved, kept, k.bad);
	count_launch();
	size_t temp = k.temp_bytes;
	RGS_TRY(cub::DeviceSelect::Flagged(k.temp, temp, k.moved, kept, reinterpret_cast<P3*>(cropped), k.num, N, s));
	count_launch();
	unsigned long long h[2];
	RGS_TRY(cudaMemcpyAsync(&h[0], k.num, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaMemcpyAsync(&h[1], k.bad, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaStreamSynchronize(s));
	*num_kept = (int64_t)h[0];
	if (h[1]) return cudaErrorInvalidValue;
	return cudaGetLastError();
}

// ---- voxel downsample ----

struct VoxelScratch {
	uint64_t *keys_in, *keys_out;
	int32_t *ids_in, *ids_out, *head, *incl, *start;
	char* temp;
	size_t temp_bytes;
};

static VoxelScratch carve_voxel(char* base, int N, size_t* total) {
	size_t sort_bytes = 0, scan_bytes = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr, N);
	cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (const int32_t*)nullptr, (int32_t*)nullptr, N);
	Carver c(base);
	VoxelScratch k;
	k.keys_in = c.take<uint64_t>(N);
	k.keys_out = c.take<uint64_t>(N);
	k.ids_in = c.take<int32_t>(N);
	k.ids_out = c.take<int32_t>(N);
	k.head = c.take<int32_t>(N);
	k.incl = c.take<int32_t>(N);
	k.start = c.take<int32_t>((size_t)N + 1);
	k.temp_bytes = std::max(sort_bytes, scan_bytes);
	k.temp = c.take<char>(k.temp_bytes);
	if (total) *total = c.size();
	return k;
}

size_t tnt_bounds_scratch_bytes() { return 8 * sizeof(unsigned long long); }

size_t tnt_voxel_scratch_bytes(int N) {
	size_t t = 0;
	carve_voxel(nullptr, N, &t);
	return t;
}

cudaError_t launch_tnt_bounds(int N, const double* pts, char* scratch, double* lo, double* hi, int64_t* nonfinite, cudaStream_t s) {
	unsigned long long* bits = reinterpret_cast<unsigned long long*>(scratch);
	RGS_TRY(cudaMemsetAsync(bits, 0xff, 3 * sizeof(unsigned long long), s));
	RGS_TRY(cudaMemsetAsync(bits + 3, 0, 5 * sizeof(unsigned long long), s));
	const int blocks = (int)std::min<int64_t>((N + 255) / 256, 4 * sm_count());
	tnt_bounds_kernel<<<blocks, 256, 0, s>>>(N, pts, bits);
	count_launch();
	unsigned long long h[8];
	RGS_TRY(cudaMemcpyAsync(h, bits, sizeof(h), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaStreamSynchronize(s));
	for (int a = 0; a < 3; a++) {
		lo[a] = ord2d(h[a]);
		hi[a] = ord2d(h[3 + a]);
	}
	*nonfinite = (int64_t)h[6];
	return cudaGetLastError();
}

cudaError_t launch_tnt_voxel_sort(int N, const double* pts, const double* origin, double voxel, char* scratch, int32_t* num_voxels, cudaStream_t s) {
	VoxelScratch k = carve_voxel(scratch, N, nullptr);
	VoxelGrid g;
	for (int a = 0; a < 3; a++) g.origin[a] = origin[a];
	g.voxel = voxel;
	const unsigned blocks = (unsigned)((N + 255) / 256);
	tnt_voxel_key_kernel<<<blocks, 256, 0, s>>>(N, pts, g, k.keys_in, k.ids_in);
	size_t temp = k.temp_bytes;
	RGS_TRY(cub::DeviceRadixSort::SortPairs(k.temp, temp, k.keys_in, k.keys_out, k.ids_in, k.ids_out, N, 0, 3 * VOXEL_BITS, s));
	tnt_voxel_head_kernel<<<blocks, 256, 0, s>>>(N, k.keys_out, k.head);
	temp = k.temp_bytes;
	RGS_TRY(cub::DeviceScan::InclusiveSum(k.temp, temp, k.head, k.incl, N, s));
	tnt_voxel_start_kernel<<<blocks, 256, 0, s>>>(N, k.head, k.incl, k.start);
	count_launch(5);
	RGS_TRY(cudaMemcpyAsync(num_voxels, k.incl + (N - 1), sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaStreamSynchronize(s));
	return cudaGetLastError();
}

cudaError_t launch_tnt_voxel_mean(int N, const double* pts, int V, char* scratch, double* means, int64_t* counts, cudaStream_t s) {
	VoxelScratch k = carve_voxel(scratch, N, nullptr);
	tnt_voxel_mean_kernel<<<(unsigned)(((int64_t)V * 32 + 255) / 256), 256, 0, s>>>(V, pts, k.ids_out, k.start, means, counts);
	count_launch();
	return cudaGetLastError();
}

// ---- ICP moments ----

size_t tnt_moments_scratch_bytes(int64_t N) {
	const int64_t P = std::max<int64_t>(1, (N + MOM_CHUNK - 1) / MOM_CHUNK);
	Carver c(nullptr);
	c.take<double>(32);
	c.take<double>((size_t)P * MOM_B);
	return c.size();
}

cudaError_t launch_tnt_moments(int64_t N, const double* src, int64_t M, const double* tgt, const double* dist, const int64_t* index, double thr,
                               char* scratch, double* moments_host, cudaStream_t s) {
	const int64_t P = std::max<int64_t>(1, (N + MOM_CHUNK - 1) / MOM_CHUNK);
	Carver c(scratch);
	double* mom = c.take<double>(32);
	double* partial = c.take<double>((size_t)P * MOM_B);
	if (N == 0) {
		RGS_TRY(cudaMemsetAsync(partial, 0, (size_t)MOM_B * sizeof(double), s));
	} else {
		tnt_mom_a_kernel<<<(unsigned)P, MOM_THREADS, 0, s>>>(N, src, M, tgt, dist, index, thr, partial);
		count_launch();
	}
	tnt_mom_final_kernel<MOM_A><<<1, MOM_THREADS, 0, s>>>(P, partial, mom);
	if (N > 0) {
		tnt_mom_b_kernel<<<(unsigned)P, MOM_THREADS, 0, s>>>(N, src, M, tgt, dist, index, thr, mom, partial);
		count_launch();
	}
	tnt_mom_final_kernel<MOM_B><<<1, MOM_THREADS, 0, s>>>(P, partial, mom);
	count_launch(2);
	RGS_TRY(cudaMemcpyAsync(moments_host, mom, 19 * sizeof(double), cudaMemcpyDeviceToHost, s));
	RGS_TRY(cudaStreamSynchronize(s));
	if (moments_host[18] != 0.0) return cudaErrorInvalidValue;
	return cudaGetLastError();
}

}  // namespace
}  // namespace rgs

using namespace rgs;

extern "C" {

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
	if (N == 0) return RGS_OK;
	tnt_xform_kernel<<<(unsigned)((N + 255) / 256), 256, 0, (cudaStream_t)cuda_stream>>>(N, points, make_xform(transform));
	count_launch();
	return cuda_status(cudaGetLastError(), "tnt transform", kNonFinitePoint);
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

}  // extern "C"

// rgs_densify.cu -- GaussianModel.densify_and_prune and reset_opacity (reference scene/gaussian_model.py:495-513, :662-741) as
// a handful of passes over the Gaussians instead of three rounds of concatenate / mask-index over every parameter and moment.
//
//   select   gradient averages, the integer count behind `ratio`, sort of grads_abs (CUB radix sort of the fp32 keys), the
//            quantile threshold Q on the device, then one flag byte per Gaussian: clone, split, and whether the original row,
//            its clone and its split children survive the final prune.  Per-CTA counts of the five flags are scanned; the
//            totals are the one host read of the call (they size the draws and the outputs).
//   plan     every output row's source row and draw index, and exp(scaling) rows of the selected Gaussians packed as the
//            `std` of the caller's torch.normal draws.
//   gather   every output row written once from its source: the sampled offset R * sample + xyz and the split scaling
//            log(exp(s) / 1.6) on new rows, every other column copied, zeros for the moments of new rows.
// The floating-point contract (bit-exactness, operation order) is stated in include/rgs_b200.h.
//
// This file also holds the C-ABI entry points rgs_densify_* and rgs_reset_opacity (include/rgs_b200.h).
#include <cub/cub.cuh>

#include "rgs_common.cuh"

namespace rgs {

constexpr int DENSIFY_CTA = 256;
// flag byte of a Gaussian
constexpr uint8_t F_CLONE = 1, F_SPLIT = 2, F_KEEP = 4, F_CLONE_KEEP = 8, F_CHILD_KEEP = 16;

// torch.max(dim=1) over three values: NaN wins
__device__ __forceinline__ float max3_nan(float a, float b, float c) {
	if (isnan(a)) return a;
	if (isnan(b)) return b;
	if (isnan(c)) return c;
	return fmaxf(fmaxf(a, b), c);
}

// grads = accum / denom with NaN -> 0 (0/0 and NaN inputs); a positive value over 0 stays +inf
__device__ __forceinline__ float grad_average(float accum, float denom) {
	const float g = __fdiv_rn(accum, denom);
	return isnan(g) ? 0.0f : g;
}

// torch.norm of a one-element row on CUDA: sqrt of the fp32 square (|g| except where g*g under- or overflows)
__device__ __forceinline__ float norm1(float g) { return sqrtf(__fmul_rn(g, g)); }

__global__ void __launch_bounds__(DENSIFY_CTA) densify_grads_kernel(int P, const float* __restrict__ accum, const float* __restrict__ accum_abs,
                                                                    const float* __restrict__ denom, float max_grad, float* __restrict__ keys,
                                                                    unsigned long long* __restrict__ count) {
	const int i = blockIdx.x * DENSIFY_CTA + threadIdx.x;
	bool hit = false;
	if (i < P) {
		const float d = denom[i];
		keys[i] = grad_average(accum_abs[i], d);
		hit = norm1(grad_average(accum[i], d)) >= max_grad;
	}
	const int n = __syncthreads_count(hit);
	if (threadIdx.x == 0 && n) atomicAdd(count, (unsigned long long)n);
}

// ratio = mean(hit) as ATen's CUDA mean computes it (the fp32 sum times the fp32 reciprocal of P);
// Q = torch.quantile(grads_abs, 1 - ratio), linear interpolation, lerp's two-branch formula (contracted to FMA as nvcc builds it)
__global__ void densify_quantile_kernel(int P, const float* __restrict__ sorted, const unsigned long long* __restrict__ count, float* __restrict__ ratio_q) {
	if (threadIdx.x != 0) return;
	const float ratio = __fmul_rn(__ull2float_rn(*count), __fdiv_rn(1.0f, __int2float_rn(P)));
	const float q = __fsub_rn(1.0f, ratio);
	const float rank = __fmul_rn(q, __int2float_rn(P - 1));
	const long long lo = (long long)rank;              // ranks.toType(kLong)
	const long long hi = (long long)ceilf(rank);
	const float w = __fsub_rn(rank, __ll2float_rn(lo));
	// above 2^24 rows (float)(P - 1) can round up past the last index: clamp (torch refuses these sizes)
	const float a = sorted[lo < P ? lo : P - 1], b = sorted[hi < P ? hi : P - 1];
	const float d = __fsub_rn(b, a);
	ratio_q[0] = ratio;
	ratio_q[1] = fabsf(w) < 0.5f ? __fmaf_rn(w, d, a) : __fmaf_rn(-d, __fsub_rn(1.0f, w), b);
}

struct SelectArgs {
	float max_grad, dense, min_opacity, max_screen_size, world, inv_split;
	int prune_large;
};

// five 12-bit counters in one word: a CTA of 256 never carries into the next field
__device__ __forceinline__ unsigned long long pack_flags(uint8_t f) {
	return (unsigned long long)(f & F_CLONE) | (unsigned long long)((f >> 1) & 1) << 12 | (unsigned long long)((f >> 2) & 1) << 24 |
	       (unsigned long long)((f >> 3) & 1) << 36 | (unsigned long long)((f >> 4) & 1) << 48;
}
__device__ __forceinline__ int field(unsigned long long v, int k) { return (int)((v >> (12 * k)) & 0xfff); }

__global__ void __launch_bounds__(DENSIFY_CTA) densify_flags_kernel(int P, const float* __restrict__ accum, const float* __restrict__ accum_abs,
                                                                    const float* __restrict__ denom, const float* __restrict__ scaling,
                                                                    const float* __restrict__ opacity, const float* __restrict__ ratio_q, SelectArgs a,
                                                                    uint8_t* __restrict__ flags, int* __restrict__ block_counts) {
	using Reduce = cub::BlockReduce<unsigned long long, DENSIFY_CTA>;
	__shared__ typename Reduce::TempStorage tmp;
	const int i = blockIdx.x * DENSIFY_CTA + threadIdx.x;
	uint8_t f = 0;
	if (i < P) {
		const float Q = ratio_q[1];
		const float d = denom[i];
		const float g = grad_average(accum[i], d), ga = grad_average(accum_abs[i], d);
		float e[3], c[3];
#pragma unroll
		for (int k = 0; k < 3; k++) {
			e[k] = expf(scaling[3 * i + k]);
			c[k] = expf(logf(__fmul_rn(e[k], a.inv_split)));   // exp of the split child's scaling
		}
		const float big = max3_nan(e[0], e[1], e[2]), big_child = max3_nan(c[0], c[1], c[2]);
		const bool clone = (norm1(g) >= a.max_grad || norm1(ga) >= Q) && big <= a.dense;
		const bool split = (g >= a.max_grad || ga >= Q) && big > a.dense;
		const bool faint = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-opacity[i]))) < a.min_opacity;
		// max_radii2D is all zeros when the prune runs (densification_postfix reset it): its test is 0 > max_screen_size
		const bool radius = 0.0f > a.max_screen_size;
		const bool prune = faint || (a.prune_large && (radius || big > a.world));
		const bool prune_child = faint || (a.prune_large && (radius || big_child > a.world));
		f = (clone ? F_CLONE : 0) | (split ? F_SPLIT : 0) | (!split && !prune ? F_KEEP : 0) | (clone && !prune ? F_CLONE_KEEP : 0) |
		    (split && !prune_child ? F_CHILD_KEEP : 0);
		flags[i] = f;
	}
	const unsigned long long sum = Reduce(tmp).Sum(pack_flags(f));
	if (threadIdx.x == 0)
		for (int k = 0; k < 5; k++) block_counts[5 * blockIdx.x + k] = field(sum, k);
}

// exclusive scan of the per-CTA counts in place, totals[5] after the last CTA
__global__ void __launch_bounds__(1024) densify_scan_kernel(int blocks, int* __restrict__ block_counts, int* __restrict__ totals) {
	using Scan = cub::BlockScan<int, 1024>;
	__shared__ typename Scan::TempStorage tmp;
	for (int k = 0; k < 5; k++) {
		int carry = 0;
		for (int base = 0; base < blocks; base += 1024) {
			const int b = base + threadIdx.x;
			const int v = b < blocks ? block_counts[5 * b + k] : 0;
			int ex, chunk;
			Scan(tmp).ExclusiveSum(v, ex, chunk);
			if (b < blocks) block_counts[5 * b + k] = carry + ex;
			carry += chunk;
			__syncthreads();
		}
		if (threadIdx.x == 0) totals[k] = carry;
	}
}

struct PlanTotals {
	int C, S, K0, K1, K2;
};

__global__ void __launch_bounds__(DENSIFY_CTA) densify_plan_kernel(int P, const uint8_t* __restrict__ flags, const int* __restrict__ block_offsets,
                                                                   PlanTotals t, const float* __restrict__ scaling, int* __restrict__ src,
                                                                   int* __restrict__ draw, float* __restrict__ std_clone, float* __restrict__ std_split) {
	using Scan = cub::BlockScan<unsigned long long, DENSIFY_CTA>;
	__shared__ typename Scan::TempStorage tmp;
	const int i = blockIdx.x * DENSIFY_CTA + threadIdx.x;
	const uint8_t f = i < P ? flags[i] : 0;
	unsigned long long ex;
	Scan(tmp).ExclusiveSum(pack_flags(f), ex);
	if (i >= P || f == 0) return;
	const int* bo = block_offsets + 5 * blockIdx.x;
	const int clone_rank = bo[0] + field(ex, 0), split_rank = bo[1] + field(ex, 1);
	if (f & (F_CLONE | F_SPLIT)) {
		float e[3];
#pragma unroll
		for (int k = 0; k < 3; k++) e[k] = expf(scaling[3 * i + k]);
		float* dst = (f & F_CLONE) ? std_clone + 3 * (size_t)clone_rank : std_split + 3 * (size_t)split_rank;
#pragma unroll
		for (int k = 0; k < 3; k++) dst[k] = e[k];
		if (f & F_SPLIT)  // stds.repeat(2, 1): the second child's draw reads the same row again, S rows later
#pragma unroll
			for (int k = 0; k < 3; k++) dst[3 * (size_t)t.S + k] = e[k];
	}
	if (f & F_KEEP) {
		const int j = bo[2] + field(ex, 2);
		src[j] = i;
		draw[j] = -1;
	}
	if (f & F_CLONE_KEEP) {
		const int j = t.K0 + bo[3] + field(ex, 3);
		src[j] = i;
		draw[j] = clone_rank;
	}
	if (f & F_CHILD_KEEP) {
		const int j = t.K0 + t.K1 + bo[4] + field(ex, 4);
		src[j] = i;
		draw[j] = t.C + split_rank;
		src[j + t.K2] = i;
		draw[j + t.K2] = t.C + t.S + split_rank;
	}
}

// xyz and scaling of every output row.  New rows: R(rotation) * sample + xyz, build_rotation's expressions
// (utils/general_utils.py:80-101) one rounded operation at a time, the matrix-vector product summed left to right.
__global__ void __launch_bounds__(DENSIFY_CTA) densify_rows_kernel(int N, const int* __restrict__ src, const int* __restrict__ draw, int C,
                                                                   const float* __restrict__ xyz, const float* __restrict__ rotation,
                                                                   const float* __restrict__ scaling, const float* __restrict__ sample_clone,
                                                                   const float* __restrict__ sample_split, float inv_split, float* __restrict__ xyz_out,
                                                                   float* __restrict__ scaling_out) {
	const int j = blockIdx.x * DENSIFY_CTA + threadIdx.x;
	if (j >= N) return;
	const int s = src[j], d = draw[j];
	const float px = xyz[3 * (size_t)s], py = xyz[3 * (size_t)s + 1], pz = xyz[3 * (size_t)s + 2];
	if (d < 0) {
		xyz_out[3 * (size_t)j] = px;
		xyz_out[3 * (size_t)j + 1] = py;
		xyz_out[3 * (size_t)j + 2] = pz;
#pragma unroll
		for (int k = 0; k < 3; k++) scaling_out[3 * (size_t)j + k] = scaling[3 * (size_t)s + k];
		return;
	}
	const float* smp = d < C ? sample_clone + 3 * (size_t)d : sample_split + 3 * (size_t)(d - C);
	const float4 q4 = *reinterpret_cast<const float4*>(rotation + 4 * (size_t)s);
	const float n = sqrtf(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q4.x, q4.x), __fmul_rn(q4.y, q4.y)), __fmul_rn(q4.z, q4.z)), __fmul_rn(q4.w, q4.w)));
	const float r = __fdiv_rn(q4.x, n), x = __fdiv_rn(q4.y, n), y = __fdiv_rn(q4.z, n), z = __fdiv_rn(q4.w, n);
	const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
	const float xy = __fmul_rn(x, y), xz = __fmul_rn(x, z), yz = __fmul_rn(y, z);
	const float rx = __fmul_rn(r, x), ry = __fmul_rn(r, y), rz = __fmul_rn(r, z);
	const float R[9] = {__fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(yy, zz))), __fmul_rn(2.0f, __fsub_rn(xy, rz)), __fmul_rn(2.0f, __fadd_rn(xz, ry)),
	                    __fmul_rn(2.0f, __fadd_rn(xy, rz)), __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(xx, zz))), __fmul_rn(2.0f, __fsub_rn(yz, rx)),
	                    __fmul_rn(2.0f, __fsub_rn(xz, ry)), __fmul_rn(2.0f, __fadd_rn(yz, rx)), __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(xx, yy)))};
	const float s0 = smp[0], s1 = smp[1], s2 = smp[2];
	const float p[3] = {px, py, pz};
#pragma unroll
	for (int k = 0; k < 3; k++) {
		const float v = __fadd_rn(__fadd_rn(__fmul_rn(R[3 * k], s0), __fmul_rn(R[3 * k + 1], s1)), __fmul_rn(R[3 * k + 2], s2));
		xyz_out[3 * (size_t)j + k] = __fadd_rn(v, p[k]);
	}
	const bool child = d >= C;
#pragma unroll
	for (int k = 0; k < 3; k++) {
		const float raw = scaling[3 * (size_t)s + k];
		scaling_out[3 * (size_t)j + k] = child ? logf(__fmul_rn(expf(raw), inv_split)) : raw;
	}
}

struct GatherColumns {
	rgs_densify_column c[RGS_DENSIFY_MAX_COLUMNS];
};

// one column per blockIdx.y: out[j, :] = in[src[j], :], or zeros on new rows of a moment column
__global__ void __launch_bounds__(DENSIFY_CTA) densify_gather_kernel(int N, const int* __restrict__ src, const int* __restrict__ draw, GatherColumns cols) {
	const rgs_densify_column col = cols.c[blockIdx.y];
	const int64_t W = col.width, total = (int64_t)N * W;
	for (int64_t e = (int64_t)blockIdx.x * DENSIFY_CTA + threadIdx.x; e < total; e += (int64_t)gridDim.x * DENSIFY_CTA) {
		const int64_t j = e / W, k = e - j * W;
		col.out[e] = (col.zero_new_rows && draw[j] >= 0) ? 0.0f : col.in[(int64_t)src[j] * W + k];
	}
}

// reset_opacity: inverse_sigmoid(min(sigmoid(o) * coef, 0.01) / coef), coef the Mip-Splatting 3D-filter factor with products
// taken left to right
__global__ void __launch_bounds__(DENSIFY_CTA) reset_opacity_kernel(int P, const float* __restrict__ scaling, const float* __restrict__ opacity,
                                                                    const float* __restrict__ filter_3D, float* __restrict__ out) {
	const int i = blockIdx.x * DENSIFY_CTA + threadIdx.x;
	if (i >= P) return;
	const float f = filter_3D[i], f2 = __fmul_rn(f, f);
	float sq[3], after[3];
#pragma unroll
	for (int k = 0; k < 3; k++) {
		const float s = expf(scaling[3 * i + k]);
		sq[k] = __fmul_rn(s, s);
		after[k] = __fadd_rn(sq[k], f2);
	}
	const float det1 = __fmul_rn(__fmul_rn(sq[0], sq[1]), sq[2]);
	const float det2 = __fmul_rn(__fmul_rn(after[0], after[1]), after[2]);
	const float coef = sqrtf(__fdiv_rn(det1, det2));
	const float o = __fmul_rn(__fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-opacity[i]))), coef);
	const float m = (isnan(o) || o < 0.01f) ? o : 0.01f;   // torch.min: NaN propagates
	const float x = __fdiv_rn(m, coef);
	out[i] = logf(__fdiv_rn(x, __fsub_rn(1.0f, x)));
}

static int densify_blocks(int P) { return (P + DENSIFY_CTA - 1) / DENSIFY_CTA; }

static size_t densify_select_scratch_bytes(int P) {
	size_t sort_bytes = 0;
	cub::DeviceRadixSort::SortKeys(nullptr, sort_bytes, (const float*)nullptr, (float*)nullptr, P);
	Carver c(nullptr);
	c.take<float>(P);
	c.take<float>(P);
	c.take<unsigned long long>(1);
	c.take<char>(sort_bytes);
	return c.size();
}

static cudaError_t launch_densify_select(int P, const float* accum, const float* accum_abs, const float* denom, const float* scaling,
                                         const float* opacity, const rgs_densify_thresholds& th, uint8_t* flags, int* block_offsets, float* ratio_q,
                                         int* totals, char* scratch, cudaStream_t s) {
	size_t sort_bytes = 0;
	RGS_TRY(cub::DeviceRadixSort::SortKeys(nullptr, sort_bytes, (const float*)nullptr, (float*)nullptr, P));
	Carver c(scratch);
	float* keys = c.take<float>(P);
	float* sorted = c.take<float>(P);
	unsigned long long* count = c.take<unsigned long long>(1);
	char* temp = c.take<char>(sort_bytes);
	const int blocks = densify_blocks(P);
	RGS_TRY(cudaMemsetAsync(count, 0, sizeof(unsigned long long), s));
	densify_grads_kernel<<<blocks, DENSIFY_CTA, 0, s>>>(P, accum, accum_abs, denom, th.max_grad, keys, count);
	RGS_TRY(cub::DeviceRadixSort::SortKeys(temp, sort_bytes, keys, sorted, P, 0, 32, s));
	densify_quantile_kernel<<<1, 32, 0, s>>>(P, sorted, count, ratio_q);
	const SelectArgs a{th.max_grad, th.dense, th.min_opacity, th.max_screen_size, th.world, th.inv_split, th.prune_large};
	densify_flags_kernel<<<blocks, DENSIFY_CTA, 0, s>>>(P, accum, accum_abs, denom, scaling, opacity, ratio_q, a, flags, block_offsets);
	densify_scan_kernel<<<1, 1024, 0, s>>>(blocks, block_offsets, totals);
	count_launch(5);
	return cudaGetLastError();
}

}  // namespace rgs

using namespace rgs;

extern "C" {

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
	const PlanTotals t{c[0], c[1], c[2], c[3], c[4]};
	densify_plan_kernel<<<densify_blocks(P), DENSIFY_CTA, 0, (cudaStream_t)cuda_stream>>>(P, flags, block_offsets, t, scaling, src, draw, std_clone, std_split);
	count_launch();
	return cuda_status(cudaGetLastError(), "densify plan");
}

int32_t rgs_densify_gather(int32_t N, const int32_t* src, const int32_t* draw, int32_t C, const float* xyz, const float* rotation, const float* scaling,
                           const float* sample_clone, const float* sample_split, float inv_split, float* xyz_out, float* scaling_out, int32_t n_cols,
                           const rgs_densify_column* cols, void* cuda_stream) {
	if (N < 0 || C < 0 || n_cols < 0 || n_cols > RGS_DENSIFY_MAX_COLUMNS) return fail(RGS_E_INVALID, "densify gather: bad sizes");
	if (N == 0) return RGS_OK;
	if (!src || !draw || !xyz || !rotation || !scaling || !xyz_out || !scaling_out || (n_cols && !cols)) return fail(RGS_E_INVALID, "null pointer");
	for (int k = 0; k < n_cols; k++)
		if (!cols[k].in || !cols[k].out || cols[k].width <= 0) return fail(RGS_E_INVALID, "densify gather: bad column");
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	densify_rows_kernel<<<densify_blocks(N), DENSIFY_CTA, 0, s>>>(N, src, draw, C, xyz, rotation, scaling, sample_clone, sample_split, inv_split, xyz_out,
	                                                              scaling_out);
	count_launch();
	if (n_cols > 0) {
		GatherColumns g{};
		for (int k = 0; k < n_cols; k++) g.c[k] = cols[k];
		int64_t widest = 0;
		for (int k = 0; k < n_cols; k++) widest = widest > cols[k].width ? widest : cols[k].width;
		const int64_t want = ((int64_t)N * widest + DENSIFY_CTA - 1) / DENSIFY_CTA;
		const int grid_x = (int)(want < 8 * (int64_t)sm_count() ? (want > 0 ? want : 1) : 8 * (int64_t)sm_count());
		densify_gather_kernel<<<dim3(grid_x, n_cols), DENSIFY_CTA, 0, s>>>(N, src, draw, g);
		count_launch();
	}
	return cuda_status(cudaGetLastError(), "densify gather");
}

int32_t rgs_reset_opacity(int32_t P, const float* scaling, const float* opacity, const float* filter_3D, float* out, void* cuda_stream) {
	if (P < 0) return fail(RGS_E_INVALID, "negative Gaussian count");
	if (P == 0) return RGS_OK;
	if (!scaling || !opacity || !filter_3D || !out) return fail(RGS_E_INVALID, "null pointer");
	reset_opacity_kernel<<<densify_blocks(P), DENSIFY_CTA, 0, (cudaStream_t)cuda_stream>>>(P, scaling, opacity, filter_3D, out);
	count_launch();
	return cuda_status(cudaGetLastError(), "reset opacity");
}

}  // extern "C"

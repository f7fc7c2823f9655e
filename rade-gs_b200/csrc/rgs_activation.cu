// rgs_activation.cu -- the per-Gaussian arithmetic that sits directly before and after the rasterizer call in the
// reference's training step, fused (SURVEY.md 8f row 1, opt-in: render() itself stays valid without it).
//
//   activate_forward/backward  replaces, with one kernel each, the ~12 + ~20 torch element-wise kernels of
//       GaussianModel.get_scaling_n_opacity_with_3D_filter (reference scene/gaussian_model.py:156-166: exp, square,
//       prod, the Mip-Splatting 3D filter, sqrt, sigmoid * coef) and get_rotation (:125-126, F.normalize);
//   densification_stats        replaces train.py:187-188 + GaussianModel.add_densification_stats
//       (scene/gaussian_model.py:743-747: masked row norms of means2D.grad[:, :2] and [:, 2:], running max, counter)
//       -- five masked-index torch passes over [P] tensors -- with one pass.
// Operation order follows the torch expressions; products and sums that torch rounds separately are kept from
// contracting into FMAs (__fmul_rn / __fadd_rn) so the results match the eager reference to the last bit or two.
//
// This file also holds the C-ABI entry points rgs_activate_*, rgs_densification_stats and rgs_compute_3d_filter (include/rgs_b200.h).
#include "rgs_common.cuh"

namespace rgs {

__global__ void __launch_bounds__(256) activate_forward_kernel(int P, const float* __restrict__ raw_scaling, const float* __restrict__ raw_opacity,
                                                                const float* __restrict__ raw_rotation, const float* __restrict__ filter_3D,
                                                                float* __restrict__ scales, float* __restrict__ opacity, float* __restrict__ rotations) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	const float f = filter_3D[i], f2 = __fmul_rn(f, f);
	float sq[3], after[3];
#pragma unroll
	for (int k = 0; k < 3; k++) {
		const float s = expf(raw_scaling[3 * i + k]);
		sq[k] = __fmul_rn(s, s);
		after[k] = __fadd_rn(sq[k], f2);
		scales[3 * i + k] = sqrtf(after[k]);
	}
	const float det1 = __fmul_rn(__fmul_rn(sq[0], sq[1]), sq[2]);
	const float det2 = __fmul_rn(__fmul_rn(after[0], after[1]), after[2]);
	const float coef = sqrtf(det1 / det2);
	const float o = 1.0f / (1.0f + expf(-raw_opacity[i]));
	opacity[i] = __fmul_rn(o, coef);
	const float4 r = *reinterpret_cast<const float4*>(raw_rotation + 4 * i);
	const float n = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(r.x, r.x), __fmul_rn(r.y, r.y)), __fadd_rn(__fmul_rn(r.z, r.z), __fmul_rn(r.w, r.w))));
	const float d = fmaxf(n, 1e-12f);  // F.normalize: x / max(||x||, eps)
	*reinterpret_cast<float4*>(rotations + 4 * i) = make_float4(r.x / d, r.y / d, r.z / d, r.w / d);
}

__global__ void __launch_bounds__(256) activate_backward_kernel(int P, const float* __restrict__ raw_scaling, const float* __restrict__ raw_opacity,
                                                                 const float* __restrict__ raw_rotation, const float* __restrict__ filter_3D,
                                                                 const float* __restrict__ g_scales, const float* __restrict__ g_opacity,
                                                                 const float* __restrict__ g_rotations, float* __restrict__ d_raw_scaling,
                                                                 float* __restrict__ d_raw_opacity, float* __restrict__ d_raw_rotation) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	const float f = filter_3D[i], f2 = f * f;
	float s[3], sq[3], after[3];
#pragma unroll
	for (int k = 0; k < 3; k++) {
		s[k] = expf(raw_scaling[3 * i + k]);
		sq[k] = s[k] * s[k];
		after[k] = sq[k] + f2;
	}
	const float det1 = sq[0] * sq[1] * sq[2], det2 = after[0] * after[1] * after[2];
	const float coef = sqrtf(det1 / det2);
	const float o = 1.0f / (1.0f + expf(-raw_opacity[i]));
	const float go = g_opacity[i];
	// opacity_out = o * coef
	d_raw_opacity[i] = go * coef * o * (1.0f - o);
	// coef = sqrt(prod_j sq_j / after_j) with after_j = sq_j + f^2 and sq_j = exp(2 raw_j), so
	//   d coef / d raw_k = coef * (1 - sq_k / after_k) = coef * f^2 / after_k.
	// Autograd's chain through det1 and det2 subtracts two terms of size d_coef * coef that nearly cancel, and its
	// -d_q * det1 / det2^2 underflows: det2 >= f^6 reaches 1e-24 at f = 1e-4, and det2 * det2 leaves the fp32 range.
	// This form has no quotient by det2^2 and no cancellation: every factor is a product of positive terms.
	const float d_coef_f2 = go * o * coef * f2;
#pragma unroll
	for (int k = 0; k < 3; k++) {
		const float scale_out = sqrtf(after[k]);
		// scales_out_k = sqrt(after_k): d / d raw_k = g / (2 scale_out) * 2 s^2
		const float d_scale = g_scales[3 * i + k] / (2.0f * scale_out) * 2.0f * s[k] * s[k];
		d_raw_scaling[3 * i + k] = d_coef_f2 / after[k] + d_scale;
	}
	const float4 r = *reinterpret_cast<const float4*>(raw_rotation + 4 * i);
	const float4 g = *reinterpret_cast<const float4*>(g_rotations + 4 * i);
	const float n = sqrtf(r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w);
	float4 dr;
	if (n > 1e-12f) {
		const float inv = 1.0f / n;
		const float4 u = make_float4(r.x * inv, r.y * inv, r.z * inv, r.w * inv);
		const float ug = u.x * g.x + u.y * g.y + u.z * g.z + u.w * g.w;
		dr = make_float4((g.x - u.x * ug) * inv, (g.y - u.y * ug) * inv, (g.z - u.z * ug) * inv, (g.w - u.w * ug) * inv);
	} else {
		dr = make_float4(g.x / 1e-12f, g.y / 1e-12f, g.z / 1e-12f, g.w / 1e-12f);  // clamp_min branch: denominator is the constant
	}
	*reinterpret_cast<float4*>(d_raw_rotation + 4 * i) = dr;
}

__global__ void __launch_bounds__(256) densification_stats_kernel(int P, const float* __restrict__ means2D_grad, const int* __restrict__ radii,
                                                                   float* __restrict__ grad_accum, float* __restrict__ grad_accum_abs,
                                                                   float* __restrict__ grad_accum_abs_max, float* __restrict__ denom,
                                                                   float* __restrict__ max_radii2D) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	const int r = radii[i];
	if (!(r > 0)) return;  // update_filter = visibility_filter = radii > 0 (gaussian_renderer/__init__.py:90)
	const float gx = means2D_grad[3 * i], gy = means2D_grad[3 * i + 1], ga = means2D_grad[3 * i + 2];
	const float n2 = sqrtf(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)));  // torch.norm(grad[:, :2], dim=-1)
	const float na = fabsf(ga);                                              // torch.norm(grad[:, 2:], dim=-1) of one element
	grad_accum[i] += n2;
	grad_accum_abs[i] += na;
	grad_accum_abs_max[i] = fmaxf(grad_accum_abs_max[i], na);
	denom[i] += 1.0f;
	if (max_radii2D != nullptr) max_radii2D[i] = fmaxf(max_radii2D[i], (float)r);  // train.py:187
}

// ---- 3D smoothing filter (GaussianModel.compute_3D_filter, scene/gaussian_model.py:179-232) ----------------------------------
// The reference loops over the training cameras in Python, ~15 torch kernels per camera over all P points (a few
// thousand launches per call at DTU scale).  Here one thread owns a point and walks the camera table (16 floats per
// camera: R row-major as Camera.R, T, focal_x, focal_y, W, H); the closest valid camera-space depth decides the
// filter size.  Pass 1 leaves min z (or -1 when no camera sees the point) and the maximum over the seen points;
// pass 2 gives unseen points that maximum and scales: filter = distance / focal_length * sqrt(0.2).
constexpr int CAM_FLOATS = 16;
constexpr int CAM_CHUNK = 256;  // cameras staged in shared memory at a time (16 KiB)

__global__ void __launch_bounds__(256) filter3d_distance_kernel(int P, const float* __restrict__ xyz, int n_cams, const float* __restrict__ cams,
                                                                 float* __restrict__ distance, unsigned int* __restrict__ max_bits) {
	__shared__ float s_cam[CAM_CHUNK * CAM_FLOATS];
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	const bool live = i < P;
	const float x = live ? xyz[3 * i] : 0.f, y = live ? xyz[3 * i + 1] : 0.f, z = live ? xyz[3 * i + 2] : 0.f;
	float dist = 100000.0f;
	bool seen = false;
	for (int base = 0; base < n_cams; base += CAM_CHUNK) {
		const int chunk = min(CAM_CHUNK, n_cams - base);
		__syncthreads();
		for (int k = threadIdx.x; k < chunk * CAM_FLOATS; k += blockDim.x) s_cam[k] = cams[(size_t)base * CAM_FLOATS + k];
		__syncthreads();
		for (int c = 0; c < chunk; c++) {
			const float* C = s_cam + c * CAM_FLOATS;
			// xyz @ R + T : one fp32 dot product per column, then the bias
			const float xc = __fadd_rn(fmaf(z, C[6], fmaf(y, C[3], __fmul_rn(x, C[0]))), C[9]);
			const float yc = __fadd_rn(fmaf(z, C[7], fmaf(y, C[4], __fmul_rn(x, C[1]))), C[10]);
			const float zc = __fadd_rn(fmaf(z, C[8], fmaf(y, C[5], __fmul_rn(x, C[2]))), C[11]);
			const bool valid_depth = zc > 0.2f;
			const float zz = fmaxf(zc, 0.001f);
			const float W = C[14], H = C[15];
			const float px = __fadd_rn(__fmul_rn(__fdiv_rn(xc, zz), C[12]), W * 0.5f);
			const float py = __fadd_rn(__fmul_rn(__fdiv_rn(yc, zz), C[13]), H * 0.5f);
			// "similar tangent space filtering as in the paper": 15% margin around the image
			const bool in_screen = px >= (float)(-0.15 * (double)W) && px <= (float)((double)W * 1.15) && py >= (float)(-0.15 * (double)H) &&
			                       py <= (float)(1.15 * (double)H);
			if (valid_depth && in_screen) {
				dist = fminf(dist, zz);
				seen = true;
			}
		}
	}
	const float best = (live && seen) ? dist : -1.0f;
	if (live) distance[i] = best;
	// maximum over the seen points (distances are positive: their bit patterns order like unsigned integers)
	float m = fmaxf(best, 0.0f);
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
	if ((threadIdx.x & 31) == 0 && m > 0.0f) atomicMax(max_bits, __float_as_uint(m));
}

__global__ void __launch_bounds__(256) filter3d_finish_kernel(int P, const unsigned int* __restrict__ max_bits, float inv_focal, float scale,
                                                               float* __restrict__ filter_3D) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	float d = filter_3D[i];
	if (d < 0.0f) d = __uint_as_float(*max_bits);
	// torch divides by a Python scalar as a multiplication with its fp32 reciprocal
	filter_3D[i] = __fmul_rn(__fmul_rn(d, inv_focal), scale);
}

}  // namespace rgs

using namespace rgs;

extern "C" {

int32_t rgs_activate_forward(int32_t P, const float* raw_scaling, const float* raw_opacity, const float* raw_rotation, const float* filter_3D,
                             float* scales, float* opacity, float* rotations, void* cuda_stream) {
	if (P < 0) return fail(RGS_E_INVALID, "negative Gaussian count");
	if (P == 0) return RGS_OK;
	if (!raw_scaling || !raw_opacity || !raw_rotation || !filter_3D || !scales || !opacity || !rotations) return fail(RGS_E_INVALID, "null pointer");
	activate_forward_kernel<<<(P + 255) / 256, 256, 0, (cudaStream_t)cuda_stream>>>(P, raw_scaling, raw_opacity, raw_rotation, filter_3D, scales, opacity,
	                                                                                rotations);
	count_launch();
	return cuda_status(cudaGetLastError(), "activate forward");
}

int32_t rgs_activate_backward(int32_t P, const float* raw_scaling, const float* raw_opacity, const float* raw_rotation, const float* filter_3D,
                              const float* g_scales, const float* g_opacity, const float* g_rotations, float* d_raw_scaling, float* d_raw_opacity,
                              float* d_raw_rotation, void* cuda_stream) {
	if (P < 0) return fail(RGS_E_INVALID, "negative Gaussian count");
	if (P == 0) return RGS_OK;
	if (!raw_scaling || !raw_opacity || !raw_rotation || !filter_3D || !g_scales || !g_opacity || !g_rotations || !d_raw_scaling || !d_raw_opacity ||
	    !d_raw_rotation)
		return fail(RGS_E_INVALID, "null pointer");
	activate_backward_kernel<<<(P + 255) / 256, 256, 0, (cudaStream_t)cuda_stream>>>(P, raw_scaling, raw_opacity, raw_rotation, filter_3D, g_scales, g_opacity,
	                                                                                 g_rotations, d_raw_scaling, d_raw_opacity, d_raw_rotation);
	count_launch();
	return cuda_status(cudaGetLastError(), "activate backward");
}

int32_t rgs_densification_stats(int32_t P, const float* means2D_grad, const int32_t* radii, float* grad_accum, float* grad_accum_abs,
                                float* grad_accum_abs_max, float* denom, float* max_radii2D, void* cuda_stream) {
	if (P < 0) return fail(RGS_E_INVALID, "negative Gaussian count");
	if (P == 0) return RGS_OK;
	if (!means2D_grad || !radii || !grad_accum || !grad_accum_abs || !grad_accum_abs_max || !denom) return fail(RGS_E_INVALID, "null pointer");
	densification_stats_kernel<<<(P + 255) / 256, 256, 0, (cudaStream_t)cuda_stream>>>(P, means2D_grad, radii, grad_accum, grad_accum_abs,
	                                                                                    grad_accum_abs_max, denom, max_radii2D);
	count_launch();
	return cuda_status(cudaGetLastError(), "densification stats");
}

int32_t rgs_compute_3d_filter(int32_t P, const float* xyz, int32_t n_cams, const float* cams, float focal_length, float* filter_3D,
                              float* max_distance, void* cuda_stream) {
	if (P < 0 || n_cams < 0) return fail(RGS_E_INVALID, "negative count");
	if (P == 0) return RGS_OK;
	if (!xyz || !filter_3D || !max_distance || (n_cams > 0 && !cams)) return fail(RGS_E_INVALID, "null pointer");
	if (!(focal_length > 0.0f)) return fail(RGS_E_INVALID, "focal_length must be positive");
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	unsigned int* max_bits = reinterpret_cast<unsigned int*>(max_distance);
	cudaMemsetAsync(max_bits, 0, sizeof(unsigned int), s);
	filter3d_distance_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, xyz, n_cams, cams, filter_3D, max_bits);
	count_launch();
	filter3d_finish_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, max_bits, 1.0f / focal_length, (float)0.4472135954999579 /* 0.2 ** 0.5 */, filter_3D);
	count_launch();
	return cuda_status(cudaGetLastError(), "compute 3d filter");
}

}  // extern "C"

// rgs_render_common.cuh -- helpers shared by the forward and backward tile kernels.
#pragma once
#include "rgs_common.cuh"

namespace rgs {

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
	const uint32_t dst = (uint32_t)__cvta_generic_to_shared(smem_dst);
	asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(dst), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }

// Two-lane float ops on the (x, y) pairs the records keep side by side.  Hopper has no packed fp32x2 pipe, so each lane is
// one scalar op; the _rn intrinsics keep every product and sum separately rounded (no contraction into FMAs), which is
// the rounding the blend and its gradient were validated with.
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }

// Conservative test: can splat (centre c, conic A,B,C, opacity o) reach alpha >= 1/255 anywhere in the
// pixel box [x0,x1]x[y0,y1]?  alpha = o*exp(-q), q = 0.5(A dx^2 + C dy^2) + B dx dy, so the splat matters
// only where q <= ln(255 o).  q is convex when the conic is positive definite; its minimum over a box is
// 0 if the centre is inside, else it lies on one of the four edges (1-D quadratics, closed form).
__device__ __forceinline__ bool splat_hits_box(float cx, float cy, float A, float B, float C, float o, float x0, float x1, float y0, float y1) {
	if (!(A > 0.f && C > 0.f && A * C - B * B > 0.f)) return true;  // not PD: no claim, let the exact path decide
	const float tau = __logf(255.0f * o);                            // o <= 0 -> NaN/-inf -> compare below fails -> culled only if tau<0
	if (!(o > 0.f)) return false;                                    // alpha = o*G <= 0 < 1/255 everywhere
	const float dxl = cx - x1, dxh = cx - x0;                        // d = centre - pixel
	const float dyl = cy - y1, dyh = cy - y0;
	if (dxl <= 0.f && dxh >= 0.f && dyl <= 0.f && dyh >= 0.f) return tau >= -1e-3f;
	const float iA = 1.0f / A, iC = 1.0f / C;
	float qmin;
	{
		// edges dx = const: minimise over dy in [dyl, dyh]
		float dy = fminf(fmaxf(-B * dxl * iC, dyl), dyh);
		qmin = 0.5f * (A * dxl * dxl + C * dy * dy) + B * dxl * dy;
		dy = fminf(fmaxf(-B * dxh * iC, dyl), dyh);
		qmin = fminf(qmin, 0.5f * (A * dxh * dxh + C * dy * dy) + B * dxh * dy);
		// edges dy = const
		float dx = fminf(fmaxf(-B * dyl * iA, dxl), dxh);
		qmin = fminf(qmin, 0.5f * (A * dx * dx + C * dyl * dyl) + B * dx * dyl);
		dx = fminf(fmaxf(-B * dyh * iA, dxl), dxh);
		qmin = fminf(qmin, 0.5f * (A * dx * dx + C * dyh * dyh) + B * dx * dyh);
	}
	// margin: absolute 1e-3 plus relative 1e-4 of the magnitudes involved (fp32 evaluation noise is ~1e-6 rel.)
	return !(qmin > tau + 1e-3f + 1e-4f * fabsf(tau));
}

}  // namespace rgs

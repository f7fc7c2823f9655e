// rgs_image_loss.cu -- the image-side consumers of the rasterizer's maps in the reference's training step, fused
// (SURVEY.md 8f row 2, opt-in).
//
//   ssim_l1_forward / backward   utils/loss_utils.py:17-18 (l1_loss) and :35-63 (ssim: five depthwise 11x11 Gaussian
//       convolutions with zero padding + ~15 element-wise kernels, and autograd's transposed convolutions in backward)
//       -> two kernels that do the separable convolutions out of shared memory.  Forward leaves the three partial
//       derivatives of the SSIM map per pixel; backward convolves them once more (the window is symmetric) and adds the
//       L1 sign term, i.e. d[(1-l) L1 + l (1 - SSIM)] / d image in one pass.
//   normal_consistency           train.py:143-156 + utils/graphics_utils.py:97-126 (depths_double_to_points,
//       point_double_to_normal): back-project two depth maps (or take two coordinate maps), central differences, cross
//       product, normalise, 1 - <rendered normal, n>, weighted mean -- ~40 torch kernels forward and about twice that
//       backward -- as one kernel that also emits the gradients of the loss w.r.t. the normal map and both depth
//       (coordinate) maps.  Gradients are gathered through shared memory, so the result is deterministic.
//
// All maps are planar fp32 [C,H,W] as the rasterizer writes them.  Scalar sums are accumulated in double.
//
// This file also holds the C-ABI entry points rgs_ssim_l1_* and rgs_normal_consistency* (include/rgs_b200.h).
#include "rgs_common.cuh"

namespace rgs {

namespace {

constexpr int SW = 11, SR = 5;  // window, radius (loss_utils.py:35 window_size=11, padding 5)
constexpr int TW = 32, TH = 16; // output tile of one CTA (256 threads, two rows per thread)
constexpr int IH = TH + 2 * SR, IW = TW + 2 * SR;

struct Window {
	float g[SW];
};

// block-wide sum of `v` into *dst (double), 256 threads
__device__ __forceinline__ void block_add(double* dst, float v, float* s_red) {
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	if (lane == 0) s_red[warp] = v;
	__syncthreads();
	if (threadIdx.x == 0) {
		double t = 0.0;
		for (int w = 0; w < (int)(blockDim.x >> 5); w++) t += (double)s_red[w];
		atomicAdd(dst, t);
	}
	__syncthreads();
}

// Rows [row_lo, row_hi) are the rows whose SSIM-map / L1 values are counted (the whole image on one GPU; a rank's slab in the
// row-sharded multi-GPU loss, where the neighbouring ranks' 5 halo rows around the slab are present in `img` but not counted);
// block rows start at by0.
__global__ void __launch_bounds__(256) ssim_l1_forward_kernel(int H, int W, int row_lo, int row_hi, int by0, Window win, const float* __restrict__ img,
                                                               const float* __restrict__ gt, float* __restrict__ dmaps, size_t map_stride,
                                                               double* __restrict__ sums) {
	__shared__ float sA[IH][IW + 1], sB[IH][IW + 1];
	__shared__ float sh[5][IH][TW];
	__shared__ float s_red[8];
	const int plane = blockIdx.z;
	const int x0 = blockIdx.x * TW, y0 = (blockIdx.y + by0) * TH;
	const float* A = img + (size_t)plane * H * W;
	const float* B = gt + (size_t)plane * H * W;
	for (int i = threadIdx.x; i < IH * IW; i += 256) {
		const int r = i / IW, c = i - r * IW;
		const int gy = y0 + r - SR, gx = x0 + c - SR;
		const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
		sA[r][c] = in ? __ldg(A + (size_t)gy * W + gx) : 0.f;  // zero padding (F.conv2d padding=5)
		sB[r][c] = in ? __ldg(B + (size_t)gy * W + gx) : 0.f;
	}
	__syncthreads();
	// horizontal pass over the IH rows: mu1, mu2, E[x^2], E[y^2], E[xy]
	for (int i = threadIdx.x; i < IH * TW; i += 256) {
		const int r = i / TW, c = i - r * TW;
		float m1 = 0.f, m2 = 0.f, e11 = 0.f, e22 = 0.f, e12 = 0.f;
#pragma unroll
		for (int k = 0; k < SW; k++) {
			const float a = sA[r][c + k], b = sB[r][c + k], w = win.g[k];
			const float wa = w * a, wb = w * b;
			m1 += wa; m2 += wb;
			e11 = fmaf(wa, a, e11); e22 = fmaf(wb, b, e22); e12 = fmaf(wa, b, e12);
		}
		sh[0][r][c] = m1; sh[1][r][c] = m2; sh[2][r][c] = e11; sh[3][r][c] = e22; sh[4][r][c] = e12;
	}
	__syncthreads();
	const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
	float ssim_sum = 0.f, l1_sum = 0.f;
#pragma unroll
	for (int half = 0; half < 2; half++) {
		const int ry = ty + 8 * half;
		const int gy = y0 + ry, gx = x0 + tx;
		if (gy >= row_lo && gy < row_hi && gx < W) {
			float mu1 = 0.f, mu2 = 0.f, e11 = 0.f, e22 = 0.f, e12 = 0.f;
#pragma unroll
			for (int k = 0; k < SW; k++) {
				const float w = win.g[k];
				mu1 = fmaf(w, sh[0][ry + k][tx], mu1); mu2 = fmaf(w, sh[1][ry + k][tx], mu2);
				e11 = fmaf(w, sh[2][ry + k][tx], e11); e22 = fmaf(w, sh[3][ry + k][tx], e22);
				e12 = fmaf(w, sh[4][ry + k][tx], e12);
			}
			const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;  // loss_utils.py:57-58
			const float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2, mu12 = mu1 * mu2;
			const float s1 = e11 - mu1_sq, s2 = e22 - mu2_sq, s12 = e12 - mu12;
			const float a_ = mu1_sq + mu2_sq + C1, b_ = s1 + s2 + C2, c_ = 2.f * mu12 + C1, d_ = 2.f * s12 + C2;
			const float inv_ab = 1.0f / (a_ * b_);
			ssim_sum += c_ * d_ * inv_ab;
			const float x = sA[ry + SR][tx + SR], y = sB[ry + SR][tx + SR];
			l1_sum += fabsf(x - y);
			if (dmaps != nullptr) {
				// partial derivatives of the SSIM map w.r.t. the convolved quantities mu1, E[x^2], E[xy] (E[.] held fixed)
				const size_t o = (size_t)plane * H * W + (size_t)gy * W + gx;
				const float cd = c_ * d_;
				dmaps[o] = 2.f * mu2 * (d_ - c_) * inv_ab - 2.f * mu1 * cd * (b_ - a_) * inv_ab * inv_ab;
				dmaps[o + map_stride] = -cd * inv_ab / b_;
				dmaps[o + 2 * map_stride] = 2.f * c_ * inv_ab;
			}
		}
	}
	block_add(sums, ssim_sum, s_red);
	block_add(sums + 1, l1_sum, s_red);
}

// d_img is written for the rows of the launched blocks; only SSIM-map rows [row_lo, row_hi) contribute (dmaps outside are not read),
// so rows further than 5 from that range come out as zero.
__global__ void __launch_bounds__(256) ssim_l1_backward_kernel(int H, int W, int row_lo, int row_hi, int by0, Window win, const float* __restrict__ img,
                                                                const float* __restrict__ gt, const float* __restrict__ dmaps, size_t map_stride,
                                                                float w_ssim, float w_l1, const float* __restrict__ upstream, float* __restrict__ d_img) {
	__shared__ float sM[3][IH][IW + 1];
	__shared__ float sh[3][IH][TW];
	const int plane = blockIdx.z;
	const int x0 = blockIdx.x * TW, y0 = (blockIdx.y + by0) * TH;
	const size_t base = (size_t)plane * H * W;
	for (int i = threadIdx.x; i < IH * IW; i += 256) {
		const int r = i / IW, c = i - r * IW;
		const int gy = y0 + r - SR, gx = x0 + c - SR;
		const bool in = gy >= row_lo && gy < row_hi && gx >= 0 && gx < W;
		const size_t o = base + (size_t)gy * W + gx;
		sM[0][r][c] = in ? __ldg(dmaps + o) : 0.f;
		sM[1][r][c] = in ? __ldg(dmaps + o + map_stride) : 0.f;
		sM[2][r][c] = in ? __ldg(dmaps + o + 2 * map_stride) : 0.f;
	}
	__syncthreads();
	for (int i = threadIdx.x; i < IH * TW; i += 256) {
		const int r = i / TW, c = i - r * TW;
		float t0 = 0.f, t1 = 0.f, t2 = 0.f;
#pragma unroll
		for (int k = 0; k < SW; k++) {
			const float w = win.g[k];
			t0 = fmaf(w, sM[0][r][c + k], t0); t1 = fmaf(w, sM[1][r][c + k], t1); t2 = fmaf(w, sM[2][r][c + k], t2);
		}
		sh[0][r][c] = t0; sh[1][r][c] = t1; sh[2][r][c] = t2;
	}
	__syncthreads();
	const float up = upstream != nullptr ? __ldg(upstream) : 1.0f;
	const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
	for (int half = 0; half < 2; half++) {
		const int ry = ty + 8 * half;
		const int gy = y0 + ry, gx = x0 + tx;
		if (gy < H && gx < W) {
			float t0 = 0.f, t1 = 0.f, t2 = 0.f;
#pragma unroll
			for (int k = 0; k < SW; k++) {
				const float w = win.g[k];
				t0 = fmaf(w, sh[0][ry + k][tx], t0); t1 = fmaf(w, sh[1][ry + k][tx], t1); t2 = fmaf(w, sh[2][ry + k][tx], t2);
			}
			const size_t o = base + (size_t)gy * W + gx;
			const float x = __ldg(img + o), y = __ldg(gt + o);
			const float diff = x - y;
			float sgn = diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f);  // torch.abs backward: sign(0) = 0
			if (gy < row_lo || gy >= row_hi) sgn = 0.f;                  // L1 term of a row another rank counts
			d_img[o] = up * (w_ssim * (t0 + 2.f * x * t1 + y * t2) + w_l1 * sgn);
		}
	}
}

// ---- normal consistency ------------------------------------------------------------------------------------------------

constexpr int NT = 16;           // output tile (NT x NT pixels, 256 threads)
constexpr int NP = NT + 4;       // points region: tile + 2 (a halo pixel's own neighbours)
constexpr int NG = NT + 2;       // region of stencil centres whose gradients reach the tile

struct V3f {
	float x, y, z;
};
__device__ __forceinline__ V3f vsub(V3f a, V3f b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ V3f vcross(V3f a, V3f b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
__device__ __forceinline__ float vdot(V3f a, V3f b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

// The rows one launch covers.  Loss rows [lo, hi) are counted and their gradients written; blocks start at tile row by0.  The
// buffers are row windows of the image: the two maps hold rows [m_lo, m_lo + m_rows), the rendered normal [n_lo, n_lo + n_rows),
// the outputs [lo, hi).  The whole image is lo = 0, hi = H with every window the whole image.
struct NcRows {
	int lo, hi, by0, m_lo, m_rows, n_lo, n_rows;
};

template <bool FROM_DEPTH>
__global__ void __launch_bounds__(256) normal_consistency_kernel(int H, int W, NcRows R, float inv_fx, float inv_fy, float cx, float cy,
                                                                  const float* __restrict__ rendered_normal, const float* __restrict__ map_e,
                                                                  const float* __restrict__ map_m, float w_e, float w_m, double* __restrict__ loss_sum,
                                                                  float* __restrict__ d_normal, float* __restrict__ d_e, float* __restrict__ d_m) {
	__shared__ V3f sP[2][NP][NP];
	__shared__ V3f sGx[2][NG][NG], sGy[2][NG][NG];  // dL/d(dx), dL/d(dy) of the stencil centred on that pixel
	__shared__ float s_red[8];
	const int x0 = blockIdx.x * NT, y0 = (blockIdx.y + R.by0) * NT;
	const size_t MP = (size_t)R.m_rows * W, NPL = (size_t)R.n_rows * W, OP = (size_t)(R.hi - R.lo) * W;  // plane strides
	for (int i = threadIdx.x; i < NP * NP; i += 256) {
		const int r = i / NP, c = i - r * NP;
		const int gy = y0 + r - 2, gx = x0 + c - 2;
		V3f p0 = {0.f, 0.f, 0.f}, p1 = {0.f, 0.f, 0.f};
		// rows outside the window feed only stencils whose results are not used
		if (gy >= R.m_lo && gy < R.m_lo + R.m_rows && gx >= 0 && gx < W) {
			const size_t o = (size_t)(gy - R.m_lo) * W + gx;
			if (FROM_DEPTH) {
				// rays_d = K^-1 (x + 0.5, y + 0.5, 1) (graphics_utils.py:101-109), points = depth * rays_d
				const float rx = inv_fx * ((float)gx + 0.5f) + cx, ry = inv_fy * ((float)gy + 0.5f) + cy;
				const float d0 = __ldg(map_e + o), d1 = __ldg(map_m + o);
				p0 = {d0 * rx, d0 * ry, d0};
				p1 = {d1 * rx, d1 * ry, d1};
			} else {
				p0 = {__ldg(map_e + o), __ldg(map_e + MP + o), __ldg(map_e + 2 * MP + o)};
				p1 = {__ldg(map_m + o), __ldg(map_m + MP + o), __ldg(map_m + 2 * MP + o)};
			}
		}
		sP[0][r][c] = p0;
		sP[1][r][c] = p1;
	}
	__syncthreads();
	float loss = 0.f;
	for (int i = threadIdx.x; i < NG * NG; i += 256) {
		const int r = i / NG, c = i - r * NG;
		const int gy = y0 + r - 1, gx = x0 + c - 1;
		const bool in_image = gy >= 0 && gy < H && gx >= 0 && gx < W;
		const bool interior = gy >= 1 && gy < H - 1 && gx >= 1 && gx < W - 1;  // output[..., 1:-1, 1:-1] (graphics_utils.py:119)
		const bool own = in_image && r >= 1 && r <= NT && c >= 1 && c <= NT && gy >= R.lo && gy < R.hi;
		V3f rn = {0.f, 0.f, 0.f};
		if (interior && gy >= R.n_lo && gy < R.n_lo + R.n_rows) {
			const size_t o = (size_t)(gy - R.n_lo) * W + gx;
			rn = {__ldg(rendered_normal + o), __ldg(rendered_normal + NPL + o), __ldg(rendered_normal + 2 * NPL + o)};
		}
		V3f dn = {0.f, 0.f, 0.f};
#pragma unroll
		for (int k = 0; k < 2; k++) {
			V3f gdx = {0.f, 0.f, 0.f}, gdy = {0.f, 0.f, 0.f};
			const float w = k == 0 ? w_e : w_m;
			if (interior) {
				// "dx" runs along the image rows' index (H), "dy" along W -- the reference's naming (graphics_utils.py:116-117)
				const V3f dx = vsub(sP[k][r + 2][c + 1], sP[k][r][c + 1]);
				const V3f dy = vsub(sP[k][r + 1][c + 2], sP[k][r + 1][c]);
				const V3f cr = vcross(dx, dy);
				const float len = sqrtf(vdot(cr, cr));
				const float den = fmaxf(len, 1e-12f);  // F.normalize eps
				const V3f n = {cr.x / den, cr.y / den, cr.z / den};
				const float nr = vdot(n, rn);
				if (own) {
					loss += w * (1.0f - nr);
					dn.x -= w * n.x; dn.y -= w * n.y; dn.z -= w * n.z;
				}
				// d(-w <rn, n>)/d(cr): through the normalisation unless the clamp is active
				V3f gc;
				if (len > 1e-12f) gc = {-w * (rn.x - n.x * nr) / den, -w * (rn.y - n.y * nr) / den, -w * (rn.z - n.z * nr) / den};
				else gc = {-w * rn.x / den, -w * rn.y / den, -w * rn.z / den};
				gdx = vcross(dy, gc);  // cr = dx x dy
				gdy = vcross(gc, dx);
			} else if (own) {
				loss += w;  // border pixels keep a zero normal: error 1 (train.py:155)
			}
			sGx[k][r][c] = gdx;
			sGy[k][r][c] = gdy;
		}
		if (own) {
			const size_t o = (size_t)(gy - R.lo) * W + gx;
			d_normal[o] = dn.x; d_normal[OP + o] = dn.y; d_normal[2 * OP + o] = dn.z;
		}
	}
	__syncthreads();
	{
		const int tx = threadIdx.x & (NT - 1), ty = threadIdx.x / NT;
		const int gy = y0 + ty, gx = x0 + tx;
		if (gy >= R.lo && gy < R.hi && gx < W) {
			const int r = ty + 1, c = tx + 1;  // position in the NG region
			const size_t o = (size_t)(gy - R.lo) * W + gx;
#pragma unroll
			for (int k = 0; k < 2; k++) {
				// the stencil centred one row up (r-1) reads this pixel as its +row neighbour, the one a row down as its -row one
				const V3f a = sGx[k][r - 1][c], b = sGx[k][r + 1][c], e = sGy[k][r][c - 1], f = sGy[k][r][c + 1];
				const V3f g = {a.x - b.x + e.x - f.x, a.y - b.y + e.y - f.y, a.z - b.z + e.z - f.z};
				float* dst = k == 0 ? d_e : d_m;
				if (FROM_DEPTH) {
					const float rx = inv_fx * ((float)gx + 0.5f) + cx, ry = inv_fy * ((float)gy + 0.5f) + cy;
					dst[o] = g.x * rx + g.y * ry + g.z;
				} else {
					dst[o] = g.x; dst[OP + o] = g.y; dst[2 * OP + o] = g.z;
				}
			}
		}
	}
	block_add(loss_sum, loss, s_red);
}

Window make_window() {
	// loss_utils.py:23-25: exp(-(x - 5)^2 / (2 * 1.5^2)) in double -> float32 tensor, divided by its float32 sum
	Window w;
	float sum = 0.f;
	for (int x = 0; x < SW; x++) {
		w.g[x] = (float)exp(-(double)((x - SW / 2) * (x - SW / 2)) / (2.0 * 1.5 * 1.5));
		sum += w.g[x];
	}
	for (int x = 0; x < SW; x++) w.g[x] /= sum;
	return w;
}

}  // namespace

}  // namespace rgs

using namespace rgs;

extern "C" {

int32_t rgs_ssim_l1_forward_rows(int32_t planes, int32_t H, int32_t W, int32_t row_lo, int32_t row_hi, const float* img, const float* gt, float* dmaps,
                                 double* sums, void* cuda_stream) {
	if (planes < 0 || H <= 0 || W <= 0) return fail(RGS_E_INVALID, "image size must be positive");
	if (row_lo < 0 || row_hi > H || row_lo > row_hi) return fail(RGS_E_INVALID, "row range out of the image");
	if (!img || !gt || !sums) return fail(RGS_E_INVALID, "null pointer");
	if (planes > 65535) return fail(RGS_E_INVALID, "too many image planes");
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	cudaMemsetAsync(sums, 0, 2 * sizeof(double), s);
	if (row_hi > row_lo) {
		const int by0 = row_lo / TH, by1 = (row_hi + TH - 1) / TH;
		const dim3 grid((W + TW - 1) / TW, by1 - by0, planes);
		ssim_l1_forward_kernel<<<grid, 256, 0, s>>>(H, W, row_lo, row_hi, by0, make_window(), img, gt, dmaps, (size_t)planes * H * W, sums);
		count_launch();
	}
	return cuda_status(cudaGetLastError(), "ssim l1 forward");
}

int32_t rgs_ssim_l1_backward_rows(int32_t planes, int32_t H, int32_t W, int32_t row_lo, int32_t row_hi, const float* img, const float* gt,
                                  const float* dmaps, float w_ssim, float w_l1, const float* upstream, float* d_img, void* cuda_stream) {
	if (planes < 0 || H <= 0 || W <= 0) return fail(RGS_E_INVALID, "image size must be positive");
	if (row_lo < 0 || row_hi > H || row_lo > row_hi) return fail(RGS_E_INVALID, "row range out of the image");
	if (!img || !gt || !dmaps || !d_img) return fail(RGS_E_INVALID, "null pointer");
	if (planes > 65535) return fail(RGS_E_INVALID, "too many image planes");
	if (row_hi > row_lo) {
		const int by0 = max(0, row_lo - SR) / TH, by1 = (min(H, row_hi + SR) + TH - 1) / TH;
		const dim3 grid((W + TW - 1) / TW, by1 - by0, planes);
		ssim_l1_backward_kernel<<<grid, 256, 0, (cudaStream_t)cuda_stream>>>(H, W, row_lo, row_hi, by0, make_window(), img, gt, dmaps, (size_t)planes * H * W,
		                                                                     w_ssim, w_l1, upstream, d_img);
		count_launch();
	}
	return cuda_status(cudaGetLastError(), "ssim l1 backward");
}

int32_t rgs_ssim_l1_forward(int32_t planes, int32_t H, int32_t W, const float* img, const float* gt, float* dmaps, double* sums, void* cuda_stream) {
	return rgs_ssim_l1_forward_rows(planes, H, W, 0, H, img, gt, dmaps, sums, cuda_stream);
}

int32_t rgs_ssim_l1_backward(int32_t planes, int32_t H, int32_t W, const float* img, const float* gt, const float* dmaps, float w_ssim, float w_l1,
                             const float* upstream, float* d_img, void* cuda_stream) {
	return rgs_ssim_l1_backward_rows(planes, H, W, 0, H, img, gt, dmaps, w_ssim, w_l1, upstream, d_img, cuda_stream);
}

int32_t rgs_normal_consistency_rows(int32_t H, int32_t W, int32_t row_lo, int32_t row_hi, int32_t from_depth, float inv_fx, float inv_fy, float cx,
                                    float cy, const float* rendered_normal, const float* map_expected, const float* map_median, float w_expected,
                                    float w_median, double* loss_sum, float* d_normal, float* d_expected, float* d_median, void* cuda_stream) {
	if (H <= 0 || W <= 0) return fail(RGS_E_INVALID, "image size must be positive");
	if (row_lo < 0 || row_hi > H || row_lo > row_hi) return fail(RGS_E_INVALID, "row range out of the image");
	if (!loss_sum) return fail(RGS_E_INVALID, "null pointer");
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	cudaMemsetAsync(loss_sum, 0, sizeof(double), s);
	if (row_hi > row_lo) {
		if (!rendered_normal || !map_expected || !map_median || !d_normal || !d_expected || !d_median) return fail(RGS_E_INVALID, "null pointer");
		NcRows R;
		R.lo = row_lo; R.hi = row_hi; R.by0 = row_lo / NT;
		R.m_lo = max(0, row_lo - 2); R.m_rows = min(H, row_hi + 2) - R.m_lo;
		R.n_lo = max(0, row_lo - 1); R.n_rows = min(H, row_hi + 1) - R.n_lo;
		const dim3 grid((W + NT - 1) / NT, (row_hi + NT - 1) / NT - R.by0);
		if (from_depth)
			normal_consistency_kernel<true><<<grid, 256, 0, s>>>(H, W, R, inv_fx, inv_fy, cx, cy, rendered_normal, map_expected, map_median, w_expected,
			                                                     w_median, loss_sum, d_normal, d_expected, d_median);
		else
			normal_consistency_kernel<false><<<grid, 256, 0, s>>>(H, W, R, inv_fx, inv_fy, cx, cy, rendered_normal, map_expected, map_median, w_expected,
			                                                      w_median, loss_sum, d_normal, d_expected, d_median);
		count_launch();
	}
	return cuda_status(cudaGetLastError(), "normal consistency");
}

int32_t rgs_normal_consistency(int32_t H, int32_t W, int32_t from_depth, float inv_fx, float inv_fy, float cx, float cy, const float* rendered_normal,
                               const float* map_expected, const float* map_median, float w_expected, float w_median, double* loss_sum,
                               float* d_normal, float* d_expected, float* d_median, void* cuda_stream) {
	if (H <= 0 || W <= 0) return fail(RGS_E_INVALID, "image size must be positive");
	if (!rendered_normal || !map_expected || !map_median || !loss_sum || !d_normal || !d_expected || !d_median) return fail(RGS_E_INVALID, "null pointer");
	return rgs_normal_consistency_rows(H, W, 0, H, from_depth, inv_fx, inv_fy, cx, cy, rendered_normal, map_expected, map_median, w_expected, w_median,
	                                   loss_sum, d_normal, d_expected, d_median, cuda_stream);
}

}  // extern "C"

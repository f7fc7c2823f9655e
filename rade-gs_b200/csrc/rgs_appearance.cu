// rgs_appearance.cu -- train.py:37-58 (L1_loss_appearance with GOF's AppearanceNetwork, scene/appearance_network.py), the
// parts that run at the crop's resolution or touch the image.  The network's low-resolution head (conv1, up1..up4) is in
// rgs_appearance_head.cu; everything else is here, in FP32 FFMA, without floating-point atomics:
//
//   downsample          center crop (a multiple of 32 per axis) -> bilinear, align_corners=True, to H/32 x W/32
//   downsample_backward adds each low-resolution sample's <= 4 taps into d_image; taps of different samples are disjoint
//                       (the stride is above 32 when an axis has 2 or more samples), so a plain read-modify-write suffices
//   tail_forward        per 30 x 14 pixel tile: x2 bilinear upsample of up4's output into shared memory with a 2-pixel halo,
//                       conv2 + bias + ReLU on the tile and a 1-pixel halo, conv3 + bias + sigmoid, mapping * crop and
//                       |. - gt|.  Writes conv2's activations (64 B per pixel) for backward, and per-CTA loss partials.
//   tail_backward       per tile: conv3 and the L1/sigmoid derivative on a 2-pixel halo from the stored activations, d_image,
//                       conv3^T and the ReLU mask on a 1-pixel halo, conv2^T; the weight/bias gradients of conv2 and conv3
//                       accumulate per CTA over a fixed set of tiles into one partial row.  Writes d(upsampled map).
//   upsample_transpose  d(up4 output) as a gather over the pixels whose bilinear taps reach each sample
//   finish kernels      fixed-order sums of the per-CTA rows
//
// Zero padding of conv2 and conv3 is at the borders of the crop-sized maps.  Backward reads the activations instead of
// recomputing them: a recompute would need conv2 on a 3-pixel halo around each tile (about 1.7x forward's conv2 FMAs).
//
// Row windows (rgs_appearance_*_rows, for row-sharded training).  A slab counts crop rows [c0, c1); every kernel takes its
// rows as parameters (`Rows`) and the whole-image entry points pass c0 = 0, c1 = H, so they run these same kernels over the
// same tiles, CTA for CTA.  The halos follow from the x2 upsample's tap rule: with sy = (H/2 - 1) / (H - 1) < 1/2, crop row y
// names the up4 rows floor(sy y) and floor(sy y) + 1, which lie in [(y - 2) / 2, (y + 2) / 2], so the gather of up4 row u
// reads d_x rows [2u - 2, 2u + 2] (it reads a row when either tap names u, also with weight 0).  A slab owns the up4 rows u
// with 2u in [c0, c1), hence:
//   d_x        rows [c0 - 2, c1 + 2)  (backward's tile rows; the tile grid starts at the window's first row)
//   d(conv2)   rows [c0 - 3, c1 + 3)
//   image, gt  rows [c0 - 4, c1 + 4)  (the loss derivative on d(conv3)'s rows)
//   act        rows [c0 - 5, c1 + 5)  (forward's tile rows)
// each clipped to the crop.  Rows a tile covers outside these windows are computed from zeros and never stored.
//
// This file also holds the C-ABI entry points rgs_appearance_* (include/rgs_b200.h).
#include <algorithm>

#include "rgs_common.cuh"

namespace rgs {

namespace {

constexpr int NT = 256;
constexpr int TW = 30, TH = 14;                    // pixel tile; conv2's region (TW+2) x (TH+2) is 256 column pairs
constexpr int NCTA = RGS_APPEARANCE_CTAS;
constexpr int GRAD_FLOATS = RGS_APPEARANCE_GRAD_FLOATS;
constexpr int OFF_B2 = 2304, OFF_W3 = 2320, OFF_B3 = 2752;  // partial row: dW2 [16,16,3,3], db2, dW3 [3,16,3,3], db3

// forward shared memory (floats): odd row strides keep the two rows a warp touches in different banks
constexpr int FXS = TW + 5, FXP = (TH + 4) * FXS;  // upsampled map, tile + 2
constexpr int FAS = TW + 3, FAP = (TH + 2) * FAS;  // conv2 activations, tile + 1
constexpr int F_SMEM = 2304 + 576 + 16 * FXP + 16 * FAP + 8;
// backward shared memory (floats)
constexpr int BAS = TW + 7, BAP = (TH + 6) * BAS;  // activations, tile + 3
constexpr int BSS = TW + 5, BSP = (TH + 4) * BSS;  // d(conv3 pre-activation), tile + 2
constexpr int BZS = TW + 3, BZP = (TH + 2) * BZS;  // d(conv2 pre-activation), tile + 1
constexpr int BXS = TW + 3, BXP = (TH + 2) * BXS + 1;  // upsampled map, tile + 1 (aliases the activations); odd plane stride
constexpr int B_SMEM = 576 + 432 + 2304 + 16 * BAP + 3 * BSP + 16 * BZP;
static_assert(16 * BXP <= 16 * BAP && 240 * 10 * 2 <= 16 * BAP, "aliases must fit in the activation buffer");

struct Crop {
	int H0, W0, H, W, top, left, h, w, Hu, Wu, tiles_x, tiles;
	float sy, sx;  // x2 upsample source scales (Hu-1)/(H-1), (Wu-1)/(W-1) in fp32, as torch computes them
};

Crop make_crop(int H0, int W0) {
	Crop k;
	k.H0 = H0; k.W0 = W0;
	k.H = H0 / 32 * 32; k.W = W0 / 32 * 32;
	k.top = H0 / 2 - k.H / 2; k.left = W0 / 2 - k.W / 2;  // train.py:40-46
	k.h = k.H / 32; k.w = k.W / 32;
	k.Hu = k.H / 2; k.Wu = k.W / 2;
	k.tiles_x = (k.W + TW - 1) / TW;
	k.tiles = k.tiles_x * ((k.H + TH - 1) / TH);
	k.sy = (float)(k.Hu - 1) / (float)(k.H - 1);
	k.sx = (float)(k.Wu - 1) / (float)(k.W - 1);
	return k;
}

constexpr int IMG_HALO = 4, ACT_HALO = 5, DX_HALO = 2;  // see the file comment

// The crop rows one call works on.  Windows are whole rows: the image / gt window holds IMAGE rows [i_row0, i_row0 + i_rows)
// (of which crop rows [i_lo, i_hi) may be read), d_image IMAGE rows [o_row0, o_row0 + o_rows); act and d_x are crop rows.
struct Rows {
	int lo, hi;            // counted rows [c0, c1): loss, weight gradients, d_image
	int t_lo, t_hi, tiles; // rows the tiles cover, the grid starting at t_lo; forward's act and backward's d_x hold these rows
	int a_lo, a_hi;        // backward: rows the activation window holds
	int i_lo, i_hi, i_row0, i_rows;
	int o_row0, o_rows;
};

// torch's align_corners=True source index: scale * dst in fp32, the tap below, the next one unless at the last row, the weight
struct Tap {
	int i0, step;
	float l1;
};
__device__ __forceinline__ Tap src_tap(float scale, int dst, int in) {
	const float s = scale * (float)dst;
	const int i0 = (int)s;
	return {i0, i0 < in - 1 ? 1 : 0, s - (float)i0};
}

__device__ __forceinline__ float bilerp(const float* __restrict__ p, Tap ty, Tap tx, int stride) {
	const float* q = p + (size_t)ty.i0 * stride + tx.i0;
	const int dy = ty.step * stride, dx = tx.step;
	const float h1 = ty.l1, h0 = 1.f - h1, w1 = tx.l1, w0 = 1.f - w1;
	return h0 * (w0 * __ldg(q) + w1 * __ldg(q + dx)) + h1 * (w0 * __ldg(q + dy) + w1 * __ldg(q + dy + dx));
}

// ---- downsample -----------------------------------------------------------------------------------------------------

// low-resolution rows [oy_lo, oy_lo + oy_rows) -> down [3, oy_rows, w]; img holds image rows [i_row0, i_row0 + i_rows)
__global__ void downsample_kernel(Crop k, float scy, float scx, int oy_lo, int oy_rows, int i_row0, int i_rows, const float* __restrict__ img,
                                  float* __restrict__ down) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= 3 * oy_rows * k.w) return;
	const int c = i / (oy_rows * k.w), oy = oy_lo + (i / k.w) % oy_rows, ox = i % k.w;
	const float* p = img + (size_t)c * i_rows * k.W0 + k.left;
	Tap ty = src_tap(scy, oy, k.H);
	ty.i0 += k.top - i_row0;  // the window's row of the upper tap
	down[i] = bilerp(p, ty, src_tap(scx, ox, k.W), k.W0);
}

// every sample's taps that land in d_img's rows: d_img holds image rows [o_row0, o_row0 + o_rows)
__global__ void downsample_backward_kernel(Crop k, float scy, float scx, int o_row0, int o_rows, const float* __restrict__ d_down,
                                           float* __restrict__ d_img) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= 3 * k.h * k.w) return;
	const int c = i / (k.h * k.w), oy = (i / k.w) % k.h, ox = i % k.w;
	const Tap ty = src_tap(scy, oy, k.H), tx = src_tap(scx, ox, k.W);
	const float g = __ldg(d_down + i);
	const float h1 = ty.l1, h0 = 1.f - h1, w1 = tx.l1, w0 = 1.f - w1;
	float* q = d_img + (size_t)c * o_rows * k.W0 + k.left + tx.i0;
	const int y0 = k.top + ty.i0 - o_row0, y1 = y0 + ty.step, dx = tx.step;
	// the same order as torch's backward scatter; when a step is 0 the second add lands on the same element
	if (y0 >= 0 && y0 < o_rows) {
		q[(size_t)y0 * k.W0] += h0 * w0 * g;
		q[(size_t)y0 * k.W0 + dx] += h0 * w1 * g;
	}
	if (y1 >= 0 && y1 < o_rows) {
		q[(size_t)y1 * k.W0] += h1 * w0 * g;
		q[(size_t)y1 * k.W0 + dx] += h1 * w1 * g;
	}
}

// ---- fused tail -------------------------------------------------------------------------------------------------------

__device__ __forceinline__ bool in_crop(const Crop& k, int y, int x) { return y >= 0 && y < k.H && x >= 0 && x < k.W; }

// fixed-order block sum (256 threads) returned to thread 0
__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
	if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
	__syncthreads();
	float s = 0.f;
	if (threadIdx.x == 0)
		for (int w = 0; w < NT / 32; w++) s += red[w];
	return s;
}

// Stage the x2-upsampled up4 map on crop rows y0 + [r0, r0 + rows), columns x0 + [c0, c0 + cols); zero outside the crop.
__device__ __forceinline__ void stage_upsampled(const Crop& k, const float* __restrict__ up4, int y0, int x0, int r0, int c0, int rows, int cols,
                                                float* s, int stride, int plane) {
	const size_t up_plane = (size_t)k.Hu * k.Wu;
	for (int i = threadIdx.x; i < 16 * rows * cols; i += NT) {
		const int c = i / (rows * cols), r = (i / cols) % rows, q = i % cols;
		const int y = y0 + r0 + r, x = x0 + c0 + q;
		s[c * plane + r * stride + q] = in_crop(k, y, x) ? bilerp(up4 + c * up_plane, src_tap(k.sy, y, k.Hu), src_tap(k.sx, x, k.Wu), k.Wu) : 0.f;
	}
}

// 3x3 convolution over two horizontally adjacent outputs, 16 output channels: a0/a1 += sum_ci,dy,dx w[ci][dy][dx][co] * in.
// `in` points at input row `dy = 0` of the pair's first output column; FLIP reads taps mirrored (a transposed convolution).
template <int CIN, bool FLIP>
__device__ __forceinline__ void conv16_pair(const float* in, int plane, int stride, const float* w, float (&a0)[16], float (&a1)[16]) {
#pragma unroll 2
	for (int ci = 0; ci < CIN; ci++) {
#pragma unroll
		for (int dy = 0; dy < 3; dy++) {
			const float* row = in + ci * plane + (FLIP ? 2 - dy : dy) * stride;
			const float v[4] = {row[0], row[1], row[2], row[3]};
#pragma unroll
			for (int dx = 0; dx < 3; dx++) {
				const float p0 = v[FLIP ? 2 - dx : dx], p1 = v[FLIP ? 3 - dx : dx + 1];
				const float4* wr = reinterpret_cast<const float4*>(w + ((ci * 3 + dy) * 3 + dx) * 16);
#pragma unroll
				for (int j = 0; j < 4; j++) {
					const float4 q = wr[j];
					a0[4 * j] = fmaf(q.x, p0, a0[4 * j]); a0[4 * j + 1] = fmaf(q.y, p0, a0[4 * j + 1]);
					a0[4 * j + 2] = fmaf(q.z, p0, a0[4 * j + 2]); a0[4 * j + 3] = fmaf(q.w, p0, a0[4 * j + 3]);
					a1[4 * j] = fmaf(q.x, p1, a1[4 * j]); a1[4 * j + 1] = fmaf(q.y, p1, a1[4 * j + 1]);
					a1[4 * j + 2] = fmaf(q.z, p1, a1[4 * j + 2]); a1[4 * j + 3] = fmaf(q.w, p1, a1[4 * j + 3]);
				}
			}
		}
	}
}

// conv3 (16 -> 3) over two adjacent outputs; w is [ci][dy][dx][4] (the 4th lane is padding)
__device__ __forceinline__ void conv3_pair(const float* in, int plane, int stride, const float* w, float (&s0)[3], float (&s1)[3]) {
#pragma unroll 4
	for (int ci = 0; ci < 16; ci++) {
#pragma unroll
		for (int dy = 0; dy < 3; dy++) {
			const float* row = in + ci * plane + dy * stride;
			const float v[4] = {row[0], row[1], row[2], row[3]};
#pragma unroll
			for (int dx = 0; dx < 3; dx++) {
				const float4 q = reinterpret_cast<const float4*>(w)[(ci * 3 + dy) * 3 + dx];
				s0[0] = fmaf(q.x, v[dx], s0[0]); s0[1] = fmaf(q.y, v[dx], s0[1]); s0[2] = fmaf(q.z, v[dx], s0[2]);
				s1[0] = fmaf(q.x, v[dx + 1], s1[0]); s1[1] = fmaf(q.y, v[dx + 1], s1[1]); s1[2] = fmaf(q.z, v[dx + 1], s1[2]);
			}
		}
	}
}

__device__ __forceinline__ float sigmoid(float s) { return 1.f / (1.f + expf(-s)); }  // torch's CUDA sigmoid

// conv3's weights [3,16,3,3] -> [ci][tap][4]
__device__ __forceinline__ void load_w3_fwd(const float* __restrict__ w3, float* s) {
	for (int i = threadIdx.x; i < 576; i += NT) {
		const int co = i & 3, tap = (i >> 2) % 9, ci = i / 36;
		s[i] = co < 3 ? __ldg(w3 + (co * 16 + ci) * 9 + tap) : 0.f;
	}
}

__global__ void __launch_bounds__(NT, 2) tail_forward_kernel(Crop k, Rows R, const float* __restrict__ img, const float* __restrict__ gt,
                                                             const float* __restrict__ up4, const float* __restrict__ w2,
                                                             const float* __restrict__ b2, const float* __restrict__ w3,
                                                             const float* __restrict__ b3, float* __restrict__ act, float* __restrict__ out,
                                                             double* __restrict__ partials) {
	extern __shared__ float4 smem_f4[];
	float* sW2 = reinterpret_cast<float*>(smem_f4);  // [ci][tap][co]
	float* sW3 = sW2 + 2304;                         // [ci][tap][4]
	float* sX = sW3 + 576;
	float* sA = sX + 16 * FXP;
	float* red = sA + 16 * FAP;
	const int t = threadIdx.x;
	for (int i = t; i < 2304; i += NT) {
		const int co = i / 144, ci = (i / 9) % 16, tap = i % 9;
		sW2[(ci * 9 + tap) * 16 + co] = __ldg(w2 + i);
	}
	load_w3_fwd(w3, sW3);
	const size_t plane0 = (size_t)R.i_rows * k.W0, crop_plane = (size_t)k.H * k.W, act_plane = (size_t)(R.t_hi - R.t_lo) * k.W;
	const size_t org = (size_t)(k.top - R.i_row0) * k.W0 + k.left;  // wraps below the window's first row, which is never read
	double acc = 0.0;
	for (int tile = blockIdx.x; tile < R.tiles; tile += gridDim.x) {
		const int y0 = R.t_lo + (tile / k.tiles_x) * TH, x0 = (tile % k.tiles_x) * TW;
		__syncthreads();  // the previous tile's readers are done
		stage_upsampled(k, up4, y0, x0, -2, -2, TH + 4, TW + 4, sX, FXS, FXP);
		__syncthreads();
		{  // conv2 + bias + ReLU on the tile + 1: row t / 16, columns 2 (t % 16) + {0, 1}
			const int r = t >> 4, q = (t & 15) * 2;
			float a0[16], a1[16];
#pragma unroll
			for (int j = 0; j < 16; j++) a0[j] = a1[j] = 0.f;
			conv16_pair<16, false>(sX + r * FXS + q, FXP, FXS, sW2, a0, a1);
			const int y = y0 - 1 + r;
#pragma unroll
			for (int e = 0; e < 2; e++) {
				const int x = x0 - 1 + q + e;
				const bool in = in_crop(k, y, x);
				const bool own = in && r >= 1 && r <= TH && q + e >= 1 && q + e <= TW && y < R.t_hi;
#pragma unroll
				for (int co = 0; co < 16; co++) {
					const float v = in ? fmaxf((e ? a1[co] : a0[co]) + __ldg(b2 + co), 0.f) : 0.f;
					sA[co * FAP + r * FAS + q + e] = v;
					if (own && act != nullptr) act[co * act_plane + (size_t)(y - R.t_lo) * k.W + x] = v;
				}
			}
		}
		__syncthreads();
		float l1 = 0.f;
		if (t < TH * (TW / 2)) {  // conv3 + sigmoid, mapping * crop, |. - gt| on the tile
			const int r = t / (TW / 2), q = (t % (TW / 2)) * 2;
			float s0[3] = {0.f, 0.f, 0.f}, s1[3] = {0.f, 0.f, 0.f};
			conv3_pair(sA + r * FAS + q, FAP, FAS, sW3, s0, s1);
			const int y = y0 + r;
#pragma unroll
			for (int e = 0; e < 2; e++) {
				const int x = x0 + q + e;
				if (y >= R.lo && y < R.hi && x < k.W) {
#pragma unroll
					for (int c = 0; c < 3; c++) {
						const float m = sigmoid((e ? s1[c] : s0[c]) + __ldg(b3 + c));
						const size_t o = c * plane0 + org + (size_t)y * k.W0 + x;
						const float tv = m * __ldg(img + o);
						l1 += fabsf(tv - __ldg(gt + o));
						if (out != nullptr) out[c * crop_plane + (size_t)y * k.W + x] = tv;
					}
				}
			}
		}
		const float s = block_sum(l1, red);
		if (t == 0) acc += (double)s;
	}
	if (t == 0) partials[blockIdx.x] = acc;
}

// the mean as float32 into loss, or (a row form) the fp64 sum into sum
__global__ void loss_finish_kernel(const double* __restrict__ partials, int rows, double n, float* __restrict__ loss, double* __restrict__ sum) {
	double s = 0.0;
	for (int b = 0; b < rows; b++) s += partials[b];
	if (sum != nullptr) sum[0] = s;
	else loss[0] = (float)(s / n);
}

// Weight gradient of one 3x3 convolution over the tile's pixels: acc[dy*3+dx] += sum_p dout[p] * in[p + (dy-1, dx-1)], and
// bias += sum_p dout[p].  dout is addressed at the pixel, in at the pixel's (dy, dx) = (0, 0) tap; rows r0, r0 + rstep, ...
__device__ __forceinline__ void wgrad_rows(const float* dout, int dstride, const float* in, int istride, int rows, int cols, int r0, int rstep,
                                           float (&w)[9], float& b) {
	for (int r = r0; r < rows; r += rstep) {
		const float* d = dout + r * dstride;
		const float* x = in + r * istride;
		float a[3][3];
#pragma unroll
		for (int dy = 0; dy < 3; dy++) { a[dy][1] = x[dy * istride]; a[dy][2] = x[dy * istride + 1]; }
		for (int c = 0; c < cols; c++) {
#pragma unroll
			for (int dy = 0; dy < 3; dy++) { a[dy][0] = a[dy][1]; a[dy][1] = a[dy][2]; a[dy][2] = x[dy * istride + c + 2]; }
			const float g = d[c];
			b += g;
#pragma unroll
			for (int dy = 0; dy < 3; dy++)
#pragma unroll
				for (int dx = 0; dx < 3; dx++) w[dy * 3 + dx] = fmaf(g, a[dy][dx], w[dy * 3 + dx]);
		}
	}
}

__global__ void __launch_bounds__(NT, 2) tail_backward_kernel(Crop k, Rows R, const float* __restrict__ img, const float* __restrict__ gt,
                                                              const float* __restrict__ up4, const float* __restrict__ act, const float* __restrict__ w2,
                                                              const float* __restrict__ w3, const float* __restrict__ b3,
                                                              const float* __restrict__ upstream, float* __restrict__ d_img,
                                                              float* __restrict__ d_x, double* __restrict__ partials) {
	extern __shared__ float4 smem_f4[];
	float* sW3f = reinterpret_cast<float*>(smem_f4);  // [ci][tap][4]
	float* sW3b = sW3f + 576;                         // [co][tap][ci]
	float* sW2b = sW3b + 432;                         // [co][tap][ci]
	float* sA = sW2b + 2304;
	float* sS = sA + 16 * BAP;
	float* sZ = sS + 3 * BSP;
	float* sX = sA;  // once the activations are no longer read
	const int t = threadIdx.x;
	load_w3_fwd(w3, sW3f);
	for (int i = t; i < 432; i += NT) {
		const int co = i / 144, ci = (i / 9) % 16, tap = i % 9;
		sW3b[(co * 9 + tap) * 16 + ci] = __ldg(w3 + i);
	}
	for (int i = t; i < 2304; i += NT) {
		const int co = i / 144, ci = (i / 9) % 16, tap = i % 9;
		sW2b[(co * 9 + tap) * 16 + ci] = __ldg(w2 + i);
	}
	const float gup = (upstream != nullptr ? __ldg(upstream) : 1.f) / (float)(3 * k.H * k.W);  // mean's backward
	const size_t plane0 = (size_t)R.i_rows * k.W0, out_plane = (size_t)R.o_rows * k.W0;
	const size_t act_plane = (size_t)(R.a_hi - R.a_lo) * k.W, dx_plane = (size_t)(R.t_hi - R.t_lo) * k.W;
	const size_t org = (size_t)(k.top - R.i_row0) * k.W0 + k.left, out_org = (size_t)(k.top - R.o_row0) * k.W0 + k.left;  // may wrap, as in forward
	// weight-gradient ownership: conv2 (co, ci) = (t / 16, t % 16); conv3 (co, ci) = ((t % 48) / 16, t % 16), rows t / 48 + 5j
	const int c2o = t >> 4, c2i = t & 15, c3p = t % 48, c3g = t / 48;
	float g2[10], g3[10];  // across this CTA's tiles (at most a few dozen tile sums); rows are added across CTAs in fp64
#pragma unroll
	for (int j = 0; j < 10; j++) g2[j] = g3[j] = 0.f;
	for (int tile = blockIdx.x; tile < R.tiles; tile += gridDim.x) {
		const int y0 = R.t_lo + (tile / k.tiles_x) * TH, x0 = (tile % k.tiles_x) * TW;
		// the weight gradients count the tile's rows in [c0, c1) only
		const int rows_lo = max(0, R.lo - y0), rows = min(TH, R.hi - y0), cols = min(TW, k.W - x0);
		__syncthreads();
		for (int i = t; i < 16 * (TH + 6) * (TW + 6); i += NT) {  // activations on the tile + 3, zero outside the crop
			const int c = i / ((TH + 6) * (TW + 6)), r = (i / (TW + 6)) % (TH + 6), q = i % (TW + 6);
			const int y = y0 - 3 + r, x = x0 - 3 + q;
			const bool held = in_crop(k, y, x) && y >= R.a_lo && y < R.a_hi;
			sA[c * BAP + r * BAS + q] = held ? __ldg(act + c * act_plane + (size_t)(y - R.a_lo) * k.W + x) : 0.f;
		}
		__syncthreads();
		for (int p = t; p < (TH + 4) * ((TW + 4) / 2); p += NT) {  // conv3 + the loss derivative on the tile + 2
			const int r = p / ((TW + 4) / 2), q = (p % ((TW + 4) / 2)) * 2;
			float s0[3] = {0.f, 0.f, 0.f}, s1[3] = {0.f, 0.f, 0.f};
			conv3_pair(sA + r * BAS + q, BAP, BAS, sW3f, s0, s1);
			const int y = y0 - 2 + r;
#pragma unroll
			for (int e = 0; e < 2; e++) {
				const int x = x0 - 2 + q + e;
				const bool in = in_crop(k, y, x) && y >= R.i_lo && y < R.i_hi;
				const bool own = in && r >= 2 && r < TH + 2 && q + e >= 2 && q + e < TW + 2 && y >= R.lo && y < R.hi;
#pragma unroll
				for (int c = 0; c < 3; c++) {
					float ds = 0.f;
					if (in) {
						const float m = sigmoid((e ? s1[c] : s0[c]) + __ldg(b3 + c));
						const size_t o = c * plane0 + org + (size_t)y * k.W0 + x;
						const float iv = __ldg(img + o), diff = m * iv - __ldg(gt + o);
						const float dt = (diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f)) * gup;  // abs backward: sgn(0) = 0
						if (own) d_img[c * out_plane + out_org + (size_t)y * k.W0 + x] = dt * m;
						ds = dt * iv * (1.f - m) * m;  // mul backward, then sigmoid_backward: grad * (1 - y) * y
					}
					sS[c * BSP + r * BSS + q + e] = ds;
				}
			}
		}
		__syncthreads();
		{  // conv3^T and the ReLU mask on the tile + 1
			const int r = t >> 4, q = (t & 15) * 2;
			float a0[16], a1[16];
#pragma unroll
			for (int j = 0; j < 16; j++) a0[j] = a1[j] = 0.f;
			conv16_pair<3, true>(sS + r * BSS + q, BSP, BSS, sW3b, a0, a1);
#pragma unroll
			for (int e = 0; e < 2; e++)
#pragma unroll
				for (int ci = 0; ci < 16; ci++)
					sZ[ci * BZP + r * BZS + q + e] = sA[ci * BAP + (r + 2) * BAS + q + e + 2] > 0.f ? (e ? a1[ci] : a0[ci]) : 0.f;
		}
		if (c3g < 5) {  // conv3's weight gradient: d(pre-sigmoid) on the tile x activations on the tile + 1
			float w[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, b = 0.f;
			wgrad_rows(sS + (c3p >> 4) * BSP + 2 * BSS + 2, BSS, sA + c2i * BAP + 2 * BAS + 2, BAS, rows, cols, rows_lo + c3g, 5, w, b);
#pragma unroll
			for (int j = 0; j < 9; j++) g3[j] += w[j];
			g3[9] += b;
		}
		__syncthreads();
		stage_upsampled(k, up4, y0, x0, -1, -1, TH + 2, TW + 2, sX, BXS, BXP);
		__syncthreads();
		{  // conv2's weight gradient: d(pre-ReLU) on the tile x upsampled map on the tile + 1
			float w[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, b = 0.f;
			wgrad_rows(sZ + c2o * BZP + BZS + 1, BZS, sX + c2i * BXP, BXS, rows, cols, rows_lo, 1, w, b);
#pragma unroll
			for (int j = 0; j < 9; j++) g2[j] += w[j];
			g2[9] += b;
		}
		if (t < TH * (TW / 2)) {  // conv2^T on the tile -> d(upsampled map)
			const int r = t / (TW / 2), q = (t % (TW / 2)) * 2;
			float a0[16], a1[16];
#pragma unroll
			for (int j = 0; j < 16; j++) a0[j] = a1[j] = 0.f;
			conv16_pair<16, true>(sZ + r * BZS + q, BZP, BZS, sW2b, a0, a1);
			const int y = y0 + r;
#pragma unroll
			for (int e = 0; e < 2; e++) {
				const int x = x0 + q + e;
				if (y < R.t_hi && x < k.W)
#pragma unroll
					for (int ci = 0; ci < 16; ci++) d_x[ci * dx_plane + (size_t)(y - R.t_lo) * k.W + x] = e ? a1[ci] : a0[ci];
			}
		}
	}
	// this CTA's partial row; conv3's five row groups are added in group order
	double* row = partials + (size_t)blockIdx.x * GRAD_FLOATS;
#pragma unroll
	for (int j = 0; j < 9; j++) row[(c2o * 16 + c2i) * 9 + j] = g2[j];
	if (c2i == 0) row[OFF_B2 + c2o] = g2[9];
	__syncthreads();
	double* red = reinterpret_cast<double*>(sA);
	if (c3g < 5)
#pragma unroll
		for (int j = 0; j < 10; j++) red[t * 10 + j] = g3[j];
	__syncthreads();
	if (t < 48) {
		for (int j = 0; j < 10; j++) {
			double s = 0.0;
			for (int g = 0; g < 5; g++) s += red[(g * 48 + t) * 10 + j];
			if (j < 9) row[OFF_W3 + t * 9 + j] = s;
			else if (c2i == 0) row[OFF_B3 + (t >> 4)] = s;
		}
	}
}

// the partial rows summed in row order, cast into d_w2, d_b2, d_w3, d_b3, or (a row form) kept in fp64 in sum_row
__global__ void grad_finish_kernel(const double* __restrict__ partials, int rows, float* __restrict__ d_w2, float* __restrict__ d_b2, float* __restrict__ d_w3,
                                   float* __restrict__ d_b3, double* __restrict__ sum_row) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= GRAD_FLOATS) return;
	double s = 0.0;
	for (int b = 0; b < rows; b++) s += partials[(size_t)b * GRAD_FLOATS + i];
	if (sum_row != nullptr) {
		sum_row[i] = s;
		return;
	}
	const float v = (float)s;
	if (i < OFF_B2) d_w2[i] = v;
	else if (i < OFF_W3) d_b2[i - OFF_B2] = v;
	else if (i < OFF_B3) d_w3[i - OFF_W3] = v;
	else d_b3[i - OFF_B3] = v;
}

// Transpose of the x2 upsample as a gather: d_up4[c][u][v] = sum over crop pixels (y, x) whose taps reach (u, v) of
// (row weight) * (column weight) * d_x[c][y][x], with the taps decided exactly as in forward.  scale < 1/2 bounds the
// candidates to y in [2u - 3, 2u + 4]; the rows actually read are [2u - 2, 2u + 2] (the file comment).
__device__ __forceinline__ float tap_weight(float scale, int y, int u, int in) {
	const Tap tp = src_tap(scale, y, in);
	return (tp.i0 == u ? 1.f - tp.l1 : 0.f) + (tp.i0 + tp.step == u ? tp.l1 : 0.f);
}

// up4 rows [u_lo, u_lo + u_rows) -> d_up4 [16, u_rows, Wu]; d_x holds crop rows [x_row0, x_row0 + x_rows)
__global__ void upsample_transpose_kernel(Crop k, int u_lo, int u_rows, int x_row0, int x_rows, const float* __restrict__ d_x, float* __restrict__ d_up4) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= 16 * u_rows * k.Wu) return;
	const int c = i / (u_rows * k.Wu), u = u_lo + (i / k.Wu) % u_rows, v = i % k.Wu;
	const float* p = d_x + (size_t)c * x_rows * k.W;
	const int x_lo = max(0, 2 * v - 3), x_hi = min(k.W - 1, 2 * v + 4);
	float acc = 0.f;
	for (int y = max(0, 2 * u - 3); y <= min(k.H - 1, 2 * u + 4); y++) {
		const Tap ty = src_tap(k.sy, y, k.Hu);
		if (ty.i0 != u && ty.i0 + ty.step != u) continue;
		const float wy = tap_weight(k.sy, y, u, k.Hu);
		float r = 0.f;
		for (int x = x_lo; x <= x_hi; x++) {
			const Tap tx = src_tap(k.sx, x, k.Wu);
			if (tx.i0 != v && tx.i0 + tx.step != v) continue;
			r = fmaf(tap_weight(k.sx, x, v, k.Wu), __ldg(p + (size_t)(y - x_row0) * k.W + x), r);
		}
		acc = fmaf(wy, r, acc);
	}
	d_up4[i] = acc;
}

float down_scale(int in, int out) { return out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f; }  // torch: 0 for one sample

size_t g_fwd_smem[64], g_bwd_smem[64];

int32_t appearance_size(int32_t H0, int32_t W0) {
	if (H0 < 32 || W0 < 32) return fail(RGS_E_INVALID, "appearance loss: the image must be at least 32 x 32");
	if ((int64_t)H0 * W0 > (int64_t)1 << 28) return fail(RGS_E_INVALID, "appearance loss: image too large");
	return RGS_OK;
}

// What the slab of image rows [row_lo, row_hi) counts, owns and reads (include/rgs_b200.h, rgs_appearance_row_windows).
// Every range is [lo, hi) and empty when the slab holds no crop row.
struct Slab {
	int c0, c1;        // crop rows counted
	int oy_lo, oy_hi;  // low-resolution rows whose upper tap (int)(scy oy) is in [c0, c1)
	int u_lo, u_hi;    // up4 rows u with 2u in [c0, c1)
	int a_lo, a_hi;    // activations: [c0 - 5, c1 + 5) in the crop
	int x_lo, x_hi;    // d_x: [c0 - 2, c1 + 2) in the crop
	int i_lo, i_hi;    // image and gt rows backward reads: [c0 - 4, c1 + 4) in the crop
};

Slab make_slab(const Crop& k, int row_lo, int row_hi) {
	Slab s;
	s.c0 = std::min(std::max(row_lo - k.top, 0), k.H);
	s.c1 = std::min(std::max(row_hi - k.top, 0), k.H);
	if (s.c1 <= s.c0) {
		s.c1 = s.c0;
		s.oy_lo = s.oy_hi = s.u_lo = s.u_hi = 0;
		s.a_lo = s.a_hi = s.x_lo = s.x_hi = s.i_lo = s.i_hi = s.c0;
		return s;
	}
	// the device's source index, in the same fp32 arithmetic (src_tap); it does not decrease with oy, so the rows are contiguous
	const float scy = down_scale(k.H, k.h);
	s.oy_lo = s.oy_hi = 0;
	for (int oy = 0, any = 0; oy < k.h; oy++) {
		const int i0 = (int)(scy * (float)oy);
		if (i0 < s.c0 || i0 >= s.c1) continue;
		if (!any) s.oy_lo = oy;
		s.oy_hi = oy + 1;
		any = 1;
	}
	s.u_lo = (s.c0 + 1) / 2;
	s.u_hi = (s.c1 + 1) / 2;
	s.a_lo = std::max(0, s.c0 - ACT_HALO); s.a_hi = std::min(k.H, s.c1 + ACT_HALO);
	s.x_lo = std::max(0, s.c0 - DX_HALO); s.x_hi = std::min(k.H, s.c1 + DX_HALO);
	s.i_lo = std::max(0, s.c0 - IMG_HALO); s.i_hi = std::min(k.H, s.c1 + IMG_HALO);
	return s;
}

int32_t row_range(int32_t H0, int32_t row_lo, int32_t row_hi) {
	if (row_lo < 0 || row_hi > H0 || row_lo > row_hi) return fail(RGS_E_INVALID, "appearance loss: row range out of the image");
	return RGS_OK;
}

// The image (and gt) window [image_lo, image_lo + image_rows) must lie in the image and hold crop rows [need_lo, need_hi).
int32_t image_window(const Crop& k, int32_t image_lo, int32_t image_rows, int need_lo, int need_hi) {
	if (image_lo < 0 || image_rows < 0 || (int64_t)image_lo + image_rows > k.H0)
		return fail(RGS_E_INVALID, "appearance loss: the image window [" + std::to_string(image_lo) + ", " + std::to_string((int64_t)image_lo + image_rows) +
		                               ") is not inside the image's " + std::to_string(k.H0) + " rows");
	if (need_lo < need_hi && (k.top + need_lo < image_lo || k.top + need_hi > image_lo + image_rows))
		return fail(RGS_E_INVALID, "appearance loss: the image window [" + std::to_string(image_lo) + ", " + std::to_string(image_lo + image_rows) +
		                               ") lacks halo rows: it must hold image rows [" + std::to_string(k.top + need_lo) + ", " +
		                               std::to_string(k.top + need_hi) + ")");
	return RGS_OK;
}

Rows tail_rows(const Crop& k, const Slab& s, int t_lo, int t_hi, int32_t image_lo, int32_t image_rows, int32_t row_lo, int32_t row_hi) {
	Rows R;
	R.lo = s.c0; R.hi = s.c1;
	R.t_lo = t_lo; R.t_hi = t_hi;
	R.tiles = k.tiles_x * ((t_hi - t_lo + TH - 1) / TH);
	R.a_lo = s.a_lo; R.a_hi = s.a_hi;
	// the crop rows the window holds
	R.i_lo = std::max(0, image_lo - k.top); R.i_hi = std::min(k.H, image_lo + image_rows - k.top);
	R.i_row0 = image_lo; R.i_rows = image_rows;
	R.o_row0 = row_lo; R.o_rows = row_hi - row_lo;
	return R;
}

int32_t l1_forward(const Crop& k, const Slab& s, int32_t image_lo, int32_t image_rows, int32_t row_lo, int32_t row_hi, const float* image, const float* gt,
                   const float* up4, const float* w2, const float* b2, const float* w3, const float* b3, float* act, float* transformed,
                   double* partials, float* loss, double* loss_sum, cudaStream_t st) {
	if (s.c1 == s.c0) {  // no crop row: nothing counted
		RGS_CUDA_TRY(cudaMemsetAsync(loss_sum, 0, sizeof(double), st));
		return RGS_OK;
	}
	const Rows R = tail_rows(k, s, s.a_lo, s.a_hi, image_lo, image_rows, row_lo, row_hi);
	const size_t bytes = F_SMEM * sizeof(float);
	ensure_dynamic_smem(tail_forward_kernel, bytes, g_fwd_smem);
	tail_forward_kernel<<<NCTA, NT, bytes, st>>>(k, R, image, gt, up4, w2, b2, w3, b3, act, transformed, partials);
	loss_finish_kernel<<<1, 1, 0, st>>>(partials, NCTA, 3.0 * k.H * k.W, loss, loss_sum);
	count_launch(2);
	return cuda_status(cudaGetLastError(), "appearance l1 forward");
}

int32_t l1_backward(const Crop& k, const Slab& s, int32_t image_lo, int32_t image_rows, int32_t row_lo, int32_t row_hi, const float* image, const float* gt,
                    const float* up4, const float* act, const float* w2, const float* w3, const float* b3, const float* upstream, float* d_image,
                    float* d_up4, float* d_w2, float* d_b2, float* d_w3, float* d_b3, double* grad_row, double* partials, float* d_x, cudaStream_t st) {
	// outside the crop (slice_backward's zero fill)
	RGS_CUDA_TRY(cudaMemsetAsync(d_image, 0, (size_t)3 * (row_hi - row_lo) * k.W0 * sizeof(float), st));
	if (s.c1 == s.c0) {
		RGS_CUDA_TRY(cudaMemsetAsync(grad_row, 0, GRAD_FLOATS * sizeof(double), st));
		return RGS_OK;
	}
	const Rows R = tail_rows(k, s, s.x_lo, s.x_hi, image_lo, image_rows, row_lo, row_hi);
	const size_t bytes = B_SMEM * sizeof(float);
	ensure_dynamic_smem(tail_backward_kernel, bytes, g_bwd_smem);
	tail_backward_kernel<<<NCTA, NT, bytes, st>>>(k, R, image, gt, up4, act, w2, w3, b3, upstream, d_image, d_x, partials);
	grad_finish_kernel<<<(GRAD_FLOATS + 255) / 256, 256, 0, st>>>(partials, NCTA, d_w2, d_b2, d_w3, d_b3, grad_row);
	const int n = 16 * (s.u_hi - s.u_lo) * k.Wu;
	if (n > 0) upsample_transpose_kernel<<<(n + 255) / 256, 256, 0, st>>>(k, s.u_lo, s.u_hi - s.u_lo, s.x_lo, s.x_hi - s.x_lo, d_x, d_up4);
	count_launch(n > 0 ? 3 : 2);
	return cuda_status(cudaGetLastError(), "appearance l1 backward");
}

}  // namespace
}  // namespace rgs

using namespace rgs;

extern "C" {

int32_t rgs_appearance_row_windows(int32_t H0, int32_t W0, int32_t row_lo, int32_t row_hi, int32_t* windows) {
	if (const int32_t rc = appearance_size(H0, W0)) return rc;
	if (const int32_t rc = row_range(H0, row_lo, row_hi)) return rc;
	if (!windows) return fail(RGS_E_INVALID, "null pointer");
	const Slab s = make_slab(make_crop(H0, W0), row_lo, row_hi);
	const int32_t out[RGS_APPEARANCE_WINDOWS] = {s.c0, s.c1, s.oy_lo, s.oy_hi, s.u_lo, s.u_hi, s.a_lo, s.a_hi, s.x_lo, s.x_hi, s.i_lo, s.i_hi};
	for (int i = 0; i < RGS_APPEARANCE_WINDOWS; i++) windows[i] = out[i];
	return RGS_OK;
}

int32_t rgs_appearance_downsample_rows(int32_t H0, int32_t W0, int32_t row_lo, int32_t row_hi, const float* image, int32_t image_lo, int32_t image_rows,
                                       float* down, void* cuda_stream) {
	if (const int32_t rc = appearance_size(H0, W0)) return rc;
	if (const int32_t rc = row_range(H0, row_lo, row_hi)) return rc;
	const Crop k = make_crop(H0, W0);
	const Slab s = make_slab(k, row_lo, row_hi);
	const int n = 3 * (s.oy_hi - s.oy_lo) * k.w;
	if (n == 0) return RGS_OK;
	if (!image || !down) return fail(RGS_E_INVALID, "null pointer");
	// the owned samples' taps: rows [c0, c1] of the crop, the last one only below the slab
	if (const int32_t rc = image_window(k, image_lo, image_rows, s.c0, std::min(k.H, s.c1 + 1))) return rc;
	downsample_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)cuda_stream>>>(k, down_scale(k.H, k.h), down_scale(k.W, k.w), s.oy_lo, s.oy_hi - s.oy_lo,
	                                                                          image_lo, image_rows, image, down);
	count_launch();
	return cuda_status(cudaGetLastError(), "appearance downsample");
}

int32_t rgs_appearance_downsample(int32_t H0, int32_t W0, const float* image, float* down, void* cuda_stream) {
	if (const int32_t rc = appearance_size(H0, W0)) return rc;
	if (!image || !down) return fail(RGS_E_INVALID, "null pointer");
	return rgs_appearance_downsample_rows(H0, W0, 0, H0, image, 0, H0, down, cuda_stream);
}

int32_t rgs_appearance_downsample_backward_rows(int32_t H0, int32_t W0, int32_t row_lo, int32_t row_hi, const float* d_down, float* d_image,
                                                void* cuda_stream) {
	if (const int32_t rc = appearance_size(H0, W0)) return rc;
	if (const int32_t rc = row_range(H0, row_lo, row_hi)) return rc;
	if (row_hi == row_lo) return RGS_OK;
	if (!d_down || !d_image) return fail(RGS_E_INVALID, "null pointer");
	const Crop k = make_crop(H0, W0);
	const int n = 3 * k.h * k.w;
	downsample_backward_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)cuda_stream>>>(k, down_scale(k.H, k.h), down_scale(k.W, k.w), row_lo, row_hi - row_lo,
	                                                                                   d_down, d_image);
	count_launch();
	return cuda_status(cudaGetLastError(), "appearance downsample backward");
}

int32_t rgs_appearance_downsample_backward(int32_t H0, int32_t W0, const float* d_down, float* d_image, void* cuda_stream) {
	if (const int32_t rc = appearance_size(H0, W0)) return rc;
	if (!d_down || !d_image) return fail(RGS_E_INVALID, "null pointer");
	return rgs_appearance_downsample_backward_rows(H0, W0, 0, H0, d_down, d_image, cuda_stream);
}

int32_t rgs_appearance_l1_forward_rows(int32_t H0, int32_t W0, int32_t row_lo, int32_t row_hi, const float* image, const float* gt, int32_t image_lo,
                                       int32_t image_rows, const float* up4, const float* w2, const float* b2, const float* w3, const float* b3, float* act,
                                       double* partials, double* loss_sum, void* cuda_stream) {
	if (const int32_t rc = appearance_size(H0, W0)) return rc;
	if (const int32_t rc = row_range(H0, row_lo, row_hi)) return rc;
	if (!loss_sum) return fail(RGS_E_INVALID, "null pointer");
	const Crop k = make_crop(H0, W0);
	const Slab s = make_slab(k, row_lo, row_hi);
	if (s.c1 > s.c0) {
		if (!image || !gt || !up4 || !w2 || !b2 || !w3 || !b3 || !act || !partials) return fail(RGS_E_INVALID, "null pointer");
		if (const int32_t rc = image_window(k, image_lo, image_rows, s.c0, s.c1)) return rc;
	}
	return l1_forward(k, s, image_lo, image_rows, row_lo, row_hi, image, gt, up4, w2, b2, w3, b3, act, nullptr, partials, nullptr, loss_sum,
	                  (cudaStream_t)cuda_stream);
}

int32_t rgs_appearance_l1_forward(int32_t H0, int32_t W0, const float* image, const float* gt, const float* up4, const float* w2, const float* b2,
                                  const float* w3, const float* b3, float* act, float* transformed, double* partials, float* loss, void* cuda_stream) {
	if (const int32_t rc = appearance_size(H0, W0)) return rc;
	if (!image || !gt || !up4 || !w2 || !b2 || !w3 || !b3 || !partials || !loss) return fail(RGS_E_INVALID, "null pointer");
	const Crop k = make_crop(H0, W0);
	return l1_forward(k, make_slab(k, 0, H0), 0, H0, 0, H0, image, gt, up4, w2, b2, w3, b3, act, transformed, partials, loss, nullptr,
	                  (cudaStream_t)cuda_stream);
}

int32_t rgs_appearance_l1_backward_rows(int32_t H0, int32_t W0, int32_t row_lo, int32_t row_hi, const float* image, const float* gt, int32_t image_lo,
                                        int32_t image_rows, const float* up4, const float* act, const float* w2, const float* w3, const float* b3,
                                        const float* upstream, float* d_image, float* d_up4, double* grad_row, double* partials, float* d_x,
                                        void* cuda_stream) {
	if (const int32_t rc = appearance_size(H0, W0)) return rc;
	if (const int32_t rc = row_range(H0, row_lo, row_hi)) return rc;
	if (!grad_row || (row_hi > row_lo && !d_image)) return fail(RGS_E_INVALID, "null pointer");
	const Crop k = make_crop(H0, W0);
	const Slab s = make_slab(k, row_lo, row_hi);
	if (s.c1 > s.c0) {
		// a slab of one odd crop row owns no up4 row: its d_up4 is empty and may be NULL
		if (!image || !gt || !up4 || !act || !w2 || !w3 || !b3 || (!d_up4 && s.u_hi > s.u_lo) || !partials || !d_x)
			return fail(RGS_E_INVALID, "null pointer");
		if (const int32_t rc = image_window(k, image_lo, image_rows, s.i_lo, s.i_hi)) return rc;
	}
	return l1_backward(k, s, image_lo, image_rows, row_lo, row_hi, image, gt, up4, act, w2, w3, b3, upstream, d_image, d_up4, nullptr, nullptr, nullptr,
	                   nullptr, grad_row, partials, d_x, (cudaStream_t)cuda_stream);
}

int32_t rgs_appearance_l1_backward(int32_t H0, int32_t W0, const float* image, const float* gt, const float* up4, const float* act, const float* w2,
                                   const float* w3, const float* b3, const float* upstream, float* d_image, float* d_up4, float* d_w2, float* d_b2,
                                   float* d_w3, float* d_b3, double* partials, float* d_x, void* cuda_stream) {
	if (const int32_t rc = appearance_size(H0, W0)) return rc;
	if (!image || !gt || !up4 || !act || !w2 || !w3 || !b3 || !d_image || !d_up4 || !d_w2 || !d_b2 || !d_w3 || !d_b3 || !partials || !d_x)
		return fail(RGS_E_INVALID, "null pointer");
	const Crop k = make_crop(H0, W0);
	return l1_backward(k, make_slab(k, 0, H0), 0, H0, 0, H0, image, gt, up4, act, w2, w3, b3, upstream, d_image, d_up4, d_w2, d_b2, d_w3, d_b3, nullptr,
	                   partials, d_x, (cudaStream_t)cuda_stream);
}

}  // extern "C"

// rgs_appearance_head.cu -- the low-resolution head of GOF's AppearanceNetwork (scene/appearance_network.py): conv1 (67 -> 256)
// + ReLU, then up1..up4, each PixelShuffle(2), a 3x3 convolution and a ReLU, forward and backward, in FP32 FFMA without
// floating-point atomics.  Layer L's convolution maps [CIN, Hi, Wi] to [COUT, Hi, Wi] with Hi = 2^L h, Wi = 2^L w:
//
//   L  layer  CIN  COUT  input
//   0  conv1   67   256  down [3, h, w] and the embedding row (64 floats) on every pixel, zero in the padding ring
//   1  up1     64   128  PixelShuffle(2) of conv1's output
//   2  up2     32    64  ... of up1's
//   3  up3     16    32  ... of up2's
//   4  up4      8    16  ... of up3's; the output [16, 16h, 16w] is the tail's up4
//
// Neither the concatenated input of conv1 nor any shuffled map is materialised: a convolution reads its input through torch's
// PixelShuffle index rule in[c][2y+i][2x+j] = prev[4c+2i+j][y][x] (head_in), and the data gradient writes through the same rule.
//
//   forward_kernel  one thread per output pixel and 16 output channels; the CTA's 16 output channels' weights in shared memory
//   dgrad_kernel    per input pixel and CIB input channels, SPLIT threads each over COUT / SPLIT output channels, their
//                   sums added in group order: the flipped-weight convolution of d(pre-ReLU), read as (a > 0 ? g : 0) from
//                   the layer's output a and d(output) g; written through the inverse shuffle
//   wgrad_kernel    per CTA up to 32 input and 32 output channels and a band of 4 x 32 (up4: 8 x 32) pixel tiles: each tile's
//                   d(pre-ReLU) and input (+1 halo) staged in shared memory, a thread's 4 x 9 weight sums and 4 bias sums in
//                   fp32 over the band's tiles, pixel groups added in order; one fp64 partial row per band
//   wgrad_finish    the band rows summed in band order in fp64, one cast
//   emb_grad        d_emb[c] = sum over pixels of conv1's input gradient on channel 3 + c: fp32 per thread over a fixed stride,
//                   fp64 over the threads in order
//
// The band count per layer aims at 528 CTAs and caps the fp64 band rows at 16 MB: the low-resolution layers have many weights
// and few pixels, the high-resolution ones few weights and many pixels.  rgs_appearance_head_scratch_bytes states the total.
// Every load of an input or gradient map outside shared-memory staging is unconditional (from a clamped address, the value
// then selected), so that a thread's loads issue together.
//
// This file also holds the C-ABI entry points rgs_appearance_head_* (include/rgs_b200.h).
#include <algorithm>

#include "rgs_common.cuh"

namespace rgs {

namespace {

constexpr int HT = 256;           // threads per CTA
constexpr int COB = 16;           // forward: output channels per thread
constexpr int WGRAD_CTAS = 528;                    // weight gradient: CTAs per layer to aim for (4 per SM)
constexpr size_t WGRAD_PARTIAL_DOUBLES = 2u << 20;  // and at most 16 MB of fp64 band rows
constexpr int LAYERS = 5;
constexpr int CIN_OF[LAYERS] = {67, 64, 32, 16, 8};
constexpr int COUT_OF[LAYERS] = {256, 128, 64, 32, 16};
// the stored activations: conv1, up1, up2, up3 outputs back to back, in units of h * w floats
constexpr int ACT_OFF[4] = {0, 256, 256 + 512, 256 + 512 + 1024};
constexpr int ACT_PER_HW = RGS_APPEARANCE_HEAD_ACT_PER_HW;
static_assert(ACT_OFF[3] + 2048 == ACT_PER_HW, "the activation layout");

// The convolution input of a layer at channel c, row Y, column X of its [CIN, Hi, Wi] map, zero outside it.  FIRST: conv1's
// input, down [3, Hi, Wi] then the embedding row; otherwise src is the previous layer's output [4 CIN, Hi / 2, Wi / 2].
template <bool FIRST>
__device__ __forceinline__ float head_in(const float* __restrict__ src, const float* __restrict__ emb, int c, int Y, int X, int Hi, int Wi) {
	const bool in = (unsigned)Y < (unsigned)Hi && (unsigned)X < (unsigned)Wi;
	const int y = min(max(Y, 0), Hi - 1), x = min(max(X, 0), Wi - 1);
	float v;
	if (FIRST) v = c < 3 ? __ldg(src + ((size_t)c * Hi + y) * Wi + x) : __ldg(emb + c - 3);
	else v = __ldg(src + ((size_t)(4 * c + 2 * (y & 1) + (x & 1)) * (Hi >> 1) + (y >> 1)) * (Wi >> 1) + (x >> 1));
	return in ? v : 0.f;
}

// conv + bias + ReLU: out [COUT, Hi, Wi]; grid (pixel blocks, COUT / COB)
template <int CIN, bool FIRST>
__global__ void __launch_bounds__(HT) forward_kernel(int Hi, int Wi, const float* __restrict__ src, const float* __restrict__ emb,
                                                    const float* __restrict__ w, const float* __restrict__ b, float* __restrict__ out) {
	__shared__ float4 sw4[CIN * 9 * COB / 4];  // [ci][tap][co]
	float* sw = reinterpret_cast<float*>(sw4);
	const int co0 = blockIdx.y * COB;
	for (int i = threadIdx.x; i < CIN * 9 * COB; i += HT) {
		const int co = i % COB, tap = (i / COB) % 9, ci = i / (9 * COB);
		sw[i] = __ldg(w + ((size_t)(co0 + co) * CIN + ci) * 9 + tap);
	}
	__syncthreads();
	const int n = Hi * Wi, p = blockIdx.x * HT + threadIdx.x;
	if (p >= n) return;
	const int Y = p / Wi, X = p % Wi;
	float acc[COB];
#pragma unroll
	for (int j = 0; j < COB; j++) acc[j] = 0.f;
#pragma unroll 1
	for (int ci = 0; ci < CIN; ci++) {
#pragma unroll
		for (int tap = 0; tap < 9; tap++) {
			const float v = head_in<FIRST>(src, emb, ci, Y + tap / 3 - 1, X + tap % 3 - 1, Hi, Wi);
			const float4* wr = sw4 + (ci * 9 + tap) * (COB / 4);
#pragma unroll
			for (int j = 0; j < COB / 4; j++) {
				const float4 q = wr[j];
				acc[4 * j] = fmaf(q.x, v, acc[4 * j]); acc[4 * j + 1] = fmaf(q.y, v, acc[4 * j + 1]);
				acc[4 * j + 2] = fmaf(q.z, v, acc[4 * j + 2]); acc[4 * j + 3] = fmaf(q.w, v, acc[4 * j + 3]);
			}
		}
	}
#pragma unroll
	for (int j = 0; j < COB; j++) out[(size_t)(co0 + j) * n + p] = fmaxf(acc[j] + __ldg(b + co0 + j), 0.f);
}

// d(pre-ReLU) of a layer at row yo, column xo of channel co's map (zero outside it): ReLU's backward as torch's
// threshold_backward, a <= 0 -> 0.  Both loads are unconditional, from a clamped address.
__device__ __forceinline__ float masked(const float* __restrict__ g, const float* __restrict__ a, int co, int yo, int xo, int Hi, int Wi) {
	const bool in = (unsigned)yo < (unsigned)Hi && (unsigned)xo < (unsigned)Wi;
	const size_t o = ((size_t)co * Hi + min(max(yo, 0), Hi - 1)) * Wi + min(max(xo, 0), Wi - 1);
	const float av = __ldg(a + o), gv = __ldg(g + o);
	return in && av > 0.f ? gv : 0.f;
}

// The data gradient of one layer: d_in[ci][Y][X] = sum_co,dy,dx w[co][ci][dy][dx] dz[co][Y+1-dy][X+1-dx], dz = masked(g, a).
// Written through the inverse shuffle into d_prev [4 CIN, Hi / 2, Wi / 2], or (FIRST) into d_down [3, Hi, Wi] and the
// embedding channels' map d_emb_map [64, Hi, Wi].  A CTA holds HT / SPLIT pixels; SPLIT threads per pixel each sum COUT / SPLIT
// consecutive output channels, and the SPLIT partial sums are added in group order.  grid (pixel blocks, ceil(CIN / CIB))
template <int CIN, int COUT, int CIB, int SPLIT, bool FIRST>
__global__ void __launch_bounds__(HT) dgrad_kernel(int Hi, int Wi, const float* __restrict__ g, const float* __restrict__ a, const float* __restrict__ w,
                                                  float* __restrict__ d_prev, float* __restrict__ d_down, float* __restrict__ d_emb_map) {
	constexpr int PIX = HT / SPLIT, CO_PER = COUT / SPLIT;
	__shared__ float4 sw4[COUT * 9 * CIB / 4];  // [co][tap][ci]
	__shared__ float red[SPLIT * CIB * PIX];
	float* sw = reinterpret_cast<float*>(sw4);
	const int ci0 = blockIdx.y * CIB;
	for (int i = threadIdx.x; i < COUT * 9 * CIB; i += HT) {
		const int ci = i % CIB, tap = (i / CIB) % 9, co = i / (9 * CIB);
		sw[i] = ci0 + ci < CIN ? __ldg(w + ((size_t)co * CIN + ci0 + ci) * 9 + tap) : 0.f;
	}
	__syncthreads();
	const int n = Hi * Wi, q = threadIdx.x % PIX, grp = threadIdx.x / PIX, p = blockIdx.x * PIX + q;
	const int pc = min(p, n - 1);  // a pixel past the map computes on the last one and stores nothing
	const int Y = pc / Wi, X = pc % Wi;
	float acc[CIB];
#pragma unroll
	for (int j = 0; j < CIB; j++) acc[j] = 0.f;
#pragma unroll 1
	for (int co = grp * CO_PER; co < (grp + 1) * CO_PER; co++) {
#pragma unroll
		for (int tap = 0; tap < 9; tap++) {
			const float v = masked(g, a, co, Y + 1 - tap / 3, X + 1 - tap % 3, Hi, Wi);
			const float4* wr = sw4 + (co * 9 + tap) * (CIB / 4);
#pragma unroll
			for (int j = 0; j < CIB / 4; j++) {
				const float4 c = wr[j];
				acc[4 * j] = fmaf(c.x, v, acc[4 * j]); acc[4 * j + 1] = fmaf(c.y, v, acc[4 * j + 1]);
				acc[4 * j + 2] = fmaf(c.z, v, acc[4 * j + 2]); acc[4 * j + 3] = fmaf(c.w, v, acc[4 * j + 3]);
			}
		}
	}
#pragma unroll
	for (int j = 0; j < CIB; j++) red[(grp * CIB + j) * PIX + q] = acc[j];
	__syncthreads();
	if (grp != 0 || p >= n) return;
#pragma unroll
	for (int j = 0; j < CIB; j++) {
		float s = red[j * PIX + q];
		for (int k = 1; k < SPLIT; k++) s += red[(k * CIB + j) * PIX + q];
		const int ci = ci0 + j;
		if (ci >= CIN) break;
		if (FIRST) {
			if (ci < 3) d_down[(size_t)ci * n + p] = s;
			else d_emb_map[(size_t)(ci - 3) * n + p] = s;
		} else {
			d_prev[((size_t)(4 * ci + 2 * (Y & 1) + (X & 1)) * (Hi >> 1) + (Y >> 1)) * (Wi >> 1) + (X >> 1)] = s;
		}
	}
}

// The weight gradient's tiling for a layer with CIN inputs and COUT outputs: a CTA owns CI_B input and CO_B output channels
// and a band of TR x TC pixel tiles.  Per tile it stages d(pre-ReLU) of its output channels [CO_B][TR][TC] (the ReLU mask applied
// once) and its input channels on the tile + 1 [CI_B][TR + 2][TC + 2] (through head_in's shuffle rule) in shared memory.  Thread
// (ci, 4 output channels) of pixel group pg sums the 4 x 9 tap products and the 4 bias terms over rows pg, pg + PG, ... of each
// tile, column by column, in fp32; the PG groups are added in group order at the end of the band.
template <int CIN, int COUT>
struct WTile {
	static constexpr int CI_B = CIN < 32 ? CIN : 32, CO_B = COUT < 32 ? COUT : 32, NTH = CI_B * CO_B / 4, PG = HT / NTH;
	static constexpr int TR = PG > 4 ? PG : 4, TC = 32, RS = TC + 3, PLANE = (TR + 2) * RS + 1;  // odd plane stride: no conflicts
	static constexpr int D_FLOATS = CO_B * TR * TC, I_FLOATS = CI_B * PLANE, RED = PG > 1 ? NTH * 40 : 0;
	static constexpr int SMEM = D_FLOATS + I_FLOATS > RED ? D_FLOATS + I_FLOATS : RED;
};

// partials [nbands][COUT * CIN * 9 + COUT]: band b = blockIdx.x sums tiles [b ntiles / nbands, (b + 1) ntiles / nbands) in fp32
template <int CIN, int COUT, bool FIRST>
__global__ void __launch_bounds__(HT) wgrad_kernel(int Hi, int Wi, int tiles_x, int ntiles, const float* __restrict__ src,
                                                  const float* __restrict__ emb, const float* __restrict__ g, const float* __restrict__ a,
                                                  double* __restrict__ partials) {
	using T = WTile<CIN, COUT>;
	__shared__ float sm[T::SMEM];
	float* sD = sm;
	float* sI = sm + T::D_FLOATS;
	const int band = blockIdx.x, nbands = gridDim.x, co0 = blockIdx.y * T::CO_B, ci0 = blockIdx.z * T::CI_B;
	const int t = threadIdx.x, tn = t % T::NTH, pg = t / T::NTH, ci_l = tn % T::CI_B, cq = tn / T::CI_B;
	const int tile_lo = (int)((int64_t)band * ntiles / nbands), tile_hi = (int)((int64_t)(band + 1) * ntiles / nbands);
	const size_t plane = (size_t)Hi * Wi;
	float acc[4][9], bs[4];
#pragma unroll
	for (int j = 0; j < 4; j++) {
		bs[j] = 0.f;
#pragma unroll
		for (int k = 0; k < 9; k++) acc[j][k] = 0.f;
	}
	for (int tile = tile_lo; tile < tile_hi; tile++) {
		const int y0 = (tile / tiles_x) * T::TR, x0 = (tile % tiles_x) * T::TC;
		__syncthreads();  // the previous tile's readers are done
		for (int i = t; i < T::D_FLOATS; i += HT) {
			const int c = i % T::TC, r = (i / T::TC) % T::TR, co = i / (T::TR * T::TC), y = y0 + r, x = x0 + c;
			float v = 0.f;
			if (y < Hi && x < Wi) {
				const size_t o = (size_t)(co0 + co) * plane + (size_t)y * Wi + x;
				v = __ldg(a + o) > 0.f ? __ldg(g + o) : 0.f;  // threshold_backward: a <= 0 -> 0
			}
			sD[i] = v;
		}
		for (int i = t; i < T::CI_B * (T::TR + 2) * (T::TC + 2); i += HT) {
			const int c = i % (T::TC + 2), r = (i / (T::TC + 2)) % (T::TR + 2), ci = i / ((T::TR + 2) * (T::TC + 2));
			sI[ci * T::PLANE + r * T::RS + c] = ci0 + ci < CIN ? head_in<FIRST>(src, emb, ci0 + ci, y0 - 1 + r, x0 - 1 + c, Hi, Wi) : 0.f;
		}
		__syncthreads();
		for (int r = pg; r < T::TR; r += T::PG) {
			const float* ip = sI + ci_l * T::PLANE + r * T::RS;
			const float* dp = sD + cq * 4 * T::TR * T::TC + r * T::TC;
			float w[3][3];
#pragma unroll
			for (int dy = 0; dy < 3; dy++) {
				w[dy][1] = ip[dy * T::RS];
				w[dy][2] = ip[dy * T::RS + 1];
			}
#pragma unroll 4
			for (int c = 0; c < T::TC; c++) {
#pragma unroll
				for (int dy = 0; dy < 3; dy++) {
					w[dy][0] = w[dy][1];
					w[dy][1] = w[dy][2];
					w[dy][2] = ip[dy * T::RS + c + 2];
				}
#pragma unroll
				for (int j = 0; j < 4; j++) {
					const float d = dp[j * T::TR * T::TC + c];
					bs[j] += d;
#pragma unroll
					for (int k = 0; k < 9; k++) acc[j][k] = fmaf(d, w[k / 3][k % 3], acc[j][k]);
				}
			}
		}
	}
	for (int k = 1; k < T::PG; k++) {  // the pixel groups, added in group order
		__syncthreads();
		if (pg == k) {
#pragma unroll
			for (int j = 0; j < 4; j++) {
				sm[tn * 40 + 36 + j] = bs[j];
#pragma unroll
				for (int q = 0; q < 9; q++) sm[tn * 40 + j * 9 + q] = acc[j][q];
			}
		}
		__syncthreads();
		if (pg == 0) {
#pragma unroll
			for (int j = 0; j < 4; j++) {
				bs[j] += sm[tn * 40 + 36 + j];
#pragma unroll
				for (int q = 0; q < 9; q++) acc[j][q] += sm[tn * 40 + j * 9 + q];
			}
		}
	}
	const int ci = ci0 + ci_l;
	if (pg != 0 || ci >= CIN) return;
	double* out = partials + (size_t)band * (COUT * CIN * 9 + COUT);
#pragma unroll
	for (int j = 0; j < 4; j++) {
		const int co = co0 + cq * 4 + j;
#pragma unroll
		for (int k = 0; k < 9; k++) out[((size_t)co * CIN + ci) * 9 + k] = acc[j][k];
		if (ci == 0) out[(size_t)COUT * CIN * 9 + co] = bs[j];
	}
}

// the band rows summed in band order, cast once: dw [cout, cin, 3, 3] then db [cout]
__global__ void wgrad_finish_kernel(const double* __restrict__ partials, int nbands, int nweights, int nw, float* __restrict__ dw, float* __restrict__ db) {
	const int j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= nw) return;
	double s = 0.0;
	for (int b = 0; b < nbands; b++) s += partials[(size_t)b * nw + j];
	if (j < nweights) dw[j] = (float)s;
	else db[j - nweights] = (float)s;
}

// d_emb[c] = sum over the n pixels of d_emb_map[c]: thread t sums pixels t, t + HT, ... in fp32, thread 0 the HT sums in fp64
__global__ void __launch_bounds__(HT) emb_grad_kernel(int n, const float* __restrict__ d_emb_map, float* __restrict__ d_emb) {
	__shared__ double part[HT];
	const float* m = d_emb_map + (size_t)blockIdx.x * n;
	float s = 0.f;
	for (int p = threadIdx.x; p < n; p += HT) s += __ldg(m + p);
	part[threadIdx.x] = s;
	__syncthreads();
	if (threadIdx.x == 0) {
		double t = 0.0;
		for (int i = 0; i < HT; i++) t += part[i];
		d_emb[blockIdx.x] = (float)t;
	}
}

struct Layer {
	int cin, cout, Hi, Wi, tiles_x, ntiles, nbands;
	size_t nweights, nw;  // weights, then weights + biases per partial row
};

template <int CIN, int COUT>
void wgrad_bands(Layer& y) {
	using T = WTile<CIN, COUT>;
	y.tiles_x = (y.Wi + T::TC - 1) / T::TC;
	y.ntiles = y.tiles_x * ((y.Hi + T::TR - 1) / T::TR);
	const int ctas = COUT / T::CO_B * ((CIN + T::CI_B - 1) / T::CI_B);
	const int cap = (int)std::max<size_t>(1, WGRAD_PARTIAL_DOUBLES / y.nw);
	y.nbands = std::min(y.ntiles, std::min(cap, std::max(1, (WGRAD_CTAS + ctas - 1) / ctas)));
}

Layer layer(int L, int h, int w) {
	Layer y;
	y.cin = CIN_OF[L]; y.cout = COUT_OF[L];
	y.Hi = h << L; y.Wi = w << L;
	y.nweights = (size_t)y.cin * y.cout * 9;
	y.nw = y.nweights + y.cout;
	switch (L) {
		case 0: wgrad_bands<67, 256>(y); break;
		case 1: wgrad_bands<64, 128>(y); break;
		case 2: wgrad_bands<32, 64>(y); break;
		case 3: wgrad_bands<16, 32>(y); break;
		default: wgrad_bands<8, 16>(y); break;
	}
	return y;
}

int32_t head_size(int32_t h, int32_t w) {
	if (h < 1 || w < 1) return fail(RGS_E_INVALID, "appearance head: h and w must be at least 1");
	if ((int64_t)h * w > (int64_t)1 << 18) return fail(RGS_E_INVALID, "appearance head: input map too large");
	return RGS_OK;
}

// scratch layout: the fp64 partial rows (the largest layer's), then d(output) buffers of 2048 h w and 1024 h w floats
size_t partial_doubles(int h, int w) {
	size_t m = 0;
	for (int L = 0; L < LAYERS; L++) {
		const Layer y = layer(L, h, w);
		m = std::max(m, (size_t)y.nbands * y.nw);
	}
	return m;
}

size_t scratch_bytes(int h, int w) { return partial_doubles(h, w) * sizeof(double) + (size_t)3072 * h * w * sizeof(float); }

template <int CIN, bool FIRST>
void launch_forward(const Layer& y, const float* src, const float* emb, const float* w, const float* b, float* out, cudaStream_t st) {
	const dim3 grid((y.Hi * y.Wi + HT - 1) / HT, y.cout / COB);
	forward_kernel<CIN, FIRST><<<grid, HT, 0, st>>>(y.Hi, y.Wi, src, emb, w, b, out);
}

template <int CIN, int COUT, int CIB, int SPLIT, bool FIRST>
void launch_dgrad(const Layer& y, const float* g, const float* a, const float* w, float* d_prev, float* d_down, float* d_emb_map, cudaStream_t st) {
	const dim3 grid((y.Hi * y.Wi + HT / SPLIT - 1) / (HT / SPLIT), (CIN + CIB - 1) / CIB);
	dgrad_kernel<CIN, COUT, CIB, SPLIT, FIRST><<<grid, HT, 0, st>>>(y.Hi, y.Wi, g, a, w, d_prev, d_down, d_emb_map);
}

template <int CIN, int COUT, bool FIRST>
void launch_wgrad(const Layer& y, const float* src, const float* emb, const float* g, const float* a, double* partials, float* dw, float* db,
                  cudaStream_t st) {
	using T = WTile<CIN, COUT>;
	const dim3 grid(y.nbands, COUT / T::CO_B, (CIN + T::CI_B - 1) / T::CI_B);
	wgrad_kernel<CIN, COUT, FIRST><<<grid, HT, 0, st>>>(y.Hi, y.Wi, y.tiles_x, y.ntiles, src, emb, g, a, partials);
	wgrad_finish_kernel<<<(int)((y.nw + 255) / 256), 256, 0, st>>>(partials, y.nbands, (int)y.nweights, (int)y.nw, dw, db);
}

}  // namespace
}  // namespace rgs

using namespace rgs;

extern "C" {

int32_t rgs_appearance_head_scratch_bytes(int32_t h, int32_t w, size_t* bytes) {
	if (const int32_t rc = head_size(h, w)) return rc;
	if (!bytes) return fail(RGS_E_INVALID, "null pointer");
	*bytes = scratch_bytes(h, w);
	return RGS_OK;
}

int32_t rgs_appearance_head_forward(int32_t h, int32_t w, const float* down, const float* emb, const float* w1, const float* b1, const float* wu1,
                                    const float* bu1, const float* wu2, const float* bu2, const float* wu3, const float* bu3, const float* wu4,
                                    const float* bu4, float* act, float* up4, void* cuda_stream) {
	if (const int32_t rc = head_size(h, w)) return rc;
	if (!down || !emb || !w1 || !b1 || !wu1 || !bu1 || !wu2 || !bu2 || !wu3 || !bu3 || !wu4 || !bu4 || !act || !up4)
		return fail(RGS_E_INVALID, "null pointer");
	const cudaStream_t st = (cudaStream_t)cuda_stream;
	const size_t hw = (size_t)h * w;
	float* a[4] = {act + ACT_OFF[0] * hw, act + ACT_OFF[1] * hw, act + ACT_OFF[2] * hw, act + ACT_OFF[3] * hw};
	launch_forward<67, true>(layer(0, h, w), down, emb, w1, b1, a[0], st);
	launch_forward<64, false>(layer(1, h, w), a[0], nullptr, wu1, bu1, a[1], st);
	launch_forward<32, false>(layer(2, h, w), a[1], nullptr, wu2, bu2, a[2], st);
	launch_forward<16, false>(layer(3, h, w), a[2], nullptr, wu3, bu3, a[3], st);
	launch_forward<8, false>(layer(4, h, w), a[3], nullptr, wu4, bu4, up4, st);
	count_launch(5);
	return cuda_status(cudaGetLastError(), "appearance head forward");
}

int32_t rgs_appearance_head_backward(int32_t h, int32_t w, const float* down, const float* emb, const float* w1, const float* wu1, const float* wu2,
                                     const float* wu3, const float* wu4, const float* act, const float* up4, const float* d_up4, float* d_down,
                                     float* d_emb, float* d_w1, float* d_b1, float* d_wu1, float* d_bu1, float* d_wu2, float* d_bu2, float* d_wu3,
                                     float* d_bu3, float* d_wu4, float* d_bu4, void* scratch, void* cuda_stream) {
	if (const int32_t rc = head_size(h, w)) return rc;
	if (!down || !emb || !w1 || !wu1 || !wu2 || !wu3 || !wu4 || !act || !up4 || !d_up4 || !d_down || !d_emb || !d_w1 || !d_b1 || !d_wu1 || !d_bu1 ||
	    !d_wu2 || !d_bu2 || !d_wu3 || !d_bu3 || !d_wu4 || !d_bu4 || !scratch)
		return fail(RGS_E_INVALID, "null pointer");
	const cudaStream_t st = (cudaStream_t)cuda_stream;
	const size_t hw = (size_t)h * w;
	const float* a[4] = {act + ACT_OFF[0] * hw, act + ACT_OFF[1] * hw, act + ACT_OFF[2] * hw, act + ACT_OFF[3] * hw};
	double* partials = static_cast<double*>(scratch);
	float* A = reinterpret_cast<float*>(partials + partial_doubles(h, w));  // 2048 h w floats: d(up3), d(up1), the embedding map
	float* B = A + 2048 * hw;                                               // 1024 h w floats: d(up2), d(conv1)
	Layer y = layer(4, h, w);
	launch_wgrad<8, 16, false>(y, a[3], nullptr, d_up4, up4, partials, d_wu4, d_bu4, st);
	launch_dgrad<8, 16, 8, 1, false>(y, d_up4, up4, wu4, A, nullptr, nullptr, st);
	y = layer(3, h, w);
	launch_wgrad<16, 32, false>(y, a[2], nullptr, A, a[3], partials, d_wu3, d_bu3, st);
	launch_dgrad<16, 32, 8, 2, false>(y, A, a[3], wu3, B, nullptr, nullptr, st);
	y = layer(2, h, w);
	launch_wgrad<32, 64, false>(y, a[1], nullptr, B, a[2], partials, d_wu2, d_bu2, st);
	launch_dgrad<32, 64, 8, 4, false>(y, B, a[2], wu2, A, nullptr, nullptr, st);
	y = layer(1, h, w);
	launch_wgrad<64, 128, false>(y, a[0], nullptr, A, a[1], partials, d_wu1, d_bu1, st);
	launch_dgrad<64, 128, 8, 8, false>(y, A, a[1], wu1, B, nullptr, nullptr, st);
	y = layer(0, h, w);
	launch_wgrad<67, 256, true>(y, down, emb, B, a[0], partials, d_w1, d_b1, st);
	launch_dgrad<67, 256, 4, 8, true>(y, B, a[0], w1, nullptr, d_down, A, st);
	emb_grad_kernel<<<64, HT, 0, st>>>((int)hw, A, d_emb);
	count_launch(16);
	return cuda_status(cudaGetLastError(), "appearance head backward");
}

}  // extern "C"

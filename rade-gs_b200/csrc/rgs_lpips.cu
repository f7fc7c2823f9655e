// rgs_lpips.cu -- the VGG16 trunk of LPIPS v0.1 up to relu5_3 and its distance (contract at rgs_lpips_* in include/rgs_b200.h).
//
// Activations are NHWC fp32 for the pair of images, [2, H, W, C].  conv1_1 (3 -> 64) is a SIMT fp32 kernel that reads
// the two CHW images and applies the z-score on the way in.  The twelve 3x3 layers after it are one implicit GEMM,
// M = 2 H W pixels, N = C_out, K = 9 C_in, on wgmma.mma_async TF32 with both operands K-major in shared memory: A is
// gathered from the NHWC activations tap by tap (a 32-channel K slice never straddles a tap because C_in % 32 == 0),
// B is the weight repacked to [C_out][ky][kx][C_in].  Every layer rounds its output to TF32 (cvt.rna) in the epilogue
// and the weights come rounded the same way, so the tensor cores see exact TF32 operands and drop no bits.
//
// Staging: cp.async 16-byte copies (zero-fill for padding and for rows past M) into a 5-stage ring, prefetch distance 3.
// A stage holds A [128 x 32] and B [BN x 32] in the no-swizzle K-major canonical layout: 16-byte chunk kc of row r sits
// at kc * (rows * 16) + r * 16, so a core matrix (8 rows x 16 bytes) is 128 contiguous bytes, the stride between 8-row
// groups (SBO) is 128 bytes and the stride between the two K halves of one k8 step (LBO) is rows * 16 bytes.  Stage
// kt - 2 is refilled only after the barrier of iteration kt, when every warpgroup has retired its wgmma of kt - 2
// (wgmma.wait_group 1 at the end of each iteration).
//
// This file also holds the C-ABI entry points rgs_lpips_* (include/rgs_b200.h).
#include <algorithm>
#include <cmath>

#include "rgs_common.cuh"

namespace rgs {
namespace {

constexpr int LP_BM = 128;     // pixels per CTA: two warpgroups of m64
constexpr int LP_BK = 32;      // K per stage: four k8 steps
constexpr int LP_STAGES = 5;
constexpr int LP_AHEAD = 3;    // prefetch distance: LP_STAGES - 2 (see the ring rule above)
constexpr int LP_THREADS = 256;

template <int BN>
struct ConvCfg {
	static constexpr int A_BYTES = LP_BM * LP_BK * 4;
	static constexpr int B_BYTES = BN * LP_BK * 4;
	static constexpr int STAGE = A_BYTES + B_BYTES;
	static constexpr int SMEM = LP_STAGES * STAGE;
	static constexpr int ACC = BN / 2;   // fp32 accumulators per thread: 64 x BN over a warpgroup
};

__device__ __forceinline__ float round_tf32(float v) {
	uint32_t u;
	asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
	return __uint_as_float(u);
}

__device__ __forceinline__ float relu(float v) { return v < 0.f ? 0.f : v; }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
	asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// shared-memory matrix descriptor, no swizzle: start address, LBO and SBO in 16-byte units
__device__ __forceinline__ uint64_t smem_desc(uint32_t addr, uint32_t lbo, uint32_t sbo) {
	return (uint64_t)((addr & 0x3ffff) >> 4) | ((uint64_t)((lbo >> 4) & 0x3fff) << 16) | ((uint64_t)((sbo >> 4) & 0x3fff) << 32);
}

__device__ __forceinline__ void wgmma_tf32(float (&d)[32], uint64_t da, uint64_t db) {
	asm volatile(
	    "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
	    "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, "
	    "%19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n}\n"
	    : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
	      "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
	      "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
	      "+f"(d[31])
	    : "l"(da), "l"(db), "n"(1));
}

__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t da, uint64_t db) {
	asm volatile(
	    "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
	    "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, "
	    "%18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, "
	    "%45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n}\n"
	    : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
	      "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
	      "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
	      "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
	      "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]),
	      "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]),
	      "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
	    : "l"(da), "l"(db), "n"(1));
}

// ---- conv1_1: z-score, 3x3 conv 3 -> 64, bias, ReLU, TF32 rounding; fp32 SIMT ------------------------------------------

__global__ void __launch_bounds__(128) lpips_input_conv_kernel(int H, int W, const float* __restrict__ x, const float* __restrict__ y,
                                                               const float* __restrict__ weight, const float* __restrict__ bias, float* __restrict__ out) {
	__shared__ float sw[64 * 27];
	__shared__ float sb[64];
	for (int i = threadIdx.x; i < 64 * 27; i += blockDim.x) sw[i] = weight[i];
	if (threadIdx.x < 64) sb[threadIdx.x] = bias[threadIdx.x];
	__syncthreads();
	const int HW = H * W;
	const int p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p >= HW) return;
	const int img = blockIdx.y;
	const float* im = img ? y : x;
	const int py = p / W, px = p - py * W;
	// lpipsPyTorch's BaseNet.z_score on [0, 1] inputs: (x - mean) / std in fp32; the conv pads the z-scored image with 0
	const float mean[3] = {-.030f, -.088f, -.188f}, stdv[3] = {.458f, .448f, .450f};
	float in[27];
#pragma unroll
	for (int c = 0; c < 3; c++)
#pragma unroll
		for (int ky = 0; ky < 3; ky++)
#pragma unroll
			for (int kx = 0; kx < 3; kx++) {
				const int yy = py + ky - 1, xx = px + kx - 1;
				in[c * 9 + ky * 3 + kx] = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? (im[(size_t)c * HW + (size_t)yy * W + xx] - mean[c]) / stdv[c] : 0.f;
			}
	float4* o = reinterpret_cast<float4*>(out + ((size_t)img * HW + p) * 64);
#pragma unroll 1
	for (int g = 0; g < 16; g++) {
		float r[4];
#pragma unroll
		for (int t = 0; t < 4; t++) {
			const float* w = sw + (g * 4 + t) * 27;
			float acc = 0.f;
#pragma unroll
			for (int k = 0; k < 27; k++) acc = fmaf(w[k], in[k], acc);
			r[t] = round_tf32(relu(acc + sb[g * 4 + t]));
		}
		o[g] = make_float4(r[0], r[1], r[2], r[3]);
	}
}

// ---- conv1_2 ... conv5_3: implicit-GEMM 3x3 conv on wgmma TF32 --------------------------------------------------------

template <int BN>
__global__ void __launch_bounds__(LP_THREADS, 1) lpips_conv3x3_kernel(int H, int W, int Cin, int Cout, const float* __restrict__ in,
                                                                      const float* __restrict__ weight, const float* __restrict__ bias,
                                                                      float* __restrict__ out) {
	using Cfg = ConvCfg<BN>;
	extern __shared__ __align__(128) unsigned char smem[];
	const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(smem);
	const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
	const int NT = Cout / BN;
	const int nt = blockIdx.x % NT;
	const int64_t HW = (int64_t)H * W, M = 2 * HW;
	const int64_t m0 = (int64_t)(blockIdx.x / NT) * LP_BM;
	const int n0 = nt * BN;
	const int K = 9 * Cin, KT = K / LP_BK;

	// copy assignment: a warp fills 8 consecutive rows x 4 chunks per unit (a quarter-warp writes 128 contiguous bytes);
	// for A this thread's rows are row groups 2 warp and 2 warp + 1, row lane & 7, chunks (lane >> 3) and 4 + (lane >> 3)
	const int rlo = lane & 7, kq = lane >> 3;
	int py[2], px[2];
	const float* pimg[2];
	bool prow[2];
#pragma unroll
	for (int h = 0; h < 2; h++) {
		const int64_t m = m0 + (2 * warp + h) * 8 + rlo;
		prow[h] = m < M;
		const int64_t mm = prow[h] ? m : 0;
		const int b = (int)(mm / HW);
		const int rem = (int)(mm - b * HW);
		py[h] = rem / W;
		px[h] = rem - py[h] * W;
		pimg[h] = in + (size_t)b * HW * Cin;
	}

	auto load = [&](int kt, int stage) {
		const int k0 = kt * LP_BK;
		const int tap = k0 / Cin, c0 = k0 - tap * Cin;
		const int dy = tap / 3 - 1, dx = tap % 3 - 1;
		const uint32_t sA = sbase + stage * Cfg::STAGE, sB = sA + Cfg::A_BYTES;
#pragma unroll
		for (int i = 0; i < 4; i++) {
			const int h = i >> 1, kc = (i & 1) * 4 + kq, row = (2 * warp + h) * 8 + rlo;
			const int yy = py[h] + dy, xx = px[h] + dx;
			const bool ok = prow[h] && yy >= 0 && yy < H && xx >= 0 && xx < W;
			const float* src = ok ? pimg[h] + ((size_t)yy * W + xx) * Cin + c0 + kc * 4 : in;
			cp_async16(sA + kc * (LP_BM * 16) + row * 16, src, ok ? 16 : 0);
		}
#pragma unroll
		for (int i = 0; i < BN / 32; i++) {
			const int u = warp * (BN / 32) + i;
			const int kc = (u & 1) * 4 + kq, row = (u >> 1) * 8 + rlo;
			cp_async16(sB + kc * (BN * 16) + row * 16, weight + (size_t)(n0 + row) * K + k0 + kc * 4, 16);
		}
	};

	float acc[Cfg::ACC];
#pragma unroll
	for (int i = 0; i < Cfg::ACC; i++) acc[i] = 0.f;

#pragma unroll
	for (int s = 0; s < LP_AHEAD; s++) {
		if (s < KT) load(s, s);
		cp_async_commit();
	}
	const int wg = warp >> 2;
#pragma unroll 1
	for (int kt = 0; kt < KT; kt++) {
		cp_async_wait<LP_AHEAD - 1>();
		fence_proxy_async();   // this thread's copies, written through the generic proxy, become visible to wgmma's async proxy
		__syncthreads();
		if (kt + LP_AHEAD < KT) load(kt + LP_AHEAD, (kt + LP_AHEAD) % LP_STAGES);
		cp_async_commit();
		const uint32_t sA = sbase + (kt % LP_STAGES) * Cfg::STAGE + wg * 64 * 16, sB = sbase + (kt % LP_STAGES) * Cfg::STAGE + Cfg::A_BYTES;
		wgmma_fence();
#pragma unroll
		for (int ks = 0; ks < LP_BK / 8; ks++)
			wgmma_tf32(acc, smem_desc(sA + ks * 2 * LP_BM * 16, LP_BM * 16, 128), smem_desc(sB + ks * 2 * BN * 16, BN * 16, 128));
		wgmma_commit();
		wgmma_wait<1>();
	}
	wgmma_wait<0>();

	// epilogue: accumulator fragment of m64nBNk8 -- row 16 (warp & 3) + (lane >> 2) + 8 i, columns 8 j + 2 (lane & 3) + {0, 1}
	const int wrow = (warp & 3) * 16 + (lane >> 2);
#pragma unroll
	for (int j = 0; j < BN / 8; j++) {
		const int col = n0 + 8 * j + 2 * (lane & 3);
		const float b0 = bias[col], b1 = bias[col + 1];
#pragma unroll
		for (int i = 0; i < 2; i++) {
			const int64_t m = m0 + wg * 64 + wrow + 8 * i;
			if (m < M) {
				const float2 v = make_float2(round_tf32(relu(acc[j * 4 + i * 2] + b0)), round_tf32(relu(acc[j * 4 + i * 2 + 1] + b1)));
				*reinterpret_cast<float2*>(out + (size_t)m * Cout + col) = v;
			}
		}
	}
}

// ---- 2x2 max-pool, stride 2, floor (torch.max_pool2d's scan order and NaN rule) ---------------------------------------

__device__ __forceinline__ void max_into(float& m, float v) {
	if (v > m || v != v) m = v;
}

__global__ void lpips_maxpool_kernel(int H, int W, int C, const float* __restrict__ in, float* __restrict__ out) {
	const int Ho = H / 2, Wo = W / 2, C4 = C / 4;
	const int64_t total = (int64_t)2 * Ho * Wo * C4;
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= total) return;
	const int c4 = (int)(i % C4);
	int64_t t = i / C4;
	const int xo = (int)(t % Wo);
	t /= Wo;
	const int yo = (int)(t % Ho);
	const int b = (int)(t / Ho);
	float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
#pragma unroll
	for (int dy = 0; dy < 2; dy++)
#pragma unroll
		for (int dx = 0; dx < 2; dx++) {
			const float4 v = reinterpret_cast<const float4*>(in + (((size_t)b * H + 2 * yo + dy) * W + 2 * xo + dx) * C)[c4];
			max_into(m.x, v.x);
			max_into(m.y, v.y);
			max_into(m.z, v.z);
			max_into(m.w, v.w);
		}
	reinterpret_cast<float4*>(out)[i] = m;
}

// ---- LPIPS distance of one target layer ---------------------------------------------------------------------------------
// One warp per pixel, lane l holding channels l + 32 j.  Both channel sums go through the same xor butterfly, so every lane
// ends with the same value.  A warp's pixel values are summed in fp64 in pixel order, a CTA's eight warps in warp order,
// then lpips_mean_kernel sums the CTA partials in a fixed tree: the layer mean does not depend on scheduling.

constexpr int LD_WARPS = 8;
constexpr int LD_PIX_PER_WARP = 16;
constexpr int LD_PIX_PER_CTA = LD_WARPS * LD_PIX_PER_WARP;
constexpr int LM_THREADS = 512;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
	return v;
}

template <int C>
__global__ void __launch_bounds__(LD_WARPS * 32) lpips_distance_kernel(int HW, const float* __restrict__ f, const float* __restrict__ lin,
                                                                       float* __restrict__ map, double* __restrict__ partial) {
	constexpr int J = C / 32;
	__shared__ double wsum[LD_WARPS];
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	float w[J];
#pragma unroll
	for (int j = 0; j < J; j++) w[j] = lin[lane + 32 * j];
	double s = 0.0;
	const int first = blockIdx.x * LD_PIX_PER_CTA + warp * LD_PIX_PER_WARP;
#pragma unroll 1
	for (int k = 0; k < LD_PIX_PER_WARP; k++) {
		const int p = first + k;
		if (p >= HW) break;
		const float* fx = f + (size_t)p * C;
		const float* fy = f + ((size_t)HW + p) * C;
		float a[J], b[J], sa = 0.f, sb = 0.f;
#pragma unroll
		for (int j = 0; j < J; j++) {
			a[j] = fx[lane + 32 * j];
			b[j] = fy[lane + 32 * j];
			sa = fmaf(a[j], a[j], sa);
			sb = fmaf(b[j], b[j], sb);
		}
		const float na = sqrtf(warp_sum(sa)) + 1e-10f, nb = sqrtf(warp_sum(sb)) + 1e-10f;
		float d = 0.f;
#pragma unroll
		for (int j = 0; j < J; j++) {
			const float e = a[j] / na - b[j] / nb;
			d = fmaf(w[j], e * e, d);
		}
		d = warp_sum(d);
		if (lane == 0) map[p] = d;
		s += (double)d;
	}
	if (lane == 0) wsum[warp] = s;
	__syncthreads();
	if (threadIdx.x == 0) {
		double t = 0.0;
		for (int i = 0; i < LD_WARPS; i++) t += wsum[i];
		partial[blockIdx.x] = t;
	}
}

__global__ void __launch_bounds__(LM_THREADS) lpips_mean_kernel(int n, int HW, const double* __restrict__ partial, double* __restrict__ mean) {
	__shared__ double s[LM_THREADS];
	double t = 0.0;
	for (int i = threadIdx.x; i < n; i += LM_THREADS) t += partial[i];
	s[threadIdx.x] = t;
	__syncthreads();
	for (int o = LM_THREADS / 2; o > 0; o >>= 1) {
		if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
		__syncthreads();
	}
	if (threadIdx.x == 0) *mean = s[0] / (double)HW;
}

template <int BN>
cudaError_t launch_conv(int H, int W, int Cin, int Cout, const float* in, const float* weight, const float* bias, float* out, cudaStream_t s) {
	static size_t configured[64] = {};
	ensure_dynamic_smem(lpips_conv3x3_kernel<BN>, ConvCfg<BN>::SMEM, configured);
	const int64_t mtiles = ((int64_t)2 * H * W + LP_BM - 1) / LP_BM;
	lpips_conv3x3_kernel<BN><<<(unsigned)(mtiles * (Cout / BN)), LP_THREADS, ConvCfg<BN>::SMEM, s>>>(H, W, Cin, Cout, in, weight, bias, out);
	count_launch();
	return cudaGetLastError();
}

int lpips_distance_blocks(int HW) { return (HW + LD_PIX_PER_CTA - 1) / LD_PIX_PER_CTA; }   // fp64 partial sums the distance of one layer writes

template <int C>
void launch_distance_c(int HW, const float* feats, const float* lin, float* map, double* partial, cudaStream_t s) {
	lpips_distance_kernel<C><<<lpips_distance_blocks(HW), LD_WARPS * 32, 0, s>>>(HW, feats, lin, map, partial);
}

// the activation sizes every LPIPS stage accepts: [2, H, W, C] with 2 H W C < 2^31 elements
int lpips_size(int32_t H, int32_t W, int64_t C, int32_t min_side, const char* what) {
	if (H < min_side || W < min_side)
		return fail(RGS_E_INVALID, std::string(what) + ": the image must be at least " + std::to_string(min_side) + " x " + std::to_string(min_side) +
		                               " pixels, got " + std::to_string(H) + " x " + std::to_string(W));
	if ((int64_t)H * W * C * 2 > INT32_MAX) return fail(RGS_E_INVALID, std::string(what) + ": the activations exceed 2^31 elements");
	return RGS_OK;
}

}  // namespace
}  // namespace rgs

using namespace rgs;

extern "C" {

int32_t rgs_lpips_input_conv(int32_t H, int32_t W, const float* x, const float* y, const float* weight, const float* bias, float* out, void* cuda_stream) {
	if (const int rc = lpips_size(H, W, 64, 16, "lpips input conv")) return rc;
	if (!x || !y || !weight || !bias || !out) return fail(RGS_E_INVALID, "null pointer");
	lpips_input_conv_kernel<<<dim3((H * W + 127) / 128, 2), 128, 0, (cudaStream_t)cuda_stream>>>(H, W, x, y, weight, bias, out);
	count_launch();
	return cuda_status(cudaGetLastError(), "lpips input conv");
}

int32_t rgs_lpips_conv3x3(int32_t H, int32_t W, int32_t C_in, int32_t C_out, const float* in, const float* weight, const float* bias, float* out,
                          void* cuda_stream) {
	if (C_in <= 0 || C_in % 32 || C_in > 512 || C_out <= 0 || C_out % 64 || C_out > 512)
		return fail(RGS_E_INVALID, "lpips conv3x3: C_in must be a multiple of 32 and C_out of 64, both at most 512");
	if (const int rc = lpips_size(H, W, std::max(C_in, C_out), 1, "lpips conv3x3")) return rc;
	if (!in || !weight || !bias || !out) return fail(RGS_E_INVALID, "null pointer");
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	return cuda_status(C_out % 128 == 0 ? launch_conv<128>(H, W, C_in, C_out, in, weight, bias, out, s) : launch_conv<64>(H, W, C_in, C_out, in, weight, bias, out, s),
	                   "lpips conv3x3");
}

int32_t rgs_lpips_maxpool(int32_t H, int32_t W, int32_t C, const float* in, float* out, void* cuda_stream) {
	if (C <= 0 || C % 4) return fail(RGS_E_INVALID, "lpips maxpool: C must be a positive multiple of 4");
	if (const int rc = lpips_size(H, W, C, 2, "lpips maxpool")) return rc;
	if (!in || !out) return fail(RGS_E_INVALID, "null pointer");
	const int64_t total = (int64_t)2 * (H / 2) * (W / 2) * (C / 4);
	if (total > 0) {
		lpips_maxpool_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)cuda_stream>>>(H, W, C, in, out);
		count_launch();
	}
	return cuda_status(cudaGetLastError(), "lpips maxpool");
}

int32_t rgs_lpips_distance(int32_t H, int32_t W, int32_t C, const float* feats, const float* lin, float* map, double* mean, rgs_resize_fn resize,
                           void* scratch_user, void* cuda_stream) {
	if (C != 64 && C != 128 && C != 256 && C != 512) return fail(RGS_E_INVALID, "lpips distance: C must be 64, 128, 256 or 512");
	if (const int rc = lpips_size(H, W, C, 1, "lpips distance")) return rc;
	if (!feats || !lin || !map || !mean || !resize) return fail(RGS_E_INVALID, "null pointer");
	const int HW = H * W;
	char* buf = nullptr;
	if (const int rc = grow(resize, scratch_user, sizeof(double) * lpips_distance_blocks(HW), buf, "lpips distance scratch")) return rc;
	const cudaStream_t s = (cudaStream_t)cuda_stream;
	double* partial = reinterpret_cast<double*>(buf);
	switch (C) {
		case 64: launch_distance_c<64>(HW, feats, lin, map, partial, s); break;
		case 128: launch_distance_c<128>(HW, feats, lin, map, partial, s); break;
		case 256: launch_distance_c<256>(HW, feats, lin, map, partial, s); break;
		default: launch_distance_c<512>(HW, feats, lin, map, partial, s); break;
	}
	lpips_mean_kernel<<<1, LM_THREADS, 0, s>>>(lpips_distance_blocks(HW), HW, partial, mean);
	count_launch(2);
	return cuda_status(cudaGetLastError(), "lpips distance");
}

}  // extern "C"

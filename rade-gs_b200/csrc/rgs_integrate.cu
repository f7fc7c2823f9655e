// rgs_integrate.cu -- opacity integration at query points (`integrate_gaussians_to_points`, SURVEY.md 8f row 3):
// the rasterizer entry point marching-tetrahedra mesh extraction calls once per training view.
//
// What the reference does (forward.cu:857-900, 938-1372; rasterizer_impl.cu:573-844): bin the Gaussians as for a
// render, bin the query points by the tile they project into, then one CTA per tile in which every PIXEL thread
//   1. walks the tile's depth-sorted list, evaluating each splat at five positions (pixel centre + four corners) and
//      remembering which list entries contributed at any of them (a per-thread array of up to 2048 uint16 ids),
//   2. scans the tile's POINT list for points inside its pixel (up to 256 at a time, in a loop), and for each batch
//      re-walks the whole Gaussian list to pick out the remembered entries and composite them with the 3D ray-space
//      Gaussian at every one of its points.
// Step 2 makes every pixel thread scan all points and all Gaussians of its tile again per batch of points.
//
// Design: the contribution sets go to HBM as bit masks (one bit per list entry and pixel, written coalesced by the
// pixel threads), and step 2 becomes POINT-parallel: points are sorted by pixel (CUB radix sort on the pixel index),
// one thread per point walks only the set bits of its pixel's mask.  Neighbouring lanes hold points of the same or
// adjacent pixels, so mask words and splat records are broadcast loads.  No per-thread id arrays (no local-memory
// traffic), no 256-point batching, no re-scan of the lists.  Per-point accumulation order is the list order, as in
// the reference, so results agree to float rounding.
//
// Parity envelope (tests/golden/integrate_*.npz come from the unmodified reference): the reference reads an
// uninitialised matrix for ill-conditioned covariances (forward.cu:214 assigns a shadowed local) -- here those get a
// zero matrix; it truncates list positions to 16 bits -- here positions are exact; it stops a pixel that collects
// 2048 contributions with a printf -- here the pixel stops the same way and the call reports how many did.
#include <cub/cub.cuh>

#include "rgs_common.cuh"
#include "rgs_geom.cuh"

namespace rgs {

namespace {

constexpr int IB = 256;                      // splats staged per round (= threads per CTA)
constexpr int MAX_CONTRIB = 512 * 4;         // MAX_NUM_CONTRIBUTORS * 4 (auxiliary.h:31, forward.cu:1126)
constexpr uint32_t NO_PIXEL = 0xFFFFFFFFu;

// ---- computeCov2D<INTE> extras (forward.cu:187-235): inverse covariance in (pixel x, pixel y, ray depth) space ----------
__global__ void __launch_bounds__(256) inte_geometry_kernel(FwdParams p, const float* __restrict__ sigma_inv, const int* __restrict__ radii,
                                                             float* __restrict__ invray) {
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= p.P) return;
	float4 o0 = make_float4(0.f, 0.f, 0.f, 0.f), o1 = make_float4(0.f, 0.f, 0.f, 0.f);
	if (radii[idx] > 0) {
		const float4* sv = reinterpret_cast<const float4*>(sigma_inv + (size_t)idx * SIGMA_INV_FLOATS);
		const float4 s0 = sv[0], s1 = sv[1], s2 = sv[2];
		const M3 Vinv = m3(s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w, s2.x);
		const int flags = __float_as_int(s2.y);
		const bool well = flags & 1, solved = flags & 2;
		const float* V = p.viewmatrix;
		const float3 p_orig = {p.means3D[3 * idx], p.means3D[3 * idx + 1], p.means3D[3 * idx + 2]};
		float3 t = xform4x3(p_orig, V);
		const float limx = 1.3f * p.tan_fovx, limy = 1.3f * p.tan_fovy;
		float txtz = t.x / t.z, tytz = t.y / t.z;
		t.x = min(limx, max(-limx, txtz)) * t.z;
		t.y = min(limy, max(-limy, tytz)) * t.z;
		txtz = t.x / t.z;
		tytz = t.y / t.z;
		const M3 Wm = m3(V[0], V[4], V[8], V[1], V[5], V[9], V[2], V[6], V[10]);
		const M3 cov_cam_inv = transpose(Wm) * Vinv * Wm;
		const V3 uvh = {txtz, tytz, 1.f};
		const V3 uvh_m = mulcol(cov_cam_inv, uvh);
		const V3 uvh_mn = uvh_m * (1.0f / sqrtf(dot3(uvh_m, uvh_m)));
		o1.z = well ? 1.f : 0.f;  // `condition` (forward.cu:377-380)
		if (!isnan(uvh_mn.x) && solved && well) {
			const float u2 = txtz * txtz, v2 = tytz * tytz, uv = txtz * tytz;
			const float l = sqrt(t.x * t.x + t.y * t.y + t.z * t.z);
			const float ltz = u2 + v2 + 1;
			const float f = t.z / (u2 + v2 + 1);
			M3 full = m3(v2 + 1, -uv, txtz / l * ltz, -uv, u2 + 1, tytz / l * ltz, -txtz, -tytz, 1 / l * ltz);
			full.c[0] = full.c[0] * f; full.c[1] = full.c[1] * f; full.c[2] = full.c[2] * f;
			const M3 T2 = Wm * transpose(full);
			M3 inv = transpose(T2) * Vinv * T2;
			const M3 sc = m3(1 / p.focal_x, 0.f, 0.f, 0.f, 1 / p.focal_y, 0.f, 0.f, 0.f, 1.f);
			inv = sc * inv * sc;
			o0 = make_float4(inv.c[0].x, inv.c[0].y, inv.c[0].z, inv.c[1].y);
			o1.x = inv.c[1].z;
			o1.y = inv.c[2].z;
		}
	}
	float4* dst = reinterpret_cast<float4*>(invray + (size_t)idx * 8);
	dst[0] = o0;
	dst[1] = o1;
}

// ---- phase A: five-sample render of every tile, contribution bit masks out -----------------------------------------------------
// masks: word w of pixel t of a tile lives at [(mask_base(tile) + w) * 256 + t]; aux: two float4 per pixel
// (mid_depth_center, mid_plane.xy, mid_mean2d.x | mid_mean2d.y, last contributor (bits), 0, 0).
__host__ __device__ inline size_t mask_base(uint32_t range_begin, int tile) { return (size_t)((range_begin + 31) / 32) + (size_t)tile; }

__global__ void __launch_bounds__(IB) integrate_render_kernel(FwdParams p, const float* __restrict__ records, int RF,
                                                               const uint32_t* __restrict__ point_list, const uint2* __restrict__ ranges,
                                                               uint32_t* __restrict__ masks, float* __restrict__ out_color, float4* __restrict__ aux,
                                                               int* __restrict__ overflow_count) {
	__shared__ float4 s_rec[3][IB];
	const int tile = blockIdx.y * p.grid_x + blockIdx.x;
	const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
	const int px = blockIdx.x * TILE_X + tx, py = blockIdx.y * TILE_Y + ty;
	const bool inside = px < p.W && py < p.H;
	const float pxf = (float)px + 0.5f, pyf = (float)py + 0.5f;  // forward.cu:985
	const uint2 range = ranges[tile];
	const int total = (int)(range.y - range.x);
	const int rounds = (total + IB - 1) / IB;
	const size_t mbase = mask_base(range.x, tile);

	bool done = !inside;
	float T = 1.0f, C0 = 0.f, C1 = 0.f, C2 = 0.f, Cd = 0.f, Cmed = 0.f, Cmax = 0.f, Ca = 0.f;
	float mid_dc = 0.f, mid_px = 0.f, mid_py = 0.f, mid_mx = 0.f, mid_my = 0.f;
	float cT1 = 1.f, cT2 = 1.f, cT3 = 1.f, cT4 = 1.f;  // corner transmittances; the centre's is T itself
	uint32_t contributor = 0, last = 0;
	int n_contrib = 0;

	for (int i = 0; i < rounds; i++) {
		if (__syncthreads_count(done) == IB) break;
		const int fetch = i * IB + threadIdx.x;
		if (fetch < total) {
			const float4* rec = reinterpret_cast<const float4*>(records + (size_t)point_list[range.x + fetch] * RF);
			s_rec[0][threadIdx.x] = __ldg(rec);
			s_rec[1][threadIdx.x] = __ldg(rec + 1);
			s_rec[2][threadIdx.x] = __ldg(rec + 2);
		}
		__syncthreads();
		const int cnt = min(IB, total - i * IB);
		for (int w = 0; w * 32 < cnt; w++) {
			uint32_t bits = 0;
			const int jend = min(32, cnt - w * 32);
			for (int jj = 0; jj < jend && !done; jj++) {
				const int j = w * 32 + jj;
				contributor++;
				const float4 a = s_rec[0][j], b = s_rec[1][j], c = s_rec[2][j];  // (mx my cx cy) (cz opac rayx rayy) (r g b t)
				bool used = false;
#pragma unroll
				for (int k = 0; k < 5; k++) {
					const float ox = (k == 0) ? 0.0f : ((k & 1) ? -0.5f : 0.5f);
					const float oy = (k == 0) ? 0.0f : ((k <= 2) ? -0.5f : 0.5f);
					const float dx = a.x - pxf - ox, dy = a.y - pyf - oy;
					const float depth = c.w + (b.z * dx + b.w * dy);
					const float power = -0.5f * (a.z * dx * dx + b.x * dy * dy) - a.w * dx * dy;
					if (power > 0.0f) continue;
					const float alpha = min(0.99f, b.y * expf(power));
					if (alpha < 1.0f / 255.0f) continue;
					float& Tk = (k == 0) ? T : (k == 1) ? cT1 : (k == 2) ? cT2 : (k == 3) ? cT3 : cT4;
					const float test_T = Tk * (1 - alpha);
					if (test_T < 0.0001f) continue;
					if (k == 0) {
						C0 += c.x * alpha * T;
						C1 += c.y * alpha * T;
						C2 += c.z * alpha * T;
					}
					if (depth > Cmax) Cmax = depth;
					if (k == 0) {
						Ca += alpha * T;
						Cd += depth * alpha * T;
						if (T > 0.5f) {
							Cmed = depth;
							mid_dc = c.w; mid_px = b.z; mid_py = b.w; mid_mx = a.x; mid_my = a.y;
						}
					}
					Tk = test_T;
					used = true;
				}
				if (used) {
					last = contributor;
					bits |= 1u << jj;
					if (++n_contrib >= MAX_CONTRIB) {
						done = true;
						atomicAdd(overflow_count, 1);
					}
				}
			}
			if (inside) masks[(mbase + (size_t)i * (IB / 32) + w) * 256 + threadIdx.x] = bits;
		}
	}
	if (inside) {
		const size_t HW = (size_t)p.W * p.H, pix = (size_t)py * p.W + px;
		out_color[pix] = C0 + T * p.background[0];
		out_color[HW + pix] = C1 + T * p.background[1];
		out_color[2 * HW + pix] = C2 + T * p.background[2];
		out_color[3 * HW + pix] = Cd;
		out_color[4 * HW + pix] = Cmed;
		out_color[5 * HW + pix] = 0.f;
		out_color[6 * HW + pix] = Cmax;  // DEPTH_OFFSET
		out_color[7 * HW + pix] = Ca;    // ALPHA_OFFSET
		out_color[8 * HW + pix] = 0.f;   // DISTORTION_OFFSET: points per pixel, counted by the point kernel
		aux[2 * pix] = make_float4(mid_dc, mid_px, mid_py, mid_mx);
		aux[2 * pix + 1] = make_float4(mid_my, __uint_as_float(last), 0.f, 0.f);
	}
}

// ---- query points: projection (forward.cu:857-900), defaults of rasterize_points.cu:313-316 -----------------------------------
__global__ void __launch_bounds__(256) integrate_points_project_kernel(FwdParams p, int PN, const float* __restrict__ points3D,
                                                                        uint32_t* __restrict__ pix_key, uint32_t* __restrict__ pid,
                                                                        float2* __restrict__ pxy, float* __restrict__ pdepth,
                                                                        float* __restrict__ out_alpha, float* __restrict__ out_color_int,
                                                                        float* __restrict__ out_coord, float* __restrict__ out_sdf) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= PN) return;
	out_alpha[i] = 1.0f;
	out_color_int[3 * i] = 0.f; out_color_int[3 * i + 1] = 0.f; out_color_int[3 * i + 2] = 0.f;
	out_coord[2 * i] = 0.f; out_coord[2 * i + 1] = 0.f;
	out_sdf[i] = -1000.0f;
	uint32_t key = NO_PIXEL;
	const float3 q = {points3D[3 * i], points3D[3 * i + 1], points3D[3 * i + 2]};
	const float3 v = xform4x3(q, p.viewmatrix);
	if (v.z > 0.2f) {  // in_frustum (auxiliary.h:170)
		const float2 im = {float(p.focal_x * v.x / (v.z + 0.0000001f) + p.W / 2.), float(p.focal_y * v.y / (v.z + 0.0000001f) + p.H / 2.)};
		if (!(im.x < 0 || im.x >= p.W || im.y < 0 || im.y >= p.H)) {
			pdepth[i] = sqrt(v.x * v.x + v.y * v.y + v.z * v.z);
			pxy[i] = im;
			// the pixel whose half-open box holds the point (forward.cu:1212-1213)
			key = (uint32_t)((int)im.y * p.W + (int)im.x);
		}
	}
	pix_key[i] = key;
	pid[i] = (uint32_t)i;
}

// ---- phase B: one thread per (pixel-sorted) point, walking the set bits of its pixel's mask ---------------------------------------
__global__ void __launch_bounds__(256) integrate_points_kernel(FwdParams p, int PN, const uint32_t* __restrict__ sorted_key,
                                                                const uint32_t* __restrict__ sorted_pid, const float2* __restrict__ pxy,
                                                                const float* __restrict__ pdepth, const float* __restrict__ records, int RF,
                                                                const float* __restrict__ invray, const uint32_t* __restrict__ point_list,
                                                                const uint2* __restrict__ ranges, const uint32_t* __restrict__ masks,
                                                                const float4* __restrict__ aux, float* __restrict__ out_color,
                                                                float* __restrict__ out_alpha, float* __restrict__ out_color_int,
                                                                float* __restrict__ out_coord, float* __restrict__ out_sdf) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= PN) return;
	const uint32_t pix = sorted_key[i];
	if (pix == NO_PIXEL) return;
	const uint32_t id = sorted_pid[i];
	const int px = (int)(pix % (uint32_t)p.W), py = (int)(pix / (uint32_t)p.W);
	const int tile = (py / TILE_Y) * p.grid_x + px / TILE_X;
	const int tpix = (py % TILE_Y) * TILE_X + (px % TILE_X);
	const uint2 range = ranges[tile];
	const float4 a0 = aux[2 * (size_t)pix], a1 = aux[2 * (size_t)pix + 1];
	const uint32_t last = __float_as_uint(a1.y);
	const float2 q = pxy[id];
	const float qd = pdepth[id];
	const uint32_t* mw = masks + mask_base(range.x, tile) * 256 + tpix;
	float pa = 0.f, pT = 1.f;
	const uint32_t nwords = (last + 31) / 32;
	for (uint32_t w = 0; w < nwords; w++) {
		uint32_t bits = __ldg(mw + (size_t)w * 256);
		while (bits) {
			const int b = __ffs(bits) - 1;
			bits &= bits - 1;
			const uint32_t g = point_list[range.x + w * 32 + b];
			const float4* rec = reinterpret_cast<const float4*>(records + (size_t)g * RF);
			const float4 ra = __ldg(rec), rb = __ldg(rec + 1);
			const float tcen = __ldg(records + (size_t)g * RF + 11);
			const float4* iv = reinterpret_cast<const float4*>(invray + (size_t)g * 8);
			const float4 i0 = __ldg(iv), i1 = __ldg(iv + 1);
			const float dx = ra.x - q.x, dy = ra.y - q.y;
			const float depth = tcen + (rb.z * dx + rb.w * dy);
			float dz;
			if (i1.z != 0.f) dz = tcen - min(qd, depth);
			else if (qd < depth) continue;  // alpha = 0 (forward.cu:1317-1318)
			else dz = tcen;
			// glm::dot(delta, M * delta) with the symmetric M from the six stored entries (forward.cu:1300-1312)
			const float m0 = i0.x * dx + i0.y * dy + i0.z * dz;
			const float m1 = i0.y * dx + i0.w * dy + i1.x * dz;
			const float m2 = i0.z * dx + i1.x * dy + i1.y * dz;
			const float power = -0.5f * (dx * m0 + dy * m1 + dz * m2);
			const float alpha = min(0.99f, rb.y * expf(power));
			if (alpha < 1.0f / 255.0f) continue;
			pa += alpha * pT;
			pT = pT * (1 - alpha);
		}
	}
	const size_t HW = (size_t)p.W * p.H;
	out_alpha[id] = pa;
	out_color_int[3 * id] = out_color[pix];
	out_color_int[3 * id + 1] = out_color[HW + pix];
	out_color_int[3 * id + 2] = out_color[2 * HW + pix];
	out_coord[2 * id] = q.x;
	out_coord[2 * id + 1] = q.y;
	if (qd > 0) {
		const float dx = a0.w - q.x, dy = a1.x - q.y;
		out_sdf[id] = (a0.x + (a0.y * dx + a0.z * dy)) - qd;
	}
	atomicAdd(out_color + 8 * HW + pix, 1.0f);  // small integers: exact and order-independent
}

}  // namespace

size_t integrate_sort_temp_bytes(int PN) {
	size_t bytes = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr, PN);
	return bytes;
}

size_t integrate_mask_words(int64_t R, int tiles) { return ((size_t)(R + 31) / 32 + (size_t)tiles + 2) * 256; }

void launch_integrate(const FwdParams& p, GeomView g, BinView b, ImgView img, const int* radii, IntegrateView v, IntegrateOut out, cudaStream_t s) {
	const int RF = rec_floats(p.coord);
	inte_geometry_kernel<<<(p.P + 255) / 256, 256, 0, s>>>(p, g.sigma_inv, radii, v.invray);
	count_launch();
	cudaMemsetAsync(v.overflow, 0, sizeof(int), s);
	const dim3 grid(p.grid_x, p.grid_y);
	integrate_render_kernel<<<grid, IB, 0, s>>>(p, g.records, RF, b.point_list, img.ranges, v.masks, out.out_color, v.aux, v.overflow);
	count_launch();
	integrate_points_project_kernel<<<(v.PN + 255) / 256, 256, 0, s>>>(p, v.PN, v.points3D, v.key_in, v.pid_in, v.pxy, v.pdepth, out.out_alpha,
	                                                                    out.out_color_int, out.out_coord, out.out_sdf);
	count_launch();
	size_t temp = v.sort_temp_bytes;
	cub::DeviceRadixSort::SortPairs(v.sort_temp, temp, v.key_in, v.key_out, v.pid_in, v.pid_out, v.PN, 0, 32, s);
	count_launch();
	integrate_points_kernel<<<(v.PN + 255) / 256, 256, 0, s>>>(p, v.PN, v.key_out, v.pid_out, v.pxy, v.pdepth, g.records, RF, v.invray, b.point_list,
	                                                            img.ranges, v.masks, v.aux, out.out_color, out.out_alpha, out.out_color_int,
	                                                            out.out_coord, out.out_sdf);
	count_launch();
}

}  // namespace rgs

// rgs_render_fwd.cu -- per-tile forward alpha blend for sm_90a.
//
// Replaces renderCUDA<3,COORD,DEPTH,NORMAL> forward (reference: cuda_rasterizer/forward.cu:428-693,
// dispatch :696-742).  Same tile size (16x16, part of the key contract), same per-pixel arithmetic
// and thresholds; what changes is how the work is fed:
//   * one CTA per tile, 8 warps, each warp owns an 8x4 pixel block (tighter culling than 16x2 rows);
//   * the tile's sorted instance list is gathered in batches of 256 packed records with cp.async
//     (LDGSTS, 16 B per request, L2-only) into a 2-stage shared-memory ring: the gather of batch k+1
//     overlaps the blend of batch k, ids are prefetched one batch further ahead;
//   * each warp first tests 32 staged splats at a time (one per lane) against its pixel block with a
//     conservative minimum of the conic form over the block -- a splat whose best pixel cannot reach
//     alpha >= 1/255 is skipped for the whole warp (result-identical: the reference would `continue`
//     on every one of those pixels, forward.cu:566-567) -- and only the survivors (ballot) are blended;
//   * the ballots are also stored (one word per pixel block per 32 instances): backward-render reuses them instead of
//     repeating the test;
//   * warp-ballot early-out when all 32 pixels are saturated, block-wide exit as in the reference;
//   * every output plane is written by the kernel (zeros for the planes of a disabled variant), so the
//     host side allocates with empty() instead of seven fill kernels (rasterize_points.cu:71-78).
#include "rgs_render_common.cuh"

namespace rgs {

template <bool COORD, bool DEPTH>
__global__ void __launch_bounds__(NTHREADS, (COORD ? 4 : 5)) render_forward_kernel(
    const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list, const float* __restrict__ records,
    int W, int H, int py_off, int Hs, int grid_x, int row_begin, float focal_x, float focal_y, const float* __restrict__ bg_color,
    float* __restrict__ out_color, float* __restrict__ out_coord, float* __restrict__ out_mcoord, float* __restrict__ out_alpha,
    float* __restrict__ out_normal, float* __restrict__ out_depth, float* __restrict__ out_mdepth,
    uint32_t* __restrict__ n_contrib, float* __restrict__ accum_depth, float* __restrict__ accum_coord, float* __restrict__ normal_length,
    const uint32_t* __restrict__ chunk_base, uint32_t* __restrict__ hitmask) {
	constexpr bool GEO = COORD || DEPTH;
	constexpr int RFQ = COORD ? 6 : 4;  // float4 chunks per record
	extern __shared__ float4 smem[];    // [2][RFQ][BATCH]

	const int tid = threadIdx.x;
	const int warp = tid >> 5, lane = tid & 31;
	const int tile_x = blockIdx.x, tile_y = blockIdx.y + row_begin;
	const int bx0 = tile_x * TILE_X + (warp & 1) * 8, by0 = tile_y * TILE_Y + (warp >> 1) * 4;
	const int px = bx0 + (lane & 7), py = by0 + (lane >> 3);
	const bool inside = px < W && py < H;
	const float pxf = (float)px, pyf = (float)py;
	// box of valid pixels of this warp (clipped to the image)
	const float wx0 = (float)bx0, wx1 = (float)min(bx0 + 7, W - 1), wy0 = (float)by0, wy1 = (float)min(by0 + 3, H - 1);
	const bool warp_has_pixels = bx0 < W && by0 < H;

	const uint2 range = ranges[tile_y * grid_x + tile_x];
	const int n = (int)(range.y - range.x);
	// this warp's column of the tile's hit-mask block: one ballot word per 32 instances, kept for backward-render
	uint32_t* my_mask = hitmask + (size_t)chunk_base[tile_y * grid_x + tile_x] * 8 + warp;
	const int rounds = (n + BATCH - 1) / BATCH;

	bool done = !inside;
	float T = 1.0f;
	uint32_t last_contributor = 0, max_contributor = 0xFFFFFFFFu;
	float2 C01 = {0.f, 0.f}, C2D = {0.f, 0.f}, N01 = {0.f, 0.f}, N2W = {0.f, 0.f};  // (r,g) (b,depth) (nx,ny) (nz,weight)
	float Coord[3] = {0.f, 0.f, 0.f}, mCoord[3] = {0.f, 0.f, 0.f};
	float mDepth = 0.f;

	// ---- pipeline prologue: gather batch 0, prefetch ids of batch 1 ----
	const size_t rec_stride = (size_t)RFQ * 4;
	auto issue_gather = [&](int stage, int id) {
		if (id >= 0) {
			const float4* src = reinterpret_cast<const float4*>(records + (size_t)id * rec_stride);
			float4* dst = smem + (size_t)stage * RFQ * BATCH + tid;
#pragma unroll
			for (int c = 0; c < RFQ; c++) cp_async16(dst + c * BATCH, src + c);
		}
		cp_async_commit();
	};
	int id_cur = (tid < n) ? (int)point_list[range.x + tid] : -1;
	issue_gather(0, id_cur);
	int id_next = (BATCH + tid < n) ? (int)point_list[range.x + BATCH + tid] : -1;

	for (int i = 0; i < rounds; i++) {
		cp_async_wait_all();
		// all threads: batch i landed, batch i-1 fully consumed; vote on block-wide completion
		if (__syncthreads_and(done)) break;
		if (i + 1 < rounds) {
			issue_gather((i + 1) & 1, id_next);
			const int nxt = (i + 2) * BATCH + tid;
			id_next = (nxt < n) ? (int)point_list[range.x + nxt] : -1;
		}
		const float4* s = smem + (size_t)(i & 1) * RFQ * BATCH;
		const int cnt = min(BATCH, n - i * BATCH);

		if (!warp_has_pixels || __all_sync(0xffffffffu, done)) continue;

		unsigned batch_mask = 0;
		for (int c0 = 0; c0 < cnt; c0 += 32) {
			const int j = c0 + lane;
			bool hit = false;
			if (j < cnt) {
				const float4 a = s[j], b = s[BATCH + j];
				hit = splat_hits_box(a.x, a.y, a.z, a.w, b.x, b.y, wx0, wx1, wy0, wy1);
			}
			unsigned m = __ballot_sync(0xffffffffu, hit);
			if (lane == (c0 >> 5)) batch_mask = m;  // lane c keeps the ballot of chunk c; stored once per batch below
			while (m) {
				const int bpos = __ffs(m) - 1;
				m &= m - 1;
				const int jj = c0 + bpos;
				const float4 q0 = s[jj], q1 = s[BATCH + jj];
				const float dx = q0.x - pxf, dy = q0.y - pyf;
				const float power = -0.5f * (q0.z * dx * dx + q1.x * dy * dy) - q0.w * dx * dy;
				bool ok = !done && !(power > 0.0f);
				const float alpha = min(0.99f, q1.y * expf(power));
				ok = ok && !(alpha < 1.0f / 255.0f);
				const float test_T = T * (1 - alpha);
				if (ok && test_T < 0.0001f) {
					done = true;
					ok = false;
				}
				if (!__any_sync(0xffffffffu, ok)) {
					if (__all_sync(0xffffffffu, done)) { m = 0; c0 = cnt; }
					continue;
				}
				const uint32_t contributor = (uint32_t)(i * BATCH + jj + 1);
				const float4 q2 = s[2 * BATCH + jj];  // r g b t_center
				if (ok) {
					const float aT = alpha * T;
					const float2 aT2 = make_float2(aT, aT);
					// (r,g), (b,t), (nx,ny), (nz,1) are blended as pairs: four two-lane FMAs cover 8 channels
					C01 = ffma2(make_float2(q2.x, q2.y), aT2, C01);
					const bool before_median = T > 0.5;
					float t = 0.f;
					if constexpr (DEPTH) t = q2.w + (q1.z * dx + q1.w * dy);
					C2D = ffma2(make_float2(q2.z, t), aT2, C2D);  // (blue, ray-space depth)
					if constexpr (GEO) {
						const float4 q3 = s[3 * BATCH + jj];
						if constexpr (COORD) {
							const float4 q4 = s[4 * BATCH + jj], q5 = s[5 * BATCH + jj];
							// camera_plane: 0,1 -> x row; 2,3 -> y row; 4,5 -> z row
							const float cx = q4.x + q4.w * dx + q5.x * dy;
							const float cy = q4.y + q5.y * dx + q5.z * dy;
							const float cz = q4.z + q5.w * dx + q3.w * dy;
							Coord[0] += cx * aT;
							Coord[1] += cy * aT;
							Coord[2] += cz * aT;
							if (before_median) { mCoord[0] = cx; mCoord[1] = cy; mCoord[2] = cz; }
						}
						if constexpr (DEPTH) {
							if (before_median) mDepth = t;
						}
						N01 = ffma2(make_float2(q3.x, q3.y), aT2, N01);
						N2W = ffma2(make_float2(q3.z, 1.f), aT2, N2W);  // (normal z, weight)
						if (before_median) max_contributor = contributor;
					} else {
						N2W.y += aT;
					}
					T = test_T;
					last_contributor = contributor;
				}
			}
		}
		if (lane < ((cnt + 31) >> 5)) my_mask[(size_t)(i * (BATCH / 32) + lane) * 8] = batch_mask;  // only this tile's chunks; untested ones read as 0
	}

	if (inside) {
		const float C[3] = {C01.x, C01.y, C2D.x};
		const float Depth = C2D.y, weight = N2W.y;
		const float Normal[3] = {N01.x, N01.y, N2W.x};
		const int pix_id = W * (py - py_off) + px;  // maps hold pixel rows [py_off, py_off + Hs): the whole image, or this call's slab
		const size_t HW = (size_t)Hs * W;
		n_contrib[pix_id] = last_contributor;
		n_contrib[pix_id + HW] = max_contributor;
#pragma unroll
		for (int ch = 0; ch < 3; ch++) out_color[ch * HW + pix_id] = C[ch] + T * bg_color[ch];
		out_alpha[pix_id] = weight;
		if constexpr (COORD) {
#pragma unroll
			for (int ch = 0; ch < 3; ch++) {
				out_coord[ch * HW + pix_id] = last_contributor ? Coord[ch] / weight : 0.f;
				accum_coord[ch * HW + pix_id] = Coord[ch];
				out_mcoord[ch * HW + pix_id] = mCoord[ch];
			}
		} else {
#pragma unroll
			for (int ch = 0; ch < 3; ch++) {
				out_coord[ch * HW + pix_id] = 0.f;
				out_mcoord[ch * HW + pix_id] = 0.f;
			}
		}
		if constexpr (DEPTH) {
			const float pnx = (pxf - W / 2.f) / focal_x, pny = (pyf - H / 2.f) / focal_y;
			const float ln = sqrt(pnx * pnx + pny * pny + 1);
			const float depth_ln = Depth / ln;
			accum_depth[pix_id] = depth_ln;
			out_depth[pix_id] = last_contributor ? depth_ln / weight : 0.f;
			out_mdepth[pix_id] = mDepth / ln;
		} else {
			out_depth[pix_id] = 0.f;
			out_mdepth[pix_id] = 0.f;
		}
		if constexpr (GEO) {
			if (last_contributor) {
				float len_normal = sqrt(Normal[0] * Normal[0] + Normal[1] * Normal[1] + Normal[2] * Normal[2]);
				normal_length[pix_id] = len_normal;
				len_normal = max(len_normal, 1.0E-12F);
#pragma unroll
				for (int ch = 0; ch < 3; ch++) out_normal[ch * HW + pix_id] = Normal[ch] / len_normal;
			} else {
				normal_length[pix_id] = 1;
#pragma unroll
				for (int ch = 0; ch < 3; ch++) out_normal[ch * HW + pix_id] = 0.f;
			}
		} else {
#pragma unroll
			for (int ch = 0; ch < 3; ch++) out_normal[ch * HW + pix_id] = 0.f;
		}
	}
}

template <bool COORD, bool DEPTH>
static void launch_variant(const FwdParams& p, GeomView g, BinView b, ImgView img, RenderOut out, cudaStream_t s) {
	constexpr int RFQ = COORD ? 6 : 4;
	const size_t smem = (size_t)2 * RFQ * BATCH * sizeof(float4);
	auto kern = render_forward_kernel<COORD, DEPTH>;
	static size_t configured[64] = {};
	ensure_dynamic_smem(kern, smem, configured);
	dim3 grid(p.grid_x, p.row_end - p.row_begin, 1);
	kern<<<grid, NTHREADS, smem, s>>>(img.ranges, b.point_list, g.records, p.W, p.H, p.py_off, p.Hs, p.grid_x, p.row_begin, p.focal_x, p.focal_y, p.background,
	                                 out.color, out.coord, out.mcoord, out.alpha, out.normal, out.depth, out.mdepth, img.n_contrib,
	                                 img.accum_depth, img.accum_coord, img.normal_length, img.chunk_base, b.hitmask);
	count_launch();
}

void launch_render_forward(const FwdParams& p, GeomView g, BinView b, ImgView img, RenderOut out, cudaStream_t s) {
	if (p.row_end <= p.row_begin) return;
	// variant selection as forward.cu:732-739
	if (p.coord && p.depth)
		launch_variant<true, true>(p, g, b, img, out, s);
	else if (p.coord)
		launch_variant<true, false>(p, g, b, img, out, s);
	else if (p.depth)
		launch_variant<false, true>(p, g, b, img, out, s);
	else
		launch_variant<false, false>(p, g, b, img, out, s);
}

}  // namespace rgs

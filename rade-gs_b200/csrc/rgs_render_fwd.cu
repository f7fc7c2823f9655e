// rgs_render_fwd.cu -- per-tile forward alpha blend for sm_90a.
//
// Replaces renderCUDA<3,COORD,DEPTH,NORMAL> forward (reference: cuda_rasterizer/forward.cu:428-693,
// dispatch :696-742).  Same tile size (16x16, part of the key contract), same per-pixel arithmetic
// and thresholds; what changes is how the work is fed:
//   * one CTA of 4 warps per tile, each warp owns an 8x8 pixel block and each lane two pixels of it, (l & 7, l >> 3) and
//     (l & 7, (l >> 3) + 4) -- the pixels the backward lane owns -- so the record loads, votes and box tests of a splat are
//     paid once per 64 pixels;
//   * the tile's sorted instance list is gathered in batches of 128 packed records with cp.async
//     (LDGSTS, 16 B per request, L2-only, one record per thread) into a 2-stage shared-memory ring: the gather of batch k+1
//     overlaps the blend of batch k, ids are prefetched one batch further ahead;
//   * each warp first tests 32 staged splats at a time (one per lane) against its pixel block with a
//     conservative minimum of the conic form over the block -- a splat whose best pixel cannot reach
//     alpha >= 1/255 is skipped for the whole warp (result-identical: the reference would `continue`
//     on every one of those pixels, forward.cu:566-567) -- and only the survivors (ballot) are blended, each pixel taking
//     a survivor or not by its own exact test;
//   * the ballots are also stored for backward-render, in its format of one word per 8x4 half-block per 32 instances: the
//     warp writes its 8x8 ballot into the slots of both of its halves;
//   * warp-ballot early-out when all 64 pixels are saturated, block-wide exit as in the reference;
//   * every output plane is written by the kernel (zeros for the planes of a disabled variant), so the
//     host side allocates with empty() instead of seven fill kernels (rasterize_points.cu:71-78).
#include "rgs_render_common.cuh"

namespace rgs {

namespace {

// 4 warps per 16x16 tile: warp w owns the 8x8 block at tile columns 8 (w & 1) .. +7 and rows 8 (w >> 1) .. +7.
constexpr int FWD_THREADS = 128;
// Records staged per round, one per thread.  The hit-mask words are indexed by list position, so the round size is
// forward's own choice; 128 rather than 256 halves the ring, so that one more CTA fits per SM.
constexpr int FWD_BATCH = 128;
constexpr int FWD_GATHERS = FWD_BATCH / FWD_THREADS;
static_assert(FWD_BATCH % FWD_THREADS == 0 && FWD_BATCH % 32 == 0, "whole records per thread, whole 32-instance chunks per round");

// Resident CTAs per SM (228 KB shared memory, 64 K registers), -Xptxas -v of the sm_90a build, no spills:
//   none / depth:           16 KB ring, 56 / 72 registers -> 7 CTAs (8 would leave 64 registers, fewer than depth uses);
//   coord / coord + depth:  24 KB ring, 87 / 92 registers -> 5 CTAs (6 would leave 80).
template <bool COORD>
constexpr int forward_ctas() { return COORD ? 5 : 7; }
template <bool COORD>
constexpr size_t forward_smem_bytes() { return (size_t)2 * (COORD ? 6 : 4) * FWD_BATCH * sizeof(float4); }
// 228 KB of shared memory per SM, 1 KB of it reserved per resident CTA
static_assert(forward_ctas<false>() * (forward_smem_bytes<false>() + 1024) <= 228 * 1024, "none / depth: CTAs per SM");
static_assert(forward_ctas<true>() * (forward_smem_bytes<true>() + 1024) <= 228 * 1024, "coord: CTAs per SM");
// the register budget the launch bounds leave ptxas (64 K registers per SM): 72 (none / depth) and 96 (coord) per thread
static_assert(forward_ctas<false>() * FWD_THREADS * 72 <= 64 * 1024, "none / depth: CTAs per SM");
static_assert(forward_ctas<true>() * FWD_THREADS * 96 <= 64 * 1024, "coord: CTAs per SM");

// What a lane keeps of one of its pixels across the walk.
struct Pixel {
	float x, y;
	bool done;
	float T;
	uint32_t last_contributor, max_contributor;
	float2 C01, C2D, N01, N2W;  // (r,g) (b,depth) (nx,ny) (nz,weight)
	float Coord[3], mCoord[3];  // coord variants only
	float mDepth;
};

}  // namespace

template <bool COORD, bool DEPTH>
__global__ void __launch_bounds__(FWD_THREADS, forward_ctas<COORD>()) render_forward_kernel(
    const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list, const float* __restrict__ records,
    int W, int H, int py_off, int Hs, int grid_x, int row_begin, float focal_x, float focal_y, const float* __restrict__ bg_color,
    float* __restrict__ out_color, float* __restrict__ out_coord, float* __restrict__ out_mcoord, float* __restrict__ out_alpha,
    float* __restrict__ out_normal, float* __restrict__ out_depth, float* __restrict__ out_mdepth,
    uint32_t* __restrict__ n_contrib, float* __restrict__ accum_depth, float* __restrict__ accum_coord, float* __restrict__ normal_length,
    const uint32_t* __restrict__ chunk_base, uint32_t* __restrict__ hitmask) {
	constexpr bool GEO = COORD || DEPTH;
	constexpr int RFQ = COORD ? 6 : 4;  // float4 chunks per record
	constexpr int BATCH = FWD_BATCH;
	extern __shared__ float4 smem[];    // [2][RFQ][BATCH]

	const int tid = threadIdx.x;
	const int warp = tid >> 5, lane = tid & 31;
	const int tile_x = blockIdx.x, tile_y = blockIdx.y + row_begin;
	const int bx0 = tile_x * TILE_X + (warp & 1) * 8, by0 = tile_y * TILE_Y + (warp >> 1) * 8;
	// box of valid pixels of this warp (clipped to the image)
	const float wx0 = (float)bx0, wx1 = (float)min(bx0 + 7, W - 1), wy0 = (float)by0, wy1 = (float)min(by0 + 7, H - 1);
	const bool warp_has_pixels = bx0 < W && by0 < H;

	const uint2 range = ranges[tile_y * grid_x + tile_x];
	const int n = (int)(range.y - range.x);
	// the tile's hit-mask block holds one ballot word per 8x4 half-block and 32 instances; this warp's halves are the slots
	// 4 (warp >> 1) + (warp & 1) (upper) and that + 2 (lower), and both get the warp's 8x8 ballot
	uint32_t* my_mask = hitmask + (size_t)chunk_base[tile_y * grid_x + tile_x] * 8 + 4 * (warp >> 1) + (warp & 1);
	const int rounds = (n + BATCH - 1) / BATCH;

	// pixel a in the upper 8x4 half of the block, pixel b four rows below it in the lower half
	auto init_pixel = [&](int px, int py) {
		Pixel p;
		p.x = (float)px;
		p.y = (float)py;
		p.done = !(px < W && py < H);
		p.T = 1.0f;
		p.last_contributor = 0;
		p.max_contributor = 0xFFFFFFFFu;
		p.C01 = p.C2D = p.N01 = p.N2W = make_float2(0.f, 0.f);
#pragma unroll
		for (int ch = 0; ch < 3; ch++) p.Coord[ch] = p.mCoord[ch] = 0.f;
		p.mDepth = 0.f;
		return p;
	};
	const int px = bx0 + (lane & 7), py = by0 + (lane >> 3);
	Pixel pa = init_pixel(px, py), pb = init_pixel(px, py + 4);

	// ---- pipeline prologue: gather batch 0, prefetch ids of batch 1 ----
	const size_t rec_stride = (size_t)RFQ * 4;
	auto issue_gather = [&](int stage, const int (&id)[FWD_GATHERS]) {
#pragma unroll
		for (int g = 0; g < FWD_GATHERS; g++) {
			if (id[g] >= 0) {
				const float4* src = reinterpret_cast<const float4*>(records + (size_t)id[g] * rec_stride);
				float4* dst = smem + (size_t)stage * RFQ * BATCH + g * FWD_THREADS + tid;
#pragma unroll
				for (int c = 0; c < RFQ; c++) cp_async16(dst + c * BATCH, src + c);
			}
		}
		cp_async_commit();
	};
	auto fetch_ids = [&](int round, int (&id)[FWD_GATHERS]) {
#pragma unroll
		for (int g = 0; g < FWD_GATHERS; g++) {
			const int pos = round * BATCH + g * FWD_THREADS + tid;
			id[g] = pos < n ? (int)point_list[range.x + pos] : -1;
		}
	};
	int id_cur[FWD_GATHERS], id_next[FWD_GATHERS];
	fetch_ids(0, id_cur);
	issue_gather(0, id_cur);
	fetch_ids(1, id_next);

	for (int i = 0; i < rounds; i++) {
		cp_async_wait_all();
		// all threads: batch i landed, batch i-1 fully consumed; vote on block-wide completion
		if (__syncthreads_and(pa.done && pb.done)) break;
		if (i + 1 < rounds) {
			issue_gather((i + 1) & 1, id_next);
			fetch_ids(i + 2, id_next);
		}
		const float4* s = smem + (size_t)(i & 1) * RFQ * BATCH;
		const int cnt = min(BATCH, n - i * BATCH);

		if (!warp_has_pixels || __all_sync(0xffffffffu, pa.done && pb.done)) continue;

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
				// the reference's per-pixel test (forward.cu:560-580), once per pixel of the lane
				auto reach = [&](Pixel& p, float& dx, float& dy, float& alpha, float& test_T) {
					dx = q0.x - p.x;
					dy = q0.y - p.y;
					const float power = -0.5f * (q0.z * dx * dx + q1.x * dy * dy) - q0.w * dx * dy;
					bool ok = !p.done && !(power > 0.0f);
					alpha = min(0.99f, q1.y * expf(power));
					ok = ok && !(alpha < 1.0f / 255.0f);
					test_T = p.T * (1 - alpha);
					if (ok && test_T < 0.0001f) {
						p.done = true;
						ok = false;
					}
					return ok;
				};
				float dxa, dya, alpha_a, test_Ta, dxb, dyb, alpha_b, test_Tb;
				const bool ok_a = reach(pa, dxa, dya, alpha_a, test_Ta);
				const bool ok_b = reach(pb, dxb, dyb, alpha_b, test_Tb);
				if (!__any_sync(0xffffffffu, ok_a || ok_b)) {
					if (__all_sync(0xffffffffu, pa.done && pb.done)) { m = 0; c0 = cnt; }
					continue;
				}
				const uint32_t contributor = (uint32_t)(i * BATCH + jj + 1);
				const float4 q2 = s[2 * BATCH + jj];  // r g b t_center
				float4 q3, q4, q5;
				if constexpr (GEO) q3 = s[3 * BATCH + jj];
				if constexpr (COORD) {
					q4 = s[4 * BATCH + jj];
					q5 = s[5 * BATCH + jj];
				}
				auto blend = [&](Pixel& p, const float dx, const float dy, const float alpha, const float test_T) {
					const float aT = alpha * p.T;
					const float2 aT2 = make_float2(aT, aT);
					// (r,g), (b,t), (nx,ny), (nz,1) are blended as pairs: four two-lane FMAs cover 8 channels
					p.C01 = ffma2(make_float2(q2.x, q2.y), aT2, p.C01);
					const bool before_median = p.T > 0.5;
					float t = 0.f;
					if constexpr (DEPTH) t = q2.w + (q1.z * dx + q1.w * dy);
					p.C2D = ffma2(make_float2(q2.z, t), aT2, p.C2D);  // (blue, ray-space depth)
					if constexpr (GEO) {
						if constexpr (COORD) {
							// camera_plane: 0,1 -> x row; 2,3 -> y row; 4,5 -> z row
							const float cx = q4.x + q4.w * dx + q5.x * dy;
							const float cy = q4.y + q5.y * dx + q5.z * dy;
							const float cz = q4.z + q5.w * dx + q3.w * dy;
							p.Coord[0] += cx * aT;
							p.Coord[1] += cy * aT;
							p.Coord[2] += cz * aT;
							if (before_median) { p.mCoord[0] = cx; p.mCoord[1] = cy; p.mCoord[2] = cz; }
						}
						if constexpr (DEPTH) {
							if (before_median) p.mDepth = t;
						}
						p.N01 = ffma2(make_float2(q3.x, q3.y), aT2, p.N01);
						p.N2W = ffma2(make_float2(q3.z, 1.f), aT2, p.N2W);  // (normal z, weight)
						if (before_median) p.max_contributor = contributor;
					} else {
						p.N2W.y += aT;
					}
					p.T = test_T;
					p.last_contributor = contributor;
				};
				if (ok_a) blend(pa, dxa, dya, alpha_a, test_Ta);
				if (ok_b) blend(pb, dxb, dyb, alpha_b, test_Tb);
			}
		}
		if (lane < ((cnt + 31) >> 5)) {  // only this tile's chunks; untested ones read as 0
			uint32_t* w = my_mask + (size_t)(i * (BATCH / 32) + lane) * 8;
			w[0] = batch_mask;
			w[2] = batch_mask;
		}
	}

	auto store = [&](const Pixel& p) {
		const int px = (int)p.x, py = (int)p.y;
		if (!(px < W && py < H)) return;
		const float pxf = p.x, pyf = p.y;
		const float T = p.T;
		const uint32_t last_contributor = p.last_contributor;
		const float C[3] = {p.C01.x, p.C01.y, p.C2D.x};
		const float Depth = p.C2D.y, weight = p.N2W.y;
		const float Normal[3] = {p.N01.x, p.N01.y, p.N2W.x};
		const int pix_id = W * (py - py_off) + px;  // maps hold pixel rows [py_off, py_off + Hs): the whole image, or this call's slab
		const size_t HW = (size_t)Hs * W;
		n_contrib[pix_id] = last_contributor;
		n_contrib[pix_id + HW] = p.max_contributor;
#pragma unroll
		for (int ch = 0; ch < 3; ch++) out_color[ch * HW + pix_id] = C[ch] + T * bg_color[ch];
		out_alpha[pix_id] = weight;
		if constexpr (COORD) {
#pragma unroll
			for (int ch = 0; ch < 3; ch++) {
				out_coord[ch * HW + pix_id] = last_contributor ? p.Coord[ch] / weight : 0.f;
				accum_coord[ch * HW + pix_id] = p.Coord[ch];
				out_mcoord[ch * HW + pix_id] = p.mCoord[ch];
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
			out_mdepth[pix_id] = p.mDepth / ln;
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
	};
	store(pa);
	store(pb);
}

template <bool COORD, bool DEPTH>
static void launch_variant(const FwdParams& p, GeomView g, BinView b, ImgView img, RenderOut out, cudaStream_t s) {
	const size_t smem = forward_smem_bytes<COORD>();
	auto kern = render_forward_kernel<COORD, DEPTH>;
	static size_t configured[64] = {};
	ensure_dynamic_smem(kern, smem, configured);
	dim3 grid(p.grid_x, p.row_end - p.row_begin, 1);
	kern<<<grid, FWD_THREADS, smem, s>>>(img.ranges, b.point_list, g.records, p.W, p.H, p.py_off, p.Hs, p.grid_x, p.row_begin, p.focal_x, p.focal_y, p.background,
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

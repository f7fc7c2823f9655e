// rgs_render_bwd.cu -- per-tile backward of the alpha blend for sm_90a.
//
// Replaces renderCUDA<3,COORD,DEPTH,NORMAL> backward (reference: cuda_rasterizer/backward.cu:631-1016,
// dispatch :1101-1163).  The per-pixel recurrence (back-to-front re-traversal, T recovered by division,
// running suffix blends, median terms) is the reference's; the gradient scatter is not:
//   * the reference issues 10/16/22/25 scalar global atomicAdds per contributing (pixel, splat) pair
//     (backward.cu:878-1013).  Here a warp owns an 8x8 pixel block, each lane two pixels of it, and the warp evaluates
//     the same splat at all 64 pixels in lock-step; each lane adds its two pixels' 16 (or 25) partial gradients of the hit
//     in registers and writes the sum to shared memory, and after every group of K hits the warp sums the group through
//     that transpose: lane -> (hit, 4-float slice, 8 of the 32 pixel pairs), a two-step shuffle tail, and one 16-byte
//     red.global.add.v4.f32 per (hit, slice) into a packed accumulator row;
//   * constant factors (0.5*W, 0.5*H, 1/focal) are pulled out of the sums and applied once per Gaussian
//     in backward-preprocess;
//   * the tile list is cut at the block-wide maximum of last_contributor (nothing behind it can receive
//     gradient, backward.cu:838-839), each warp additionally skips splats behind ITS maximum and splats
//     that cannot reach alpha >= 1/255 inside either 8x4 half of its block -- read from the ballots forward-render stored;
//   * records are gathered with cp.async into a 2-stage ring, like forward, but walking the list from
//     the back.
#include "rgs_render_common.cuh"

namespace rgs {

namespace {

// 4 warps per 16x16 tile, one 8x8 pixel block each.  Lane l owns pixels (l & 7, l >> 3) and (l & 7, (l >> 3) + 4) of its block:
// one in each of the two 8x4 halves that forward-render gives a warp of its own.  Two pixels per lane halve the shared-memory
// bytes of the transpose per pixel-hit and pay the per-hit record loads, mask shuffles and vote once per 64 pixels.
constexpr int BWD_THREADS = 128;
// Records staged per round, one per thread.  The hit-mask words are indexed by list position, so the round size is backward's
// own choice.
constexpr int BWD_BATCH = 128;

// Gradient rows of the hits a warp has queued but not yet summed.  Per warp [K][NQ][S] float4: row (hit, slice) holds
// that slice of the hit's partial gradients for the 32 lanes, each the sum of the lane's two pixels (lane-contiguous, so each
// store of the queueing side is one conflict-free 512-B warp store).  At a flush lane l sums row (l / L) over the lanes
// (l % L) + L*t, t < PIX, and the L lanes of a row finish with a shuffle butterfly.  The row stride S = 32 + L puts the 8 lanes
// of a quarter-warp on 8 different 16-B bank groups while every lane walks its pixels at constant immediate offsets.
//
// Resident CTAs per SM (228 KB shared memory, 64 K registers), -Xptxas -v of the sm_90a build, no spills:
//   none:  K = 2, 17 + 18 KB shared,    78 registers -> 6 CTAs (the bound asks for 5);
//   depth: K = 2, 17 + 18 KB shared,    91 registers -> 5 CTAs (at 6, i.e. <= 80 registers, ptxas spills);
//   coord: K = 1, 25 + 15.75 KB shared, 108 / 117 registers (coord / coord + depth) -> 4 CTAs.
// K = 4 would double the hit groups to 36 KB and leave room for 4 CTAs of none / depth.
template <bool COORD>
struct HitGroup {
	static constexpr int NC = (COORD ? GRAD_FLOATS_COORD : GRAD_FLOATS_BASE) / 4;  // float4 slices of an accumulator row
	static constexpr int NQ = COORD ? 7 : 4;  // slices that carry data: floats 25..31 of a coord row are padding
	static constexpr int K = COORD ? 1 : 2;  // hits per group: K * NC = 8 rows, 4 lanes per row
	static constexpr int CTAS = COORD ? 4 : 5;
	static constexpr int L = 32 / (K * NC);
	static constexpr int PIX = 32 / L;
	static constexpr int S = 32 + L;
	static constexpr int WARP_FLOAT4 = K * NQ * S;
	static_assert(K * NC <= 32 && 32 % (K * NC) == 0 && PIX >= 8, "lanes must split evenly over (hit, slice) rows");
};

template <bool COORD>
constexpr size_t backward_smem_bytes() {
	constexpr int RFQ = COORD ? 6 : 4;
	return (size_t)2 * RFQ * BWD_BATCH * sizeof(float4) + (size_t)2 * BWD_BATCH * sizeof(int) +
	       (size_t)(BWD_THREADS / 32) * HitGroup<COORD>::WARP_FLOAT4 * sizeof(float4);
}
// 228 KB of shared memory per SM, 1 KB of it reserved per resident CTA
static_assert(HitGroup<false>::CTAS * (backward_smem_bytes<false>() + 1024 + 64) <= 228 * 1024, "none / depth: CTAs per SM");
static_assert(HitGroup<true>::CTAS * (backward_smem_bytes<true>() + 1024 + 64) <= 228 * 1024, "coord: CTAs per SM");
// the register budget the launch bounds leave ptxas (64 K registers per SM): 96 (none / depth) and 128 (coord) per thread
static_assert(HitGroup<false>::CTAS * BWD_THREADS * 96 <= 64 * 1024, "none / depth: CTAs per SM");
static_assert(HitGroup<true>::CTAS * BWD_THREADS * 128 <= 64 * 1024, "coord: CTAs per SM");

__device__ __forceinline__ float rcp_approx(float x) {
	float r;
	asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
	return r;
}
__device__ __forceinline__ int lds32(uint32_t addr) {
	int v;
	asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
	return v;
}
__device__ __forceinline__ float4 lds128(uint32_t addr) {
	float4 v;
	asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
	return v;
}

// What a lane keeps of one of its pixels across the walk: the forward state, the upstream gradients in the pairing of the
// record fields (see the loop body), and the two running values of the recurrence (T, B).
struct Pixel {
	float T, B;
	int last_contributor, max_contributor;
	float dL_dalpha, dL_dpixel_mt;
	float2 npix, g_rg, g_bt, g_nxy;
	float g_nz;
	float dL_dpixel_coord[3], dL_dpixel_mcoord[3];  // coord variants only
};

}  // namespace

template <bool COORD, bool DEPTH>
__global__ void __launch_bounds__(BWD_THREADS, HitGroup<COORD>::CTAS) render_backward_kernel(
    const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list, const float* __restrict__ records,
    int W, int H, int py_off, int Hs, int grid_x, int row_begin, float focal_x, float focal_y, const float* __restrict__ bg_color,
    const float* __restrict__ alphas, const float* __restrict__ normalmap, const uint32_t* __restrict__ n_contrib,
    const float* __restrict__ accum_depth, const float* __restrict__ accum_coord, const float* __restrict__ normal_length,
    const float* __restrict__ dL_dpixels, const float* __restrict__ dL_dpixel_coords, const float* __restrict__ dL_dpixel_mcoords,
    const float* __restrict__ dL_dpixel_depths, const float* __restrict__ dL_dpixel_mdepths, const float* __restrict__ dL_dalphas,
    const float* __restrict__ dL_dpixel_normals, float* __restrict__ grad_accum, const uint32_t* __restrict__ chunk_base,
    const uint32_t* __restrict__ hitmask) {
	constexpr bool GEO = COORD || DEPTH;
	constexpr int RFQ = COORD ? 6 : 4;
	constexpr int GF = COORD ? GRAD_FLOATS_COORD : GRAD_FLOATS_BASE;
	constexpr int BATCH = BWD_BATCH;
	using HG = HitGroup<COORD>;
	extern __shared__ float4 smem[];  // [2][RFQ][BATCH] records, [2][BATCH] ids, then per warp the HitGroup rows
	int* s_ids = reinterpret_cast<int*>(smem + 2 * RFQ * BATCH);
	const uint32_t smem_base = (uint32_t)__cvta_generic_to_shared(smem);
	__shared__ int s_block_last[BWD_THREADS / 32];

	const int tid = threadIdx.x;
	const int warp = tid >> 5, lane = tid & 31;
	float4* grp = smem + 2 * RFQ * BATCH + 2 * BATCH / 4 + warp * HG::WARP_FLOAT4;
	const int tile_x = blockIdx.x, tile_y = blockIdx.y + row_begin;
	const int bx0 = tile_x * TILE_X + (warp & 1) * 8, by0 = tile_y * TILE_Y + (warp >> 1) * 8;
	const size_t HW = (size_t)Hs * W;

	const uint2 range = ranges[tile_y * grid_x + tile_x];
	// forward-render's ballot columns of the block's two 8x4 halves: forward warps 4 (warp >> 1) + (warp & 1) and that + 2
	const uint32_t* my_mask = hitmask + (size_t)chunk_base[tile_y * grid_x + tile_x] * 8 + 4 * (warp >> 1) + (warp & 1);

	// ---- per-pixel state from forward (backward.cu:704-781) ----
	auto load_pixel = [&](int px, int py) {
		Pixel p;
		const bool inside = px < W && py < H;
		const float pxf = (float)px, pyf = (float)py;
		const int pix_id = W * (py - py_off) + px;  // maps hold pixel rows [py_off, py_off + Hs)
		const float T_final = inside ? (1 - alphas[pix_id]) : 0;
		const float w_final = inside ? alphas[pix_id] : 0;
		p.T = T_final;
		p.last_contributor = inside ? (int)n_contrib[pix_id] : 0;
		p.max_contributor = inside ? (int)n_contrib[pix_id + HW] : 0;

		float dL_dpixel[3] = {0.f, 0.f, 0.f};
		float dL_dpixel_t = 0.f, dL_dpixel_mt = 0.f, dL_dalpha = 0.f;
		float dL_dpixel_normal[3] = {0.f, 0.f, 0.f};
#pragma unroll
		for (int i = 0; i < 3; i++) p.dL_dpixel_coord[i] = p.dL_dpixel_mcoord[i] = 0.f;
		if (inside) {
#pragma unroll
			for (int i = 0; i < 3; i++) dL_dpixel[i] = dL_dpixels[i * HW + pix_id];
			dL_dalpha = dL_dalphas[pix_id];
			if constexpr (GEO) {
				const float ww = w_final * w_final;
				if constexpr (COORD) {
#pragma unroll
					for (int i = 0; i < 3; i++) {
						const float g = dL_dpixel_coords[i * HW + pix_id];
						dL_dalpha -= g * accum_coord[i * HW + pix_id] / ww;
						p.dL_dpixel_coord[i] = g / w_final;
						p.dL_dpixel_mcoord[i] = dL_dpixel_mcoords[i * HW + pix_id];
					}
				}
				if constexpr (DEPTH) {
					const float pnx = (pxf - W / 2.f) / focal_x, pny = (pyf - H / 2.f) / focal_y;
					const float ln = sqrt(pnx * pnx + pny * pny + 1);
					const float g = dL_dpixel_depths[pix_id];
					dL_dalpha -= g * accum_depth[pix_id] / ww;
					dL_dpixel_t = g / w_final / ln;
					dL_dpixel_mt = dL_dpixel_mdepths[pix_id] / ln;
				}
				{
					const float gx = dL_dpixel_normals[pix_id], gy = dL_dpixel_normals[HW + pix_id], gz = dL_dpixel_normals[2 * HW + pix_id];
					const float nx = normalmap[pix_id], ny = normalmap[HW + pix_id], nz = normalmap[2 * HW + pix_id];
					const float nlen = normal_length[pix_id];
					if (nlen < 1.0E-12F) {
						dL_dpixel_normal[0] = gx / 1.0E-12F;
						dL_dpixel_normal[1] = gy / 1.0E-12F;
						dL_dpixel_normal[2] = gz / 1.0E-12F;
					} else {
						const float d = gx * nx + gy * ny + gz * nz;
						dL_dpixel_normal[0] = (gx - d * nx) / nlen;
						dL_dpixel_normal[1] = (gy - d * ny) / nlen;
						dL_dpixel_normal[2] = (gz - d * nz) / nlen;
					}
				}
			}
		}
		if (p.last_contributor == 0) {
			// pixels nothing was blended into: w_final = 0 makes the normalisation terms 0/0.  They never receive a splat
			// (`ok` is false for every pair) but the straight-line body multiplies by them, so clear them.
			dL_dalpha = 0.f; dL_dpixel_t = 0.f; dL_dpixel_mt = 0.f;
#pragma unroll
			for (int i = 0; i < 3; i++) { dL_dpixel[i] = 0.f; p.dL_dpixel_coord[i] = 0.f; p.dL_dpixel_mcoord[i] = 0.f; dL_dpixel_normal[i] = 0.f; }
		}
		float bg_dot_dpixel = 0;
#pragma unroll
		for (int i = 0; i < 3; i++) bg_dot_dpixel += bg_color[i] * dL_dpixel[i];
		// running sum over the splats behind the current one (see the loop body); starts with the background layer
		p.B = T_final * bg_dot_dpixel;
		p.dL_dalpha = dL_dalpha;
		p.dL_dpixel_mt = dL_dpixel_mt;
		p.g_rg = make_float2(dL_dpixel[0], dL_dpixel[1]);
		p.g_bt = make_float2(dL_dpixel[2], dL_dpixel_t);
		p.g_nxy = make_float2(dL_dpixel_normal[0], dL_dpixel_normal[1]);
		p.g_nz = dL_dpixel_normal[2];
		p.npix = make_float2(-pxf, -pyf);
		return p;
	};
	// pixel a in the upper 8x4 half of the block, pixel b four rows below it in the lower half
	const int px = bx0 + (lane & 7), py = by0 + (lane >> 3);
	Pixel pa = load_pixel(px, py), pb = load_pixel(px, py + 4);

	// ---- cut the list at the last splat that contributed to any pixel of the block / warp ----
	int warp_last = max(pa.last_contributor, pb.last_contributor);
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) warp_last = max(warp_last, __shfl_xor_sync(0xffffffffu, warp_last, o));
	if (lane == 0) s_block_last[warp] = warp_last;
	__syncthreads();
	int n = 0;
#pragma unroll
	for (int w = 0; w < BWD_THREADS / 32; w++) n = max(n, s_block_last[w]);
	n = min(n, (int)(range.y - range.x));  // defensive; last_contributor <= list length by construction
	const int rounds = (n + BATCH - 1) / BATCH;

	const float ddelx_dx = 0.5 * W;
	const float ddely_dy = 0.5 * H;

	// staged index j of round i is list position  n-1 - (i*BATCH + j); thread tid stages index tid
	static_assert(BATCH == BWD_THREADS, "one staged record per thread");
	const size_t rec_stride = (size_t)RFQ * 4;
	auto issue_gather = [&](int stage, int id) {
		if (id >= 0) {
			const float4* src = reinterpret_cast<const float4*>(records + (size_t)id * rec_stride);
			float4* dst = smem + (size_t)stage * RFQ * BATCH + tid;
#pragma unroll
			for (int c = 0; c < RFQ; c++) cp_async16(dst + c * BATCH, src + c);
		}
		s_ids[stage * BATCH + tid] = id;
		cp_async_commit();
	};
	int id_cur = tid < n ? (int)point_list[range.x + n - 1 - tid] : -1;
	issue_gather(0, id_cur);
	int id_next = BATCH + tid < n ? (int)point_list[range.x + n - 1 - BATCH - tid] : -1;

	// Queue of hits whose gradient rows wait in `grp` (q of them, warp-uniform); lane h holds the Gaussian id of hit h.  The
	// queue lives in registers and its own shared memory, not in the record ring, so it carries over batch boundaries and is
	// summed when it holds K hits and once after the last batch.
	int q = 0, qid = 0;
	const int f_row = lane / HG::L, f_sub = lane % HG::L;
	const int f_hit = f_row / HG::NC, f_slice = f_row % HG::NC;
	const float4* f_src = grp + (f_hit * HG::NQ + f_slice) * HG::S + f_sub;
	auto flush = [&](int nq) {
		__syncwarp();
		const bool live = f_hit < nq && f_slice < HG::NQ;
		float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
		if (live) {
			a = f_src[0];
#pragma unroll
			for (int t = 1; t < HG::PIX; t++) {
				const float4 b = f_src[t * HG::L];
				a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
			}
		}
#pragma unroll
		for (int o = 1; o < HG::L; o <<= 1) {
			a.x += __shfl_xor_sync(0xffffffffu, a.x, o);
			a.y += __shfl_xor_sync(0xffffffffu, a.y, o);
			a.z += __shfl_xor_sync(0xffffffffu, a.z, o);
			a.w += __shfl_xor_sync(0xffffffffu, a.w, o);
		}
		const int id = __shfl_sync(0xffffffffu, qid, f_hit);
		if (live && f_sub == 0) red_add_v4(grad_accum + (size_t)id * GF + 4 * f_slice, a);
		__syncwarp();  // the rows are rewritten by the next hits
	};

	for (int i = 0; i < rounds; i++) {
		cp_async_wait_all();
		__syncthreads();
		if (i + 1 < rounds) {
			issue_gather((i + 1) & 1, id_next);
			const int nxt = (i + 2) * BATCH + tid;
			id_next = nxt < n ? (int)point_list[range.x + n - 1 - nxt] : -1;
		}
		const uint32_t s_addr = smem_base + (uint32_t)((i & 1) * RFQ * BATCH * 16);
		const uint32_t ids_addr = smem_base + (uint32_t)(2 * RFQ * BATCH * 16 + (i & 1) * BATCH * 4);
		const int cnt = min(BATCH, n - i * BATCH);
		const int pos0 = n - 1 - i * BATCH;  // list position of staged index 0
		if (pos0 - (cnt - 1) >= warp_last) continue;  // whole batch is behind this warp's last contributor

		// hit masks of forward-render for the positions of this batch: word k covers list positions [32k, 32k+32), the OR of
		// the two halves' words; lane l fetches word (pos0>>5) - l, chunks below pick theirs up with a shuffle
		const int k_hi = pos0 >> 5;
		uint32_t wl = 0;
		if (lane <= BATCH / 32 + 1 && k_hi - lane >= 0) {
			const uint32_t* wp = my_mask + (size_t)(k_hi - lane) * 8;
			wl = __ldg(wp) | __ldg(wp + 2);
		}

		for (int c0 = 0; c0 < cnt; c0 += 32) {
			// staged index j of this chunk <-> list position hi - j
			const int hi = pos0 - c0, lo_pos = hi - 31;
			const int k0 = lo_pos >> 5;  // floor, -1 when the chunk reaches below position 0
			const uint32_t w0 = __shfl_sync(0xffffffffu, wl, (k_hi - k0) & 31);
			const uint32_t w1 = __shfl_sync(0xffffffffu, wl, (k_hi - k0 - 1) & 31);
			unsigned m = __brev(__funnelshift_r(w0, w1, lo_pos & 31));  // bit j <-> position hi - j
			const int valid = min(32, cnt - c0);                       // staged entries in this chunk
			if (valid < 32) m &= (1u << valid) - 1u;
			const int behind = hi - warp_last + 1;                      // entries j < behind sit at or behind warp_last
			if (behind > 0) m = behind >= 32 ? 0u : (m & ~((1u << behind) - 1u));
			while (m) {
				const int bpos = __ffs(m) - 1;
				m &= m - 1;
				const int jj = c0 + bpos;
				const int contributor = pos0 - jj;  // 0-based position in the tile list (backward.cu:837)
				const uint32_t sa = s_addr + (uint32_t)jj * 16u;
				const float4 q0 = lds128(sa), q1 = lds128(sa + BATCH * 16u);  // (mx my A B) (C o ray.x ray.y)
				auto reach = [&](const Pixel& p, float2& d, float& G, float& alpha_raw) {
					d = fadd2(make_float2(q0.x, q0.y), p.npix);  // centre - pixel
					const float power = -0.5f * (q0.z * d.x * d.x + q1.x * d.y * d.y) - q0.w * d.x * d.y;
					G = expf(power);
					alpha_raw = min(0.99f, q1.y * G);
					return contributor < p.last_contributor && !(power > 0.0f) && !(alpha_raw < 1.0f / 255.0f);
				};
				float2 da, db;
				float Ga, Gb, alpha_a, alpha_b;
				const bool ok_a = reach(pa, da, Ga, alpha_a), ok_b = reach(pb, db, Gb, alpha_b);
				if (!__any_sync(0xffffffffu, ok_a || ok_b)) continue;

				const float4 q2 = lds128(sa + 2 * BATCH * 16u);  // r g b t_center
				float4 q3, q4, q5;
				if constexpr (GEO) q3 = lds128(sa + 3 * BATCH * 16u);
				if constexpr (COORD) {
					q4 = lds128(sa + 4 * BATCH * 16u);
					q5 = lds128(sa + 5 * BATCH * 16u);
				}
				// Straight-line body, once per pixel of the lane; the two calls share nothing but the record, so their
				// chains interleave.  A pixel that does not receive this splat runs it with alpha = 0: a layer of zero
				// opacity leaves T and the running sum below unchanged, its channel weights are alpha*T = 0, and the terms
				// that would not vanish (they all carry the factor G) are masked through G.
				//
				// Blend backward in "dot-product" form.  The reference keeps, per channel, the normalised blend of everything
				// behind the current splat (accum_rec, backward.cu:870-962) and forms sum_ch (c_ch - accum_rec_ch) g_ch * T.
				// With B = sum over the splats behind of (alpha T) * S, S = sum_ch c_ch g_ch (g = the pixel's upstream
				// gradients, alpha channel c = 1, background folded in as the last layer) that is exactly
				//      dL/dalpha = T * S - B / (1 - alpha),       B += alpha T S
				// -- one running scalar instead of 8 running blends + 8 "last" values (same algebra, different rounding).
				//
				// Channels that share a factor are kept in aligned register pairs -- (r,g) (b,t) (nx,ny) on the record side,
				// (g_r,g_g) (g_b,g_t) (g_nx,g_ny) on the pixel side -- and go through the two-lane helpers fmul2 / ffma2.
				auto body = [&](Pixel& p, const float2 d, const float G, const float alpha_raw, const bool ok, float* gv) {
					const float dx = d.x, dy = d.y;
					const float alpha = ok ? alpha_raw : 0.f;
					float4 c2 = q2;
					const float inv = rcp_approx(1.f - alpha);  // 1 - alpha in [0.01, 1]: bare MUFU.RCP; shared by T/(1-alpha) and B/(1-alpha)
					p.T = p.T * inv;
					const float T = p.T;
					const float w = alpha * T;  // dchannel_dcolor
					const float2 w2 = make_float2(w, w);
					if constexpr (DEPTH) c2.w = c2.w + (q1.z * dx + q1.w * dy);  // t = t_center + ray . d
					float2 S2 = ffma2(make_float2(c2.x, c2.y), p.g_rg, make_float2(p.dL_dalpha, 0.f));
					S2 = ffma2(make_float2(c2.z, c2.w), p.g_bt, S2);
					const float2 c_rg = fmul2(w2, p.g_rg);
					const float2 c_bt = fmul2(w2, p.g_bt);  // (dL_dcolor.b, dL_dt before the median term)
					gv[G_COL + 0] = c_rg.x;
					gv[G_COL + 1] = c_rg.y;
					gv[G_COL + 2] = c_bt.x;
					float dL_dcoords[3] = {0.f, 0.f, 0.f};
					const bool is_median = ok && contributor == p.max_contributor - 1;
					if constexpr (COORD) {
						const float coord[3] = {q4.x + q4.w * dx + q5.x * dy, q4.y + q5.y * dx + q5.z * dy, q4.z + q5.w * dx + q3.w * dy};
#pragma unroll
						for (int ch = 0; ch < 3; ch++) {
							S2.x = fmaf(coord[ch], p.dL_dpixel_coord[ch], S2.x);
							dL_dcoords[ch] = w * p.dL_dpixel_coord[ch];
							if (is_median) dL_dcoords[ch] += p.dL_dpixel_mcoord[ch];
							gv[G_VP + ch] = dL_dcoords[ch];
							gv[G_CP + 2 * ch] = dL_dcoords[ch] * dx;      // 1/focal_x applied in backward-preprocess
							gv[G_CP + 2 * ch + 1] = dL_dcoords[ch] * dy;  // 1/focal_y
						}
					}
					float dL_dt = 0.f;
					if constexpr (DEPTH) {
						dL_dt = c_bt.y;
						if (is_median) dL_dt += p.dL_dpixel_mt;
					}
					gv[G_T] = dL_dt;
					const float2 g_ray = fmul2(make_float2(dL_dt, dL_dt), d);
					gv[G_RAYX] = g_ray.x;
					gv[G_RAYY] = g_ray.y;
					float S;
					if constexpr (GEO) {
						S2 = ffma2(make_float2(q3.x, q3.y), p.g_nxy, S2);
						const float2 c_n = fmul2(w2, p.g_nxy);
						S = fmaf(q3.z, p.g_nz, S2.x + S2.y);
						gv[G_NRM + 0] = c_n.x;
						gv[G_NRM + 1] = c_n.y;
						gv[G_NRM + 2] = w * p.g_nz;
					} else {
						S = S2.x + S2.y;
						gv[G_NRM] = gv[G_NRM + 1] = gv[G_NRM + 2] = 0.f;
					}
					const float dL_dopa = T * S - inv * p.B;
					p.B = fmaf(w, S, p.B);
					const float Gm = ok ? G : 0.f;  // the reference skips this pair entirely: every term below carries a factor G

					const float dL_dG = q1.y * dL_dopa;
					const float2 gd = fmul2(make_float2(Gm, Gm), d);  // (G dx, G dy)
					const float dG_ddelx = -gd.x * q0.z - gd.y * q0.w;
					const float dG_ddely = -gd.y * q1.x - gd.x * q0.w;
					float2 dL_ddel = fmul2(make_float2(dL_dG, dL_dG), make_float2(dG_ddelx, dG_ddely));
					const float2 ab = fmul2(dL_ddel, make_float2(ddelx_dx, ddely_dy));
					gv[G_MABS] = abs(ab.x) + abs(ab.y);
					if constexpr (COORD) {
						dL_ddel.x += dL_dcoords[0] * q4.w + dL_dcoords[1] * q5.y + dL_dcoords[2] * q5.w;
						dL_ddel.y += dL_dcoords[0] * q5.x + dL_dcoords[1] * q5.z + dL_dcoords[2] * q3.w;
					}
					if constexpr (DEPTH) dL_ddel = ffma2(make_float2(dL_dt, dL_dt), make_float2(q1.z, q1.w), dL_ddel);
					gv[G_MX] = dL_ddel.x;  // * 0.5 W in backward-preprocess
					gv[G_MY] = dL_ddel.y;  // * 0.5 H
					const float hG = -0.5f * dL_dG;
					const float2 cxy = fmul2(fmul2(make_float2(gd.x, gd.x), d), make_float2(hG, hG));
					gv[G_CONX] = cxy.x;
					gv[G_CONY] = cxy.y;
					gv[G_CONW] = gd.y * dy * hG;
					gv[G_OPA] = Gm * dL_dopa;
				};
				constexpr int NG = 4 * HG::NQ;  // floats 25..31 of a coord row are padding, stored as zeros
				float ga[NG], gb[NG];
				if constexpr (COORD) {
#pragma unroll
					for (int k = 25; k < NG; k++) ga[k] = gb[k] = 0.f;
				}
				body(pa, da, Ga, alpha_a, ok_a, ga);
				body(pb, db, Gb, alpha_b, ok_b, gb);
				float4* slot = grp + q * (HG::NQ * HG::S) + lane;
#pragma unroll
				for (int c = 0; c < HG::NQ; c++)
					slot[c * HG::S] = make_float4(ga[4 * c] + gb[4 * c], ga[4 * c + 1] + gb[4 * c + 1], ga[4 * c + 2] + gb[4 * c + 2], ga[4 * c + 3] + gb[4 * c + 3]);
				const int hit_id = lds32(ids_addr + (uint32_t)jj * 4u);
				if (lane == q) qid = hit_id;
				if (++q == HG::K) {
					flush(HG::K);
					q = 0;
				}
			}
		}
	}
	if (q > 0) flush(q);
}

template <bool COORD, bool DEPTH>
static void launch_variant(const FwdParams& p, GeomView g, BinView b, ImgView img, RenderGradIn gin, float* grad_accum, cudaStream_t s) {
	const size_t smem = backward_smem_bytes<COORD>();
	auto kern = render_backward_kernel<COORD, DEPTH>;
	static size_t configured[64] = {};
	ensure_dynamic_smem(kern, smem, configured);
	dim3 grid(p.grid_x, p.row_end - p.row_begin, 1);
	kern<<<grid, BWD_THREADS, smem, s>>>(img.ranges, b.point_list, g.records, p.W, p.H, p.py_off, p.Hs, p.grid_x, p.row_begin, p.focal_x, p.focal_y, p.background,
	                                     gin.out_alpha, gin.out_normal, img.n_contrib, img.accum_depth, img.accum_coord, img.normal_length,
	                                     gin.d_color, gin.d_coord, gin.d_mcoord, gin.d_depth, gin.d_mdepth, gin.d_alpha, gin.d_normal, grad_accum, img.chunk_base, b.hitmask);
	count_launch();
}

void launch_render_backward(const FwdParams& p, GeomView g, BinView b, ImgView img, RenderGradIn gin, float* grad_accum, cudaStream_t s, bool zero_first) {
	if (zero_first) {
		cudaMemsetAsync(grad_accum, 0, (size_t)p.P * grad_floats(p.coord) * sizeof(float), s);
		count_launch();
	}
	if (p.row_end <= p.row_begin) return;
	if (p.coord && p.depth)
		launch_variant<true, true>(p, g, b, img, gin, grad_accum, s);
	else if (p.coord)
		launch_variant<true, false>(p, g, b, img, gin, grad_accum, s);
	else if (p.depth)
		launch_variant<false, true>(p, g, b, img, gin, grad_accum, s);
	else
		launch_variant<false, false>(p, g, b, img, gin, grad_accum, s);
}

}  // namespace rgs

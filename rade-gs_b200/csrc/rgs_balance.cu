// rgs_balance.cu -- balanced row sharding (include/rgs_b200.h, rgs_forward_balanced): the per-row work of a frame, the partition
// rule, and the restriction of a whole-image tile scan to one rank's slab.
//
// A balanced call preprocesses and scans the whole image, so its tile ranges, chunk offsets, totals and per-splat tile counts
// are those of the whole image.  slab_restrict_kernel turns them into what the scan of a fixed-slab call over the same rows
// leaves, in that call's image buffer: binning, sort, blend and backward then see exactly that call's state and need no change.
#include "rgs_common.cuh"

namespace rgs {

// Per tile row y: stats[y] = instances of the row, stats[grid_y + y] = its longest tile list, stats[2 grid_y + y] = its
// 32-instance chunks (hit-mask words per pixel block, the unit of chunk_base).  One warp per row.
__global__ void __launch_bounds__(256) row_stats_kernel(int grid_x, int grid_y, const uint32_t* __restrict__ tile_count,
                                                        uint32_t* __restrict__ stats) {
	const int lane = threadIdx.x & 31;
	const int y = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
	if (y >= grid_y) return;
	uint32_t sum = 0, longest = 0, chunks = 0;
	for (int x = lane; x < grid_x; x += 32) {
		const uint32_t c = tile_count[(size_t)y * grid_x + x];
		sum += c;
		longest = max(longest, c);
		chunks += (c + 31u) >> 5;
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
		sum += __shfl_xor_sync(0xffffffffu, sum, o);
		longest = max(longest, __shfl_xor_sync(0xffffffffu, longest, o));
		chunks += __shfl_xor_sync(0xffffffffu, chunks, o);
	}
	if (lane == 0) {
		stats[y] = sum;
		stats[grid_y + y] = longest;
		stats[2 * grid_y + y] = chunks;
	}
}

void launch_row_stats(const FwdParams& p, ImgView img, uint32_t* stats, cudaStream_t s) {
	row_stats_kernel<<<(p.grid_y + 7) / 8, 256, 0, s>>>(p.grid_x, p.grid_y, img.tile_count, stats);
	count_launch();
}

// The first `tile_blocks` CTAs write the slab's per-tile state into `dst` from the whole image's in `src`, the rest clip the
// per-splat tile counts in place:
//   tiles of the slab   : count as is, range and chunk_base shifted down by what the rows above the slab hold (an empty tile
//                         keeps (0, 0));
//   tiles outside it    : count 0, range (0, 0), chunk_base 0 above the slab and the slab's chunk total below it;
//   splats              : tile count of the rectangle clipped to the slab rows, as preprocess computes it for a fixed slab;
//   totals              : the slab's instances and longest list.
__global__ void __launch_bounds__(256) slab_restrict_kernel(int P, int grid_x, int grid_y, int row_begin, int row_end, int tile_blocks,
                                                            uint32_t range_off, uint32_t chunk_off, uint32_t chunk_total, uint32_t slab_rendered,
                                                            uint32_t slab_longest, ImgView src, ImgView dst, const float* __restrict__ records,
                                                            int rec_f, const int* __restrict__ radii, uint32_t* __restrict__ tiles_touched) {
	if ((int)blockIdx.x < tile_blocks) {
		const int t = blockIdx.x * blockDim.x + threadIdx.x;
		if (t == 0) {
			dst.totals[0] = slab_rendered;
			dst.totals[1] = slab_longest;
		}
		if (t >= grid_x * grid_y) return;
		const int y = t / grid_x;
		if (y >= row_begin && y < row_end) {
			const uint2 rg = src.ranges[t];
			dst.tile_count[t] = src.tile_count[t];
			dst.ranges[t] = rg.y > rg.x ? make_uint2(rg.x - range_off, rg.y - range_off) : make_uint2(0u, 0u);
			dst.chunk_base[t] = src.chunk_base[t] - chunk_off;
		} else {
			dst.tile_count[t] = 0;
			dst.ranges[t] = make_uint2(0u, 0u);
			dst.chunk_base[t] = y < row_begin ? 0u : chunk_total;
		}
		return;
	}
	const int idx = (blockIdx.x - tile_blocks) * blockDim.x + threadIdx.x;
	if (idx >= P || tiles_touched[idx] == 0) return;
	const float2 xy = *reinterpret_cast<const float2*>(records + (size_t)idx * rec_f);
	uint2 rmin, rmax;
	tile_rect(xy, radii[idx], grid_x, grid_y, rmin, rmax);
	const int ry0 = max((int)rmin.y, row_begin), ry1 = min((int)rmax.y, row_end);
	tiles_touched[idx] = (rmax.x - rmin.x) * (uint32_t)max(0, ry1 - ry0);
}

void launch_slab_restrict(const FwdParams& slab, GeomView g, ImgView whole, ImgView img, const int* radii, const SlabShift& sh, cudaStream_t s) {
	const int tile_blocks = (slab.grid_x * slab.grid_y + 255) / 256;
	const int blocks = tile_blocks + (slab.P + 255) / 256;
	slab_restrict_kernel<<<blocks, 256, 0, s>>>(slab.P, slab.grid_x, slab.grid_y, slab.row_begin, slab.row_end, tile_blocks, sh.range_off, sh.chunk_off,
	                                            sh.chunk_total, sh.rendered, sh.longest, whole, img, g.records, rec_floats(slab.coord), radii,
	                                            g.tiles_touched);
	count_launch();
}

}  // namespace rgs

using namespace rgs;

extern "C" int32_t rgs_balance_partition(int32_t grid_y, int32_t grid_x, int32_t world_size, const uint32_t* row_instances, int32_t* row_cuts) {
	if (world_size <= 0 || grid_x <= 0 || grid_y < 0) return fail(RGS_E_INVALID, "balanced partition: world_size and grid_x must be positive");
	if (grid_y < world_size) return fail(RGS_E_INVALID, "balanced partition: fewer tile rows than ranks (every slab needs a tile row)");
	if (!row_cuts || (!row_instances && grid_y > 0)) return fail(RGS_E_INVALID, "balanced partition: null pointer");
	const uint64_t fixed = (uint64_t)RGS_BALANCE_TILE_COST * (uint64_t)grid_x;
	uint64_t total = 0, heaviest = 0;
	for (int y = 0; y < grid_y; y++) {
		const uint64_t w = row_instances[y] + fixed;
		total += w;
		heaviest = w > heaviest ? w : heaviest;
	}
	// least number of contiguous slabs of weight <= B (every row fits alone once B >= heaviest)
	auto slabs_needed = [&](uint64_t B) {
		int n = 1;
		uint64_t acc = 0;
		for (int y = 0; y < grid_y; y++) {
			const uint64_t w = row_instances[y] + fixed;
			if (acc + w > B) { n++; acc = 0; }
			acc += w;
		}
		return n;
	};
	// B* by bisection: with grid_y >= world_size a partition into fewer slabs splits into exactly world_size without growing its largest
	uint64_t lo = heaviest, hi = total;
	while (lo < hi) {
		const uint64_t mid = lo + (hi - lo) / 2;
		if (slabs_needed(mid) <= world_size) hi = mid; else lo = mid + 1;
	}
	const uint64_t best = lo;
	int y = 0;
	row_cuts[0] = 0;
	for (int r = 0; r + 1 < world_size; r++) {
		uint64_t acc = 0;
		const int last = grid_y - (world_size - r - 1);  // rows [last, grid_y) stay for the later ranks
		do { acc += row_instances[y] + fixed; y++; } while (y < last && acc + row_instances[y] + fixed <= best);
		row_cuts[r + 1] = y;
	}
	row_cuts[world_size] = grid_y;
	return RGS_OK;
}

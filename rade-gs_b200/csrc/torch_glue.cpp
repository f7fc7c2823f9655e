// torch_glue.cpp -- pybind11 module `diff_gaussian_rasterization._C` on top of the C ABI.
//
// Drop-in for the reference's torch glue: same four Python-callable symbols, argument order, tuple layouts
// and error behaviour (reference: submodules/diff-gaussian-rasterization/rasterize_points.{h,cu},
// ext.cpp:15-20).  Everything that touches the GPU goes through include/rgs_b200.h; this file only
// allocates tensors, converts the "empty tensor == absent" convention to NULL pointers and forwards.
//
// Differences that are deliberate:
//   * outputs are allocated with empty(): the kernels write every element (the reference zero-fills 15 image
//     planes and 14 gradient tensors first, rasterize_points.cu:71-78,180-193);
//   * work is queued on torch's CURRENT stream of the tensors' device (the reference uses the legacy default
//     stream, SURVEY.md 8b);
//   * three extra symbols (`*_slab`, `*_backward_render`, `*_backward_preprocess`) expose the tile-row slab and
//     the two backward stages for the multi-GPU path; the reference has no equivalent.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <algorithm>
#include <array>
#include <string>
#include <tuple>
#include <vector>

#include "rgs_b200.h"

namespace {

const float* opt_ptr(const torch::Tensor& t) { return t.numel() == 0 ? nullptr : t.data_ptr<float>(); }

const char* dtype_name(torch::ScalarType t) {
	switch (t) {
		case torch::kFloat32: return "float32";
		case torch::kFloat64: return "float64";
		case torch::kInt32: return "int32";
		case torch::kInt64: return "int64";
		case torch::kUInt8: return "uint8";
		default: return c10::toString(t);
	}
}

// COPY hands the kernels a contiguous copy when needed; REJECT refuses a non-contiguous tensor instead, for tensors the
// kernels write in place and for the arrays the TSDF grid owns.
enum Contiguity { COPY, REJECT };

// The check of one tensor argument: `dtype`, sizes matching `dims` (-1 matches any size; no dims: any shape; `shape` is the
// pattern as messages print it, e.g. "[H, W, 3]"), on a CUDA device, `like`'s device when given.
torch::Tensor arg(const torch::Tensor& t, const char* name, torch::ScalarType dtype, std::initializer_list<int64_t> dims = {}, const char* shape = "",
                  const torch::Tensor* like = nullptr, Contiguity mode = COPY) {
	TORCH_CHECK(t.scalar_type() == dtype, name, " must be ", dtype_name(dtype), ", got ", t.scalar_type());
	bool fits = dims.size() == 0 || t.dim() == (int64_t)dims.size();
	for (int64_t i = 0; fits && i < (int64_t)dims.size(); i++) fits = dims.begin()[i] < 0 || t.size(i) == dims.begin()[i];
	TORCH_CHECK(fits, name, " must be ", shape, ", got ", t.sizes());
	TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor: no CPU path");
	TORCH_CHECK(!like || t.device() == like->device(), name, " must be on the same device as the other inputs");
	if (mode == COPY) return t.contiguous();
	TORCH_CHECK(t.is_contiguous(), name, " must be contiguous");
	return t;
}

// the rasterizer's optional float32 inputs: an empty tensor (torch.Tensor([]) on the CPU) is absent and stays so
torch::Tensor as_input(const torch::Tensor& t, const torch::Tensor& like, const char* name) {
	return t.numel() == 0 ? t : arg(t, name, torch::kFloat32, {}, "", &like);
}

// an empty byte tensor on `like`'s device, for the C ABI's resize callback to grow
torch::Tensor bytes(const torch::Tensor& like) { return torch::empty({0}, like.options().dtype(torch::kByte)); }

// the first n rows of `dtype` values shaped `k` in a byte buffer the C ABI resized
torch::Tensor rows(const torch::Tensor& buffer, torch::ScalarType dtype, int64_t n, std::initializer_list<int64_t> k) {
	std::vector<int64_t> shape{n};
	shape.insert(shape.end(), k);
	return buffer.narrow(0, 0, c10::multiply_integers(shape) * (int64_t)c10::elementSize(dtype)).view(dtype).view(shape);
}

// Debug aid (`_C.set_poison(byte)`, tests only): every scratch buffer and every empty()-allocated output is filled with
// `byte` before the kernels run, so a read of memory the kernels did not write themselves changes the result instead of
// silently depending on what the caching allocator handed out (fresh pages in one process, stale data in another).
int g_poison = -1;

void poison(const torch::Tensor& t) {
	if (g_poison >= 0 && t.defined() && t.numel() > 0 && t.is_cuda())
		cudaMemsetAsync(t.data_ptr(), g_poison, t.nbytes(), at::cuda::getCurrentCUDAStream(t.device().index()).stream());
}

torch::Tensor new_empty(at::IntArrayRef shape, const torch::TensorOptions& o) {
	torch::Tensor t = torch::empty(shape, o);
	poison(t);
	return t;
}

char* resize_cb(void* user, size_t bytes) {
	auto* t = reinterpret_cast<torch::Tensor*>(user);
	t->resize_({(long long)bytes});
	poison(*t);
	return reinterpret_cast<char*>(t->data_ptr());
}

void check(int64_t rc) {
	if (rc < 0) throw std::runtime_error(std::string(rgs_last_error()));
}

// The rasterizer has no CPU fallback: refuse host tensors, then run on the device of means3D.
c10::Device rasterizer_device(const torch::Tensor& means3D, const torch::Tensor* points3D = nullptr) {
	TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor: no CPU path");
	TORCH_CHECK(!points3D || points3D->is_cuda(), "points3D must be a CUDA tensor: no CPU path");
	return means3D.device();
}

// number of SH coefficients per Gaussian for either layout
int sh_coeffs(const torch::Tensor& sh, const torch::Tensor& sh_rest = torch::Tensor()) {
	int M = 0;
	if (sh.size(0) != 0) M = sh.size(1);
	if (sh_rest.defined() && sh_rest.numel() != 0) M += sh_rest.size(1);
	return M;
}

// One rasterizer call's camera and Gaussians as the C ABI takes them, built from the reference's arguments, with the tensors behind
// their pointers.  Building it checks means3D (and integrate's query points) and switches to the device of means3D for the call.
// With `sh_rest` (split-SH symbols) the SH coefficients come split into `sh` [P,1,3] and `sh_rest` [P,M-1,3].
struct Frame {
	c10::cuda::CUDAGuard guard;
	torch::Tensor bg, view, proj, pos, means, opac, shs, shs_rest, cols, scale, rot, cov;
	rgs_camera cam;
	rgs_gaussians g;

	static c10::Device checked_device(const torch::Tensor& means3D, const torch::Tensor* points3D) {
		if (means3D.ndimension() != 2 || means3D.size(1) != 3) {
			AT_ERROR("means3D must have dimensions (num_points, 3)");
		}
		if (points3D && (points3D->ndimension() != 2 || points3D->size(1) != 3)) {
			AT_ERROR("points3D must have dimensions (num_points, 3)");
		}
		return rasterizer_device(means3D, points3D);
	}

	Frame(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors, const torch::Tensor& opacity,
	      const torch::Tensor& scales, const torch::Tensor& rotations, float scale_modifier, const torch::Tensor& cov3D_precomp,
	      const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, float tan_fovx, float tan_fovy, float kernel_size, int H, int W,
	      const torch::Tensor& sh, int degree, const torch::Tensor& campos, bool prefiltered, bool require_coord, bool require_depth, bool debug,
	      int row_begin, int row_end, bool compact, const torch::Tensor& sh_rest = torch::Tensor(), const torch::Tensor* points3D = nullptr)
	    : guard(checked_device(means3D, points3D)) {
		bg = as_input(background, means3D, "background");
		view = as_input(viewmatrix, means3D, "viewmatrix");
		proj = as_input(projmatrix, means3D, "projmatrix");
		pos = as_input(campos, means3D, "campos");
		cam = rgs_camera{W, H, tan_fovx, tan_fovy, kernel_size, scale_modifier, view.data_ptr<float>(), proj.data_ptr<float>(), pos.data_ptr<float>(),
		                 bg.data_ptr<float>(), degree, sh_coeffs(sh, sh_rest), require_coord, require_depth, prefiltered, debug, row_begin, row_end,
		                 compact};
		means = as_input(means3D, means3D, "means3D");
		opac = as_input(opacity, means3D, "opacity");
		shs = as_input(sh, means3D, "sh");
		cols = as_input(colors, means3D, "colors_precomp");
		scale = as_input(scales, means3D, "scales");
		rot = as_input(rotations, means3D, "rotations");
		cov = as_input(cov3D_precomp, means3D, "cov3D_precomp");
		g = rgs_gaussians{(int)means3D.size(0), opt_ptr(means), opt_ptr(opac), opt_ptr(shs), opt_ptr(cols), opt_ptr(scale), opt_ptr(rot), opt_ptr(cov), nullptr};
		if (sh_rest.defined() && sh_rest.numel() != 0) {
			TORCH_CHECK(sh.dim() == 3 && sh.size(1) == 1 && sh_rest.dim() == 3 && sh_rest.size(0) == sh.size(0) && sh_rest.size(2) == 3,
			            "split SH layout needs shs_dc [P,1,3] and shs_rest [P,M-1,3]");
			shs_rest = as_input(sh_rest, means3D, "shs_rest");
			g.shs_rest = shs_rest.data_ptr<float>();
		}
	}
};

// Pixel rows of tile rows [row_begin, row_end) in an H-row image: the height of compact slab maps, as slab_height in rgs_api.cu
// gives it for compact_slab.
int compact_rows(int H, int row_begin, int row_end) { return std::max(0, std::min(row_end * 16, H) - row_begin * 16); }

// The seven maps of a forward: [C, H, W], or with `compact` only the slab's pixel rows.  They are zero-filled when nothing is drawn,
// and so are full-size maps of a slab that is not the whole image, whose rows outside the slab the library does not write.
struct Maps {
	torch::TensorOptions opts;
	int H, W;
	bool compact;
	torch::Tensor color, coord, mcoord, alpha, normal, depth, mdepth;

	int height(int row_begin, int row_end) const { return compact ? compact_rows(H, row_begin, row_end) : H; }

	void make(int row_begin, int row_end, bool zero) {  // tile rows [row_begin, row_end); row_end < 0: to the last
		const int grid_y = (H + 15) / 16;
		if (row_end < 0) row_end = grid_y;
		const bool fill = zero || (!compact && !(row_begin == 0 && row_end == grid_y));
		const int h = height(row_begin, row_end);
		auto img = [&](int ch) { return fill ? torch::zeros({ch, h, W}, opts) : new_empty({ch, h, W}, opts); };
		color = img(3), depth = img(1), mdepth = img(1), coord = img(3), mcoord = img(3), alpha = img(1), normal = img(3);
	}

	void point(rgs_forward_out& out) const {
		out.out_color = color.data_ptr<float>();
		out.out_coord = coord.data_ptr<float>();
		out.out_mcoord = mcoord.data_ptr<float>();
		out.out_alpha = alpha.data_ptr<float>();
		out.out_normal = normal.data_ptr<float>();
		out.out_depth = depth.data_ptr<float>();
		out.out_mdepth = mdepth.data_ptr<float>();
	}
};

// rgs_forward_balanced's maps callback: the maps of the slab the library chose
int32_t balanced_maps_cb(void* user, int32_t row_begin, int32_t row_end, int32_t height, rgs_forward_out* out) {
	auto* m = reinterpret_cast<Maps*>(user);
	if (height != m->height(row_begin, row_end)) return 1;
	try {
		m->make(row_begin, row_end, false);
	} catch (const std::exception&) {
		return 1;
	}
	m->point(*out);
	return 0;
}

// A balanced forward's rank of `world_size`, and what it returns beyond the slab's outputs: the partition (world_size + 1 tile-row
// cuts) and the per-row statistics [2, grid_y] (instances, longest tile list) on the host.
struct Balance {
	int world_size, rank;
	std::vector<int32_t> cuts;
	torch::Tensor stats;
};

using FwdResult = std::tuple<int, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor,
                             torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>;

// The forward of tile rows [row_begin, row_end) (the whole image: 0, -1), or with `balance` of the slab the frame's own tile
// counts give its rank, or with `preset` of the whole image binned into the preset's capacities (rgs_forward_preset; num_rendered
// is then preset->instances).
FwdResult forward_impl(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors, const torch::Tensor& opacity,
                       const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier, const torch::Tensor& cov3D_precomp,
                       const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy,
                       const float kernel_size, const int image_height, const int image_width, const torch::Tensor& sh, const int degree,
                       const torch::Tensor& campos, const bool prefiltered, const bool require_coord, const bool require_depth, const bool debug,
                       int row_begin, int row_end, const torch::Tensor& sh_rest = torch::Tensor(), bool compact = false, Balance* balance = nullptr,
                       const rgs_preset* preset = nullptr) {
	const Frame f(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
	              kernel_size, image_height, image_width, sh, degree, campos, prefiltered, require_coord, require_depth, debug, row_begin, row_end, compact,
	              sh_rest);
	const int P = f.g.P, H = image_height, W = image_width;
	Maps m{means3D.options().dtype(torch::kFloat32), H, W, compact};
	if (!balance) m.make(row_begin, row_end, P == 0);  // P == 0: the reference returns all-zero maps (rasterize_points.cu:90)
	torch::Tensor radii = P == 0 ? torch::zeros({P}, means3D.options().dtype(torch::kInt32)) : new_empty({P}, means3D.options().dtype(torch::kInt32));
	torch::Tensor geomBuffer = bytes(means3D), binningBuffer = bytes(means3D), imgBuffer = bytes(means3D);
	rgs_buffers bufs{resize_cb, &geomBuffer, resize_cb, &binningBuffer, resize_cb, &imgBuffer};
	rgs_forward_out fo{};
	fo.radii = radii.data_ptr<int>();
	const cudaStream_t stream = at::cuda::getCurrentCUDAStream().stream();
	int64_t rc = 0;
	if (!balance) {
		m.point(fo);
		if (preset) rc = P != 0 ? rgs_forward_preset(&f.cam, &f.g, &fo, &bufs, preset, stream) : preset->instances;
		else if (P != 0) rc = rgs_forward(&f.cam, &f.g, &fo, &bufs, stream);
		check(rc);
	} else {
		const int grid_x = (W + 15) / 16, grid_y = (H + 15) / 16;
		TORCH_CHECK(balance->world_size > 0 && balance->rank >= 0 && balance->rank < balance->world_size, "rank ", balance->rank, " is not a rank of ",
		            balance->world_size);
		TORCH_CHECK(H > 0 && W > 0, "image size must be positive");
		balance->cuts.resize(balance->world_size + 1);
		balance->stats = torch::zeros({2, grid_y}, torch::dtype(torch::kInt64));
		std::vector<uint32_t> row_stats((size_t)2 * grid_y, 0u);
		if (P == 0) {  // nothing to render: the partition of empty rows and all-zero maps, as rasterize_gaussians_slab returns them
			check(rgs_balance_partition(grid_y, grid_x, balance->world_size, row_stats.data(), balance->cuts.data()));
			m.make(balance->cuts[balance->rank], balance->cuts[balance->rank + 1], true);
		} else {
			check(rc = rgs_forward_balanced(&f.cam, &f.g, balance->world_size, balance->rank, &fo, balanced_maps_cb, &m, &bufs, balance->cuts.data(),
			                                row_stats.data(), stream));
			auto acc = balance->stats.accessor<int64_t, 2>();
			for (int y = 0; y < grid_y; y++) {
				acc[0][y] = row_stats[y];
				acc[1][y] = row_stats[grid_y + y];
			}
		}
	}
	return std::make_tuple((int)rc, m.color, m.coord, m.mcoord, m.alpha, m.normal, m.depth, m.mdepth, radii, geomBuffer, binningBuffer, imgBuffer);
}

// rasterize_gaussians_slab's 12-tuple for the slab the frame's tile counts give rank `rank` of `world_size`, then the partition and
// the per-row statistics
py::tuple RasterizeBalanced(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors, const torch::Tensor& opacity,
                            const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier, const torch::Tensor& cov3D_precomp,
                            const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy,
                            const float kernel_size, const int image_height, const int image_width, const torch::Tensor& sh, const int degree,
                            const torch::Tensor& campos, const bool prefiltered, const bool require_coord, const bool require_depth, const bool debug,
                            const int world_size, const int rank, const bool compact) {
	Balance b{world_size, rank};
	const FwdResult out = forward_impl(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix,
	                                   tan_fovx, tan_fovy, kernel_size, image_height, image_width, sh, degree, campos, prefiltered, require_coord,
	                                   require_depth, debug, 0, -1, torch::Tensor(), compact, &b);
	py::list cuts;
	for (int32_t c : b.cuts) cuts.append(c);
	return std::apply([&](const auto&... o) { return py::make_tuple(o..., cuts, b.stats); }, out);
}

// the library's partition of `row_instances` (one count per tile row) over `world_size` ranks: world_size + 1 tile-row cuts
std::vector<int32_t> BalancePartition(const std::vector<int64_t>& row_instances, const int grid_x, const int world_size) {
	std::vector<uint32_t> rows(row_instances.size());
	for (size_t y = 0; y < rows.size(); y++) {
		TORCH_CHECK(row_instances[y] >= 0 && row_instances[y] <= (int64_t)UINT32_MAX, "row instance counts must fit in 32 bits");
		rows[y] = (uint32_t)row_instances[y];
	}
	std::vector<int32_t> cuts(std::max(world_size, 0) + 1);
	check(rgs_balance_partition((int32_t)rows.size(), grid_x, world_size, rows.data(), cuts.data()));
	return cuts;
}

// `_graph.rasterize_gaussians`: rasterize_gaussians (split SH when sh_rest is not empty) binned into the capacities `instances` and
// `longest_list`, with no host read, so that it can be captured in a CUDA graph.  `status` int32 [4] on the device of means3D is
// accumulated in place (rgs_preset in include/rgs_b200.h).
FwdResult RasterizePreset(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors, const torch::Tensor& opacity,
                          const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier, const torch::Tensor& cov3D_precomp,
                          const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy,
                          const float kernel_size, const int image_height, const int image_width, const torch::Tensor& sh, const int degree,
                          const torch::Tensor& campos, const bool prefiltered, const bool require_coord, const bool require_depth, const bool debug,
                          const torch::Tensor& sh_rest, const int64_t instances, const int64_t longest_list, const torch::Tensor& status) {
	TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor: no CPU path");
	const torch::Tensor st = arg(status, "status", torch::kInt32, {4}, "[4]", &means3D, REJECT);
	TORCH_CHECK(instances >= 0 && longest_list >= 0 && longest_list <= INT32_MAX, "instances and longest_list must be non-negative (longest_list < 2^31)");
	const rgs_preset preset{instances, (int32_t)longest_list, reinterpret_cast<uint32_t*>(st.data_ptr<int32_t>())};
	return forward_impl(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
	                    kernel_size, image_height, image_width, sh, degree, campos, prefiltered, require_coord, require_depth, debug, 0, -1, sh_rest, false,
	                    nullptr, &preset);
}

// ---- the reference's four symbols ------------------------------------------------------------------------------

FwdResult RasterizeGaussiansCUDA(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors,
                                 const torch::Tensor& opacity, const torch::Tensor& scales, const torch::Tensor& rotations,
                                 const float scale_modifier, const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix,
                                 const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy, const float kernel_size,
                                 const int image_height, const int image_width, const torch::Tensor& sh, const int degree,
                                 const torch::Tensor& campos, const bool prefiltered, const bool require_coord, const bool require_depth,
                                 const bool debug) {
	return forward_impl(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx,
	                    tan_fovy, kernel_size, image_height, image_width, sh, degree, campos, prefiltered, require_coord, require_depth, debug, 0, -1);
}

// The inputs of the backward stages: the frame and rgs_backward_in.  The whole backward and stage 1 pass `maps`: the upstream
// gradients of the seven maps (color, coord, mcoord, depth, mdepth, alpha, normal), then the forward's normal and alpha maps.  Their
// height is read off the colour gradient like the reference does (rasterize_points.cu:171-172), except for compact slab maps, which
// need the image height.  Stage 2 reads no maps nor the binning and image buffers: it passes no maps and the image size.
struct Backward {
	Frame f;
	torch::Tensor maps[9], radii, geom, binning, image;
	rgs_backward_in in{};

	Backward(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& radii_, const torch::Tensor& colors,
	         const torch::Tensor& opacity, const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier,
	         const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx,
	         const float tan_fovy, const float kernel_size, std::initializer_list<torch::Tensor> maps_, const torch::Tensor& sh, const int degree,
	         const torch::Tensor& campos, const torch::Tensor& geomBuffer, const int R, const torch::Tensor& binningBuffer,
	         const torch::Tensor& imageBuffer, const bool require_coord, const bool require_depth, const bool debug, int row_begin, int row_end,
	         bool compact, int image_height, int image_width, const torch::Tensor& sh_rest = torch::Tensor())
	    : f(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
	        kernel_size, maps_.size() == 0 || (compact && image_height > 0) ? image_height : maps_.begin()[0].size(1),
	        maps_.size() == 0 ? image_width : maps_.begin()[0].size(2), sh, degree, campos, false, require_coord, require_depth, debug, row_begin,
	        row_end, compact, sh_rest) {
		TORCH_CHECK(!compact || image_height > 0, "compact slab maps need the full image height");
		static const char* const names[9] = {"dL_dout_color", "dL_dout_coord", "dL_dout_mcoord", "dL_dout_depth", "dL_dout_mdepth",
		                                     "dL_dout_alpha", "dL_dout_normal", "normalmap", "alphas"};
		const float** ptrs[9] = {&in.dL_dout_color, &in.dL_dout_coord, &in.dL_dout_mcoord, &in.dL_dout_depth, &in.dL_dout_mdepth,
		                         &in.dL_dout_alpha, &in.dL_dout_normal, &in.out_normal, &in.out_alpha};
		for (size_t i = 0; i < maps_.size(); i++) {
			maps[i] = as_input(maps_.begin()[i], means3D, names[i]);
			*ptrs[i] = maps[i].data_ptr<float>();
		}
		radii = radii_.contiguous();
		geom = geomBuffer.contiguous();
		binning = binningBuffer.contiguous();
		image = imageBuffer.contiguous();
		in.radii = radii.data_ptr<int>();
		in.geom_buffer = reinterpret_cast<const char*>(geom.data_ptr());
		in.binning_buffer = reinterpret_cast<const char*>(binning.data_ptr());
		in.image_buffer = reinterpret_cast<const char*>(image.data_ptr());
		in.num_rendered = R;
	}
};

using BwdResult = std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>;

struct GradTensors {
	torch::Tensor means3D, means2D, colors, opacity, cov3D, sh, sh_rest, scales, rotations;
	rgs_backward_out out;
	BwdResult reference_tuple() const { return std::make_tuple(means2D, colors, opacity, means3D, cov3D, sh, scales, rotations); }
};

void alloc_grads(GradTensors& t, const torch::Tensor& means3D, int P, int M, bool split_sh = false) {
	auto o = means3D.options();
	auto mk = [&](std::initializer_list<int64_t> shape) { return P == 0 ? torch::zeros(shape, o) : new_empty(shape, o); };
	t.means3D = mk({P, 3});
	t.means2D = mk({P, 3});
	t.colors = mk({P, 3});
	t.opacity = mk({P, 1});
	t.cov3D = mk({P, 6});
	t.sh = mk({P, split_sh ? 1 : M, 3});
	if (split_sh) t.sh_rest = mk({P, M - 1, 3});
	t.scales = mk({P, 3});
	t.rotations = mk({P, 4});
	t.out.dL_dmeans2D = t.means2D.data_ptr<float>();
	t.out.dL_dcolors = t.colors.data_ptr<float>();
	t.out.dL_dopacity = t.opacity.data_ptr<float>();
	t.out.dL_dmeans3D = t.means3D.data_ptr<float>();
	t.out.dL_dcov3D = t.cov3D.data_ptr<float>();
	t.out.dL_dsh = M > 0 ? t.sh.data_ptr<float>() : nullptr;
	t.out.dL_dscales = t.scales.data_ptr<float>();
	t.out.dL_drotations = t.rotations.data_ptr<float>();
	t.out.dL_dsh_rest = split_sh ? t.sh_rest.data_ptr<float>() : nullptr;
}

// the reference's backward; with `sh_rest` (split-SH symbol) the SH coefficients come split into `sh` [P,1,3] and `sh_rest` [P,M-1,3]
GradTensors backward_impl(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& radii, const torch::Tensor& colors,
                          const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier, const torch::Tensor& cov3D_precomp,
                          const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy,
                          const float kernel_size, const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_coord,
                          const torch::Tensor& dL_dout_mcoord, const torch::Tensor& dL_dout_depth, const torch::Tensor& dL_dout_mdepth,
                          const torch::Tensor& dL_dout_alpha, const torch::Tensor& dL_dout_normal, const torch::Tensor& normalmap,
                          const torch::Tensor& sh, const int degree, const torch::Tensor& campos, const torch::Tensor& geomBuffer, const int R,
                          const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer, const torch::Tensor& alphas, const bool require_coord,
                          const bool require_depth, const bool debug, const torch::Tensor& sh_rest) {
	// backward does not receive the opacities (rasterize_points.h:43-76)
	const Backward b(background, means3D, radii, colors, torch::empty({0}), scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix,
	                 tan_fovx, tan_fovy, kernel_size,
	                 {dL_dout_color, dL_dout_coord, dL_dout_mcoord, dL_dout_depth, dL_dout_mdepth, dL_dout_alpha, dL_dout_normal, normalmap, alphas}, sh,
	                 degree, campos, geomBuffer, R, binningBuffer, imageBuffer, require_coord, require_depth, debug, 0, -1, false, -1, -1, sh_rest);
	TORCH_CHECK(!sh_rest.defined() || sh_rest.numel() != 0, "split SH layout needs a non-empty shs_rest");
	GradTensors gt;
	alloc_grads(gt, means3D, b.f.g.P, b.f.cam.sh_coeffs, sh_rest.defined());
	if (b.f.g.P != 0) {
		torch::Tensor scratch = bytes(means3D);
		check(rgs_backward(&b.f.cam, &b.f.g, &b.in, &gt.out, resize_cb, &scratch, at::cuda::getCurrentCUDAStream().stream()));
	}
	return gt;
}

BwdResult RasterizeGaussiansBackwardCUDA(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& radii,
                                         const torch::Tensor& colors, const torch::Tensor& scales, const torch::Tensor& rotations,
                                         const float scale_modifier, const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix,
                                         const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy, const float kernel_size,
                                         const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_coord,
                                         const torch::Tensor& dL_dout_mcoord, const torch::Tensor& dL_dout_depth,
                                         const torch::Tensor& dL_dout_mdepth, const torch::Tensor& dL_dout_alpha,
                                         const torch::Tensor& dL_dout_normal, const torch::Tensor& normalmap, const torch::Tensor& sh,
                                         const int degree, const torch::Tensor& campos, const torch::Tensor& geomBuffer, const int R,
                                         const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer, const torch::Tensor& alphas,
                                         const bool require_coord, const bool require_depth, const bool debug) {
	return backward_impl(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx,
	                     tan_fovy, kernel_size, dL_dout_color, dL_dout_coord, dL_dout_mcoord, dL_dout_depth, dL_dout_mdepth, dL_dout_alpha,
	                     dL_dout_normal, normalmap, sh, degree, campos, geomBuffer, R, binningBuffer, imageBuffer, alphas, require_coord,
	                     require_depth, debug, torch::Tensor())
	    .reference_tuple();
}

torch::Tensor markVisible(torch::Tensor& means3D, torch::Tensor& viewmatrix, torch::Tensor& projmatrix) {
	const int P = means3D.size(0);
	torch::Tensor present = torch::full({P}, false, means3D.options().dtype(at::kBool));
	if (P != 0) {
		const c10::cuda::CUDAGuard guard(rasterizer_device(means3D));
		torch::Tensor m = means3D.contiguous(), v = viewmatrix.contiguous(), pr = projmatrix.contiguous();
		check(rgs_mark_visible(P, m.data_ptr<float>(), v.data_ptr<float>(), pr.data_ptr<float>(), reinterpret_cast<uint8_t*>(present.data_ptr<bool>()),
		                       at::cuda::getCurrentCUDAStream().stream()));
	}
	return present;
}

// GOF-style opacity integration at query points (rasterize_points.h:83-107, rasterize_points.cu:269-388): the call
// marching-tetrahedra mesh extraction makes once per view.  Same argument list and 10-tuple as the reference
// (view2gaussian_precomp and subpixel_offset are accepted and unused there as well).
std::tuple<int, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
IntegrateGaussiansToPointsCUDA(const torch::Tensor& background, const torch::Tensor& points3D, const torch::Tensor& means3D, const torch::Tensor& colors,
                               const torch::Tensor& opacity, const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier,
                               const torch::Tensor& cov3D_precomp, const torch::Tensor& view2gaussian_precomp, const torch::Tensor& viewmatrix,
                               const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy, const float kernel_size,
                               const torch::Tensor& subpixel_offset, const int image_height, const int image_width, const torch::Tensor& sh,
                               const int degree, const torch::Tensor& campos, const bool prefiltered, const bool debug) {
	const Frame f(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
	              kernel_size, image_height, image_width, sh, degree, campos, prefiltered, false, true, debug, 0, -1, false, torch::Tensor(), &points3D);
	const int PN = points3D.size(0), P = f.g.P, H = image_height, W = image_width;
	auto int_opts = means3D.options().dtype(torch::kInt32);
	auto float_opts = means3D.options().dtype(torch::kFloat32);
	const bool run = P != 0 && PN != 0;  // rasterize_points.cu:341: otherwise the fill values below are returned
	torch::Tensor out_color = run ? new_empty({9, H, W}, float_opts) : torch::zeros({9, H, W}, float_opts);
	torch::Tensor radii = run ? new_empty({P}, int_opts) : torch::zeros({P}, int_opts);
	torch::Tensor out_alpha_integrated = run ? new_empty({PN}, float_opts) : torch::full({PN}, 1.0, float_opts);
	torch::Tensor out_color_integrated = run ? new_empty({PN, 3}, float_opts) : torch::zeros({PN, 3}, float_opts);
	torch::Tensor out_coordinate2d = run ? new_empty({PN, 2}, float_opts) : torch::zeros({PN, 2}, float_opts);
	torch::Tensor out_sdf = run ? new_empty({PN}, float_opts) : torch::full({PN}, -1000.0, float_opts);
	torch::Tensor geomBuffer = bytes(means3D), binningBuffer = bytes(means3D), imgBuffer = bytes(means3D), pointBuffer = bytes(means3D);
	int rendered = 0;
	if (run) {
		torch::Tensor pts = as_input(points3D, means3D, "points3D");
		rgs_integrate_io io{PN, pts.data_ptr<float>(), out_color.data_ptr<float>(), out_alpha_integrated.data_ptr<float>(),
		                    out_color_integrated.data_ptr<float>(), out_coordinate2d.data_ptr<float>(), out_sdf.data_ptr<float>(), radii.data_ptr<int>()};
		rgs_buffers bufs{resize_cb, &geomBuffer, resize_cb, &binningBuffer, resize_cb, &imgBuffer};
		int32_t overflowed = 0;
		const int64_t rc = rgs_integrate(&f.cam, &f.g, &io, &bufs, resize_cb, &pointBuffer, &overflowed,  // always read: 4 bytes on a call that synchronises anyway
		                                 at::cuda::getCurrentCUDAStream().stream());
		check(rc);
		rendered = (int)rc;
		if (overflowed > 0) printf("ERROR: Maximal contributors are met in %d pixels. This should be fixed!\n", overflowed);  // forward.cu:1128
	}
	return std::make_tuple(rendered, out_color, out_alpha_integrated, out_color_integrated, out_coordinate2d, out_sdf, radii, geomBuffer, binningBuffer,
	                       imgBuffer);
}

// ---- multi-GPU extras ---------------------------------------------------------------------------------------------

// stage 1: the packed screen-space gradient accumulator [P, rgs_grad_stride] (additive across slabs).  Without an exchange
// in a fresh tensor; with one, the rows SUMMED over the ranks, as a view of the exchange's result buffer that stays valid
// until the next call on this exchange.
torch::Tensor backward_render_impl(rgs_exchange* ex, const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& radii,
                                   const torch::Tensor& colors, const torch::Tensor& scales, const torch::Tensor& rotations,
                                   const float scale_modifier, const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix,
                                   const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy, const float kernel_size,
                                   const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_coord, const torch::Tensor& dL_dout_mcoord,
                                   const torch::Tensor& dL_dout_depth, const torch::Tensor& dL_dout_mdepth, const torch::Tensor& dL_dout_alpha,
                                   const torch::Tensor& dL_dout_normal, const torch::Tensor& normalmap, const torch::Tensor& sh, const int degree,
                                   const torch::Tensor& campos, const torch::Tensor& geomBuffer, const int R, const torch::Tensor& binningBuffer,
                                   const torch::Tensor& imageBuffer, const torch::Tensor& alphas, const bool require_coord, const bool require_depth,
                                   const bool debug, const int tile_row_begin, const int tile_row_end, const bool compact, const int image_height) {
	const Backward b(background, means3D, radii, colors, torch::empty({0}), scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix,
	                 tan_fovx, tan_fovy, kernel_size,
	                 {dL_dout_color, dL_dout_coord, dL_dout_mcoord, dL_dout_depth, dL_dout_mdepth, dL_dout_alpha, dL_dout_normal, normalmap, alphas}, sh,
	                 degree, campos, geomBuffer, R, binningBuffer, imageBuffer, require_coord, require_depth, debug, tile_row_begin, tile_row_end,
	                 compact, image_height, -1);
	const int P = b.f.g.P;
	const int GS = rgs_grad_stride(require_coord, require_depth);
	torch::Tensor acc = ex ? torch::Tensor() : P == 0 ? torch::zeros({P, GS}, means3D.options()) : new_empty({P, GS}, means3D.options());
	if (P != 0) {
		const cudaStream_t stream = at::cuda::getCurrentCUDAStream().stream();
		check(ex ? rgs_backward_render_exchange(&b.f.cam, &b.f.g, &b.in, ex, stream)
		         : rgs_backward_render(&b.f.cam, &b.f.g, &b.in, acc.data_ptr<float>(), stream));
	}
	return ex ? torch::from_blob(const_cast<float*>(rgs_exchange_result(ex)), {P, GS}, means3D.options().dtype(torch::kFloat32)) : acc;
}

// The two Python symbols of stage 1 call `impl` without an exchange, or with one passed as an integer handle.  The arguments
// they share (`A`) are deduced from `impl`, so that the 36-name list is written once.
template <class... A>
auto without_exchange(torch::Tensor (*impl)(rgs_exchange*, A...)) {
	return [impl](A... a) { return impl(nullptr, a...); };
}

template <class... A>
auto with_exchange(torch::Tensor (*impl)(rgs_exchange*, A...)) {
	return [impl](const int64_t ex, A... a) {
		TORCH_CHECK(ex != 0, "null exchange handle");
		return impl(reinterpret_cast<rgs_exchange*>(ex), a...);
	};
}

// ---- device-side exchange of the accumulator rows over peer memory (rgs_exchange_*) ----
// The exchange object is handed to Python as an integer handle; the IPC handle as a CPU uint8 tensor [64] the caller
// all-gathers with torch.distributed before `exchange_connect`.
std::tuple<int64_t, torch::Tensor> ExchangeCreate(const int rank, const int world, const int64_t capacity_rows, const int row_floats, const int device) {
	const c10::cuda::CUDAGuard guard(c10::Device(c10::kCUDA, device));
	rgs_exchange* ex = nullptr;
	torch::Tensor handle = torch::zeros({RGS_IPC_HANDLE_BYTES}, torch::kUInt8);
	check(rgs_exchange_create(rank, world, capacity_rows, row_floats, &ex, handle.data_ptr()));
	return std::make_tuple((int64_t)reinterpret_cast<intptr_t>(ex), handle);
}

void ExchangeConnect(const int64_t ex, const torch::Tensor& all_handles, const int device) {
	const c10::cuda::CUDAGuard guard(c10::Device(c10::kCUDA, device));
	torch::Tensor h = all_handles.to(torch::kCPU).contiguous();
	TORCH_CHECK(h.scalar_type() == torch::kUInt8 && h.numel() % RGS_IPC_HANDLE_BYTES == 0, "handles must be a uint8 tensor [world, 64]");
	check(rgs_exchange_connect(reinterpret_cast<rgs_exchange*>(ex), h.data_ptr()));
}

// views of the exchange's persistent local accumulator / result rows, and the bare exchange step (self-check, tools)
torch::Tensor ExchangeAccumulator(const int64_t ex, const int P, const int row_floats, const int device) {
	return torch::from_blob(rgs_exchange_accumulator(reinterpret_cast<rgs_exchange*>(ex)), {P, row_floats},
	                        torch::TensorOptions().dtype(torch::kFloat32).device(torch::kCUDA, device));
}

torch::Tensor ExchangeResult(const int64_t ex, const int P, const int row_floats, const int device) {
	return torch::from_blob(const_cast<float*>(rgs_exchange_result(reinterpret_cast<rgs_exchange*>(ex))), {P, row_floats},
	                        torch::TensorOptions().dtype(torch::kFloat32).device(torch::kCUDA, device));
}

void ExchangeRows(const int64_t ex, const torch::Tensor& tiles_touched, const torch::Tensor& radii) {
	const torch::Tensor t = arg(tiles_touched, "tiles_touched", torch::kInt32), r = arg(radii, "radii", torch::kInt32);
	const c10::cuda::CUDAGuard guard(r.device());
	check(rgs_exchange_rows(reinterpret_cast<rgs_exchange*>(ex), (int)r.numel(), reinterpret_cast<const uint32_t*>(t.data_ptr<int>()), r.data_ptr<int>(),
	                        at::cuda::getCurrentCUDAStream().stream()));
}

int ExchangeStatus(const int64_t ex) {
	const int rc = rgs_exchange_status(reinterpret_cast<rgs_exchange*>(ex), at::cuda::getCurrentCUDAStream().stream());
	check(rc);
	return rc;
}

void ExchangeDestroy(const int64_t ex) { rgs_exchange_destroy(reinterpret_cast<rgs_exchange*>(ex)); }


// stage 2: accumulator (after the cross-rank sum) -> the reference's 8-tuple of parameter gradients
BwdResult BackwardPreprocessCUDA(const torch::Tensor& grad_accum, const torch::Tensor& background, const torch::Tensor& means3D,
                                 const torch::Tensor& radii, const torch::Tensor& colors, const torch::Tensor& opacity, const torch::Tensor& scales,
                                 const torch::Tensor& rotations, const float scale_modifier, const torch::Tensor& cov3D_precomp,
                                 const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy,
                                 const float kernel_size, const int image_height, const int image_width, const torch::Tensor& sh, const int degree,
                                 const torch::Tensor& campos, const torch::Tensor& geomBuffer, const bool require_coord, const bool require_depth,
                                 const bool debug) {
	const Backward b(background, means3D, radii, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx,
	                 tan_fovy, kernel_size, {}, sh, degree, campos, geomBuffer, 0, geomBuffer, geomBuffer, require_coord, require_depth, debug, 0, -1,
	                 false, image_height, image_width);
	GradTensors gt;
	alloc_grads(gt, means3D, b.f.g.P, b.f.cam.sh_coeffs);
	if (b.f.g.P != 0) {
		torch::Tensor acc = as_input(grad_accum, means3D, "grad_accum");
		check(rgs_backward_preprocess(&b.f.cam, &b.f.g, &b.in, acc.data_ptr<float>(), &gt.out, at::cuda::getCurrentCUDAStream().stream()));
	}
	return gt.reference_tuple();
}

// ---- fused activations / densification statistics (opt-in, SURVEY.md 8f row 1) --------------------------------------------

std::tuple<torch::Tensor, torch::Tensor, torch::Tensor> ActivateForward(const torch::Tensor& raw_scaling, const torch::Tensor& raw_opacity,
                                                                        const torch::Tensor& raw_rotation, const torch::Tensor& filter_3D) {
	const torch::Tensor s = arg(raw_scaling, "raw_scaling", torch::kFloat32), o = as_input(raw_opacity, s, "raw_opacity"),
	                    r = as_input(raw_rotation, s, "raw_rotation"), f = as_input(filter_3D, s, "filter_3D");
	const c10::cuda::CUDAGuard guard(s.device());
	const int P = s.size(0);
	TORCH_CHECK(s.numel() == 3 * (int64_t)P && o.numel() == P && r.numel() == 4 * (int64_t)P && f.numel() == P, "activate: shapes must be [P,3] [P,1] [P,4] [P,1]");
	torch::Tensor scales = new_empty({P, 3}, s.options()), opacity = new_empty({P, 1}, s.options()), rot = new_empty({P, 4}, s.options());
	if (P)
		check(rgs_activate_forward(P, s.data_ptr<float>(), o.data_ptr<float>(), r.data_ptr<float>(), f.data_ptr<float>(), scales.data_ptr<float>(),
		                           opacity.data_ptr<float>(), rot.data_ptr<float>(), at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(scales, opacity, rot);
}

std::tuple<torch::Tensor, torch::Tensor, torch::Tensor> ActivateBackward(const torch::Tensor& raw_scaling, const torch::Tensor& raw_opacity,
                                                                         const torch::Tensor& raw_rotation, const torch::Tensor& filter_3D,
                                                                         const torch::Tensor& g_scales, const torch::Tensor& g_opacity,
                                                                         const torch::Tensor& g_rotations) {
	const torch::Tensor s = arg(raw_scaling, "raw_scaling", torch::kFloat32), o = as_input(raw_opacity, s, "raw_opacity"),
	                    r = as_input(raw_rotation, s, "raw_rotation"), f = as_input(filter_3D, s, "filter_3D"), gs = as_input(g_scales, s, "g_scales"),
	                    go = as_input(g_opacity, s, "g_opacity"), gr = as_input(g_rotations, s, "g_rotations");
	const c10::cuda::CUDAGuard guard(s.device());
	const int P = s.size(0);
	TORCH_CHECK(gs.numel() == 3 * (int64_t)P && go.numel() == P && gr.numel() == 4 * (int64_t)P, "activate backward: gradient shapes must be [P,3] [P,1] [P,4]");
	torch::Tensor ds = new_empty({P, 3}, s.options()), dop = new_empty({P, 1}, s.options()), dr = new_empty({P, 4}, s.options());
	if (P)
		check(rgs_activate_backward(P, s.data_ptr<float>(), o.data_ptr<float>(), r.data_ptr<float>(), f.data_ptr<float>(), gs.data_ptr<float>(),
		                            go.data_ptr<float>(), gr.data_ptr<float>(), ds.data_ptr<float>(), dop.data_ptr<float>(), dr.data_ptr<float>(),
		                            at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(ds, dop, dr);
}

void DensificationStats(const torch::Tensor& means2D_grad, const torch::Tensor& radii, torch::Tensor& grad_accum, torch::Tensor& grad_accum_abs,
                        torch::Tensor& grad_accum_abs_max, torch::Tensor& denom, torch::Tensor& max_radii2D) {
	const torch::Tensor g = arg(means2D_grad, "means2D.grad", torch::kFloat32);
	const c10::cuda::CUDAGuard guard(g.device());
	const int P = g.size(0);
	if (P == 0) return;
	torch::Tensor rad = radii.contiguous();
	const std::pair<const char*, const torch::Tensor*> stats[] = {
	    {"grad_accum", &grad_accum}, {"grad_accum_abs", &grad_accum_abs}, {"grad_accum_abs_max", &grad_accum_abs_max}, {"denom", &denom}};
	for (const auto& [name, t] : stats) {
		arg(*t, name, torch::kFloat32, {}, "", &g, REJECT);
		TORCH_CHECK(t->numel() == P, "densification statistics must be [P,1] tensors");
	}
	float* mr = nullptr;
	if (max_radii2D.numel() != 0) {
		arg(max_radii2D, "max_radii2D", torch::kFloat32, {}, "", &g, REJECT);
		TORCH_CHECK(max_radii2D.numel() == P, "max_radii2D must be [P]");
		mr = max_radii2D.data_ptr<float>();
	}
	check(rgs_densification_stats(P, g.data_ptr<float>(), rad.data_ptr<int>(), grad_accum.data_ptr<float>(), grad_accum_abs.data_ptr<float>(),
	                              grad_accum_abs_max.data_ptr<float>(), denom.data_ptr<float>(), mr, at::cuda::getCurrentCUDAStream().stream()));
}

// returns (filter_3D [P,1], max_distance [1])
std::tuple<torch::Tensor, torch::Tensor> Compute3DFilter(const torch::Tensor& xyz, const torch::Tensor& cams, const double focal_length) {
	const torch::Tensor x = arg(xyz, "xyz", torch::kFloat32), c = as_input(cams, x, "camera table");
	const c10::cuda::CUDAGuard guard(x.device());
	const int P = x.size(0);
	TORCH_CHECK(c.numel() % 16 == 0, "camera table must be [n_cams,16]");
	const int n = (int)(c.numel() / 16);
	torch::Tensor out = new_empty({P, 1}, x.options()), mx = torch::zeros({1}, x.options());
	if (P)
		check(rgs_compute_3d_filter(P, x.data_ptr<float>(), n, n ? c.data_ptr<float>() : nullptr, (float)focal_length, out.data_ptr<float>(),
		                            mx.data_ptr<float>(), at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(out, mx);
}

// ---- fused image-side losses (opt-in, SURVEY.md 8f row 2) -----------------------------------------------------------------

// returns (sums [2] float64: sum of the SSIM map, sum |img - gt|; dmaps [3, planes, H, W] or empty)
std::tuple<torch::Tensor, torch::Tensor> SsimL1Forward(const torch::Tensor& img, const torch::Tensor& gt, const bool need_grad, const int row_lo_in,
                                                        const int row_hi_in) {
	TORCH_CHECK(img.dim() >= 2 && img.numel() == gt.numel() && img.size(-1) == gt.size(-1) && img.size(-2) == gt.size(-2),
	            "ssim: images must have the same number of elements and the same [H, W]");
	const torch::Tensor a = arg(img, "img1", torch::kFloat32), b = arg(gt, "img2", torch::kFloat32, {}, "", &a);
	const c10::cuda::CUDAGuard guard(a.device());
	const int H = a.size(-2), W = a.size(-1);
	const int planes = (int)(a.numel() / ((int64_t)H * W));
	torch::Tensor sums = new_empty({2}, a.options().dtype(torch::kFloat64));
	torch::Tensor dmaps = need_grad ? new_empty({3, planes, H, W}, a.options()) : torch::empty({0}, a.options());
	const int row_lo = row_lo_in, row_hi = row_hi_in < 0 ? H : row_hi_in;  // (0, -1): the whole image
	check(rgs_ssim_l1_forward_rows(planes, H, W, row_lo, row_hi, a.data_ptr<float>(), b.data_ptr<float>(), need_grad ? dmaps.data_ptr<float>() : nullptr,
	                               sums.data_ptr<double>(), at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(sums, dmaps);
}

torch::Tensor SsimL1Backward(const torch::Tensor& img, const torch::Tensor& gt, const torch::Tensor& dmaps, const double w_ssim, const double w_l1,
                             const torch::Tensor& upstream, const int row_lo_in, const int row_hi_in) {
	const torch::Tensor a = arg(img, "img1", torch::kFloat32), b = arg(gt, "img2", torch::kFloat32, {}, "", &a),
	                    d = arg(dmaps, "dmaps", torch::kFloat32, {}, "", &a);
	const c10::cuda::CUDAGuard guard(a.device());
	const int H = a.size(-2), W = a.size(-1);
	const int planes = (int)(a.numel() / ((int64_t)H * W));
	TORCH_CHECK(d.numel() == 3 * a.numel(), "ssim backward: dmaps do not belong to these images");
	torch::Tensor up;
	const float* up_ptr = nullptr;
	if (upstream.defined() && upstream.numel() != 0) {
		TORCH_CHECK(upstream.numel() == 1, "ssim backward: upstream gradient must be a scalar");
		up = arg(upstream, "upstream gradient", torch::kFloat32, {}, "", &a);
		up_ptr = up.data_ptr<float>();
	}
	const int row_lo = row_lo_in, row_hi = row_hi_in < 0 ? H : row_hi_in;
	const bool whole = row_lo == 0 && row_hi == H;
	torch::Tensor out = whole ? new_empty(a.sizes(), a.options()) : torch::zeros(a.sizes(), a.options());  // slab: rows far from the slab stay zero
	check(rgs_ssim_l1_backward_rows(planes, H, W, row_lo, row_hi, a.data_ptr<float>(), b.data_ptr<float>(), d.data_ptr<float>(), (float)w_ssim,
	                                (float)w_l1, up_ptr, out.data_ptr<float>(), at::cuda::getCurrentCUDAStream().stream()));
	return out.view(img.sizes());
}

// returns (loss_sum [1] float64, d_normal [3,H,W], d_expected, d_median)
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor> NormalConsistency(const torch::Tensor& rendered_normal,
                                                                                           const torch::Tensor& map_expected,
                                                                                           const torch::Tensor& map_median, const bool from_depth,
                                                                                           const double inv_fx, const double inv_fy, const double cx,
                                                                                           const double cy, const double w_expected,
                                                                                           const double w_median) {
	const torch::Tensor n = arg(rendered_normal, "rendered_normal", torch::kFloat32, {3, -1, -1}, "[3,H,W]"),
	                    e = arg(map_expected, "expected map", torch::kFloat32, {}, "", &n), m = arg(map_median, "median map", torch::kFloat32, {}, "", &n);
	const c10::cuda::CUDAGuard guard(n.device());
	const int H = n.size(1), W = n.size(2);
	const int64_t want = (from_depth ? 1 : 3) * (int64_t)H * W;
	TORCH_CHECK(e.numel() == want && m.numel() == want, from_depth ? "depth maps must be [1,H,W]" : "coordinate maps must be [3,H,W]");
	torch::Tensor loss = new_empty({1}, n.options().dtype(torch::kFloat64));
	torch::Tensor dn = new_empty(n.sizes(), n.options()), de = new_empty(e.sizes(), e.options()), dm = new_empty(m.sizes(), m.options());
	check(rgs_normal_consistency(H, W, from_depth ? 1 : 0, (float)inv_fx, (float)inv_fy, (float)cx, (float)cy, n.data_ptr<float>(), e.data_ptr<float>(),
	                             m.data_ptr<float>(), (float)w_expected, (float)w_median, loss.data_ptr<double>(), dn.data_ptr<float>(),
	                             de.data_ptr<float>(), dm.data_ptr<float>(), at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(loss, dn, de.view(map_expected.sizes()), dm.view(map_median.sizes()));
}

// Row-sharded form: loss rows [row_lo, row_hi) of an H-row image.  The maps hold rows [row_lo - 2, row_hi + 2) and the normal
// rows [row_lo - 1, row_hi + 1), both clipped to the image; returns (loss_sum [1] float64, d_normal, d_expected, d_median), each
// gradient [C, row_hi - row_lo, W].
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor> NormalConsistencyRows(
    const torch::Tensor& rendered_normal, const torch::Tensor& map_expected, const torch::Tensor& map_median, const bool from_depth, const double inv_fx,
    const double inv_fy, const double cx, const double cy, const double w_expected, const double w_median, const int64_t H, const int64_t row_lo,
    const int64_t row_hi) {
	TORCH_CHECK(H > 0 && 0 <= row_lo && row_lo <= row_hi && row_hi <= H, "normal consistency rows: need 0 <= row_lo <= row_hi <= H, got [", row_lo, ", ",
	            row_hi, ") of ", H);
	const int64_t C = from_depth ? 1 : 3;
	const int64_t m_rows = std::min(H, row_hi + 2) - std::max<int64_t>(0, row_lo - 2), n_rows = std::min(H, row_hi + 1) - std::max<int64_t>(0, row_lo - 1);
	const torch::Tensor n = arg(rendered_normal, "rendered_normal", torch::kFloat32, {3, n_rows, -1}, "[3, rows row_lo - 1 .. row_hi + 1, W]");
	const char* map_shape = from_depth ? "[1, rows row_lo - 2 .. row_hi + 2, W]" : "[3, rows row_lo - 2 .. row_hi + 2, W]";
	const int64_t W = n.size(2);
	const torch::Tensor e = arg(map_expected, "expected map", torch::kFloat32, {C, m_rows, W}, map_shape, &n),
	                    m = arg(map_median, "median map", torch::kFloat32, {C, m_rows, W}, map_shape, &n);
	const c10::cuda::CUDAGuard guard(n.device());
	torch::Tensor loss = new_empty({1}, n.options().dtype(torch::kFloat64));
	torch::Tensor dn = new_empty({3, row_hi - row_lo, W}, n.options()), de = new_empty({C, row_hi - row_lo, W}, n.options()),
	              dm = new_empty({C, row_hi - row_lo, W}, n.options());
	check(rgs_normal_consistency_rows((int)H, (int)W, (int)row_lo, (int)row_hi, from_depth ? 1 : 0, (float)inv_fx, (float)inv_fy, (float)cx, (float)cy,
	                                  n.data_ptr<float>(), e.data_ptr<float>(), m.data_ptr<float>(), (float)w_expected, (float)w_median,
	                                  loss.data_ptr<double>(), dn.data_ptr<float>(), de.data_ptr<float>(), dm.data_ptr<float>(),
	                                  at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(loss, dn, de, dm);
}

// ---- decoupled-appearance L1 loss (train.py:37-58; rgs_appearance_*) -------------------------------------------------------

// image [3,H0,W0] -> the center crop's bilinear downsample [3, H/32, W/32]
torch::Tensor AppearanceDownsample(const torch::Tensor& image) {
	const torch::Tensor a = arg(image, "image", torch::kFloat32, {3, -1, -1}, "[3, H, W]");
	TORCH_CHECK(a.size(1) >= 32 && a.size(2) >= 32, "appearance loss: the image must be at least 32 x 32, got ", a.sizes());
	const c10::cuda::CUDAGuard guard(a.device());
	const int H0 = a.size(1), W0 = a.size(2);
	torch::Tensor down = new_empty({3, H0 / 32, W0 / 32}, a.options());
	check(rgs_appearance_downsample(H0, W0, a.data_ptr<float>(), down.data_ptr<float>(), at::cuda::getCurrentCUDAStream().stream()));
	return down;
}

// d_image += the downsample's transpose applied to d_down (in place)
void AppearanceDownsampleBackward(const torch::Tensor& d_down, torch::Tensor& d_image) {
	arg(d_image, "d_image", torch::kFloat32, {3, -1, -1}, "[3, H, W]", nullptr, REJECT);
	const int H0 = d_image.size(1), W0 = d_image.size(2);
	TORCH_CHECK(H0 >= 32 && W0 >= 32, "appearance loss: the image must be at least 32 x 32, got ", d_image.sizes());
	const torch::Tensor g = arg(d_down, "d_down", torch::kFloat32, {}, "", &d_image);
	TORCH_CHECK(g.numel() == 3 * (int64_t)(H0 / 32) * (W0 / 32), "d_down does not belong to this image");
	const c10::cuda::CUDAGuard guard(d_image.device());
	check(rgs_appearance_downsample_backward(H0, W0, g.data_ptr<float>(), d_image.data_ptr<float>(), at::cuda::getCurrentCUDAStream().stream()));
}

struct AppearanceArgs {
	torch::Tensor image, gt, up4, w2, b2, w3, b3;
	int H0, W0;
};

AppearanceArgs appearance_args(const torch::Tensor& image, const torch::Tensor& gt, const torch::Tensor& up4, const torch::Tensor& w2, const torch::Tensor& b2,
                               const torch::Tensor& w3, const torch::Tensor& b3) {
	AppearanceArgs a;
	a.image = arg(image, "image", torch::kFloat32, {3, -1, -1}, "[3, H, W]");
	a.H0 = image.size(1);
	a.W0 = image.size(2);
	TORCH_CHECK(a.H0 >= 32 && a.W0 >= 32, "appearance loss: the image must be at least 32 x 32, got ", image.sizes());
	TORCH_CHECK(gt.sizes() == image.sizes(), "gt must have the image's shape");
	a.gt = arg(gt, "gt", torch::kFloat32, {}, "", &image);
	const int64_t H = a.H0 / 32 * 32, W = a.W0 / 32 * 32;
	a.up4 = arg(up4, "up4 output", torch::kFloat32, {}, "", &image);
	TORCH_CHECK(a.up4.numel() == 16 * (H / 2) * (W / 2), "up4 output must be [1, 16, ", H / 2, ", ", W / 2, "], got ", up4.sizes());
	a.w2 = arg(w2, "conv2 weight", torch::kFloat32, {}, "", &image);
	a.b2 = arg(b2, "conv2 bias", torch::kFloat32, {}, "", &image);
	a.w3 = arg(w3, "conv3 weight", torch::kFloat32, {}, "", &image);
	a.b3 = arg(b3, "conv3 bias", torch::kFloat32, {}, "", &image);
	TORCH_CHECK(a.w2.sizes() == torch::IntArrayRef({16, 16, 3, 3}) && a.b2.numel() == 16, "conv2 must be 16 -> 16 with 3x3 kernels");
	TORCH_CHECK(a.w3.sizes() == torch::IntArrayRef({3, 16, 3, 3}) && a.b3.numel() == 3, "conv3 must be 16 -> 3 with 3x3 kernels");
	return a;
}

// returns (loss [] float32, act [16, H, W] or empty, transformed [3, H, W] or empty)
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor> AppearanceL1Forward(const torch::Tensor& image, const torch::Tensor& gt, const torch::Tensor& up4,
                                                                             const torch::Tensor& w2, const torch::Tensor& b2, const torch::Tensor& w3,
                                                                             const torch::Tensor& b3, const bool need_act, const bool want_transformed) {
	const AppearanceArgs a = appearance_args(image, gt, up4, w2, b2, w3, b3);
	const c10::cuda::CUDAGuard guard(a.image.device());
	const int64_t H = a.H0 / 32 * 32, W = a.W0 / 32 * 32;
	const auto o = a.image.options();
	torch::Tensor act = need_act ? new_empty({16, H, W}, o) : torch::empty({0}, o);
	torch::Tensor out = want_transformed ? new_empty({3, H, W}, o) : torch::empty({0}, o);
	torch::Tensor partials = new_empty({RGS_APPEARANCE_CTAS}, o.dtype(torch::kFloat64));
	torch::Tensor loss = new_empty({}, o);
	check(rgs_appearance_l1_forward(a.H0, a.W0, a.image.data_ptr<float>(), a.gt.data_ptr<float>(), a.up4.data_ptr<float>(), a.w2.data_ptr<float>(),
	                                a.b2.data_ptr<float>(), a.w3.data_ptr<float>(), a.b3.data_ptr<float>(), need_act ? act.data_ptr<float>() : nullptr,
	                                want_transformed ? out.data_ptr<float>() : nullptr, partials.data_ptr<double>(), loss.data_ptr<float>(),
	                                at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(loss, act, out);
}

// returns (d_image [3,H0,W0] (crop term only), d_up4 shaped like up4, d_w2, d_b2, d_w3, d_b3)
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor> AppearanceL1Backward(
    const torch::Tensor& image, const torch::Tensor& gt, const torch::Tensor& up4, const torch::Tensor& act, const torch::Tensor& w2, const torch::Tensor& b2,
    const torch::Tensor& w3, const torch::Tensor& b3, const torch::Tensor& upstream) {
	const AppearanceArgs a = appearance_args(image, gt, up4, w2, b2, w3, b3);
	const c10::cuda::CUDAGuard guard(a.image.device());
	const int64_t H = a.H0 / 32 * 32, W = a.W0 / 32 * 32;
	const torch::Tensor ac = arg(act, "activations", torch::kFloat32, {}, "", &image);
	TORCH_CHECK(ac.numel() == 16 * H * W, "activations do not belong to this image");
	const float* up_ptr = nullptr;
	torch::Tensor up;
	if (upstream.defined() && upstream.numel() != 0) {
		TORCH_CHECK(upstream.numel() == 1, "appearance loss backward: upstream gradient must be a scalar");
		up = arg(upstream, "upstream gradient", torch::kFloat32, {}, "", &image);
		up_ptr = up.data_ptr<float>();
	}
	const auto o = a.image.options();
	torch::Tensor d_img = new_empty(a.image.sizes(), o), d_up4 = new_empty(up4.sizes(), o);
	torch::Tensor d_w2 = new_empty(w2.sizes(), o), d_b2 = new_empty(b2.sizes(), o), d_w3 = new_empty(w3.sizes(), o), d_b3 = new_empty(b3.sizes(), o);
	torch::Tensor partials = new_empty({RGS_APPEARANCE_CTAS, RGS_APPEARANCE_GRAD_FLOATS}, o.dtype(torch::kFloat64));
	torch::Tensor d_x = new_empty({16, H, W}, o);
	check(rgs_appearance_l1_backward(a.H0, a.W0, a.image.data_ptr<float>(), a.gt.data_ptr<float>(), a.up4.data_ptr<float>(), ac.data_ptr<float>(),
	                                 a.w2.data_ptr<float>(), a.w3.data_ptr<float>(), a.b3.data_ptr<float>(), up_ptr, d_img.data_ptr<float>(),
	                                 d_up4.data_ptr<float>(), d_w2.data_ptr<float>(), d_b2.data_ptr<float>(), d_w3.data_ptr<float>(), d_b3.data_ptr<float>(),
	                                 partials.data_ptr<double>(), d_x.data_ptr<float>(), at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(d_img, d_up4, d_w2, d_b2, d_w3, d_b3);
}

// Row-sharded forms (rgs_appearance_*_rows).  The image and gt windows hold image rows [image_lo, image_lo + rows) of an
// H0-row image; the slab is image rows [row_lo, row_hi).

// (c0, c1, oy_lo, oy_hi, u_lo, u_hi, act_lo, act_hi, dx_lo, dx_hi, img_lo, img_hi); host only
std::vector<int64_t> AppearanceRowWindows(const int64_t H0, const int64_t W0, const int64_t row_lo, const int64_t row_hi) {
	int32_t w[RGS_APPEARANCE_WINDOWS];
	check(rgs_appearance_row_windows((int)H0, (int)W0, (int)row_lo, (int)row_hi, w));
	return std::vector<int64_t>(w, w + RGS_APPEARANCE_WINDOWS);
}

struct AppearanceSlab {
	int32_t H0, W0, row_lo, row_hi, image_lo, win[RGS_APPEARANCE_WINDOWS];
};

AppearanceSlab appearance_slab(const torch::Tensor& window, const int64_t image_lo, const int64_t H0, const int64_t row_lo, const int64_t row_hi) {
	AppearanceSlab s;
	s.H0 = (int32_t)H0; s.W0 = (int32_t)window.size(2); s.row_lo = (int32_t)row_lo; s.row_hi = (int32_t)row_hi; s.image_lo = (int32_t)image_lo;
	check(rgs_appearance_row_windows(s.H0, s.W0, s.row_lo, s.row_hi, s.win));
	return s;
}

// image window [3, rows, W0] -> the owned low-res rows [3, oy_hi - oy_lo, W0 / 32]
torch::Tensor AppearanceDownsampleRows(const torch::Tensor& image, const int64_t image_lo, const int64_t H0, const int64_t row_lo, const int64_t row_hi) {
	const torch::Tensor a = arg(image, "image window", torch::kFloat32, {3, -1, -1}, "[3, rows, W]");
	const c10::cuda::CUDAGuard guard(a.device());
	const AppearanceSlab s = appearance_slab(a, image_lo, H0, row_lo, row_hi);
	torch::Tensor down = new_empty({3, s.win[3] - s.win[2], s.W0 / 32}, a.options());
	check(rgs_appearance_downsample_rows(s.H0, s.W0, s.row_lo, s.row_hi, a.data_ptr<float>(), s.image_lo, (int32_t)a.size(1), down.data_ptr<float>(),
	                                     at::cuda::getCurrentCUDAStream().stream()));
	return down;
}

// d_image [3, row_hi - row_lo, W0] += the taps of d_down [3, H/32, W/32] in the slab's rows (in place)
void AppearanceDownsampleBackwardRows(const torch::Tensor& d_down, torch::Tensor& d_image, const int64_t H0, const int64_t row_lo, const int64_t row_hi) {
	arg(d_image, "d_image", torch::kFloat32, {3, row_hi - row_lo, -1}, "[3, row_hi - row_lo, W]", nullptr, REJECT);
	const int32_t W0 = (int32_t)d_image.size(2);
	const torch::Tensor g = arg(d_down, "d_down", torch::kFloat32, {3, H0 / 32, W0 / 32}, "[3, H/32, W/32]", &d_image);
	const c10::cuda::CUDAGuard guard(d_image.device());
	check(rgs_appearance_downsample_backward_rows((int32_t)H0, W0, (int32_t)row_lo, (int32_t)row_hi, g.data_ptr<float>(), d_image.data_ptr<float>(),
	                                              at::cuda::getCurrentCUDAStream().stream()));
}

AppearanceArgs appearance_rows_args(const torch::Tensor& image, const torch::Tensor& gt, const torch::Tensor& up4, const torch::Tensor& w2,
                                    const torch::Tensor& b2, const torch::Tensor& w3, const torch::Tensor& b3, const int64_t H0) {
	AppearanceArgs a;
	a.image = arg(image, "image window", torch::kFloat32, {3, -1, -1}, "[3, rows, W]");
	a.H0 = (int)H0;
	a.W0 = (int)image.size(2);
	TORCH_CHECK(gt.sizes() == image.sizes(), "gt window must have the image window's shape");
	a.gt = arg(gt, "gt window", torch::kFloat32, {}, "", &a.image);
	const int64_t H = H0 / 32 * 32, W = a.W0 / 32 * 32;
	a.up4 = arg(up4, "up4 output", torch::kFloat32, {}, "", &a.image);
	TORCH_CHECK(a.up4.numel() == 16 * (H / 2) * (W / 2), "up4 output must be [1, 16, ", H / 2, ", ", W / 2, "], got ", up4.sizes());
	a.w2 = arg(w2, "conv2 weight", torch::kFloat32, {16, 16, 3, 3}, "[16, 16, 3, 3]", &a.image);
	a.b2 = arg(b2, "conv2 bias", torch::kFloat32, {16}, "[16]", &a.image);
	a.w3 = arg(w3, "conv3 weight", torch::kFloat32, {3, 16, 3, 3}, "[3, 16, 3, 3]", &a.image);
	a.b3 = arg(b3, "conv3 bias", torch::kFloat32, {3}, "[3]", &a.image);
	return a;
}

// returns (loss_sum [1] float64, act [16, act_hi - act_lo, W])
std::tuple<torch::Tensor, torch::Tensor> AppearanceL1ForwardRows(const torch::Tensor& image, const torch::Tensor& gt, const int64_t image_lo, const int64_t H0,
                                                                 const int64_t row_lo, const int64_t row_hi, const torch::Tensor& up4, const torch::Tensor& w2,
                                                                 const torch::Tensor& b2, const torch::Tensor& w3, const torch::Tensor& b3) {
	const AppearanceArgs a = appearance_rows_args(image, gt, up4, w2, b2, w3, b3, H0);
	const c10::cuda::CUDAGuard guard(a.image.device());
	const AppearanceSlab s = appearance_slab(a.image, image_lo, H0, row_lo, row_hi);
	const auto o = a.image.options();
	torch::Tensor act = new_empty({16, s.win[7] - s.win[6], a.W0 / 32 * 32}, o);
	torch::Tensor partials = new_empty({RGS_APPEARANCE_CTAS}, o.dtype(torch::kFloat64));
	torch::Tensor loss_sum = new_empty({1}, o.dtype(torch::kFloat64));
	check(rgs_appearance_l1_forward_rows(s.H0, s.W0, s.row_lo, s.row_hi, a.image.data_ptr<float>(), a.gt.data_ptr<float>(), s.image_lo, (int32_t)a.image.size(1),
	                                     a.up4.data_ptr<float>(), a.w2.data_ptr<float>(), a.b2.data_ptr<float>(), a.w3.data_ptr<float>(), a.b3.data_ptr<float>(),
	                                     act.data_ptr<float>(), partials.data_ptr<double>(), loss_sum.data_ptr<double>(), at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(loss_sum, act);
}

// returns (d_image [3, row_hi - row_lo, W0] (crop term only), d_up4 owned rows [16, u_hi - u_lo, W/2], grad_row [2755] float64)
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor> AppearanceL1BackwardRows(
    const torch::Tensor& image, const torch::Tensor& gt, const int64_t image_lo, const int64_t H0, const int64_t row_lo, const int64_t row_hi,
    const torch::Tensor& up4, const torch::Tensor& act, const torch::Tensor& w2, const torch::Tensor& b2, const torch::Tensor& w3, const torch::Tensor& b3,
    const torch::Tensor& upstream) {
	const AppearanceArgs a = appearance_rows_args(image, gt, up4, w2, b2, w3, b3, H0);
	const c10::cuda::CUDAGuard guard(a.image.device());
	const AppearanceSlab s = appearance_slab(a.image, image_lo, H0, row_lo, row_hi);
	const int64_t W = a.W0 / 32 * 32;
	const torch::Tensor ac = arg(act, "activations", torch::kFloat32, {16, s.win[7] - s.win[6], W}, "[16, act_hi - act_lo, W]", &a.image);
	const float* up_ptr = nullptr;
	torch::Tensor up;
	if (upstream.defined() && upstream.numel() != 0) {
		TORCH_CHECK(upstream.numel() == 1, "appearance loss backward: upstream gradient must be a scalar");
		up = arg(upstream, "upstream gradient", torch::kFloat32, {}, "", &a.image);
		up_ptr = up.data_ptr<float>();
	}
	const auto o = a.image.options();
	torch::Tensor d_img = new_empty({3, row_hi - row_lo, a.W0}, o), d_up4 = new_empty({16, s.win[5] - s.win[4], W / 2}, o);
	torch::Tensor grad_row = new_empty({RGS_APPEARANCE_GRAD_FLOATS}, o.dtype(torch::kFloat64));
	torch::Tensor partials = new_empty({RGS_APPEARANCE_CTAS, RGS_APPEARANCE_GRAD_FLOATS}, o.dtype(torch::kFloat64));
	torch::Tensor d_x = new_empty({16, s.win[9] - s.win[8], W}, o);
	check(rgs_appearance_l1_backward_rows(s.H0, s.W0, s.row_lo, s.row_hi, a.image.data_ptr<float>(), a.gt.data_ptr<float>(), s.image_lo,
	                                      (int32_t)a.image.size(1), a.up4.data_ptr<float>(), ac.data_ptr<float>(), a.w2.data_ptr<float>(), a.w3.data_ptr<float>(),
	                                      a.b3.data_ptr<float>(), up_ptr, d_img.data_ptr<float>(), d_up4.data_ptr<float>(), grad_row.data_ptr<double>(),
	                                      partials.data_ptr<double>(), d_x.data_ptr<float>(), at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(d_img, d_up4, grad_row);
}

// The network's head (rgs_appearance_head_*): down [3, h, w], the embedding row [64] and the ten head parameters in the
// module's order (conv1.weight, conv1.bias, up1.conv.weight, ..., up4.conv.bias).
struct AppearanceHeadArgs {
	torch::Tensor down, emb;
	std::vector<torch::Tensor> p;
	int h, w;
};

AppearanceHeadArgs appearance_head_args(const torch::Tensor& down, const torch::Tensor& emb, const std::vector<torch::Tensor>& params) {
	static const char* names[10] = {"conv1 weight", "conv1 bias", "up1 weight", "up1 bias", "up2 weight", "up2 bias", "up3 weight", "up3 bias", "up4 weight", "up4 bias"};
	static const int64_t cin[5] = {67, 64, 32, 16, 8}, cout[5] = {256, 128, 64, 32, 16};
	AppearanceHeadArgs a;
	a.down = arg(down, "down", torch::kFloat32, {3, -1, -1}, "[3, h, w]");
	a.h = (int)a.down.size(1);
	a.w = (int)a.down.size(2);
	a.emb = arg(emb, "embedding row", torch::kFloat32, {64}, "[64]", &a.down);
	TORCH_CHECK(params.size() == 10, "appearance head: 10 parameters (conv1, up1..up4 weights and biases), got ", params.size());
	for (int i = 0; i < 10; i++) {
		const int l = i / 2;
		if (i % 2 == 0) {
			const std::string shape = "[" + std::to_string(cout[l]) + ", " + std::to_string(cin[l]) + ", 3, 3]";
			a.p.push_back(arg(params[i], names[i], torch::kFloat32, {cout[l], cin[l], 3, 3}, shape.c_str(), &a.down));
		} else {
			const std::string shape = "[" + std::to_string(cout[l]) + "]";
			a.p.push_back(arg(params[i], names[i], torch::kFloat32, {cout[l]}, shape.c_str(), &a.down));
		}
	}
	return a;
}

const float* fp(const torch::Tensor& t) { return t.data_ptr<float>(); }

// returns (act [3840 h w], up4 [1, 16, 16h, 16w])
std::tuple<torch::Tensor, torch::Tensor> AppearanceHeadForward(const torch::Tensor& down, const torch::Tensor& emb, const std::vector<torch::Tensor>& params) {
	const AppearanceHeadArgs a = appearance_head_args(down, emb, params);
	const c10::cuda::CUDAGuard guard(a.down.device());
	const auto o = a.down.options();
	torch::Tensor act = new_empty({(int64_t)RGS_APPEARANCE_HEAD_ACT_PER_HW * a.h * a.w}, o), up4 = new_empty({1, 16, 16 * a.h, 16 * a.w}, o);
	const auto& p = a.p;
	check(rgs_appearance_head_forward(a.h, a.w, fp(a.down), fp(a.emb), fp(p[0]), fp(p[1]), fp(p[2]), fp(p[3]), fp(p[4]), fp(p[5]), fp(p[6]), fp(p[7]),
	                                  fp(p[8]), fp(p[9]), act.data_ptr<float>(), up4.data_ptr<float>(), at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(act, up4);
}

// returns [d_down [3, h, w], d_emb [64], the ten parameter gradients]
std::vector<torch::Tensor> AppearanceHeadBackward(const torch::Tensor& down, const torch::Tensor& emb, const std::vector<torch::Tensor>& params,
                                                  const torch::Tensor& act, const torch::Tensor& up4, const torch::Tensor& d_up4) {
	const AppearanceHeadArgs a = appearance_head_args(down, emb, params);
	const c10::cuda::CUDAGuard guard(a.down.device());
	const int64_t h = a.h, w = a.w;
	const torch::Tensor ac = arg(act, "head activations", torch::kFloat32, {RGS_APPEARANCE_HEAD_ACT_PER_HW * h * w}, "[3840 h w]", &a.down);
	const torch::Tensor u = arg(up4, "up4 output", torch::kFloat32, {1, 16, 16 * h, 16 * w}, "[1, 16, 16h, 16w]", &a.down);
	const torch::Tensor du = arg(d_up4, "d_up4", torch::kFloat32, {}, "", &a.down);
	TORCH_CHECK(du.numel() == u.numel(), "d_up4 must have up4's ", u.numel(), " elements, got ", d_up4.sizes());
	size_t bytes = 0;
	check(rgs_appearance_head_scratch_bytes(a.h, a.w, &bytes));
	const auto o = a.down.options();
	torch::Tensor scratch = new_empty({(int64_t)bytes}, o.dtype(torch::kByte));
	std::vector<torch::Tensor> out{new_empty({3, h, w}, o), new_empty({64}, o)};
	for (const torch::Tensor& t : a.p) out.push_back(new_empty(t.sizes(), o));
	float* g[12];
	for (int i = 0; i < 12; i++) g[i] = out[i].data_ptr<float>();
	const auto& p = a.p;
	check(rgs_appearance_head_backward(a.h, a.w, fp(a.down), fp(a.emb), fp(p[0]), fp(p[2]), fp(p[4]), fp(p[6]), fp(p[8]), fp(ac), fp(u), fp(du), g[0], g[1],
	                                   g[2], g[3], g[4], g[5], g[6], g[7], g[8], g[9], g[10], g[11], scratch.data_ptr(),
	                                   at::cuda::getCurrentCUDAStream().stream()));
	return out;
}

// ---- densify-and-prune and opacity reset (scene/gaussian_model.py:495-513, :662-741; rgs_densify_*, rgs_reset_opacity) ----------

// a per-Gaussian input: float32 on `like`'s device with `width` floats per row over P rows
torch::Tensor per_gaussian(const torch::Tensor& t, const char* name, int64_t P, int64_t width, const torch::Tensor* like) {
	const torch::Tensor a = arg(t, name, torch::kFloat32, {}, "", like);
	TORCH_CHECK(a.dim() >= 1 && a.size(0) == P && a.numel() == P * width, "densify: ", name, " must have ", width, " float(s) per row over ", P,
	            " rows, got ", t.sizes());
	return a;
}

// returns (flags [P] uint8, block_offsets int32, ratio_q [2] float32 = (ratio, Q), counts (C, S, K0, K1, K2))
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, std::vector<int64_t>> DensifySelect(
    const torch::Tensor& grad_accum, const torch::Tensor& grad_accum_abs, const torch::Tensor& denom, const torch::Tensor& scaling,
    const torch::Tensor& opacity, const double max_grad, const double dense, const double min_opacity, const bool prune_large,
    const double max_screen_size, const double world) {
	const torch::Tensor acc = arg(grad_accum, "xyz_gradient_accum", torch::kFloat32);
	TORCH_CHECK(acc.dim() >= 1 && acc.size(0) > 0, "densify: the model has no Gaussians");
	TORCH_CHECK(acc.size(0) <= INT32_MAX, "densify: at most 2^31 - 1 Gaussians");
	const int64_t P = acc.size(0);
	per_gaussian(acc, "xyz_gradient_accum", P, 1, nullptr);
	const torch::Tensor ab = per_gaussian(grad_accum_abs, "xyz_gradient_accum_abs", P, 1, &acc), dn = per_gaussian(denom, "denom", P, 1, &acc),
	                    sc = per_gaussian(scaling, "_scaling", P, 3, &acc), op = per_gaussian(opacity, "_opacity", P, 1, &acc);
	const c10::cuda::CUDAGuard guard(acc.device());
	const auto o = acc.options();
	torch::Tensor flags = new_empty({P}, o.dtype(torch::kUInt8));
	torch::Tensor offsets = new_empty({5 * (int64_t)rgs_densify_blocks((int)P) + 5}, o.dtype(torch::kInt32));
	torch::Tensor ratio_q = new_empty({2}, o), scratch = bytes(acc);
	rgs_densify_thresholds th;
	th.max_grad = (float)max_grad;
	th.dense = (float)dense;
	th.min_opacity = (float)min_opacity;
	th.max_screen_size = (float)max_screen_size;
	th.world = (float)world;
	th.inv_split = 1.0f / (float)(0.8 * 2);
	th.prune_large = prune_large ? 1 : 0;
	int32_t counts[5];
	check(rgs_densify_select((int)P, acc.data_ptr<float>(), ab.data_ptr<float>(), dn.data_ptr<float>(), sc.data_ptr<float>(), op.data_ptr<float>(), &th,
	                         flags.data_ptr<uint8_t>(), offsets.data_ptr<int32_t>(), ratio_q.data_ptr<float>(), counts, resize_cb, &scratch,
	                         at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(flags, offsets, ratio_q, std::vector<int64_t>(counts, counts + 5));
}

// returns (src [N] int32, draw [N] int32, std_clone [C,3], std_split [2S,3]), N = K0 + K1 + 2 K2
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor> DensifyPlan(const torch::Tensor& flags, const torch::Tensor& block_offsets,
                                                                                   const std::vector<int64_t>& counts, const torch::Tensor& scaling) {
	const torch::Tensor f = arg(flags, "flags", torch::kUInt8, {-1}, "[P]");
	const int64_t P = f.size(0);
	TORCH_CHECK(P > 0 && P <= INT32_MAX, "densify: the model has no Gaussians");
	const torch::Tensor bo = arg(block_offsets, "block_offsets", torch::kInt32, {5 * (int64_t)rgs_densify_blocks((int)P) + 5}, "[5 * blocks + 5]", &f);
	const torch::Tensor sc = per_gaussian(scaling, "_scaling", P, 3, &f);
	TORCH_CHECK(counts.size() == 5, "densify plan: five counts");
	int32_t c[5];
	for (int k = 0; k < 5; k++) {
		TORCH_CHECK(counts[k] >= 0 && counts[k] <= P, "densify plan: counts out of range");
		c[k] = (int32_t)counts[k];
	}
	const c10::cuda::CUDAGuard guard(f.device());
	const auto o = sc.options();
	const int64_t N = (int64_t)c[2] + c[3] + 2 * (int64_t)c[4];
	torch::Tensor src = new_empty({N}, o.dtype(torch::kInt32)), draw = new_empty({N}, o.dtype(torch::kInt32));
	torch::Tensor std_clone = new_empty({c[0], 3}, o), std_split = new_empty({2 * (int64_t)c[1], 3}, o);
	check(rgs_densify_plan((int)P, f.data_ptr<uint8_t>(), bo.data_ptr<int32_t>(), c, sc.data_ptr<float>(), N ? src.data_ptr<int32_t>() : nullptr,
	                       N ? draw.data_ptr<int32_t>() : nullptr, c[0] ? std_clone.data_ptr<float>() : nullptr,
	                       c[1] ? std_split.data_ptr<float>() : nullptr, at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(src, draw, std_clone, std_split);
}

// returns (xyz [N,3], scaling [N,3], one tensor [N, *column.shape[1:]] per column); columns: (tensor [P, ...], zero on new rows)
std::tuple<torch::Tensor, torch::Tensor, std::vector<torch::Tensor>> DensifyGather(const torch::Tensor& src, const torch::Tensor& draw, const int64_t C,
                                                                                    const torch::Tensor& xyz, const torch::Tensor& rotation,
                                                                                    const torch::Tensor& scaling, const torch::Tensor& sample_clone,
                                                                                    const torch::Tensor& sample_split,
                                                                                    const std::vector<std::tuple<torch::Tensor, bool>>& columns) {
	const torch::Tensor x = arg(xyz, "_xyz", torch::kFloat32);
	const int64_t P = x.size(0);
	per_gaussian(x, "_xyz", P, 3, nullptr);
	const torch::Tensor r = per_gaussian(rotation, "_rotation", P, 4, &x), sc = per_gaussian(scaling, "_scaling", P, 3, &x);
	const torch::Tensor s = arg(src, "src", torch::kInt32, {-1}, "[N]", &x), d = arg(draw, "draw", torch::kInt32, {-1}, "[N]", &x);
	const int64_t N = s.size(0);
	TORCH_CHECK(d.size(0) == N, "densify gather: src and draw differ in length");
	TORCH_CHECK(C >= 0 && C <= P, "densify gather: clone count out of range");
	const torch::Tensor smc = arg(sample_clone, "clone draws", torch::kFloat32, {C, 3}, "[C, 3]", &x);
	const torch::Tensor sms = arg(sample_split, "split draws", torch::kFloat32, {-1, 3}, "[2S, 3]", &x);
	TORCH_CHECK((int64_t)columns.size() <= RGS_DENSIFY_MAX_COLUMNS, "densify gather: at most ", RGS_DENSIFY_MAX_COLUMNS, " columns");
	const c10::cuda::CUDAGuard guard(x.device());
	const auto o = x.options();
	std::vector<torch::Tensor> ins, outs;
	std::vector<rgs_densify_column> cols;
	for (const auto& [t, zero_new] : columns) {
		const torch::Tensor in = arg(t, "column", torch::kFloat32, {}, "", &x);
		TORCH_CHECK(in.dim() >= 1 && in.size(0) == P, "densify gather: every column must have the model's ", P, " rows, got ", t.sizes());
		std::vector<int64_t> shape(in.sizes().begin(), in.sizes().end());
		shape[0] = N;
		torch::Tensor out = new_empty(shape, o);
		const int64_t width = P ? in.numel() / P : 0;
		if (width > 0 && N > 0) cols.push_back(rgs_densify_column{in.data_ptr<float>(), out.data_ptr<float>(), width, zero_new ? 1 : 0});
		ins.push_back(in);
		outs.push_back(out);
	}
	torch::Tensor xyz_out = new_empty({N, 3}, o), scaling_out = new_empty({N, 3}, o);
	check(rgs_densify_gather((int)N, s.data_ptr<int32_t>(), d.data_ptr<int32_t>(), (int)C, x.data_ptr<float>(), r.data_ptr<float>(), sc.data_ptr<float>(),
	                         C ? smc.data_ptr<float>() : nullptr, sms.size(0) ? sms.data_ptr<float>() : nullptr, 1.0f / (float)(0.8 * 2),
	                         xyz_out.data_ptr<float>(), scaling_out.data_ptr<float>(), (int)cols.size(), cols.data(),
	                         at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(xyz_out, scaling_out, outs);
}

// GaussianModel.reset_opacity's new raw opacity [P,1]
torch::Tensor ResetOpacity(const torch::Tensor& scaling, const torch::Tensor& opacity, const torch::Tensor& filter_3D) {
	const torch::Tensor op = arg(opacity, "_opacity", torch::kFloat32);
	const int64_t P = op.size(0);
	TORCH_CHECK(P > 0 && P <= INT32_MAX, "reset_opacity: the model has no Gaussians");
	per_gaussian(op, "_opacity", P, 1, nullptr);
	const torch::Tensor sc = per_gaussian(scaling, "_scaling", P, 3, &op), f = per_gaussian(filter_3D, "filter_3D", P, 1, &op);
	const c10::cuda::CUDAGuard guard(op.device());
	torch::Tensor out = new_empty({P, 1}, op.options());
	check(rgs_reset_opacity((int)P, sc.data_ptr<float>(), op.data_ptr<float>(), f.data_ptr<float>(), out.data_ptr<float>(),
	                        at::cuda::getCurrentCUDAStream().stream()));
	return out;
}

// simple_knn's distCUDA2 (reference scene/gaussian_model.py:315-316): points [P,3] float32 on a CUDA device -> [P] float32,
// the mean squared distance to the 3 nearest other points (rgs_knn_mean_dist2).  Non-contiguous input is accepted.
torch::Tensor KnnMeanDist2(const torch::Tensor& points) {
	const torch::Tensor x = arg(points, "distCUDA2: points", torch::kFloat32, {-1, 3}, "(num_points, 3)");
	TORCH_CHECK(x.size(0) <= INT32_MAX, "distCUDA2: at most 2^31 - 1 points");
	const c10::cuda::CUDAGuard guard(x.device());
	const int P = (int)x.size(0);
	torch::Tensor out = new_empty({P}, x.options()), scratch = bytes(x);
	if (P) check(rgs_knn_mean_dist2(P, x.data_ptr<float>(), out.data_ptr<float>(), resize_cb, &scratch, at::cuda::getCurrentCUDAStream().stream()));
	return out;
}

// ---- TSDF voxel-block grid (rgs_tsdf_*; Python side rade_gs_b200.tsdf.VoxelBlockGrid, which owns every array) ----------------

torch::Tensor grid_array(const py::object& grid, const char* name, torch::ScalarType type) {
	return arg(grid.attr(name).cast<torch::Tensor>(), name, type, {}, "", nullptr, REJECT);
}

// the C view of the grid; the Python object keeps the tensors alive
rgs_tsdf_grid tsdf_grid(const py::object& grid) {
	rgs_tsdf_grid g;
	torch::Tensor keys = grid_array(grid, "hash_keys", torch::kInt64), frame = grid_array(grid, "frame_keys", torch::kInt64);
	g.voxel_size = grid.attr("voxel_size").cast<float>();
	g.capacity = grid_array(grid, "stamps", torch::kInt32).numel();
	g.hash_slots = keys.numel();
	g.hash_keys = reinterpret_cast<uint64_t*>(keys.data_ptr<int64_t>());
	g.hash_values = grid_array(grid, "hash_values", torch::kInt32).data_ptr<int32_t>();
	g.tsdf = grid_array(grid, "tsdf", torch::kFloat32).data_ptr<float>();
	g.weight = grid_array(grid, "weight", torch::kFloat32).data_ptr<float>();
	g.color = grid_array(grid, "color", torch::kFloat32).data_ptr<float>();
	g.stamps = grid_array(grid, "stamps", torch::kInt32).data_ptr<int32_t>();
	g.frame_slots = frame.numel();
	g.frame_keys = reinterpret_cast<uint64_t*>(frame.data_ptr<int64_t>());
	g.frame_list = reinterpret_cast<uint64_t*>(grid_array(grid, "frame_list", torch::kInt64).data_ptr<int64_t>());
	g.counters = grid_array(grid, "counters", torch::kInt32).data_ptr<int32_t>();
	return g;
}

// intrinsic [3,3] and extrinsic [4,4] as CPU float64 tensors -> the fp32 camera of the contract (one conversion, here)
rgs_tsdf_camera tsdf_camera(const torch::Tensor& depth, const torch::Tensor& intrinsic, const torch::Tensor& extrinsic, double depth_scale, double depth_max,
                            double trunc_voxel_multiplier) {
	TORCH_CHECK(intrinsic.device().is_cpu() && intrinsic.scalar_type() == torch::kFloat64 && intrinsic.numel() == 9, "intrinsic must be a 3x3 matrix");
	TORCH_CHECK(extrinsic.device().is_cpu() && extrinsic.scalar_type() == torch::kFloat64 && extrinsic.numel() == 16, "extrinsic must be a 4x4 matrix");
	const torch::Tensor K = intrinsic.contiguous(), E = extrinsic.contiguous();
	const double* k = K.data_ptr<double>();
	const double* e = E.data_ptr<double>();
	rgs_tsdf_camera c;
	c.height = (int32_t)depth.size(0);
	c.width = (int32_t)depth.size(1);
	c.fx = (float)k[0];
	c.fy = (float)k[4];
	c.cx = (float)k[2];
	c.cy = (float)k[5];
	for (int r = 0; r < 3; r++) {
		for (int q = 0; q < 3; q++) c.R[3 * r + q] = (float)e[4 * r + q];
		c.t[r] = (float)e[4 * r + 3];
	}
	c.depth_scale = (float)depth_scale;
	c.depth_max = (float)depth_max;
	c.trunc_voxel_multiplier = (float)trunc_voxel_multiplier;
	return c;
}

// returns (number of touched blocks, or -1 when the frame-local hash is full; block coordinates int32 [n, 3]; allocated blocks)
std::tuple<int64_t, torch::Tensor, int64_t> TsdfTouch(const py::object& grid, const torch::Tensor& depth, const torch::Tensor& intrinsic,
                                                      const torch::Tensor& extrinsic, double depth_scale, double depth_max, double trunc_voxel_multiplier) {
	const torch::Tensor keys = grid_array(grid, "hash_keys", torch::kInt64);
	const c10::cuda::CUDAGuard guard(keys.device());
	const torch::Tensor d = arg(depth, "depth", torch::kFloat32, {-1, -1}, "[H, W]", &keys, REJECT);
	const rgs_tsdf_grid g = tsdf_grid(grid);
	const rgs_tsdf_camera c = tsdf_camera(d, intrinsic, extrinsic, depth_scale, depth_max, trunc_voxel_multiplier);
	torch::Tensor out = new_empty({g.frame_slots / 2, 3}, keys.options().dtype(torch::kInt32)), scratch = bytes(keys);
	int64_t allocated = 0;
	const int64_t n = rgs_tsdf_touch(&g, &c, d.data_ptr<float>(), out.data_ptr<int32_t>(), &allocated, resize_cb, &scratch,
	                                 at::cuda::getCurrentCUDAStream().stream());
	if (n == RGS_E_CAPACITY) return std::make_tuple((int64_t)-1, out.narrow(0, 0, 0), allocated);
	check(n);
	return std::make_tuple(n, out.narrow(0, 0, n).clone(), allocated);
}

void TsdfIntegrate(const py::object& grid, const torch::Tensor& block_coords, const torch::Tensor& depth, const torch::Tensor& color,
                   const torch::Tensor& intrinsic, const torch::Tensor& extrinsic, double depth_scale, double depth_max, double trunc_voxel_multiplier,
                   int call_id) {
	const torch::Tensor keys = grid_array(grid, "hash_keys", torch::kInt64);
	const c10::cuda::CUDAGuard guard(keys.device());
	arg(block_coords, "block_coords", torch::kInt32, {-1, 3}, "[N, 3]", &keys, REJECT);
	const torch::Tensor d = arg(depth, "depth", torch::kFloat32, {-1, -1}, "[H, W]", &keys, REJECT),
	                    col = arg(color, "color", torch::kFloat32, {-1, -1, 3}, "[H, W, 3]", &keys, REJECT);
	TORCH_CHECK(col.size(0) == d.size(0) && col.size(1) == d.size(1), "color and depth must have the same [H, W]");
	const rgs_tsdf_grid g = tsdf_grid(grid);
	const rgs_tsdf_camera c = tsdf_camera(d, intrinsic, extrinsic, depth_scale, depth_max, trunc_voxel_multiplier);
	torch::Tensor scratch = bytes(keys);
	check(rgs_tsdf_integrate(&g, &c, block_coords.size(0), block_coords.data_ptr<int32_t>(), d.data_ptr<float>(), col.data_ptr<float>(), call_id, resize_cb,
	                         &scratch, at::cuda::getCurrentCUDAStream().stream()));
}

void TsdfRehash(const py::object& grid, const torch::Tensor& old_keys, const torch::Tensor& old_values) {
	const torch::Tensor keys = grid_array(grid, "hash_keys", torch::kInt64);
	const c10::cuda::CUDAGuard guard(keys.device());
	arg(old_keys, "old hash keys", torch::kInt64, {}, "", &keys, REJECT);
	arg(old_values, "old hash values", torch::kInt32, {}, "", &keys, REJECT);
	TORCH_CHECK(old_keys.numel() == old_values.numel(), "old hash keys and values must have one length");
	const rgs_tsdf_grid g = tsdf_grid(grid);
	check(rgs_tsdf_rehash(&g, reinterpret_cast<const uint64_t*>(old_keys.data_ptr<int64_t>()), old_values.data_ptr<int32_t>(), old_keys.numel(),
	                      at::cuda::getCurrentCUDAStream().stream()));
}

// returns (keys int64 [N] ascending, pool indices int32 [N])
std::tuple<torch::Tensor, torch::Tensor> TsdfActiveBlocks(const py::object& grid) {
	const torch::Tensor hk = grid_array(grid, "hash_keys", torch::kInt64);
	const c10::cuda::CUDAGuard guard(hk.device());
	const rgs_tsdf_grid g = tsdf_grid(grid);
	torch::Tensor keys = new_empty({g.capacity}, hk.options()), pools = new_empty({g.capacity}, hk.options().dtype(torch::kInt32)), scratch = bytes(hk);
	const int64_t n = rgs_tsdf_active_blocks(&g, reinterpret_cast<uint64_t*>(keys.data_ptr<int64_t>()), pools.data_ptr<int32_t>(), resize_cb, &scratch,
	                                         at::cuda::getCurrentCUDAStream().stream());
	check(n);
	return std::make_tuple(keys.narrow(0, 0, n), pools.narrow(0, 0, n));
}

// returns (vertices f32 [V,3], colors f32 [V,3], triangles int32 [F,3])
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor> TsdfExtract(const py::object& grid, double weight_threshold) {
	const torch::Tensor hk = grid_array(grid, "hash_keys", torch::kInt64);
	const c10::cuda::CUDAGuard guard(hk.device());
	const rgs_tsdf_grid g = tsdf_grid(grid);
	torch::Tensor v = bytes(hk), c = bytes(hk), t = bytes(hk), scratch = bytes(hk);
	rgs_tsdf_mesh_out out{&v, &c, &t, 0, 0};
	check(rgs_tsdf_extract(&g, (float)weight_threshold, resize_cb, &out, &scratch, at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(rows(v, torch::kFloat32, out.num_vertices, {3}), rows(c, torch::kFloat32, out.num_vertices, {3}),
	                       rows(t, torch::kInt32, out.num_triangles, {3}));
}

torch::Tensor TsdfVertexNormals(const torch::Tensor& vertices, const torch::Tensor& triangles) {
	arg(vertices, "vertices", torch::kFloat32, {-1, 3}, "[V, 3]", nullptr, REJECT);
	arg(triangles, "triangles", torch::kInt32, {-1, 3}, "[F, 3]", &vertices, REJECT);
	const c10::cuda::CUDAGuard guard(vertices.device());
	const int64_t V = vertices.size(0), F = triangles.size(0);
	if (F > 0) {
		const auto mm = torch::aminmax(triangles);
		TORCH_CHECK(std::get<0>(mm).item<int32_t>() >= 0 && std::get<1>(mm).item<int32_t>() < V, "triangle vertex index out of [0, V)");
	}
	torch::Tensor normals = new_empty({V, 3}, vertices.options()), scratch = bytes(vertices);
	check(rgs_tsdf_vertex_normals(V, vertices.data_ptr<float>(), F, triangles.data_ptr<int32_t>(), normals.data_ptr<float>(), resize_cb, &scratch,
	                              at::cuda::getCurrentCUDAStream().stream()));
	return normals;
}

// ---- bounded TSDF, Open3D's legacy ScalableTSDFVolume (rgs_scalable_*; Python side rade_gs_b200.tsdf.ScalableTSDFVolume) ------

// rgb f32 [3,H,W], depth f32 [1,H,W] or [H,W], mask (None or H*W floats) -> (color uint8 [H,W,3], depth f32 [H,W])
std::tuple<torch::Tensor, torch::Tensor> ScalableRgbd(const torch::Tensor& rgb, const torch::Tensor& depth, double depth_trunc,
                                                     const c10::optional<torch::Tensor>& mask) {
	const torch::Tensor c = arg(rgb, "rgb", torch::kFloat32, {3, -1, -1}, "[3, H, W]");
	const int64_t H = c.size(1), W = c.size(2);
	const torch::Tensor d = arg(depth, "depth", torch::kFloat32, {}, "", &c);
	TORCH_CHECK(d.numel() == H * W && (d.dim() == 2 || (d.dim() == 3 && d.size(0) == 1)), "depth must be [1, H, W] or [H, W] like rgb ", c.sizes(),
	            ", got ", d.sizes());
	torch::Tensor m;
	if (mask && mask->defined()) {
		m = arg(*mask, "mask", torch::kFloat32, {}, "", &c);
		TORCH_CHECK(m.numel() == H * W, "mask must have H * W = ", H * W, " values, got ", m.sizes());
	}
	TORCH_CHECK(H <= INT32_MAX && W <= INT32_MAX, "image too large");
	const c10::cuda::CUDAGuard guard(c.device());
	torch::Tensor col = new_empty({H, W, 3}, c.options().dtype(torch::kUInt8)), dout = new_empty({H, W}, c.options());
	check(rgs_scalable_rgbd((int32_t)H, (int32_t)W, c.data_ptr<float>(), d.data_ptr<float>(), m.defined() ? m.data_ptr<float>() : nullptr, depth_trunc,
	                        col.data_ptr<uint8_t>(), dout.data_ptr<float>(), at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(col, dout);
}

// image f32 [3,H,W] -> uint8 [H,W,3] as save_img_u8 converts image * scale + offset
torch::Tensor ScalableImageU8(const torch::Tensor& image, double scale, double offset) {
	const torch::Tensor x = arg(image, "image", torch::kFloat32, {3, -1, -1}, "[3, H, W]");
	TORCH_CHECK(x.size(1) <= INT32_MAX && x.size(2) <= INT32_MAX, "image too large");
	const c10::cuda::CUDAGuard guard(x.device());
	torch::Tensor out = new_empty({x.size(1), x.size(2), 3}, x.options().dtype(torch::kUInt8));
	check(rgs_scalable_image_u8((int32_t)x.size(1), (int32_t)x.size(2), x.data_ptr<float>(), (float)scale, (float)offset, out.data_ptr<uint8_t>(),
	                            at::cuda::getCurrentCUDAStream().stream()));
	return out;
}

// returns (number of touched units, or -1 when the frame-local hash is full; unit coordinates int32 [n, 3]; allocated units)
std::tuple<int64_t, torch::Tensor, int64_t> ScalableTouch(const py::object& volume, const torch::Tensor& depth, const torch::Tensor& intrinsic,
                                                          const torch::Tensor& extrinsic, double sdf_trunc) {
	const torch::Tensor keys = grid_array(volume, "hash_keys", torch::kInt64);
	const c10::cuda::CUDAGuard guard(keys.device());
	const torch::Tensor d = arg(depth, "depth", torch::kFloat32, {-1, -1}, "[H, W]", &keys, REJECT);
	const rgs_tsdf_grid g = tsdf_grid(volume);
	const rgs_tsdf_camera c = tsdf_camera(d, intrinsic, extrinsic, 1.0, 1.0, 1.0);
	torch::Tensor out = new_empty({g.frame_slots / 2, 3}, keys.options().dtype(torch::kInt32)), scratch = bytes(keys);
	int64_t allocated = 0;
	const int64_t n = rgs_scalable_touch(&g, &c, (float)sdf_trunc, d.data_ptr<float>(), out.data_ptr<int32_t>(), &allocated, resize_cb, &scratch,
	                                     at::cuda::getCurrentCUDAStream().stream());
	if (n == RGS_E_CAPACITY) return std::make_tuple((int64_t)-1, out.narrow(0, 0, 0), allocated);
	check(n);
	return std::make_tuple(n, out.narrow(0, 0, n).clone(), allocated);
}

void ScalableIntegrate(const py::object& volume, const torch::Tensor& unit_coords, const torch::Tensor& depth, const torch::Tensor& color,
                       const torch::Tensor& intrinsic, const torch::Tensor& extrinsic, double sdf_trunc, int call_id) {
	const torch::Tensor keys = grid_array(volume, "hash_keys", torch::kInt64);
	const c10::cuda::CUDAGuard guard(keys.device());
	arg(unit_coords, "unit_coords", torch::kInt32, {-1, 3}, "[N, 3]", &keys, REJECT);
	const torch::Tensor d = arg(depth, "depth", torch::kFloat32, {-1, -1}, "[H, W]", &keys, REJECT),
	                    col = arg(color, "color", torch::kUInt8, {-1, -1, 3}, "[H, W, 3]", &keys, REJECT);
	TORCH_CHECK(col.size(0) == d.size(0) && col.size(1) == d.size(1), "color and depth must have the same [H, W]");
	const rgs_tsdf_grid g = tsdf_grid(volume);
	const rgs_tsdf_camera c = tsdf_camera(d, intrinsic, extrinsic, 1.0, 1.0, 1.0);
	torch::Tensor scratch = bytes(keys);
	check(rgs_scalable_integrate(&g, &c, (float)sdf_trunc, unit_coords.size(0), unit_coords.data_ptr<int32_t>(), d.data_ptr<float>(), col.data_ptr<uint8_t>(),
	                             call_id, resize_cb, &scratch, at::cuda::getCurrentCUDAStream().stream()));
}

// ---- DTU evaluation (rgs_dtu_*; Python side rade_gs_b200.dtu_eval) -------------------------------------------------------

// vertices f64 [V,3], faces int32 [F,3] -> the vertices followed by the surface samples, f64 [V + S, 3]
torch::Tensor DtuSampleMesh(const torch::Tensor& vertices, const torch::Tensor& faces, double density) {
	const torch::Tensor v = arg(vertices, "vertices", torch::kFloat64, {-1, 3}, "[N, 3]");
	const torch::Tensor f = arg(faces, "faces", torch::kInt32, {-1, 3}, "[F, 3]", &v);
	const c10::cuda::CUDAGuard guard(v.device());
	torch::Tensor pts = bytes(v), scratch = bytes(v), row_scratch = bytes(v);
	rgs_dtu_samples_out out{&pts, &scratch, &row_scratch, 0};
	check(rgs_dtu_sample_mesh(v.size(0), v.data_ptr<double>(), f.size(0), f.data_ptr<int32_t>(), density, resize_cb, &out,
	                          at::cuda::getCurrentCUDAStream().stream()));
	return rows(pts, torch::kFloat64, out.num_points, {3});
}

// points f64 [N,3] in processing order -> (kept bool [N], rounds)
std::tuple<torch::Tensor, int32_t> DtuRadiusDownsample(const torch::Tensor& points, double radius) {
	const torch::Tensor p = arg(points, "points", torch::kFloat64, {-1, 3}, "[N, 3]");
	const c10::cuda::CUDAGuard guard(p.device());
	torch::Tensor kept = new_empty({p.size(0)}, p.options().dtype(torch::kBool)), scratch = bytes(p);
	int32_t rounds = 0;
	check(rgs_dtu_radius_downsample(p.size(0), p.data_ptr<double>(), radius, reinterpret_cast<uint8_t*>(kept.data_ptr<bool>()), &rounds, resize_cb, &scratch,
	                                at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(kept, rounds);
}

// reference f64 [M,3], query f64 [N,3] -> (distance f64 [N], index int64 [N])
std::tuple<torch::Tensor, torch::Tensor> DtuNearest(const torch::Tensor& reference, const torch::Tensor& query) {
	const torch::Tensor r = arg(reference, "reference", torch::kFloat64, {-1, 3}, "[N, 3]"), q = arg(query, "query", torch::kFloat64, {-1, 3}, "[N, 3]", &r);
	const c10::cuda::CUDAGuard guard(r.device());
	torch::Tensor dist = new_empty({q.size(0)}, q.options()), index = new_empty({q.size(0)}, q.options().dtype(torch::kInt64)), scratch = bytes(r);
	check(rgs_dtu_nearest(r.size(0), r.data_ptr<double>(), q.size(0), q.data_ptr<double>(), dist.data_ptr<double>(), index.data_ptr<int64_t>(), resize_cb,
	                      &scratch, at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(dist, index);
}

// masks uint8 [n, H, W] (nonzero = set) -> disk(6) dilation, uint8 [n, H, W]
torch::Tensor DtuDilateMasks(const torch::Tensor& masks) {
	const torch::Tensor m = arg(masks, "masks", torch::kUInt8, {-1, -1, -1}, "[n, H, W]");
	const c10::cuda::CUDAGuard guard(m.device());
	torch::Tensor out = new_empty(m.sizes(), m.options());
	check(rgs_dtu_dilate_masks((int32_t)m.size(0), (int32_t)m.size(1), (int32_t)m.size(2), m.data_ptr<uint8_t>(), out.data_ptr<uint8_t>(),
	                           at::cuda::getCurrentCUDAStream().stream()));
	return out;
}

// vertices f64 [V,3], proj f64 [n,3,4], dilated uint8 [n,H,W] -> keep bool [V]
torch::Tensor DtuCullVertices(const torch::Tensor& vertices, const torch::Tensor& proj, const torch::Tensor& dilated) {
	const torch::Tensor v = arg(vertices, "vertices", torch::kFloat64, {-1, 3}, "[N, 3]");
	const torch::Tensor P = arg(proj, "proj", torch::kFloat64, {-1, 3, 4}, "[n, 3, 4]", &v),
	                    m = arg(dilated, "dilated", torch::kUInt8, {P.size(0), -1, -1}, "[n, H, W] with one mask per view", &v);
	const c10::cuda::CUDAGuard guard(v.device());
	torch::Tensor keep = new_empty({v.size(0)}, v.options().dtype(torch::kBool));
	check(rgs_dtu_cull_vertices(v.size(0), v.data_ptr<double>(), (int32_t)P.size(0), (int32_t)m.size(1), (int32_t)m.size(2), P.data_ptr<double>(),
	                            m.data_ptr<uint8_t>(), reinterpret_cast<uint8_t*>(keep.data_ptr<bool>()), at::cuda::getCurrentCUDAStream().stream()));
	return keep;
}

// ---- TNT evaluation (rgs_tnt_*; Python side rade_gs_b200.tnt_eval) -------------------------------------------------------

// a 4x4 transform as 16 host doubles (row-major), or an empty tensor for none
torch::Tensor tnt_host_transform(const torch::Tensor& T) {
	if (T.numel() == 0) return T;
	TORCH_CHECK(T.dim() == 2 && T.size(0) == 4 && T.size(1) == 4, "transform must be [4, 4], got ", T.sizes());
	return T.to(torch::kCPU, torch::kFloat64).contiguous();
}

// points f64 [N,3], transform f64 [4,4] or empty, polygon f64 [K,2] (CUDA) or empty -> (kept bool [N], cropped f64 [n,3])
std::tuple<torch::Tensor, torch::Tensor> TntCrop(const torch::Tensor& points, const torch::Tensor& transform, int64_t axis, double axis_min, double axis_max,
                                                 const torch::Tensor& polygon) {
	const torch::Tensor p = arg(points, "points", torch::kFloat64, {-1, 3}, "[N, 3]");
	const c10::cuda::CUDAGuard guard(p.device());
	const torch::Tensor T = tnt_host_transform(transform);
	torch::Tensor poly;
	rgs_tnt_crop_volume vol{};
	if (polygon.numel() > 0) {
		poly = arg(polygon, "polygon", torch::kFloat64, {-1, 2}, "[K, 2]", &p);
		vol = rgs_tnt_crop_volume{(int32_t)axis, (int32_t)poly.size(0), axis_min, axis_max, poly.data_ptr<double>()};
	}
	torch::Tensor kept = new_empty({p.size(0)}, p.options().dtype(torch::kBool)), cropped = new_empty({p.size(0), 3}, p.options()), scratch = bytes(p);
	int64_t n = 0;
	check(rgs_tnt_crop(p.size(0), p.data_ptr<double>(), T.numel() ? T.data_ptr<double>() : nullptr, polygon.numel() ? &vol : nullptr,
	                   reinterpret_cast<uint8_t*>(kept.data_ptr<bool>()), cropped.data_ptr<double>(), &n, resize_cb, &scratch,
	                   at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(kept, cropped.narrow(0, 0, n));
}

// points f64 [N,3] (contiguous CUDA), overwritten with T p
void TntTransform(torch::Tensor points, const torch::Tensor& transform) {
	arg(points, "points", torch::kFloat64, {-1, 3}, "[N, 3]", nullptr, REJECT);
	TORCH_CHECK(transform.numel() == 16, "transform must be [4, 4]");
	const c10::cuda::CUDAGuard guard(points.device());
	const torch::Tensor T = tnt_host_transform(transform);
	check(rgs_tnt_transform(points.size(0), points.data_ptr<double>(), T.data_ptr<double>(), at::cuda::getCurrentCUDAStream().stream()));
}

// points f64 [N,3] -> (means f64 [V,3] in ascending voxel key order, counts int64 [V])
std::tuple<torch::Tensor, torch::Tensor> TntVoxelDownsample(const torch::Tensor& points, double voxel) {
	const torch::Tensor p = arg(points, "points", torch::kFloat64, {-1, 3}, "[N, 3]");
	const c10::cuda::CUDAGuard guard(p.device());
	torch::Tensor means = bytes(p), counts = bytes(p), scratch = bytes(p);
	rgs_tnt_voxel_out out{&means, &counts, &scratch, 0};
	check(rgs_tnt_voxel_downsample(p.size(0), p.data_ptr<double>(), voxel, resize_cb, &out, at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(rows(means, torch::kFloat64, out.num_voxels, {3}), rows(counts, torch::kInt64, out.num_voxels, {}));
}

// source f64 [N,3], target f64 [M,3], dist f64 [N], index int64 [N] -> the 18 moments (CPU float64)
torch::Tensor TntIcpMoments(const torch::Tensor& source, const torch::Tensor& target, const torch::Tensor& dist, const torch::Tensor& index, double threshold) {
	const torch::Tensor s = arg(source, "source", torch::kFloat64, {-1, 3}, "[N, 3]"), t = arg(target, "target", torch::kFloat64, {-1, 3}, "[M, 3]", &s),
	                    d = arg(dist, "dist", torch::kFloat64, {s.size(0)}, "[N]", &s), ix = arg(index, "index", torch::kInt64, {s.size(0)}, "[N]", &s);
	const c10::cuda::CUDAGuard guard(s.device());
	torch::Tensor scratch = bytes(s), mom = torch::empty({19}, torch::TensorOptions().dtype(torch::kFloat64));
	check(rgs_tnt_icp_moments(s.size(0), s.data_ptr<double>(), t.size(0), t.data_ptr<double>(), d.data_ptr<double>(), ix.data_ptr<int64_t>(), threshold,
	                          mom.data_ptr<double>(), resize_cb, &scratch, at::cuda::getCurrentCUDAStream().stream()));
	return mom.narrow(0, 0, 18);
}

// ---- tetrahedra mesh extraction (rgs_tetra_*; Python side rade_gs_b200.tetra) ----------------------------------------------

// xyz, scaling f32 [P,3], rotation f32 [P,4] -> (points f32 [9P,3], scales f32 [9P,1])
std::tuple<torch::Tensor, torch::Tensor> TetraPoints(const torch::Tensor& xyz, const torch::Tensor& scaling, const torch::Tensor& rotation) {
	const torch::Tensor x = arg(xyz, "xyz", torch::kFloat32, {-1, 3}, "[P, 3]"), s = arg(scaling, "scaling", torch::kFloat32, {x.size(0), 3}, "[P, 3]", &x),
	                    r = arg(rotation, "rotation", torch::kFloat32, {x.size(0), 4}, "[P, 4]", &x);
	const c10::cuda::CUDAGuard guard(x.device());
	const int64_t P = x.size(0);
	torch::Tensor pts = new_empty({9 * P, 3}, x.options()), scl = new_empty({9 * P, 1}, x.options());
	check(rgs_tetra_points(P, x.data_ptr<float>(), s.data_ptr<float>(), r.data_ptr<float>(), pts.data_ptr<float>(), scl.data_ptr<float>(),
	                       at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(pts, scl);
}

// accumulates one view into final_alpha f32 [N] and weight int32 [N] (contiguous, in place)
void TetraCullAdd(const torch::Tensor& alpha, const torch::Tensor& coord, const torch::Tensor& render7, const torch::Tensor& gt_mask, torch::Tensor final_alpha,
                  torch::Tensor weight) {
	arg(final_alpha, "final_alpha", torch::kFloat32, {-1}, "[N]", nullptr, REJECT);
	const int64_t N = final_alpha.size(0);
	arg(weight, "weight", torch::kInt32, {N}, "[N]", &final_alpha, REJECT);
	const torch::Tensor a = arg(alpha.reshape({-1}), "alpha_integrated", torch::kFloat32, {N}, "[N]", &final_alpha),
	                    c = arg(coord, "point_coordinate", torch::kFloat32, {N, 2}, "[N, 2]", &final_alpha),
	                    r7 = arg(render7, "render7", torch::kFloat32, {-1, -1}, "[H, W]", &final_alpha);
	torch::Tensor gt;
	if (gt_mask.numel() > 0) gt = arg(gt_mask.reshape({-1}), "gt_mask", torch::kFloat32, {r7.numel()}, "the image's H x W values", &final_alpha);
	const c10::cuda::CUDAGuard guard(final_alpha.device());
	check(rgs_tetra_cull_add(N, a.data_ptr<float>(), c.data_ptr<float>(), (int32_t)r7.size(0), (int32_t)r7.size(1), r7.data_ptr<float>(),
	                         gt.defined() ? gt.data_ptr<float>() : nullptr, final_alpha.data_ptr<float>(), weight.data_ptr<int32_t>(),
	                         at::cuda::getCurrentCUDAStream().stream()));
}

torch::Tensor TetraCullFinish(const torch::Tensor& final_alpha, const torch::Tensor& weight) {
	const torch::Tensor f = arg(final_alpha, "final_alpha", torch::kFloat32, {-1}, "[N]"), w = arg(weight, "weight", torch::kInt32, {f.size(0)}, "[N]", &f);
	const c10::cuda::CUDAGuard guard(f.device());
	torch::Tensor sdf = new_empty({f.size(0)}, f.options());
	check(rgs_tetra_cull_finish(f.size(0), f.data_ptr<float>(), w.data_ptr<int32_t>(), sdf.data_ptr<float>(), at::cuda::getCurrentCUDAStream().stream()));
	return sdf;
}

// points f32 [N,3], sdf f32 [N], scales f32 [N] or [N,1], tets int64 [T,4]
//   -> (ends f32 [M,2,3], end_sdf f32 [M,2,1], end_scales f32 [M,2,1], faces int64 [F,3], interp_v int64 [M,2])
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor> TetraMarching(const torch::Tensor& points, const torch::Tensor& sdf,
                                                                                                   const torch::Tensor& scales, const torch::Tensor& tets) {
	const torch::Tensor p = arg(points, "vertices", torch::kFloat32, {-1, 3}, "[N, 3]"),
	                    d = arg(sdf.reshape({-1}), "sdf", torch::kFloat32, {p.size(0)}, "one value per vertex", &p),
	                    s = arg(scales.reshape({-1}), "scales", torch::kFloat32, {p.size(0)}, "one value per vertex", &p),
	                    t = arg(tets, "tets", torch::kInt64, {-1, 4}, "[T, 4]", &p);
	const c10::cuda::CUDAGuard guard(p.device());
	torch::Tensor interp = bytes(p), ends = bytes(p), esdf = bytes(p), escl = bytes(p), faces = bytes(p), scratch = bytes(p), sort = bytes(p);
	rgs_tetra_march_out out{&interp, &ends, &esdf, &escl, &faces, &scratch, &sort, 0, 0};
	check(rgs_tetra_marching(p.size(0), p.data_ptr<float>(), d.data_ptr<float>(), s.data_ptr<float>(), t.size(0), t.data_ptr<int64_t>(), resize_cb, &out,
	                         at::cuda::getCurrentCUDAStream().stream()));
	const int64_t M = out.num_vertices, F = out.num_faces;
	return std::make_tuple(rows(ends, torch::kFloat32, M, {2, 3}), rows(esdf, torch::kFloat32, M, {2, 1}), rows(escl, torch::kFloat32, M, {2, 1}),
	                       rows(faces, torch::kInt64, F, {3}), rows(interp, torch::kInt64, M, {2}));
}

// one bisection step in place: left, right f32 [M,3], left_sdf, right_sdf f32 [M] (or [M,1]), mid f32 [M,3]; mid_sdf f32 [M] or empty
void TetraBisect(const torch::Tensor& mid_sdf, torch::Tensor left, torch::Tensor right, torch::Tensor left_sdf, torch::Tensor right_sdf, torch::Tensor mid) {
	arg(left, "left", torch::kFloat32, {-1, 3}, "[M, 3]", nullptr, REJECT);
	const int64_t M = left.size(0);
	arg(right, "right", torch::kFloat32, {M, 3}, "[M, 3]", &left, REJECT);
	arg(mid, "mid", torch::kFloat32, {M, 3}, "[M, 3]", &left, REJECT);
	arg(left_sdf, "left_sdf", torch::kFloat32, {M}, "[M]", &left, REJECT);
	arg(right_sdf, "right_sdf", torch::kFloat32, {M}, "[M]", &left, REJECT);
	torch::Tensor m;
	if (mid_sdf.numel() > 0) m = arg(mid_sdf.reshape({-1}), "mid_sdf", torch::kFloat32, {M}, "one value per vertex", &left);
	const c10::cuda::CUDAGuard guard(left.device());
	check(rgs_tetra_bisect(M, m.defined() ? m.data_ptr<float>() : nullptr, left.data_ptr<float>(), right.data_ptr<float>(), left_sdf.data_ptr<float>(),
	                       right_sdf.data_ptr<float>(), mid.data_ptr<float>(), at::cuda::getCurrentCUDAStream().stream()));
}

// points f32 [M,3], ends f32 [M,2,3], end_scales f32 [M,2(,1)], faces int64 [F,3] -> (vertices f32 [V',3], faces int64 [F',3])
std::tuple<torch::Tensor, torch::Tensor> TetraFilter(const torch::Tensor& points, const torch::Tensor& ends, const torch::Tensor& end_scales,
                                                     const torch::Tensor& faces) {
	const torch::Tensor p = arg(points, "points", torch::kFloat32, {-1, 3}, "[M, 3]"),
	                    e = arg(ends, "ends", torch::kFloat32, {p.size(0), 2, 3}, "[M, 2, 3]", &p),
	                    s = arg(end_scales.reshape({-1}), "end_scales", torch::kFloat32, {2 * p.size(0)}, "[M, 2]", &p),
	                    f = arg(faces, "faces", torch::kInt64, {-1, 3}, "[F, 3]", &p);
	const c10::cuda::CUDAGuard guard(p.device());
	torch::Tensor verts = bytes(p), fout = bytes(p), scratch = bytes(p);
	rgs_tetra_filter_out out{&verts, &fout, &scratch, 0, 0};
	check(rgs_tetra_filter(p.size(0), p.data_ptr<float>(), e.data_ptr<float>(), s.data_ptr<float>(), f.size(0), f.data_ptr<int64_t>(), resize_cb, &out,
	                       at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(rows(verts, torch::kFloat32, out.num_vertices, {3}), rows(fout, torch::kInt64, out.num_faces, {3}));
}

// points f32 [N,3] -> (cells int32 [T,4], statistics {rounds, max_cavity, overflowed, alone, mesh_growths})
std::tuple<torch::Tensor, py::dict> DelaunayTriangulate(const torch::Tensor& points) {
	const torch::Tensor p = arg(points, "points", torch::kFloat32, {-1, 3}, "[N, 3]");
	const c10::cuda::CUDAGuard guard(p.device());
	torch::Tensor cells = bytes(p), pts = bytes(p), mesh0 = bytes(p), mesh1 = bytes(p), slab = bytes(p), sort = bytes(p);
	rgs_delaunay_out out{&cells, &pts, {&mesh0, &mesh1}, &slab, &sort, 0, 0, 0, 0, 0, 0};
	check(rgs_delaunay(p.size(0), p.data_ptr<float>(), resize_cb, &out, at::cuda::getCurrentCUDAStream().stream()));
	py::dict st;
	st["rounds"] = out.rounds;
	st["max_cavity"] = out.max_cavity;
	st["overflowed"] = out.overflowed;
	st["alone"] = out.alone;
	st["mesh_growths"] = out.mesh_growths;
	return std::make_tuple(rows(cells, torch::kInt32, out.num_cells, {4}), st);
}

// points f32 [N,3], tuples int32 [M,5] -> int8 [M,3] (orient3d, insphere, perturbed insphere)
torch::Tensor DelaunayPredicates(const torch::Tensor& points, const torch::Tensor& tuples) {
	const torch::Tensor p = arg(points, "points", torch::kFloat32, {-1, 3}, "[N, 3]"), t = arg(tuples, "tuples", torch::kInt32, {-1, 5}, "[M, 5]", &p);
	const c10::cuda::CUDAGuard guard(p.device());
	torch::Tensor signs = new_empty({t.size(0), 3}, p.options().dtype(torch::kInt8)), scratch = bytes(p);
	check(rgs_delaunay_predicates(p.size(0), p.data_ptr<float>(), t.size(0), t.data_ptr<int32_t>(), signs.data_ptr<int8_t>(), resize_cb, &scratch,
	                              at::cuda::getCurrentCUDAStream().stream()));
	return signs;
}

// ---- LPIPS-VGG stages (rgs_lpips_*; Python side rade_gs_b200.metrics) ------------------------------------------------------
// Each stage writes its [2, H, W, C] activations into `buffer` (a byte tensor grown through resize_cb, a fresh one when
// None): rade_gs_b200.metrics alternates two of them, so only two activation maps of the trunk are alive at a time.

torch::Tensor activation_out(const c10::optional<torch::Tensor>& buffer, const torch::Tensor& like, const torch::Tensor& input, int64_t H, int64_t W,
                             int64_t C) {
	torch::Tensor b = buffer.has_value() ? *buffer : bytes(like);
	TORCH_CHECK(b.scalar_type() == torch::kUInt8 && b.dim() == 1 && b.is_contiguous(), "buffer must be a contiguous 1-D uint8 tensor");
	TORCH_CHECK(b.device() == like.device(), "buffer must be on the same device as the other inputs");
	TORCH_CHECK(!b.is_alias_of(input), "buffer must not hold the input");
	resize_cb(&b, (size_t)(2 * H * W * C) * sizeof(float));
	return rows(b, torch::kFloat32, 2, {H, W, C});
}

// x, y f32 [3,H,W], weight f32 [64,3,3,3], bias f32 [64] -> f32 [2,H,W,64]
torch::Tensor LpipsInputConv(const torch::Tensor& x, const torch::Tensor& y, const torch::Tensor& weight, const torch::Tensor& bias,
                             const c10::optional<torch::Tensor>& buffer) {
	const torch::Tensor a = arg(x, "x", torch::kFloat32, {3, -1, -1}, "[3, H, W]"), b = arg(y, "y", torch::kFloat32, {3, a.size(1), a.size(2)}, "[3, H, W] like x", &a),
	                    w = arg(weight, "weight", torch::kFloat32, {64, 3, 3, 3}, "[64, 3, 3, 3]", &a), bs = arg(bias, "bias", torch::kFloat32, {64}, "[64]", &a);
	const c10::cuda::CUDAGuard guard(a.device());
	torch::Tensor out = activation_out(buffer, a, a, a.size(1), a.size(2), 64);
	check(rgs_lpips_input_conv(a.size(1), a.size(2), a.data_ptr<float>(), b.data_ptr<float>(), w.data_ptr<float>(), bs.data_ptr<float>(), out.data_ptr<float>(),
	                           at::cuda::getCurrentCUDAStream().stream()));
	return out;
}

// input f32 [2,H,W,C_in], weight f32 [C_out,3,3,C_in] (TF32 values), bias f32 [C_out] -> f32 [2,H,W,C_out]
torch::Tensor LpipsConv3x3(const torch::Tensor& input, const torch::Tensor& weight, const torch::Tensor& bias, const c10::optional<torch::Tensor>& buffer) {
	const torch::Tensor in = arg(input, "input", torch::kFloat32, {2, -1, -1, -1}, "[2, H, W, C_in]"),
	                    w = arg(weight, "weight", torch::kFloat32, {-1, 3, 3, in.size(3)}, "[C_out, 3, 3, C_in]", &in),
	                    bs = arg(bias, "bias", torch::kFloat32, {w.size(0)}, "[C_out]", &in);
	const c10::cuda::CUDAGuard guard(in.device());
	torch::Tensor out = activation_out(buffer, in, input, in.size(1), in.size(2), w.size(0));
	check(rgs_lpips_conv3x3(in.size(1), in.size(2), in.size(3), w.size(0), in.data_ptr<float>(), w.data_ptr<float>(), bs.data_ptr<float>(), out.data_ptr<float>(),
	                        at::cuda::getCurrentCUDAStream().stream()));
	return out;
}

// input f32 [2,H,W,C] -> f32 [2,H/2,W/2,C]
torch::Tensor LpipsMaxpool(const torch::Tensor& input, const c10::optional<torch::Tensor>& buffer) {
	const torch::Tensor in = arg(input, "input", torch::kFloat32, {2, -1, -1, -1}, "[2, H, W, C]");
	const c10::cuda::CUDAGuard guard(in.device());
	torch::Tensor out = activation_out(buffer, in, input, in.size(1) / 2, in.size(2) / 2, in.size(3));
	check(rgs_lpips_maxpool(in.size(1), in.size(2), in.size(3), in.data_ptr<float>(), out.data_ptr<float>(), at::cuda::getCurrentCUDAStream().stream()));
	return out;
}

// feats f32 [2,H,W,C], lin f32 [C] -> (map f32 [H,W], mean f64 [1])
std::tuple<torch::Tensor, torch::Tensor> LpipsDistance(const torch::Tensor& feats, const torch::Tensor& lin) {
	const torch::Tensor f = arg(feats, "feats", torch::kFloat32, {2, -1, -1, -1}, "[2, H, W, C]"),
	                    l = arg(lin.reshape({-1}), "lin", torch::kFloat32, {f.size(3)}, "C values", &f);
	const c10::cuda::CUDAGuard guard(f.device());
	torch::Tensor map = new_empty({f.size(1), f.size(2)}, f.options()), mean = new_empty({1}, f.options().dtype(torch::kFloat64)), scratch = bytes(f);
	check(rgs_lpips_distance(f.size(1), f.size(2), f.size(3), f.data_ptr<float>(), l.data_ptr<float>(), map.data_ptr<float>(), mean.data_ptr<double>(), resize_cb,
	                         &scratch, at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(map, mean);
}

// ---- unbounded mesh stages (rgs_unbounded_*; Python side rade_gs_b200.unbounded) -------------------------------------------

std::array<float, 3> vec3f(const std::vector<double>& v, const char* name) {
	TORCH_CHECK(v.size() == 3, name, " must have 3 values");
	return {(float)v[0], (float)v[1], (float)v[2]};  // round to nearest, as np.float32
}

// points f32 [N,3] -> (out f32 [N,3], norms f32 [N])
std::tuple<torch::Tensor, torch::Tensor> UnboundedContract(const torch::Tensor& points, const std::vector<double>& center, double radius, bool inverse,
                                                           double max_range) {
	const torch::Tensor p = arg(points, "points", torch::kFloat32, {-1, 3}, "[N, 3]");
	const c10::cuda::CUDAGuard guard(p.device());
	const std::array<float, 3> c = vec3f(center, "center");
	torch::Tensor out = new_empty({p.size(0), 3}, p.options()), norms = new_empty({p.size(0)}, p.options());
	check(rgs_unbounded_contract(p.size(0), p.data_ptr<float>(), c.data(), (float)radius, inverse, (float)max_range, out.data_ptr<float>(), norms.data_ptr<float>(),
	                             at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(out, norms);
}

// xs, ys, zs f32 [n], full_proj f32 [V,4,4], depth f32 [V,H,W] -> sdf f32 [n,n,n]
torch::Tensor UnboundedSdf(const torch::Tensor& xs, const torch::Tensor& ys, const torch::Tensor& zs, const torch::Tensor& full_proj, const torch::Tensor& depth,
                           const std::vector<double>& center, double radius, double trunc) {
	const torch::Tensor x = arg(xs, "xs", torch::kFloat32, {-1}, "[n]"), y = arg(ys, "ys", torch::kFloat32, {x.size(0)}, "[n] like xs", &x),
	                    z = arg(zs, "zs", torch::kFloat32, {x.size(0)}, "[n] like xs", &x),
	                    pr = arg(full_proj, "full_proj", torch::kFloat32, {-1, 4, 4}, "[V, 4, 4]", &x),
	                    d = arg(depth, "depth", torch::kFloat32, {pr.size(0), -1, -1}, "[V, H, W] with V like full_proj", &x);
	const c10::cuda::CUDAGuard guard(x.device());
	const std::array<float, 3> c = vec3f(center, "center");
	const int64_t n = x.size(0);
	TORCH_CHECK(n >= 1 && n <= RGS_UNBOUNDED_MAX_CROP, "crop size must be in [1, ", RGS_UNBOUNDED_MAX_CROP, "], got ", n);
	torch::Tensor sdf = new_empty({n, n, n}, x.options());
	check(rgs_unbounded_sdf((int32_t)n, x.data_ptr<float>(), y.data_ptr<float>(), z.data_ptr<float>(), (int32_t)pr.size(0), (int32_t)d.size(1), (int32_t)d.size(2),
	                        pr.data_ptr<float>(), d.data_ptr<float>(), c.data(), (float)radius, (float)trunc, sdf.data_ptr<float>(),
	                        at::cuda::getCurrentCUDAStream().stream()));
	return sdf;
}

// points f32 [N,3], full_proj f32 [V,4,4], depth f32 [V,H,W], rgb f32 [V,3,H,W] -> colors f32 [N,3]
torch::Tensor UnboundedColors(const torch::Tensor& points, const torch::Tensor& full_proj, const torch::Tensor& depth, const torch::Tensor& rgb, double trunc) {
	const torch::Tensor p = arg(points, "points", torch::kFloat32, {-1, 3}, "[N, 3]"),
	                    pr = arg(full_proj, "full_proj", torch::kFloat32, {-1, 4, 4}, "[V, 4, 4]", &p),
	                    d = arg(depth, "depth", torch::kFloat32, {pr.size(0), -1, -1}, "[V, H, W] with V like full_proj", &p),
	                    c = arg(rgb, "rgb", torch::kFloat32, {pr.size(0), 3, d.size(1), d.size(2)}, "[V, 3, H, W] like depth", &p);
	const c10::cuda::CUDAGuard guard(p.device());
	torch::Tensor out = new_empty({p.size(0), 3}, p.options());
	check(rgs_unbounded_colors(p.size(0), p.data_ptr<float>(), (int32_t)pr.size(0), (int32_t)d.size(1), (int32_t)d.size(2), pr.data_ptr<float>(), d.data_ptr<float>(),
	                           c.data_ptr<float>(), (float)trunc, out.data_ptr<float>(), at::cuda::getCurrentCUDAStream().stream()));
	return out;
}

// sdf f32 [n,n,n], lo / spacing 3 doubles -> (vertices f64 [V,3], triangles int32 [F,3])
std::tuple<torch::Tensor, torch::Tensor> UnboundedMcubes(const torch::Tensor& sdf, const std::vector<double>& lo, const std::vector<double>& spacing) {
	const torch::Tensor f = arg(sdf, "sdf", torch::kFloat32, {-1, -1, -1}, "[n, n, n]");
	TORCH_CHECK(f.size(1) == f.size(0) && f.size(2) == f.size(0), "sdf must be [n, n, n], got ", f.sizes());
	TORCH_CHECK(lo.size() == 3 && spacing.size() == 3, "lo and spacing must have 3 values");
	TORCH_CHECK(f.size(0) >= 2 && f.size(0) <= RGS_UNBOUNDED_MAX_CROP, "crop size must be in [2, ", RGS_UNBOUNDED_MAX_CROP, "], got ", f.size(0));
	const c10::cuda::CUDAGuard guard(f.device());
	torch::Tensor verts = bytes(f), tris = bytes(f), scratch = bytes(f);
	rgs_unbounded_mesh_out out{&verts, &tris, 0, 0};
	check(rgs_unbounded_mcubes((int32_t)f.size(0), f.data_ptr<float>(), lo.data(), spacing.data(), resize_cb, &out, &scratch, at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(rows(verts, torch::kFloat64, out.num_vertices, {3}), rows(tris, torch::kInt32, out.num_triangles, {3}));
}

// vertices f64 [V,3], triangles int32 [F,3] -> (vertices f32 [U,3], triangles int32 [F,3])
std::tuple<torch::Tensor, torch::Tensor> UnboundedMerge(const torch::Tensor& vertices, const torch::Tensor& triangles) {
	const torch::Tensor v = arg(vertices, "vertices", torch::kFloat64, {-1, 3}, "[V, 3]"), t = arg(triangles, "triangles", torch::kInt32, {-1, 3}, "[F, 3]", &v);
	const c10::cuda::CUDAGuard guard(v.device());
	torch::Tensor merged = bytes(v), scratch = bytes(v), tout = new_empty({t.size(0), 3}, t.options());
	int64_t U = 0;
	check(rgs_unbounded_merge(v.size(0), v.data_ptr<double>(), t.size(0), t.data_ptr<int32_t>(), tout.data_ptr<int32_t>(), resize_cb, &merged, &U, &scratch,
	                          at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(rows(merged, torch::kFloat32, U, {3}), tout);
}

// triangles int32 [F,3] over num_vertices vertices -> (kept vertex indices int32 [V'], triangles int32 [F',3],
// {num_clusters, threshold})
std::tuple<torch::Tensor, torch::Tensor, py::dict> UnboundedClusters(int64_t num_vertices, const torch::Tensor& triangles, int64_t cluster_to_keep) {
	const torch::Tensor t = arg(triangles, "triangles", torch::kInt32, {-1, 3}, "[F, 3]");
	const c10::cuda::CUDAGuard guard(t.device());
	torch::Tensor vidx = bytes(t), tout = bytes(t), scratch = bytes(t);
	rgs_unbounded_clusters_out out{&vidx, &tout, 0, 0, 0, 0};
	check(rgs_unbounded_clusters(num_vertices, t.size(0), t.data_ptr<int32_t>(), cluster_to_keep, resize_cb, &out, &scratch, at::cuda::getCurrentCUDAStream().stream()));
	py::dict st;
	st["num_clusters"] = out.num_clusters;
	st["threshold"] = out.threshold;
	return std::make_tuple(rows(vidx, torch::kInt32, out.num_vertices, {}), rows(tout, torch::kInt32, out.num_triangles, {3}), st);
}

// ---- Tanks and Temples mesh cull (rgs_tnt_mesh_depth / rgs_tnt_visibility_count; Python side rade_gs_b200.tnt_cull) --------

std::array<float, 12> w2c_rows(const std::vector<double>& w2c) {
	TORCH_CHECK(w2c.size() == 12, "w2c must hold rows 0..2 of the 4x4 (12 values), got ", w2c.size());
	std::array<float, 12> m;
	for (int k = 0; k < 12; k++) m[k] = (float)w2c[k];
	return m;
}

// vertices f32 [V,3], faces int32 [F,3] -> depth f32 [H,W]
torch::Tensor TntMeshDepth(const torch::Tensor& vertices, const torch::Tensor& faces, const std::vector<double>& w2c, double fx, double fy, double cx,
                           double cy, int64_t H, int64_t W, double znear, double zfar) {
	const torch::Tensor v = arg(vertices, "vertices", torch::kFloat32, {-1, 3}, "[V, 3]"), f = arg(faces, "faces", torch::kInt32, {-1, 3}, "[F, 3]", &v);
	const c10::cuda::CUDAGuard guard(v.device());
	const std::array<float, 12> m = w2c_rows(w2c);
	TORCH_CHECK(H > 0 && W > 0 && H <= 32768 && W <= 32768, "H and W must lie in [1, 32768], got ", H, " x ", W);
	torch::Tensor depth = new_empty({H, W}, v.options()), scratch = bytes(v);
	check(rgs_tnt_mesh_depth(v.size(0), v.data_ptr<float>(), f.size(0), f.data_ptr<int32_t>(), m.data(), (float)fx, (float)fy, (float)cx, (float)cy, (int32_t)H,
	                         (int32_t)W, (float)znear, (float)zfar, depth.data_ptr<float>(), resize_cb, &scratch, at::cuda::getCurrentCUDAStream().stream()));
	return depth;
}

// points f32 [N,3], depth f32 [H,W], counts int32 [N] (added to in place)
void TntVisibilityCount(const torch::Tensor& points, const torch::Tensor& depth, const std::vector<double>& w2c, double fx, double fy, double cx, double cy,
                        double eps, const torch::Tensor& counts) {
	const torch::Tensor p = arg(points, "points", torch::kFloat32, {-1, 3}, "[N, 3]"), d = arg(depth, "depth", torch::kFloat32, {-1, -1}, "[H, W]", &p),
	                    c = arg(counts, "counts", torch::kInt32, {p.size(0)}, "[N] like points", &p, REJECT);
	const c10::cuda::CUDAGuard guard(p.device());
	const std::array<float, 12> m = w2c_rows(w2c);
	check(rgs_tnt_visibility_count(p.size(0), p.data_ptr<float>(), d.data_ptr<float>(), m.data(), (float)fx, (float)fy, (float)cx, (float)cy, (int32_t)d.size(0),
	                               (int32_t)d.size(1), (float)eps, c.data_ptr<int32_t>(), at::cuda::getCurrentCUDAStream().stream()));
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
	m.def("rasterize_gaussians", &RasterizeGaussiansCUDA);
	m.def("integrate_gaussians_to_points", &IntegrateGaussiansToPointsCUDA);
	m.def("rasterize_gaussians_backward", &RasterizeGaussiansBackwardCUDA);
	m.def("mark_visible", &markVisible);
	// extras (not in the reference)
	m.def("rasterize_gaussians_slab",
	      [](const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors, const torch::Tensor& opacity,
	         const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier, const torch::Tensor& cov3D_precomp,
	         const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy, const float kernel_size,
	         const int image_height, const int image_width, const torch::Tensor& sh, const int degree, const torch::Tensor& campos,
	         const bool prefiltered, const bool require_coord, const bool require_depth, const bool debug, const int tile_row_begin,
	         const int tile_row_end, const bool compact) {
		      return forward_impl(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix,
		                          tan_fovx, tan_fovy, kernel_size, image_height, image_width, sh, degree, campos, prefiltered, require_coord,
		                          require_depth, debug, tile_row_begin, tile_row_end, torch::Tensor(), compact);
	      },
	      py::arg("background"), py::arg("means3D"), py::arg("colors"), py::arg("opacity"), py::arg("scales"), py::arg("rotations"), py::arg("scale_modifier"), py::arg("cov3D_precomp"), py::arg("viewmatrix"), py::arg("projmatrix"), py::arg("tan_fovx"), py::arg("tan_fovy"), py::arg("kernel_size"), py::arg("image_height"), py::arg("image_width"), py::arg("sh"), py::arg("degree"), py::arg("campos"), py::arg("prefiltered"), py::arg("require_coord"), py::arg("require_depth"), py::arg("debug"), py::arg("tile_row_begin"), py::arg("tile_row_end"), py::arg("compact") = false);
	// stage 1 with and without the exchange: by name, so that callers can pass the slab tail by keyword
#define BACKWARD_RENDER_ARGS py::arg("background"), py::arg("means3D"), py::arg("radii"), py::arg("colors"), py::arg("scales"), py::arg("rotations"), py::arg("scale_modifier"), py::arg("cov3D_precomp"), py::arg("viewmatrix"), py::arg("projmatrix"), py::arg("tan_fovx"), py::arg("tan_fovy"), py::arg("kernel_size"), py::arg("dL_dout_color"), py::arg("dL_dout_coord"), py::arg("dL_dout_mcoord"), py::arg("dL_dout_depth"), py::arg("dL_dout_mdepth"), py::arg("dL_dout_alpha"), py::arg("dL_dout_normal"), py::arg("normalmap"), py::arg("sh"), py::arg("degree"), py::arg("campos"), py::arg("geomBuffer"), py::arg("R"), py::arg("binningBuffer"), py::arg("imageBuffer"), py::arg("alphas"), py::arg("require_coord"), py::arg("require_depth"), py::arg("debug"), py::arg("tile_row_begin"), py::arg("tile_row_end"), py::arg("compact") = false, py::arg("image_height") = -1
	m.def("rasterize_gaussians_backward_render", without_exchange(&backward_render_impl), BACKWARD_RENDER_ARGS);
	m.def("rasterize_gaussians_backward_preprocess", &BackwardPreprocessCUDA);
	m.def("exchange_create", &ExchangeCreate);
	m.def("exchange_connect", &ExchangeConnect);
	m.def("exchange_destroy", &ExchangeDestroy);
	m.def("exchange_accumulator", &ExchangeAccumulator);
	m.def("exchange_result", &ExchangeResult);
	m.def("exchange_rows", &ExchangeRows);
	m.def("exchange_status", &ExchangeStatus);
	m.def("rasterize_gaussians_backward_render_exchange", with_exchange(&backward_render_impl), py::arg("ex"), BACKWARD_RENDER_ARGS);
#undef BACKWARD_RENDER_ARGS
	// split SH layout (opt-in, SURVEY.md 8f row 1): features_dc / features_rest stay two tensors, no torch.cat per iteration
	m.def("rasterize_gaussians_split_sh",
	      [](const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors, const torch::Tensor& opacity,
	         const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier, const torch::Tensor& cov3D_precomp,
	         const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy, const float kernel_size,
	         const int image_height, const int image_width, const torch::Tensor& sh_dc, const torch::Tensor& sh_rest, const int degree,
	         const torch::Tensor& campos, const bool prefiltered, const bool require_coord, const bool require_depth, const bool debug) {
		      return forward_impl(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix,
		                          tan_fovx, tan_fovy, kernel_size, image_height, image_width, sh_dc, degree, campos, prefiltered, require_coord,
		                          require_depth, debug, 0, -1, sh_rest);
	      });
	// returns (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh_dc, dL_dsh_rest, dL_dscales, dL_drotations)
	m.def("rasterize_gaussians_backward_split_sh",
	      [](const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& radii, const torch::Tensor& colors,
	         const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier, const torch::Tensor& cov3D_precomp,
	         const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy, const float kernel_size,
	         const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_coord, const torch::Tensor& dL_dout_mcoord,
	         const torch::Tensor& dL_dout_depth, const torch::Tensor& dL_dout_mdepth, const torch::Tensor& dL_dout_alpha,
	         const torch::Tensor& dL_dout_normal, const torch::Tensor& normalmap, const torch::Tensor& sh_dc, const torch::Tensor& sh_rest,
	         const int degree, const torch::Tensor& campos, const torch::Tensor& geomBuffer, const int R, const torch::Tensor& binningBuffer,
	         const torch::Tensor& imageBuffer, const torch::Tensor& alphas, const bool require_coord, const bool require_depth, const bool debug) {
		      const GradTensors g = backward_impl(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix,
		                                          projmatrix, tan_fovx, tan_fovy, kernel_size, dL_dout_color, dL_dout_coord, dL_dout_mcoord,
		                                          dL_dout_depth, dL_dout_mdepth, dL_dout_alpha, dL_dout_normal, normalmap, sh_dc, degree, campos,
		                                          geomBuffer, R, binningBuffer, imageBuffer, alphas, require_coord, require_depth, debug, sh_rest);
		      return std::make_tuple(g.means2D, g.colors, g.opacity, g.means3D, g.cov3D, g.sh, g.sh_rest, g.scales, g.rotations);
	      });
	m.def("compute_3d_filter", &Compute3DFilter);
	m.def("ssim_l1_forward", &SsimL1Forward, py::arg("img"), py::arg("gt"), py::arg("need_grad"), py::arg("row_lo") = 0, py::arg("row_hi") = -1);
	m.def("ssim_l1_backward", &SsimL1Backward, py::arg("img"), py::arg("gt"), py::arg("dmaps"), py::arg("w_ssim"), py::arg("w_l1"), py::arg("upstream"),
	      py::arg("row_lo") = 0, py::arg("row_hi") = -1);
	m.def("normal_consistency", &NormalConsistency);
	m.def("appearance_downsample", &AppearanceDownsample, py::arg("image"));
	m.def("appearance_downsample_backward", &AppearanceDownsampleBackward, py::arg("d_down"), py::arg("d_image"));
	m.def("appearance_l1_forward", &AppearanceL1Forward, py::arg("image"), py::arg("gt"), py::arg("up4"), py::arg("w2"), py::arg("b2"), py::arg("w3"),
	      py::arg("b3"), py::arg("need_act"), py::arg("want_transformed"));
	m.def("appearance_l1_backward", &AppearanceL1Backward, py::arg("image"), py::arg("gt"), py::arg("up4"), py::arg("act"), py::arg("w2"), py::arg("b2"),
	      py::arg("w3"), py::arg("b3"), py::arg("upstream"));
	m.def("activate_forward", &ActivateForward);
	m.def("activate_backward", &ActivateBackward);
	m.def("densification_stats", &DensificationStats);
	// densify-and-prune: one private submodule, called by rade_gs_b200.densify (the stages are not a public API of their own)
	py::module_ d = m.def_submodule("_densify", "densify-and-prune stages behind rade_gs_b200.densify");
	d.def("select", &DensifySelect, py::arg("grad_accum"), py::arg("grad_accum_abs"), py::arg("denom"), py::arg("scaling"), py::arg("opacity"),
	      py::arg("max_grad"), py::arg("dense"), py::arg("min_opacity"), py::arg("prune_large"), py::arg("max_screen_size"), py::arg("world"));
	d.def("plan", &DensifyPlan, py::arg("flags"), py::arg("block_offsets"), py::arg("counts"), py::arg("scaling"));
	d.def("gather", &DensifyGather, py::arg("src"), py::arg("draw"), py::arg("C"), py::arg("xyz"), py::arg("rotation"), py::arg("scaling"),
	      py::arg("sample_clone"), py::arg("sample_split"), py::arg("columns"));
	d.def("reset_opacity", &ResetOpacity, py::arg("scaling"), py::arg("opacity"), py::arg("filter_3D"));
	m.def("knn_mean_dist2", &KnnMeanDist2, py::arg("points"));
	m.def("tsdf_touch", &TsdfTouch);
	m.def("tsdf_integrate", &TsdfIntegrate);
	m.def("tsdf_rehash", &TsdfRehash);
	m.def("tsdf_active_blocks", &TsdfActiveBlocks);
	m.def("tsdf_extract", &TsdfExtract);
	m.def("tsdf_vertex_normals", &TsdfVertexNormals);
	// bounded TSDF (Open3D's legacy ScalableTSDFVolume): a private submodule behind rade_gs_b200.tsdf.ScalableTSDFVolume
	py::module_ sc = m.def_submodule("_scalable_tsdf", "bounded-TSDF stages behind rade_gs_b200.tsdf.ScalableTSDFVolume");
	sc.def("rgbd", &ScalableRgbd, py::arg("rgb"), py::arg("depth"), py::arg("depth_trunc"), py::arg("mask") = py::none());
	sc.def("image_u8", &ScalableImageU8, py::arg("image"), py::arg("scale") = 1.0, py::arg("offset") = 0.0);
	sc.def("touch", &ScalableTouch, py::arg("volume"), py::arg("depth"), py::arg("intrinsic"), py::arg("extrinsic"), py::arg("sdf_trunc"));
	sc.def("integrate", &ScalableIntegrate, py::arg("volume"), py::arg("unit_coords"), py::arg("depth"), py::arg("color"), py::arg("intrinsic"),
	       py::arg("extrinsic"), py::arg("sdf_trunc"), py::arg("call_id"));
	m.def("dtu_sample_mesh", &DtuSampleMesh, py::arg("vertices"), py::arg("faces"), py::arg("density"));
	m.def("dtu_radius_downsample", &DtuRadiusDownsample, py::arg("points"), py::arg("radius"));
	m.def("dtu_nearest", &DtuNearest, py::arg("reference"), py::arg("query"));
	m.def("dtu_dilate_masks", &DtuDilateMasks, py::arg("masks"));
	m.def("dtu_cull_vertices", &DtuCullVertices, py::arg("vertices"), py::arg("proj"), py::arg("dilated"));
	m.def("tnt_crop", &TntCrop, py::arg("points"), py::arg("transform"), py::arg("axis"), py::arg("axis_min"), py::arg("axis_max"), py::arg("polygon"));
	m.def("tnt_transform", &TntTransform, py::arg("points"), py::arg("transform"));
	m.def("tnt_voxel_downsample", &TntVoxelDownsample, py::arg("points"), py::arg("voxel"));
	m.def("tnt_icp_moments", &TntIcpMoments, py::arg("source"), py::arg("target"), py::arg("dist"), py::arg("index"), py::arg("threshold"));
	m.def("tetra_points", &TetraPoints, py::arg("xyz"), py::arg("scaling"), py::arg("rotation"));
	m.def("tetra_cull_add", &TetraCullAdd, py::arg("alpha"), py::arg("coord"), py::arg("render7"), py::arg("gt_mask"), py::arg("final_alpha"), py::arg("weight"));
	m.def("tetra_cull_finish", &TetraCullFinish, py::arg("final_alpha"), py::arg("weight"));
	m.def("tetra_marching", &TetraMarching, py::arg("vertices"), py::arg("sdf"), py::arg("scales"), py::arg("tets"));
	m.def("tetra_bisect", &TetraBisect, py::arg("mid_sdf"), py::arg("left"), py::arg("right"), py::arg("left_sdf"), py::arg("right_sdf"), py::arg("mid"));
	m.def("tetra_filter", &TetraFilter, py::arg("points"), py::arg("ends"), py::arg("end_scales"), py::arg("faces"));
	// exact Delaunay of the tetra points: a private submodule behind rade_gs_b200.tetra.delaunay
	py::module_ dt = m.def_submodule("_delaunay", "exact Delaunay tetrahedralization behind rade_gs_b200.tetra.delaunay");
	dt.def("triangulate", &DelaunayTriangulate, py::arg("points"));
	dt.def("predicates", &DelaunayPredicates, py::arg("points"), py::arg("tuples"));
	// LPIPS-VGG trunk and distance: a private submodule behind rade_gs_b200.metrics.lpips
	py::module_ lp = m.def_submodule("_lpips", "LPIPS-VGG stages behind rade_gs_b200.metrics.lpips");
	lp.def("input_conv", &LpipsInputConv, py::arg("x"), py::arg("y"), py::arg("weight"), py::arg("bias"), py::arg("buffer") = py::none());
	lp.def("conv3x3", &LpipsConv3x3, py::arg("input"), py::arg("weight"), py::arg("bias"), py::arg("buffer") = py::none());
	lp.def("maxpool", &LpipsMaxpool, py::arg("input"), py::arg("buffer") = py::none());
	lp.def("distance", &LpipsDistance, py::arg("feats"), py::arg("lin"));
	// contracted-space TSDF mesh of unbounded scenes: a private submodule behind rade_gs_b200.unbounded
	py::module_ ub = m.def_submodule("_unbounded", "unbounded-scene mesh stages behind rade_gs_b200.unbounded");
	ub.def("contract", &UnboundedContract, py::arg("points"), py::arg("center"), py::arg("radius"), py::arg("inverse"), py::arg("max_range"));
	ub.def("sdf", &UnboundedSdf, py::arg("xs"), py::arg("ys"), py::arg("zs"), py::arg("full_proj"), py::arg("depth"), py::arg("center"), py::arg("radius"),
	       py::arg("trunc"));
	ub.def("colors", &UnboundedColors, py::arg("points"), py::arg("full_proj"), py::arg("depth"), py::arg("rgb"), py::arg("trunc"));
	ub.def("mcubes", &UnboundedMcubes, py::arg("sdf"), py::arg("lo"), py::arg("spacing"));
	ub.def("merge", &UnboundedMerge, py::arg("vertices"), py::arg("triangles"));
	ub.def("clusters", &UnboundedClusters, py::arg("num_vertices"), py::arg("triangles"), py::arg("cluster_to_keep"));
	// Tanks and Temples mesh cull: a private submodule behind rade_gs_b200.tnt_cull
	py::module_ tc = m.def_submodule("_tnt_cull", "depth rasterizer and visibility count behind rade_gs_b200.tnt_cull");
	tc.def("mesh_depth", &TntMeshDepth, py::arg("vertices"), py::arg("faces"), py::arg("w2c"), py::arg("fx"), py::arg("fy"), py::arg("cx"), py::arg("cy"),
	       py::arg("H"), py::arg("W"), py::arg("znear"), py::arg("zfar"));
	tc.def("visibility_count", &TntVisibilityCount, py::arg("points"), py::arg("depth"), py::arg("w2c"), py::arg("fx"), py::arg("fy"), py::arg("cx"),
	       py::arg("cy"), py::arg("eps"), py::arg("counts"));
	// slab-local forms of the training losses: a private submodule behind rade_gs_b200.multigpu
	py::module_ sl = m.def_submodule("_slab", "row-sharded training-loss stages behind rade_gs_b200.multigpu");
	sl.def("normal_consistency_rows", &NormalConsistencyRows, py::arg("rendered_normal"), py::arg("map_expected"), py::arg("map_median"),
	       py::arg("from_depth"), py::arg("inv_fx"), py::arg("inv_fy"), py::arg("cx"), py::arg("cy"), py::arg("w_expected"), py::arg("w_median"), py::arg("H"),
	       py::arg("row_lo"), py::arg("row_hi"));
	sl.def("rasterize_balanced", &RasterizeBalanced, py::arg("background"), py::arg("means3D"), py::arg("colors"), py::arg("opacity"), py::arg("scales"),
	       py::arg("rotations"), py::arg("scale_modifier"), py::arg("cov3D_precomp"), py::arg("viewmatrix"), py::arg("projmatrix"), py::arg("tan_fovx"),
	       py::arg("tan_fovy"), py::arg("kernel_size"), py::arg("image_height"), py::arg("image_width"), py::arg("sh"), py::arg("degree"), py::arg("campos"),
	       py::arg("prefiltered"), py::arg("require_coord"), py::arg("require_depth"), py::arg("debug"), py::arg("world_size"), py::arg("rank"),
	       py::arg("compact") = false);
	sl.def("balance_partition", &BalancePartition, py::arg("row_instances"), py::arg("grid_x"), py::arg("world_size"));
	sl.attr("BALANCE_TILE_COST") = RGS_BALANCE_TILE_COST;
	sl.def("appearance_row_windows", &AppearanceRowWindows, py::arg("H0"), py::arg("W0"), py::arg("row_lo"), py::arg("row_hi"));
	sl.def("appearance_downsample_rows", &AppearanceDownsampleRows, py::arg("image"), py::arg("image_lo"), py::arg("H0"), py::arg("row_lo"),
	       py::arg("row_hi"));
	sl.def("appearance_downsample_backward_rows", &AppearanceDownsampleBackwardRows, py::arg("d_down"), py::arg("d_image"), py::arg("H0"), py::arg("row_lo"),
	       py::arg("row_hi"));
	sl.def("appearance_l1_forward_rows", &AppearanceL1ForwardRows, py::arg("image"), py::arg("gt"), py::arg("image_lo"), py::arg("H0"), py::arg("row_lo"),
	       py::arg("row_hi"), py::arg("up4"), py::arg("w2"), py::arg("b2"), py::arg("w3"), py::arg("b3"));
	sl.def("appearance_l1_backward_rows", &AppearanceL1BackwardRows, py::arg("image"), py::arg("gt"), py::arg("image_lo"), py::arg("H0"), py::arg("row_lo"),
	       py::arg("row_hi"), py::arg("up4"), py::arg("act"), py::arg("w2"), py::arg("b2"), py::arg("w3"), py::arg("b3"), py::arg("upstream"));
	// the forward without a host read, for CUDA-graph capture: a private submodule behind diff_gaussian_rasterization's reserve path
	py::module_ gr = m.def_submodule("_graph", "rasterizer forward binned into preset capacities behind rade_gs_b200.graphs");
	gr.def("rasterize_gaussians", &RasterizePreset, py::arg("background"), py::arg("means3D"), py::arg("colors"), py::arg("opacity"), py::arg("scales"),
	       py::arg("rotations"), py::arg("scale_modifier"), py::arg("cov3D_precomp"), py::arg("viewmatrix"), py::arg("projmatrix"), py::arg("tan_fovx"),
	       py::arg("tan_fovy"), py::arg("kernel_size"), py::arg("image_height"), py::arg("image_width"), py::arg("sh"), py::arg("degree"), py::arg("campos"),
	       py::arg("prefiltered"), py::arg("require_coord"), py::arg("require_depth"), py::arg("debug"), py::arg("sh_rest"), py::arg("instances"),
	       py::arg("longest_list"), py::arg("status"));
	// the decoupled-appearance network's head: a private submodule behind rade_gs_b200.appearance and multigpu
	py::module_ ah = m.def_submodule("_appearance_head", "conv1 and up1..up4 of the appearance network behind rade_gs_b200.appearance");
	ah.def("forward", &AppearanceHeadForward, py::arg("down"), py::arg("emb"), py::arg("params"));
	ah.def("backward", &AppearanceHeadBackward, py::arg("down"), py::arg("emb"), py::arg("params"), py::arg("act"), py::arg("up4"), py::arg("d_up4"));
	m.def("grad_stride",[](bool require_coord, bool require_depth) { return rgs_grad_stride(require_coord, require_depth); });
	m.def("set_poison", [](int byte) { g_poison = byte; });
	m.def("launch_count", []() { return rgs_launch_count(); });
	m.def("abi_version", []() { return rgs_abi_version(); });
	m.def("stage_timing", [](bool on) { rgs_stage_timing(on); });
	m.def("stage_times", []() {
		const char* names[16]; double ms[16]; int64_t n[16];
		const int k = rgs_stage_times(names, ms, n, 16);
		py::dict d;
		for (int i = 0; i < k; i++) d[names[i]] = py::make_tuple(ms[i], n[i]);
		return d;
	});
}

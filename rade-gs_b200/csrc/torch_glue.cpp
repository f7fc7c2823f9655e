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
#include <string>
#include <tuple>
#include <vector>

#include "rgs_b200.h"

namespace {

const float* opt_ptr(const torch::Tensor& t) { return t.numel() == 0 ? nullptr : t.data_ptr<float>(); }

torch::Tensor as_input(const torch::Tensor& t, const torch::Tensor& like, const char* name) {
	if (t.numel() == 0) return t;  // absent (torch.Tensor([]) on the CPU), stays absent
	TORCH_CHECK(t.scalar_type() == torch::kFloat32, name, " must be float32");
	TORCH_CHECK(t.device() == like.device(), name, " must be on the same device as means3D");
	return t.contiguous();
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

struct CamHolder {
	torch::Tensor bg, view, proj, campos;
	rgs_camera cam;
};

void fill_camera(CamHolder& h, const torch::Tensor& like, const torch::Tensor& background, const torch::Tensor& viewmatrix,
                 const torch::Tensor& projmatrix, const torch::Tensor& campos, float tan_fovx, float tan_fovy, float kernel_size,
                 float scale_modifier, int H, int W, int degree, int M, bool prefiltered, bool require_coord, bool require_depth, bool debug,
                 int row_begin, int row_end, bool compact = false) {
	h.bg = as_input(background, like, "background");
	h.view = as_input(viewmatrix, like, "viewmatrix");
	h.proj = as_input(projmatrix, like, "projmatrix");
	h.campos = as_input(campos, like, "campos");
	rgs_camera& c = h.cam;
	c.width = W;
	c.height = H;
	c.tan_fovx = tan_fovx;
	c.tan_fovy = tan_fovy;
	c.kernel_size = kernel_size;
	c.scale_modifier = scale_modifier;
	c.viewmatrix = h.view.data_ptr<float>();
	c.projmatrix = h.proj.data_ptr<float>();
	c.cam_pos = h.campos.data_ptr<float>();
	c.background = h.bg.data_ptr<float>();
	c.sh_degree = degree;
	c.sh_coeffs = M;
	c.require_coord = require_coord;
	c.require_depth = require_depth;
	c.prefiltered = prefiltered;
	c.debug = debug;
	c.tile_row_begin = row_begin;
	c.tile_row_end = row_end;
	c.compact_slab = compact ? 1 : 0;
}

struct GaussHolder {
	torch::Tensor means, opac, sh, sh_rest, colors, scales, rots, cov;
	rgs_gaussians g;
};

void fill_gaussians(GaussHolder& h, const torch::Tensor& means3D, const torch::Tensor& opacity, const torch::Tensor& sh, const torch::Tensor& colors,
                    const torch::Tensor& scales, const torch::Tensor& rotations, const torch::Tensor& cov3D_precomp,
                    const torch::Tensor& sh_rest = torch::Tensor()) {
	h.means = as_input(means3D, means3D, "means3D");
	h.opac = as_input(opacity, means3D, "opacity");
	h.sh = as_input(sh, means3D, "sh");
	h.colors = as_input(colors, means3D, "colors_precomp");
	h.scales = as_input(scales, means3D, "scales");
	h.rots = as_input(rotations, means3D, "rotations");
	h.cov = as_input(cov3D_precomp, means3D, "cov3D_precomp");
	h.g.P = (int)means3D.size(0);
	h.g.means3D = opt_ptr(h.means);
	h.g.opacities = opt_ptr(h.opac);
	h.g.shs = opt_ptr(h.sh);
	h.g.colors_precomp = opt_ptr(h.colors);
	h.g.scales = opt_ptr(h.scales);
	h.g.rotations = opt_ptr(h.rots);
	h.g.cov3D_precomp = opt_ptr(h.cov);
	h.g.shs_rest = nullptr;
	if (sh_rest.defined() && sh_rest.numel() != 0) {  // split layout: `sh` is [P,1,3], sh_rest [P,M-1,3]
		TORCH_CHECK(sh.dim() == 3 && sh.size(1) == 1 && sh_rest.dim() == 3 && sh_rest.size(0) == sh.size(0) && sh_rest.size(2) == 3,
		            "split SH layout needs shs_dc [P,1,3] and shs_rest [P,M-1,3]");
		h.sh_rest = as_input(sh_rest, means3D, "shs_rest");
		h.g.shs_rest = h.sh_rest.data_ptr<float>();
	}
}

// number of SH coefficients per Gaussian for either layout
int sh_coeffs(const torch::Tensor& sh, const torch::Tensor& sh_rest) {
	int M = 0;
	if (sh.size(0) != 0) M = sh.size(1);
	if (sh_rest.defined() && sh_rest.numel() != 0) M += sh_rest.size(1);
	return M;
}

using FwdResult = std::tuple<int, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor,
                             torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>;

FwdResult forward_impl(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors, const torch::Tensor& opacity,
                       const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier, const torch::Tensor& cov3D_precomp,
                       const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy,
                       const float kernel_size, const int image_height, const int image_width, const torch::Tensor& sh, const int degree,
                       const torch::Tensor& campos, const bool prefiltered, const bool require_coord, const bool require_depth, const bool debug,
                       int row_begin, int row_end, const torch::Tensor& sh_rest = torch::Tensor(), bool compact = false) {
	if (means3D.ndimension() != 2 || means3D.size(1) != 3) {
		AT_ERROR("means3D must have dimensions (num_points, 3)");
	}
	TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor: this rasterizer has no CPU path");
	const c10::cuda::CUDAGuard guard(means3D.device());
	const int P = means3D.size(0);
	const int H = image_height, W = image_width;
	auto int_opts = means3D.options().dtype(torch::kInt32);
	auto float_opts = means3D.options().dtype(torch::kFloat32);
	auto byte_opts = means3D.options().dtype(torch::kByte);
	const int grid_y = (H + 15) / 16;
	const bool whole = (row_begin == 0 && (row_end < 0 || row_end == grid_y));
	// compact: the maps hold the slab's pixel rows only ([ch, Hs, W]) and are fully written by the kernels
	const int r1 = row_end < 0 ? grid_y : row_end;
	const int Hm = compact ? std::max(0, std::min(r1 * 16, H) - row_begin * 16) : H;
	const bool fill = (P == 0) || (!whole && !compact);  // P == 0: the reference returns all-zero maps (rasterize_points.cu:90)
	auto img = [&](int ch) { return fill ? torch::zeros({ch, Hm, W}, float_opts) : new_empty({ch, Hm, W}, float_opts); };
	torch::Tensor out_color = img(3), out_depth = img(1), out_mdepth = img(1), out_coord = img(3), out_mcoord = img(3), out_alpha = img(1),
	              out_normal = img(3);
	torch::Tensor radii = P == 0 ? torch::zeros({P}, int_opts) : new_empty({P}, int_opts);
	torch::Tensor geomBuffer = torch::empty({0}, byte_opts), binningBuffer = torch::empty({0}, byte_opts), imgBuffer = torch::empty({0}, byte_opts);

	int rendered = 0;
	if (P != 0) {
		const int M = sh_coeffs(sh, sh_rest);
		CamHolder ch;
		fill_camera(ch, means3D, background, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, kernel_size, scale_modifier, H, W, degree, M,
		            prefiltered, require_coord, require_depth, debug, row_begin, row_end, compact);
		GaussHolder gh;
		fill_gaussians(gh, means3D, opacity, sh, colors, scales, rotations, cov3D_precomp, sh_rest);
		rgs_forward_out fo{out_color.data_ptr<float>(), out_coord.data_ptr<float>(), out_mcoord.data_ptr<float>(), out_alpha.data_ptr<float>(),
		                   out_normal.data_ptr<float>(), out_depth.data_ptr<float>(), out_mdepth.data_ptr<float>(), radii.data_ptr<int>()};
		rgs_buffers bufs{resize_cb, &geomBuffer, resize_cb, &binningBuffer, resize_cb, &imgBuffer};
		const int64_t rc = rgs_forward(&ch.cam, &gh.g, &fo, &bufs, at::cuda::getCurrentCUDAStream().stream());
		check(rc);
		rendered = (int)rc;
	}
	return std::make_tuple(rendered, out_color, out_coord, out_mcoord, out_alpha, out_normal, out_depth, out_mdepth, radii, geomBuffer,
	                       binningBuffer, imgBuffer);
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

struct BackwardCtx {
	CamHolder ch;
	GaussHolder gh;
	torch::Tensor g_color, g_coord, g_mcoord, g_depth, g_mdepth, g_alpha, g_normal, normalmap, alphas, radii, geom, binning, image;
	rgs_backward_in in;
};

void fill_backward(BackwardCtx& c, const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& radii,
                   const torch::Tensor& colors, const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier,
                   const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx,
                   const float tan_fovy, const float kernel_size, const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_coord,
                   const torch::Tensor& dL_dout_mcoord, const torch::Tensor& dL_dout_depth, const torch::Tensor& dL_dout_mdepth,
                   const torch::Tensor& dL_dout_alpha, const torch::Tensor& dL_dout_normal, const torch::Tensor& normalmap, const torch::Tensor& sh,
                   const int degree, const torch::Tensor& campos, const torch::Tensor& geomBuffer, const int R, const torch::Tensor& binningBuffer,
                   const torch::Tensor& imageBuffer, const torch::Tensor& alphas, const bool require_coord, const bool require_depth,
                   const bool debug, int row_begin, int row_end, const torch::Tensor& sh_rest = torch::Tensor(), bool compact = false,
                   int image_height = -1) {
	// the image height is read off the gradient map like the reference does (rasterize_points.cu:171-172), except for compact slab maps
	const int H = (compact && image_height > 0) ? image_height : dL_dout_color.size(1), W = dL_dout_color.size(2);
	TORCH_CHECK(!compact || image_height > 0, "compact slab maps need the full image height");
	const int M = sh_coeffs(sh, sh_rest);
	fill_camera(c.ch, means3D, background, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, kernel_size, scale_modifier, H, W, degree, M, false,
	            require_coord, require_depth, debug, row_begin, row_end, compact);
	torch::Tensor no_opacity = torch::empty({0});  // backward does not receive the opacities (rasterize_points.h:43-76)
	fill_gaussians(c.gh, means3D, no_opacity, sh, colors, scales, rotations, cov3D_precomp, sh_rest);
	c.g_color = as_input(dL_dout_color, means3D, "dL_dout_color");
	c.g_coord = as_input(dL_dout_coord, means3D, "dL_dout_coord");
	c.g_mcoord = as_input(dL_dout_mcoord, means3D, "dL_dout_mcoord");
	c.g_depth = as_input(dL_dout_depth, means3D, "dL_dout_depth");
	c.g_mdepth = as_input(dL_dout_mdepth, means3D, "dL_dout_mdepth");
	c.g_alpha = as_input(dL_dout_alpha, means3D, "dL_dout_alpha");
	c.g_normal = as_input(dL_dout_normal, means3D, "dL_dout_normal");
	c.normalmap = as_input(normalmap, means3D, "normalmap");
	c.alphas = as_input(alphas, means3D, "alphas");
	c.radii = radii.contiguous();
	c.geom = geomBuffer.contiguous();
	c.binning = binningBuffer.contiguous();
	c.image = imageBuffer.contiguous();
	c.in.dL_dout_color = c.g_color.data_ptr<float>();
	c.in.dL_dout_coord = c.g_coord.data_ptr<float>();
	c.in.dL_dout_mcoord = c.g_mcoord.data_ptr<float>();
	c.in.dL_dout_depth = c.g_depth.data_ptr<float>();
	c.in.dL_dout_mdepth = c.g_mdepth.data_ptr<float>();
	c.in.dL_dout_alpha = c.g_alpha.data_ptr<float>();
	c.in.dL_dout_normal = c.g_normal.data_ptr<float>();
	c.in.out_alpha = c.alphas.data_ptr<float>();
	c.in.out_normal = c.normalmap.data_ptr<float>();
	c.in.radii = c.radii.data_ptr<int>();
	c.in.geom_buffer = reinterpret_cast<const char*>(c.geom.data_ptr());
	c.in.binning_buffer = reinterpret_cast<const char*>(c.binning.data_ptr());
	c.in.image_buffer = reinterpret_cast<const char*>(c.image.data_ptr());
	c.in.num_rendered = R;
}

using BwdResult = std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>;

struct GradTensors {
	torch::Tensor means3D, means2D, colors, opacity, cov3D, sh, sh_rest, scales, rotations;
	rgs_backward_out out;
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
	TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor: this rasterizer has no CPU path");
	const c10::cuda::CUDAGuard guard(means3D.device());
	const int P = means3D.size(0);
	int M = 0;
	if (sh.size(0) != 0) M = sh.size(1);
	GradTensors gt;
	alloc_grads(gt, means3D, P, M);
	if (P != 0) {
		BackwardCtx c;
		fill_backward(c, background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx,
		              tan_fovy, kernel_size, dL_dout_color, dL_dout_coord, dL_dout_mcoord, dL_dout_depth, dL_dout_mdepth, dL_dout_alpha,
		              dL_dout_normal, normalmap, sh, degree, campos, geomBuffer, R, binningBuffer, imageBuffer, alphas, require_coord, require_depth,
		              debug, 0, -1);
		torch::Tensor scratch = torch::empty({0}, means3D.options().dtype(torch::kByte));
		check(rgs_backward(&c.ch.cam, &c.gh.g, &c.in, &gt.out, resize_cb, &scratch, at::cuda::getCurrentCUDAStream().stream()));
	}
	return std::make_tuple(gt.means2D, gt.colors, gt.opacity, gt.means3D, gt.cov3D, gt.sh, gt.scales, gt.rotations);
}

torch::Tensor markVisible(torch::Tensor& means3D, torch::Tensor& viewmatrix, torch::Tensor& projmatrix) {
	const int P = means3D.size(0);
	torch::Tensor present = torch::full({P}, false, means3D.options().dtype(at::kBool));
	if (P != 0) {
		TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor: this rasterizer has no CPU path");
		const c10::cuda::CUDAGuard guard(means3D.device());
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
	if (means3D.ndimension() != 2 || means3D.size(1) != 3) {
		AT_ERROR("means3D must have dimensions (num_points, 3)");
	}
	if (points3D.ndimension() != 2 || points3D.size(1) != 3) {
		AT_ERROR("points3D must have dimensions (num_points, 3)");
	}
	TORCH_CHECK(means3D.is_cuda() && points3D.is_cuda(), "means3D / points3D must be CUDA tensors: this rasterizer has no CPU path");
	const c10::cuda::CUDAGuard guard(means3D.device());
	const int PN = points3D.size(0), P = means3D.size(0), H = image_height, W = image_width;
	auto int_opts = means3D.options().dtype(torch::kInt32);
	auto float_opts = means3D.options().dtype(torch::kFloat32);
	auto byte_opts = means3D.options().dtype(torch::kByte);
	const bool run = P != 0 && PN != 0;  // rasterize_points.cu:341: otherwise the fill values below are returned
	torch::Tensor out_color = run ? new_empty({9, H, W}, float_opts) : torch::zeros({9, H, W}, float_opts);
	torch::Tensor radii = run ? new_empty({P}, int_opts) : torch::zeros({P}, int_opts);
	torch::Tensor out_alpha_integrated = run ? new_empty({PN}, float_opts) : torch::full({PN}, 1.0, float_opts);
	torch::Tensor out_color_integrated = run ? new_empty({PN, 3}, float_opts) : torch::zeros({PN, 3}, float_opts);
	torch::Tensor out_coordinate2d = run ? new_empty({PN, 2}, float_opts) : torch::zeros({PN, 2}, float_opts);
	torch::Tensor out_sdf = run ? new_empty({PN}, float_opts) : torch::full({PN}, -1000.0, float_opts);
	torch::Tensor geomBuffer = torch::empty({0}, byte_opts), binningBuffer = torch::empty({0}, byte_opts), imgBuffer = torch::empty({0}, byte_opts),
	              pointBuffer = torch::empty({0}, byte_opts);
	int rendered = 0;
	if (run) {
		int M = 0;
		if (sh.size(0) != 0) M = sh.size(1);
		CamHolder ch;
		fill_camera(ch, means3D, background, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, kernel_size, scale_modifier, H, W, degree, M,
		            prefiltered, false, true, debug, 0, -1);
		GaussHolder gh;
		fill_gaussians(gh, means3D, opacity, sh, colors, scales, rotations, cov3D_precomp);
		torch::Tensor pts = as_input(points3D, means3D, "points3D");
		rgs_integrate_io io{PN, pts.data_ptr<float>(), out_color.data_ptr<float>(), out_alpha_integrated.data_ptr<float>(),
		                    out_color_integrated.data_ptr<float>(), out_coordinate2d.data_ptr<float>(), out_sdf.data_ptr<float>(), radii.data_ptr<int>()};
		rgs_buffers bufs{resize_cb, &geomBuffer, resize_cb, &binningBuffer, resize_cb, &imgBuffer};
		int32_t overflowed = 0;
		const int64_t rc = rgs_integrate(&ch.cam, &gh.g, &io, &bufs, resize_cb, &pointBuffer, &overflowed,  // always read: 4 bytes on a call that synchronises anyway
		                                 at::cuda::getCurrentCUDAStream().stream());
		check(rc);
		rendered = (int)rc;
		if (overflowed > 0) printf("ERROR: Maximal contributors are met in %d pixels. This should be fixed!\n", overflowed);  // forward.cu:1128
	}
	return std::make_tuple(rendered, out_color, out_alpha_integrated, out_color_integrated, out_coordinate2d, out_sdf, radii, geomBuffer, binningBuffer,
	                       imgBuffer);
}

// ---- multi-GPU extras ---------------------------------------------------------------------------------------------

FwdResult RasterizeGaussiansSlabCUDA(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors,
                                     const torch::Tensor& opacity, const torch::Tensor& scales, const torch::Tensor& rotations,
                                     const float scale_modifier, const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix,
                                     const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy, const float kernel_size,
                                     const int image_height, const int image_width, const torch::Tensor& sh, const int degree,
                                     const torch::Tensor& campos, const bool prefiltered, const bool require_coord, const bool require_depth,
                                     const bool debug, const int tile_row_begin, const int tile_row_end, const bool compact) {
	return forward_impl(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx,
	                    tan_fovy, kernel_size, image_height, image_width, sh, degree, campos, prefiltered, require_coord, require_depth, debug,
	                    tile_row_begin, tile_row_end, torch::Tensor(), compact);
}

// stage 1: returns the packed screen-space gradient accumulator [P, rgs_grad_stride] (additive across slabs)
torch::Tensor BackwardRenderCUDA(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& radii,
                                 const torch::Tensor& colors, const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier,
                                 const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix,
                                 const float tan_fovx, const float tan_fovy, const float kernel_size, const torch::Tensor& dL_dout_color,
                                 const torch::Tensor& dL_dout_coord, const torch::Tensor& dL_dout_mcoord, const torch::Tensor& dL_dout_depth,
                                 const torch::Tensor& dL_dout_mdepth, const torch::Tensor& dL_dout_alpha, const torch::Tensor& dL_dout_normal,
                                 const torch::Tensor& normalmap, const torch::Tensor& sh, const int degree, const torch::Tensor& campos,
                                 const torch::Tensor& geomBuffer, const int R, const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer,
                                 const torch::Tensor& alphas, const bool require_coord, const bool require_depth, const bool debug,
                                 const int tile_row_begin, const int tile_row_end, const bool compact, const int image_height) {
	TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor: this rasterizer has no CPU path");
	const c10::cuda::CUDAGuard guard(means3D.device());
	const int P = means3D.size(0);
	const int GS = rgs_grad_stride(require_coord, require_depth);
	torch::Tensor acc = P == 0 ? torch::zeros({P, GS}, means3D.options()) : new_empty({P, GS}, means3D.options());
	if (P != 0) {
		BackwardCtx c;
		fill_backward(c, background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx,
		              tan_fovy, kernel_size, dL_dout_color, dL_dout_coord, dL_dout_mcoord, dL_dout_depth, dL_dout_mdepth, dL_dout_alpha,
		              dL_dout_normal, normalmap, sh, degree, campos, geomBuffer, R, binningBuffer, imageBuffer, alphas, require_coord, require_depth,
		              debug, tile_row_begin, tile_row_end, torch::Tensor(), compact, image_height);
		check(rgs_backward_render(&c.ch.cam, &c.gh.g, &c.in, acc.data_ptr<float>(), at::cuda::getCurrentCUDAStream().stream()));
	}
	return acc;
}

// ---- device-side exchange of the accumulator rows over peer memory (rgs_exchange_*) ----
// The exchange object is handed to Python as an integer handle; the IPC handle as a CPU uint8 tensor [64] the caller
// all-gathers with torch.distributed before `exchange_connect`.
std::tuple<int64_t, torch::Tensor> ExchangeCreate(const int rank, const int world, const int64_t capacity_rows, const int row_floats, const int device) {
	const c10::cuda::CUDAGuard guard(c10::Device(c10::kCUDA, device));
	rgs_exchange* ex = nullptr;
	torch::Tensor handle = torch::zeros({RGS_IPC_HANDLE_BYTES}, torch::kUInt8);
	if (rgs_exchange_create(rank, world, capacity_rows, row_floats, &ex, handle.data_ptr()) != RGS_OK) throw std::runtime_error(rgs_exchange_last_error());
	return std::make_tuple((int64_t)reinterpret_cast<intptr_t>(ex), handle);
}

int64_t ExchangeWindowBytes(const int world, const int64_t capacity_rows, const int row_floats) {
	return (int64_t)rgs_exchange_window_bytes(world, capacity_rows, row_floats);
}

int64_t ExchangeAttach(const int rank, const int world, const int64_t capacity_rows, const int row_floats, const std::vector<int64_t>& window_ptrs,
                       const int64_t multicast_ptr, const int device) {
	const c10::cuda::CUDAGuard guard(c10::Device(c10::kCUDA, device));
	TORCH_CHECK((int)window_ptrs.size() == world, "one window pointer per rank");
	std::vector<uint64_t> ptrs(window_ptrs.begin(), window_ptrs.end());
	rgs_exchange* ex = nullptr;
	if (rgs_exchange_attach(rank, world, capacity_rows, row_floats, ptrs.data(), (uint64_t)multicast_ptr, &ex) != RGS_OK)
		throw std::runtime_error(rgs_exchange_last_error());
	return (int64_t)reinterpret_cast<intptr_t>(ex);
}

void ExchangeConnect(const int64_t ex, const torch::Tensor& all_handles, const int device) {
	const c10::cuda::CUDAGuard guard(c10::Device(c10::kCUDA, device));
	torch::Tensor h = all_handles.to(torch::kCPU).contiguous();
	TORCH_CHECK(h.scalar_type() == torch::kUInt8 && h.numel() % RGS_IPC_HANDLE_BYTES == 0, "handles must be a uint8 tensor [world, 64]");
	if (rgs_exchange_connect(reinterpret_cast<rgs_exchange*>(ex), h.data_ptr()) != RGS_OK) throw std::runtime_error(rgs_exchange_last_error());
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
	TORCH_CHECK(tiles_touched.is_cuda() && radii.is_cuda() && tiles_touched.scalar_type() == torch::kInt32 && radii.scalar_type() == torch::kInt32,
	            "tiles_touched / radii must be CUDA int32 tensors");
	const c10::cuda::CUDAGuard guard(radii.device());
	torch::Tensor t = tiles_touched.contiguous(), r = radii.contiguous();
	if (rgs_exchange_rows(reinterpret_cast<rgs_exchange*>(ex), (int)r.numel(), reinterpret_cast<const uint32_t*>(t.data_ptr<int>()), r.data_ptr<int>(),
	                      at::cuda::getCurrentCUDAStream().stream()) != RGS_OK)
		throw std::runtime_error(rgs_exchange_last_error());
}

int ExchangeStatus(const int64_t ex) { return rgs_exchange_status(reinterpret_cast<rgs_exchange*>(ex), at::cuda::getCurrentCUDAStream().stream()); }

void ExchangeDestroy(const int64_t ex) { rgs_exchange_destroy(reinterpret_cast<rgs_exchange*>(ex)); }

// stage 1 + exchange: same arguments as BackwardRenderCUDA after the handle; returns the SUMMED rows [P, stride] (a view
// of the exchange's result buffer: valid until the next call on this exchange)
torch::Tensor BackwardRenderExchangeCUDA(const int64_t ex, const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& radii,
                                         const torch::Tensor& colors, const torch::Tensor& scales, const torch::Tensor& rotations,
                                         const float scale_modifier, const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix,
                                         const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy, const float kernel_size,
                                         const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_coord, const torch::Tensor& dL_dout_mcoord,
                                         const torch::Tensor& dL_dout_depth, const torch::Tensor& dL_dout_mdepth, const torch::Tensor& dL_dout_alpha,
                                         const torch::Tensor& dL_dout_normal, const torch::Tensor& normalmap, const torch::Tensor& sh, const int degree,
                                         const torch::Tensor& campos, const torch::Tensor& geomBuffer, const int R, const torch::Tensor& binningBuffer,
                                         const torch::Tensor& imageBuffer, const torch::Tensor& alphas, const bool require_coord,
                                         const bool require_depth, const bool debug, const int tile_row_begin, const int tile_row_end,
                                         const bool compact, const int image_height) {
	TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor: this rasterizer has no CPU path");
	const c10::cuda::CUDAGuard guard(means3D.device());
	const int P = means3D.size(0);
	const int GS = rgs_grad_stride(require_coord, require_depth);
	rgs_exchange* x = reinterpret_cast<rgs_exchange*>(ex);
	TORCH_CHECK(x != nullptr, "null exchange handle");
	if (P != 0) {
		BackwardCtx c;
		fill_backward(c, background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx,
		              tan_fovy, kernel_size, dL_dout_color, dL_dout_coord, dL_dout_mcoord, dL_dout_depth, dL_dout_mdepth, dL_dout_alpha,
		              dL_dout_normal, normalmap, sh, degree, campos, geomBuffer, R, binningBuffer, imageBuffer, alphas, require_coord, require_depth,
		              debug, tile_row_begin, tile_row_end, torch::Tensor(), compact, image_height);
		check(rgs_backward_render_exchange(&c.ch.cam, &c.gh.g, &c.in, x, at::cuda::getCurrentCUDAStream().stream()));
	}
	return torch::from_blob(const_cast<float*>(rgs_exchange_result(x)), {P, GS}, means3D.options().dtype(torch::kFloat32));
}

// stage 2: accumulator (after the cross-rank sum) -> the reference's 8-tuple of parameter gradients
BwdResult BackwardPreprocessCUDA(const torch::Tensor& grad_accum, const torch::Tensor& background, const torch::Tensor& means3D,
                                 const torch::Tensor& radii, const torch::Tensor& colors, const torch::Tensor& opacity, const torch::Tensor& scales,
                                 const torch::Tensor& rotations, const float scale_modifier, const torch::Tensor& cov3D_precomp,
                                 const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy,
                                 const float kernel_size, const int image_height, const int image_width, const torch::Tensor& sh, const int degree,
                                 const torch::Tensor& campos, const torch::Tensor& geomBuffer, const bool require_coord, const bool require_depth,
                                 const bool debug) {
	TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor: this rasterizer has no CPU path");
	const c10::cuda::CUDAGuard guard(means3D.device());
	const int P = means3D.size(0);
	int M = 0;
	if (sh.size(0) != 0) M = sh.size(1);
	GradTensors gt;
	alloc_grads(gt, means3D, P, M);
	if (P != 0) {
		CamHolder ch;
		fill_camera(ch, means3D, background, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, kernel_size, scale_modifier, image_height,
		            image_width, degree, M, false, require_coord, require_depth, debug, 0, -1);
		GaussHolder gh;
		fill_gaussians(gh, means3D, opacity, sh, colors, scales, rotations, cov3D_precomp);
		torch::Tensor acc = as_input(grad_accum, means3D, "grad_accum");
		torch::Tensor geom = geomBuffer.contiguous(), rad = radii.contiguous();
		rgs_backward_in in;
		memset(&in, 0, sizeof(in));
		in.radii = rad.data_ptr<int>();
		in.geom_buffer = reinterpret_cast<const char*>(geom.data_ptr());
		in.image_buffer = in.geom_buffer;    // not read by stage 2
		in.binning_buffer = in.geom_buffer;  // not read by stage 2
		check(rgs_backward_preprocess(&ch.cam, &gh.g, &in, acc.data_ptr<float>(), &gt.out, at::cuda::getCurrentCUDAStream().stream()));
	}
	return std::make_tuple(gt.means2D, gt.colors, gt.opacity, gt.means3D, gt.cov3D, gt.sh, gt.scales, gt.rotations);
}

// ---- split SH layout (opt-in, SURVEY.md 8f row 1): features_dc / features_rest stay two tensors, no torch.cat per iteration ----

FwdResult RasterizeGaussiansSplitShCUDA(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors,
                                        const torch::Tensor& opacity, const torch::Tensor& scales, const torch::Tensor& rotations,
                                        const float scale_modifier, const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix,
                                        const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy, const float kernel_size,
                                        const int image_height, const int image_width, const torch::Tensor& sh_dc, const torch::Tensor& sh_rest,
                                        const int degree, const torch::Tensor& campos, const bool prefiltered, const bool require_coord,
                                        const bool require_depth, const bool debug) {
	return forward_impl(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx,
	                    tan_fovy, kernel_size, image_height, image_width, sh_dc, degree, campos, prefiltered, require_coord, require_depth, debug, 0,
	                    -1, sh_rest);
}

using BwdSplitResult = std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor,
                                  torch::Tensor, torch::Tensor>;

// returns (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh_dc, dL_dsh_rest, dL_dscales, dL_drotations)
BwdSplitResult RasterizeGaussiansBackwardSplitShCUDA(
    const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& radii, const torch::Tensor& colors,
    const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier, const torch::Tensor& cov3D_precomp,
    const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy, const float kernel_size,
    const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_coord, const torch::Tensor& dL_dout_mcoord, const torch::Tensor& dL_dout_depth,
    const torch::Tensor& dL_dout_mdepth, const torch::Tensor& dL_dout_alpha, const torch::Tensor& dL_dout_normal, const torch::Tensor& normalmap,
    const torch::Tensor& sh_dc, const torch::Tensor& sh_rest, const int degree, const torch::Tensor& campos, const torch::Tensor& geomBuffer,
    const int R, const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer, const torch::Tensor& alphas, const bool require_coord,
    const bool require_depth, const bool debug) {
	TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor: this rasterizer has no CPU path");
	TORCH_CHECK(sh_rest.defined() && sh_rest.numel() != 0, "split SH layout needs a non-empty shs_rest");
	const c10::cuda::CUDAGuard guard(means3D.device());
	const int P = means3D.size(0);
	GradTensors gt;
	alloc_grads(gt, means3D, P, sh_coeffs(sh_dc, sh_rest), true);
	if (P != 0) {
		BackwardCtx c;
		fill_backward(c, background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx,
		              tan_fovy, kernel_size, dL_dout_color, dL_dout_coord, dL_dout_mcoord, dL_dout_depth, dL_dout_mdepth, dL_dout_alpha,
		              dL_dout_normal, normalmap, sh_dc, degree, campos, geomBuffer, R, binningBuffer, imageBuffer, alphas, require_coord,
		              require_depth, debug, 0, -1, sh_rest);
		torch::Tensor scratch = torch::empty({0}, means3D.options().dtype(torch::kByte));
		check(rgs_backward(&c.ch.cam, &c.gh.g, &c.in, &gt.out, resize_cb, &scratch, at::cuda::getCurrentCUDAStream().stream()));
	}
	return std::make_tuple(gt.means2D, gt.colors, gt.opacity, gt.means3D, gt.cov3D, gt.sh, gt.sh_rest, gt.scales, gt.rotations);
}

// ---- fused activations / densification statistics (opt-in, SURVEY.md 8f row 1) --------------------------------------------

std::tuple<torch::Tensor, torch::Tensor, torch::Tensor> ActivateForward(const torch::Tensor& raw_scaling, const torch::Tensor& raw_opacity,
                                                                        const torch::Tensor& raw_rotation, const torch::Tensor& filter_3D) {
	TORCH_CHECK(raw_scaling.is_cuda(), "raw_scaling must be a CUDA tensor: no CPU path");
	const c10::cuda::CUDAGuard guard(raw_scaling.device());
	const int P = raw_scaling.size(0);
	torch::Tensor s = as_input(raw_scaling, raw_scaling, "raw_scaling"), o = as_input(raw_opacity, raw_scaling, "raw_opacity"),
	              r = as_input(raw_rotation, raw_scaling, "raw_rotation"), f = as_input(filter_3D, raw_scaling, "filter_3D");
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
	const c10::cuda::CUDAGuard guard(raw_scaling.device());
	const int P = raw_scaling.size(0);
	torch::Tensor s = as_input(raw_scaling, raw_scaling, "raw_scaling"), o = as_input(raw_opacity, raw_scaling, "raw_opacity"),
	              r = as_input(raw_rotation, raw_scaling, "raw_rotation"), f = as_input(filter_3D, raw_scaling, "filter_3D"),
	              gs = as_input(g_scales, raw_scaling, "g_scales"), go = as_input(g_opacity, raw_scaling, "g_opacity"),
	              gr = as_input(g_rotations, raw_scaling, "g_rotations");
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
	const c10::cuda::CUDAGuard guard(means2D_grad.device());
	const int P = means2D_grad.size(0);
	if (P == 0) return;
	torch::Tensor g = as_input(means2D_grad, means2D_grad, "means2D.grad");
	torch::Tensor rad = radii.contiguous();
	for (const torch::Tensor* t : {&grad_accum, &grad_accum_abs, &grad_accum_abs_max, &denom})
		TORCH_CHECK(t->is_contiguous() && t->scalar_type() == torch::kFloat32 && t->numel() == P, "densification statistics must be contiguous float32 [P,1] tensors");
	float* mr = nullptr;
	if (max_radii2D.numel() != 0) {
		TORCH_CHECK(max_radii2D.is_contiguous() && max_radii2D.scalar_type() == torch::kFloat32 && max_radii2D.numel() == P, "max_radii2D must be contiguous float32 [P]");
		mr = max_radii2D.data_ptr<float>();
	}
	check(rgs_densification_stats(P, g.data_ptr<float>(), rad.data_ptr<int>(), grad_accum.data_ptr<float>(), grad_accum_abs.data_ptr<float>(),
	                              grad_accum_abs_max.data_ptr<float>(), denom.data_ptr<float>(), mr, at::cuda::getCurrentCUDAStream().stream()));
}

// returns (filter_3D [P,1], max_distance [1])
std::tuple<torch::Tensor, torch::Tensor> Compute3DFilter(const torch::Tensor& xyz, const torch::Tensor& cams, const double focal_length) {
	TORCH_CHECK(xyz.is_cuda(), "xyz must be a CUDA tensor: no CPU path");
	const c10::cuda::CUDAGuard guard(xyz.device());
	torch::Tensor x = as_input(xyz, xyz, "xyz"), c = as_input(cams, xyz, "camera table");
	const int P = xyz.size(0);
	TORCH_CHECK(c.numel() % 16 == 0, "camera table must be [n_cams,16]");
	const int n = (int)(c.numel() / 16);
	torch::Tensor out = new_empty({P, 1}, x.options()), mx = torch::zeros({1}, x.options());
	if (P)
		check(rgs_compute_3d_filter(P, x.data_ptr<float>(), n, n ? c.data_ptr<float>() : nullptr, (float)focal_length, out.data_ptr<float>(),
		                            mx.data_ptr<float>(), at::cuda::getCurrentCUDAStream().stream()));
	return std::make_tuple(out, mx);
}

// ---- fused image-side losses (opt-in, SURVEY.md 8f row 2) -----------------------------------------------------------------

torch::Tensor image_input(const torch::Tensor& t, const torch::Tensor& like, const char* name) {
	TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor: no CPU path");
	TORCH_CHECK(t.scalar_type() == torch::kFloat32, name, " must be float32");
	TORCH_CHECK(t.device() == like.device(), name, " must be on the same device as the image");
	return t.contiguous();
}

// returns (sums [2] float64: sum of the SSIM map, sum |img - gt|; dmaps [3, planes, H, W] or empty)
std::tuple<torch::Tensor, torch::Tensor> SsimL1Forward(const torch::Tensor& img, const torch::Tensor& gt, const bool need_grad, const int row_lo_in,
                                                        const int row_hi_in) {
	TORCH_CHECK(img.dim() >= 2 && img.numel() == gt.numel() && img.size(-1) == gt.size(-1) && img.size(-2) == gt.size(-2),
	            "ssim: images must have the same number of elements and the same [H, W]");
	torch::Tensor a = image_input(img, img, "img1"), b = image_input(gt, img, "img2");
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
	torch::Tensor a = image_input(img, img, "img1"), b = image_input(gt, img, "img2"), d = image_input(dmaps, img, "dmaps");
	const c10::cuda::CUDAGuard guard(a.device());
	const int H = a.size(-2), W = a.size(-1);
	const int planes = (int)(a.numel() / ((int64_t)H * W));
	TORCH_CHECK(d.numel() == 3 * a.numel(), "ssim backward: dmaps do not belong to these images");
	torch::Tensor up;
	const float* up_ptr = nullptr;
	if (upstream.defined() && upstream.numel() != 0) {
		TORCH_CHECK(upstream.numel() == 1, "ssim backward: upstream gradient must be a scalar");
		up = image_input(upstream, img, "upstream gradient");
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
	torch::Tensor n = image_input(rendered_normal, rendered_normal, "rendered_normal"), e = image_input(map_expected, rendered_normal, "expected map"),
	              m = image_input(map_median, rendered_normal, "median map");
	const c10::cuda::CUDAGuard guard(n.device());
	TORCH_CHECK(n.dim() == 3 && n.size(0) == 3, "rendered_normal must be [3,H,W]");
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

// simple_knn's distCUDA2 (reference scene/gaussian_model.py:315-316): points [P,3] float32 on a CUDA device -> [P] float32,
// the mean squared distance to the 3 nearest other points (rgs_knn_mean_dist2).  Non-contiguous input is accepted.
torch::Tensor KnnMeanDist2(const torch::Tensor& points) {
	TORCH_CHECK(points.dim() == 2 && points.size(1) == 3, "distCUDA2: points must have dimensions (num_points, 3), got ", points.sizes());
	TORCH_CHECK(points.scalar_type() == torch::kFloat32, "distCUDA2: points must be float32, got ", points.scalar_type());
	TORCH_CHECK(points.is_cuda(), "distCUDA2: points must be a CUDA tensor: no CPU path");
	TORCH_CHECK(points.size(0) <= INT32_MAX, "distCUDA2: at most 2^31 - 1 points");
	const c10::cuda::CUDAGuard guard(points.device());
	const int P = (int)points.size(0);
	torch::Tensor x = points.contiguous();
	torch::Tensor out = new_empty({P}, x.options());
	torch::Tensor scratch = torch::empty({0}, x.options().dtype(torch::kByte));
	if (P) check(rgs_knn_mean_dist2(P, x.data_ptr<float>(), out.data_ptr<float>(), resize_cb, &scratch, at::cuda::getCurrentCUDAStream().stream()));
	return out;
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
	m.def("rasterize_gaussians", &RasterizeGaussiansCUDA);
	m.def("integrate_gaussians_to_points", &IntegrateGaussiansToPointsCUDA);
	m.def("rasterize_gaussians_backward", &RasterizeGaussiansBackwardCUDA);
	m.def("mark_visible", &markVisible);
	// extras (not in the reference)
	m.def("rasterize_gaussians_slab", &RasterizeGaussiansSlabCUDA, py::arg("background"), py::arg("means3D"), py::arg("colors"), py::arg("opacity"), py::arg("scales"), py::arg("rotations"), py::arg("scale_modifier"), py::arg("cov3D_precomp"), py::arg("viewmatrix"), py::arg("projmatrix"), py::arg("tan_fovx"), py::arg("tan_fovy"), py::arg("kernel_size"), py::arg("image_height"), py::arg("image_width"), py::arg("sh"), py::arg("degree"), py::arg("campos"), py::arg("prefiltered"), py::arg("require_coord"), py::arg("require_depth"), py::arg("debug"), py::arg("tile_row_begin"), py::arg("tile_row_end"), py::arg("compact") = false);
	m.def("rasterize_gaussians_backward_render", &BackwardRenderCUDA, py::arg("background"), py::arg("means3D"), py::arg("radii"), py::arg("colors"), py::arg("scales"), py::arg("rotations"), py::arg("scale_modifier"), py::arg("cov3D_precomp"), py::arg("viewmatrix"), py::arg("projmatrix"), py::arg("tan_fovx"), py::arg("tan_fovy"), py::arg("kernel_size"), py::arg("dL_dout_color"), py::arg("dL_dout_coord"), py::arg("dL_dout_mcoord"), py::arg("dL_dout_depth"), py::arg("dL_dout_mdepth"), py::arg("dL_dout_alpha"), py::arg("dL_dout_normal"), py::arg("normalmap"), py::arg("sh"), py::arg("degree"), py::arg("campos"), py::arg("geomBuffer"), py::arg("R"), py::arg("binningBuffer"), py::arg("imageBuffer"), py::arg("alphas"), py::arg("require_coord"), py::arg("require_depth"), py::arg("debug"), py::arg("tile_row_begin"), py::arg("tile_row_end"), py::arg("compact") = false, py::arg("image_height") = -1);
	m.def("rasterize_gaussians_backward_preprocess", &BackwardPreprocessCUDA);
	m.def("exchange_create", &ExchangeCreate);
	m.def("exchange_connect", &ExchangeConnect);
	m.def("exchange_window_bytes", &ExchangeWindowBytes);
	m.def("exchange_attach", &ExchangeAttach);
	m.def("exchange_destroy", &ExchangeDestroy);
	m.def("exchange_accumulator", &ExchangeAccumulator);
	m.def("exchange_result", &ExchangeResult);
	m.def("exchange_rows", &ExchangeRows);
	m.def("exchange_status", &ExchangeStatus);
	m.def("rasterize_gaussians_backward_render_exchange", &BackwardRenderExchangeCUDA, py::arg("ex"), py::arg("background"), py::arg("means3D"), py::arg("radii"), py::arg("colors"), py::arg("scales"), py::arg("rotations"), py::arg("scale_modifier"), py::arg("cov3D_precomp"), py::arg("viewmatrix"), py::arg("projmatrix"), py::arg("tan_fovx"), py::arg("tan_fovy"), py::arg("kernel_size"), py::arg("dL_dout_color"), py::arg("dL_dout_coord"), py::arg("dL_dout_mcoord"), py::arg("dL_dout_depth"), py::arg("dL_dout_mdepth"), py::arg("dL_dout_alpha"), py::arg("dL_dout_normal"), py::arg("normalmap"), py::arg("sh"), py::arg("degree"), py::arg("campos"), py::arg("geomBuffer"), py::arg("R"), py::arg("binningBuffer"), py::arg("imageBuffer"), py::arg("alphas"), py::arg("require_coord"), py::arg("require_depth"), py::arg("debug"), py::arg("tile_row_begin"), py::arg("tile_row_end"), py::arg("compact") = false, py::arg("image_height") = -1);
	m.def("rasterize_gaussians_split_sh", &RasterizeGaussiansSplitShCUDA);
	m.def("rasterize_gaussians_backward_split_sh", &RasterizeGaussiansBackwardSplitShCUDA);
	m.def("compute_3d_filter", &Compute3DFilter);
	m.def("ssim_l1_forward", &SsimL1Forward, py::arg("img"), py::arg("gt"), py::arg("need_grad"), py::arg("row_lo") = 0, py::arg("row_hi") = -1);
	m.def("ssim_l1_backward", &SsimL1Backward, py::arg("img"), py::arg("gt"), py::arg("dmaps"), py::arg("w_ssim"), py::arg("w_l1"), py::arg("upstream"),
	      py::arg("row_lo") = 0, py::arg("row_hi") = -1);
	m.def("normal_consistency", &NormalConsistency);
	m.def("activate_forward", &ActivateForward);
	m.def("activate_backward", &ActivateBackward);
	m.def("densification_stats", &DensificationStats);
	m.def("knn_mean_dist2", &KnnMeanDist2, py::arg("points"));
	m.def("grad_stride", [](bool require_coord, bool require_depth) { return rgs_grad_stride(require_coord, require_depth); });
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

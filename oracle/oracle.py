"""ctypes front-end of the CPU oracle (oracle/oracle.c).  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this module; the product never
does.  `forward()` / `backward()` mirror the tuple layouts of the reference's `_C.rasterize_gaussians[_backward]`
(reference: submodules/diff-gaussian-rasterization/rasterize_points.cu:132,245) with numpy arrays.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "_build", "liboracle.so")

_f32p = C.POINTER(C.c_float)
_f64p = C.POINTER(C.c_double)
_i32p = C.POINTER(C.c_int32)
_u32p = C.POINTER(C.c_uint32)
_u64p = C.POINTER(C.c_uint64)
_u8p = C.POINTER(C.c_uint8)


class _Scene(C.Structure):
    _fields_ = [("P", C.c_int), ("D", C.c_int), ("M", C.c_int), ("W", C.c_int), ("H", C.c_int),
                ("tan_fovx", C.c_float), ("tan_fovy", C.c_float), ("kernel_size", C.c_float), ("scale_modifier", C.c_float),
                ("means3D", _f32p), ("opacities", _f32p), ("shs", _f32p), ("colors_precomp", _f32p), ("scales", _f32p),
                ("rotations", _f32p), ("cov3D_precomp", _f32p), ("viewmatrix", _f32p), ("projmatrix", _f32p), ("cam_pos", _f32p)]


class _Geom(C.Structure):
    _fields_ = [("radii", _i32p), ("means2D", _f32p), ("depths", _f32p), ("conic_opacity", _f32p), ("rgb", _f32p), ("clamped", _u8p),
                ("cov3D", _f32p), ("ts", _f32p), ("ray_planes", _f32p), ("camera_planes", _f32p), ("normals", _f32p),
                ("view_points", _f32p), ("tiles_touched", _u32p)]


class _Image(C.Structure):
    _fields_ = [("color", _f32p), ("coord", _f32p), ("mcoord", _f32p), ("alpha", _f32p), ("normal", _f32p), ("depth", _f32p),
                ("mdepth", _f32p), ("n_contrib", _u32p), ("accum_coord", _f32p), ("accum_depth", _f32p), ("normal_length", _f32p)]


class _SGrad(C.Structure):
    _fields_ = [("mean2D", _f64p), ("conic", _f64p), ("opacity", _f64p), ("colors", _f64p), ("ts", _f64p), ("camera_planes", _f64p),
                ("ray_planes", _f64p), ("normals", _f64p), ("view_points", _f64p)]


class _Upstream(C.Structure):
    _fields_ = [("color", _f32p), ("coord", _f32p), ("mcoord", _f32p), ("depth", _f32p), ("mdepth", _f32p), ("alpha", _f32p), ("normal", _f32p)]


class _PGrad(C.Structure):
    _fields_ = [("means2D", _f32p), ("colors", _f32p), ("opacity", _f32p), ("means3D", _f32p), ("cov3D", _f32p), ("sh", _f32p),
                ("scales", _f32p), ("rotations", _f32p)]


_lib = None


def build(force: bool = False) -> str:
    src = os.path.join(HERE, "oracle.c")
    if force or not os.path.exists(LIB_PATH) or os.path.getmtime(LIB_PATH) < os.path.getmtime(src):
        subprocess.run(["make", "-C", HERE, "-B" if force else "-s"], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    return LIB_PATH


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(LIB_PATH)
        _lib.orc_binning.restype = C.c_int64
        _lib.orc_binning.argtypes = [C.c_int, C.c_int, C.c_int, _i32p, _f32p, _f32p, _u64p, _u32p, _u32p]
        _lib.orc_eig_sym3.restype = C.c_int
        _lib.orc_eig_sym3.argtypes = [_f32p, _f32p, _f32p]
    return _lib


def _p(a, t):
    return a.ctypes.data_as(t) if a is not None else C.cast(None, t)


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


class Inputs:
    """Plain container of one rasterizer call's inputs (numpy, float32)."""

    def __init__(self, means3D, opacities, viewmatrix, projmatrix, campos, bg, W, H, tanfovx, tanfovy, shs=None, colors_precomp=None,
                 scales=None, rotations=None, cov3D_precomp=None, sh_degree=0, kernel_size=0.0, scale_modifier=1.0,
                 require_coord=False, require_depth=False):
        self.means3D, self.opacities = _f32(means3D), _f32(opacities).reshape(-1)
        self.viewmatrix, self.projmatrix, self.campos, self.bg = _f32(viewmatrix), _f32(projmatrix), _f32(campos), _f32(bg)
        self.shs, self.colors_precomp, self.scales, self.rotations, self.cov3D_precomp = _f32(shs), _f32(colors_precomp), _f32(scales), _f32(rotations), _f32(cov3D_precomp)
        self.W, self.H, self.tanfovx, self.tanfovy = int(W), int(H), float(tanfovx), float(tanfovy)
        self.sh_degree, self.kernel_size, self.scale_modifier = int(sh_degree), float(kernel_size), float(scale_modifier)
        self.require_coord, self.require_depth = bool(require_coord), bool(require_depth)
        self.P = self.means3D.shape[0]
        self.M = 0 if self.shs is None else self.shs.shape[1]

    def c_scene(self):
        return _Scene(self.P, self.sh_degree, self.M, self.W, self.H, self.tanfovx, self.tanfovy, self.kernel_size, self.scale_modifier,
                      _p(self.means3D, _f32p), _p(self.opacities, _f32p), _p(self.shs, _f32p), _p(self.colors_precomp, _f32p),
                      _p(self.scales, _f32p), _p(self.rotations, _f32p), _p(self.cov3D_precomp, _f32p), _p(self.viewmatrix, _f32p),
                      _p(self.projmatrix, _f32p), _p(self.campos, _f32p))


def preprocess(inp: Inputs) -> dict:
    P = inp.P
    g = dict(radii=np.zeros(P, np.int32), means2D=np.zeros((P, 2), np.float32), depths=np.zeros(P, np.float32),
             conic_opacity=np.zeros((P, 4), np.float32), rgb=np.zeros((P, 3), np.float32), clamped=np.zeros((P, 3), np.uint8),
             cov3D=np.zeros((P, 6), np.float32), ts=np.zeros(P, np.float32), ray_planes=np.zeros((P, 2), np.float32),
             camera_planes=np.zeros((P, 6), np.float32), normals=np.zeros((P, 3), np.float32), view_points=np.zeros((P, 3), np.float32),
             tiles_touched=np.zeros(P, np.uint32))
    sc = inp.c_scene()
    cg = _c_geom(g)
    lib().orc_preprocess(C.byref(sc), C.byref(cg))
    return g


def _c_geom(g):
    return _Geom(_p(g["radii"], _i32p), _p(g["means2D"], _f32p), _p(g["depths"], _f32p), _p(g["conic_opacity"], _f32p), _p(g["rgb"], _f32p),
                 _p(g["clamped"], _u8p), _p(g["cov3D"], _f32p), _p(g["ts"], _f32p), _p(g["ray_planes"], _f32p), _p(g["camera_planes"], _f32p),
                 _p(g["normals"], _f32p), _p(g["view_points"], _f32p), _p(g["tiles_touched"], _u32p))


def binning(W: int, H: int, radii, means2D, depths, tiles_touched=None) -> dict:
    """(tile|depth) keys, stable sort, per-tile ranges for the given per-Gaussian screen state."""
    radii = np.ascontiguousarray(radii, np.int32)
    means2D = np.ascontiguousarray(means2D, np.float32)
    depths = np.ascontiguousarray(depths, np.float32)
    P = radii.shape[0]
    gx, gy = (W + 15) // 16, (H + 15) // 16
    # capacity: every visible splat can touch at most the whole grid; size from a first exact count
    if tiles_touched is None:
        cap = 0
        for i in np.nonzero(radii > 0)[0]:
            r = int(radii[i])
            x0 = min(gx, max(0, int((means2D[i, 0] - r) / 16)))
            x1 = min(gx, max(0, int((means2D[i, 0] + r + 15) / 16)))
            y0 = min(gy, max(0, int((means2D[i, 1] - r) / 16)))
            y1 = min(gy, max(0, int((means2D[i, 1] + r + 15) / 16)))
            cap += (x1 - x0) * (y1 - y0)
    else:
        cap = int(np.asarray(tiles_touched, np.int64).sum())
    cap += gx * gy + 16  # slack: float truncation above is not bit-identical to the C code
    keys = np.zeros(cap, np.uint64)
    vals = np.zeros(cap, np.uint32)
    ranges = np.zeros((gx * gy, 2), np.uint32)
    n = lib().orc_binning(P, W, H, _p(radii, _i32p), _p(means2D, _f32p), _p(depths, _f32p), _p(keys, _u64p), _p(vals, _u32p), _p(ranges, _u32p))
    return dict(num_rendered=int(n), keys=keys[:n].copy(), point_list=vals[:n].copy(), ranges=ranges)


def render_forward(inp: Inputs, g: dict, b: dict) -> dict:
    H, W = inp.H, inp.W
    img = dict(color=np.zeros((3, H, W), np.float32), coord=np.zeros((3, H, W), np.float32), mcoord=np.zeros((3, H, W), np.float32),
               alpha=np.zeros((1, H, W), np.float32), normal=np.zeros((3, H, W), np.float32), depth=np.zeros((1, H, W), np.float32),
               mdepth=np.zeros((1, H, W), np.float32), n_contrib=np.zeros((2, H, W), np.uint32), accum_coord=np.zeros((3, H, W), np.float32),
               accum_depth=np.zeros((H, W), np.float32), normal_length=np.zeros((H, W), np.float32))
    ci = _c_image(img)
    cg = _c_geom(g)
    ranges = np.ascontiguousarray(b["ranges"], np.uint32)
    pl = np.ascontiguousarray(b["point_list"], np.uint32)
    lib().orc_render_forward(C.c_int(W), C.c_int(H), C.c_float(inp.tanfovx), C.c_float(inp.tanfovy), _p(inp.bg, _f32p), C.c_int(inp.require_coord),
                             C.c_int(inp.require_depth), _p(ranges, _u32p), _p(pl, _u32p), C.byref(cg), C.byref(ci))
    return img


def _c_image(img):
    return _Image(_p(img["color"], _f32p), _p(img["coord"], _f32p), _p(img["mcoord"], _f32p), _p(img["alpha"], _f32p), _p(img["normal"], _f32p),
                  _p(img["depth"], _f32p), _p(img["mdepth"], _f32p), _p(img["n_contrib"], _u32p), _p(img["accum_coord"], _f32p),
                  _p(img["accum_depth"], _f32p), _p(img["normal_length"], _f32p))


def forward(inp: Inputs) -> dict:
    """Whole forward pass; keys follow the reference's 12-tuple plus the decoded internal state."""
    g = preprocess(inp)
    b = binning(inp.W, inp.H, g["radii"], g["means2D"], g["depths"], g["tiles_touched"])
    img = render_forward(inp, g, b)
    return dict(num_rendered=b["num_rendered"], geom=g, binning=b, image=img, radii=g["radii"],
                **{k: img[k] for k in ("color", "coord", "mcoord", "alpha", "normal", "depth", "mdepth")})


def render_backward(inp: Inputs, fwd: dict, grads: dict) -> dict:
    """Screen-space per-Gaussian gradients (what backward.cu:631-1016 scatters), float64 sums."""
    P = inp.P
    sg = dict(mean2D=np.zeros((P, 3)), conic=np.zeros((P, 4)), opacity=np.zeros(P), colors=np.zeros((P, 3)), ts=np.zeros(P),
              camera_planes=np.zeros((P, 6)), ray_planes=np.zeros((P, 2)), normals=np.zeros((P, 3)), view_points=np.zeros((P, 3)))
    up = {k: _f32(grads[k]) for k in ("color", "coord", "mcoord", "depth", "mdepth", "alpha", "normal")}
    cu = _Upstream(*[_p(up[k], _f32p) for k in ("color", "coord", "mcoord", "depth", "mdepth", "alpha", "normal")])
    csg = _SGrad(*[_p(sg[k], _f64p) for k in ("mean2D", "conic", "opacity", "colors", "ts", "camera_planes", "ray_planes", "normals", "view_points")])
    cg, ci = _c_geom(fwd["geom"]), _c_image(fwd["image"])
    ranges = np.ascontiguousarray(fwd["binning"]["ranges"], np.uint32)
    pl = np.ascontiguousarray(fwd["binning"]["point_list"], np.uint32)
    lib().orc_render_backward(C.c_int(inp.W), C.c_int(inp.H), C.c_float(inp.tanfovx), C.c_float(inp.tanfovy), _p(inp.bg, _f32p),
                              C.c_int(inp.require_coord), C.c_int(inp.require_depth), _p(ranges, _u32p), _p(pl, _u32p), C.byref(cg), C.byref(ci),
                              C.byref(cu), C.byref(csg))
    return sg


def preprocess_backward(inp: Inputs, fwd: dict, sg: dict, fix_mip_gradient: bool = False) -> dict:
    P, M = inp.P, inp.M
    out = dict(means2D=np.zeros((P, 3), np.float32), colors=np.zeros((P, 3), np.float32), opacity=np.zeros((P, 1), np.float32),
               means3D=np.zeros((P, 3), np.float32), cov3D=np.zeros((P, 6), np.float32), sh=np.zeros((P, M, 3), np.float32),
               scales=np.zeros((P, 3), np.float32), rotations=np.zeros((P, 4), np.float32))
    cp = _PGrad(*[_p(out[k], _f32p) for k in ("means2D", "colors", "opacity", "means3D", "cov3D", "sh", "scales", "rotations")])
    csg = _SGrad(*[_p(sg[k], _f64p) for k in ("mean2D", "conic", "opacity", "colors", "ts", "camera_planes", "ray_planes", "normals", "view_points")])
    sc, cg = inp.c_scene(), _c_geom(fwd["geom"])
    lib().orc_preprocess_backward(C.byref(sc), C.byref(cg), C.byref(csg), C.byref(cp), C.c_int(int(fix_mip_gradient)))
    return out


def backward(inp: Inputs, fwd: dict, grads: dict, fix_mip_gradient: bool = False) -> dict:
    sg = render_backward(inp, fwd, grads)
    out = preprocess_backward(inp, fwd, sg, fix_mip_gradient)
    out["_screen"] = sg
    return out


class _IntegrateOut(C.Structure):
    _fields_ = [(n, _f32p) for n in ("out_color", "alpha_integrated", "color_integrated", "coordinate2d", "sdf")]


def integrate(inp: Inputs, points3D) -> dict:
    """`integrate_gaussians_to_points` (rasterize_points.cu:269-388): the reference always runs it with kernel_size 0 and both
    geometry variants on; `inp` must have been built with kernel_size=0."""
    assert inp.kernel_size == 0.0, "GaussianRasterizer.integrate passes kernel_size 0.0 (diff_gaussian_rasterization/__init__.py:281)"
    points3D = np.ascontiguousarray(points3D, np.float32)
    PN, P, H, W = points3D.shape[0], inp.P, inp.H, inp.W
    g = preprocess(inp)
    b = binning(W, H, g["radii"], g["means2D"], g["depths"], g["tiles_touched"])
    invraycov = np.zeros((P, 6), np.float32)
    condition = np.zeros(P, np.uint8)
    sigma_inv = np.zeros((P, 12), np.float32)  # what orc_inte_geometry used: 9 floats column-major, the flag bits in float 9
    sc, cg = inp.c_scene(), _c_geom(g)
    lib().orc_inte_geometry(C.byref(sc), C.byref(cg), _p(invraycov, _f32p), _p(condition, _u8p), _p(sigma_inv, _f32p))
    out = dict(color=np.zeros((9, H, W), np.float32), alpha_integrated=np.ones(PN, np.float32), color_integrated=np.zeros((PN, 3), np.float32),
               point_coordinate=np.zeros((PN, 2), np.float32), point_sdf=np.full(PN, -1000.0, np.float32))
    co = _IntegrateOut(_p(out["color"], _f32p), _p(out["alpha_integrated"], _f32p), _p(out["color_integrated"], _f32p),
                       _p(out["point_coordinate"], _f32p), _p(out["point_sdf"], _f32p))
    ranges = np.ascontiguousarray(b["ranges"], np.uint32)
    pl = np.ascontiguousarray(b["point_list"], np.uint32)
    lib().orc_integrate.restype = C.c_int
    over = lib().orc_integrate(C.c_int(W), C.c_int(H), C.c_float(inp.tanfovx), C.c_float(inp.tanfovy), _p(inp.bg, _f32p), _p(ranges, _u32p),
                               _p(pl, _u32p), C.byref(cg), _p(invraycov, _f32p), _p(condition, _u8p), C.c_int(PN), _p(points3D, _f32p),
                               _p(inp.viewmatrix, _f32p), C.byref(co))
    out.update(radii=g["radii"], num_rendered=b["num_rendered"], invraycov=invraycov, condition=condition, sigma_inv=sigma_inv, overflowed=int(over), geom=g, binning=b)
    return out


def eig_sym3(cov6):
    cov6 = np.ascontiguousarray(cov6, np.float32)
    lam = np.zeros(3, np.float32)
    vec = np.zeros(9, np.float32)
    rc = lib().orc_eig_sym3(_p(cov6, _f32p), _p(lam, _f32p), _p(vec, _f32p))
    return rc, lam, vec.reshape(3, 3).T.copy()  # columns = eigenvectors

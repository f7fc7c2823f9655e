"""CPU checks of the exact Delaunay model (tests/delaunay_exact.py) and of the bindings' and the C ABI's rejections."""
import ctypes
import itertools
import os

import numpy as np
import pytest
import torch

import delaunay_exact as dx

REGULAR = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], dtype=np.float32)   # positive


def test_signs_on_hand_built_tuples():
    a, b, c, d = REGULAR
    assert dx.orient3d(a, b, c, d) == 1 and dx.orient3d(a, c, b, d) == -1
    assert dx.orient3d(a, b, c, np.float32([0.3, 0.7, 0.0])) == 0                 # coplanar
    assert dx.insphere(a, b, c, d, np.float32([0.2, 0.2, 0.2])) == 1              # inside
    assert dx.insphere(a, b, c, d, np.float32([3, 3, 3])) == -1
    assert dx.insphere(a, b, c, d, np.float32([1, 1, 1])) == 0                    # the cube's corners are cospherical
    # scaled far down and far up: the exact stage decides what the fp64 determinant cannot
    for e in (-100, -60, 0, 40, 90):
        s = np.float32(2.0 ** e)
        assert dx.orient3d(a * s, b * s, c * s, d * s) == 1
        assert dx.insphere(a * s, b * s, c * s, d * s, np.float32([1, 1, 1]) * s) == 0
    near = np.float32([1, 1, np.nextafter(np.float32(1), np.float32(2))])
    assert dx.insphere(a, b, c, d, near) == -1


def test_perturbation_decides_every_cospherical_tuple_consistently():
    cube = np.array(list(itertools.product((0, 1), repeat=3)), dtype=np.float32)
    for five in itertools.combinations(range(8), 5):
        p = cube[list(five)]
        if dx.orient3d(*p[:4]) == 0:
            continue
        base = dx.insphere_perturbed(*p)
        assert base != 0
        # swapping two of the first four flips the orientation and the sign together
        q = p[[1, 0, 2, 3, 4]]
        assert dx.insphere_perturbed(*q) == -base
    # lattice tuple with integer coordinates: sign matches the rule "largest point first"
    a, b, c, d = REGULAR
    e = np.float32([1, 1, 1])      # the lexicographically largest: it is lifted most, so it lies outside
    assert dx.insphere_perturbed(a, b, c, d, e) == -1


def test_checker_accepts_scipy_cells_once_reoriented():
    from scipy.spatial import Delaunay
    rng = np.random.default_rng(0)
    for n in (5, 60, 300):
        p = rng.normal(size=(n, 3)).astype(np.float32)
        cells = dx.reorient(p, Delaunay(p.astype(np.float64)).simplices)
        assert dx.check(p, cells) > 0 or n == 5


def test_checker_rejects_broken_meshes():
    from scipy.spatial import Delaunay
    rng = np.random.default_rng(1)
    p = rng.normal(size=(80, 3)).astype(np.float32)
    cells = dx.reorient(p, Delaunay(p.astype(np.float64)).simplices)
    flipped = cells.copy()
    flipped[0, 2], flipped[0, 3] = flipped[0, 3], flipped[0, 2]
    with pytest.raises(AssertionError, match="not positive"):
        dx.check(p, flipped)
    with pytest.raises(AssertionError):
        dx.check(p, cells[1:])                                  # a missing cell opens the boundary
    with pytest.raises(AssertionError):
        dx.check(p, np.concatenate([cells, cells[:1]]))         # a duplicated cell
    # a non-Delaunay face: flip one interior face 2-3 where the union is convex
    from collections import defaultdict
    own = defaultdict(list)
    for i, t in enumerate(cells):
        for f in itertools.combinations(sorted(t), 3):
            own[f].append(i)
    for f, cs in own.items():
        if len(cs) != 2:
            continue
        a, b, c = f
        d = [v for v in cells[cs[0]] if v not in f][0]
        e = [v for v in cells[cs[1]] if v not in f][0]
        new = [np.array(x) for x in ((d, e, a, b), (d, e, b, c), (d, e, c, a))]
        signs = {dx.orient3d(*p[t]) for t in new}
        if len(signs) != 1 or 0 in signs:   # the segment de misses the triangle abc: no 2-3 flip here
            continue
        new = [t if signs == {1} else t[[0, 1, 3, 2]] for t in new]
        bad = np.concatenate([np.delete(cells, cs, axis=0), np.stack(new)])
        with pytest.raises(AssertionError, match="locally Delaunay"):
            dx.check(p, bad)
        break
    else:
        pytest.fail("no flippable face")


def test_bindings_refuse_cpu_tensors():
    from diff_gaussian_rasterization import _C
    assert {n for n in dir(_C._delaunay) if not n.startswith("_")} == {"triangulate", "predicates"}
    with pytest.raises(RuntimeError, match="CUDA"):
        _C._delaunay.triangulate(torch.zeros(8, 3))
    with pytest.raises(RuntimeError, match="CUDA"):
        _C._delaunay.predicates(torch.zeros(8, 3), torch.zeros(2, 5, dtype=torch.int32))
    from rade_gs_b200 import tetra
    with pytest.raises(RuntimeError, match="no CPU path"):
        tetra.delaunay(torch.zeros(8, 3))


def test_c_abi_rejects_null_pointers_and_bad_counts():
    from conftest import ROOT
    lib = ctypes.CDLL(os.path.join(ROOT, "rade-gs_b200", "rade_gs_b200", "librgs_b200.so"))
    lib.rgs_last_error.restype = ctypes.c_char_p
    lib.rgs_delaunay.argtypes = [ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    fake = ctypes.c_void_p(0x1000)   # never dereferenced: rejected before the first CUDA call
    out = (ctypes.c_char * 128)()
    assert lib.rgs_delaunay(10, fake, None, out, None) == -1 and b"null" in lib.rgs_last_error()
    assert lib.rgs_delaunay(10, None, fake, out, None) == -1 and b"null" in lib.rgs_last_error()
    assert lib.rgs_delaunay(-1, fake, fake, out, None) == -1 and b"out of range" in lib.rgs_last_error()
    assert lib.rgs_delaunay((1 << 26) + 1, fake, fake, out, None) == -1 and b"out of range" in lib.rgs_last_error()

"""Backward blend with two pixels per lane: a warp owns an 8x8 pixel block, lane l the pixels (l & 7, l >> 3) and
(l & 7, (l >> 3) + 4), so each lane carries one pixel of each 8x4 half for which forward-render stored a hit-mask word
(rgs_render_bwd.cu).  The scenes here aim at what that layout adds: splats that reach only the upper half of a block, only the
lower half, or both (the hit mask is the OR of the halves' words); halves whose last contributors differ, so that the warp's
64-pixel cut is set by one half while the other half's pixels lie behind their own; images whose last block row has its lower
half outside the image (H = 20, H = 12); and hits on both sides of the 128-record batch boundary.  Every accumulator row is
checked against the fp64 blend (tests/blend_f64.py) as in test_gpu_blend_exact.py; the rows of the hidden splats and the
padding of coord rows must be exactly zero.

A "upper" / "lower" / "both" hit is a small round splat centred on a pixel of one 8x8 block; its depth is its rank in the tile,
so the tile list is in the order given below."""
import numpy as np
import pytest
import torch

import blend_scenes as bs
from rade_gs_b200 import rawapi, scenes
from test_gpu_blend_exact import DEV, VARIANTS, _C, _run

pytestmark = pytest.mark.gpu
FOCAL = 60.0


def _place(kind, bx0, by0, g):
    """centre (u, v), sigma (x, y) in pixels and opacity of one entry on the 8x8 block at (bx0, by0)"""
    r = lambda k: int(torch.randint(0, k, (1,), generator=g))
    cu = bx0 + 3 + r(2)
    if kind in ("upper", "hidden"):    # alpha >= 1/255 reaches 1.25 px: rows by0 .. by0 + 3 only
        return cu, by0 + 1 + r(2), (0.4, 0.4), 0.5
    if kind == "lower":                # rows by0 + 4 .. by0 + 7 only
        return cu, by0 + 5 + r(2), (0.4, 0.4), 0.5
    if kind == "both":                 # centred between rows 3 and 4, reaches 3.1 px up and down
        return cu, by0 + 3.5, (0.4, 1.0), 0.5
    if kind == "occluder":             # T < 1e-4 at the middle columns of the upper half after 120 of them; alpha < 0.01 in the lower
        return bx0 + 3.5, by0 + 1.5, (3.0, 0.8), 1.0
    return cu, by0 + r(8), (0.4, 0.4), 0.02   # filler


def _mixed_tile(g, n=24):
    kinds = ("upper", "lower", "both")
    return [(kinds[r % 3], int(w)) for r, w in zip(torch.randperm(3 * n, generator=g).tolist(), torch.randint(0, 4, (3 * n,), generator=g).tolist())]


def _boundary_tile(n=301):
    """n entries: fillers on block 3 keep the block's cut at n; block 0 has an upper, a lower and a "both" hit on each side of the
    128- and 256-entry batch boundaries counted from the back, block 1 one of each in the last, partial batch."""
    spec = [("filler", 3)] * n
    for b in (128, 256):
        spec[n - b - 2], spec[n - b - 1], spec[n - b] = ("upper", 0), ("lower", 0), ("both", 0)
        spec[n - b + 1] = ("both", 0)
    spec[0], spec[1], spec[2] = ("upper", 1), ("lower", 1), ("both", 1)
    return spec


def _split_cut_tile(n_occ=120):
    """Block 0: occluders over its upper half in front, then hidden upper hits interleaved with hits on both halves, and lower
    hits at the back: the upper half's last contributor sits at the occluders, the block's 64-pixel cut at the back.  Block 2
    the mirror image without occluders (its lower half's hits in front)."""
    spec = [("occluder", 0)] * n_occ
    spec += [("hidden", 0), ("both", 0), ("both", 0), ("hidden", 0), ("lower", 2), ("upper", 2)] * 4
    spec += [("lower", 0)] * 6 + [("upper", 2)] * 3
    return spec


def _scene(seed=31):
    W, H = 80, 16
    g = torch.Generator().manual_seed(seed)
    # tile 1 stays empty, so that no footprint of the later tiles (the occluders reach 10 px sideways, the hits 4 px) reaches
    # tile 0, whose list positions are counted
    tiles = [_boundary_tile(), [], _mixed_tile(g), _split_cut_tile(), _mixed_tile(g)]
    u, v, z, sig, opac, hidden = [], [], [], [], [], []
    for t, spec in enumerate(tiles):
        for rank, (kind, w) in enumerate(spec):
            cu, cv, s, o = _place(kind, 16 * t + (w & 1) * 8, (w >> 1) * 8, g)
            if kind == "hidden":
                hidden.append(len(u))
            zz = 2.0 + 0.004 * rank
            u.append(cu); v.append(cv); z.append(zz); opac.append(o)
            sig.append((s[0] * zz / FOCAL, s[1] * zz / FOCAL, 0.4 * zz / FOCAL))
    P = len(u)
    rots = torch.tensor([[1.0, 0.0, 0.0, 0.0]]).repeat(P, 1)
    sc = bs.build(W, H, FOCAL, torch.tensor(u, dtype=torch.float64), torch.tensor(v, dtype=torch.float64), torch.tensor(z, dtype=torch.float64),
                  torch.tensor(sig, dtype=torch.float64), rots, torch.tensor(opac), seed)
    return sc, hidden


def _name(fam, coord, depth):
    return f"{fam}/{'coord' if coord else ''}{'depth' if depth else ''}{'' if coord or depth else 'none'}"


def _backward(sc, coord, depth):
    scd = sc.to(DEV)
    f = rawapi.forward(_C(), scd, coord, depth, kernel_size=0.0)
    grads = {k: t.to(DEV) for k, t in scenes.make_upstream_grads(sc.height, sc.width, seed=17).items()}
    return rawapi.backward_render(_C(), scd, f, grads).cpu().numpy()


@pytest.mark.parametrize("coord,depth", VARIANTS, ids=["none", "depth", "coord", "both"])
def test_backward_block_halves(coord, depth):
    sc, hidden = _scene()
    v, _, _ = _run(sc, coord, depth, 0.0, _name("pairs", coord, depth))
    assert int(v["ranges"][0, 1] - v["ranges"][0, 0]) == 301, "tile 0 must hold exactly its own entries"
    nc = v["n_contrib"][0].cpu().numpy()
    up, low = nc[0:4, 48:56].max(), nc[4:8, 48:56].max()
    assert up < 120 < low, f"the halves of tile 3's block 0 must end at different list positions: {up} {low}"
    acc = _backward(sc, coord, depth)
    assert np.all(acc[hidden] == 0), "a splat behind every last contributor of the pixels it reaches received gradient"
    if coord:
        assert np.all(acc[:, 25:] == 0), "padding of the coord rows"


@pytest.mark.parametrize("coord,depth", VARIANTS, ids=["none", "depth", "coord", "both"])
@pytest.mark.parametrize("W,H,P,seed", [(48, 20, 300, 41), (40, 12, 200, 42)], ids=["48x20", "40x12"])
def test_backward_lower_half_outside(W, H, P, seed, coord, depth):
    """H = 20: the second tile row's blocks have rows 16..19 inside, their lower halves outside; H = 12: the first row's
    lower blocks have rows 8..11 inside, their lower halves outside."""
    sc = bs.tiny(W, H, P, seed)
    _run(sc, coord, depth, 0.0, _name(f"pairs_{W}x{H}", coord, depth))
    if coord:
        assert np.all(_backward(sc, coord, depth)[:, 25:] == 0), "padding of the coord rows"

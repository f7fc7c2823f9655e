"""Backward blend at the edges of its hit groups: a warp sums the gradient rows of its hits in groups (rgs_render_bwd.cu,
HitGroup), so the tiles here give warps 0..5 surviving hits in one batch, hits on both sides of the 128- and 256-entry batch
boundaries, a single hit in the last, partial batch, and a warp whose hits in a batch all lie behind its last contributor.
Every accumulator row is checked against the fp64 blend (tests/blend_f64.py) as in test_gpu_blend_exact.py; the rows of the
hidden splats and the padding of coord rows must be exactly zero.

Scene: a 64x16 image, four 16x16 tiles, built in camera space.  A "hit" or "filler" is a small round splat centred on a pixel
inside one warp's 8x4 block, so it reaches that block only and stays inside its tile; its depth is its rank in the tile, so
the tile list is in the order given below."""
import numpy as np
import pytest
import torch

import blend_scenes as bs
from rade_gs_b200 import rawapi, scenes
from test_gpu_blend_exact import DEV, VARIANTS, _C, _run

pytestmark = pytest.mark.gpu
FOCAL = 60.0
W, H = 64, 16


def _counts_tile(counts, g):
    """Warp w gets counts[w] hits, the warps' hits interleaved in depth."""
    order = torch.cat([torch.full((c,), w) for w, c in enumerate(counts)])
    return [("hit", int(w)) for w in order[torch.randperm(order.numel(), generator=g)]]


def _boundary_tile(n):
    """n entries: fillers on warp 7 (the last one at the back keeps the block's cut at n), warp 0 with hits at the pairs of
    positions that straddle the 128- and 256-entry batch boundaries counted from the back, warp 1 with one hit at position 0
    (inside the last, partial batch), warp 2 with hits at the positions next to warp 0's."""
    spec = [("filler", 7)] * n
    for b in (128, 256):
        spec[n - b - 1] = spec[n - b] = ("hit", 0)
        spec[n - b - 2] = spec[n - b + 1] = ("hit", 2)
    spec[0] = ("hit", 1)
    return spec


def _occluded_tile(n_occ=40, n_fill=150, hidden=(50, 120, 191, 192)):
    """n_occ opaque, wide splats over warp 3's block in front (they drive T below 1e-4 at all 32 of its pixels), then fillers
    on warp 6 with hits on warp 3 at the list positions `hidden`, all behind warp 3's last contributor."""
    spec = [("occluder", 3)] * n_occ + [("filler", 6)] * n_fill
    for p in hidden:
        spec.insert(p, ("hit", 3))
    return spec


def _scene(seed=21):
    g = torch.Generator().manual_seed(seed)
    tiles = [_counts_tile([0, 1, 2, 3, 4, 5, 1, 2], g), _counts_tile([3, 4, 5, 0, 1, 2, 3, 3], g), _boundary_tile(301),
             _occluded_tile()]
    u, v, z, sig, opac, hidden = [], [], [], [], [], []
    for t, spec in enumerate(tiles):
        for rank, (kind, w) in enumerate(spec):
            bx0, by0 = 16 * t + (w & 1) * 8, (w >> 1) * 4
            if kind == "occluder":
                cu, cv, s, o = bx0 + 3.5, by0 + 1.5, (3.0, 1.2), 1.0
            else:
                # pixel centres 3 px from the block's sides, and for hits 1 px from its top and bottom: alpha >= 1/255
                # reaches 1.25 px (hit) / 0.72 px (filler) and the tile rectangle 3 px
                cu = bx0 + 3 + int(torch.randint(0, 2, (1,), generator=g))
                cv = by0 + (1 + int(torch.randint(0, 2, (1,), generator=g)) if kind == "hit" else int(torch.randint(0, 4, (1,), generator=g)))
                s, o = (0.4, 0.4), (0.5 if kind == "hit" else 0.02)
            if kind == "hit" and t == 3:
                hidden.append(len(u))
            zz = 2.0 + 0.004 * rank
            u.append(cu); v.append(cv); z.append(zz); opac.append(o)
            sig.append((s[0] * zz / FOCAL, s[1] * zz / FOCAL, 0.4 * zz / FOCAL))
    P = len(u)
    rots = torch.tensor([[1.0, 0.0, 0.0, 0.0]]).repeat(P, 1)
    sc = bs.build(W, H, FOCAL, torch.tensor(u, dtype=torch.float64), torch.tensor(v, dtype=torch.float64), torch.tensor(z, dtype=torch.float64),
                  torch.tensor(sig, dtype=torch.float64), rots, torch.tensor(opac), seed)
    return sc, [len(s) for s in tiles], hidden


@pytest.mark.parametrize("coord,depth", VARIANTS, ids=["none", "depth", "coord", "both"])
def test_backward_hit_groups(coord, depth):
    sc, lengths, hidden = _scene()
    name = f"groups/{'coord' if coord else ''}{'depth' if depth else ''}{'' if coord or depth else 'none'}"
    v, _, _ = _run(sc, coord, depth, 0.0, name)
    n = (v["ranges"][:, 1] - v["ranges"][:, 0]).cpu().numpy()
    assert n.tolist() == lengths, "every splat must stay inside its own tile"
    scd = sc.to(DEV)
    f = rawapi.forward(_C(), scd, coord, depth, kernel_size=0.0)
    grads = {k: t.to(DEV) for k, t in scenes.make_upstream_grads(sc.height, sc.width, seed=17).items()}
    acc = rawapi.backward_render(_C(), scd, f, grads).cpu().numpy()
    assert np.all(acc[hidden] == 0), "a splat behind every last contributor of its warp received gradient"
    if coord:
        assert np.all(acc[:, 25:] == 0), "padding of the coord rows"

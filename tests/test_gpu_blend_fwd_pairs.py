"""Forward blend with two pixels per lane: a warp owns an 8x8 pixel block, lane l the pixels (l & 7, l >> 3) and (l & 7, (l >> 3) + 4),
the box test culls a staged splat once for all 64 pixels, and the warp's 8x8 ballot is stored into the hit-mask slots of both of its
8x4 halves (rgs_render_fwd.cu).  The scenes aim at what that layout adds: splats that reach only the upper half of a block, only
the lower half, or both; one half saturating early behind occluders while the other half keeps blending (the saturated pixels
must take nothing more and the warp must not stop); a whole tile saturating mid-list, so that the block exits; images whose last
block row or column lies partly outside (H = 20, H = 12, W = 44); and hits on both sides of the 128- and 256-entry boundaries.

Every map is checked against the fp64 blend and n_contrib exactly (tests/blend_f64.py, as in test_gpu_blend_exact.py).  The
stored ballots are checked too: the two half-block words of a block are equal for every chunk, and for every pixel and every list
entry the fp64 blend takes there, the entry's bit is set in both."""
import numpy as np
import pytest
import torch

import blend_f64 as bf
import blend_scenes as bs
from rade_gs_b200 import rawapi
from test_gpu_blend_exact import DEV, VARIANTS, _C, _run
from test_gpu_blend_pairs import FOCAL, _mixed_tile, _name, _place, _split_cut_tile

pytestmark = pytest.mark.gpu
UPPER_SLOTS = [0, 1, 4, 5]  # hit-mask slot of the upper 8x4 half of each 8x8 block; the lower half's is that + 2


def _boundary_tile(n=301):
    """n entries: fillers on block 3; block 0 has an upper, a lower and a "both" hit on each side of list positions 128 and 256
    (the forward walks the list from the front), block 1 one of each in the last, partial round."""
    spec = [("filler", 3)] * n
    for b in (128, 256):
        spec[b - 2], spec[b - 1], spec[b], spec[b + 1] = ("upper", 0), ("lower", 0), ("both", 0), ("both", 0)
    spec[n - 3], spec[n - 2], spec[n - 1] = ("upper", 1), ("lower", 1), ("both", 1)
    return spec


def _wall_tile(n_wall=10, n_behind=300):
    """Wide opaque splats centred on the tile (alpha >= 0.67 at every pixel of it, so T < 1e-4 after at most ten), then more
    than a round of hits behind them on every block: the whole tile saturates inside the first round and the block exits."""
    g = torch.Generator().manual_seed(5)
    kinds = ("upper", "lower", "both", "filler")
    return [("wall", 0)] * n_wall + [(kinds[k % 4], w) for k, w in enumerate(torch.randint(0, 4, (n_behind,), generator=g).tolist())]


def _scene(seed=37):
    # tiles 1 and 4..6 stay empty: the hits reach 4 px and the occluders 10 px sideways, the walls of tile 7 36 px
    tiles = [_boundary_tile(), [], _mixed_tile(torch.Generator().manual_seed(seed)), _split_cut_tile(), [], [], [], _wall_tile()]
    W, H = 16 * len(tiles), 16
    g = torch.Generator().manual_seed(seed)
    u, v, z, sig, opac = [], [], [], [], []
    for t, spec in enumerate(tiles):
        for rank, (kind, w) in enumerate(spec):
            if kind == "wall":
                cu, cv, s, o = 16 * t + 7.5, 7.5, (12.0, 12.0), 1.0
            else:
                cu, cv, s, o = _place(kind, 16 * t + (w & 1) * 8, (w >> 1) * 8, g)
            zz = 2.0 + 0.004 * rank
            u.append(cu); v.append(cv); z.append(zz); opac.append(o)
            sig.append((s[0] * zz / FOCAL, s[1] * zz / FOCAL, 0.4 * zz / FOCAL))
    P = len(u)
    rots = torch.tensor([[1.0, 0.0, 0.0, 0.0]]).repeat(P, 1)
    return bs.build(W, H, FOCAL, torch.tensor(u, dtype=torch.float64), torch.tensor(v, dtype=torch.float64), torch.tensor(z, dtype=torch.float64),
                    torch.tensor(sig, dtype=torch.float64), rots, torch.tensor(opac), seed)


def _check_ballots(sc, coord, depth, name):
    """Both half-block words equal for every chunk; every (pixel, entry) pair the fp64 blend takes has its bit set in both."""
    scd = sc.to(DEV)
    f = rawapi.forward(_C(), scd, coord, depth, kernel_size=0.0)
    v = rawapi.ours_views(f, scd)
    words = v["hitmask"].view(-1, 8).cpu().numpy().view(np.uint32)
    up = np.array(UPPER_SLOTS)
    assert np.array_equal(words[:, up], words[:, up + 2]), f"{name}: the two half-block words of a block differ"

    bl = bf.make_blend(dict(means2D=v["means2D"], conic_opacity=v["conic_opacity"], rgb=v["rgb"], ranges=v["ranges"], point_list=v["point_list"]),
                       sc.width, sc.height, sc.tanfovx, sc.tanfovy, sc.bg.numpy(), False, False, device=DEV)
    last = bf.forward(bl)["n_contrib"][0].reshape(-1)
    chunk_base = v["chunk_base"].long().to(DEV)
    hm = v["hitmask"].long().to(DEV) & 0xFFFFFFFF
    tiles = torch.nonzero(bl.ranges[:, 1] > bl.ranges[:, 0]).flatten()
    for t in tiles.tolist():
        tt = torch.tensor([t], device=DEV)
        L = int(bl.ranges[t, 1] - bl.ranges[t, 0])
        _, _, inside, pix = bf._pixels(bl, tt)
        e = bf._pairs(bl, tt, L, last=torch.where(inside, last[pix], torch.zeros_like(pix)))
        take = (e["contrib"] & ~e["amb"])[0]                                   # [256 pixels, L]
        loc, pos = torch.nonzero(take, as_tuple=True)
        if loc.numel() == 0:
            continue
        slot = ((loc // 16) // 4) * 2 + (loc % 16) // 8                      # the pixel's own 8x4 half
        other = torch.where((slot // 2) % 2 == 0, slot + 2, slot - 2)          # the other half of its 8x8 block
        word = (chunk_base[t] + pos // 32) * 8
        for s in (slot, other):
            bit = (hm[word + s] >> (pos % 32)) & 1
            bad = torch.nonzero(bit == 0).flatten()
            assert bad.numel() == 0, (f"{name}: tile {t}: list entry {int(pos[bad[0]])} taken at tile pixel {int(loc[bad[0]])} "
                                      f"but clear in hit-mask slot {int(s[bad[0]])} ({bad.numel()} such pairs)")


@pytest.mark.parametrize("coord,depth", VARIANTS, ids=["none", "depth", "coord", "both"])
def test_forward_block_halves(coord, depth):
    sc = _scene()
    name = _name("fwd_pairs", coord, depth)
    v, _, _ = _run(sc, coord, depth, 0.0, name)
    n = (v["ranges"][:, 1] - v["ranges"][:, 0]).cpu().numpy()
    assert n[0] == 301, "tile 0 must hold exactly its own entries"
    assert n[7] > 256, "the wall tile's list must run past the first round"
    nc = v["n_contrib"][0].cpu().numpy()
    up, low = nc[0:4, 48:56].max(), nc[4:8, 48:56].max()
    assert up < 120 < low, f"the halves of tile 3's block 0 must end at different list positions: {up} {low}"
    assert nc[:, 112:128].max() <= 10, "every pixel of the wall tile must saturate behind the walls"
    _check_ballots(sc, coord, depth, name)


@pytest.mark.parametrize("coord,depth", VARIANTS, ids=["none", "depth", "coord", "both"])
@pytest.mark.parametrize("W,H,P,seed", [(48, 20, 300, 51), (40, 12, 200, 52), (44, 40, 400, 53)], ids=["48x20", "40x12", "44x40"])
def test_forward_blocks_partly_outside(W, H, P, seed, coord, depth):
    """H = 20 and H = 12: a block row with its lower half (partly) outside the image; W = 44: the last block column has
    4 of its 8 columns inside."""
    sc = bs.tiny(W, H, P, seed)
    name = _name(f"fwd_pairs_{W}x{H}", coord, depth)
    _run(sc, coord, depth, 0.0, name)
    _check_ballots(sc, coord, depth, name)

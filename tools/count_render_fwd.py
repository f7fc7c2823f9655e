"""Count the work of the forward blend (render_forward_kernel, rgs_render_fwd.cu) at a bench config, from the hit-mask words one
forward stores: the (warp, hit) pairs its ffs loops walk and the (warp, 32-entry chunk) box tests its warps run.

A warp stores its ballot (the staged entries its box test kept) for every chunk it tests.  A build with 8x4 blocks stores one word
per 8x4 block (8 warps per tile); a build with 8x8 blocks stores its 4 warps' words twice, into the slots of both 8x4 halves, so
only the upper halves' slots 0, 1, 4, 5 are counted.  Counted per warp:
  pairs        bits set in the words it stored: the hits that enter its ffs loop (a warp that stops mid-chunk is counted to the
               end of that chunk);
  chunk tests  between the chunks up to its last nonzero word (it tested at least those) and all chunks of the tile's list
               (a warp with an unsaturated pixel tests them all).

Usage: python tools/count_render_fwd.py --layout 8x8 [--config C2] [--package DIR]
  --package  the directory holding `diff_gaussian_rasterization` and `rade_gs_b200` of the build to count (default: this tree's)
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def popcount32(x):
    """bits set per element of an int64 tensor holding 32-bit words"""
    x = x & 0xFFFFFFFF
    n = x.new_zeros(x.shape)
    for b in range(32):
        n += (x >> b) & 1
    return n


def counts(v, layout):
    import torch
    ranges = v["ranges"].long()
    n = (ranges[:, 1] - ranges[:, 0]).clamp(min=0)
    tiles = n.numel()
    dev = n.device
    nch = (n + 31) // 32
    t_of = torch.repeat_interleave(torch.arange(tiles, device=dev), nch)
    k = torch.arange(t_of.numel(), device=dev) - torch.repeat_interleave(torch.cumsum(nch, 0) - nch, nch)
    words = v["hitmask"].long().view(-1, 8)[v["chunk_base"].long()[t_of] + k] & 0xFFFFFFFF  # [chunk, slot]
    slots = [0, 1, 2, 3, 4, 5, 6, 7] if layout == "8x4" else [0, 1, 4, 5]
    w = words[:, slots]
    pairs = int(popcount32(w).sum().item())
    # last chunk with a nonzero word, per (tile, warp)
    kk = torch.where(w != 0, k[:, None].expand_as(w), torch.full_like(w, -1))
    last = torch.full((tiles, len(slots)), -1, dtype=torch.int64, device=dev)
    last.scatter_reduce_(0, t_of[:, None].expand_as(kk), kk, reduce="amax")
    tests_lo = int((last + 1).sum().item())
    tests_hi = int((nch * len(slots)).sum().item())
    live = int((n > 0).sum().item())
    return {"layout": layout, "warps_per_tile": len(slots), "tiles": tiles, "tiles_with_splats": live, "instances": int(n.sum().item()),
            "pairs": pairs, "pairs_per_tile": pairs / max(live, 1), "chunk_tests_min": tests_lo, "chunk_tests_max": tests_hi}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layout", choices=["8x4", "8x8"], required=True, help="the pixel-block layout of the build being counted")
    ap.add_argument("--config", default="C2")
    ap.add_argument("--package", default=os.path.join(ROOT, "rade-gs_b200"))
    a = ap.parse_args()
    for p in (ROOT, a.package):
        if p not in sys.path:
            sys.path.insert(0, p)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("count_render_fwd.py needs a CUDA device: the rasterizer has no CPU path")
    import diff_gaussian_rasterization as dgr
    from rade_gs_b200 import rawapi, scenes
    sc_cpu, coord, depth = scenes.make_config(a.config)
    sc = sc_cpu.to(torch.device("cuda:0"))
    f = rawapi.forward(dgr._C, sc, coord, depth)
    c = counts(rawapi.ours_views(f, sc), a.layout)
    torch.cuda.synchronize()
    print(json.dumps({"config": a.config, "W": sc.width, "H": sc.height, "require_depth": depth, "require_coord": coord,
                      "package": os.path.relpath(os.path.abspath(a.package), ROOT), **c}), flush=True)


if __name__ == "__main__":
    main()

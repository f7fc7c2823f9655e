"""Time the backward blend (render_backward_kernel, rgs_render_bwd.cu) at a bench config and count the (warp, hit) pairs it
walks, for the two pixel-block layouts the kernel can give a warp.

A warp of the backward blend walks the tile list from the back and runs its per-hit body for every list entry whose bit is
set in the hit mask forward-render stored for its pixel block, up to the last contributor of any pixel of the block.  The
forward stores one ballot word per 32 list entries per 8x4 half-block: the ballot of the 8x8 block holding it (a build whose
forward warps own 8x4 blocks stores each half's own ballot).  Counted from the buffers one forward leaves:
  8x4   one warp per 8x4 block (32 pixels, one per lane): the half's word, cut at the half's max(n_contrib);
  8x8   one warp per 8x8 block (64 pixels, two per lane): the OR of the words of its two 8x4 halves, cut at the 64-pixel max.
With the 8x8 forward the 8x4 count uses 8x8 ballots, so it is not what an 8x4 backward walked after an 8x4 forward.
Each counted pair moves its 16-float gradient row through the warp's shared-memory transpose: every lane stores 64 B and the
flush reads them back, 4 KB per pair in either layout, so per pixel-hit the 8x8 layout moves half the bytes.

The stage time is the library's own CUDA-event timing of the render_backward stage (`stage_timing`, as bench.py reports it),
averaged over --launches forward+backward steps after --warmup.  Prints one JSON line, with the card name, power limit and SM
clocks read in the same run.

Usage: python tools/bench_render_bwd.py [--config C2] [--launches 100] [--warmup 5]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "rade-gs_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

TRANSPOSE_BYTES_PER_PAIR = 32 * 64 * 2  # 32 lanes store 16 floats each, the flush reads them back


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, power, sm, sm_max = [x.strip() for x in out.splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # the timing below stands without it, labelled so
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"not read ({type(e).__name__})"}


def popcount32(x):
    """bits set per element of an int64 tensor holding 32-bit words"""
    x = x & 0xFFFFFFFF
    n = torch.zeros_like(x)
    for b in range(32):
        n += (x >> b) & 1
    return n


def pair_counts(v, W, H):
    """(warp, hit) pairs the backward blend walks with 8x4 and with 8x8 pixel blocks, from one forward's buffers."""
    dev = v["ranges"].device
    ranges = v["ranges"].long()
    n = (ranges[:, 1] - ranges[:, 0]).clamp(min=0)
    tiles = n.numel()
    gx, gy = (W + 15) // 16, (H + 15) // 16
    # last contributor per 8x4 block: [tile, forward warp w] with w = 2 * (row block) + (column block)
    nc = torch.zeros(gy * 16, gx * 16, dtype=torch.int64, device=dev)
    nc[:H, :W] = v["n_contrib"][0].long()
    last84 = nc.view(gy, 4, 4, gx, 2, 8).amax(dim=(2, 5)).permute(0, 2, 1, 3).reshape(tiles, 8)
    # the 8x8 block (row pair r, column c) joins forward warps 4 r + c and 4 r + c + 2
    top = torch.tensor([0, 1, 4, 5], device=dev)
    last88 = torch.maximum(last84[:, top], last84[:, top + 2])

    nch = (n + 31) // 32
    t_of = torch.repeat_interleave(torch.arange(tiles, device=dev), nch)
    k = torch.arange(t_of.numel(), device=dev) - torch.repeat_interleave(torch.cumsum(nch, 0) - nch, nch)
    words = v["hitmask"].long().view(-1, 8)[v["chunk_base"].long()[t_of] + k]  # [chunk, forward warp]

    def kept(w, last):
        lim = (last - 32 * k[:, None]).clamp(0, 32)  # bit b of word k <-> list position 32 k + b
        return popcount32(w & ((1 << lim) - 1)).sum().item()

    p84 = kept(words, last84[t_of])
    p88 = kept(words[:, top] | words[:, top + 2], last88[t_of])
    live = int((n > 0).sum().item())
    return {"tiles": tiles, "tiles_with_splats": live, "instances": int(n.sum().item()),
            "pairs_8x4": p84, "pairs_8x8": p88, "pairs_ratio_8x8_over_8x4": p88 / max(p84, 1),
            "pairs_per_tile_8x4": p84 / max(live, 1), "pairs_per_tile_8x8": p88 / max(live, 1),
            "transpose_bytes_per_pair": TRANSPOSE_BYTES_PER_PAIR,
            "transpose_bytes_per_pixel_hit_8x4": TRANSPOSE_BYTES_PER_PAIR / 32, "transpose_bytes_per_pixel_hit_8x8": TRANSPOSE_BYTES_PER_PAIR / 64,
            "transpose_MB_8x4": p84 * TRANSPOSE_BYTES_PER_PAIR / 1e6, "transpose_MB_8x8": p88 * TRANSPOSE_BYTES_PER_PAIR / 1e6}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2")
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_render_bwd.py needs a CUDA device: the rasterizer has no CPU path")
    import diff_gaussian_rasterization as dgr
    from rade_gs_b200 import rawapi, scenes
    C = dgr._C
    dev = torch.device("cuda:0")
    sc_cpu, coord, depth = scenes.make_config(a.config)
    sc = sc_cpu.to(dev)
    grads = scenes.make_upstream_grads(sc.height, sc.width, device=dev)

    def step():
        f = rawapi.forward(C, sc, coord, depth)
        return f, rawapi.backward(C, sc, f, grads)

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    C.stage_timing(True)
    for _ in range(a.launches):
        step()
    torch.cuda.synchronize()
    stages = C.stage_times()
    C.stage_timing(False)
    tot, cnt = stages["render_backward"]

    f = rawapi.forward(C, sc, coord, depth)
    counts = pair_counts(rawapi.ours_views(f, sc), sc.width, sc.height)
    torch.cuda.synchronize()
    print(json.dumps({"config": a.config, "W": sc.width, "H": sc.height, "require_depth": depth, "require_coord": coord,
                      "render_backward_ms": tot / max(cnt, 1), "launches": cnt,
                      "stage_ms": {k: t / max(c, 1) for k, (t, c) in stages.items()}, "counts": counts, "device": card()}), flush=True)


if __name__ == "__main__":
    main()

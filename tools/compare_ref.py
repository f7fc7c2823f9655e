"""GPU-side parity report: this build vs the reference build (oracle/_ref/ref_dgr_C.so) on the same inputs.

Needs a GPU:  python tools/compare_ref.py [--cfg small|C1|C2|C3] [--ks 0.0] [--coord 0/1] [--depth 0/1] [--time]
Prints exact-match counts for the integer contract (radii, num_rendered, sorted ids, tile ranges, n_contrib) and
error statistics for images / gradients.  Test infrastructure, not product.
"""
from __future__ import annotations

import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import torch  # noqa: E402

from rade_gs_b200 import rawapi, scenes  # noqa: E402


def stats(name, a, b, mask=None):
    a, b = a.float(), b.float()
    if mask is not None:
        a, b = a[mask], b[mask]
    if a.numel() == 0:
        print(f"  {name:14s} empty")
        return
    d = (a - b).abs()
    bad = torch.isnan(a) != torch.isnan(b)
    d = torch.nan_to_num(d, nan=0.0)
    rel = d.norm() / (b.nan_to_num().norm() + 1e-30)
    print(f"  {name:14s} max|d|={d.max().item():.3e}  mean|d|={d.mean().item():.3e}  relL2={rel.item():.3e}  max|ref|={b.nan_to_num().abs().max().item():.3e}"
          f"  nan-mismatch={int(bad.sum())}  frac>1e-4={(d > 1e-4 + 1e-4 * b.abs()).float().mean().item():.2e}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg", default="small")
    ap.add_argument("--ks", type=float, default=0.0)
    ap.add_argument("--coord", type=int, default=-1)
    ap.add_argument("--depth", type=int, default=-1)
    ap.add_argument("--time", action="store_true")
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()

    import build_ref
    import diff_gaussian_rasterization as dgr
    ours, ref = dgr._C, build_ref.load()

    dev = torch.device("cuda:0")
    if a.cfg == "small":
        sc = scenes.make_scene(20000, 320, 240, 300.0, -3.6, view=scenes.look_at_view((0.4, -0.3, -0.5), (0.1, 0.05, 6.0)), bg=(0.1, 0.2, 0.3))
        coord, depth = False, True
    else:
        sc, coord, depth = scenes.make_config(a.cfg)
    if a.coord >= 0:
        coord = bool(a.coord)
    if a.depth >= 0:
        depth = bool(a.depth)
    sc = sc.to(dev)
    grads = scenes.make_upstream_grads(sc.height, sc.width, device=dev)
    print(f"cfg={a.cfg} P={sc.means3D.shape[0]} {sc.width}x{sc.height} coord={coord} depth={depth} ks={a.ks}")

    fo = rawapi.forward(ours, sc, coord, depth, kernel_size=a.ks)
    fr = rawapi.forward(ref, sc, coord, depth, kernel_size=a.ks)
    torch.cuda.synchronize()
    print(f"num_rendered ours={fo['num_rendered']} ref={fr['num_rendered']}")
    vo, vr = rawapi.ours_views(fo, sc), rawapi.ref_views(fr, sc)
    print("integer contract:")
    print("  radii mismatches      :", int((fo["radii"] != fr["radii"]).sum()), "of", fo["radii"].numel(), " visible:", int((fr["radii"] > 0).sum()))
    vis = fr["radii"] > 0
    both = vis & (fo["radii"] > 0)
    print("  tiles_touched mismatch:", int((vo["tiles_touched"] != vr["tiles_touched"]).sum()))
    print("  depth bits mismatch   :", int((vo["depths"][both].view(torch.int32) != vr["depths"][both].view(torch.int32)).sum()))
    print("  means2D bits mismatch :", int((vo["means2D"][both].contiguous().view(torch.int32) != vr["means2D"][both].contiguous().view(torch.int32)).sum()))
    if fo["num_rendered"] == fr["num_rendered"]:
        print("  sorted ids mismatch   :", int((vo["point_list"] != vr["point_list"]).sum()), "of", fo["num_rendered"])
        print("  sorted keys mismatch  :", int((vo["keys"] != vr["keys"]).sum()))
        print("  tile ranges mismatch  :", int((vo["ranges"] != vr["ranges"]).sum()))
    nc = (vo["n_contrib"] != vr["n_contrib"])
    print("  n_contrib mismatch    : last", int(nc[0].sum()), " median", int(nc[1].sum()), "of", nc[0].numel())
    print("preprocess (visible only):")
    for k in ("conic_opacity", "rgb", "ts", "ray_planes", "normals"):
        stats(k, vo[k], vr[k], both)
    if coord:
        stats("camera_planes", vo["camera_planes"], vr["camera_planes"], both)
        stats("view_points", vo["view_points"], vr["view_points"], both)
    print("  clamped mismatch      :", int(((vo["clamped"][both][:, None] >> torch.arange(3, device=dev)) & 1 != vr["clamped"][both]).sum()))
    print("images:")
    for k in ("color", "alpha", "depth", "mdepth", "normal", "coord", "mcoord"):
        stats(k, fo[k], fr[k])

    bo = rawapi.backward(ours, sc, fo, grads)
    br = rawapi.backward(ref, sc, fr, grads)
    br2 = rawapi.backward(ref, sc, fr, grads)
    torch.cuda.synchronize()
    print("gradients (ours vs ref; then ref vs ref run-to-run):")
    for k in rawapi.BWD_KEYS:
        stats(k, bo[k], br[k])
    for k in ("means3D", "scales"):
        stats("ref/ref " + k, br2[k], br[k])

    if a.time:
        def timeit(C):
            ts = []
            for it in range(a.iters + 3):
                torch.cuda.synchronize()
                e0, e1, e2 = torch.cuda.Event(True), torch.cuda.Event(True), torch.cuda.Event(True)
                e0.record()
                f = rawapi.forward(C, sc, coord, depth, kernel_size=a.ks)
                e1.record()
                rawapi.backward(C, sc, f, grads)
                e2.record()
                torch.cuda.synchronize()
                if it >= 3:
                    ts.append((e0.elapsed_time(e1), e1.elapsed_time(e2)))
            f = sorted(t[0] for t in ts)[len(ts) // 2]
            b = sorted(t[1] for t in ts)[len(ts) // 2]
            return f, b
        fo_t, bo_t = timeit(ours)
        fr_t, br_t = timeit(ref)
        mp = sc.width * sc.height / 1e6
        print(f"time ours fwd {fo_t:.3f} ms bwd {bo_t:.3f} ms -> {mp / ((fo_t + bo_t) * 1e-3):.1f} Mpix/s")
        print(f"time ref  fwd {fr_t:.3f} ms bwd {br_t:.3f} ms -> {mp / ((fr_t + br_t) * 1e-3):.1f} Mpix/s")
        print(f"speedup fwd {fr_t / fo_t:.2f}x bwd {br_t / bo_t:.2f}x total {(fr_t + br_t) / (fo_t + bo_t):.2f}x")


if __name__ == "__main__":
    main()

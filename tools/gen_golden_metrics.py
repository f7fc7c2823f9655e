"""Generate tests/golden/metrics/lpips.npz from the REFERENCE'S OWN lpipsPyTorch and metric.py (on CPU; the reference
checkout beside the repository, or $RADE_GS_REFERENCE).

The two downloads are replaced by seeded weights, the modules are imported unmodified:
  * torchvision.models.vgg16(weights=IMAGENET1K_V1) becomes vgg16(weights=None) filled with tests/lpips_f64.seeded_weights;
  * torch.hub.load_state_dict_from_url returns the seeded lin0..lin4 heads of the same set.
`.cuda()` means the CPU for the duration of the run (the shim of tools/gen_golden_fused.py).

Stored: the seed and the SHA-256 of the regenerated weights (never the weights); eight image pairs; per pair the five
layer means and the total of lpipsPyTorch.lpips in fp32 and of the same modules converted to fp64; and the results.json /
per_view.json that metric.py's evaluate() writes for a scene/test/ours_1/{renders,gt} tree of the pairs that are exact
8-bit images (their PNGs are rebuilt from the stored arrays by the tests).

    python tools/gen_golden_metrics.py
"""
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("RADE_GS_REFERENCE") or os.path.join(os.path.dirname(ROOT), "reference")
sys.path[:0] = [os.path.join(ROOT, "tests", "ref_stubs"), os.path.join(ROOT, "tests"), REF]
torch.Tensor.cuda = lambda self, *a, **k: self            # noqa: E731  CPU run of code that says .cuda()
torch.nn.Module.cuda = lambda self, *a, **k: self         # noqa: E731

import torchvision                                        # noqa: E402
from PIL import Image                                     # noqa: E402

import lpips_f64                                          # noqa: E402

SEED = 20261017
WEIGHTS = lpips_f64.seeded_weights(SEED)
_vgg16 = torchvision.models.vgg16


def _seeded_vgg16(*a, **k):
    m = _vgg16(weights=None)
    m.features.load_state_dict({k[len("features."):]: v for k, v in WEIGHTS.items() if k.startswith("features.")})
    return m


def _seeded_heads(url, *a, **k):
    assert url.endswith("/v0.1/vgg.pth"), url
    return {k: v.clone() for k, v in WEIGHTS.items() if k.startswith("lin")}


torchvision.models.vgg16 = _seeded_vgg16
torch.hub.load_state_dict_from_url = _seeded_heads

from lpipsPyTorch import lpips                            # noqa: E402
from lpipsPyTorch.modules.lpips import LPIPS              # noqa: E402
import metric                                             # noqa: E402


def pairs():
    g = np.random.default_rng(7)
    q = lambda a: np.round(a * 255) / 255                 # noqa: E731  render.py's 8-bit PNG
    out = []
    for h, w in [(16, 16), (17, 31), (64, 48), (97, 53)]:
        x = g.random((3, h, w))
        out.append((f"rand_{h}x{w}", x, np.clip(x + g.normal(0, 0.1, x.shape), 0, 1), False))
    x = q(g.random((3, 40, 33)))
    out.append(("identical_40x33", x, x.copy(), True))
    out.append(("saturated_24x20", (g.random((3, 24, 20)) < 0.5) * 1.0, (g.random((3, 24, 20)) < 0.5) * 1.0, True))
    for h, w in [(48, 64), (33, 57)]:
        yy, xx = np.mgrid[0:h, 0:w]
        base = 0.5 + 0.4 * np.sin(xx[None] / 5.0 + np.arange(3)[:, None, None]) * np.cos(yy[None] / 7.0)
        out.append((f"quantized_{h}x{w}", q(np.clip(base + g.normal(0, 0.03, (3, h, w)), 0, 1)), q(base), True))
    return [(n, x.astype(np.float32), y.astype(np.float32), png) for n, x, y, png in out]


def layer_means(crit, x, y):
    got = []
    hooks = [lin.register_forward_hook(lambda mod, i, o: got.append(o.mean((2, 3)).reshape(()))) for lin in crit.lin]
    total = crit(x, y).reshape(())
    for h in hooks:
        h.remove()
    return torch.stack(got).numpy(), total.numpy()


def main():
    torch.set_num_threads(8)
    data = {"seed": np.int64(SEED), "digest": np.array(lpips_f64.digest(WEIGHTS))}
    crit64 = LPIPS("vgg", "0.1").double()
    names = []
    for n, x, y, png in pairs():
        tx, ty = torch.from_numpy(x)[None], torch.from_numpy(y)[None]
        total32 = lpips(tx, ty, net_type="vgg").reshape(()).numpy()
        m32, t32 = layer_means(LPIPS("vgg", "0.1"), tx, ty)
        assert t32 == total32
        m64, t64 = layer_means(crit64, tx.double(), ty.double())
        data.update({f"{n}/x": x, f"{n}/y": y, f"{n}/png": np.bool_(png), f"{n}/layers_f32": m32, f"{n}/total_f32": t32,
                     f"{n}/layers_f64": m64, f"{n}/total_f64": t64})
        names.append(n)
        print(f"{n:20s} f32 {float(t32):.9g}  f64 {float(t64):.17g}")
    data["names"] = np.array(names)
    with tempfile.TemporaryDirectory() as tmp:
        scene = os.path.join(tmp, "scene")
        for sub in ("renders", "gt"):
            os.makedirs(os.path.join(scene, "test", "ours_1", sub))
        for n, x, y, png in pairs():
            if png:
                for sub, a in (("renders", x), ("gt", y)):
                    Image.fromarray(np.round(a.transpose(1, 2, 0) * 255).astype(np.uint8)).save(os.path.join(scene, "test", "ours_1", sub, n + ".png"))
        metric.evaluate([scene])
        for f in ("results.json", "per_view.json"):
            with open(os.path.join(scene, f)) as fp:
                data[f] = np.array(fp.read())
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "metrics", "lpips.npz"), **data)


if __name__ == "__main__":
    main()

"""Generate tests/golden/fused_appearance.npz from the REFERENCE'S OWN `L1_loss_appearance` (on CPU; the reference checkout beside
the repository, or $RADE_GS_REFERENCE).

train.py cannot be imported here (tensorboard, matplotlib and the renderer at module level), so the function is taken out of it:
the file is parsed and that one `def` is executed, with `torch` and utils/loss_utils.py's `l1_loss` in its namespace.  The
network is scene/appearance_network.py's AppearanceNetwork, imported as it is.  Each case runs in float32 and again in float64
(the arbiter for tolerances; stored as a float32 residual against the float32 run) and records the loss, d_image, d(embedding
row), every parameter's gradient and the transformed image, as tests/appearance_f64.recorded keeps them: the head's weight
gradients and the transformed image at fixed sample indices, to keep the file small.  The inputs are
regenerated from seeds by tests/appearance_f64.make_inputs; the fixture stores their digest.

    python tools/gen_golden_appearance.py
"""
import ast
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("RADE_GS_REFERENCE") or os.path.join(os.path.dirname(ROOT), "reference")
sys.path[:0] = [os.path.join(ROOT, "tests", "ref_stubs"), os.path.join(ROOT, "tests"), REF]
torch.Tensor.cuda = lambda self, *a, **k: self            # noqa: E731  CPU run of code that says .cuda()
torch.nn.Module.cuda = lambda self, *a, **k: self         # noqa: E731

from scene.appearance_network import AppearanceNetwork    # noqa: E402
from utils.loss_utils import l1_loss                      # noqa: E402
import appearance_f64 as af                               # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "fused_appearance.npz")


def reference_function():
    src = open(os.path.join(REF, "train.py")).read()
    tree = ast.parse(src)
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "L1_loss_appearance")
    ns = {"torch": torch, "l1_loss": l1_loss}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), os.path.join(REF, "train.py"), "exec"), ns)
    return ns["L1_loss_appearance"]


def run(fn, inp, dtype):
    net = AppearanceNetwork(3 + 64, 3).to(dtype)
    with torch.no_grad():
        for p, v in zip(net.parameters(), inp["params"]):
            p.copy_(torch.from_numpy(v))
    table = torch.nn.Parameter(torch.from_numpy(inp["table"]).to(dtype))
    gaussians = SimpleNamespace(appearance_network=net, get_apperance_embedding=lambda i: table[i])
    image = torch.from_numpy(inp["image"]).to(dtype).requires_grad_(True)
    gt = torch.from_numpy(inp["gt"]).to(dtype)
    loss = fn(image, gt, gaussians, af.VIEW_IDX)
    loss.backward()
    with torch.no_grad():
        transformed = fn(image, gt, gaussians, af.VIEW_IDX, return_transformed_image=True)
    out = {"loss": loss.detach().numpy(), "d_image": image.grad.numpy(), "d_emb": table.grad[af.VIEW_IDX].numpy(),
           "transformed": af.recorded("transformed", transformed.numpy())}
    assert not table.grad[[i for i in range(table.shape[0]) if i != af.VIEW_IDX]].any()
    for name, p in zip(af.PARAM_NAMES, net.parameters()):
        out["g_" + name] = af.recorded(name, p.grad.numpy())
    return out


def main():
    fn = reference_function()
    torch.set_num_threads(4)
    data = {}
    for case in af.CASES:
        inp = af.make_inputs(case)
        data[case + "/digest"] = np.array(af.inputs_digest(inp))
        for dtype, suf in ((torch.float32, ""), (torch.float64, "_f64")):
            for k, v in run(fn, inp, dtype).items():
                if suf:  # float64 as a float32 residual against the float32 run: exact to ~1e-14 relative, half the bytes
                    data[f"{case}/{k}_f64d"] = (v - data[f"{case}/{k}"].astype(np.float64)).astype(np.float32)
                else:
                    data[f"{case}/{k}"] = v
    np.savez_compressed(OUT, **data)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()

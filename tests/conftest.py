"""Shared test plumbing.  `-m "not gpu"` runs without a GPU; `-m gpu` needs an H100."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tools"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
_ALL_GOLDEN = sorted(f[:-4] for f in os.listdir(GOLDEN_DIR) if f.endswith(".npz")) if os.path.isdir(GOLDEN_DIR) else []
GOLDEN_CASES = [c for c in _ALL_GOLDEN if not c.startswith(("integrate_", "fused_", "refbuild_"))]  # rasterize fwd/bwd (tools/gen_golden.py)
INTEGRATE_CASES = [c for c in _ALL_GOLDEN if c.startswith("integrate_")]        # integrate (tools/gen_golden_integrate.py)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """Plain `pytest tests` on a box without a CUDA device: GPU tests are skipped, not errors.  (On a GPU box nothing is
    skipped here -- and the product itself still fails loudly without its extension, see tests/test_abi_host.py.)"""
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (run with -m gpu on an H100)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    """A fixture as a dict of arrays.  Fixtures made from seeded scenes store a digest of their inputs instead of the inputs:
    those are regenerated (tools/golden_inputs.py) and must match it bit for bit."""
    d = dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz")))
    if "inputs_digest" in d:
        import golden_inputs
        inputs = golden_inputs.inputs_of(name)
        assert golden_inputs.digest(inputs) == str(d.pop("inputs_digest")), f"{name}: the regenerated inputs differ from the fixture's"
        d.update(inputs)
    return d


def golden_oracle_inputs(d):
    """oracle.Inputs for a golden fixture."""
    import oracle
    kw = {}
    if "in_colors_precomp" in d:
        kw["colors_precomp"] = d["in_colors_precomp"]
    else:
        kw["shs"] = d["in_shs"]
    if "in_cov3D_precomp" in d:
        kw["cov3D_precomp"] = d["in_cov3D_precomp"]
    else:
        kw["scales"], kw["rotations"] = d["in_scales"], d["in_rotations"]
    return oracle.Inputs(d["in_means3D"], d["in_opacities"], d["in_viewmatrix"], d["in_projmatrix"], d["in_campos"], d["in_bg"],
                         int(d["meta_W"]), int(d["meta_H"]), float(d["in_tanfov"][0]), float(d["in_tanfov"][1]), sh_degree=int(d["meta_deg"]),
                         kernel_size=float(d["meta_ks"]), require_coord=bool(d["meta_coord"]), require_depth=bool(d["meta_depth"]), **kw)


def integrate_oracle_inputs(d):
    """oracle.Inputs for an integrate fixture: kernel_size 0, SH truncated to the fixture's degree (as the generator passed it)."""
    import oracle
    M = (int(d["meta_deg"]) + 1) ** 2
    return oracle.Inputs(d["in_means3D"], d["in_opacities"], d["in_viewmatrix"], d["in_projmatrix"], d["in_campos"], d["in_bg"],
                         int(d["meta_W"]), int(d["meta_H"]), float(d["in_tanfov"][0]), float(d["in_tanfov"][1]), sh_degree=int(d["meta_deg"]),
                         kernel_size=0.0, require_coord=True, require_depth=True, shs=np.ascontiguousarray(d["in_shs"][:, :M]),
                         scales=d["in_scales"], rotations=d["in_rotations"])


def golden_upstream(d):
    return {k: d["gin_" + k] for k in ("color", "coord", "mcoord", "depth", "mdepth", "alpha", "normal")}


@pytest.fixture(params=GOLDEN_CASES)
def golden(request):
    return request.param, load_golden(request.param)

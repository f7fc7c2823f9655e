"""Inputs of the golden fixtures under tests/golden/, regenerated from their seeds.

The rasterize fixtures (tools/gen_golden.py) and the integrate fixtures (tools/gen_golden_integrate.py) are made from seeded
synthetic scenes.  They store the reference's outputs and only a SHA-256 of their inputs (`inputs_digest`): the inputs are
rebuilt here by the same case builders, and tests/conftest.py:load_golden() checks them against the digest before a test
sees them.  The scene synthesis runs on one CPU thread (rade_gs_b200.scenes), so the bits do not depend on the host's core
count; they could still depend on the CPU's vector instruction set, which the digest check would report.
"""
from __future__ import annotations

import hashlib

import numpy as np

SCENE_KEYS = ("means3D", "scales", "rotations", "opacities", "shs", "viewmatrix", "projmatrix", "campos", "bg")


def digest(arrays: dict) -> str:
    h = hashlib.sha256()
    for k in sorted(arrays):
        h.update(k.encode())
        h.update(np.ascontiguousarray(arrays[k]).tobytes())
    return h.hexdigest()


def rasterize_inputs(name: str) -> dict:
    """in_* (scene, precomputed colours / covariances) and gin_* (upstream gradients) of a gen_golden.py case."""
    import gen_golden
    from rade_gs_b200 import scenes
    c = gen_golden.CASES[name]
    sc, extra = gen_golden.build_case(c)
    rec = {"in_" + k: getattr(sc, k).numpy() for k in SCENE_KEYS}
    rec.update({"in_" + k: v.numpy() for k, v in extra.items()})
    rec.update({"gin_" + k: v.numpy() for k, v in scenes.make_upstream_grads(sc.height, sc.width, seed=4321 + c["seed"]).items()})
    return rec


def integrate_inputs(name: str) -> dict:
    """in_* (scene and query points) of a gen_golden_integrate.py case."""
    import gen_golden_integrate
    sc, pts = gen_golden_integrate.build_case(gen_golden_integrate.CASES[name])
    rec = {"in_" + k: getattr(sc, k).numpy() for k in SCENE_KEYS}
    rec["in_points3D"] = pts.numpy()
    return rec


def inputs_of(name: str) -> dict:
    return integrate_inputs(name) if name.startswith("integrate_") else rasterize_inputs(name)

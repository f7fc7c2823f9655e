"""Call sites of `diff_gaussian_rasterization` in the reference's own caller, `gaussian_renderer.render()` (reference
gaussian_renderer/__init__.py:19-95), extracted once into tests/golden/render_call_sites.json for tests/test_dropin_static.py:
the names it imports, the keywords it passes to `GaussianRasterizationSettings(...)`, `rasterizer(...)` and `.integrate(...)`,
and how many outputs it unpacks from the rasterizer call.

Usage:  python tools/gen_golden_callsites.py <reference checkout>/gaussian_renderer/__init__.py
"""
from __future__ import annotations

import ast
import json
import os
import sys

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "render_call_sites.json")


def extract(src: str) -> dict:
    tree = ast.parse(src)
    calls = {"settings": [], "rasterizer": [], "integrate": []}
    for node in ast.walk(tree):
        if not isinstance(node, ast.Call):
            continue
        kws = sorted(k.arg for k in node.keywords)
        if isinstance(node.func, ast.Name) and node.func.id == "GaussianRasterizationSettings":
            calls["settings"].append(kws)
        elif isinstance(node.func, ast.Name) and node.func.id == "rasterizer":
            calls["rasterizer"].append(kws)
        elif isinstance(node.func, ast.Attribute) and node.func.attr == "integrate":
            calls["integrate"].append(kws)
    unpack = [len(n.targets[0].elts) for n in ast.walk(tree) if isinstance(n, ast.Assign) and isinstance(n.targets[0], ast.Tuple)
              and isinstance(n.value, ast.Call) and isinstance(n.value.func, ast.Name) and n.value.func.id == "rasterizer"]
    imported = [a.name for n in ast.walk(tree) if isinstance(n, ast.ImportFrom) and n.module == "diff_gaussian_rasterization" for a in n.names]
    return {"imported": imported, "calls": calls, "rasterizer_unpack": unpack}


if __name__ == "__main__":
    with open(sys.argv[1]) as f:
        facts = extract(f.read())
    with open(OUT, "w") as f:
        json.dump(facts, f, indent=1)
        f.write("\n")
    print(OUT)

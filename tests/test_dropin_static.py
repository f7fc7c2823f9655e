"""Static drop-in check against the reference's own caller, `gaussian_renderer.render()` (reference
gaussian_renderer/__init__.py:19-95): every name it imports from `diff_gaussian_rasterization`, every keyword it passes to
`GaussianRasterizationSettings(...)`, to `rasterizer(...)` and to `.integrate(...)`, and the 8-tuple it unpacks must exist in this
repo's package.  The call sites were extracted from the reference into tests/golden/render_call_sites.json
(tools/gen_golden_callsites.py)."""
import inspect
import json
import os

from conftest import GOLDEN_DIR


def test_render_call_sites_fit_our_package():
    import diff_gaussian_rasterization as dgr
    with open(os.path.join(GOLDEN_DIR, "render_call_sites.json")) as f:
        facts = json.load(f)
    imported = facts["imported"]
    assert imported and all(hasattr(dgr, name) for name in imported), imported
    fields = set(dgr.GaussianRasterizationSettings._fields)
    fwd_params = set(inspect.signature(dgr.GaussianRasterizer.forward).parameters) - {"self"}
    integ_params = set(inspect.signature(dgr.GaussianRasterizer.integrate).parameters) - {"self"}
    for kws in facts["calls"]["settings"]:
        assert kws and set(kws) <= fields, set(kws) - fields
    for kws in facts["calls"]["rasterizer"]:
        assert set(kws) <= fwd_params, set(kws) - fwd_params
    for kws in facts["calls"]["integrate"]:
        assert set(kws) <= integ_params, set(kws) - integ_params
    assert len(facts["calls"]["settings"]) >= 1 and len(facts["calls"]["rasterizer"]) >= 1
    # render() unpacks 8 outputs from the rasterizer call (reference :71)
    assert facts["rasterizer_unpack"] and facts["rasterizer_unpack"][0] == 8

"""CPU checks of densify-and-prune: the eager model (tests/densify_model.py) against the reference's own method
(tests/golden/fused_densify.npz) bit for bit, the numpy quantile model against torch.quantile, and the wrapper's rejections."""
import os

import numpy as np
import pytest
import torch

import densify_model as dm
from conftest import GOLDEN_DIR

FIXTURE = dm.load_fixture(os.path.join(GOLDEN_DIR, "fused_densify.npz"))


@pytest.mark.parametrize("case", sorted(FIXTURE))
def test_model_reproduces_the_reference_bit_for_bit(case):
    d = FIXTURE[case]
    m = dm.from_fixture(d, "cpu")
    with dm.replay([d["draw_clone"], d["draw_split"]]):
        result, sel = dm.densify_and_prune(m, *dm.arguments(d))
    assert result == tuple(d["result"])
    assert np.array_equal(sel["clone"].numpy(), d["clone"]) and np.array_equal(sel["split"].numpy(), d["split"])
    assert np.array_equal(sel["Q"].numpy(), d["Q"], equal_nan=True) and sel["ratio"].numpy() == d["ratio"]
    got = dm.state_of(m)
    want = {k[4:]: v for k, v in d.items() if k.startswith("out_") and k[4:] in got}
    assert sorted(got) == sorted(want)
    for k, v in want.items():
        assert got[k].shape == v.shape and np.array_equal(got[k], v), k
    for k in ("xyz_gradient_accum", "xyz_gradient_accum_abs", "xyz_gradient_accum_abs_max", "denom", "max_radii2D", "filter_3D"):
        assert np.array_equal(getattr(m, k).numpy(), d["out_" + k]), k
    fresh = dm.from_fixture(d, "cpu")
    dm.reset_opacity(fresh)
    for k, v in dm.state_of(fresh).items():
        if k.startswith("opacity"):
            assert np.array_equal(v, d["reset_" + k]), k


def test_fixture_covers_the_issue_cases():
    assert {int(d["sh_degree"]) for d in FIXTURE.values()} >= {0, 3}
    assert tuple(FIXTURE["nothing_selected"]["result"][:2]) == (0, 0)
    d = FIXTURE["all_pruned"]
    assert d["out_xyz"].shape[0] == 0 and d["result"][2] == d["in_xyz"].shape[0] + d["result"][0] + d["result"][1]
    assert FIXTURE["ratio_zero"]["ratio"] == 0 and FIXTURE["ratio_one"]["ratio"] == 1
    assert "f_rest.exp_avg" not in {k[3:] for k in FIXTURE["no_state"] if k.startswith("in_")}
    assert (FIXTURE["deg3_none"]["in_denom"] == 0).any()
    # the rounding case: ATen's CUDA mean rounds differently from the CPU's, and the fixture holds the CUDA threshold too
    r = FIXTURE["ratio_rounding"]
    P = r["in_xyz"].shape[0]
    count = int(round(float(r["ratio"]) * P))
    assert dm.ratio_np(count, P, cuda=False) == r["ratio"] != dm.ratio_np(count, P, cuda=True)


def test_planted_threshold_rows_decide_as_fp32_comparisons():
    d = FIXTURE["boundary_dense"]
    # rows 0-3 have max exp(s) = 1 against dense = 0.99999999907, which is 1.0f: as fp32 comparisons they are clones, not splits
    assert float(d["percent_dense"] * d["extent"]) < 1.0 == np.float32(d["percent_dense"] * d["extent"])
    assert (d["in_scaling"][:4].max(axis=1) == 0).all() and d["clone"][:4].all() and not d["split"][:4].any()
    # rows 1-3: sigmoid(0) = 0.5 is not below min_opacity 0.5 + 2^-30 once that is rounded to fp32: row and clone both survive
    assert float(d["min_opacity"]) > 0.5 == np.float32(d["min_opacity"])
    for i in (1, 2, 3):
        assert (d["out_f_dc"] == d["in_f_dc"][i]).all(axis=(1, 2)).sum() == 2
    w = FIXTURE["boundary_world"]
    assert 0.1 * float(w["extent"]) > 1.0 == np.float32(0.1 * float(w["extent"]))
    assert not w["clone"][1:4].any() and not w["split"][1:4].any()      # rows 1-3 stay, max exp(s) = 1 is not > 1.0f
    kept = w["out_xyz"][: (~w["split"]).sum()]
    assert all((kept == w["in_xyz"][i]).all(axis=1).any() for i in (1, 2, 3))


@pytest.mark.parametrize("P", [1, 2, 3, 1000, 65537, 2 ** 20 + 7, 2 ** 24])
def test_numpy_quantile_model_matches_torch(P):
    g = torch.Generator().manual_seed(P)
    v = torch.rand(P, generator=g) * torch.randint(0, 2, (P,), generator=g)     # ties and zeros, as grads_abs has
    for q in (0.0, 1.0, 0.5, 0.123456789, float(np.float32(1) - np.float32(1) / np.float32(3)), torch.rand(1, generator=g).item()):
        qt = torch.tensor(q, dtype=torch.float32)
        assert np.array_equal(np.float32(torch.quantile(v, qt).item()), dm.quantile_np(v.numpy(), qt.numpy())), q


def test_model_quantile_follows_the_formula_beyond_torchs_limit():
    P = 2 ** 24 + 3
    g = torch.Generator().manual_seed(5)
    v = torch.rand(P, generator=g)
    for q in (0.0, 1.0, 0.3, 0.999999):
        qt = torch.tensor(q, dtype=torch.float32)
        assert np.float32(dm.quantile(v, qt).item()) == dm.quantile_np(v.numpy(), qt.numpy()), q
    with pytest.raises(RuntimeError, match="too large"):
        torch.quantile(v, torch.tensor(0.5))


def test_wrapper_rejects_cpu_models():
    from rade_gs_b200.densify import densify_and_prune, reset_opacity
    d = FIXTURE["deg0_screen20"]
    m = dm.from_fixture(d, "cpu")
    with pytest.raises(RuntimeError, match="no CPU path"):
        densify_and_prune(m, *dm.arguments(d))
    with pytest.raises(RuntimeError, match="no CPU path"):
        reset_opacity(m)
    m.optimizer.param_groups = [g for g in m.optimizer.param_groups if g["name"] != "rotation"]
    with pytest.raises(ValueError, match="no group"):
        densify_and_prune(m, *dm.arguments(d))


def test_bindings_refuse_cpu_tensors():
    from diff_gaussian_rasterization import _C
    P, f32 = 4, torch.zeros
    entries = {
        "select": [f32(P, 1), f32(P, 1), f32(P, 1), f32(P, 3), f32(P, 1), 0.0002, 0.04, 0.05, True, 20.0, 0.4],
        "plan": [torch.zeros(P, dtype=torch.uint8), torch.zeros(10, dtype=torch.int32), [0, 0, P, 0, 0], f32(P, 3)],
        "gather": [torch.zeros(P, dtype=torch.int32), torch.zeros(P, dtype=torch.int32), 0, f32(P, 3), f32(P, 4), f32(P, 3), f32(0, 3),
                   f32(0, 3), [(f32(P, 1), False)]],
        "reset_opacity": [f32(P, 3), f32(P, 1), f32(P, 1)],
    }
    assert {n for n in dir(_C._densify) if not n.startswith("_")} == set(entries)
    for name, args in entries.items():
        with pytest.raises(RuntimeError, match="CUDA"):
            getattr(_C._densify, name)(*args)


def test_c_abi_rejects_empty_models_and_null_pointers():
    import ctypes
    from conftest import ROOT
    lib = ctypes.CDLL(os.path.join(ROOT, "rade-gs_b200", "rade_gs_b200", "librgs_b200.so"))
    lib.rgs_last_error.restype = ctypes.c_char_p
    fake = ctypes.c_void_p(0x1000)   # never dereferenced: rejected before the first CUDA call
    assert lib.rgs_densify_select(ctypes.c_int32(0), *([fake] * 11), None, None, None) == -1
    assert b"no Gaussians" in lib.rgs_last_error()
    args = [ctypes.c_int32(10)] + [fake] * 11 + [None, None, None]
    args[3] = None
    assert lib.rgs_densify_select(*args) == -1 and b"null" in lib.rgs_last_error()
    assert lib.rgs_reset_opacity(ctypes.c_int32(4), fake, None, fake, fake, None) == -1

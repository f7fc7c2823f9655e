"""Densify-and-prune and reset_opacity (rade_gs_b200.densify) on the GPU: against the reference's own method
(tests/golden/fused_densify.npz, draws replayed), against the eager model (tests/densify_model.py) run on the GPU with the same seeded
draws, the quantile past torch's 2^24 limit, continuity of training after the call, reproducibility and rejections."""
import os

import numpy as np
import pytest
import torch

import densify_model as dm
from conftest import GOLDEN_DIR

pytestmark = pytest.mark.gpu
FIXTURE = dm.load_fixture(os.path.join(GOLDEN_DIR, "fused_densify.npz"))
STATS = ("xyz_gradient_accum", "xyz_gradient_accum_abs", "xyz_gradient_accum_abs_max", "denom", "max_radii2D")


def _densify():
    from rade_gs_b200 import densify
    return densify


@pytest.mark.parametrize("case", sorted(FIXTURE))
def test_kernels_against_the_reference(case):
    d = FIXTURE[case]
    m = dm.from_fixture(d, "cuda")
    with dm.replay([d["draw_clone"], d["draw_split"]]):
        result = _densify().densify_and_prune(m, *dm.arguments(d))
    assert result == tuple(d["result"])
    got = dm.state_of(m)
    want = {k[4:]: v for k, v in d.items() if k.startswith("out_") and k[4:] in got}
    assert sorted(got) == sorted(want)
    for k, v in want.items():
        assert got[k].shape == v.shape, k
        if k == "xyz":
            # new rows: the CPU build's vectorised sqrt (the quaternion norm) is not correctly rounded, CUDA's is
            n_keep, samples = _new_rows(d)
            assert np.array_equal(got[k][:n_keep], v[:n_keep])
            bound = 2.0 ** -21 * (np.abs(samples).sum(axis=1, keepdims=True) + np.abs(v[n_keep:]))
            assert (np.abs(got[k][n_keep:] - v[n_keep:]) <= bound).all()
        elif k == "scaling":
            # children: log(exp(s) * (1 / 1.6f)) with libdevice exp / log here, log(exp(s) / 1.6f) with the CPU's SLEEF there
            assert np.abs(got[k] - v).max(initial=0) <= 4e-6
            assert np.array_equal(got[k][: v.shape[0] - _children_rows(d)], v[: v.shape[0] - _children_rows(d)])
        else:
            assert np.array_equal(got[k], v), k
    for k in STATS:
        assert getattr(m, k).shape == d["out_" + k].shape and not getattr(m, k).any(), k
    assert getattr(m, "filter_3D").shape == d["out_filter_3D"].shape
    fresh = dm.from_fixture(d, "cuda")
    _densify().reset_opacity(fresh)
    for k, v in dm.state_of(fresh).items():
        if k.startswith("opacity"):
            assert np.allclose(v, d["reset_" + k], rtol=0, atol=1e-5) and v.shape == d["reset_" + k].shape, k


def _new_rows(d):
    """Rows of the fixture's output before the new ones, and the draw of every new row."""
    m = dm.from_fixture(d, "cpu")
    sel = dm.select(m, *dm.arguments(d))
    clone, split, prune, prune_child = (sel[k].numpy() for k in ("clone", "split", "prune", "prune_child"))
    S = int(split.sum())
    live_c, live_s = ~prune[clone], ~prune_child[split]
    samples = np.concatenate([d["draw_clone"][live_c], d["draw_split"][:S][live_s], d["draw_split"][S:][live_s]])
    return int((~split & ~prune).sum()), samples


def _children_rows(d):
    """Rows of the fixture's output that are split children (the last ones)."""
    n_out = d["out_xyz"].shape[0]
    return n_out - _kept_and_clones(d)


def _kept_and_clones(d):
    m = dm.from_fixture(d, "cpu")
    sel = dm.select(m, *dm.arguments(d))
    keep = int((~sel["split"] & ~sel["prune"]).sum())
    return keep + int((sel["clone"] & ~sel["prune"]).sum())


@pytest.mark.parametrize("case", sorted(FIXTURE))
def test_select_binding_ratio_and_threshold(case):
    from diff_gaussian_rasterization import _C
    d = FIXTURE[case]
    m = dm.from_fixture(d, "cuda")
    mg, mo, ext, mss = dm.arguments(d)
    _, _, ratio_q, counts = _C._densify.select(m.xyz_gradient_accum, m.xyz_gradient_accum_abs, m.denom, m._scaling.detach(), m._opacity.detach(),
                                              mg, m.percent_dense * ext, mo, bool(mss), float(mss or 0), 0.1 * ext)
    P = d["in_xyz"].shape[0]
    ratio, Q = ratio_q.cpu().numpy()
    count = int(round(float(d["ratio"]) * P))
    assert ratio == dm.ratio_np(count, P, cuda=True)
    assert np.array_equal(np.float32(Q), d["Q_cuda"], equal_nan=True)
    assert counts[:2] == [int(d["clone"].sum()), int(d["split"].sum())]


def _random_model(P, deg, seed, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    d = {"percent_dense": np.float64(0.01)}
    d["in_xyz"] = (torch.rand(P, 3, generator=g) * 4 - 2).numpy()
    d["in_f_dc"] = torch.randn(P, 1, 3, generator=g).numpy()
    d["in_f_rest"] = (0.1 * torch.randn(P, (deg + 1) ** 2 - 1, 3, generator=g)).numpy()
    d["in_opacity"] = (torch.randn(P, 1, generator=g) * 2).numpy()
    d["in_scaling"] = (torch.randn(P, 3, generator=g) * 0.8 - 3.3).numpy()
    d["in_rotation"] = torch.randn(P, 4, generator=g).numpy()
    denom = torch.randint(0, 6, (P, 1), generator=g).float()
    d["in_denom"] = denom.numpy()
    d["in_xyz_gradient_accum"] = (torch.rand(P, 1, generator=g) * 0.0003 * denom).numpy()
    d["in_xyz_gradient_accum_abs"] = (torch.rand(P, 1, generator=g) * 0.004 * denom).numpy()
    d["in_xyz_gradient_accum_abs_max"] = torch.rand(P, 1, generator=g).numpy()
    d["in_max_radii2D"] = torch.randint(0, 40, (P,), generator=g).float().numpy()
    d["in_filter_3D"] = torch.exp(torch.randn(P, 1, generator=g) * 0.8 - 4.0).numpy()
    for name in dm.GROUPS:
        d[f"in_{name}.exp_avg"] = (torch.randn(d["in_" + name].shape, generator=g) * 1e-3).numpy()
        d[f"in_{name}.exp_avg_sq"] = (torch.rand(d["in_" + name].shape, generator=g) * 1e-6).numpy()
        d[f"in_{name}.step"] = np.float64(7)
    return d


def _assert_same(a, b):
    sa, sb = dm.state_of(a), dm.state_of(b)
    assert sorted(sa) == sorted(sb)
    for k in sa:
        assert sa[k].shape == sb[k].shape and np.array_equal(sa[k], sb[k]), k
    for k in STATS:
        assert torch.equal(getattr(a, k), getattr(b, k)), k


@pytest.mark.parametrize("P", [1, 257, 100_003, 1_000_000])
@pytest.mark.parametrize("mss", [None, 20])
def test_kernels_match_the_model_on_the_gpu(P, mss):
    d = _random_model(P, 3, P)
    ours, model = dm.from_fixture(d, "cuda"), dm.from_fixture(d, "cuda")
    torch.manual_seed(P)
    r_ours = _densify().densify_and_prune(ours, 0.0002, 0.05, 4.0, mss)
    torch.manual_seed(P)
    r_model, _ = dm.densify_and_prune(model, 0.0002, 0.05, 4.0, mss)
    assert r_ours == r_model
    _assert_same(ours, model)
    if P >= 100_000:
        assert min(r_ours) > 0


def test_two_runs_give_identical_bits():
    d = _random_model(200_000, 3, 11)
    runs = []
    for _ in range(2):
        m = dm.from_fixture(d, "cuda")
        torch.manual_seed(3)
        _densify().densify_and_prune(m, 0.0002, 0.05, 4.0, 20)
        runs.append(m)
    _assert_same(*runs)


def test_select_beyond_two_to_the_24():
    from diff_gaussian_rasterization import _C
    P = 2 ** 24 + 3
    g = torch.Generator(device="cuda").manual_seed(9)
    denom = torch.randint(0, 4, (P, 1), device="cuda", generator=g).float()
    accum = torch.rand(P, 1, device="cuda", generator=g) * 0.0004 * denom
    accum_abs = torch.rand(P, 1, device="cuda", generator=g) * denom
    scaling, opacity = torch.zeros(P, 3, device="cuda"), torch.zeros(P, 1, device="cuda")
    _, _, ratio_q, counts = _C._densify.select(accum, accum_abs, denom, scaling, opacity, 0.0002, 0.5, 0.05, False, 0.0, 1e9)
    ga = torch.nan_to_num(accum_abs / denom, nan=0.0).cpu().numpy().reshape(-1)
    gr = torch.nan_to_num(accum / denom, nan=0.0).cpu().numpy().reshape(-1)
    count = int((gr >= np.float32(0.0002)).sum())
    ratio = dm.ratio_np(count, P, cuda=True)
    Q = dm.quantile_np(ga, np.float32(1) - ratio)
    assert ratio_q[0].item() == ratio and np.float32(ratio_q[1].item()) == Q
    assert counts[0] == 0 and counts[1] == int(((gr >= np.float32(0.0002)) | (ga >= Q)).sum())   # max exp(0) = 1 > 0.5: split


def test_training_continues_after_densification():
    d = _random_model(50_000, 3, 21)
    ours, model = dm.from_fixture(d, "cuda"), dm.from_fixture(d, "cuda")
    for m in (ours, model):
        m.optimizer = torch.optim.Adam(m.optimizer.param_groups, lr=0.0, eps=1e-15, fused=True)
        for name, attr in dm.GROUPS.items():
            p = getattr(m, attr)
            m.optimizer.state[p] = {"step": torch.tensor(float(d[f"in_{name}.step"]), device="cuda"),
                                    "exp_avg": torch.tensor(d[f"in_{name}.exp_avg"], device="cuda"),
                                    "exp_avg_sq": torch.tensor(d[f"in_{name}.exp_avg_sq"], device="cuda")}
    torch.manual_seed(5)
    _densify().densify_and_prune(ours, 0.0002, 0.05, 4.0, None)
    torch.manual_seed(5)
    dm.densify_and_prune(model, 0.0002, 0.05, 4.0, None)
    for m in (ours, model):
        g = torch.Generator(device="cuda").manual_seed(1)
        for attr in dm.GROUPS.values():
            p = getattr(m, attr)
            p.grad = torch.randn(p.shape, device="cuda", generator=g) * 1e-2
        m.optimizer.step()
    _assert_same(ours, model)
    # the optimizer state round-trips through state_dict, as a checkpoint (capture / restore) stores it
    sd = ours.optimizer.state_dict()
    again = dm.from_fixture(d, "cuda")
    for name, attr in dm.GROUPS.items():
        setattr(again, attr, torch.nn.Parameter(getattr(ours, attr).detach().clone()))
    groups = [{"params": [getattr(again, attr)], "lr": 0.0, "name": name} for name, attr in dm.GROUPS.items()]
    groups += [{"params": list(again.appearance_network.parameters()), "lr": 0.0, "name": "appearance_network"},
               {"params": [again._appearance_embeddings], "lr": 0.0, "name": "appearance_embeddings"}]
    again.optimizer = torch.optim.Adam(groups, lr=0.0, eps=1e-15, fused=True)
    again.optimizer.load_state_dict(sd)
    for attr in dm.GROUPS.values():
        a, b = ours.optimizer.state[getattr(ours, attr)], again.optimizer.state[getattr(again, attr)]
        assert torch.equal(a["exp_avg"], b["exp_avg"]) and torch.equal(a["exp_avg_sq"], b["exp_avg_sq"]) and torch.equal(a["step"], b["step"])


def test_rasterizer_renders_the_densified_model():
    from rade_gs_b200 import rawapi, scenes
    from diff_gaussian_rasterization import _C
    d = _random_model(20_000, 3, 31)
    m = dm.from_fixture(d, "cuda")
    torch.manual_seed(2)
    _densify().densify_and_prune(m, 0.0002, 0.05, 4.0, 20)
    sc = scenes.make_scene(2000, 128, 96, 110.0, -2.6, seed=77, view=scenes.look_at_view((0.2, -0.1, -0.3), (0.0, 0.0, 6.0)), bg=(0.1, 0.2, 0.3))
    scd = sc.to("cuda")
    P = m._xyz.shape[0]
    scd.means3D = m._xyz.detach() + torch.tensor([0.0, 0.0, 6.0], device="cuda")
    scd.opacities = torch.sigmoid(m._opacity.detach())
    scd.scales = torch.exp(m._scaling.detach())
    scd.rotations = torch.nn.functional.normalize(m._rotation.detach())
    scd.shs = torch.cat([m._features_dc.detach(), m._features_rest.detach()], dim=1).contiguous()
    f = rawapi.forward(_C, scd, False, True, kernel_size=0.1)
    torch.cuda.synchronize()
    assert f["radii"].shape[0] == P and (f["radii"] > 0).any() and torch.isfinite(f["color"]).all()


def test_bad_input_is_rejected():
    from diff_gaussian_rasterization import _C
    d = _random_model(100, 0, 41)
    m = dm.from_fixture(d, "cuda")
    with pytest.raises(RuntimeError, match="rows"):
        _C._densify.select(m.xyz_gradient_accum[:99], m.xyz_gradient_accum_abs, m.denom, m._scaling.detach(), m._opacity.detach(),
                          0.0002, 0.04, 0.05, False, 0.0, 0.4)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        _C._densify.select(m.xyz_gradient_accum.cpu(), m.xyz_gradient_accum_abs, m.denom, m._scaling.detach(), m._opacity.detach(),
                          0.0002, 0.04, 0.05, False, 0.0, 0.4)
    e = torch.empty(0, 1, device="cuda")
    with pytest.raises(RuntimeError, match="no Gaussians"):
        _C._densify.select(e, e, e, torch.empty(0, 3, device="cuda"), e, 0.0002, 0.04, 0.05, False, 0.0, 0.4)
    m._xyz.data = m._xyz.data.cpu()
    with pytest.raises(RuntimeError, match="no CPU path"):
        _densify().densify_and_prune(m, 0.0002, 0.05, 4.0, None)

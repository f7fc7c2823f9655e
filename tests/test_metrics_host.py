"""CPU checks of rade_gs_b200.metrics: the fp64 restatement against the reference's fixture, weight loading from local
files only, and the argument checks that run before any device is touched."""
import os

import numpy as np
import pytest
import torch

import lpips_f64 as ref

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "metrics", "lpips.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def seeded(golden):
    sd = ref.seeded_weights(int(golden["seed"]))
    assert ref.digest(sd) == str(golden["digest"])
    return sd


@pytest.fixture()
def files(seeded, tmp_path):
    vgg, lin = tmp_path / "vgg16-397923af.pth", tmp_path / "vgg.pth"
    torch.save({k: v for k, v in seeded.items() if k.startswith("features.")}, vgg)
    torch.save({k: v for k, v in seeded.items() if k.startswith("lin")}, lin)
    return str(vgg), str(lin)


@pytest.fixture()
def no_download(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("a download was attempted")
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)


def test_fp64_restatement_matches_the_reference_fixture(golden, seeded):
    for n in golden["names"]:
        n = str(n)
        x, y = torch.from_numpy(golden[f"{n}/x"]), torch.from_numpy(golden[f"{n}/y"])
        got = ref.layer_means(x, y, seeded)
        want = golden[f"{n}/layers_f64"]
        for g, w in zip(got, want):
            assert abs(g.item() - w) <= 1e-12 * abs(w) + 1e-300, n
        total = float(golden[f"{n}/total_f64"])
        assert abs(ref.lpips(x, y, seeded).item() - total) <= 1e-12 * abs(total), n
        assert abs(float(golden[f"{n}/total_f32"]) - total) <= 1e-5 * abs(total) + 1e-9, n


def test_loader_maps_keys_and_repacks(files, seeded, no_download):
    from rade_gs_b200.metrics import load_lpips_weights, round_tf32
    w = load_lpips_weights(*files)
    assert len(w["convs"]) == 13 and len(w["heads"]) == 5
    order = [i for b in ref.BLOCKS for i in b]
    w0, b0 = w["convs"][0]
    assert torch.equal(w0, seeded["features.0.weight"]) and torch.equal(b0, seeded["features.0.bias"])
    for (wk, bk), i in zip(w["convs"][1:], order[1:]):
        src = seeded[f"features.{i}.weight"]
        assert wk.shape == (src.shape[0], 3, 3, src.shape[1])
        assert torch.equal(wk, round_tf32(src.permute(0, 2, 3, 1).contiguous()))
        assert torch.equal(bk, seeded[f"features.{i}.bias"])
        assert ((wk - src.permute(0, 2, 3, 1)).abs() <= src.permute(0, 2, 3, 1).abs() * 2.0 ** -11).all()
    for k, h in enumerate(w["heads"]):
        assert torch.equal(h, seeded[f"lin{k}.model.1.weight"].reshape(-1))


def test_round_tf32_is_nearest_ties_away():
    from rade_gs_b200.metrics import round_tf32
    one = 1.0
    ulp = 2.0 ** -10
    x = torch.tensor([one, one + ulp / 2, one + ulp / 2 - 2.0 ** -23, -(one + ulp / 2), one + 3 * ulp / 2, 0.0, -0.0], dtype=torch.float32)
    want = torch.tensor([one, one + ulp, one, -(one + ulp), one + 2 * ulp, 0.0, -0.0], dtype=torch.float32)
    got = round_tf32(x)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))


def test_missing_file_names_the_path(files, tmp_path, no_download):
    from rade_gs_b200.metrics import load_lpips_weights
    missing = str(tmp_path / "nowhere" / "vgg.pth")
    with pytest.raises(FileNotFoundError, match="nowhere/vgg.pth") as e:
        load_lpips_weights(files[0], missing)
    assert "vgg.pth" in str(e.value)
    with pytest.raises(FileNotFoundError, match="vgg16-397923af.pth"):
        load_lpips_weights(str(tmp_path / "none.pth"), files[1])


def test_default_location_is_the_hub_checkpoints(files, tmp_path, monkeypatch, no_download):
    from rade_gs_b200.metrics import load_lpips_weights
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    with pytest.raises(FileNotFoundError, match=str(tmp_path / "hub" / "checkpoints")):
        load_lpips_weights()
    os.makedirs(tmp_path / "hub" / "checkpoints")
    for f in files:
        os.symlink(f, tmp_path / "hub" / "checkpoints" / os.path.basename(f))
    assert len(load_lpips_weights()["convs"]) == 13


def test_wrong_shapes_and_missing_keys_are_rejected(seeded, tmp_path, files, no_download):
    from rade_gs_b200.metrics import load_lpips_weights
    bad = {k: v for k, v in seeded.items() if k.startswith("features.")}
    bad["features.7.weight"] = bad["features.7.weight"][:, :64]
    torch.save(bad, tmp_path / "bad_vgg.pth")
    with pytest.raises(ValueError, match=r"features.7.weight has shape \(128, 64, 3, 3\)"):
        load_lpips_weights(str(tmp_path / "bad_vgg.pth"), files[1])
    heads = {k: v for k, v in seeded.items() if k.startswith("lin") and not k.startswith("lin3")}
    torch.save(heads, tmp_path / "bad_lin.pth")
    with pytest.raises(ValueError, match="lin3.model.1.weight"):
        load_lpips_weights(files[0], str(tmp_path / "bad_lin.pth"))


@pytest.mark.parametrize("case", ["side15", "batch2", "channels4", "fp64", "mismatch"])
def test_lpips_rejects_bad_images_before_touching_a_device(case, no_download):
    from rade_gs_b200.metrics import lpips
    x = {"side15": torch.rand(3, 15, 40), "batch2": torch.rand(2, 3, 32, 32), "channels4": torch.rand(1, 4, 32, 32),
         "fp64": torch.rand(3, 32, 32, dtype=torch.float64), "mismatch": torch.rand(3, 32, 32)}[case]
    y = torch.rand(3, 32, 33) if case == "mismatch" else x.clone()
    with pytest.raises(ValueError):
        lpips(x, y, vgg_path="/nonexistent/a.pth", lin_path="/nonexistent/b.pth")


def test_only_vgg_is_implemented():
    from rade_gs_b200.metrics import lpips
    x = torch.rand(3, 32, 32)
    with pytest.raises(NotImplementedError, match="alex"):
        lpips(x, x, net_type="alex")


def test_cpu_images_are_refused_naming_cuda(no_download):
    from rade_gs_b200.metrics import lpips
    x = torch.rand(3, 32, 32)
    with pytest.raises(ValueError, match="CUDA"):
        lpips(x, x)


def test_every_lpips_entry_refuses_cpu_tensors():
    from diff_gaussian_rasterization import _C
    L = _C._lpips
    assert {n for n in dir(L) if not n.startswith("_")} == {"input_conv", "conv3x3", "maxpool", "distance"}
    img = torch.rand(3, 16, 16)
    calls = {
        "input_conv": lambda: L.input_conv(img, img, torch.rand(64, 3, 3, 3), torch.rand(64)),
        "conv3x3": lambda: L.conv3x3(torch.rand(2, 4, 4, 64), torch.rand(64, 3, 3, 64), torch.rand(64)),
        "maxpool": lambda: L.maxpool(torch.rand(2, 4, 4, 64)),
        "distance": lambda: L.distance(torch.rand(2, 4, 4, 64), torch.rand(64)),
    }
    for name, call in calls.items():
        with pytest.raises(RuntimeError, match="CUDA"):
            call()


def test_psnr_is_the_reference_formula():
    from rade_gs_b200.metrics import psnr
    g = torch.Generator().manual_seed(1)
    a, b = torch.rand(1, 3, 20, 30, generator=g), torch.rand(1, 3, 20, 30, generator=g)
    mse = ((a.double() - b.double()) ** 2).mean()
    assert psnr(a, b).shape == (1, 1)
    assert abs(psnr(a, b).item() - (20 * torch.log10(1 / mse.sqrt())).item()) < 1e-4

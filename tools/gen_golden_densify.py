"""Generate tests/golden/fused_densify.npz by running the REFERENCE'S OWN GaussianModel.densify_and_prune and reset_opacity
(scene/gaussian_model.py:495-513, :662-741) on the CPU, each on a model with a live torch.optim.Adam holding the state of one
real step.

The reference allocates with device="cuda" and calls .cuda() (gaussian_model.py:65-68, :665-676, utils/general_utils.py:85);
for the duration of this run those mean the CPU -- an environment shim, the reference files are imported as they are.  Every
torch.normal draw is recorded so the tests can replay it.  Keys are "<case>__<name>".

The inputs are not stored: tests/densify_model.py regenerates them from a seed (make_inputs), checked by `inputs_digest`.  Of the
outputs the fixture keeps the source row of every output row (`src`, `n_keep` original rows first), the columns computed on new
rows (`out_xyz`, `out_scaling`) and `reset_opacity`; every other output is a copy of an input row or zero.  This script checks
that rebuilding them (densify_model.expand) reproduces the reference's arrays bit for bit and stores their `outputs_digest`,
which the tests check again.  Each case also checks that the CUDA rounding of `ratio` and of the quantile selects the same rows
as the CPU run recorded here.

    python tools/gen_golden_densify.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("RADE_GS_REFERENCE") or os.path.join(os.path.dirname(ROOT), "reference")
sys.path[:0] = [os.path.join(ROOT, "tests", "ref_stubs"), REF, os.path.join(ROOT, "tests")]
torch.Tensor.cuda = lambda self, *a, **k: self            # noqa: E731  CPU run of code that says .cuda()
torch.nn.Module.cuda = lambda self, *a, **k: self         # noqa: E731


def _on_cpu(fn):
    def call(*a, **k):
        if str(k.get("device", "")).startswith("cuda"):
            k["device"] = "cpu"
        return fn(*a, **k)
    return call


for _name in ("tensor", "zeros", "ones", "empty"):
    setattr(torch, _name, _on_cpu(getattr(torch, _name)))

from scene.gaussian_model import GaussianModel   # noqa: E402
import densify_model as dm                         # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "fused_densify.npz")
torch.set_num_threads(4)


def make_model(d):
    """The reference's GaussianModel holding the inputs, with a live Adam over the reference's groups and the inputs' state."""
    pc = GaussianModel(int(d["sh_degree"]))
    pc.percent_dense = float(d["percent_dense"])
    pc.active_sh_degree = int(d["sh_degree"])
    for name, attr in dm.GROUPS.items():
        setattr(pc, attr, torch.nn.Parameter(torch.tensor(d["in_" + name])))
    for k in dm.STATS:
        setattr(pc, k, torch.tensor(d["in_" + k]))
    groups = [{"params": [getattr(pc, attr)], "lr": 1e-3, "name": name} for name, attr in dm.GROUPS.items()]
    groups += [{"params": list(pc.appearance_network.parameters()), "lr": 1e-3, "name": "appearance_network"},
               {"params": [pc._appearance_embeddings], "lr": 1e-3, "name": "appearance_embeddings"}]
    pc.optimizer = torch.optim.Adam(groups, lr=0.0, eps=1e-15)
    for name, attr in dm.GROUPS.items():
        if f"in_{name}.exp_avg" in d:
            pc.optimizer.state[getattr(pc, attr)] = {"step": torch.tensor(float(d[f"in_{name}.step"])),
                                                     "exp_avg": torch.tensor(d[f"in_{name}.exp_avg"]),
                                                     "exp_avg_sq": torch.tensor(d[f"in_{name}.exp_avg_sq"])}
    return pc


def snapshot(pc, prefix):
    out = {}
    for name, attr in dm.GROUPS.items():
        p = getattr(pc, attr)
        out[f"{prefix}{name}"] = p.detach().numpy().copy()
        st = pc.optimizer.state.get(p, None)
        if st is not None:
            out[f"{prefix}{name}.exp_avg"] = st["exp_avg"].numpy().copy()
            out[f"{prefix}{name}.exp_avg_sq"] = st["exp_avg_sq"].numpy().copy()
            out[f"{prefix}{name}.step"] = np.asarray(float(st["step"]))
    return out


def gen_case(case):
    d = dm.make_inputs(case)
    args = dm.arguments(d)
    pc = make_model(d)
    rec = {k: v for k, v in d.items() if not k.startswith("in_")}
    rec["inputs_digest"] = np.asarray(dm.digest(d))
    sel = dm.select(pc, *args)
    src, n_keep = dm.rows(sel)
    rec.update(ratio=sel["ratio"].numpy(), Q=sel["Q"].numpy(), clone=sel["clone"].numpy(), split=sel["split"].numpy(),
               src=src.numpy().astype(np.int32), n_keep=np.int64(n_keep))
    # the CUDA roundings of ratio and Q must select the same rows as this CPU run
    with np.errstate(invalid="ignore", divide="ignore"):
        g, ga = d["in_xyz_gradient_accum"] / d["in_denom"], d["in_xyz_gradient_accum_abs"] / d["in_denom"]
        g, ga = np.where(np.isnan(g), 0, g).reshape(-1), np.where(np.isnan(ga), 0, ga).reshape(-1)
        count = int((np.abs(g) >= np.float32(args[0])).sum())
        Q_cuda = dm.quantile_np(ga, np.float32(1) - dm.ratio_np(count, g.size, cuda=True))
        assert np.array_equal(ga >= Q_cuda, ga >= sel["Q"].numpy()), case
    rec["Q_cuda"] = np.asarray(Q_cuda, np.float32)
    draws = []
    normal = torch.normal

    def recording_normal(*a, **k):
        out = normal(*a, **k)
        draws.append(out.detach().clone())
        return out

    torch.normal = recording_normal
    try:
        result = pc.densify_and_prune(*args)
    finally:
        torch.normal = normal
    assert [tuple(t.shape) for t in draws] == [(int(sel["clone"].sum()), 3), (2 * int(sel["split"].sum()), 3)], case
    rec.update(draw_clone=draws[0].numpy(), draw_split=draws[1].numpy(), result=np.asarray(result, np.int64))
    ref = {f"out_{k}": v for k, v in snapshot(pc, "").items()}
    ref.update({f"out_{k}": getattr(pc, k).numpy().copy() for k in dm.STATS})
    fresh = make_model(d)                                  # reset_opacity on the inputs (the densified model's filter_3D is stale)
    fresh.reset_opacity()
    ref.update({f"reset_{k}": v for k, v in snapshot(fresh, "").items() if k.startswith("opacity")})
    rec.update(out_xyz=ref["out_xyz"], out_scaling=ref["out_scaling"], reset_opacity=ref["reset_opacity"])
    rebuilt = dm.expand({**d, **rec})
    assert sorted(rebuilt) == sorted(ref), case
    for k, v in ref.items():
        assert rebuilt[k].dtype == v.dtype and rebuilt[k].shape == v.shape and np.array_equal(rebuilt[k], v), (case, k)
    rec["outputs_digest"] = np.asarray(dm.digest(ref))
    print(f"{case:18s} P={len(d['in_xyz']):4d} ratio={float(rec['ratio']):.6g} Q={float(rec['Q']):.6g} (cloned, split, pruned)={result}")
    return rec


def main():
    out = {}
    for case in dm.CASES:
        for k, v in gen_case(case).items():
            out[f"{case}__{k}"] = np.asarray(v)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()

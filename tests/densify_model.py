"""Eager torch model of densify_and_prune and reset_opacity (reference scene/gaussian_model.py:495-513, :662-741), written as the
kernels decompose the work: every decision first, over the original rows, then one index_select per tensor.  It runs on the
CPU (where it must reproduce tests/golden/fused_densify.npz, made by the reference's own method, bit for bit) and on the GPU (where
the kernels must reproduce it bit for bit).  Device-dependent roundings come from torch itself: the mean behind `ratio` and
the division of the split scaling by a Python scalar.

quantile_np is a numpy model of torch.quantile's linear interpolation, usable beyond torch's 2^24-element limit.
"""
from fractions import Fraction

import numpy as np
import torch

GROUPS = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "scaling": "_scaling", "rotation": "_rotation"}


def build_rotation(r):
    """R of the normalised quaternion, each operation rounded on its own (utils/general_utils.py:80-101)."""
    norm = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    w, x, y, z = q.unbind(1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                        2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                        2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], 1).view(-1, 3, 3)


def offset(rotation, sample, xyz):
    """R * sample + xyz, products and sums rounded one at a time, left to right (torch.bmm's order on the CPU)."""
    R = build_rotation(rotation)
    return ((R[:, :, 0] * sample[:, None, 0] + R[:, :, 1] * sample[:, None, 1]) + R[:, :, 2] * sample[:, None, 2]) + xyz


def _fma32(a, b, c):
    """fp32 fused multiply-add, correctly rounded (exact rational arithmetic, then round to nearest even)."""
    a, b, c = (np.float32(v) for v in (a, b, c))
    if not (np.isfinite(a) and np.isfinite(b) and np.isfinite(c)):
        return np.float32(a * b + c)
    exact = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    r = np.float32(float(exact))
    best = r
    for cand in (np.nextafter(r, np.float32(-np.inf)), np.nextafter(r, np.float32(np.inf))):
        d0, d1 = abs(Fraction(float(best)) - exact), abs(Fraction(float(cand)) - exact)
        if d1 < d0 or (d1 == d0 and (cand.view(np.uint32) & 1) == 0):
            best = cand
    return np.float32(best)


def ratio_np(count, P, cuda=True):
    """mean() of `count` ones over P rows: ATen on CUDA multiplies the fp32 sum by the fp32 reciprocal of P; on the CPU it divides."""
    s, n = np.float32(count), np.float32(P)
    return np.float32(s * (np.float32(1) / n)) if cuda else np.float32(s / n)


def quantile_np(values, q):
    """torch.quantile(values, q), linear interpolation, at any size: indices clamped to the last element."""
    v = np.sort(np.asarray(values, np.float32).reshape(-1), kind="stable")
    P = v.size
    rank = np.float32(np.float32(q) * np.float32(P - 1))
    lo = int(rank)
    hi = int(np.ceil(rank))
    w = np.float32(rank - np.float32(lo))
    a, b = v[min(lo, P - 1)], v[min(hi, P - 1)]
    d = np.float32(b - a)
    return _fma32(w, d, a) if abs(w) < 0.5 else _fma32(-d, np.float32(1) - w, b)


def quantile(values, q):
    """torch.quantile up to 2^24 elements, the same formula above it."""
    if values.numel() <= 2 ** 24:
        return torch.quantile(values, q)
    v = values.sort().values
    P = v.numel()
    rank = q * (P - 1)
    lo = rank.long().clamp_max(P - 1)
    hi = rank.ceil().long().clamp_max(P - 1)
    return v[lo].lerp(v[hi], rank - rank.long())


def select(model, max_grad, min_opacity, extent, max_screen_size):
    """The decisions of densify_and_prune over the original rows."""
    def average(accum):
        g = accum / model.denom
        return torch.where(g.isnan(), torch.zeros_like(g), g)

    grads, grads_abs = average(model.xyz_gradient_accum), average(model.xyz_gradient_accum_abs)
    norm, norm_abs = torch.norm(grads, dim=-1), torch.norm(grads_abs, dim=-1)
    ratio = (norm >= max_grad).float().mean()
    Q = quantile(grads_abs.reshape(-1), 1 - ratio)
    scales = torch.exp(model._scaling)
    big = scales.max(dim=1).values
    dense = model.percent_dense * extent
    clone = ((norm >= max_grad) | (norm_abs >= Q)) & (big <= dense)
    split = ((grads.squeeze(-1) >= max_grad) | (grads_abs.squeeze(-1) >= Q)) & (big > dense)
    child_scaling = torch.log(scales / (0.8 * 2))
    faint = (torch.sigmoid(model._opacity) < min_opacity).squeeze(-1)
    prune, prune_child = faint, faint
    if max_screen_size:
        radius = torch.zeros_like(big) > max_screen_size     # max_radii2D was zeroed by densification_postfix
        prune = faint | radius | (big > 0.1 * extent)
        prune_child = faint | radius | (torch.exp(child_scaling).max(dim=1).values > 0.1 * extent)
    return dict(ratio=ratio, Q=Q, clone=clone, split=split, prune=prune, prune_child=prune_child, scales=scales, child_scaling=child_scaling)


@torch.no_grad()
def densify_and_prune(model, max_grad, min_opacity, extent, max_screen_size):
    """Mutates `model` as the reference's method does; returns (cloned, split, pruned) and the decisions."""
    sel = select(model, max_grad, min_opacity, extent, max_screen_size)
    clone_idx, split_idx = sel["clone"].nonzero().squeeze(1), sel["split"].nonzero().squeeze(1)
    C, S = clone_idx.numel(), split_idx.numel()
    dev = model._xyz.device
    sample_clone = torch.normal(mean=torch.zeros((C, 3), device=dev), std=sel["scales"][clone_idx])
    sample_split = torch.normal(mean=torch.zeros((2 * S, 3), device=dev), std=sel["scales"][split_idx].repeat(2, 1))
    clone_live, child_live = ~sel["prune"][clone_idx], ~sel["prune_child"][split_idx]
    src, n_keep = rows(sel)
    n_clone = int(clone_live.sum())
    new_sample = torch.cat([sample_clone[clone_live], sample_split[:S][child_live], sample_split[S:][child_live]])
    new_src = src[n_keep:]

    opt = model.optimizer
    for group in opt.param_groups:
        if group["name"] not in GROUPS:
            continue
        old = group["params"][0]
        out = old.detach().index_select(0, src)
        if group["name"] == "xyz":
            out[n_keep:] = offset(model._rotation.detach()[new_src], new_sample, old.detach()[new_src])
        elif group["name"] == "scaling":
            out[n_keep + n_clone:] = sel["child_scaling"][new_src[n_clone:]]
        state = opt.state.get(old, None)
        new = torch.nn.Parameter(out.requires_grad_(True))
        if state is not None:
            for key in ("exp_avg", "exp_avg_sq"):
                m = state[key].index_select(0, src)
                m[n_keep:] = 0
                state[key] = m
            del opt.state[old]
            opt.state[new] = state
        group["params"][0] = new
        setattr(model, GROUPS[group["name"]], new)
    N = src.numel()
    for name in ("xyz_gradient_accum", "xyz_gradient_accum_abs", "xyz_gradient_accum_abs_max", "denom"):
        setattr(model, name, torch.zeros((N, 1), device=dev))
    model.max_radii2D = torch.zeros((N,), device=dev)
    P = sel["clone"].numel()
    return (C, S, P + C + S - N), sel


@torch.no_grad()
def reset_opacity(model):
    scales = torch.exp(model._scaling)
    sq = scales * scales
    after = sq + model.filter_3D * model.filter_3D
    coef = torch.sqrt((sq[:, 0] * sq[:, 1] * sq[:, 2]) / (after[:, 0] * after[:, 1] * after[:, 2]))[:, None]
    o = torch.sigmoid(model._opacity) * coef
    x = torch.min(o, torch.ones_like(o) * 0.01) / coef
    new = torch.log(x / (1 - x))
    for group in model.optimizer.param_groups:
        if group["name"] != "opacity":
            continue
        old = group["params"][0]
        state = model.optimizer.state.get(old, None)
        p = torch.nn.Parameter(new.requires_grad_(True))
        if state is not None:
            state["exp_avg"], state["exp_avg_sq"] = torch.zeros_like(new), torch.zeros_like(new)
            del model.optimizer.state[old]
            model.optimizer.state[p] = state
        group["params"][0] = p
        model._opacity = p


# ---- the fixture (tests/golden/fused_densify.npz, tools/gen_golden_densify.py) ---------------------------------------------------
# The fixture stores no model: its inputs are regenerated here from a seed and must match the stored digest bit for bit.  Of the
# reference's outputs it stores the source row of every output row, the columns computed on new rows (xyz, scaling) and
# reset_opacity's result; the rest is rebuilt from the inputs, and the rebuilt arrays must match the digest of the reference's
# own outputs bit for bit.

STATS = ("xyz_gradient_accum", "xyz_gradient_accum_abs", "xyz_gradient_accum_abs_max", "denom", "max_radii2D", "filter_3D")

# case: (P, sh degree, max_grad, min_opacity, extent, max_screen_size, percent_dense, scaling mean, groups left without state)
CASES = {
    "deg3_none": (300, 3, 0.0002, 0.05, 4.0, None, 0.01, -3.3, ()),
    "deg0_screen20": (400, 0, 0.0002, 0.05, 4.0, 20, 0.01, -3.3, ()),
    "no_state": (300, 1, 0.0002, 0.05, 4.0, 20, 0.01, -3.3, ("f_rest", "rotation")),
    "nothing_selected": (200, 0, 1e9, 0.0, 4.0, None, 0.01, -3.3, ()),
    "all_pruned": (200, 0, 0.0002, 1.0, 4.0, None, 0.01, -3.3, ()),
    "ratio_zero": (250, 0, 1e9, 0.05, 4.0, None, 0.01, -3.3, ()),
    "ratio_one": (250, 0, 0.0, 0.05, 4.0, None, 0.01, -3.3, ()),
    "negative_screen": (250, 0, 0.0002, 0.05, 4.0, -1, 0.01, -3.3, ()),
    "boundary_dense": (300, 0, 0.0002, 0.5 + 2 ** -30, (1 - 2 ** -30) / 0.01, None, 0.01, 0.0, ()),
    "boundary_world": (300, 0, 0.0002, 0.05, 10.00000001, 20, 0.01, -2.0, ()),
    "ratio_rounding": (None, 0, 0.0002, 0.05, 4.0, None, 0.01, -3.3, ()),
}


def rounding_p_count():
    """A (P, count) where ATen's CUDA mean (sum * (1/P)) and its CPU mean (sum / P) round differently."""
    for P in range(200, 400):
        for count in range(P // 10, P):
            if ratio_np(count, P, cuda=True) != ratio_np(count, P, cuda=False):
                return P, count
    raise AssertionError("no such P")


def _away(x, thresholds, rel=1e-5):
    """Move float64 values within `rel` (relative) of an fp32-rounded threshold to 2 rel above it."""
    for t in thresholds:
        t = float(np.float32(t))
        x = np.where(np.abs(x - t) <= rel * abs(t), t * (1 + 2 * rel) if t >= 0 else t * (1 - 2 * rel), x)
    return x


def make_inputs(case):
    """The inputs of a fixture case (in_* arrays and the call's arguments), seeded, after one real torch.optim.Adam step with
    lr 0: the parameters are as drawn, the moments and step as Adam leaves them.  Every value that is compared with a threshold
    sits at least 1e-5 (relative) away from it, so exp and sigmoid, whose last bit differs between torch's CPU and CUDA builds,
    decide nothing; the planted rows of the boundary cases use exp(0) = 1 and sigmoid(0) = 0.5, exact on both."""
    P, deg, max_grad, min_opacity, extent, mss, pd, smean, no_state = CASES[case]
    count = None
    if P is None:
        P, count = rounding_p_count()
    rng = np.random.default_rng(1000 + list(CASES).index(case))
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)     # noqa: E731
    raw_s = rng.standard_normal((P, 3)) * 0.8 + smean
    dense, world = pd * extent, 0.1 * extent
    for _ in range(3):   # each threshold the largest scale, and the split child's, is compared with
        big = np.exp(raw_s).max(axis=1)
        raw_s = raw_s + np.log(_away(big, [dense, world] + ([world * 1.6] if mss else [])) / big)[:, None]
    opa = rng.standard_normal((P, 1)) * 2
    if min_opacity not in (0.0, 1.0):
        sig = _away(1 / (1 + np.exp(-opa)), [min_opacity])
        opa = np.log(sig / (1 - sig))
    denom = rng.integers(0, 6, (P, 1)).astype(np.float64)
    accum = rng.random((P, 1)) * 0.0012 * denom
    accum_abs = rng.random((P, 1)) * 0.004 * denom
    zero_denom = np.nonzero(denom[:, 0] == 0)[0]
    if case != "ratio_zero":                      # there q = 1 picks the largest grads_abs: keep it finite
        accum_abs[zero_denom[::3]] = 0.01         # x / 0 = +inf in grads_abs; the rest 0 / 0 = NaN -> 0
    if case == "nothing_selected":
        accum_abs[zero_denom[:2]] = 0.01          # the top two grads_abs are +inf: Q = lerp(inf, inf, 0) = NaN
    if count is not None:                         # exactly `count` rows with |g| >= max_grad
        order = rng.permutation(P)
        denom[:] = 1
        accum[order[:count]] = 0.0003 + 0.0001 * rng.random((count, 1))
        accum[order[count:]] = 0.0001 * rng.random((P - count, 1))
    if case.startswith("boundary"):
        # planted rows: g = max_grad in row 0; exp(0) = 1 in rows 0-3 against thresholds that round to 1.0f;
        # boundary_dense: rows 1-3 are selected (clones); boundary_world: they are not, and face the world-size test
        accum[0], denom[0] = float(np.float32(0.0002)), 1.0
        raw_s[0:4] = [0.0, -5.0, -5.0]
        accum[1:4], accum_abs[1:4], denom[1:4] = 0.0, (1.0 if case == "boundary_dense" else 0.0), 1.0
        opa[1:4] = 0.0                            # sigmoid(0) = 0.5 against min_opacity 0.5 + 2^-30 -> 0.5f
    d = {"in_xyz": f32(rng.random((P, 3)) * 4 - 2), "in_f_dc": f32(rng.standard_normal((P, 1, 3))),
         "in_f_rest": f32(0.1 * rng.standard_normal((P, (deg + 1) ** 2 - 1, 3))), "in_opacity": f32(opa), "in_scaling": f32(raw_s),
         "in_rotation": f32(rng.standard_normal((P, 4))), "in_filter_3D": f32(np.exp(rng.standard_normal((P, 1)) * 0.8 - 4.0)),
         "in_xyz_gradient_accum": f32(accum), "in_xyz_gradient_accum_abs": f32(accum_abs), "in_denom": f32(denom),
         "in_xyz_gradient_accum_abs_max": f32(rng.random((P, 1))), "in_max_radii2D": f32(rng.integers(0, 40, P))}
    params = {name: torch.nn.Parameter(torch.tensor(d["in_" + name])) for name in GROUPS}
    opt = torch.optim.Adam([{"params": [p], "lr": 0.0, "name": name} for name, p in params.items()], eps=1e-15)
    for name, p in params.items():               # groups without a gradient get no state
        p.grad = None if name in no_state else torch.tensor(f32(rng.standard_normal(p.shape) * 0.01))
    opt.step()
    for name, p in params.items():
        assert np.array_equal(p.detach().numpy(), d["in_" + name])
        st = opt.state.get(p, None)
        if st is not None:
            d[f"in_{name}.exp_avg"], d[f"in_{name}.exp_avg_sq"] = st["exp_avg"].numpy().copy(), st["exp_avg_sq"].numpy().copy()
            d[f"in_{name}.step"] = np.asarray(float(st["step"]))
    d.update(percent_dense=np.float64(pd), sh_degree=np.int64(deg), max_grad=np.float64(max_grad), min_opacity=np.float64(min_opacity),
             extent=np.float64(extent), max_screen_size=np.float64(np.nan if mss is None else mss))
    return d


def digest(arrays):
    """sha256 over the names, dtypes, shapes and bytes of a dict of arrays."""
    import hashlib
    h = hashlib.sha256()
    for k in sorted(arrays):
        a = np.ascontiguousarray(arrays[k])
        h.update(f"{k}|{a.dtype.str}|{a.shape}|".encode())
        h.update(a.tobytes())
    return h.hexdigest()


def rows(sel):
    """(source row of every output row, number of original rows kept): the output's row order."""
    clone_idx, split_idx = sel["clone"].nonzero().squeeze(1), sel["split"].nonzero().squeeze(1)
    keep = (~sel["split"] & ~sel["prune"]).nonzero().squeeze(1)
    clone_live, child_live = ~sel["prune"][clone_idx], ~sel["prune_child"][split_idx]
    return torch.cat([keep, clone_idx[clone_live], split_idx[child_live], split_idx[child_live]]), keep.numel()


def expand(d):
    """Every out_* and reset_* array of a case from its inputs and the stored columns (see the note above)."""
    src, n_keep = d["src"].astype(np.int64), int(d["n_keep"])
    out = {}
    for name in GROUPS:
        out["out_" + name] = d["out_" + name] if name in ("xyz", "scaling") else d["in_" + name][src]
        if f"in_{name}.exp_avg" in d:
            for key in ("exp_avg", "exp_avg_sq"):
                m = d[f"in_{name}.{key}"][src]
                m[n_keep:] = 0
                out[f"out_{name}.{key}"] = m
            out[f"out_{name}.step"] = d[f"in_{name}.step"]
    for k in STATS:
        out["out_" + k] = d["in_filter_3D"] if k == "filter_3D" else np.zeros((len(src),) + d["in_" + k].shape[1:], np.float32)
    out["reset_opacity"] = d["reset_opacity"]
    if "in_opacity.exp_avg" in d:
        out["reset_opacity.exp_avg"] = out["reset_opacity.exp_avg_sq"] = np.zeros_like(d["reset_opacity"])
        out["reset_opacity.step"] = d["in_opacity.step"]
    return out


def load_fixture(path):
    """{case: {name: array}}: the fixture's arrays, the regenerated inputs and the rebuilt outputs, each checked by its digest."""
    cases = {}
    with np.load(path) as z:
        for key in z.files:
            case, name = key.split("__", 1)
            cases.setdefault(case, {})[name] = z[key]
    for case, d in cases.items():
        inputs = make_inputs(case)
        assert digest(inputs) == str(d["inputs_digest"]), f"{case}: the regenerated inputs differ from the fixture's"
        d.update(inputs)
        outputs = expand(d)
        assert digest(outputs) == str(d["outputs_digest"]), f"{case}: the rebuilt outputs differ from the reference's"
        d.update(outputs)
    return cases


class Model:
    """The attributes of the reference's GaussianModel that densify_and_prune and reset_opacity touch."""


def from_fixture(d, device, prefix="in_"):
    m = Model()
    for name, attr in GROUPS.items():
        setattr(m, attr, torch.nn.Parameter(torch.tensor(d[prefix + name], device=device)))
    for k in ("xyz_gradient_accum", "xyz_gradient_accum_abs", "xyz_gradient_accum_abs_max", "denom", "max_radii2D", "filter_3D"):
        setattr(m, k, torch.tensor(d[prefix + k], device=device))
    m.percent_dense = float(d["percent_dense"])
    m.appearance_network = torch.nn.Linear(3, 3).to(device)
    m._appearance_embeddings = torch.nn.Parameter(torch.zeros(4, 8, device=device))
    groups = [{"params": [getattr(m, attr)], "lr": 1e-3, "name": name} for name, attr in GROUPS.items()]
    groups += [{"params": list(m.appearance_network.parameters()), "lr": 1e-3, "name": "appearance_network"},
               {"params": [m._appearance_embeddings], "lr": 1e-3, "name": "appearance_embeddings"}]
    m.optimizer = torch.optim.Adam(groups, lr=0.0, eps=1e-15)
    for name, attr in GROUPS.items():
        if prefix + name + ".exp_avg" in d:
            p = getattr(m, attr)
            m.optimizer.state[p] = {"step": torch.tensor(float(d[prefix + name + ".step"])),
                                    "exp_avg": torch.tensor(d[prefix + name + ".exp_avg"], device=device),
                                    "exp_avg_sq": torch.tensor(d[prefix + name + ".exp_avg_sq"], device=device)}
    return m


def arguments(d):
    mss = float(d["max_screen_size"])
    return float(d["max_grad"]), float(d["min_opacity"]), float(d["extent"]), None if np.isnan(mss) else int(mss)


class replay:
    """torch.normal returns the given draws, in order, on the device it was asked for, while the context is open."""

    def __init__(self, draws):
        self.draws = list(draws)

    def __enter__(self):
        self.normal = torch.normal

        def fake(mean, std, *a, **k):
            want = self.draws.pop(0)
            assert tuple(want.shape) == tuple(std.shape), (tuple(want.shape), tuple(std.shape))
            return torch.as_tensor(want).to(std.device)
        torch.normal = fake
        return self

    def __exit__(self, *exc):
        torch.normal = self.normal
        assert exc[0] is not None or not self.draws, "not every recorded draw was consumed"


def state_of(m):
    """{name: array} of the parameters, their moments and step, as the fixture's snapshot names them."""
    out = {}
    for name, attr in GROUPS.items():
        p = getattr(m, attr)
        out[name] = p.detach().cpu().numpy()
        st = m.optimizer.state.get(p, None)
        if st is not None:
            out[name + ".exp_avg"] = st["exp_avg"].cpu().numpy()
            out[name + ".exp_avg_sq"] = st["exp_avg_sq"].cpu().numpy()
            out[name + ".step"] = np.asarray(float(st["step"]))
    return out

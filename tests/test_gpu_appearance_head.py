"""The decoupled-appearance network's head in the project's kernels (csrc/rgs_appearance_head.cu, `_C._appearance_head`):

  - the head alone (conv1, up1..up4 forward, every stored activation, and backward from a d(up4) with exact zeros and a wide
    dynamic range) against the fp64 model of tests/appearance_f64.py, at the fixture cases and the recipes' image sizes, within
    test_fused_golden._close's bar against torch's fp32 evaluation without cuDNN;
  - `L1_loss_appearance` on the reference's own fixture (tests/golden/fused_appearance.npz) under torch's default flags;
  - every output bit-identical across cuDNN / TF32 / deterministic / benchmark settings and across calls;
  - the entries on poisoned memory and on a late-ready side stream;
  - `slab_L1_loss_appearance` over 2, 3, 4 and 8 slabs, its ranks run as threads of one process over an in-memory stand-in for
    the collectives: head, embedding and d_image gradients bit for bit those of `L1_loss_appearance`;
  - the wrapper's shape rejections before any launch."""
import threading
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn as nn

import appearance_f64 as af
from conftest import GOLDEN_DIR
from test_fused_golden import _close
from test_gpu_appearance import _check_all, _recipe_inputs, _run, _setup
from test_gpu_stale_memory import Case, check_case, poisoned_allocator  # noqa: F401  (the fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda"
SIZES = [(600, 800), (546, 979), (1200, 1600)]
HEAD_NAMES = af.PARAM_NAMES[:10]


def _C():
    import diff_gaussian_rasterization as dgr
    return dgr._C


def _inputs(inp, seed):
    """down (the downsample kernel's), the view's embedding row, the ten head parameters, and a d(up4) with a quarter exact
    zeros and magnitudes over six decades."""
    image = torch.as_tensor(inp["image"]).to(DEV)
    down = _C().appearance_downsample(image)
    h, w = down.shape[1:]
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(1, 16, 16 * h, 16 * w, generator=g) * 10.0 ** (6.0 * torch.rand(1, 16, 16 * h, 16 * w, generator=g) - 4.0)
    d[torch.rand(d.shape, generator=g) < 0.25] = 0.0
    return {"down": down, "emb": torch.as_tensor(inp["table"][af.VIEW_IDX]).to(DEV),
            "head": [torch.as_tensor(p).to(DEV) for p in inp["params"][:10]], "d_up4": d.to(DEV)}


def _split(act, h, w):
    sizes = [(256, h, w), (128, 2 * h, 2 * w), (64, 4 * h, 4 * w), (32, 8 * h, 8 * w)]
    out, o = [], 0
    for s in sizes:
        n = s[0] * s[1] * s[2]
        out.append(act[o:o + n].view(s))
        o += n
    assert o == act.numel()
    return out


def _fused(x):
    C = _C()
    act, up4 = C._appearance_head.forward(x["down"], x["emb"], x["head"])
    g = C._appearance_head.backward(x["down"], x["emb"], x["head"], act, up4, x["d_up4"])
    h, w = x["down"].shape[1:]
    return {"acts": _split(act, h, w), "up4": up4[0], "d_down": g[0], "d_emb": g[1], "grads": list(g[2:])}


def _torch(x, dtype):
    """The head as torch layers, without cuDNN: at the fixture cases' 1x2 .. 3x4 head inputs cuDNN may pick Winograd / FFT
    algorithms whose fp32 error (~1e-4) would loosen the bar; torch's native convolution keeps plain fp32 accuracy."""
    import torch.nn.functional as F
    down, emb = (x[k].to(dtype).clone().requires_grad_(True) for k in ("down", "emb"))
    p = [t.to(dtype).clone().requires_grad_(True) for t in x["head"]]
    h, w = down.shape[1:]
    a = torch.relu(F.conv2d(torch.cat([down, emb[:, None, None].expand(64, h, w)])[None], p[0], p[1], padding=1))
    acts = [a]
    for k in range(1, 5):
        a = torch.relu(F.conv2d(F.pixel_shuffle(a, 2), p[2 * k], p[2 * k + 1], padding=1))
        acts.append(a)
    grads = torch.autograd.grad(a, [down, emb, *p], x["d_up4"].to(dtype))
    return {"acts": [t[0] for t in acts[:4]], "up4": a[0], "d_down": grads[0], "d_emb": grads[1], "grads": list(grads[2:])}


def _model(x, masks=None):
    """The fp64 model: appearance_f64's conv, conv_T, conv_wgrad and (un)shuffle.  Backward uses the five ReLU masks `masks` when
    given (else its own), and the pre-activations are returned with the result."""
    down, emb = (x[k].double().cpu().numpy() for k in ("down", "emb"))
    p = [t.double().cpu().numpy() for t in x["head"]]
    h, w = down.shape[1:]
    x0 = np.concatenate([down, np.broadcast_to(emb[:, None, None], (64, h, w))])
    pre = [af.conv(x0, p[0], p[1])]
    ins, acts = [x0], [np.maximum(pre[0], 0)]
    for k in range(1, 5):
        ins.append(af.pixel_shuffle(acts[-1]))
        pre.append(af.conv(ins[-1], p[2 * k], p[2 * k + 1]))
        acts.append(np.maximum(pre[-1], 0))
    masks = masks if masks is not None else [a > 0 for a in acts]
    grads = [None] * 10
    d_a = x["d_up4"][0].double().cpu().numpy()
    for k in range(4, 0, -1):
        dz = d_a * masks[k]
        grads[2 * k], grads[2 * k + 1] = af.conv_wgrad(dz, ins[k])
        d_a = af.pixel_unshuffle(af.conv_T(dz, p[2 * k]))
    dz = d_a * masks[0]
    grads[0], grads[1] = af.conv_wgrad(dz, x0)
    d_x0 = af.conv_T(dz, p[0])
    return {"acts": acts[:4], "up4": acts[4], "d_down": d_x0[:3], "d_emb": d_x0[3:].sum(axis=(1, 2)), "grads": grads, "pre": pre}


def _flat(r):
    names = [f"act{i}" for i in range(4)] + ["up4", "d_down", "d_emb"] + [f"d {n}" for n in HEAD_NAMES]
    vals = list(r["acts"]) + [r["up4"], r["d_down"], r["d_emb"]] + list(r["grads"])
    return dict(zip(names, [v.detach().double().cpu().numpy() if torch.is_tensor(v) else v for v in vals]))


_HEAD_CASES = [("case", c) for c in af.CASES] + [("size", s) for s in SIZES]


@pytest.mark.parametrize("kind,which", _HEAD_CASES, ids=[c if k == "case" else f"{c[0]}x{c[1]}" for k, c in _HEAD_CASES])
def test_head_alone_against_fp64(kind, which):
    inp = af.make_inputs(which) if kind == "case" else _recipe_inputs(*which, sum(which))
    x = _inputs(inp, 17)
    with torch.backends.cudnn.flags(enabled=False):
        r32 = _flat(_torch(x, torch.float32))
    fused = _fused(x)
    # A ReLU input within fp32 rounding of 0 may fall on either side in any fp32 summation order, and a flipped mask is no error
    # of either implementation (appearance_f64.RELU_MARGIN): the fp64 backward takes the kernels' masks, and every place where
    # they differ from fp64's own must be such an input.
    ours_masks = [(t > 0).cpu().numpy() for t in fused["acts"]] + [(fused["up4"] > 0).cpu().numpy()]
    m64 = _model(x, ours_masks)
    for k, (z, m) in enumerate(zip(m64["pre"], ours_masks)):
        flips = m != (z > 0)
        assert np.abs(z[flips]).max(initial=0.0) <= 1e-5 * np.abs(z).max(), f"layer {k}: a mask flip away from 0"
    ours, r64 = _flat(fused), _flat(m64)
    failures = []
    for k in r64:
        assert ours[k].shape == r64[k].shape, (k, ours[k].shape, r64[k].shape)
        try:
            _close(ours[k], r32[k], r64[k], k, 2e-6)
        except AssertionError as e:
            failures.append(str(e).split("\n")[0])
    assert not failures, failures


@pytest.mark.parametrize("case", list(af.CASES))
def test_fixture_parity_under_default_flags(case):
    """The reference's own function (fp32 and fp64) pins the whole loss, head gradients included, with torch's default cuDNN
    flags: the head no longer runs on cuDNN, so no flag needs setting."""
    from rade_gs_b200.appearance import L1_loss_appearance
    d = af.load_fixture(f"{GOLDEN_DIR}/fused_appearance.npz")[case]
    inp = af.make_inputs(case)
    assert af.inputs_digest(inp) == str(d["digest"])
    ours = _run(L1_loss_appearance, inp)
    r32 = {k: d[k] for k in ("loss", "d_image", "d_emb", "transformed")}
    r64 = {k: d[k + "_f64"] for k in r32}
    r32["grads"] = [d["g_" + n] for n in af.PARAM_NAMES]
    r64["grads"] = [d["g_" + n + "_f64"] for n in af.PARAM_NAMES]
    _check_all(ours, r32, r64, sub=af.recorded)


FLAGS = [dict(enabled=False, allow_tf32=False, deterministic=False, benchmark=False),
         dict(enabled=True, allow_tf32=False, deterministic=False, benchmark=False),
         dict(enabled=True, allow_tf32=True, deterministic=False, benchmark=True),
         dict(enabled=True, allow_tf32=True, deterministic=True, benchmark=False)]


def test_outputs_do_not_depend_on_cudnn_flags():
    from rade_gs_b200.appearance import L1_loss_appearance
    inp = _recipe_inputs(546, 979, 5)
    runs = []
    for f in FLAGS:
        with torch.backends.cudnn.flags(**f):
            for _ in range(2):
                r = _run(L1_loss_appearance, inp)
                runs.append((f, [np.asarray(r["loss"])] + [r[k] for k in ("d_image", "d_emb", "transformed")] + r["grads"]))
    names = ["loss", "d_image", "d_emb", "transformed"] + af.PARAM_NAMES
    for f, vals in runs[1:]:
        for n, a, b in zip(names, vals, runs[0][1]):
            assert np.array_equal(np.atleast_1d(a).view(np.uint8), np.atleast_1d(b).view(np.uint8)), (f, n)


def test_head_entries_on_poisoned_memory_and_a_side_stream(poisoned_allocator):
    x = _inputs(_recipe_inputs(546, 979, 9), 3)

    def run(x):
        r = _fused(x)
        out = {f"act{i}": a for i, a in enumerate(r["acts"])}
        out.update({"up4": r["up4"], "d_down": r["d_down"], "d_emb": r["d_emb"]})
        out.update({n: g for n, g in zip(HEAD_NAMES, r["grads"])})
        return out
    check_case(Case(x, run), poisoned_allocator)


# ---- the sharded loss: ranks as threads of one process ----------------------------------------------------------------

class _ThreadCollectives:
    """What multigpu's slab losses call of torch.distributed (all_gather, P2POp / isend / irecv / batch_isend_irecv), for ranks
    that are threads of one process on one device.  Every rank enqueues on the device's default stream, so a copy a receiver
    enqueues after the sender's clone runs after it."""

    def __init__(self, world):
        self.world, self.local, self.cv = world, threading.local(), threading.Condition()
        self.slots, self.calls = {}, {}
        self.isend, self.irecv = "send", "recv"

    def P2POp(self, op, tensor, peer, group=None):
        return (op, tensor, peer)

    def _take(self, key, pop):
        with self.cv:
            if not self.cv.wait_for(lambda: key in self.slots, timeout=300):
                raise TimeoutError(f"rank {self.local.rank}: nothing arrived for {key}")
            return self.slots.pop(key) if pop else self.slots[key]

    def batch_isend_irecv(self, ops):
        r = self.local.rank
        with self.cv:
            for op, t, peer in ops:
                if op == "send":
                    self.slots[("p2p", r, peer)] = t.clone()
            self.cv.notify_all()
        for op, t, peer in ops:
            if op == "recv":
                t.copy_(self._take(("p2p", peer, r), True))
        return []

    def all_gather(self, parts, t, group=None):
        r = self.local.rank
        n = self.calls[r] = self.calls.get(r, 0) + 1
        with self.cv:
            self.slots[("ag", n, r)] = t.clone()
            self.cv.notify_all()
        for i, p in enumerate(parts):
            p.copy_(self._take(("ag", n, i), False))


class _Ctx:
    def save_for_backward(self, *t):
        self.saved_tensors = t


def _slab_ranks(inp, rows, view):
    """Each rank's forward and backward of multigpu._SlabAppearanceL1 in its own thread; returns the per-rank gradients."""
    from rade_gs_b200 import multigpu
    from rade_gs_b200.appearance import _head_params
    world = len(rows)
    fake = _ThreadCollectives(world)
    g, image, gt = _setup(inp)
    net = g.appearance_network
    params = _head_params(net) + [net.conv2.weight, net.conv2.bias, net.conv3.weight, net.conv3.bias]
    emb = g.table[view].detach()
    H0 = image.shape[1]
    out, errors = [None] * world, []

    def rank_main(rank):
        try:
            fake.local.rank = rank
            ctx = _Ctx()
            with torch.no_grad():
                multigpu._SlabAppearanceL1.forward(ctx, image.detach(), gt, emb, net, (H0, rows, rank, world, None), multigpu._CudaAppearanceRows,
                                                   *[p.detach() for p in params])
            out[rank] = multigpu._SlabAppearanceL1.backward(ctx, torch.ones((), device=DEV))
        except BaseException as e:  # noqa: BLE001  (re-raised on the main thread)
            errors.append((rank, e))

    old = multigpu.dist
    multigpu.dist = fake
    try:
        threads = [threading.Thread(target=rank_main, args=(r,)) for r in range(world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    finally:
        multigpu.dist = old
    torch.cuda.synchronize()
    if errors:
        raise errors[0][1]
    return out


def _partitions(H0):
    from rade_gs_b200 import multigpu
    n = multigpu.tile_rows(H0)
    out = {f"{world}eq": multigpu.partition_tile_rows(n, world) for world in (2, 3, 4, 8)}
    wts = [1.0 + 20.0 * (y > 2 * n // 3) for y in range(n)]
    out.update({f"{world}wt": multigpu.partition_tile_rows(n, world, wts) for world in (3, 8)})
    return {k: [(min(b * 16, H0), min(e * 16, H0)) for b, e in v] for k, v in out.items()}


def _bits(name, a, b):
    assert a.shape == b.shape, (name, tuple(a.shape), tuple(b.shape))
    bad = int((a.contiguous().view(torch.int32) != b.contiguous().view(torch.int32)).sum())
    assert bad == 0, f"{name}: {bad} of {a.numel()} elements differ"


@pytest.mark.parametrize("H0,W0", [(1200, 1600), (546, 979)])
def test_sharded_head_is_the_single_gpu_head_bit_for_bit(H0, W0):
    """No cuDNN flag is set: the head's gradients are the same bits on every rank as in the single-GPU call."""
    from rade_gs_b200.appearance import L1_loss_appearance
    inp = _recipe_inputs(H0, W0, 31 + H0)
    view = 2
    g, image, gt = _setup(inp)
    L1_loss_appearance(image, gt, g, view).backward()
    head_ref = [p.grad for p in list(g.appearance_network.parameters())[:10]]
    for name, rows in _partitions(H0).items():
        per_rank = _slab_ranks(inp, rows, view)
        d_image = torch.full_like(image, float("nan"))
        for rank, ((r0, r1), grads) in enumerate(zip(rows, per_rank)):
            d_image[:, r0:r1] = grads[0][:, r0:r1]
            _bits(f"{name} rank {rank} d_emb", grads[2], g.table.grad[view])
            for n, a, b in zip(HEAD_NAMES, grads[6:16], head_ref):
                _bits(f"{name} rank {rank} {n}", a, b)
        _bits(f"{name} d_image", d_image, image.grad)


def test_rejections_before_any_launch():
    from rade_gs_b200 import multigpu
    from rade_gs_b200.appearance import L1_loss_appearance
    C = _C()
    inp = af.make_inputs("odd_offsets")
    bad_nets = {"conv1": lambda n: setattr(n, "conv1", nn.Conv2d(67, 128, 3, padding=1)),
                "up2": lambda n: setattr(n.up2, "conv", nn.Conv2d(32, 64, 5, padding=2)),
                "up4": lambda n: setattr(n.up4, "conv", nn.Conv2d(8, 16, 3, padding=1, bias=False)),
                "up3": lambda n: delattr(n, "up3")}
    for layer, spoil in bad_nets.items():
        g, image, gt = _setup(inp)
        spoil(g.appearance_network)
        g.appearance_network.to(DEV)
        torch.cuda.synchronize()
        n0 = C.launch_count()
        with pytest.raises(ValueError, match=f"{layer} must be"):
            L1_loss_appearance(image, gt, g, af.VIEW_IDX)
        with pytest.raises(ValueError, match=f"{layer} must be"):
            multigpu.slab_L1_loss_appearance(image, gt, g, af.VIEW_IDX, (0, image.shape[1]), all_pixel_rows=[(0, image.shape[1])])
        assert C.launch_count() == n0, layer
    g, image, gt = _setup(inp)
    wide = torch.zeros(8, 65, device=DEV)
    g2 = SimpleNamespace(appearance_network=g.appearance_network, get_apperance_embedding=lambda i: wide[i])
    n0 = C.launch_count()
    for fn in (lambda: L1_loss_appearance(image, gt, g2, 0), lambda: multigpu.slab_L1_loss_appearance(image, gt, g2, 0, (0, 67), all_pixel_rows=[(0, 67)])):
        with pytest.raises(ValueError, match="embedding"):
            fn()
    assert C.launch_count() == n0

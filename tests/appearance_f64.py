"""fp64 numpy model of the decoupled-appearance L1 loss (train.py:37-58 with GOF's AppearanceNetwork), forward and backward,
in the decomposition csrc/rgs_appearance.cu uses: the 4-tap downsample and its scatter transpose, the x2 upsample and its
transpose as a gather (each sample sums the pixels whose taps reach it), conv3^T / conv2^T as transposed convolutions, and
the conv2 / conv3 weight gradients as per-CTA partial rows over fixed tile sets, summed in row order.

Also the seeded inputs of the fixture cases (tools/gen_golden_appearance.py -> tests/golden/fused_appearance.npz): the
network's ~250 k parameters are regenerated here from a seed rather than stored, and checked against the fixture's digest."""
import hashlib

import numpy as np

TW, TH, NCTA = 30, 14, 264                 # the kernels' pixel tile and CTA count (RGS_APPEARANCE_CTAS)
PARAM_SHAPES = [(256, 67, 3, 3), (256,), (128, 64, 3, 3), (128,), (64, 32, 3, 3), (64,), (32, 16, 3, 3), (32,), (16, 8, 3, 3), (16,),
                (16, 16, 3, 3), (16,), (3, 16, 3, 3), (3,)]
PARAM_NAMES = ["conv1.weight", "conv1.bias"] + [f"up{i}.conv.{k}" for i in range(1, 5) for k in ("weight", "bias")] + \
              ["conv2.weight", "conv2.bias", "conv3.weight", "conv3.bias"]
# seeds chosen so that every ReLU input lies at least RELU_MARGIN x its layer's largest magnitude away from 0: nearer than that,
# fp32 rounding in any summation order can flip the mask, and a flipped mask is not an error of either implementation
CASES = {"odd_offsets": (67, 67, 13), "one_sample_axis": (35, 64, 12), "ragged_tiles": (71, 99, 93)}
RELU_MARGIN = 3e-6
VIEW_IDX = 5
# The fixture keeps it under half a megabyte: loss, d_image, d(embedding row), the tail's and the biases' gradients whole; the head's
# weight gradients and the transformed image (whose final resize is F.interpolate on both sides) at SUBSET fixed indices each.
SUBSET = 1024


def make_inputs(case):
    """image, gt [3,H0,W0]; embedding table [8,64] (std 0.5, far from the reference's 1e-4 init); the 14 parameters (He-scaled
    weights, so about half the ReLUs are dead and the sigmoid's input is O(1)).  torch CPU generator: the same bits everywhere."""
    import torch
    H0, W0, seed = CASES[case]
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(3, H0, W0, generator=g)
    image = (0.8 * gt + 0.1 + 0.1 * torch.randn(3, H0, W0, generator=g)).clamp(0, 1)
    table = 0.5 * torch.randn(8, 64, generator=g)
    params = []
    for shp in PARAM_SHAPES:
        if len(shp) == 4:
            params.append(torch.randn(*shp, generator=g) * (2.0 / (shp[1] * 9)) ** 0.5)
        else:
            params.append(0.05 * torch.randn(*shp, generator=g))
    return {"image": image.numpy(), "gt": gt.numpy(), "table": table.numpy(), "params": [p.numpy() for p in params]}


def inputs_digest(inp):
    h = hashlib.sha256()
    for a in [inp["image"], inp["gt"], inp["table"], *inp["params"]]:
        h.update(np.ascontiguousarray(a, np.float32).tobytes())
    return h.hexdigest()


def load_fixture(path):
    """{case: {key: value}} with the float64 results restored: the file keeps them as float32 residuals against the float32 run."""
    raw = dict(np.load(path))
    out = {}
    for k, v in raw.items():
        case, key = k.split("/")
        if key.endswith("_f64d"):
            key, v = key[:-1], raw[f"{case}/{key[:-5]}"].astype(np.float64) + v
        out.setdefault(case, {})[key] = v
    return out


def recorded(name, a):
    """What the fixture keeps of output `name` (a key of forward_backward, or a parameter name for a gradient)."""
    a = np.asarray(a)
    if (name == "transformed" or (a.ndim == 4 and name in PARAM_NAMES[:10])) and a.size > SUBSET:
        return a.reshape(-1)[subset_indices(a.shape)]
    return a


def subset_indices(shape, k=SUBSET):
    n = int(np.prod(shape))
    return np.random.default_rng(n).choice(n, size=min(k, n), replace=False)


# ---- geometry ------------------------------------------------------------------------------------------------------------

def crop_box(H0, W0):
    H, W = H0 // 32 * 32, W0 // 32 * 32
    return H0 // 2 - H // 2, W0 // 2 - W // 2, H, W


def interp_matrix(n_in, n_out):
    """[n_out, n_in]: bilinear, align_corners=True; source = scale * dst with scale = (in-1)/(out-1), 0 for one sample."""
    scale = (n_in - 1) / (n_out - 1) if n_out > 1 else 0.0
    R = np.zeros((n_out, n_in))
    for d in range(n_out):
        s = scale * d
        i0 = int(s)
        step = 1 if i0 < n_in - 1 else 0
        R[d, i0] += 1.0 - (s - i0)
        R[d, i0 + step] += s - i0
    return R


def resample(x, Ry, Rx):                          # x [C, in_h, in_w] -> [C, out_h, out_w]
    return np.einsum("yi,cij,xj->cyx", Ry, x, Rx)


def resample_T(g, Ry, Rx):                        # the transpose: each input sample gathers the outputs its taps feed
    return np.einsum("yi,cyx,xj->cij", Ry, g, Rx)


# ---- convolutions --------------------------------------------------------------------------------------------------------

def conv(x, w, b):
    _, H, W = x.shape
    xp = np.pad(x, ((0, 0), (1, 1), (1, 1)))
    out = np.zeros((w.shape[0], H, W))
    for dy in range(3):
        for dx in range(3):
            out += np.einsum("oc,chw->ohw", w[:, :, dy, dx], xp[:, dy:dy + H, dx:dx + W])
    return out + b[:, None, None]


def conv_T(g, w):
    """d(input) = the transposed convolution: taps mirrored over d(output) with a 1-pixel zero border."""
    _, H, W = g.shape
    gp = np.pad(g, ((0, 0), (1, 1), (1, 1)))
    out = np.zeros((w.shape[1], H, W))
    for dy in range(3):
        for dx in range(3):
            out += np.einsum("oc,ohw->chw", w[:, :, dy, dx], gp[:, 2 - dy:2 - dy + H, 2 - dx:2 - dx + W])
    return out


def conv_wgrad(g, x):
    _, H, W = g.shape
    xp = np.pad(x, ((0, 0), (1, 1), (1, 1)))
    dw = np.zeros((g.shape[0], x.shape[0], 3, 3))
    for dy in range(3):
        for dx in range(3):
            dw[:, :, dy, dx] = np.einsum("ohw,chw->oc", g, xp[:, dy:dy + H, dx:dx + W])
    return dw, g.sum(axis=(1, 2))


def conv_wgrad_partials(g, x):
    """conv_wgrad as the backward kernel sums it: CTA b owns tiles b, b + NCTA, ...; one partial row per CTA; rows in order."""
    _, H, W = g.shape
    tx, ty = -(-W // TW), -(-H // TH)
    rows_w = np.zeros((NCTA, g.shape[0], x.shape[0], 3, 3))
    rows_b = np.zeros((NCTA, g.shape[0]))
    xp = np.pad(x, ((0, 0), (1, 1), (1, 1)))
    for t in range(tx * ty):
        y0, x0 = (t // tx) * TH, (t % tx) * TW
        gt = g[:, y0:y0 + TH, x0:x0 + TW]
        xt = xp[:, y0:y0 + gt.shape[1] + 2, x0:x0 + gt.shape[2] + 2]
        dw, db = _tile_wgrad(gt, xt)
        rows_w[t % NCTA] += dw
        rows_b[t % NCTA] += db
    return rows_w.sum(axis=0), rows_b.sum(axis=0)


def _tile_wgrad(g, xp_tile):
    _, h, w = g.shape
    dw = np.zeros((g.shape[0], xp_tile.shape[0], 3, 3))
    for dy in range(3):
        for dx in range(3):
            dw[:, :, dy, dx] = np.einsum("ohw,chw->oc", g, xp_tile[:, dy:dy + h, dx:dx + w])
    return dw, g.sum(axis=(1, 2))


def pixel_shuffle(x):                            # [4C, h, w] -> [C, 2h, 2w]
    C4, h, w = x.shape
    return x.reshape(C4 // 4, 2, 2, h, w).transpose(0, 3, 1, 4, 2).reshape(C4 // 4, 2 * h, 2 * w)


def pixel_unshuffle(x):                          # its inverse (and transpose)
    C, H, W = x.shape
    return x.reshape(C, H // 2, 2, W // 2, 2).transpose(0, 2, 4, 1, 3).reshape(4 * C, H // 2, W // 2)


def relu_margin(inp):
    """Smallest |ReLU input| / max |ReLU input| over the six ReLU layers, in fp64."""
    m = forward_backward(inp["image"], inp["gt"], inp["table"][VIEW_IDX], inp["params"])
    return min(np.abs(z).min() / np.abs(z).max() for z in m["pre"])


# ---- the loss ------------------------------------------------------------------------------------------------------------

def forward_backward(image, gt, emb, params, upstream=1.0):
    """Returns loss, d_image, d_emb, the 14 parameter gradients, transformed (mapping * crop resized to the image, as the
    reference returns it) and the intermediate maps."""
    image, gt, emb = (np.asarray(a, np.float64) for a in (image, gt, emb))
    p = [np.asarray(a, np.float64) for a in params]
    _, H0, W0 = image.shape
    top, left, H, W = crop_box(H0, W0)
    crop, crop_gt = image[:, top:top + H, left:left + W], gt[:, top:top + H, left:left + W]
    h, w = H // 32, W // 32
    Dy, Dx = interp_matrix(H, h), interp_matrix(W, w)
    down = resample(crop, Dy, Dx)
    x0 = np.concatenate([down, np.broadcast_to(emb[:, None, None], (64, h, w))], axis=0)
    # head
    acts = [x0]
    z = conv(x0, p[0], p[1])
    a = np.maximum(z, 0)
    pre = [z]
    ins = [x0]
    for k in range(4):
        s = pixel_shuffle(a)
        ins.append(s)
        z = conv(s, p[2 + 2 * k], p[3 + 2 * k])
        pre.append(z)
        a = np.maximum(z, 0)
    up4 = a
    Uy, Ux = interp_matrix(H // 2, H), interp_matrix(W // 2, W)
    X = resample(up4, Uy, Ux)
    Z = conv(X, p[10], p[11])
    pre.append(Z)
    A = np.maximum(Z, 0)
    S = conv(A, p[12], p[13])
    M = 1.0 / (1.0 + np.exp(-S))
    T = M * crop
    n = T.size
    loss = np.abs(T - crop_gt).mean() * upstream
    # tail backward
    dT = np.sign(T - crop_gt) * (upstream / n)
    d_image = np.zeros_like(image)
    d_image[:, top:top + H, left:left + W] = dT * M
    dS = dT * crop * (1.0 - M) * M
    dW3, db3 = conv_wgrad_partials(dS, A)
    dZ = conv_T(dS, p[12]) * (A > 0)
    dW2, db2 = conv_wgrad_partials(dZ, X)
    dX = conv_T(dZ, p[10])
    d_a = resample_T(dX, Uy, Ux)
    # head backward
    grads = [None] * 14
    grads[10], grads[11], grads[12], grads[13] = dW2, db2, dW3, db3
    for k in range(3, -1, -1):
        dz = d_a * (pre[k + 1] > 0)
        grads[2 + 2 * k], grads[3 + 2 * k] = conv_wgrad(dz, ins[k + 1])
        d_a = pixel_unshuffle(conv_T(dz, p[2 + 2 * k]))
    dz = d_a * (pre[0] > 0)
    grads[0], grads[1] = conv_wgrad(dz, x0)
    d_x0 = conv_T(dz, p[0])
    d_emb = d_x0[3:].sum(axis=(1, 2))
    d_image[:, top:top + H, left:left + W] += resample_T(d_x0[:3], Dy, Dx)
    transformed = resample(T, interp_matrix(H, H0), interp_matrix(W, W0))
    return {"loss": loss, "d_image": d_image, "d_emb": d_emb, "grads": grads, "transformed": transformed, "up4": up4, "mapping": M, "pre": pre}

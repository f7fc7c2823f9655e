"""Decoupled-appearance L1 loss of the DTU and Tanks and Temples recipes (``train.py --use_decoupled_appearance``), fused.

``L1_loss_appearance(image, gt_image, gaussians, view_idx, return_transformed_image=False)`` has the signature and meaning of
the reference's function (train.py:37-58, from Gaussian Opacity Fields): center-crop the render to a multiple of 32, downsample
it by 32, append the view's appearance embedding, run ``gaussians.appearance_network`` (scene/appearance_network.py) and take
the L1 of ``mapping * crop`` against the ground truth's crop.

The whole network and the loss run in the project's kernels, in FP32 without tensor cores: the crop and downsample, the x2
upsample, conv2 + ReLU, conv3 + sigmoid and the loss in csrc/rgs_appearance.cu, the low-resolution head (conv1, relu, up1..up4)
in csrc/rgs_appearance_head.cu.  Every backward sum has a fixed order and there are no float atomics: two calls give identical
bits, whatever torch's cuDNN and TF32 settings, where torch's bilinear backward accumulates with atomics.
Gradients reach the module's parameters, the embedding table row ``view_idx`` and the image, as autograd would deliver them.
No CPU path: CUDA tensors only.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from diff_gaussian_rasterization import _C

__all__ = ["L1_loss_appearance"]


# GOF's head (scene/appearance_network.py): conv1, then up1..up4's convolutions after each PixelShuffle(2)
_HEAD_LAYERS = (("conv1", 67, 256), ("up1", 64, 128), ("up2", 32, 64), ("up3", 16, 32), ("up4", 8, 16))


def _head_convs(net):
    return [(name, getattr(net, name, None) if name == "conv1" else getattr(getattr(net, name, None), "conv", None), cin, cout)
            for name, cin, cout in _HEAD_LAYERS]


def _head_params(net):
    """conv1.weight, conv1.bias, up1.conv.weight, ..., up4.conv.bias: the module's parameter order."""
    return [p for _, conv, _, _ in _head_convs(net) for p in (conv.weight, conv.bias)]


def _check_network(net):
    tail = [(name, getattr(net, name, None), cin, cout) for name, cin, cout in (("conv2", 16, 16), ("conv3", 16, 3))]
    for name, conv, cin, cout in tail + _head_convs(net):
        w = getattr(conv, "weight", None)
        if w is None or tuple(w.shape) != (cout, cin, 3, 3) or getattr(conv, "bias", None) is None:
            raise ValueError(f"appearance network: {name} must be a {cin} -> {cout} 3x3 convolution with bias, got "
                             f"{None if w is None else tuple(w.shape)}")


def _embedding(gaussians, view_idx):
    emb = gaussians.get_apperance_embedding(view_idx)
    if tuple(emb.shape) != (64,):
        raise ValueError(f"appearance embedding: the view's row must hold 64 values, got {tuple(emb.shape)}")
    return emb


def _check_images(image, gt):
    if gt.requires_grad:
        raise ValueError("L1_loss_appearance differentiates w.r.t. the rendered image, not the ground truth")
    if image.dim() != 3 or image.shape[0] != 3 or image.shape[1] < 32 or image.shape[2] < 32:
        raise ValueError(f"L1_loss_appearance needs a [3, H, W] image with H, W >= 32, got {tuple(image.shape)}")
    if gt.shape != image.shape:
        raise ValueError(f"gt_image {tuple(gt.shape)} must have the image's shape {tuple(image.shape)}")
    if not (image.is_cuda and gt.is_cuda):
        raise RuntimeError("L1_loss_appearance needs CUDA tensors: there is no CPU path")


def _head(net, x):
    """The head as the module's own layers (for row stages without a fused head, multigpu's CPU stand-ins)."""
    x = net.relu(net.conv1(x))
    return net.up4(net.up3(net.up2(net.up1(x))))


def _head_input(down, emb):
    h, w = down.shape[1:]
    return torch.cat([down, emb[:, None, None].expand(emb.shape[0], h, w)], dim=0)[None]


class _AppearanceL1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, gt, emb, net, *params):
        image, gt = image.contiguous(), gt.contiguous()
        down, emb = _C.appearance_downsample(image), emb.detach()
        head = [p.detach() for p in params[:-4]]
        head_act, up4 = _C._appearance_head.forward(down, emb, head)
        w2, b2, w3, b3 = net.conv2.weight, net.conv2.bias, net.conv3.weight, net.conv3.bias
        loss, act, _ = _C.appearance_l1_forward(image, gt, up4, w2.detach(), b2.detach(), w3.detach(), b3.detach(), True, False)
        ctx.save_for_backward(image, gt, act, w2.detach(), b2.detach(), w3.detach(), b3.detach(), down, emb, head_act, up4, *head)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        image, gt, act, w2, b2, w3, b3, down, emb, head_act, up4, *head = ctx.saved_tensors
        d_img, d_up4, d_w2, d_b2, d_w3, d_b3 = _C.appearance_l1_backward(image, gt, up4, act, w2, b2, w3, b3, grad_out.float().reshape(1))
        grads = _C._appearance_head.backward(down, emb, head, head_act, up4, d_up4)
        _C.appearance_downsample_backward(grads[0], d_img)
        return (d_img, None, grads[1], None, *grads[2:], d_w2, d_b2, d_w3, d_b3)


def L1_loss_appearance(image: torch.Tensor, gt_image: torch.Tensor, gaussians, view_idx, return_transformed_image: bool = False):
    """train.py:37-58.  Returns the loss (a device scalar, no host synchronisation), or with ``return_transformed_image=True``
    the reference's transformed image (``mapping * crop`` resized back to the image size; forward only)."""
    net = gaussians.appearance_network
    _check_network(net)
    emb = _embedding(gaussians, view_idx)
    _check_images(image, gt_image)
    if not return_transformed_image:
        params = _head_params(net) + [net.conv2.weight, net.conv2.bias, net.conv3.weight, net.conv3.bias]
        if len(params) != len(list(net.parameters())):
            raise ValueError("appearance network: parameters outside conv1, up1..up4, conv2 and conv3 are not supported")
        return _AppearanceL1.apply(image, gt_image, emb, net, *params)
    with torch.no_grad():
        image, gt_image = image.contiguous(), gt_image.contiguous()
        _, up4 = _C._appearance_head.forward(_C.appearance_downsample(image), emb, _head_params(net))
        _, _, t = _C.appearance_l1_forward(image, gt_image, up4, net.conv2.weight, net.conv2.bias, net.conv3.weight, net.conv3.bias, False, True)
        return F.interpolate(t[None], size=tuple(image.shape[1:]), mode="bilinear", align_corners=True)[0]

"""Decoupled appearance (SURVEY.md 8(a) row a27, BASELINE config 4): the reference's AppearanceNetwork
(scene/appearance_network.py:18-46) and L1_loss_appearance (train.py:67-88) -- callers of the rasterizer, the only
GEMM-shaped math on the path.

Same module structure and parameter names as the reference (conv1, up1.conv ... up4.conv, conv2, conv3), so a reference
checkpoint's `appearance_network` state_dict loads unchanged.  Forward and data gradients of the convolutions run through torch
(cuDNN; TF32 tensor-core math is the reference's own default, torch.backends.cudnn.allow_tf32); the WEIGHT gradients of the
few-channel layers at (near) full resolution -- where cuDNN's generic fp32 engine took 40 % of the appearance step -- come from
the library's own kernel (csrc/conv_wgrad.cu, `_Conv3x3`).  DESIGN.md states the measured share of a C4 step.
What this module adds over the reference's formulation: the per-view tensors the loss re-creates every iteration (crop window,
the embedding broadcast to the 1/32 grid) are built without the `repeat().permute()` copy, and `appearance_grads_flat` /
`load_flat_grads_` pack the network's and the embedding's gradients into the view-parallel gradient bucket
(gof_dp.GradBucket(extra_sum=...)) so that they travel in the same exchange as the Gaussian gradients."""
import ctypes
import os

import torch
import torch.nn as nn
import torch.nn.functional as F

# A/B switches (developer use): GOF_APP_WGRAD=0 -> cuDNN's weight gradients, GOF_APP_NHWC=1 -> channels-last activations
_USE_WGRAD = os.environ.get("GOF_APP_WGRAD", "1") != "0"
_USE_NHWC = os.environ.get("GOF_APP_NHWC", "0") == "1"
_WGRAD_PAIRS = {(16, 16), (3, 16), (16, 8)}          # (C_out, C_in) pairs csrc/conv_wgrad.cu is instantiated for
_lib = None


def _wgrad_lib():
    global _lib
    if _lib is None:
        from diff_gaussian_rasterization import _C
        _lib = _C._lib
        _lib.gof_conv3x3_wgrad.restype = ctypes.c_int
        _lib.gof_conv3x3_wgrad.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p] * 5
    return _lib


class _Conv3x3(torch.autograd.Function):
    """3x3 / stride 1 / pad 1 convolution whose WEIGHT and BIAS gradients come from the library's kernel (csrc/conv_wgrad.cu):
    for the few-channel, full-resolution layers at the network's tail cuDNN falls back to a generic fp32 weight-gradient engine
    that takes longer than the network's whole forward.  Forward and data
    gradient stay on cuDNN."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        ctx.save_for_backward(x, weight)
        return F.conv2d(x, weight, bias, padding=1)

    @staticmethod
    def backward(ctx, gy):
        from diff_gaussian_rasterization import _C
        x, weight = ctx.saved_tensors
        gx = torch.nn.grad.conv2d_input(x.shape, weight, gy, padding=1) if ctx.needs_input_grad[0] else None
        xc, gc = x.detach().contiguous(), gy.contiguous()
        dW = torch.zeros_like(weight, memory_format=torch.contiguous_format)
        db = torch.zeros(weight.shape[0], dtype=weight.dtype, device=weight.device)
        with torch.cuda.device(x.device):
            _C._check(_wgrad_lib().gof_conv3x3_wgrad(int(weight.shape[0]), int(weight.shape[1]), int(x.shape[2]), int(x.shape[3]), xc.data_ptr(),
                                                     gc.data_ptr(), dW.data_ptr(), db.data_ptr(), _C._stream()))
        return gx, dW, db


def conv3x3(x, conv):
    """`conv(x)` for an nn.Conv2d(3x3, stride 1, pad 1), through _Conv3x3 when its weight gradient is worth taking over."""
    w = conv.weight
    if (_USE_WGRAD and x.is_cuda and x.dtype == torch.float32 and x.shape[0] == 1 and (int(w.shape[0]), int(w.shape[1])) in _WGRAD_PAIRS
            and x.shape[2] * x.shape[3] >= 128 * 128 and conv.bias is not None and torch.is_grad_enabled() and w.requires_grad):
        return _Conv3x3.apply(x, w, conv.bias)
    return conv(x)


class UpsampleBlock(nn.Module):   # scene/appearance_network.py:5-16
    def __init__(self, num_input_channels, num_output_channels):
        super().__init__()
        self.pixel_shuffle = nn.PixelShuffle(2)
        self.conv = nn.Conv2d(num_input_channels // 4, num_output_channels, 3, stride=1, padding=1)
        self.relu = nn.ReLU()

    def forward(self, x):
        return self.relu(conv3x3(self.pixel_shuffle(x), self.conv))


class AppearanceNetwork(nn.Module):   # scene/appearance_network.py:18-46
    def __init__(self, num_input_channels, num_output_channels):
        super().__init__()
        self.conv1 = nn.Conv2d(num_input_channels, 256, 3, stride=1, padding=1)
        self.up1 = UpsampleBlock(256, 128)
        self.up2 = UpsampleBlock(128, 64)
        self.up3 = UpsampleBlock(64, 32)
        self.up4 = UpsampleBlock(32, 16)
        self.conv2 = nn.Conv2d(16, 16, 3, stride=1, padding=1)
        self.conv3 = nn.Conv2d(16, num_output_channels, 3, stride=1, padding=1)
        self.relu = nn.ReLU()
        self.sigmoid = nn.Sigmoid()

    def forward(self, x):
        if x.is_cuda and _USE_NHWC:      # no gain measured (cuDNN converts back and forth around its NCHW engines)
            x = x.contiguous(memory_format=torch.channels_last)
        x = self.relu(self.conv1(x))
        x = self.up4(self.up3(self.up2(self.up1(x))))
        x = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)
        x = self.relu(conv3x3(x, self.conv2))
        return self.sigmoid(conv3x3(x, self.conv3))


def crop_window(origH, origW):
    """train.py:70-75: the centred crop to multiples of 32."""
    H, W = origH // 32 * 32, origW // 32 * 32
    left, top = origW // 2 - W // 2, origH // 2 - H // 2
    return top, left, H, W


def l1_loss_appearance(image, gt_image, network, appearance_embedding, return_transformed_image=False):
    """L1_loss_appearance (train.py:67-88) with the model pieces passed explicitly: `appearance_embedding` is the view's row
    of GaussianModel._appearance_embeddings (64 floats), `network` the AppearanceNetwork."""
    origH, origW = image.shape[1:]
    top, left, H, W = crop_window(origH, origW)
    crop_image = image[:, top:top + H, left:left + W]
    crop_gt_image = gt_image[:, top:top + H, left:left + W]
    crop_image_down = F.interpolate(crop_image[None], size=(H // 32, W // 32), mode="bilinear", align_corners=True)[0]
    emb = appearance_embedding.reshape(-1, 1, 1).expand(-1, H // 32, W // 32)      # the reference: repeat(H/32, W/32, 1).permute(2, 0, 1)
    mapping_image = network(torch.cat([crop_image_down, emb], dim=0)[None])
    transformed_image = mapping_image * crop_image
    if not return_transformed_image:
        return torch.abs(transformed_image - crop_gt_image).mean()            # utils/loss_utils.py:17-18 l1_loss
    return F.interpolate(transformed_image, size=(origH, origW), mode="bilinear", align_corners=True)[0]


def appearance_numel(network, n_embedding=64):
    return sum(p.numel() for p in network.parameters()) + int(n_embedding)


def appearance_grads_flat(network, embedding_grad, out):
    """Packs d loss / d (network parameters, this view's embedding row) into the flat tensor `out` (the `extra` view of a
    gof_dp.GradBucket) in parameter order followed by the embedding row."""
    off = 0
    for p in network.parameters():
        n = p.numel()
        if p.grad is not None:
            out[off:off + n].copy_(p.grad.reshape(-1))
        else:
            out[off:off + n].zero_()
        off += n
    out[off:off + embedding_grad.numel()].copy_(embedding_grad.reshape(-1))
    return out


def load_flat_grads_(network, flat):
    """Inverse of appearance_grads_flat for the network part: writes the exchanged sums back into .grad; returns the
    embedding-row gradient slice."""
    off = 0
    for p in network.parameters():
        n = p.numel()
        p.grad = flat[off:off + n].view_as(p).clone()
        off += n
    return flat[off:]

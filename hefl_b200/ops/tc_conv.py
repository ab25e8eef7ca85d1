"""ResNet convolutions on the hand-written tensor-core GEMM kernels (csrc/nn/gemm_tcgen05.cu): 1x1 (any stride, by
sub-sampling first) and 3x3 / pad 1 / stride 1, forward, dgrad and wgrad, bf16 with fp32 accumulation; the 1x1
forward can run in e4m3 (wgmma e4m3) with per-tensor delayed scaling.

Layout: activations are channels_last bf16, i.e. ``[pixels, C]`` matrices. A 3x3 convolution works on a
zero-padded copy ``[B, H+2, W+2, C]``: tap (r, s) is the same matrix shifted by ``(r-1)*(W+2) + (s-1)`` rows, so
the nine tap GEMMs accumulate in one register tile with nothing but a different TMA row coordinate (no im2col).

What stays on cuDNN: the 7x7 stem (3 input channels) and the three 3x3 stride-2 convolutions of a ResNet.

Replaces the convolutions Keras/TF run for the reference's ``model.fit`` (FLPyfhelin.py:193) for the scaled-up
model family of BASELINE.json configs[2] and [4].
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _ext
from . import fp8 as _fp8

ENABLE = False          # module-level default; ``set_model_tc`` switches single models


def set_model_tc(model: nn.Module, on: bool) -> int:
    """Route every eligible convolution of ``model`` through the tcgen05 kernels (or back). Returns the count."""
    n = 0
    for m in model.modules():
        if isinstance(m, (Conv3x3, _fp8.Conv1x1)):
            m.use_tc = bool(on)
            n += 1
    return n


def _nhwc2d(x: torch.Tensor) -> torch.Tensor:
    """[B,C,H,W] channels_last -> zero-copy [B*H*W, C]."""
    B, C, H, W = x.shape
    return x.permute(0, 2, 3, 1).reshape(B * H * W, C)


def _as_nchw(y2: torch.Tensor, B: int, H: int, W: int) -> torch.Tensor:
    return y2.view(B, H, W, -1).permute(0, 3, 1, 2)            # channels_last strides


def eligible(x: torch.Tensor, cin: int, cout: int) -> bool:
    return (x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 4 and cin % 64 == 0 and cout % 64 == 0
            and x.is_contiguous(memory_format=torch.channels_last))


class _Conv1x1TC(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, fp8_state):
        ops = _ext.ops()
        B, Cin, H, W = x.shape
        Cout = w.shape[0]
        x2 = _nhwc2d(x)
        wb, wT = ops.conv_weight_prep(w.detach().contiguous())            # [Cout,Cin] and its transpose, one launch
        y2 = torch.empty(B * H * W, Cout, dtype=torch.bfloat16, device=x.device)
        mx = fp8_state == "mx" and Cin % 128 == 0 and Cout % 128 == 0
        if mx:
            # block-scaled e4m3 (kind::mxf8f6f4.block_scale): one UE8M0 scale per row and 32 channels, no amax history
            xq, xs = ops.mxfp8_quantize(x2 if x2.is_contiguous() else x2.contiguous())
            wq, ws = ops.mxfp8_quantize(wb)
            ops.gemm_mxfp8(xq, wq, xs, ws, y2)
        elif fp8_state is not None and fp8_state != "mx" and Cin % 128 == 0:   # per-tensor delayed scaling (kind::f8f6f4)
            sx, sw = fp8_state
            xq = _fp8._quantize(x2, sx).view(torch.uint8)
            wq = _fp8._quantize(wb, sw).view(torch.uint8)
            ops.gemm_taps(xq, wq, y2, Cout, Cin, [], 0, 0, 0, 0, sx.inv, sw.inv)
        else:
            ops.gemm_taps(x2, wb, y2, Cout, Cin, [], 0, 0, 0, 0, None, None)
        ctx.save_for_backward(x2, wT)
        ctx.shape = (B, Cin, H, W, Cout)
        ctx.mx = mx
        return _as_nchw(y2, B, H, W)

    @staticmethod
    def backward(ctx, gy):
        ops = _ext.ops()
        x2, wT = ctx.saved_tensors
        B, Cin, H, W, Cout = ctx.shape
        g2 = gy.permute(0, 2, 3, 1).reshape(B * H * W, Cout)
        if g2.dtype != torch.bfloat16 or not g2.is_contiguous():
            g2 = g2.to(torch.bfloat16).contiguous()
        dx2 = torch.empty(B * H * W, Cin, dtype=torch.bfloat16, device=gy.device)
        if ctx.mx:                                                                              # dX = dY . W, block-scaled
            gq, gs = ops.mxfp8_quantize(g2)
            tq, ts = ops.mxfp8_quantize(wT)
            ops.gemm_mxfp8(gq, tq, gs, ts, dx2)
        else:
            ops.gemm_taps(g2, wT, dx2, Cin, Cout, [], 0, 0, 0, 0, None, None)                   # dX = dY . W
        dw = torch.empty(1, Cout, Cin, dtype=torch.float32, device=gy.device)
        ops.wgrad_taps(g2, x2, dw, 1, 0)                                                       # dW = dY^T . X
        return _as_nchw(dx2, B, H, W), dw.view(Cout, Cin, 1, 1), None


def _shifts(Wp: int):
    return [(r - 1) * Wp + (s - 1) for r in range(3) for s in range(3)]


class _Conv3x3TC(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w):
        ops = _ext.ops()
        B, Cin, H, W = x.shape
        Cout = w.shape[0]
        xp = ops.pad_nhwc(x)                                          # [B, H+2, W+2, Cin], zero border, one pass
        # wt [tap][Cout][Cin] for the forward; wd [tap][Cin][Cout] = filter rotated by 180 degrees, for dgrad
        wt, wd = ops.conv_weight_prep(w.detach().contiguous())
        y2 = torch.empty(B * H * W, Cout, dtype=torch.bfloat16, device=x.device)
        ops.gemm_taps(xp.view(-1, Cin), wt, y2, Cout, Cin, _shifts(W + 2), 1, B, H, W, None, None)
        ctx.save_for_backward(xp, wd)
        ctx.shape = (B, Cin, H, W, Cout)
        return _as_nchw(y2, B, H, W)

    @staticmethod
    def backward(ctx, gy):
        ops = _ext.ops()
        xp, wd = ctx.saved_tensors
        B, Cin, H, W, Cout = ctx.shape
        if gy.dtype != torch.bfloat16 or not gy.is_contiguous(memory_format=torch.channels_last):
            gy = gy.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        gp = ops.pad_nhwc(gy)                                         # [B, H+2, W+2, Cout]
        # dX = conv(dY, W rotated by 180 degrees, channels swapped): tap (r, s) -> W[:, :, 2-r, 2-s]^T
        dx2 = torch.empty(B * H * W, Cin, dtype=torch.bfloat16, device=gy.device)
        ops.gemm_taps(gp.view(-1, Cout), wd, dx2, Cin, Cout, _shifts(W + 2), 1, B, H, W, None, None)
        dw = torch.empty(9, Cout, Cin, dtype=torch.float32, device=gy.device)
        ops.wgrad_taps(gp.view(-1, Cout), xp.view(-1, Cin), dw, 9, W + 2)
        return _as_nchw(dx2, B, H, W), ops.conv_wgrad_unpack(dw, Cout, Cin, 3)


def conv1x1(x: torch.Tensor, w: torch.Tensor, stride: int = 1, fp8_state=None) -> torch.Tensor:
    if stride > 1:
        x = x[:, :, ::stride, ::stride].contiguous(memory_format=torch.channels_last)
    return _Conv1x1TC.apply(x, w, fp8_state)


def conv3x3(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    return _Conv3x3TC.apply(x, w)


class Conv3x3(nn.Conv2d):
    """3x3 / pad 1 convolution without bias: the tcgen05 tap-GEMM when switched on and the input qualifies
    (CUDA, channels_last bf16, channel counts multiples of 64, stride 1), a regular ``nn.Conv2d`` otherwise."""

    def __init__(self, cin: int, cout: int, stride: int = 1):
        super().__init__(cin, cout, 3, stride, 1, bias=False)
        self.use_tc: Optional[bool] = None

    def forward(self, x):
        on = ENABLE if self.use_tc is None else self.use_tc
        if on and self.stride[0] == 1 and eligible(x, self.in_channels, self.out_channels):
            return conv3x3(x, self.weight)
        return super().forward(x)

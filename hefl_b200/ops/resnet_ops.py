"""ResNet building blocks on hand-written sm_90a kernels (SURVEY.md K18): training-mode
BatchNorm over NHWC bf16 fused with the residual add and ReLU (forward and backward, 5 kernels
per BN layer and direction instead of cuDNN BN + add + ReLU + their autograd nodes) and global
average pooling. The convolutions of the ResNets stay on cuDNN (library GEMMs); everything
memory-bound around them runs here.

``bn_act`` falls back to ``F.batch_norm`` whenever the fused path does not apply (CPU, eval
mode, fp32 or NCHW-contiguous activations), so models built on it run anywhere.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _ext


ENABLE = True     # tests flip this to compare against the cuDNN/ATen path


def _v(x: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """Zero-copy [B,H,W,C] view of a channels_last tensor (what the kernels index)."""
    return None if x is None else x.permute(0, 2, 3, 1)


def _nhwc(x: torch.Tensor) -> bool:
    return x.dim() == 4 and x.is_contiguous(memory_format=torch.channels_last)


class _BNActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, res, gamma, beta, run_mean, run_var, momentum, eps, relu):
        ops = _ext.ops()
        C = x.shape[1]
        y = torch.empty_like(x)                       # keeps channels_last strides
        stats = torch.empty(4 * C, dtype=torch.float32, device=x.device)
        mean, invstd, sums = stats[:C], stats[C:2 * C], stats[2 * C:]
        ops.bn_forward(_v(x), _v(res), gamma, beta, run_mean, run_var, mean, invstd, sums, _v(y), momentum, eps, relu)
        ctx.save_for_backward(x, y, mean, invstd, gamma)
        ctx.relu = relu
        ctx.has_res = res is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        ops = _ext.ops()
        x, y, mean, invstd, gamma = ctx.saved_tensors
        C = x.shape[1]
        if dy.dtype != torch.bfloat16 or not _nhwc(dy):
            dy = dy.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        dx = torch.empty_like(x)
        dres = torch.empty_like(x) if ctx.has_res else None
        sums = torch.empty(2 * C, dtype=torch.float32, device=x.device)
        ops.bn_backward(_v(dy), _v(x), _v(y), mean, invstd, gamma, sums, _v(dx), _v(dres), ctx.relu)
        return dx, dres, sums[C:], sums[:C], None, None, None, None, None


def bn_act(bn: nn.BatchNorm2d, x: torch.Tensor, res: Optional[torch.Tensor] = None, relu: bool = True) -> torch.Tensor:
    """``relu(bn(x) + res)`` with the fused kernels when possible."""
    fused = (ENABLE and x.is_cuda and bn.training and x.dtype == torch.bfloat16 and _nhwc(x) and x.shape[1] % 8 == 0
             and x.shape[1] <= 2048 and (res is None or (res.dtype == torch.bfloat16 and _nhwc(res))))
    if fused:
        if bn.track_running_stats and bn.num_batches_tracked is not None:
            bn.num_batches_tracked.add_(1)
        return _BNActFn.apply(x, res, bn.weight, bn.bias, bn.running_mean if bn.track_running_stats else None,
                              bn.running_var if bn.track_running_stats else None,
                              bn.momentum if bn.momentum is not None else 0.1, bn.eps, relu)
    out = bn(x)
    if res is not None:
        out = out + res
    return F.relu(out) if relu else out


class _AvgPoolFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        ops = _ext.ops()
        B, C, H, W = x.shape
        out = torch.empty(B, C, dtype=torch.float32, device=x.device)
        ops.avgpool_forward(_v(x), out, B, H * W, C)
        ctx.shape = (B, C, H, W)
        return out

    @staticmethod
    def backward(ctx, dout):
        ops = _ext.ops()
        B, C, H, W = ctx.shape
        dx = torch.empty(B, C, H, W, dtype=torch.bfloat16, device=dout.device).contiguous(memory_format=torch.channels_last)
        ops.avgpool_backward(dout.float().contiguous(), _v(dx), B, H * W, C)
        return dx


def global_avgpool(x: torch.Tensor) -> torch.Tensor:
    """[B,C,H,W] -> [B,C] (fp32 on the fused path)."""
    if ENABLE and x.is_cuda and x.dtype == torch.bfloat16 and _nhwc(x):
        return _AvgPoolFn.apply(x)
    return F.adaptive_avg_pool2d(x, 1).flatten(1)

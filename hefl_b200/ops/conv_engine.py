"""Training engine for the sequential 3x3-conv CNNs on the hand-written sm_90a kernels.

Replaces Keras' ``model.fit`` compute path (FLPyfhelin.py:118-136, :193) for the medical CNN:

  input     preprocess_u8 (uint8 -> bf16 NHWC, 1/255, Philox affine augmentation; RGB: [P,4] = R, G, B, 0 by
            default (``compact0``), else [P,16] with pixels w, w+1, w+2 in its channels; grayscale: [P,16] with the
            whole 3x3 neighbourhood) into one of two X0 slots — the trainer stages batch i+1 on a side stream while
            step i runs
  forward   6 x conv_fwd_pool  (TMA-fed tensor-core tap GEMMs, bias + ReLU + 2x2 max-pool + 3-bit
                                arg-max/active code fused in the epilogue; only pooled tensors
                                reach HBM; layer 1 on the pair-row variant: the whole pooling window
                                in one thread)
            head_forward_backward (Dense 128-64-C + softmax CE, forward AND backward, one launch on a
                                   cluster of 8 CTAs)
  backward  unpool_relu / conv_dgrad chain on the main stream (layers 6..2),
            conv_wgrad (tensor cores, operands read in place, split-K partials added in a fixed order) on a
            side stream; layer 2 (CK = Co = 32 on the wide map): conv_dgrad_wgrad, both gradients from one pass
            over dY on the main stream,
            layer 1: wgrad0_gather straight from the pooled gradient (no un-pool, no dY tensor): four
                     masked GEMMs on the tensor cores (wgrad0_mma.cu), FP32-pipe gather as the fallback
  update    conv_grad_finalize + Adam + conv_weight_relayout: layers 2..6 and the head on the side
            stream under the layer-1 kernel, the 896 (RGB) or 320 (grayscale) layer-1 parameters in the
            tail (``opt`` hooks)
  head-only (personalised FL, ``head_step_staged``) forward convs without arg-max codes, the head kernel at the
            depth that yields the personal layers' gradients only, Adam over the personal layers
  Grad-CAM  (``gradcam_staged``, DESIGN.md §11) forward convs (arg-max codes from the explained stage on), the head
            seeded with a class score (head_saliency), the un-pool / dgrad chain down to that stage, gradcam
  IG        (``ig_staged``, DESIGN.md §12) per path point: the scan in slot 1 scaled into slot 0, forward convs
            with every arg-max code, the head seeded with a class score, the un-pool / dgrad chain down to X[1],
            input_grad0 (the layer-1 input gradient straight from the pooled gradient, into an fp32 accumulator)
  scoring   (``score_staged``, DESIGN.md §13) forward convs without arg-max codes, the head's logits (head_logits),
            score_stats (confusion matrix, score histograms and loss sum of one client)

All buffers are allocated once; a step is CUDA-graph capturable (one graph per input slot); every
kernel uses programmatic dependent launch (csrc/nn/launch.cuh).
"""
from __future__ import annotations

import os

import math
from typing import List

import torch
import torch.nn.functional as F

from .. import _ext
from ..config import FLConfig
from ..models.pack import ParamPack


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class MedCNNEngine:
    def __init__(self, model, pack: ParamPack, cfg: FLConfig, device: torch.device):
        if device.type != "cuda":
            raise RuntimeError("the tcgen05 engine needs a CUDA device (sm_90a)")
        self.ops = _ext.ops()
        self.model, self.pack, self.cfg, self.device = model, pack, cfg, device
        B, S = cfg.batch_size, cfg.image_size
        if cfg.in_channels not in (1, 3):
            raise ValueError(f"the tcgen05 engine supports 1- or 3-channel uint8 images, got in_channels={cfg.in_channels}")
        self.B = B
        convs = list(model.convs)
        if convs[0].in_channels != cfg.in_channels:
            raise ValueError(f"model has {convs[0].in_channels} input channels, config {cfg.in_channels}")
        self.n = len(convs)
        offs = {k: o for k, _, o, _ in pack.entries}
        keys = [k for k in pack.keras_order_keys()]
        conv_keys = [(f"c_{2 * i}_0", f"c_{2 * i}_1") for i in range(self.n)]
        self.H: List[int] = []
        self.Ci: List[int] = []
        self.CK: List[int] = []
        self.Co: List[int] = []
        h = S
        for i, c in enumerate(convs):
            ci, co = c.in_channels, c.out_channels
            ck = 16 if i == 0 else ci
            if ck not in (16, 32, 64) or co not in (32, 64, 128):
                raise ValueError(f"unsupported conv shape ({ci}->{co}) for the tcgen05 engine")
            self.H.append(h)
            self.Ci.append(ci)
            self.CK.append(ck)
            self.Co.append(co)
            h = (h - 2) // 2
        self.H.append(h)                 # feature map side
        # packed layer-1 input: RGB carries pixels (w, w+1, w+2) in its 16 channels, 3 tap-GEMMs instead of 9
        # (conv_tcgen05.cu TS=1); grayscale carries the whole 3x3 neighbourhood, one GEMM (rs layout, TS=kTapsRS)
        self.spack0 = (os.environ.get("HEFL_SPACK0", "1") != "0" and self.Ci[0] in (1, 3) and self.CK[0] == 16
                       and self.Co[0] == 32)
        # pair-row forward kernel (both columns of a pooling window in one thread, conv_tcgen05.cu G1b): on by
        # default for layer 1, where it reads the same s-packed input as the tap-GEMM forward (same outputs, tests).
        # On the small layers it runs one 128-window tile per pooled row, so HEFL_FWD_PAIR=all is only for experiments.
        mode = os.environ.get("HEFL_FWD_PAIR", "1")
        self.fwd_pair = {"0": 0, "1": 1, "all": self.n}.get(mode, 0)      # number of leading layers that may use it
        # layer-1 weight gradient by gather from the pooled gradient (csrc/nn/wgrad_gather.cu)
        self.gather_wgrad0 = (os.environ.get("HEFL_GATHER_WGRAD0", "1") != "0" and self.Co[0] == 32
                              and self.CK[0] == 16 and self.H[0] <= 256)
        self._wgrad0_mma = not os.environ.get("HEFL_WGRAD0_MMA", "1").startswith("0")     # as wgrad0_mma.cu reads it
        # layers whose data and weight gradients come from one pass over dY on the main stream (conv_dgrad_wgrad,
        # conv_tcgen05.cu G3): CK = Co = 32 on a map wider than 64 columns (layer 2), where the weight gradient on the
        # side stream was the step's tail. Same bits as conv_dgrad + conv_wgrad.
        self.dgrad_wgrad = [l > 0 and self.H[l] > 64 and self.CK[l] == 32 and self.Co[l] == 32
                            and self.ops.conv_dgrad_wgrad_supported(self.H[l], self.H[l], 32, 32)
                            for l in range(self.n)]
        bf = dict(dtype=torch.bfloat16, device=device)
        self.P = [B * self.H[l] * self.H[l] for l in range(self.n + 1)]
        # activations / gradients (all NHWC bf16 viewed as [pixels, channels])
        # layer-1 input with 8 pixels of slack: its wgrad reads 4-pixel windows (overlapping TMA rows)
        # two copies: batch i+1 is pre-processed into the other slot while step i trains (fl/trainer.py)
        # Sized for the 16-channel layouts, which the switches below may select at any time; the compact RGB layout
        # (``compact0``) uses the first quarter, so only the bytes it touches cost bandwidth.
        self._x0_bufs = [torch.zeros(self.P[0] + 8, 16, **bf) for _ in range(2)]
        self.X0 = [b[: self.P[0]] for b in self._x0_bufs]
        self._x0c = [b.view(-1)[: self.P[0] * 4].view(self.P[0], 4) for b in self._x0_bufs]
        self._x0_base = self._x0_bufs[0]
        self.X = [self.X0[0]]
        self.amax, self.dY, self.gX = [], [], [None]
        for l in range(self.n):
            hp = self.H[l + 1]
            self.X.append(torch.zeros(B * hp * hp, self.Co[l], **bf))
            self.amax.append(torch.zeros(B * hp * hp, self.Co[l], dtype=torch.uint8, device=device))
            # layer 1 normally takes the gather path (no conv-grid gradient at all): allocate lazily
            self.dY.append(None if l == 0 else torch.zeros(self.P[l], self.Co[l], **bf))
            self.gX.append(torch.zeros(B * hp * hp, self.Co[l], **bf))
        # weights
        wf_off, wd_off, dw_off = [0], [0], [0]
        for l in range(self.n):
            wf_off.append(wf_off[-1] + 9 * self.Co[l] * self.CK[l])
            wd_off.append(wd_off[-1] + 9 * self.Ci[l] * self.Co[l])
            dw_off.append(dw_off[-1] + (9 * self.CK[l] + 1) * self.Co[l])
        self.wf_off, self.wd_off, self.dw_off = wf_off, wd_off, dw_off
        self.Wf = torch.zeros(wf_off[-1], **bf)
        self.Wd = torch.zeros(wd_off[-1], **bf)
        self.dW32 = torch.zeros(dw_off[-1], dtype=torch.float32, device=device)
        self.shadow = torch.zeros(pack.n_trainable, **bf)
        rows = []
        self.b_off = []
        for l, (kw, kb) in enumerate(conv_keys):
            rows.append([self.Ci[l], self.CK[l], self.Co[l], offs[kw], offs[kb], wf_off[l], wd_off[l], dw_off[l]])
            self.b_off.append(offs[kb])
        self.table = torch.tensor(rows, dtype=torch.int64)
        self.bias = [pack.flat[self.b_off[l]: self.b_off[l] + self.Co[l]] for l in range(self.n)]
        # flat parameters [0, p0) belong to layer 1 (weights then bias come first in the pack)
        self.p0 = max(offs[conv_keys[0][0]] + 9 * self.Ci[0] * self.Co[0], self.b_off[0] + self.Co[0])
        if self.n > 1 and not (self.p0 <= offs[conv_keys[1][0]] and self.p0 <= self.b_off[1]):
            self.p0 = 0          # unexpected parameter order: never split the update
        # dense head: fused kernels when it is the reference's 3-layer shape, else PyTorch autograd
        fcs = list(model.fcs)
        self.fused_head = len(fcs) == 3 and B <= 32 and B % 2 == 0
        if self.fused_head:
            nfc = self.n * 2 + 1
            self.head_offs = []
            for i in range(3):
                self.head_offs += [offs[f"c_{nfc + i}_0"], offs[f"c_{nfc + i}_1"]]
            self.F, self.H1, self.H2, self.C = fcs[0].in_features, fcs[0].out_features, fcs[1].out_features, fcs[2].out_features
            self.h1_buf = torch.zeros(B * self.H1, dtype=torch.float32, device=device)
            self.dh1_buf = torch.zeros(B * (self.H1 + self.H2), dtype=torch.float32, device=device)
            self.dfeat = torch.zeros(B, self.F, **bf)
        # personal layers (DESIGN.md §10): a head-only step updates flat[head_lo:n_trainable]; the head kernel stops
        # after the last personal layer's gradient (depth 5 - p: 4 = dW3 only, 3 = dW2 and dW3, 2 = all, no dfeat)
        self.personal = int(cfg.personal_layers)
        self.head_lo = pack.dense_tail_start(self.personal) if self.personal else pack.n_trainable
        self.head_depth = 5 - self.personal
        self.theta = torch.zeros(B, 2, 3, dtype=torch.float32, device=device)
        self.aug_seed = (cfg.seed * 2654435761 + 12345) & 0x7FFFFFFFFFFFFFFF or 1
        self.prep_count = 0          # augmented batches pre-processed so far (keys the in-kernel Philox draw)
        self.ig_acc = None           # Integrated Gradients: fp32 [B, S, S, Ci] sum of the path's input gradients (lazy)
        # weight gradients run on a side stream, concurrently with the dgrad / un-pool chain
        self.side = torch.cuda.Stream(device)
        self.after_restore()

    @property
    def compact0(self) -> bool:
        """Layer-1 input as [P, 4] = R, G, B, 0 (8 bytes per pixel instead of 32) — the one place that picks it.
        Only the RGB defaults read it: the s-packed layer 1 on the pair-row forward and the masked-GEMM weight gradient
        (both have compact variants, conv_tcgen05.cu kPairC and wgrad0_mma.cu). Any switch that selects a layer-1
        kernel needing 16 channels (HEFL_SPACK0=0, HEFL_FWD_PAIR=0, HEFL_GATHER_WGRAD0=0, HEFL_WGRAD0_MMA=0, odd
        image sizes), or the same attributes changed after construction, gives the 16-channel layout back."""
        h = self.H[0]
        return (self.spack0 and self.Ci[0] == 3 and self.fwd_pair >= 1 and self.gather_wgrad0 and self._wgrad0_mma
                and h % 2 == 0 and h <= 256)

    def x0(self, slot: int) -> torch.Tensor:
        """Layer-1 input buffer of ``slot`` in the current layout."""
        return self._x0c[slot] if self.compact0 else self._x0_bufs[slot]

    # ------------------------------------------------------------------ weights
    def after_update(self) -> None:
        """Called after Adam wrote the bf16 shadow: rebuild the tensor-core weight layouts."""
        self.ops.conv_weight_relayout(self.shadow, self.table, self.Wf, self.Wd, 0, -1, self.spack0, self.compact0)

    def after_restore(self) -> None:
        self.shadow.copy_(self.pack.trainable())
        self.after_update()

    def _wf(self, l):
        return self.Wf[self.wf_off[l]: self.wf_off[l + 1]]

    def _wf0c(self):
        """Layer-1 weights of the compact input: [3 r][2 dx][Co][16], after the s-packed [3][Co][16] (conv_weight_relayout)."""
        return self.Wf[self.wf_off[0] + 3 * self.Co[0] * 16: self.wf_off[1]]

    def _wd(self, l):
        return self.Wd[self.wd_off[l]: self.wd_off[l + 1]]

    def _dw(self, l):
        return self.dW32[self.dw_off[l]: self.dw_off[l + 1]]

    # ------------------------------------------------------------------ forward
    def _make_theta(self, shear=0.2, zoom=0.2) -> torch.Tensor:
        B, dev = self.B, self.device
        r = torch.rand(B, 4, device=dev)
        sh = (r[:, 0] * 2 - 1) * shear * (math.pi / 180.0)
        zx = 1.0 + (r[:, 1] * 2 - 1) * zoom
        zy = 1.0 + (r[:, 2] * 2 - 1) * zoom
        flip = torch.where(r[:, 3] < 0.5, -1.0, 1.0)
        th = self.theta
        th.zero_()
        th[:, 0, 0] = zx * flip
        th[:, 0, 1] = -torch.sin(sh) * zx
        th[:, 1, 1] = torch.cos(sh) * zy
        return th

    def preprocess(self, x_u8: torch.Tensor, slot: int, train: bool, augment: bool) -> None:
        """uint8 NHWC batch -> bf16 [P,16] layer-1 input of ``slot`` (1/255 rescale + Keras-style random
        affine, FLPyfhelin.py:80-86). Augmentation parameters are drawn inside the kernel from Philox
        keyed by (seed, number of augmented batches so far, sample): reproducible and independent of
        which stream or slot the batch is staged on."""
        seed = 0
        if train and augment:
            seed = (self.aug_seed + 0x9E3779B97F4A7C15 * (self.prep_count + 1)) & 0x7FFFFFFFFFFFFFFF or 1
            self.prep_count += 1
        compact = self.compact0
        self.ops.preprocess_u8(x_u8, None, self._x0c[slot] if compact else self.X0[slot], seed, None, self.spack0,
                               compact)     # channels from x_u8

    def forward_convs(self, slot: int, train: bool, codes_from: int = 0) -> torch.Tensor:
        """The conv stack on the input of ``slot``; with ``train``, layers ``codes_from`` .. n-1 store arg-max codes."""
        x = self.X0[slot]
        for l in range(self.n):
            h = self.H[l]
            codes = self.amax[l] if train and l >= codes_from else None
            if l < self.fwd_pair and h % 2 == 0 and (h - 2) // 2 <= 128 and self.CK[l] <= 32 and self.Co[l] <= 64:
                compact = l == 0 and self.compact0
                self.ops.conv_fwd_pool_pair(x if l else self.x0(slot), self._wf0c() if compact else self._wf(l),
                                            self.bias[l], self.X[l + 1], codes, self.B, h, h,
                                            self.CK[l], self.Co[l], self.spack0 and l == 0, self.Ci[0], compact)
                x = self.X[l + 1]
                continue
            self.ops.conv_fwd_pool(x, self._wf(l), self.bias[l], self.X[l + 1], codes, self.B, h, h, self.CK[l], self.Co[l],
                                   self.spack0 and l == 0, self.Ci[0])
            x = self.X[l + 1]
        return self.X[self.n]

    def features(self, x_u8: torch.Tensor, train: bool, augment: bool, slot: int = 0) -> torch.Tensor:
        self.preprocess(x_u8, slot, train, augment)
        return self.forward_convs(slot, train)

    def _head(self, feat: torch.Tensor) -> torch.Tensor:
        x = feat
        fcs = self.model.fcs
        for fc in fcs[:-1]:
            x = F.relu(fc(x))
        return fcs[-1](x)

    # ------------------------------------------------------------------ steps
    def train_step(self, x_u8: torch.Tensor, y: torch.Tensor, out: torch.Tensor, augment: bool = True, opt=None) -> None:
        self.preprocess(x_u8, 0, True, augment)
        self.train_step_staged(0, y, out, opt)

    def train_step_staged(self, slot: int, y: torch.Tensor, out: torch.Tensor, opt=None) -> None:
        """Forward + backward on the already pre-processed batch in ``slot`` (CUDA-graph body).

        ``opt`` (optional) applies the parameter update: ``opt.bump()`` advances the step counter and
        ``opt.apply(lo, hi)`` runs Adam on flat parameters [lo, hi). Everything but layer 1 is updated on the side
        stream while layer 1's weight-gradient kernel still runs; only the layer-1 parameters (896 for RGB, 320 for
        grayscale) are left for the tail of the step."""
        feat_bf = self.forward_convs(slot, True)
        if self.fused_head:
            self.ops.head_forward_backward(feat_bf, self.pack.flat, self.pack.grad, self.head_offs, y, self.dfeat,
                                           self.h1_buf, self.dh1_buf, out, self.B, self.F, self.H1, self.H2, self.C, True)
            g = self.dfeat.view_as(feat_bf)
        else:
            feat = feat_bf.view(self.B, -1).float().requires_grad_(True)
            logits = self._head(feat)
            loss = F.cross_entropy(logits, y)
            loss.backward()
            out[0] = loss.detach()
            out[1] = (logits.argmax(1) == y).sum()
            g = feat.grad.to(torch.bfloat16).view_as(feat_bf).contiguous()
        main = torch.cuda.current_stream(self.device)
        split = False
        for l in range(self.n - 1, -1, -1):
            h = self.H[l]
            if l == 0 and self.gather_wgrad0:
                if opt is not None and self.n > 1 and self.p0 > 0:
                    split = True
                    ev = torch.cuda.Event()
                    ev.record(main)                     # dgrad of layer 2 (last reader of Wd) is enqueued
                    with torch.cuda.stream(self.side):
                        self.side.wait_event(ev)
                        opt.bump()
                        self.ops.conv_grad_finalize(self.dW32, self.table, self.pack.grad, 1, self.n)
                        opt.apply(self.p0, self.pack.n_trainable)
                        self.ops.conv_weight_relayout(self.shadow, self.table, self.Wf, self.Wd, 1, self.n)
                # 1- or 3-channel layer: weight gradient gathered straight from the pooled gradient
                self.ops.wgrad0_gather(self.x0(slot), g, self.amax[0], self._dw(0), self.B, h, h, self.spack0,
                                       self.Ci[0], self.compact0)
                break
            xin = self.X0[slot] if l == 0 else self.X[l]
            if self.dY[l] is None:
                self.dY[l] = torch.zeros(self.P[l], self.Co[l], dtype=torch.bfloat16, device=self.device)
            self.ops.unpool_relu(g, self.amax[l], self.X[l + 1], self.dY[l], self.B, h, h, self.Co[l])
            if l > 0 and self.dgrad_wgrad[l]:
                # both gradients on the main stream; the side stream's finalize of this layer waits on an event
                # recorded after it (layer 1's split below, or main.wait_stream(side) at the end)
                self.ops.conv_dgrad_wgrad(xin, self.dY[l], self._wd(l), self.gX[l], self._dw(l), self.B, h, h,
                                          self.CK[l], self.Co[l])
                g = self.gX[l]
            elif l > 0:
                # wgrad(l) only needs X[l] and dY[l]; dgrad(l) -> unpool(l-1) -> ... proceeds meanwhile
                self.side.wait_stream(main)
                with torch.cuda.stream(self.side):
                    self.ops.conv_wgrad(xin, self.dY[l], self._dw(l), self.B, h, h, self.CK[l], self.Co[l])
                self.ops.conv_dgrad(self.dY[l], self._wd(l), self.gX[l], self.B, h, h, self.Co[l], self.Ci[l])
                g = self.gX[l]
            else:
                self.ops.conv_wgrad(xin, self.dY[l], self._dw(l), self.B, h, h, self.CK[l], self.Co[l])
        main.wait_stream(self.side)
        if opt is None:
            self.ops.conv_grad_finalize(self.dW32, self.table, self.pack.grad)
        elif split:
            self.ops.conv_grad_finalize(self.dW32, self.table, self.pack.grad, 0, 1)
            opt.apply(0, self.p0)
            self.ops.conv_weight_relayout(self.shadow, self.table, self.Wf, self.Wd, 0, 1, self.spack0, self.compact0)
        else:
            opt.bump()
            self.ops.conv_grad_finalize(self.dW32, self.table, self.pack.grad)
            opt.apply(0, self.pack.n_trainable)
            self.after_update()

    def head_step_staged(self, slot: int, y: torch.Tensor, out: torch.Tensor, opt) -> None:
        """Head-only step on the pre-processed batch in ``slot`` (CUDA-graph body): the conv base is frozen, so its
        backward (un-pool, dgrad, wgrad, finalize, relayout) is dead work. Forward convs without arg-max codes, the
        head forward and backward down to the first personal layer (no ``dfeat``), then ``opt.bump()`` and Adam on
        the personal layers [head_lo, n_trainable)."""
        if not self.personal:
            raise RuntimeError("head_step_staged needs personal_layers > 0")
        feat_bf = self.forward_convs(slot, False)
        if self.fused_head:
            self.ops.head_forward_backward(feat_bf, self.pack.flat, self.pack.grad, self.head_offs, y, self.dfeat,
                                           self.h1_buf, self.dh1_buf, out, self.B, self.F, self.H1, self.H2, self.C,
                                           self.head_depth)
        else:
            fcs = self.model.fcs
            shared = len(fcs) - self.personal
            with torch.no_grad():
                x = feat_bf.view(self.B, -1).float()
                for fc in fcs[:shared]:
                    x = F.relu(fc(x))
            for j in range(shared, len(fcs)):
                x = fcs[j](x)
                if j + 1 < len(fcs):
                    x = F.relu(x)
            loss = F.cross_entropy(x, y)
            loss.backward()
            out[0] = loss.detach()
            out[1] = (x.argmax(1) == y).sum()
        opt.bump()
        opt.apply(self.head_lo, self.pack.n_trainable)

    def _saliency(self, slot: int, stage: int, codes_from: int, target: torch.Tensor,
                  logits_out: torch.Tensor) -> torch.Tensor:
        """Forward convs on the input of ``slot`` (arg-max codes of layers ``codes_from`` .. n-1), the head seeded with
        the class score of ``target`` (head_saliency; -1: the arg-max), ``logits_out`` [B, C] fp32, and the un-pool /
        dgrad chain down to stage ``stage`` (1..n). Returns d logits[b, t_b] / d X[stage] (bf16, X[stage]'s shape)."""
        feat_bf = self.forward_convs(slot, True, codes_from=codes_from)
        if self.fused_head:
            self.ops.head_saliency(feat_bf, self.pack.flat, self.head_offs, target, self.dfeat, self.h1_buf,
                                   self.dh1_buf, logits_out, self.B, self.F, self.H1, self.H2, self.C)
            g = self.dfeat.view_as(feat_bf)
        else:
            with torch.enable_grad():
                feat = feat_bf.view(self.B, -1).float().requires_grad_(True)
                logits = self._head(feat)
                t = torch.where(target < 0, logits.argmax(1), target)
                gf, = torch.autograd.grad(logits.gather(1, t[:, None]).sum(), feat)
            logits_out.copy_(logits.detach())
            g = gf.to(torch.bfloat16).view_as(feat_bf).contiguous()
        for l in range(self.n - 1, stage - 1, -1):
            h = self.H[l]
            self.ops.unpool_relu(g, self.amax[l], self.X[l + 1], self.dY[l], self.B, h, h, self.Co[l])
            self.ops.conv_dgrad(self.dY[l], self._wd(l), self.gX[l], self.B, h, h, self.Co[l], self.Ci[l])
            g = self.gX[l]
        return g

    def gradcam_staged(self, slot: int, stage: int, target: torch.Tensor, logits_out: torch.Tensor,
                       cam_out: torch.Tensor, nvalid: int) -> None:
        """Grad-CAM (DESIGN.md §11) of the batch pre-processed into ``slot`` (``preprocess(.., train=False,
        augment=False)``): ``logits_out`` [B, C] fp32 and ``cam_out`` [>= nvalid, S, S] fp32, the first ``nvalid`` maps.
        ``target`` int64 [B] on the device: the class whose score is explained per scan, -1 for the predicted one.
        ``stage`` 1..n is the pooled output X[stage] the map is taken at. Runs no weight gradient, finalize, Adam or
        relayout: only X, amax, dY, gX, dfeat and the head scratch change."""
        if not 1 <= stage <= self.n:
            raise ValueError(f"stage must be in 1..{self.n}, got {stage}")
        g = self._saliency(slot, stage, stage, target, logits_out)
        self.ops.gradcam(self.X[stage], g, cam_out, self.B, self.H[stage], self.Co[stage - 1], self.H[0], nvalid)

    def ig_staged(self, steps: int, target: torch.Tensor, logits_out: torch.Tensor, base_out: torch.Tensor,
                  attr_out: torch.Tensor, nvalid: int) -> torch.Tensor:
        """Integrated Gradients (DESIGN.md §12) of the batch pre-processed into slot 1 (``preprocess(.., 1,
        train=False, augment=False)``), black baseline, midpoint rule with ``steps`` points. ``target`` int64 [B] on
        the device (-1: the class predicted at the scan); returns it resolved. ``logits_out`` / ``base_out`` [B, C]
        fp32: the logits at the scan and at the black image. ``attr_out`` [>= nvalid, S, S] fp32, the first ``nvalid``
        maps: sum over channels of x * (1/steps) sum_k d logit_t / d x at x_k = bf16(alpha_k x), alpha_k =
        (k - 1/2) / steps; ``ig_acc`` keeps the sum over k. Path points are scaled into slot 0. Runs no weight
        gradient, finalize, Adam or relayout: only slot 0, X, amax, dY, gX, dfeat, the head scratch and ig_acc change."""
        if self.Co[0] != 32:
            raise ValueError(f"input_grad0 handles a first conv of 32 filters, this model has {self.Co[0]}")
        if not 1 <= steps <= 1024:
            raise ValueError(f"steps must be in 1..1024, got {steps}")
        B, S, ci, n = self.B, self.H[0], self.Ci[0], self.n
        if self.ig_acc is None:
            self.ig_acc = torch.zeros(B, S, S, ci, dtype=torch.float32, device=self.device)
        x1, x0 = self.x0(1), self.x0(0)
        self._saliency(1, n, n, target, logits_out)
        t = torch.where(target < 0, logits_out.argmax(1), target)
        torch.mul(x1, 0.0, out=x0)
        self._saliency(0, n, n, t, base_out)
        w_off = int(self.table[0, 3])
        w0 = self.shadow[w_off: w_off + self.Co[0] * ci * 9]           # layer 1's [Co][Ci][3][3], as the forward used
        acc = self.ig_acc
        acc[:nvalid].zero_()
        scratch = torch.empty_like(logits_out)
        for k in range(1, steps + 1):
            torch.mul(x1, (k - 0.5) / steps, out=x0)          # fp32 opmath, rounded to bf16 in every layer-1 layout
            g = self._saliency(0, 1, 0, t, scratch)
            self.ops.input_grad0(g, self.amax[0], w0, acc, B, S, ci, nvalid)
        xh = x1[: self.P[0], :ci].view(B, S, S, ci)
        attr_out[:nvalid] = (xh[:nvalid].float() * acc[:nvalid]).sum(-1) / steps
        return t

    def score_staged(self, slot: int, y: torch.Tensor, nvalid_dev: torch.Tensor, counts_row, probs_out: torch.Tensor) -> None:
        """Federated-evaluation scoring (DESIGN.md §13) of the batch pre-processed into ``slot`` (``preprocess(..,
        train=False, augment=False)``; CUDA-graph body): forward convs without arg-max codes, the head's logits
        (head_logits; autograd-free PyTorch for heads the fused kernels do not cover) into ``score_logits``, then
        score_stats. ``counts_row`` = (int32 counts [C*C*(nbins+1)], float64 loss sum [1], int32 error flag [1]) is
        added into; ``probs_out`` [B, C] fp32; ``nvalid_dev`` int32 [1] on the device: rows >= it are not counted.
        Only X, the head scratch, ``score_logits`` and the outputs change."""
        counts, loss, err = counts_row
        C = self.model.fcs[-1].out_features
        nbins = counts.numel() // (C * C) - 1
        if getattr(self, "score_logits", None) is None:
            self.score_logits = torch.zeros(self.B, C, dtype=torch.float32, device=self.device)
        feat_bf = self.forward_convs(slot, False)
        if self.fused_head:
            self.ops.head_logits(feat_bf, self.pack.flat, self.head_offs, self.h1_buf, self.dh1_buf, self.score_logits,
                                 self.B, self.F, self.H1, self.H2, self.C)
        else:
            with torch.no_grad():
                self.score_logits.copy_(self._head(feat_bf.view(self.B, -1).float()))
        self.ops.score_stats(self.score_logits, y, nvalid_dev, probs_out, counts, loss, err, nbins)

    def eval_step(self, x_u8: torch.Tensor, y: torch.Tensor, out: torch.Tensor) -> None:
        self.preprocess(x_u8, 0, False, False)
        self.eval_step_staged(0, y, out)

    def eval_step_staged(self, slot: int, y: torch.Tensor, out: torch.Tensor) -> None:
        feat_bf = self.forward_convs(slot, False)
        if self.fused_head:
            self.ops.head_forward_backward(feat_bf, self.pack.flat, self.pack.grad, self.head_offs, y, self.dfeat,
                                           self.h1_buf, self.dh1_buf, out, self.B, self.F, self.H1, self.H2, self.C, False)
            return
        feat = feat_bf.view(self.B, -1).float()
        logits = self._head(feat)
        out[0] = F.cross_entropy(logits, y)
        out[1] = (logits.argmax(1) == y).sum()

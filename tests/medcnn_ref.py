"""Plain float64 references for the medical CNN's kernels, the layer-1 input layouts they read, and the error bounds
the GPU tests hold them to.

Tensors here are NCHW and float64 unless a name says otherwise; the kernels' buffers are NHWC viewed as
[pixels, channels] (`nchw` / `nhwc` convert). Everything is plain PyTorch and runs on any device."""
import math
from typing import NamedTuple

import torch
import torch.nn.functional as F

# per-addition error allowed for the tensor-core fp32 accumulation (truncating adds: 2^-23 per add, doubled)
ACC_EPS = 2.0 ** -22
BF16_EPS = 2.0 ** -8          # bf16 unit round-off (8 significant bits)


def nchw(t, B, H, W):
    """[B*H*W(, ...), C] NHWC buffer -> [B, C, H, W] float64 (rows past B*H*W, e.g. TMA slack, are ignored)."""
    return t[: B * H * W].reshape(B, H, W, -1).permute(0, 3, 1, 2).double()


def nhwc(t):
    """[B, C, H, W] -> [B*H*W, C] (contiguous, same dtype)."""
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1]).contiguous()


def bf16_rn(t):
    """Round to bf16 (nearest even); the GPU epilogues' cvt.rn.bf16x2.f32 does the same to an exact fp32 value."""
    return t.to(torch.bfloat16)


# ---------------------------------------------------------------------------------------------- forward
class Pool(NamedTuple):
    out: torch.Tensor     # relu(max + bias), [B, Co, Hp, Wp]
    code: torch.Tensor    # uint8: bit 1 = lower row, bit 0 = right column of the arg-max, bit 2 = max + bias > 0
    S: torch.Tensor       # largest sum of |x w| (+ |bias|) over the window's four conv outputs
    gap: torch.Tensor     # largest minus second-largest conv output of the window (0 on a tie)
    act: torch.Tensor     # max + bias (before ReLU)


def fwd_pool(x, w, b, drop_last_col=False):
    """conv 3x3 (valid) -> + bias -> ReLU -> 2x2 floor max-pool, in float64, with the kernels' arg-max codes.

    Tie rule of tap_gemm_kernel and the pair kernels: within a column the lower row wins only if it is strictly
    greater; then the right column wins only if its maximum is strictly greater than the left column's. Bias and
    ReLU commute with the max, so the comparisons are on the raw conv sums. `drop_last_col` is a defect variant: the
    last conv column each pooled row reads is ignored."""
    x, w, b = x.double(), w.double(), b.double()
    conv = F.conv2d(x, w)
    S = F.conv2d(x.abs(), w.abs()) + b.abs().view(1, -1, 1, 1)
    Hp, Wp = (x.shape[2] - 2) // 2, (x.shape[3] - 2) // 2
    conv, S = conv[..., : 2 * Hp, : 2 * Wp], S[..., : 2 * Hp, : 2 * Wp]
    if drop_last_col:
        conv = conv.clone()
        conv[..., 2 * Wp - 1] = -math.inf
    v00, v01, v10, v11 = conv[..., 0::2, 0::2], conv[..., 0::2, 1::2], conv[..., 1::2, 0::2], conv[..., 1::2, 1::2]
    l0, l1 = v10 > v00, v11 > v01
    m0, m1 = torch.where(l0, v10, v00), torch.where(l1, v11, v01)
    rw = m1 > m0
    y = torch.where(rw, m1, m0) + b.view(1, -1, 1, 1)
    row = torch.where(rw, l1, l0)
    code = (row.to(torch.uint8) << 1) | rw.to(torch.uint8) | ((y > 0).to(torch.uint8) << 2)
    win = torch.stack([v00, v01, v10, v11], -1)
    top2 = win.topk(2, -1).values
    gap = top2[..., 0] - top2[..., 1]
    Swin = torch.stack([S[..., 0::2, 0::2], S[..., 0::2, 1::2], S[..., 1::2, 0::2], S[..., 1::2, 1::2]], -1).amax(-1)
    return Pool(y.clamp_min(0), code, Swin, gap, y)


# ---------------------------------------------------------------------------------------------- backward
def unpool(g, pooled, code, H, W):
    """unpool_relu_kernel: the pooled gradient g goes to the arg-max position (code bits 0-1) of windows whose pooled
    (bf16) value is > 0; every other position of the H x W grid, the dropped floor-pool edge and the two-pixel
    border of the conv grid included, is zero."""
    B, C, Hp, Wp = g.shape
    out = torch.zeros(B, C, H, W, dtype=torch.float64, device=g.device)
    on = pooled.double() > 0
    gv = torch.where(on, g.double(), torch.zeros((), dtype=torch.float64, device=g.device))
    c = code.long()
    for dy in range(2):
        for dx in range(2):
            sel = ((c >> 1) & 1 == dy) & (c & 1 == dx)
            out[:, :, dy: 2 * Hp: 2, dx: 2 * Wp: 2] = torch.where(sel, gv, torch.zeros_like(gv))
    return out


def dgrad(dy, w):
    """Full correlation: dX [B, Ci, H, W] from the conv-grid gradient dy [B, Co, H, W] (its valid part is the top-left
    (H-2) x (W-2); the rest must be zero, as unpool leaves it)."""
    H, W = dy.shape[2], dy.shape[3]
    return F.conv_transpose2d(dy[..., : H - 2, : W - 2].double(), w.double())


def dgrad_abs(dy, w):
    """Sum of |terms| of every dgrad output."""
    return dgrad(dy.abs(), w.abs())


def wgrad(x, dy, CK):
    """Weight + bias gradient of a 3x3 valid conv in the engine's dW32 layout: [(r*3 + s)*CK + ci][co] for ci < Ci
    (padded channels zero), then the bias row. x [B, Ci, H, W], dy [B, Co, H, W] (valid part top-left)."""
    x, dy = x.double(), dy.double()
    B, Ci, H, W = x.shape
    Co = dy.shape[1]
    d = dy[..., : H - 2, : W - 2]
    gw = torch.nn.grad.conv2d_weight(x, (Co, Ci, 3, 3), d)
    out = torch.zeros(9 * CK + 1, Co, dtype=torch.float64, device=x.device)
    out[: 9 * CK].view(9, CK, Co)[:, :Ci] = gw.permute(2, 3, 1, 0).reshape(9, Ci, Co)
    out[9 * CK] = d.sum((0, 2, 3))
    return out


def wgrad_abs(x, dy, CK):
    return wgrad(x.abs(), dy.abs(), CK)


def conv_grid_grad(g, code, H, W):
    """Layer-1 conv-grid gradient implied by the pooled gradient and the codes: g at the arg-max of every active
    window (code bit 2), zero elsewhere."""
    B, C, Hp, Wp = g.shape
    act = (code.long() & 4) != 0
    return unpool(torch.where(act, g.double(), torch.zeros((), dtype=torch.float64, device=g.device)),
                  act.double(), code, H, W)


def wgrad0(x, g, code, CK=16):
    """Layer-1 weight gradient straight from the pooled gradient and the codes (wgrad0_gather / wgrad0_mma*)."""
    return wgrad(x, conv_grid_grad(g, code, x.shape[2], x.shape[3]), CK)


def wgrad0_abs(x, g, code, CK=16):
    return wgrad0(x.abs(), g.abs(), code, CK)


def wgrad_to_oihw(dW, Ci, CK, Co):
    """dW32 layout -> ([Co, Ci, 3, 3] weight gradient, [Co] bias gradient)."""
    dW = dW.reshape(-1)
    w = dW[: 9 * CK * Co].reshape(9, CK, Co)[:, :Ci].permute(2, 1, 0).reshape(Co, Ci, 3, 3)
    return w, dW[9 * CK * Co: (9 * CK + 1) * Co]


# ---------------------------------------------------------------------------------------------- defect variants
def drop_tap(w, ci, r, s):
    """w with input channel ci's tap (r, s) zeroed (ci = None: the tap of every input channel)."""
    w = w.clone()
    if ci is None:
        w[:, :, r, s] = 0
    else:
        w[:, ci, r, s] = 0
    return w


def wgrad_last_unit(B, H, W):
    """(image, conv rows, conv columns) of the last work unit of wgrad_kernel's plan: units of <= 16 conv rows per
    64-column strip and image. At H = W = 127 that is the 13-row unit (rows 112-124) of the second strip (columns
    64-124, 61 of them) of the last image."""
    Ho, Wo = H - 2, W - 2
    rows_per = min(Ho, 16)
    r0 = (Ho + rows_per - 1) // rows_per * rows_per - rows_per
    c0 = (Wo + 63) // 64 * 64 - 64
    return B - 1, slice(r0, Ho), slice(c0, Wo)


def omit_unit(dy, unit):
    """dy with the conv-grid gradient of one wgrad unit zeroed (the unit's contribution omitted)."""
    b, rows, cols = unit
    dy = dy.clone()
    dy[b, :, rows, cols] = 0
    return dy


# ---------------------------------------------------------------------------------------------- bounds
def fwd_bound(ref, S, n):
    """|got - ref| allowed for a bf16 output of an n-term fp32 dot product: bf16 rounding + n accumulation errors."""
    return BF16_EPS * ref.abs() + n * ACC_EPS * S


def within(got, ref, bound):
    return bool(((got.double() - ref.double()).abs() <= bound).all())


def codes_agree(code, ref: Pool, n):
    """Kernel codes equal the reference where they are decided by a margin the accumulation error cannot cross:
    arg-max bits where the window's two largest conv outputs differ by more than twice the error, the active bit
    where |max + bias| exceeds it. Returns (agree, number of codes checked)."""
    e = n * ACC_EPS * ref.S
    c, rc = code.long(), ref.code.long()
    pos = ref.gap > 2 * e
    act = ref.act.abs() > e
    ok = bool(((c & 3) == (rc & 3))[pos].all()) and bool(((c & 4) == (rc & 4))[act].all())
    return ok, int(pos.sum())


def max_abs_sum_ok(S, limit=2 ** 24):
    """Premise of the integer tests: every output's sum of |terms| is below 2^24, so fp32 accumulation of the
    (integer) terms is exact in any order."""
    return float(S.max()) < limit


# ---------------------------------------------------------------------------------------------- layer-1 layouts
def pack_compact(img):
    """[B, H, W, 3] -> [B*H*W, 4] = R, G, B, 0 (preprocess_u8 compact)."""
    B, H, W, _ = img.shape
    out = torch.zeros(B, H, W, 4, dtype=img.dtype, device=img.device)
    out[..., :3] = img
    return out.view(-1, 4)


def pack_s(img):
    """[B, H, W, 3] -> s-packed [B*H*W, 16]: channel 3s + ci = pixel (h, w + s), 0 past the right edge."""
    B, H, W, C = img.shape
    out = torch.zeros(B, H, W, 16, dtype=img.dtype, device=img.device)
    for s in range(3):
        out[:, :, : W - s, 3 * s: 3 * s + C] = img[:, :, s:]
    return out.view(-1, 16)


def pack_rs(img):
    """[B, H, W, 1] -> rs-packed [B*H*W, 16]: channel 3r + s = pixel (h + r, w + s), 0 past the bottom or right."""
    B, H, W, _ = img.shape
    out = torch.zeros(B, H, W, 16, dtype=img.dtype, device=img.device)
    for r in range(3):
        for s in range(3):
            out[:, : H - r, : W - s, 3 * r + s] = img[:, r:, s:, 0]
    return out.view(-1, 16)


def with_slack(t, rows=8):
    """t followed by `rows` zero rows (the engine's layer-1 buffers carry this slack: layer-1 kernels read 4-pixel
    windows past the last pixel), as a view of the first t.shape[0] rows."""
    buf = torch.zeros(t.shape[0] + rows, t.shape[1], dtype=t.dtype, device=t.device)
    buf[: t.shape[0]] = t
    return buf


# ---------------------------------------------------------------------------------------------- weight layouts
MEDCNN_CI = [3, 32, 32, 32, 64, 64]
MEDCNN_CO = [32, 32, 32, 64, 64, 128]


class Layouts(NamedTuple):
    Wf: list          # per layer: forward B operand (layer 1: s-packed / rs-packed [taps][Co][16])
    Wd: list          # per layer: dgrad B operand [tap][Ci][Co] (None for layer 1)
    Wf0c: torch.Tensor   # layer 1 on the compact input, [3 r][2 dx][Co][16] (None unless compact0)
    table: torch.Tensor


def weight_layouts(ops, ws, spack0=True, compact0=False):
    """Tensor-core weight layouts of the medical CNN's six convs, built by conv_weight_relayout from a bf16 shadow
    holding ws (list of [Co, Ci, 3, 3]) the way ParamPack stores them (weights then bias per layer; biases unused)."""
    dev = ws[0].device
    rows, shadow = [], []
    off = wf = wd = dw = 0
    for w in ws:
        Co, Ci = w.shape[:2]
        CK = 16 if not rows else Ci
        rows.append([Ci, CK, Co, off, off + w.numel(), wf, wd, dw])
        shadow += [w.reshape(-1), torch.zeros(Co, device=dev)]
        off += w.numel() + Co
        wf += 9 * Co * CK
        wd += 9 * Ci * Co
        dw += (9 * CK + 1) * Co
    table = torch.tensor(rows, dtype=torch.int64)
    shadow = torch.cat(shadow).to(torch.bfloat16)
    Wf = torch.full((wf,), float("nan"), dtype=torch.bfloat16, device=dev)
    Wd = torch.full((wd,), float("nan"), dtype=torch.bfloat16, device=dev)
    ops.conv_weight_relayout(shadow, table, Wf, Wd, 0, -1, spack0, compact0)
    wf_ = [r[5] for r in rows] + [wf]
    wd_ = [r[6] for r in rows] + [wd]
    Co0, Ci0 = ws[0].shape[:2]
    taps0 = (1 if Ci0 == 1 else 3) if spack0 else 9
    f = [Wf[wf_[0]: wf_[0] + taps0 * Co0 * 16]] + [Wf[wf_[l]: wf_[l + 1]] for l in range(1, len(ws))]
    d = [None] + [Wd[wd_[l]: wd_[l + 1]] for l in range(1, len(ws))]
    f0c = Wf[wf_[0] + 3 * Co0 * 16: wf_[1]] if compact0 else None
    return Layouts(f, d, f0c, table)

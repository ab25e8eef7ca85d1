"""Plain float64 references for the ResNet kernels (csrc/nn/gemm_tcgen05.cu, csrc/nn/resnet_kernels.cu), bit-level
references of the e4m3 quantisers, and the error bounds the GPU tests hold the kernels to.

Activations are NHWC matrices `[pixels, C]` as the kernels see them; `nhwc` converts a channels_last [B, C, H, W]
tensor. Convolutions are tap GEMMs in float64 (torch.matmul: exact for integer data below 2^53), never cuDNN, so no
TF32, Winograd or FFT can hide a wrong tap. Everything is plain PyTorch and runs on any device."""
import math

import torch

U32 = 2.0 ** -24            # fp32 unit round-off
E4M3_MAX = 448.0
# Per-addition error allowed for fp32 accumulation, in units of U32: a truncating add can lose 2 U32 of the partial
# sum, doubled for margin. A K-term dot product is then off by at most C_ACC * K * U32 * sum|terms|.
C_ACC = 4
# e4m3 tensor-core MMAs (wgmma ...e4m3, mma.sync ...e4m3) are reported to add their products with fewer than fp32's
# 24 bits. Integer tests keep sum|terms| <= 2^12 so that 13 bits suffice; real-data bounds allow 2^-12 of sum|terms|
# per 32-element MMA step instead of C_ACC * U32 per addition.
FP8_INT_LIMIT = 2 ** 12
FP8_STEP_EPS = 2.0 ** -12


def nhwc(t):
    """[B, C, H, W] -> [B*H*W, C] (contiguous, same dtype)."""
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1]).contiguous()


def bf16_rn(t):
    """Round to bf16, nearest even (what cvt.rn.bf16x2.f32 does to an exact fp32 value)."""
    return t.to(torch.bfloat16)


def half_ulp_bf16(a):
    """Half a bf16 ulp at |a| (8 significant bits; subnormal spacing 2^-133 below 2^-126)."""
    a = a.double().abs()
    e = torch.floor(torch.log2(a.clamp_min(2.0 ** -126)))
    return torch.exp2(e - 8)


# ---------------------------------------------------------------------------------------------- convolutions
def shifts(Wp):
    """Row shift of tap (r, s) on a zero-padded grid of row length Wp (tc_conv._shifts)."""
    return [(r - 1) * Wp + (s - 1) for r in range(3) for s in range(3)]


def pad_grid(x2, B, H, W):
    """[B*H*W, C] -> [B*(H+2)*(W+2), C] with a zero border (pad_nhwc_kernel)."""
    C = x2.shape[1]
    xp = torch.zeros(B, H + 2, W + 2, C, dtype=x2.dtype, device=x2.device)
    xp[:, 1:H + 1, 1:W + 1] = x2.view(B, H, W, C)
    return xp.view(-1, C)


def _shifted(xp, s):
    """Rows p + s of xp, zero where p + s falls outside."""
    out = torch.zeros_like(xp)
    n = xp.shape[0]
    if s >= 0:
        out[: n - s] = xp[s:]
    else:
        out[-s:] = xp[: n + s]
    return out


def _interior(yp, B, H, W):
    return yp.view(B, H + 2, W + 2, -1)[:, 1:H + 1, 1:W + 1].reshape(B * H * W, -1)


def conv1x1_fwd(x2, w):
    """Y = X W^T; x2 [P, Cin], w [Cout, Cin] (stride 2: sub-sample x first, `subsample`)."""
    return x2.double() @ w.double().t()


def conv1x1_dgrad(dy2, w):
    """dX = dY W."""
    return dy2.double() @ w.double()


def conv1x1_wgrad(dy2, x2):
    """dW = dY^T X, [Cout, Cin]."""
    return dy2.double().t() @ x2.double()


def subsample(x2, B, H, W, stride):
    """Pixels (stride*i, stride*j) of a [B*H*W, C] map (what conv1x1 does before the GEMM)."""
    return x2.view(B, H, W, -1)[:, ::stride, ::stride].reshape(-1, x2.shape[1])


def scatter_even(dx2, B, H, W, stride):
    """Input gradient of a strided 1x1 conv: dx2 at the sampled pixels, zero elsewhere."""
    out = torch.zeros(B, H, W, dx2.shape[1], dtype=dx2.dtype, device=dx2.device)
    out[:, ::stride, ::stride] = dx2.view(B, (H + stride - 1) // stride, (W + stride - 1) // stride, -1)
    return out.view(-1, dx2.shape[1])


def conv3x3_fwd(x2, w, B, H, W, drop_tap=None):
    """3x3 / pad 1 / stride 1: Y[p] = sum_tap X_pad[p + shift(tap)] W[:, :, r, s]^T on the padded grid, interior rows
    kept. w [Cout, Cin, 3, 3]. `drop_tap` (defect variant) leaves that tap out."""
    xp = pad_grid(x2.double(), B, H, W)
    w = w.double()
    y = None
    for t, s in enumerate(shifts(W + 2)):
        if t == drop_tap:
            continue
        term = _shifted(xp, s) @ w[:, :, t // 3, t % 3].t()
        y = term if y is None else y + term
    return _interior(y, B, H, W)


def conv3x3_dgrad(dy2, w, B, H, W, rotate=True):
    """dX = 3x3 conv of dY with the filter rotated by 180 degrees and its channels swapped. `rotate=False` is the
    defect variant that forgets the rotation."""
    w = w.double()
    wr = w.flip(2, 3) if rotate else w
    return conv3x3_fwd(dy2, wr.transpose(0, 1), B, H, W)


def conv3x3_wgrad(dy2, x2, B, H, W):
    """dW[co, ci, r, s] = sum_p dY[p, co] X_pad[p + shift(r, s), ci] over the padded grid."""
    dyp = pad_grid(dy2.double(), B, H, W)
    xp = pad_grid(x2.double(), B, H, W)
    Co, Ci = dy2.shape[1], x2.shape[1]
    dw = torch.empty(Co, Ci, 3, 3, dtype=torch.float64, device=x2.device)
    for t, s in enumerate(shifts(W + 2)):
        dw[:, :, t // 3, t % 3] = dyp.t() @ _shifted(xp, s)
    return dw


def conv3x3_fwd_abs(x2, w, B, H, W):
    return conv3x3_fwd(x2.double().abs(), w.double().abs(), B, H, W)


def conv3x3_dgrad_abs(dy2, w, B, H, W):
    return conv3x3_dgrad(dy2.double().abs(), w.double().abs(), B, H, W)


def conv3x3_wgrad_abs(dy2, x2, B, H, W):
    return conv3x3_wgrad(dy2.double().abs(), x2.double().abs(), B, H, W)


def conv1x1_fwd_abs(x2, w):
    return conv1x1_fwd(x2.double().abs(), w.double().abs())


def conv1x1_dgrad_abs(dy2, w):
    return conv1x1_dgrad(dy2.double().abs(), w.double().abs())


def conv1x1_wgrad_abs(dy2, x2):
    return conv1x1_wgrad(dy2.double().abs(), x2.double().abs())


# ---------------------------------------------------------------------------------------------- guards and bounds
def assert_exact_premise(S, limit=2 ** 24):
    """Premise of an integer test: every output's sum of |terms| is below `limit` (2^24 for bf16 operands on fp32
    accumulation, FP8_INT_LIMIT for e4m3 operands), so accumulation in any order is exact."""
    m = float(S.max())
    assert m <= limit, f"sum of |terms| {m} exceeds {limit}: integer data too large for an exact test"


def gemm_bound(ref, S, n, step_eps=None, steps=0):
    """|got - ref| allowed for a bf16 output of an n-term fp32 dot product with sum of |terms| S: the bf16 rounding of
    the accumulated value plus C_ACC * n * U32 * S of accumulation error. For e4m3 MMAs pass step_eps / steps: each of
    the `steps` MMA steps may lose step_eps * S. Use n = K + splits for a weight gradient that is RED-added."""
    acc = C_ACC * n * U32 * S
    if step_eps is not None:
        acc = acc + steps * step_eps * S
    return half_ulp_bf16(ref.double().abs() + acc) + acc


def acc_bound(S, n):
    """|got - ref| allowed for an fp32 (unrounded) result of n accumulated terms with sum of |terms| S."""
    return C_ACC * n * U32 * S


def within(got, ref, bound):
    """(all within bound, message naming the worst element relative to its bound)."""
    err = (got.double() - ref.double()).abs()
    ratio = err / bound.double().clamp_min(1e-300)
    ratio = torch.where(torch.isnan(err), torch.full_like(ratio, math.inf), ratio)
    i = int(ratio.reshape(-1).argmax())
    g, r, b = got.reshape(-1)[i].item(), ref.reshape(-1)[i].item(), bound.reshape(-1)[i].item()
    worst = float(ratio.reshape(-1)[i])
    return worst <= 1.0, f"worst element {i}: got {g!r} ref {r!r} err {abs(g - r):.3e} bound {b:.3e} ({worst:.3f} of it)"


# ---------------------------------------------------------------------------------------------- BatchNorm
def bn_launch(P, C, sms):
    """(threads, rows per iteration, stats grid) of bn_forward / bn_backward's reduction kernels."""
    groups = C // 8
    threads = 256 - 256 % min(groups, 256)
    rows = threads // groups
    grid = max(1, min((P + rows * 8 - 1) // (rows * 8), sms * 4))
    return threads, rows, grid


def bn_chain(P, C, sms):
    """Longest chain of fp32 additions a per-channel statistic goes through: a thread's rows, then the shared-memory
    atomics of the CTA's row lanes, then one global atomic per CTA."""
    _, rows, grid = bn_launch(P, C, sms)
    return (P + grid * rows - 1) // (grid * rows) + rows + grid + 1


def bn_forward(x2, res2, gamma, beta, eps, relu, var_div=None, skip_res=False):
    """Training-mode BatchNorm in float64 on a [P, C] bf16 matrix: (y before rounding, mean, biased var, invstd).
    y = relu(gamma * xhat + beta + res). Defect variants: var_div (e.g. P - 1) and skip_res."""
    x = x2.double()
    P = x.shape[0]
    mean = x.mean(0)
    var = ((x - mean) ** 2).sum(0) / (var_div if var_div is not None else P)
    invstd = 1.0 / torch.sqrt(var + eps)
    z = (x - mean) * invstd * gamma.double() + beta.double()
    if res2 is not None and not skip_res:
        z = z + res2.double()
    return (z.clamp_min(0) if relu else z), z, mean, var, invstd


def bn_running(run_mean, run_var, mean, var, P, momentum):
    """Running statistics after one step; the running variance takes the unbiased variance."""
    return ((1 - momentum) * run_mean.double() + momentum * mean,
            (1 - momentum) * run_var.double() + momentum * var * P / max(P - 1, 1))


def relu_mask(y_bf16, relu):
    """The backward's mask: the bf16 output is > 0 (as bn_bwd_* read it: not zero, sign bit clear)."""
    if not relu:
        return torch.ones_like(y_bf16, dtype=torch.bool)
    return y_bf16.float() > 0


def bn_backward(dy2, x2, mask, gamma, mean, invstd):
    """(dx, dres, dgamma, dbeta) in float64 given the mask; mean / invstd are the float64 statistics."""
    d = torch.where(mask, dy2.double(), torch.zeros((), dtype=torch.float64, device=dy2.device))
    xhat = (x2.double() - mean) * invstd
    P = x2.shape[0]
    dbeta = d.sum(0)
    dgamma = (d * xhat).sum(0)
    dx = gamma.double() * invstd * (d - dbeta / P - xhat * dgamma / P)
    return dx, d, dgamma, dbeta


class BNBounds:
    """First-order error bounds of bn_forward / bn_backward's fp32 arithmetic against the float64 reference.

    Statistics: sum and sum of squares of bf16 values (squares exact in fp32) through a chain of L additions
    (`bn_chain`), so |dS| <= L U Sum|x|, |dQ| <= L U Sum x^2. From there mean = S/P, var = Q/P - mean^2 and
    invstd = rsqrtf(var + eps) (<= 2 ulp) carry those errors plus a few roundings each; the forward's fma(x, scale,
    shift) + res and the backward's sums and fma(a, dy, fma(b, x, c)) add theirs. Every rounding is charged one U32 of
    the magnitude it rounds, doubled."""

    def __init__(self, x2, gamma, beta, eps, sms, ref):
        y, z, mean, var, invstd = ref
        x = x2.double()
        P, C = x.shape
        L = bn_chain(P, C, sms)
        u = 2 * U32
        self.L, self.P = L, P
        S1, S2 = x.abs().sum(0), (x * x).sum(0)
        self.dmean = L * u * S1 / P + u * mean.abs()
        Q = S2 / P
        self.dvar = L * u * Q + 2 * mean.abs() * self.dmean + self.dmean ** 2 + 3 * u * (Q + mean * mean)
        self.rel_is = 0.5 * self.dvar / (var + eps) + 4 * U32 + u
        g, b = gamma.double(), beta.double()
        sc = g * invstd
        self.dsc = g.abs() * invstd * (self.rel_is + u)
        sh = b - mean * sc
        self.dsh = mean.abs() * self.dsc + sc.abs() * self.dmean + u * (b.abs() + 2 * (mean * sc).abs())
        self.sc, self.sh, self.mean, self.var, self.invstd = sc, sh, mean, var, invstd
        self.mean_abs, self.Q, self.eps = S1 / P, Q, eps

    def statistical(self, k=8):
        """(mean, var, invstd) bounds under the usual model of rounding errors as independent and zero-mean, so that
        the error of the L-addition chain grows like sqrt(L) U32 rather than L U32; k of those steps is a wide margin.
        Much tighter than the worst case where the mean is large next to the spread (mean / std = 16, where
        E[x^2] - E[x]^2 cancels): there a variance off by a fraction of a percent fails it."""
        s = k * math.sqrt(self.L) * U32
        dm = s * self.mean_abs + U32 * self.mean.abs()
        dvar = s * self.Q + 2 * self.mean.abs() * dm + dm ** 2 + 4 * U32 * (self.Q + self.mean ** 2)
        dis = (0.5 * dvar / (self.var + self.eps) + 6 * U32) * self.invstd
        return dm, dvar, dis

    def forward(self, x2, res2, z):
        """Bound of the bf16 output against the float64 y (ReLU is 1-Lipschitz)."""
        x = x2.double()
        r = res2.double().abs() if res2 is not None else 0.0
        e = x.abs() * self.dsc + self.dsh + 2 * U32 * 2 * ((x * self.sc).abs() + self.sh.abs() + r + z.abs())
        return half_ulp_bf16(z.abs() + e) + e, e

    def mean_bound(self):
        return self.dmean

    def invstd_bound(self):
        return self.rel_is * self.invstd

    def running(self, run_mean, run_var, momentum):
        P = self.P
        u = 2 * U32
        k = P / max(P - 1, 1)
        dm = momentum * self.dmean + 3 * u * ((1 - momentum) * run_mean.double().abs() + momentum * self.mean.abs())
        dv = momentum * k * self.dvar + 4 * u * ((1 - momentum) * run_var.double().abs() + momentum * k * self.var)
        return dm, dv

    def backward(self, x2, d, dgamma, dbeta, dx):
        """Bounds of (dgamma, dbeta, dx) given the masked gradient d of the reference."""
        P, L, u = self.P, self.L, 2 * U32
        x = x2.double()
        xhat = (x - self.mean) * self.invstd
        ad = d.abs()
        ddbeta = L * u * ad.sum(0)
        # the kernel's xhat = (x - mean') * invstd' carries dmean * invstd + |xhat| (rel_is + 2u) per term
        ddgamma = (ad.sum(0) * self.invstd * self.dmean + (ad * xhat.abs()).sum(0) * (self.rel_is + 3 * u + L * u))
        g = self.sc.abs() / self.invstd            # |gamma|
        a = g * self.invstd
        da = g * self.invstd * (self.rel_is + u)
        b = a * self.invstd * dgamma.abs() / P
        db = a * self.invstd / P * (ddgamma + dgamma.abs() * (2 * self.rel_is + 4 * u))
        c = a * dbeta.abs() / P + b * self.mean.abs()
        dc = (a / P * (ddbeta + dbeta.abs() * (self.rel_is + 2 * u)) + db * self.mean.abs() + b * self.dmean
              + 2 * u * c)
        e = ad * da + x.abs() * db + dc + 2 * u * (a * ad + b * x.abs() + c)
        return ddgamma, ddbeta, half_ulp_bf16(dx.abs() + e) + e


# ---------------------------------------------------------------------------------------------- average pool
def avgpool_fwd(x3):
    """[B, HW, C] -> [B, C] mean, float64."""
    return x3.double().mean(1)


def avgpool_fwd_bound(x3):
    """avgpool_fwd_kernel: HW sequential fp32 adds, then one division."""
    HW = x3.shape[1]
    return acc_bound(x3.double().abs().sum(1), HW) / HW + 2 * U32 * x3.double().mean(1).abs()


def avgpool_bwd(dout, HW):
    """[B, C] -> [B, HW, C] = dout / HW broadcast, float64."""
    return (dout.double() / HW).unsqueeze(1).expand(-1, HW, -1)


# ---------------------------------------------------------------------------------------------- quantisers
def mx_exponent(amax):
    """UE8M0 exponent of MX blocks: the smallest e with amax * 2^-e <= 448, by search over e = -127 ... 127 (e = -127
    for an all-zero block; 127 if none qualifies)."""
    a = amax.double()
    e = torch.full_like(a, 127.0)
    for k in range(126, -128, -1):
        e = torch.where(a * 2.0 ** -k <= E4M3_MAX, torch.full_like(a, float(k)), e)
    return e.long()


def mx_quantize(x2):
    """Bit-level reference of mxfp8_quantize on bf16 [R, K]: (e4m3 bytes [R, K] uint8, scale tiles uint8, e [R, K/32]).
    Elements are x * 2^-e rounded to e4m3 (exact scaling by a power of two, then round to nearest even). Scale bytes
    e + 127 go to the tile [128-row block][k-group of 128][lane l][quarter i][k-block] for row 32 i + l; padding rows
    of a partial last row block keep 127 (2^0)."""
    R, K = x2.shape
    xf = x2.float().view(R, K // 32, 32)
    e = mx_exponent(xf.abs().amax(-1))
    q = (xf.double() * torch.exp2(-e.double()).unsqueeze(-1)).float().to(torch.float8_e4m3fn)
    Rp = (R + 127) // 128 * 128
    eb = torch.full((Rp, K // 32), 127, dtype=torch.uint8, device=x2.device)
    eb[:R] = (e + 127).to(torch.uint8)
    sf = eb.view(Rp // 128, 4, 32, K // 128, 4).permute(0, 3, 2, 1, 4).reshape(-1)
    return q.view(torch.uint8).view(R, K), sf, e


def mx_dequantize(q, sf, R, K):
    """Float64 values of MX operands (e4m3 bytes [R, K], scale tiles)."""
    Rp = (R + 127) // 128 * 128
    e = sf.view(Rp // 128, K // 128, 32, 4, 4).permute(0, 3, 2, 1, 4).reshape(Rp, K // 32)[:R].double() - 127.0
    v = q.view(torch.float8_e4m3fn).double().view(R, K // 32, 32)
    return (v * torch.exp2(e).unsqueeze(-1)).view(R, K)


def fp8_quantize(x, scale, amax_prev=0.0):
    """Bit-level reference of fp8_quantize: (e4m3 bytes, new amax). q = sat_e4m3(x * s) with the product rounded in
    fp32 (as the kernel multiplies), clamped to +-448 before the round-to-nearest-even cast; amax = max(amax_prev,
    max |x|)."""
    p = x.float() * torch.tensor(float(scale), dtype=torch.float32, device=x.device)
    q = p.clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).view(torch.uint8)
    amax = max(float(amax_prev), float(x.float().abs().max()))
    return q, amax


def fp8_scale_update(amax, scale, target):
    """(scale, inv, amax) after fp8_scale_update: scale = target / amax in fp32 (amax floored at 1e-12), kept when
    amax == 0; amax reset."""
    a = torch.tensor(float(amax), dtype=torch.float32)
    s = torch.tensor(float(scale), dtype=torch.float32)
    if float(a) > 0:
        s = torch.tensor(float(target), dtype=torch.float32) / torch.clamp_min(a, 1e-12)
    return float(s), float(torch.tensor(1.0, dtype=torch.float32) / s), 0.0

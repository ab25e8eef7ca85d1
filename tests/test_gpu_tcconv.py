"""tcgen05 GEMM convolutions for the ResNets (csrc/nn/gemm_tcgen05.cu, ops/tc_conv.py) against F.conv2d in fp32 on
the same bf16-rounded operands: forward, input gradient, weight gradient; 1x1 (stride 1 / 2, bf16 and e4m3) and
3x3 / pad 1. Shapes are the ones ResNet-18 / ResNet-50 use at 224 x 224 (plus a pixel count that is not a multiple
of the 128-row tile)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-12))


def _mk(B, Cin, Cout, H, k, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, Cin, H, H, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5).to(torch.bfloat16).float()
    gy_shape = None
    return x, w, g


@pytest.mark.parametrize("B,Cin,Cout,H,stride", [(4, 64, 256, 56, 1), (4, 256, 64, 56, 1), (2, 256, 512, 28, 2),
                                                  (3, 1024, 2048, 7, 1), (4, 64, 128, 14, 2), (1, 512, 128, 28, 1),
                                                  (4, 256, 512, 4, 2), (4, 128, 256, 8, 2)])
def test_conv1x1_forward_backward_match_fp32(B, Cin, Cout, H, stride):
    from hefl_b200.ops import tc_conv

    x, w, g = _mk(B, Cin, Cout, H, 1, 1)
    xr = x.float().requires_grad_(True)
    wr = w.clone().requires_grad_(True)
    ref = F.conv2d(xr, wr, stride=stride)
    gy = torch.randn(ref.shape, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    ref.backward(gy.float())
    xt = x.clone().requires_grad_(True)
    wt = w.clone().requires_grad_(True)
    out = tc_conv.conv1x1(xt, wt, stride)
    assert out.shape == ref.shape and out.dtype == torch.bfloat16
    assert _rel(out, ref) < 1e-2
    out.backward(gy)
    assert _rel(xt.grad, xr.grad) < 1e-2
    assert _rel(wt.grad, wr.grad) < 1e-2


@pytest.mark.parametrize("B,C,Cout,H", [(2, 64, 64, 56), (2, 128, 128, 28), (3, 256, 256, 14), (4, 512, 512, 7),
                                        (2, 64, 128, 28), (4, 512, 512, 2), (4, 256, 256, 4), (4, 64, 64, 16)])
def test_conv3x3_forward_backward_match_fp32(B, C, Cout, H):
    from hefl_b200.ops import tc_conv

    x, w, g = _mk(B, C, Cout, H, 3, 2)
    xr = x.float().requires_grad_(True)
    wr = w.clone().requires_grad_(True)
    ref = F.conv2d(xr, wr, padding=1)
    gy = torch.randn(ref.shape, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    ref.backward(gy.float())
    xt = x.clone().requires_grad_(True)
    wt = w.clone().requires_grad_(True)
    out = tc_conv.conv3x3(xt, wt)
    assert _rel(out, ref) < 1e-2
    out.backward(gy)
    assert _rel(xt.grad, xr.grad) < 1e-2
    assert _rel(wt.grad, wr.grad) < 1e-2


def test_conv1x1_e4m3_forward_is_within_fp8_tolerance():
    from hefl_b200.ops import fp8, tc_conv

    x, w, _ = _mk(4, 256, 512, 28, 1, 3)
    st = (fp8.DelayedScale(x.device), fp8.DelayedScale(x.device))
    out = tc_conv.conv1x1(x, w, 1, st)                          # per-tensor delayed scaling, kind::f8f6f4
    ref = F.conv2d(x.float(), w)
    # e4m3 has 3 mantissa bits: relative error of a 256-term dot product of random operands ~ 2^-4 / sqrt(...)
    err = (out.float() - ref).abs().mean() / ref.abs().mean()
    assert float(err) < 0.06, float(err)
    cos = F.cosine_similarity(out.float().flatten(), ref.flatten(), dim=0)
    assert float(cos) > 0.998


def test_resnet18_step_on_the_tcgen05_convolutions_matches_the_library_arm():
    """One forward/backward of ResNet-18 (batch 4, 64 x 64) with every eligible convolution on the hand-written
    kernels vs the cuDNN arm: same loss, same gradients within bf16 tolerance."""
    from hefl_b200.models import create_model
    from hefl_b200.ops import tc_conv

    torch.manual_seed(0)
    m = create_model("resnet18", 3, 10, 64).cuda()
    x = torch.randn(4, 3, 64, 64, device="cuda").contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (4,), device="cuda")

    def run(on, amp=True):
        tc_conv.set_model_tc(m, on)
        m.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
            loss = F.cross_entropy(m(x).float(), y)
        loss.backward()
        return float(loss), torch.cat([p.grad.flatten() for p in m.parameters() if p.grad is not None]).clone()

    la, ga = run(True)
    lb, gb = run(False)
    lf, gf = run(False, amp=False)                      # fp32 reference calibrates the bf16 noise of this tiny batch
    ca = float(F.cosine_similarity(ga, gf, dim=0))
    cb = float(F.cosine_similarity(gb, gf, dim=0))
    print("loss tc / cudnn-bf16 / fp32:", la, lb, lf, " cos(tc, fp32)", ca, " cos(cudnn-bf16, fp32)", cb,
          " cos(tc, cudnn)", float(F.cosine_similarity(ga, gb, dim=0)))
    assert abs(la - lf) < 2e-2 * max(1.0, abs(lf))
    assert ca > cb - 0.02                               # as close to fp32 as the library's bf16 path is


def test_block_scaled_mxfp8_gemm_is_exact_on_its_own_quantisation():
    """kind::mxf8f6f4.block_scale with UE8M0 scales per 32 channels: the kernel's result must equal the product of
    the DE-QUANTISED operands (fp32) up to the bf16 rounding of the output -- this pins the scale-factor layout
    (tile [lane][row quarter][k-block]), the TMEM copy and the instruction descriptor; then the quantisation error
    itself against the fp32 product."""
    from hefl_b200 import _ext

    ops = _ext.ops()
    g = torch.Generator(device="cuda").manual_seed(4)
    M, N, K = 1000, 256, 512                                   # M is not a multiple of the 128-row tile
    a = torch.randn(M, K, device="cuda", generator=g) * torch.exp2((torch.arange(M, device="cuda") % 9).float() - 4).unsqueeze(1)
    b = torch.randn(N, K, device="cuda", generator=g) * torch.exp2(((torch.arange(K, device="cuda") // 32) % 5).float()).unsqueeze(0)
    qa, sa = ops.mxfp8_quantize(a.to(torch.bfloat16))
    qb, sb = ops.mxfp8_quantize(b.to(torch.bfloat16))

    def dequant(q, sf, R):
        Rp = (R + 127) // 128 * 128
        e = sf.view(Rp // 128, K // 128, 32, 4, 4).permute(0, 3, 2, 1, 4).reshape(Rp, K // 32)[:R].float() - 127.0
        return (q.view(torch.float8_e4m3fn).float().view(R, K // 32, 32) * torch.exp2(e).unsqueeze(-1)).view(R, K)

    da, db = dequant(qa, sa, M), dequant(qb, sb, N)
    out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    ops.gemm_mxfp8(qa, qb, sa, sb, out)
    ref = da @ db.t()
    assert _rel(out, ref) < 6e-3                               # bf16 output rounding only
    full = a.to(torch.bfloat16).float() @ b.to(torch.bfloat16).float().t()
    err = (out.float() - full).abs().mean() / full.abs().mean()
    assert float(err) < 0.05, float(err)                       # e4m3 with per-32 scales: ~2-3 %


def test_conv1x1_mxfp8_forward_and_dgrad_track_fp32():
    from hefl_b200.ops import tc_conv

    x, w, g = _mk(4, 256, 512, 28, 1, 5)
    xr = x.float().requires_grad_(True)
    wr = w.clone().requires_grad_(True)
    ref = F.conv2d(xr, wr)
    gy = torch.randn(ref.shape, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    ref.backward(gy.float())
    xt = x.clone().requires_grad_(True)
    wt = w.clone().requires_grad_(True)
    out = tc_conv.conv1x1(xt, wt, 1, "mx")
    out.backward(gy)
    for got, want in ((out, ref), (xt.grad, xr.grad)):
        cos = F.cosine_similarity(got.float().flatten(), want.detach().flatten(), dim=0)
        assert float(cos) > 0.998, float(cos)
    assert _rel(wt.grad, wr.grad) < 1e-2                        # the weight gradient stays in bf16

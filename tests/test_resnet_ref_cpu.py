"""The float64 references of tests/resnet_ref.py against PyTorch autograd, the quantiser references on hand-built
boundary cases, and each bound against the defect it must be able to see (no GPU needed)."""
import pytest
import torch
import torch.nn.functional as F

import resnet_ref as R

SMS = 132


def _rand(*shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g, dtype=torch.float64)


def _bf(*shape, seed, scale=1.0):
    return (_rand(*shape, seed=seed) * scale).to(torch.bfloat16)


# ---------------------------------------------------------------------------------------------- convolutions
@pytest.mark.parametrize("B,Cin,Cout,H,stride", [(2, 24, 16, 7, 1), (2, 24, 8, 7, 2), (1, 16, 24, 8, 2)])
def test_conv1x1_reference_matches_autograd(B, Cin, Cout, H, stride):
    x = _rand(B, Cin, H, H, seed=1).requires_grad_(True)
    w = _rand(Cout, Cin, 1, 1, seed=2).requires_grad_(True)
    y = F.conv2d(x, w, stride=stride)
    Ho = y.shape[2]
    gy = _rand(*y.shape, seed=3)
    y.backward(gy)
    x2 = R.nhwc(x.detach())
    xs = R.subsample(x2, B, H, H, stride)
    w2 = w.detach().view(Cout, Cin)
    dy2 = R.nhwc(gy)
    assert torch.allclose(R.conv1x1_fwd(xs, w2), R.nhwc(y.detach()), rtol=0, atol=1e-12)
    dx = R.scatter_even(R.conv1x1_dgrad(dy2, w2), B, H, H, stride)
    assert torch.allclose(dx, R.nhwc(x.grad), rtol=0, atol=1e-12)
    assert torch.allclose(R.conv1x1_wgrad(dy2, xs), w.grad.view(Cout, Cin), rtol=0, atol=1e-12)
    assert Ho == (H + stride - 1) // stride


@pytest.mark.parametrize("B,Cin,Cout,H,W", [(2, 24, 16, 7, 7), (1, 8, 24, 5, 9)])
def test_conv3x3_reference_matches_autograd(B, Cin, Cout, H, W):
    x = _rand(B, Cin, H, W, seed=4).requires_grad_(True)
    w = _rand(Cout, Cin, 3, 3, seed=5).requires_grad_(True)
    y = F.conv2d(x, w, padding=1)
    gy = _rand(*y.shape, seed=6)
    y.backward(gy)
    x2, dy2 = R.nhwc(x.detach()), R.nhwc(gy)
    assert torch.allclose(R.conv3x3_fwd(x2, w.detach(), B, H, W), R.nhwc(y.detach()), rtol=0, atol=1e-12)
    assert torch.allclose(R.conv3x3_dgrad(dy2, w.detach(), B, H, W), R.nhwc(x.grad), rtol=0, atol=1e-12)
    assert torch.allclose(R.conv3x3_wgrad(dy2, x2, B, H, W), w.grad, rtol=0, atol=1e-12)
    # the |terms| sums bound |result| and are reached by non-negative data
    assert bool((R.conv3x3_fwd(x2, w.detach(), B, H, W).abs() <= R.conv3x3_fwd_abs(x2, w.detach(), B, H, W) + 1e-12).all())
    assert torch.allclose(R.conv3x3_fwd(x2.abs(), w.detach().abs(), B, H, W), R.conv3x3_fwd_abs(x2, w.detach(), B, H, W))


def test_conv_bounds_reject_a_dropped_tap_and_a_missing_rotation():
    B, C, H = 2, 24, 7
    x2 = _bf(B * H * H, C, seed=7)
    w = _bf(C, C, 3, 3, seed=8, scale=0.2).double()
    dy2 = _bf(B * H * H, C, seed=9)
    K = 9 * C
    ref = R.conv3x3_fwd(x2, w, B, H, H)
    bound = R.gemm_bound(ref, R.conv3x3_fwd_abs(x2, w, B, H, H), K)
    assert R.within(R.bf16_rn(ref), ref, bound)[0]
    for tap in (0, 4, 8):           # a corner tap, the centre, the last
        ok, msg = R.within(R.bf16_rn(R.conv3x3_fwd(x2, w, B, H, H, drop_tap=tap)), ref, bound)
        assert not ok, (tap, msg)
    dref = R.conv3x3_dgrad(dy2, w, B, H, H)
    dbound = R.gemm_bound(dref, R.conv3x3_dgrad_abs(dy2, w, B, H, H), K)
    assert R.within(R.bf16_rn(dref), dref, dbound)[0]
    assert not R.within(R.bf16_rn(R.conv3x3_dgrad(dy2, w, B, H, H, rotate=False)), dref, dbound)[0]


# ---------------------------------------------------------------------------------------------- BatchNorm / pool
def _bn_data(P, C, seed, offset=0.0):
    x2 = (_rand(P, C, seed=seed) + offset).to(torch.bfloat16)
    res2 = _bf(P, C, seed=seed + 1)
    gamma = (1 + 0.2 * _rand(C, seed=seed + 2)).float()
    beta = (0.1 * _rand(C, seed=seed + 3)).float()
    return x2, res2, gamma, beta


@pytest.mark.parametrize("res,relu", [(True, True), (False, True), (False, False)])
def test_bn_reference_matches_autograd(res, relu):
    B, C, H = 2, 24, 7
    P = B * H * H
    x2, res2, gamma, beta = _bn_data(P, C, 10)
    res2 = res2 if res else None
    eps, mom = 1e-5, 0.1
    xt = x2.double().view(B, H, H, C).permute(0, 3, 1, 2).requires_grad_(True)
    rt = res2.double().view(B, H, H, C).permute(0, 3, 1, 2).requires_grad_(True) if res else None
    g = gamma.double().requires_grad_(True)
    b = beta.double().requires_grad_(True)
    rm, rv = torch.zeros(C, dtype=torch.float64), torch.ones(C, dtype=torch.float64)
    out = F.batch_norm(xt, rm, rv, g, b, True, mom, eps)
    if res:
        out = out + rt
    if relu:
        out = F.relu(out)
    y, z, mean, var, invstd = R.bn_forward(x2, res2, gamma, beta, eps, relu)
    assert torch.allclose(y, R.nhwc(out.detach()), rtol=0, atol=1e-12)
    m2, v2 = R.bn_running(torch.zeros(C), torch.ones(C), mean, var, P, mom)
    assert torch.allclose(m2, rm) and torch.allclose(v2, rv)
    dy2 = _bf(P, C, seed=20)
    out.backward(dy2.double().view(B, H, H, C).permute(0, 3, 1, 2))
    # float64 y is never 0 < y < bf16 underflow here, so the bf16 mask equals autograd's
    mask = R.relu_mask(R.bf16_rn(y), relu)
    dx, dres, dgamma, dbeta = R.bn_backward(dy2, x2, mask, gamma, mean, invstd)
    assert torch.allclose(dx, R.nhwc(xt.grad), rtol=0, atol=1e-12)
    assert torch.allclose(dgamma, g.grad, rtol=0, atol=1e-12) and torch.allclose(dbeta, b.grad, rtol=0, atol=1e-12)
    if res:
        assert torch.allclose(dres, R.nhwc(rt.grad), rtol=0, atol=1e-12)


def test_bn_bounds_reject_biased_running_var_p_minus_1_and_a_skipped_residual():
    P, C, eps = 98, 24, 1e-5
    x2, res2, gamma, beta = _bn_data(P, C, 30)
    ref = R.bn_forward(x2, res2, gamma, beta, eps, True)
    bb = R.BNBounds(x2, gamma, beta, eps, SMS, ref)
    bound, _ = bb.forward(x2, res2, ref[1])
    assert R.within(R.bf16_rn(ref[0]), ref[0], bound)[0]
    bad = R.bn_forward(x2, res2, gamma, beta, eps, True, var_div=P - 1)
    assert not R.within(R.bf16_rn(bad[0]), ref[0], bound)[0]
    assert not R.within(bad[4], ref[4], bb.invstd_bound())[0]
    assert not R.within(R.bf16_rn(R.bn_forward(x2, res2, gamma, beta, eps, True, skip_res=True)[0]), ref[0], bound)[0]
    # running variance: unbiased, not the biased batch variance
    rm, rv = torch.zeros(C), torch.ones(C)
    m2, v2 = R.bn_running(rm, rv, ref[2], ref[3], P, 0.1)
    dm, dv = bb.running(rm, rv, 0.1)
    assert not R.within(0.9 * rv.double() + 0.1 * ref[3], v2, dv)[0]
    assert R.within(v2.float(), v2, dv)[0] and R.within(m2.float(), m2, dm)[0]
    # backward: dx from the exact gradient is within, a skipped residual's mask is not
    dy2 = _bf(P, C, seed=40)
    mask = R.relu_mask(R.bf16_rn(ref[0]), True)
    dx, d, dgamma, dbeta = R.bn_backward(dy2, x2, mask, gamma, ref[2], ref[4])
    ddg, ddb, dxb = bb.backward(x2, d, dgamma, dbeta, dx)
    assert R.within(R.bf16_rn(dx), dx, dxb)[0]
    bad_mask = R.relu_mask(R.bf16_rn(R.bn_forward(x2, res2, gamma, beta, eps, True, skip_res=True)[0]), True)
    bdx, _, bdg, bdb = R.bn_backward(dy2, x2, bad_mask, gamma, ref[2], ref[4])
    assert not R.within(bdb, dbeta, ddb)[0] and not R.within(R.bf16_rn(bdx), dx, dxb)[0]


def test_bn_mask_comes_from_the_rounded_output():
    """A channel whose output is positive but below half the smallest bf16 subnormal rounds to 0: its gradient is
    masked. A reference that takes the mask from the unrounded output passes gradient there and is rejected."""
    P, C, eps = 98, 24, 1e-5
    x2, res2, gamma, beta = _bn_data(P, C, 50)
    gamma[0], beta[0] = 0.0, 3e-41                 # z = 3e-41 > 0 on every pixel of channel 0
    ref = R.bn_forward(x2, None, gamma, beta, eps, True)
    yb = R.bf16_rn(ref[0])
    assert bool((ref[1][:, 0] > 0).all()) and bool((yb[:, 0] == 0).all())
    bb = R.BNBounds(x2, gamma, beta, eps, SMS, ref)
    dy2 = _bf(P, C, seed=51)
    dx, d, dgamma, dbeta = R.bn_backward(dy2, x2, R.relu_mask(yb, True), gamma, ref[2], ref[4])
    ddg, ddb, _ = bb.backward(x2, d, dgamma, dbeta, dx)
    assert float(dbeta[0]) == 0.0
    _, d_bad, _, dbeta_bad = R.bn_backward(dy2, x2, ref[1] > 0, gamma, ref[2], ref[4])
    assert not torch.equal(d_bad, d)
    assert not R.within(dbeta_bad, dbeta, ddb)[0]


def test_avgpool_reference_matches_autograd():
    B, HW, C = 3, 49, 24
    x3 = _bf(B, HW, C, seed=60)
    xt = x3.double().view(B, 7, 7, C).permute(0, 3, 1, 2).requires_grad_(True)
    out = F.adaptive_avg_pool2d(xt, 1).flatten(1)
    assert torch.allclose(R.avgpool_fwd(x3), out.detach(), rtol=0, atol=1e-14)
    dout = _rand(B, C, seed=61)
    out.backward(dout)
    assert torch.allclose(R.avgpool_bwd(dout, HW), xt.grad.permute(0, 2, 3, 1).reshape(B, HW, C), rtol=0, atol=1e-14)


# ---------------------------------------------------------------------------------------------- quantisers
def test_mx_exponent_boundaries():
    cases = [0.0, 448.0, 448.0 * 2 ** 5, 448.0 * 2 ** -20, 1.0, 256.0, 2.0 ** -133, 2.0 ** -126]
    for a in cases:
        e = int(R.mx_exponent(torch.tensor([a]))[0])
        if a == 0:
            assert e == -127
            continue
        assert a * 2.0 ** -e <= 448 and (e == -127 or a * 2.0 ** -(e - 1) > 448), (a, e)
    # amax exactly 448 * 2^k -> e = k; one bf16 ulp above -> e = k + 1
    for k in (-10, 0, 7):
        a = torch.tensor([448.0 * 2 ** k], dtype=torch.bfloat16)
        up = a.float() + 2.0 ** (8 + k - 7)            # 448 = 1.75 * 2^8: the bf16 ulp there is 2^(8 - 7)
        assert float(up.to(torch.bfloat16).float()) == float(up)
        assert int(R.mx_exponent(a.float())[0]) == k
        assert int(R.mx_exponent(up)[0]) == k + 1


def _mx_block(vals):
    x = torch.zeros(1, 128, dtype=torch.bfloat16)
    x[0, : len(vals)] = torch.tensor(vals, dtype=torch.float64).to(torch.bfloat16)
    return x


def test_mx_quantize_boundary_blocks():
    x = torch.zeros(130, 256, dtype=torch.bfloat16)      # 130 rows: a partial second row block of 2 rows
    x[0, 32:64] = 448.0 * 4                              # k-block 1: amax = 448 * 2^2
    x[0, 64] = 448.0 * 4 + 8                             # k-block 2: one bf16 ulp above
    x[1, :32] = torch.tensor([2.0 ** -133 * (i % 16 + 1) for i in range(32)]).to(torch.bfloat16)   # bf16 subnormals
    x[129, 224:] = -3.0
    q, sf, e = R.mx_quantize(x)
    assert int(e[0, 0]) == -127 and int(e[0, 1]) == 2 and int(e[0, 2]) == 3 and int(e[1, 0]) == -127
    assert int(e[129, 7]) == -7                          # 3 * 2^7 = 384 <= 448 < 768
    assert sf.numel() == 2 * 2 * 512
    tiles = sf.view(2, 2, 32, 4, 4)                      # [row block][k-group][lane][quarter][k-block]
    assert int(tiles[0, 0, 0, 0, 0]) == 0 and int(tiles[0, 0, 0, 0, 1]) == 129 and int(tiles[0, 0, 0, 0, 2]) == 130
    assert int(tiles[1, 1, 1, 0, 3]) == 120              # row 129 = block 1, lane 1, quarter 0; k-block 7
    pad = tiles[1].permute(2, 1, 0, 3).reshape(128, 8)[2:]   # rows 130..255 of the last block
    assert bool((pad == 127).all())
    # element bytes: 1792 * 2^-2 = 448 = 0x7E, 0 = 0x00, the subnormals scaled by 2^127 are exact
    assert int(q[0, 32]) == 0x7E and int(q[0, 0]) == 0
    back = R.mx_dequantize(q, sf, 130, 256)
    assert torch.equal(back[1, :32], x[1, :32].double())
    assert torch.equal(back[129, 224:], x[129, 224:].double())
    assert float(back[0, 64]) == 224 * 8 != float(x[0, 64])   # 1800 / 8 = 225 rounds to 224 in e4m3


def test_mx_quantize_round_trips_small_integers_and_matches_a_closed_form():
    g = torch.Generator().manual_seed(70)
    x = torch.randint(-4, 5, (200, 384), generator=g).to(torch.bfloat16)
    q, sf, e = R.mx_quantize(x)
    assert torch.equal(R.mx_dequantize(q, sf, 200, 384), x.double())
    y = (torch.randn(200, 384, generator=g) * torch.exp2(torch.randint(-30, 30, (200, 1), generator=g).float())).to(torch.bfloat16)
    amax = y.float().view(200, 12, 32).abs().amax(-1).double()
    closed = torch.ceil(torch.log2(amax / 448.0)).long()
    assert torch.equal(R.mx_exponent(amax), closed)


def test_per_tensor_quantizer_saturates_and_records_amax():
    x = torch.tensor([0.0, 1.0, -1.0, 500.0, -1e4, 448.0, 449.0, 2.0 ** -12, 3.0], dtype=torch.bfloat16)
    q, amax = R.fp8_quantize(x, 1.0, amax_prev=0.5)
    assert q.tolist()[:6] == [0x00, 0x38, 0xB8, 0x7E, 0xFE, 0x7E]
    assert q.tolist()[6] == 0x7E and amax == 9984.0       # 1e4 is 9984 in bf16
    assert q.tolist()[7] == 0x00                           # 2^-12 is below half the smallest e4m3 subnormal 2^-9
    q2, amax2 = R.fp8_quantize(x, 0.25, amax_prev=1e5)
    assert q2.tolist()[3] == 0x70 and amax2 == 1e5         # 500 / 4 = 125 rounds to 128 (e4m3 step 8 there)
    assert q2.tolist()[8] == 0x34                          # 0.75 = 1.5 * 2^-1: exponent field 6, mantissa 100


def test_scale_update_reference():
    s, inv, amax = R.fp8_scale_update(3.0, 1.0, 224.0)
    assert s == float(torch.tensor(224.0) / torch.tensor(3.0)) and inv == float(1 / torch.tensor(s)) and amax == 0.0
    assert R.fp8_scale_update(0.0, 3.0, 224.0) == (3.0, float(1 / torch.tensor(3.0)), 0.0)      # amax 0 keeps the scale

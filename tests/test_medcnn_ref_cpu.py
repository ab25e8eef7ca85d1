"""The float64 references of tests/medcnn_ref.py against PyTorch autograd, and their bounds against the defects the GPU
tests must be able to see (no GPU needed)."""
import pytest
import torch
import torch.nn.functional as F

import medcnn_ref as R


def _rand(*shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g, dtype=torch.float64)


@pytest.mark.parametrize("B,H,Ci,Co", [(2, 10, 3, 8), (3, 13, 4, 8), (1, 9, 2, 16)])
def test_fwd_pool_matches_torch_on_tie_free_data(B, H, Ci, Co):
    x, w, b = _rand(B, Ci, H, H, seed=1), _rand(Co, Ci, 3, 3, seed=2), _rand(Co, seed=3)
    p = R.fwd_pool(x, w, b)
    conv = F.conv2d(x, w, b)
    ref, idx = F.max_pool2d(F.relu(conv), 2, return_indices=True)
    assert torch.allclose(p.out, ref, rtol=0, atol=1e-12)
    # positions, where the window's maximum is positive (ReLU leaves ties at zero otherwise)
    Wo = H - 2
    pos = ((idx // Wo) % 2) * 2 + (idx % Wo) % 2
    sel = ref > 0
    assert torch.equal((p.code.long() & 3)[sel], pos[sel])
    assert torch.equal((p.code & 4) != 0, F.max_pool2d(conv, 2) > 0)
    assert bool((p.gap > 0).all())
    # S bounds |conv| and is reached with non-negative data
    assert bool((p.act.abs() <= p.S + 1e-12).all())
    q = R.fwd_pool(x.abs(), w.abs(), b.abs())
    assert torch.allclose(q.act, q.S, rtol=1e-14, atol=0)


def _window(v00, v01, v10, v11, bias=0.0):
    """One 2x2 pooling window as the conv output of a 1x1 identity filter (3x3 kernel with only the centre tap)."""
    x = torch.zeros(1, 1, 4, 4, dtype=torch.float64)
    x[0, 0, 1:3, 1:3] = torch.tensor([[v00, v01], [v10, v11]], dtype=torch.float64)
    w = torch.zeros(1, 1, 3, 3, dtype=torch.float64)
    w[0, 0, 1, 1] = 1
    p = R.fwd_pool(x, w, torch.tensor([bias], dtype=torch.float64))
    return int(p.code.view(-1)[0]), float(p.out.view(-1)[0])


@pytest.mark.parametrize("win,bias,code", [
    ((1, 1, 1, 1), 0, 0b100),          # all equal: top-left, active
    ((0, 0, 0, 0), 0, 0b000),          # all zero: top-left, inactive (max + bias == 0 is not > 0)
    ((0, 0, 0, 0), 1, 0b100),
    ((-1, -1, -1, -1), 0, 0b000),
    ((2, 2, 2, 2), -2, 0b000),         # max + bias exactly zero
    ((1, 2, 1, 2), 0, 0b101),          # right column strictly greater, rows tie -> upper
    ((1, 1, 2, 2), 0, 0b110),          # lower row strictly greater, columns tie -> left
    ((1, 1, 1, 2), 0, 0b111),
    ((3, 1, 1, 3), 0, 0b100),          # columns tie at 3 (upper-left vs lower-right): left wins
    ((1, 3, 3, 1), 0, 0b110),          # columns tie at 3 (lower-left vs upper-right): left wins, its lower row
    ((0, -1, 0, 0), 0, 0b000),         # zero ties in the left column; right column max 0 is not greater
])
def test_tie_rule_on_hand_built_windows(win, bias, code):
    got, out = _window(*win, bias=bias)
    assert got == code, (win, bias, bin(got))
    assert out == max(max(win) + bias, 0)


def _autograd_layer(x, w, b, gp):
    x, w, b = (t.clone().requires_grad_(True) for t in (x, w, b))
    pooled = F.max_pool2d(F.relu(F.conv2d(x, w, b)), 2)
    pooled.backward(gp)
    return x.grad, w.grad, b.grad


@pytest.mark.parametrize("B,H,Ci,CK,Co", [(2, 10, 3, 16, 8), (2, 13, 4, 4, 8), (3, 11, 8, 8, 16)])
def test_backward_references_match_autograd(B, H, Ci, CK, Co):
    """unpool -> dgrad / wgrad, and wgrad0 from the pooled gradient, == autograd through conv -> ReLU -> max-pool
    (odd H included: the floor pool drops the last conv row and column)."""
    x, w, b = _rand(B, Ci, H, H, seed=4), _rand(Co, Ci, 3, 3, seed=5), _rand(Co, seed=6)
    Hp = (H - 2) // 2
    gp = _rand(B, Co, Hp, Hp, seed=7)
    gx, gw, gb = _autograd_layer(x, w, b, gp)
    p = R.fwd_pool(x, w, b)
    dy = R.unpool(gp, p.out, p.code, H, H)
    assert float(dy[..., H - 2:, :].abs().max()) == 0 and float(dy[..., H - 2:].abs().max()) == 0
    if H % 2:
        assert float(dy[..., H - 3, :].abs().max()) == 0           # dropped conv row of the floor pool
    assert torch.allclose(R.dgrad(dy, w), gx, rtol=0, atol=1e-12)
    dW = R.wgrad(x, dy, CK)
    rw, rb = R.wgrad_to_oihw(dW, Ci, CK, Co)
    assert torch.allclose(rw, gw, rtol=0, atol=1e-12) and torch.allclose(rb, gb, rtol=0, atol=1e-12)
    assert int(torch.count_nonzero(dW[: 9 * CK].view(9, CK, Co)[:, Ci:])) == 0
    assert torch.equal(R.wgrad0(x, gp, p.code, CK), dW)
    assert bool((R.wgrad_abs(x, dy, CK) >= dW.abs()).all())


def test_layer1_packers_hold_each_layouts_neighbours():
    img = torch.arange(2 * 5 * 7 * 3, dtype=torch.float32).view(2, 5, 7, 3) + 1
    c = R.pack_compact(img).view(2, 5, 7, 4)
    assert torch.equal(c[..., :3], img) and float(c[..., 3].abs().max()) == 0
    s = R.pack_s(img).view(2, 5, 7, 16)
    for sh in range(3):
        assert torch.equal(s[:, :, : 7 - sh, 3 * sh: 3 * sh + 3], img[:, :, sh:])
        assert int(torch.count_nonzero(s[:, :, 7 - sh:, 3 * sh: 3 * sh + 3])) == 0
    assert float(s[..., 9:].abs().max()) == 0
    g = img[..., :1]
    rs = R.pack_rs(g).view(2, 5, 7, 16)
    for r in range(3):
        for sh in range(3):
            assert torch.equal(rs[:, : 5 - r, : 7 - sh, 3 * r + sh], g[:, r:, sh:, 0])
    assert int((rs != 0).sum()) == sum((5 - r) * (7 - sh) for r in range(3) for sh in range(3)) * 2


def test_wgrad_last_unit_is_the_odd_layer_2_unit():
    b, rows, cols = R.wgrad_last_unit(32, 127, 127)
    assert b == 31 and (rows.start, rows.stop) == (112, 125) and (cols.start, cols.stop) == (64, 125)
    b, rows, cols = R.wgrad_last_unit(3, 6, 6)
    assert (rows.start, rows.stop) == (0, 4) and (cols.start, cols.stop) == (0, 4)


@pytest.mark.parametrize("H", [12, 13])
def test_bounds_pass_a_faithful_kernel_and_reject_the_defects(H):
    """The bounded comparisons of the GPU tests: an fp32 computation rounded to bf16 passes them, and each defect the
    GPU tests use as a tooth (one input channel's tap zeroed, the last conv column ignored by the pool, one dgrad tap
    dropped, one wgrad unit omitted) fails them."""
    B, Ci, Co = 2, 8, 16
    n = 9 * Ci
    x = R.bf16_rn(_rand(B, Ci, H, H, seed=8)).double()
    w = R.bf16_rn(_rand(Co, Ci, 3, 3, seed=9) * 0.3).double()
    b = _rand(Co, seed=10) * 0.1
    ref = R.fwd_pool(x, w, b)
    conv32 = F.conv2d(x.float(), w.float())
    got = R.bf16_rn(F.max_pool2d(F.relu(conv32[..., : 2 * ((H - 2) // 2), : 2 * ((H - 2) // 2)]
                                        + b.float().view(1, -1, 1, 1)), 2))
    assert R.within(got, ref.out, R.fwd_bound(ref.out, ref.S, n))
    for bad in (R.fwd_pool(x, R.drop_tap(w, 3, 1, 2), b), R.fwd_pool(x, w, b, drop_last_col=True)):
        assert not R.within(got, bad.out, R.fwd_bound(bad.out, bad.S, n))
    # dgrad
    Hp = (H - 2) // 2
    dy = R.unpool(R.bf16_rn(_rand(B, Co, Hp, Hp, seed=11)).double(), ref.out, ref.code, H, H)
    gx = R.bf16_rn(R.dgrad(dy.float(), w.float()))
    nd = 9 * Co
    rd, sd = R.dgrad(dy, w), R.dgrad_abs(dy, w)
    assert R.within(gx, rd, R.fwd_bound(rd, sd, nd))
    w_bad = R.drop_tap(w, None, 0, 1)
    assert not R.within(gx, R.dgrad(dy, w_bad), R.fwd_bound(R.dgrad(dy, w_bad), R.dgrad_abs(dy, w_bad), nd))
    # wgrad: the sanity bound of the GPU tests
    dW = R.wgrad(x.float(), dy.float(), Ci).double()
    rW, sW = R.wgrad(x, dy, Ci), R.wgrad_abs(x, dy, Ci)
    assert R.within(dW, rW, 2.0 ** -14 * sW)
    bad = rW.clone()
    bad[3 * Ci + 5] = 0                                     # one (tap, input channel) row not written
    assert not R.within(dW, bad, 2.0 ** -14 * sW)
    assert not torch.equal(R.wgrad(x, R.omit_unit(dy, R.wgrad_last_unit(B, H, H)), Ci), rW)

"""The fused layer-2 backward (conv_dgrad_wgrad, conv_tcgen05.cu G3): both gradients of a CK = Co = 32 layer from one
pass over dY, the same bits as the standalone conv_dgrad and conv_wgrad. The weight and bias gradient must also equal
the float64 reference exactly on integer data (every sum of |terms| below 2^24, so fp32 accumulation is exact in any
order). Outputs, dW32 margins and the workspace are NaN-poisoned first."""
import os

import pytest
import torch

import medcnn_ref as R
from kernel_trace import kernels_run, ran

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from hefl_b200 import _ext
    ops = _ext.ops()

NAN = float("nan")
C = 32
PAD = 64          # poisoned rows / floats around every output


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _weights(g, integer):
    ws = []
    for ci, co in zip(R.MEDCNN_CI, R.MEDCNN_CO):
        if integer:
            ws.append(torch.randint(-4, 5, (co, ci, 3, 3), generator=g, device="cuda").to(torch.bfloat16))
        else:
            ws.append((torch.randn((co, ci, 3, 3), generator=g, device="cuda") / (3 * ci ** 0.5)).to(torch.bfloat16))
    return ws


def _operands(B, H, g, integer):
    """X [P, 32] and dY [P, 32] with dY zero outside the valid (H-2) x (H-2) grid, as unpool_relu leaves it."""
    P = B * H * H
    if integer:
        X = torch.randint(-8, 9, (P, C), generator=g, device="cuda").to(torch.bfloat16)
        dy = torch.randint(-2, 3, (B, H, H, C), generator=g, device="cuda").to(torch.bfloat16)
    else:
        X = torch.randn((P, C), generator=g, device="cuda").to(torch.bfloat16)
        dy = torch.randn((B, H, H, C), generator=g, device="cuda").to(torch.bfloat16)
    dy[:, H - 2:] = 0
    dy[:, :, H - 2:] = 0
    return X, dy.reshape(P, C).contiguous()


def _poisoned(n, cols=None, dtype=torch.bfloat16):
    shape = (n + 2 * PAD,) if cols is None else (n + 2 * PAD, cols)
    buf = torch.full(shape, NAN, dtype=dtype, device="cuda")
    return buf, buf[PAD: PAD + n]


def _margins_nan(buf, n):
    return bool(torch.isnan(buf[:PAD].float()).all()) and bool(torch.isnan(buf[PAD + n:].float()).all())


def _poison_workspace():
    """Best-effort: a freed NaN block at least as large as the workspace, for the binding's at::empty to take."""
    t = torch.full((2 * torch.cuda.get_device_properties(0).multi_processor_count * (9 * C + 1) * C,), NAN,
                   dtype=torch.float32, device="cuda")
    del t


def _fused(X, dY, Wd, B, H):
    P = B * H * H
    dx_buf, dX = _poisoned(P, C)
    dw_buf, dW = _poisoned((9 * C + 1) * C, dtype=torch.float32)
    dW.zero_()
    _poison_workspace()
    ops.conv_dgrad_wgrad(X, dY, Wd, dX, dW, B, H, H, C, C)
    torch.cuda.synchronize()
    assert _margins_nan(dx_buf, P) and _margins_nan(dw_buf, (9 * C + 1) * C)
    return dX, dW


def _pair(X, dY, Wd, B, H):
    P = B * H * H
    dX = torch.full((P, C), NAN, dtype=torch.bfloat16, device="cuda")
    ops.conv_dgrad(dY, Wd, dX, B, H, H, C, C)
    dW = torch.zeros((9 * C + 1) * C, dtype=torch.float32, device="cuda")
    ops.conv_wgrad(X, dY, dW, B, H, H, C, C)
    return dX, dW


# B = 3 at 127 ends on a partial tile; 111 is layer 2 of a 224 x 224 input (another column-tile count)
SHAPES = [(1, 127), (3, 127), (32, 127), (8, 111)]


@pytest.mark.parametrize("B,H", SHAPES)
def test_exact_on_integer_data(B, H):
    g = _gen(10 * B + H)
    ws = _weights(g, True)
    lay = R.weight_layouts(ops, ws)
    w = ws[1].double()
    X, dY = _operands(B, H, g, True)
    (dX, dW), names = kernels_run(lambda: _fused(X, dY, lay.Wd[1], B, H))
    assert ran(names, "dgrad_wgrad_kernel") and ran(names, "reduce_partials_kernel"), sorted(names)
    assert not ran(names, "tap_gemm_kernel") and not ran(names, "wgrad_kernel"), sorted(names)
    xr, dy = R.nchw(X, B, H, H), R.nchw(dY, B, H, H)
    assert R.max_abs_sum_ok(R.dgrad_abs(dy, w)) and R.max_abs_sum_ok(R.wgrad_abs(xr, dy, C))
    assert torch.equal(dX, R.nhwc(R.bf16_rn(R.dgrad(dy, w))))
    exact = R.wgrad(xr, dy, C)
    assert torch.equal(dW.double().view(-1, C), exact)
    # teeth: the last tile's pixels reach the weight gradient
    dy_cut = dy.clone()
    dy_cut[-1, :, H - 3] = 0
    assert not torch.equal(R.wgrad(xr, dy_cut, C), exact)
    # gX is the bits of the standalone dgrad
    dX_pair, dW_pair = _pair(X, dY, lay.Wd[1], B, H)
    assert torch.equal(dX.view(torch.int16), dX_pair.view(torch.int16)) and torch.equal(dW, dW_pair)


def test_supported_shapes():
    """The 64-column strips of the weight gradient must cover the row for the data gradient: W = 66 (W - 2 = 64) is
    refused, and the engine keeps the standalone pair there."""
    assert ops.conv_dgrad_wgrad_supported(127, 127, 32, 32) and ops.conv_dgrad_wgrad_supported(111, 111, 32, 32)
    assert not ops.conv_dgrad_wgrad_supported(66, 66, 32, 32)
    assert not ops.conv_dgrad_wgrad_supported(127, 127, 32, 64)
    X = torch.zeros(66 * 66, C, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError):
        ops.conv_dgrad_wgrad(X, X, torch.zeros(9 * C * C, dtype=torch.bfloat16, device="cuda"), X.clone(),
                             torch.zeros((9 * C + 1) * C, device="cuda"), 1, 66, 66, C, C)


@pytest.mark.parametrize("B,H", [(32, 127), (8, 111)])
def test_random_data(B, H):
    g = _gen(7 * B + H)
    ws = _weights(g, False)
    lay = R.weight_layouts(ops, ws)
    X, dY = _operands(B, H, g, False)
    dX, dW = _fused(X, dY, lay.Wd[1], B, H)
    dX_pair, dW_pair = _pair(X, dY, lay.Wd[1], B, H)
    assert torch.equal(dX.view(torch.int16), dX_pair.view(torch.int16))
    xr, dy = R.nchw(X, B, H, H), R.nchw(dY, B, H, H)
    ref, S = R.wgrad(xr, dy, C), R.wgrad_abs(xr, dy, C)
    bound = 2.0 ** -14 * S
    assert R.within(dW.double().view(-1, C), ref, bound)
    assert torch.equal(dW, dW_pair)
    bad = ref.clone()
    bad[4 * C] = 0
    assert not R.within(dW.double().view(-1, C), bad, bound)
    # the same bits on a second call
    dX2, dW2 = _fused(X, dY, lay.Wd[1], B, H)
    assert torch.equal(dX2.view(torch.int16), dX.view(torch.int16)) and torch.equal(dW2, dW)


@pytest.mark.parametrize("ch", [3, 1])
def test_engine_step_fused_vs_pair(ch, monkeypatch):
    """A seeded step with the fused layer-2 backward against the same step on the standalone dgrad / wgrad pair
    (forced through the engine's dgrad_wgrad attribute): dY, gX, loss and every gradient are the same bits, and two
    fused steps are bit-identical."""
    from hefl_b200.config import FLConfig
    from hefl_b200.models import ParamPack, create_model
    from hefl_b200.ops.conv_engine import MedCNNEngine

    for k in list(os.environ):
        if k.startswith("HEFL_"):
            monkeypatch.delenv(k)
    torch.manual_seed(5)
    cfg = FLConfig(in_channels=ch)
    B, S = cfg.batch_size, cfg.image_size
    dev = torch.device("cuda")
    model = create_model("medcnn", in_channels=ch).to(dev)
    pack = ParamPack(model)
    eng = MedCNNEngine(model, pack, cfg, dev)
    assert eng.dgrad_wgrad == [False, True, False, False, False, False]
    g = _gen(40 + ch)
    x = torch.randint(0, 256, (B, S, S, ch), dtype=torch.uint8, device="cuda", generator=g)
    y = torch.randint(0, 2, (B,), device="cuda", generator=g)
    out = torch.zeros(2, device="cuda")

    def step():
        pack.grad.zero_()
        eng.train_step(x, y, out, augment=False, opt=None)
        torch.cuda.synchronize()
        return {"grad": pack.grad.clone(), "dY": [t.clone() if t is not None else None for t in eng.dY],
                "gX": [t.clone() if t is not None else None for t in eng.gX], "out": out.clone()}

    fused, names = kernels_run(step)
    assert ran(names, "dgrad_wgrad_kernel"), sorted(names)
    again = step()
    assert torch.equal(again["grad"], fused["grad"]) and torch.equal(again["out"], fused["out"])
    eng.dgrad_wgrad = [False] * eng.n
    pair, names = kernels_run(step)
    assert not ran(names, "dgrad_wgrad_kernel"), sorted(names)
    assert torch.equal(pair["out"], fused["out"])
    for a, b in zip(fused["dY"] + fused["gX"], pair["dY"] + pair["gX"]):
        assert (a is None and b is None) or torch.equal(a.view(torch.int16), b.view(torch.int16))
    # every gradient, layer 2's weights and bias included
    assert torch.equal(fused["grad"], pair["grad"])

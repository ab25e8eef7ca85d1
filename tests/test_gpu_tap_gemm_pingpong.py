"""The tap-GEMM kernel's consumer schedule: two groups of four warps take a CTA's tiles alternately (even tiles group 0,
odd tiles group 1) and each warp holds 32 GEMM rows x all output channels of its column block.

Integer tests (small-integer bf16 operands, every sum of |terms| below 2^24, so fp32 accumulation is exact in any
order) run every forward and dgrad instantiation the dispatch selects, at shapes that put the schedule's edges in
play: tile counts just below, at and just above one and two tiles per CTA slot of the grid (a CTA with a single tile
leaves its second group idle, a CTA with 3 tiles ends on group 0), a 1-image batch, the odd 127 map, the row-packed
maps (62, 30, 14, 6) and the output-channel split of the late layers. Outputs are written into NaN-filled buffers
(codes: 0xFF) with a margin on either side that must stay untouched. Each case is one launch that completes.

The step test runs two default training steps from the same seed on two engines: their pooled outputs, codes, input
gradients and weight gradients are bit-identical, and within the float64 bounds of tests/medcnn_ref.py computed from
each stage's own bf16 input."""
import pytest
import torch

import medcnn_ref as R

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from hefl_b200 import _ext
    ops = _ext.ops()

NAN = float("nan")
MARGIN = 96            # rows of poison before and after every output


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, generator=g, device="cuda").to(torch.bfloat16)


def _poisoned(n, C, dtype=torch.bfloat16):
    """(buffer, view of its rows MARGIN .. MARGIN + n): the kernel writes the view, the rest must stay poisoned."""
    fill = NAN if dtype == torch.bfloat16 else 0xFF
    buf = torch.full((n + 2 * MARGIN, C), fill, dtype=dtype, device="cuda")
    return buf, buf[MARGIN: MARGIN + n]


def _margins_untouched(buf):
    edge = torch.cat([buf[:MARGIN], buf[-MARGIN:]])
    return bool(edge.isnan().all()) if edge.dtype == torch.bfloat16 else bool((edge == 0xFF).all())


# layer (CK, Co) of the medical CNN: 1 = (32, 32), 3 = (32, 64), 4 = (64, 64), 5 = (64, 128). conv_fwd_pool halves
# the output-channel block while tiles x blocks < SMs (132), which picks <CK, 32>, <CK, 64> or <64, 128> below.
FWD_CASES = [
    # (layer, B, H, W)
    (1, 1, 127, 127),      # 62 tiles, one per CTA
    (1, 3, 127, 127),      # 186 tiles: some CTAs with 2, partial last tile column
    (1, 1, 264, 129),      # 131 tiles: one below one per SM
    (1, 1, 266, 129),      # 132 tiles
    (1, 1, 268, 129),      # 133 tiles: CTA 0 has 2
    (1, 1, 530, 129),      # 264 tiles: two per SM
    (1, 1, 532, 129),      # 265 tiles: CTA 0 has 3 (odd)
    (1, 5, 127, 127),      # 310 tiles
    (1, 2, 62, 62),        # row-packed, 62 map
    (1, 32, 62, 62),       # row-packed, 496 tiles
    (3, 1, 30, 30),        # row-packed 30 map, CO = 64 split into two 32-channel blocks
    (3, 32, 30, 30),
    (4, 1, 14, 14),        # CK = 64, channel-split column blocks
    (4, 32, 14, 14),
    (5, 1, 6, 6),          # CO = 128 over four column blocks
    (5, 32, 6, 6),
    (5, 20, 30, 30),       # CO = 128 at 75 tiles: two 64-channel blocks
    (4, 48, 30, 30),       # CO = 64 in one block
    (5, 64, 30, 30),       # CO = 128 in one block (4 passes of 32 channels)
    (3, 64, 30, 30),       # CO = 64 in one block
]


@pytest.mark.parametrize("l,B,H,W", FWD_CASES)
@pytest.mark.parametrize("train", [True, False])
def test_forward_exact_on_integer_data(l, B, H, W, train):
    CK, Co = R.MEDCNN_CI[l], R.MEDCNN_CO[l]
    g = _gen(7 * l + B + H + W)
    ws = [_ints((co, ci, 3, 3), -4, 4, g) for ci, co in zip([3] + R.MEDCNN_CI[1:], R.MEDCNN_CO)]
    lay = R.weight_layouts(ops, ws)
    w = ws[l].double()
    X = _ints((B * H * W, CK), -8, 8, g)
    bias = torch.randint(-20, 21, (Co,), generator=g, device="cuda").float()
    ref = R.fwd_pool(R.nchw(X, B, H, W), w, bias)
    assert R.max_abs_sum_ok(ref.S)
    Hp, Wp = (H - 2) // 2, (W - 2) // 2
    n = B * Hp * Wp
    obuf, out = _poisoned(n, Co)
    cbuf, am = _poisoned(n, Co, torch.uint8)
    ops.conv_fwd_pool(X, lay.Wf[l], bias, out, am if train else None, B, H, W, CK, Co)
    assert torch.equal(out, R.nhwc(R.bf16_rn(ref.out)))
    assert _margins_untouched(obuf)
    if train:
        assert torch.equal(am, R.nhwc(ref.code))
    else:
        assert bool((am == 0xFF).all())
    assert _margins_untouched(cbuf)


# dgrad tiles are 128 consecutive pixels: B = 1, H = T rows of W = 128 gives exactly T tiles. (CK, CO) of the call:
# layers 1-2 (32, 32) -> <32, 32>, layer 3 (64, 32) -> <64, 32>, layer 4 (64, 64) -> <64, 64>, layer 5 (128, 64) ->
# <128, 32> on two column blocks
DGRAD_CASES = [
    # (layer, B, H, W)
    (1, 1, 127, 127),      # 127 tiles, the last one partial
    (1, 32, 127, 127),     # 4033 tiles
    (1, 1, 131, 128), (1, 1, 132, 128), (1, 1, 133, 128),
    (1, 1, 263, 128), (1, 1, 264, 128), (1, 1, 265, 128),
    (1, 1, 527, 128), (1, 1, 528, 128), (1, 1, 529, 128),
    (2, 3, 62, 62),
    (3, 1, 30, 30),        # (CK, CO) = (64, 32)
    (3, 1, 131, 128), (3, 1, 133, 128), (3, 1, 265, 128),
    (3, 32, 30, 30),
    (4, 1, 14, 14),        # (64, 64)
    (4, 1, 133, 128), (4, 1, 265, 128),
    (4, 32, 14, 14),
    (5, 1, 6, 6),          # (128, 64): two 32-channel column blocks, one consumer group
    (5, 32, 6, 6),
    (5, 1, 133, 128),
]


@pytest.mark.parametrize("l,B,H,W", DGRAD_CASES)
def test_dgrad_exact_on_integer_data(l, B, H, W):
    Ci, Co = R.MEDCNN_CI[l], R.MEDCNN_CO[l]
    g = _gen(11 * l + B + H + W)
    ws = [_ints((co, ci, 3, 3), -4, 4, g) for ci, co in zip([3] + R.MEDCNN_CI[1:], R.MEDCNN_CO)]
    lay = R.weight_layouts(ops, ws)
    w = ws[l].double()
    dy = _ints((B, Co, H, W), -3, 3, g).double()
    dy[..., H - 2:, :] = 0          # un-pooled gradients are zero outside the valid conv grid
    dy[..., W - 2:] = 0
    assert R.max_abs_sum_ok(R.dgrad_abs(dy, w))
    dY = R.nhwc(dy).to(torch.bfloat16)
    P = B * H * W
    buf, dX = _poisoned(P, Ci)
    ops.conv_dgrad(dY, lay.Wd[l], dX, B, H, W, Co, Ci)
    assert torch.equal(dX, R.nhwc(R.bf16_rn(R.dgrad(dy, w))))
    assert _margins_untouched(buf)


def _engine_step(seed):
    from hefl_b200.config import FLConfig
    from hefl_b200.models import ParamPack, create_model
    from hefl_b200.ops.conv_engine import MedCNNEngine

    torch.manual_seed(seed)
    cfg = FLConfig()
    dev = torch.device("cuda")
    model = create_model("medcnn").to(dev)
    pack = ParamPack(model)
    eng = MedCNNEngine(model, pack, cfg, dev)
    g = _gen(seed)
    x = torch.randint(0, 256, (cfg.batch_size, cfg.image_size, cfg.image_size, 3), dtype=torch.uint8, device="cuda",
                      generator=g)
    y = torch.randint(0, 2, (cfg.batch_size,), device="cuda", generator=g)
    pack.grad.zero_()
    eng.train_step(x, y, torch.zeros(2, device="cuda"), augment=True)
    torch.cuda.synchronize()
    return eng, list(model.convs)


def test_training_step_reproducible_and_within_bounds():
    (e1, c1), (e2, c2) = _engine_step(5), _engine_step(5)
    B = e1.B
    for l in range(1, e1.n):
        assert torch.equal(e1.X[l + 1], e2.X[l + 1]), f"layer {l + 1} pooled output differs between runs"
        assert torch.equal(e1.amax[l], e2.amax[l]), f"layer {l + 1} codes differ between runs"
        assert torch.equal(e1.gX[l], e2.gX[l]), f"layer {l + 1} dgrad differs between runs"
        assert torch.equal(c1[l].weight.grad, c2[l].weight.grad), f"layer {l + 1} weight gradient differs between runs"
        H, Ci, Co, CK = e1.H[l], e1.Ci[l], e1.Co[l], e1.CK[l]
        Hp = (H - 2) // 2
        w = c1[l].weight.detach().to(torch.bfloat16).double()
        xr = R.nchw(e1.X[l], B, H, H)
        ref = R.fwd_pool(xr, w, c1[l].bias.detach())
        got = R.nchw(e1.X[l + 1], B, Hp, Hp)
        n = 9 * Ci
        assert R.within(got, ref.out, R.fwd_bound(ref.out, ref.S, n)), f"layer {l + 1} pooled output"
        ok, checked = R.codes_agree(R.nchw(e1.amax[l], B, Hp, Hp), ref, n)
        assert ok and checked > 0, f"layer {l + 1} codes"
        dy = R.nchw(e1.dY[l], B, H, H)
        rd, sd = R.dgrad(dy, w), R.dgrad_abs(dy, w)
        assert R.within(R.nchw(e1.gX[l], B, H, H), rd, R.fwd_bound(rd, sd, 9 * Co)), f"layer {l + 1} dgrad"
        rw, rb = R.wgrad_to_oihw(R.wgrad(xr, dy, CK), Ci, CK, Co)
        sw, sb = R.wgrad_to_oihw(R.wgrad_abs(xr, dy, CK), Ci, CK, Co)
        got_w = torch.cat([c1[l].weight.grad.double().reshape(-1), c1[l].bias.grad.double()])
        S = torch.cat([sw.reshape(-1), sb])
        assert R.within(got_w, torch.cat([rw.reshape(-1), rb]), 2.0 ** -14 * S), f"layer {l + 1} weight gradient"

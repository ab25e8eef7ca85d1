"""The pooled forward's output path: pooled values and arg-max codes staged in shared memory and written by TMA
stores (one box per pooled row in the pair-row kernels), against the float64 references of tests/medcnn_ref.py.

Every output and code buffer is a view into a larger allocation whose margins before and after the tensor are
poisoned; the tests assert the margins come back untouched, because a store that writes a whole box could otherwise
run past a pooled row or past the tensor. Integer data keep fp32 accumulation exact (sum of |terms| < 2^24,
asserted), so values and codes must equal the reference bit for bit; on randn data values are held to the derived
bound and codes to `codes_agree`. Evaluation (argmax=None) must leave the code buffer untouched.

Each call must launch exactly one native kernel. Which instantiation the dispatch picks at the training step's shapes
is checked by name in test_gpu_medcnn_step_shapes.py; these tests add no profiler sessions of their own."""
import pytest
import torch

import medcnn_ref as R

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from hefl_b200 import _ext
    ops = _ext.ops()

MARGIN = 512          # rows of poison before and after each output tensor
CODE_POISON = 0xA5


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, generator=g, device="cuda").to(torch.bfloat16)


class Guarded:
    """[n, Co] tensor `t` inside a poisoned [MARGIN + n + MARGIN, Co] allocation."""

    def __init__(self, n, Co, dtype):
        self.n = n
        self.buf = torch.empty(n + 2 * MARGIN, Co, dtype=dtype, device="cuda")
        if dtype == torch.uint8:
            self.buf.fill_(CODE_POISON)
        else:
            self.buf.fill_(float("nan"))
        self.poison = self.buf.clone()
        self.t = self.buf[MARGIN: MARGIN + n]

    def margins_intact(self):
        bits = lambda x: x.view(torch.uint8) if x.dtype == torch.uint8 else x.view(torch.int16)
        return (torch.equal(bits(self.buf[:MARGIN]), bits(self.poison[:MARGIN]))
                and torch.equal(bits(self.buf[MARGIN + self.n:]), bits(self.poison[MARGIN + self.n:])))

    def untouched(self):
        return torch.equal(self.buf.view(torch.uint8), self.poison.view(torch.uint8))


def _run(launch, n, Co, train):
    out, am = Guarded(n, Co, torch.bfloat16), Guarded(n, Co, torch.uint8)
    launches = int(ops.launch_count())
    launch(out.t, am.t if train else None)
    torch.cuda.synchronize()
    assert int(ops.launch_count()) == launches + 1
    assert out.margins_intact(), "pooled values written outside the tensor"
    assert am.margins_intact(), "codes written outside the tensor"
    if not train:
        assert am.untouched(), "evaluation wrote the code buffer"
    return out.t, am.t


def _layer1(ch, B, H, g, integer):
    """Layer-1 input (compact RGB or rs-packed grayscale, with the engine's slack), weights in the kernel's layout,
    bias, and the launcher of the pair-row forward."""
    img = _ints((B, H, H, ch), -8, 8, g) if integer else (torch.rand(B, H, H, ch, generator=g, device="cuda")
                                                          .to(torch.bfloat16))
    w = (_ints((32, ch, 3, 3), -4, 4, g) if integer
         else (torch.randn(32, ch, 3, 3, generator=g, device="cuda") * 0.3).to(torch.bfloat16))
    ws = [w] + [torch.zeros(co, ci, 3, 3, dtype=torch.bfloat16, device="cuda")
                for ci, co in zip(R.MEDCNN_CI[1:], R.MEDCNN_CO[1:])]
    bias = (torch.randint(-20, 21, (32,), generator=g, device="cuda").float() if integer
            else torch.randn(32, generator=g, device="cuda") * 0.1)
    lay = R.weight_layouts(ops, ws, spack0=True, compact0=ch == 3)
    P = B * H * H
    if ch == 3:
        X, wf, args = R.with_slack(R.pack_compact(img), 32)[:P], lay.Wf0c, (True, 3, True)
    else:
        X, wf, args = R.with_slack(R.pack_rs(img))[:P], lay.Wf[0], (True, 1, False)

    def launch(out, am):
        ops.conv_fwd_pool_pair(X, wf, bias, out, am, B, H, H, 16, 32, *args)
    return img.permute(0, 3, 1, 2).double(), w, bias, launch


@pytest.mark.parametrize("ch,B,H", [(3, 4, 256), (3, 3, 66), (1, 4, 256), (1, 2, 40)])
@pytest.mark.parametrize("train", [True, False])
def test_layer1_pair_store_exact(ch, B, H, train):
    """Layer 1 on the pair-row kernels (compact RGB, rs-packed grayscale): the full 127-window row of a 256 map (the
    staged window 127 is never stored) and short rows of 32 and 19 windows."""
    Hp = (H - 2) // 2
    x, w, bias, launch = _layer1(ch, B, H, _gen(7 * H + ch), True)
    ref = R.fwd_pool(x, w, bias)
    assert R.max_abs_sum_ok(ref.S)
    out, am = _run(launch, B * Hp * Hp, 32, train)
    assert torch.equal(out, R.nhwc(R.bf16_rn(ref.out)))
    if train:
        assert torch.equal(am, R.nhwc(ref.code))


@pytest.mark.parametrize("ch", [3, 1])
def test_layer1_pair_store_real_data(ch):
    """Layer 1 on [0, 1) images and randn weights at B = 32, 256 x 256: values within the derived bound, codes agree
    wherever the accumulation error cannot decide them."""
    B, H = 32, 256
    Hp = (H - 2) // 2
    x, w, bias, launch = _layer1(ch, B, H, _gen(50 + ch), False)
    ref = R.fwd_pool(x, w, bias)
    out, am = _run(launch, B * Hp * Hp, 32, True)
    n = 9 * ch
    got = R.nchw(out, B, Hp, Hp)
    assert R.within(got, ref.out, R.fwd_bound(ref.out, ref.S, n))
    ok, checked = R.codes_agree(R.nchw(am, B, Hp, Hp), ref, n)
    assert ok and checked > 0.5 * ref.code.numel()


@pytest.mark.parametrize("CK,Co,B,H", [(32, 32, 3, 62), (32, 64, 2, 62), (32, 64, 2, 258)])
@pytest.mark.parametrize("train", [True, False])
def test_plain_pair_store_exact(CK, Co, B, H, train):
    """The plain pair-row kernel (9 tap GEMMs on a [P, CK] input): Co = 64 stages rows of 128 bytes in two channel
    passes, and H = 258 fills all 128 windows of a row."""
    Hp = (H - 2) // 2
    g = _gen(CK + Co + H)
    l = R.MEDCNN_CO.index(Co) if Co == 64 else 1
    ws = [_ints((co, ci, 3, 3), -4, 4, g) for ci, co in zip(R.MEDCNN_CI, R.MEDCNN_CO)]
    lay = R.weight_layouts(ops, ws)
    X = _ints((B * H * H, CK), -8, 8, g)
    bias = torch.randint(-20, 21, (Co,), generator=g, device="cuda").float()
    ref = R.fwd_pool(R.nchw(X, B, H, H), ws[l], bias)
    assert R.max_abs_sum_ok(ref.S)

    def launch(out, am):
        ops.conv_fwd_pool_pair(X, lay.Wf[l], bias, out, am, B, H, H, CK, Co)
    out, am = _run(launch, B * Hp * Hp, Co, train)
    assert torch.equal(out, R.nhwc(R.bf16_rn(ref.out)))
    if train:
        assert torch.equal(am, R.nhwc(ref.code))


@pytest.mark.parametrize("l,B", [(1, 3), (2, 5), (4, 2), (5, 1)])
@pytest.mark.parametrize("train", [True, False])
def test_tap_gemm_pooled_store_exact(l, B, train):
    """The tap-GEMM pooled forward of layers 2-6: the odd 127 map (floor-pooled column 124 dropped), row-packed tiles
    whose last tile is partial (62 and 14 maps: 155 pairs in tiles of 2, 14 in tiles of 9), and output channels split
    over blockIdx.y (the 14 x 14 and 6 x 6 layers at these batch sizes)."""
    H, CK, Co = [256, 127, 62, 30, 14, 6][l], R.MEDCNN_CI[l], R.MEDCNN_CO[l]
    Hp = (H - 2) // 2
    g = _gen(300 + l + B)
    ws = [_ints((co, ci, 3, 3), -4, 4, g) for ci, co in zip(R.MEDCNN_CI, R.MEDCNN_CO)]
    lay = R.weight_layouts(ops, ws)
    X = _ints((B * H * H, CK), -8, 8, g)
    bias = torch.randint(-20, 21, (Co,), generator=g, device="cuda").float()
    ref = R.fwd_pool(R.nchw(X, B, H, H), ws[l], bias)
    assert R.max_abs_sum_ok(ref.S)

    def launch(out, am):
        ops.conv_fwd_pool(X, lay.Wf[l], bias, out, am, B, H, H, CK, Co)
    out, am = _run(launch, B * Hp * Hp, Co, train)
    assert torch.equal(out, R.nhwc(R.bf16_rn(ref.out)))
    if train:
        assert torch.equal(am, R.nhwc(ref.code))

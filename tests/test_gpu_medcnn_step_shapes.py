"""The medical CNN's kernels at the shapes of its training step (FLConfig() defaults: B = 32, 256 x 256 RGB, and the
grayscale variant), against the float64 references of tests/medcnn_ref.py.

Six conv layers at H = 256, 127, 62, 30, 14, 6. At B = 32 the persistent tap-GEMM kernels loop over many tiles per
CTA (layer 2: 1984 forward tiles, 4033 dgrad tiles on 132 SMs), layer 2's odd 127-pixel map drops conv row and column
124 in the floor pool, and its weight gradient has a second 64-column strip of 61 columns and a last row unit of 13
rows. Every test asks torch.profiler which kernel instantiation ran, so the shape coverage is checked, not assumed.

Integer tests: small-integer bf16 operands keep every output's sum of |terms| below 2^24 (asserted), so fp32
accumulation is exact in any order and a kernel result must equal the exactly rounded float64 one bit for bit
(torch.equal). This relies on the tensor cores' fp32 accumulation being exact for integers below 2^24, as IEEE fp32
addition is. Real-data tests hold randn operands to per-element bounds derived from the accumulation length; each
bound is shown to reject a defective reference (the teeth), so it could see a real defect.

Outputs are filled with NaN (codes with 0xFF) before every call so an unwritten element cannot pass. The weight-
gradient workspaces are allocated inside the bindings with at::empty; just before each such call a NaN block at least
as large is allocated and freed so the caching allocator will probably hand it back as the workspace. That is best-
effort: the allocator is free to pick another block. The fp32 weight-gradient buffers are accumulated into (+=) and
start at zero, as in the engine."""
import copy
import os

import pytest
import torch
import torch.nn.functional as F

import medcnn_ref as R
from kernel_trace import kernels_run, ran

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from hefl_b200 import _ext
    ops = _ext.ops()

NAN = float("nan")
H_OF = [256, 127, 62, 30, 14, 6]
CK_OF = [16, 32, 32, 32, 64, 64]
# instantiations the dispatch selects at B = 32 (layers 2..6; conv_tcgen05.cu conv_fwd_pool / conv_dgrad / wgrad_dispatch)
FWD = {1: "tap_gemm_kernel<32, 32, true, 3>", 2: "tap_gemm_kernel<32, 32, true, 3>", 3: "tap_gemm_kernel<32, 32, true, 3>",
       4: "tap_gemm_kernel<64, 32, true, 3>", 5: "tap_gemm_kernel<64, 32, true, 3>"}
DGRAD = {1: "tap_gemm_kernel<32, 32, false, 3>", 2: "tap_gemm_kernel<32, 32, false, 3>",
         3: "tap_gemm_kernel<64, 32, false, 3>", 4: "tap_gemm_kernel<64, 64, false, 3>",
         5: "tap_gemm_kernel<128, 32, false, 3>"}
WGRAD = {1: "wgrad_kernel<32, 32, false>", 2: "wgrad_kernel<32, 32, false>", 3: "wgrad_kernel<32, 64, true>",
         4: "wgrad_kernel<64, 64, true>", 5: "wgrad_kernel<64, 64, true>"}


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, generator=g, device="cuda").to(torch.bfloat16)


def _randn(shape, g, scale=1.0):
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def _nan(*shape, dtype=torch.bfloat16):
    return torch.full(shape, NAN, dtype=dtype, device="cuda")


def _codes(n, Co):
    return torch.full((n, Co), 0xFF, dtype=torch.uint8, device="cuda")


def _poison_workspace(n_floats):
    """Best-effort: leave a freed NaN block of n_floats in the caching allocator for the next at::empty."""
    t = torch.full((n_floats,), NAN, dtype=torch.float32, device="cuda")
    del t


def _ws_bound(CK, Co):
    """Upper bound of a weight-gradient workspace: at most 2 CTA columns per SM, one [9 CK + 1][Co] partial each."""
    return 2 * torch.cuda.get_device_properties(0).multi_processor_count * (9 * CK + 1) * Co


def _weights(ci0, g, integer):
    ws = []
    for l, (ci, co) in enumerate(zip([ci0] + R.MEDCNN_CI[1:], R.MEDCNN_CO)):
        ws.append(_ints((co, ci, 3, 3), -4, 4, g) if integer else _randn((co, ci, 3, 3), g, 1.0 / (3 * ci ** 0.5)))
    return ws


def _bias(Co, g, integer):
    if integer:
        return torch.randint(-20, 21, (Co,), generator=g, device="cuda").float()
    return torch.randn(Co, generator=g, device="cuda") * 0.1


def _fwd(X, Wf, bias, B, H, CK, Co, train=True):
    Hp = (H - 2) // 2
    out, am = _nan(B * Hp * Hp, Co), _codes(B * Hp * Hp, Co)
    ops.conv_fwd_pool(X, Wf, bias, out, am if train else None, B, H, H, CK, Co)
    return out, am


def _wgrad(X, dY, B, H, CK, Co):
    dW = torch.zeros((9 * CK + 1) * Co, dtype=torch.float32, device="cuda")
    _poison_workspace(_ws_bound(CK, Co))
    ops.conv_wgrad(X, dY, dW, B, H, H, CK, Co)
    return dW


# ---------------------------------------------------------------------------------------------- layer-1 layouts
def test_packers_match_preprocess_u8_on_real_images():
    """The reference packers (compact, s-packed, rs-packed) produce the layer-1 layouts preprocess_u8 writes, bit for
    bit, on 256 x 256 images: the integer tests below feed the layouts the kernels actually read."""
    B, H = 4, 256
    g = _gen(1)
    x = torch.randint(0, 256, (B, H, H, 3), dtype=torch.uint8, device="cuda", generator=g)
    P = B * H * H
    Xc, Xs = _nan(P, 4), _nan(P, 16)
    ops.preprocess_u8(x, None, Xc, 0, None, True, True)
    ops.preprocess_u8(x, None, Xs, 0, None, True)
    img = Xc.view(B, H, H, 4)[..., :3]
    assert torch.equal(img.float(), R.bf16_rn(x.float() / 255.0).float())
    assert torch.equal(Xc.view(torch.int16), R.pack_compact(img).view(torch.int16))
    assert torch.equal(Xs.view(torch.int16), R.pack_s(img).view(torch.int16))
    x1 = x[..., :1].contiguous()
    Xr = _nan(P, 16)
    ops.preprocess_u8(x1, None, Xr, 0, None, True)
    img1 = R.bf16_rn(x1.float() / 255.0)
    assert torch.equal(Xr.view(torch.int16), R.pack_rs(img1).view(torch.int16))


def _layer1_inputs(img, ch):
    """Layer-1 inputs built by the reference packers: (compact, s-packed) for RGB, (rs-packed, rs-packed) for
    grayscale, with the engine's slack behind the last pixel."""
    B, H = img.shape[0], img.shape[1]
    P = B * H * H
    if ch == 3:
        Xc = R.with_slack(R.pack_compact(img), 32)[:P]          # the engine's slack: 8 pixels of 16 channels
        Xs = R.with_slack(R.pack_s(img))
        return Xc, Xs
    Xr = R.with_slack(R.pack_rs(img))
    return Xr, Xr


def _gradient_rows(kern, ch):
    """dW32 rows a layer-1 weight-gradient kernel defines. The FP32 gather reads channels 0-2 of the shifted pixels
    whatever the input, so on the grayscale input its rows for channels 1 and 2 hold products with the rs layout's
    neighbour channels; conv_grad_finalize reads only the rows of channels < Ci. Every other kernel defines all rows
    (the padded ones as zeros)."""
    rows = torch.ones(9 * 16 + 1, dtype=torch.bool, device="cuda")
    if kern == "wgrad0_gather_kernel" and ch == 1:
        rows[: 9 * 16] = (torch.arange(9 * 16, device="cuda") % 16) < ch
    return rows


def _run_layer1(ch, img, ws, bias, gp, B, H):
    """Layer-1 forward (train and eval) and every weight-gradient kernel on the same inputs; returns the outputs and
    the kernels each step ran."""
    Co, Hp = 32, (H - 2) // 2
    P = B * H * H
    lay = R.weight_layouts(ops, ws, spack0=True, compact0=ch == 3)
    Xa, Xb = _layer1_inputs(img, ch)
    if ch == 3:
        fwd_args, wf = (True, 3, True), lay.Wf0c
        variants = {"wgrad0_mma_compact_kernel": (Xa, True, 3, True), "wgrad0_mma_kernel": (Xb, True, 3, False),
                    "wgrad0_gather_kernel": (Xb, False, 3, False)}
    else:
        fwd_args, wf = (True, 1, False), lay.Wf[0]
        variants = {"wgrad0_mma_rs_kernel": (Xa, True, 1, False), "wgrad0_gather_kernel": (Xa, False, 1, False)}

    def fwd(train):
        out, am = _nan(B * Hp * Hp, Co), _codes(B * Hp * Hp, Co)
        ops.conv_fwd_pool_pair(Xa, wf, bias, out, am if train else None, B, H, H, 16, Co,
                               *fwd_args)
        return out, am

    (out, am), names = kernels_run(lambda: fwd(True))
    assert ran(names, "pair_fwd_compact_kernel" if ch == 3 else "pair_fwd_rs_kernel"), sorted(names)
    out_eval, _ = fwd(False)
    grads = {}
    for kern, (X, spack, inch, compact) in variants.items():
        def wg():
            dW = torch.zeros((9 * 16 + 1) * Co, dtype=torch.float32, device="cuda")
            _poison_workspace(_ws_bound(16, Co))
            ops.wgrad0_gather(X, gp, am, dW, B, H, H, spack, inch, compact)
            return dW
        grads[kern], names = kernels_run(wg)
        assert ran(names, kern), (kern, sorted(names))
    return out, am, out_eval, grads


# ---------------------------------------------------------------------------------------------- (a) integer-exact
@pytest.mark.parametrize("ch", [3, 1])
def test_layer1_is_exact_on_integer_data(ch):
    """Layer 1 at B = 32, 256 x 256: the pair-row forward (compact RGB / rs-packed grayscale input) and every layer-1
    weight-gradient kernel (compact, s-packed and rs masked GEMMs, FP32 gather) equal the exact result."""
    B, H, Co = 32, 256, 32
    Hp = (H - 2) // 2
    g = _gen(10 + ch)
    img = _ints((B, H, H, ch), -8, 8, g)
    ws = _weights(ch, g, True)
    bias = _bias(Co, g, True)
    gp = _ints((B * Hp * Hp, Co), -2, 2, g)
    xr = img.permute(0, 3, 1, 2).double()
    ref = R.fwd_pool(xr, ws[0], bias)
    assert R.max_abs_sum_ok(ref.S)
    out, am, out_eval, grads = _run_layer1(ch, img, ws, bias, gp, B, H)
    assert torch.equal(out, R.nhwc(R.bf16_rn(ref.out)))
    assert torch.equal(am, R.nhwc(ref.code))
    assert torch.equal(out_eval, out)
    gpr = R.nchw(gp, B, Hp, Hp)
    assert R.max_abs_sum_ok(R.wgrad0_abs(xr, gpr, ref.code))
    exact = R.wgrad0(xr, gpr, ref.code)
    for kern, dW in grads.items():
        rows = _gradient_rows(kern, ch)
        assert torch.equal(dW.double().view(-1, Co)[rows], exact[rows]), kern
    dy = R.conv_grid_grad(gpr, ref.code, H, H)
    assert not torch.equal(R.wgrad(xr, R.omit_unit(dy, R.wgrad_last_unit(B, H, H)), 16), exact)


@pytest.mark.parametrize("l,B", [(1, 32), (2, 32), (3, 32), (4, 32), (5, 32), (1, 3)])
def test_layer_is_exact_on_integer_data(l, B):
    """Layers 2-6: forward (train and eval), unpool_relu, dgrad and weight gradient equal the exact results, the zero
    border and the dropped floor-pool edge of the odd 127 map included. B = 3 at H = 127 ends on a partial tile."""
    H, CK, Co = H_OF[l], CK_OF[l], R.MEDCNN_CO[l]
    Ci, Hp, P = CK, (H - 2) // 2, B * H * H
    g = _gen(100 + l + B)
    ws = _weights(3, g, True)
    lay = R.weight_layouts(ops, ws)
    w = ws[l].double()
    X = _ints((P, CK), -8, 8, g)
    bias = _bias(Co, g, True)
    xr = R.nchw(X, B, H, H)
    ref = R.fwd_pool(xr, w, bias)
    assert R.max_abs_sum_ok(ref.S)
    (out, am), names = kernels_run(lambda: _fwd(X, lay.Wf[l], bias, B, H, CK, Co))
    if B == 32:
        assert ran(names, FWD[l]), sorted(names)
    assert torch.equal(out, R.nhwc(R.bf16_rn(ref.out)))
    assert torch.equal(am, R.nhwc(ref.code))
    out_eval, _ = _fwd(X, lay.Wf[l], bias, B, H, CK, Co, train=False)
    assert torch.equal(out_eval, out)
    # un-pool: the whole H x W grid, zeros included
    gp = _ints((B * Hp * Hp, Co), -2, 2, g)
    dY = _nan(P, Co)
    ops.unpool_relu(gp, am, out, dY, B, H, H, Co)
    dy = R.unpool(R.nchw(gp, B, Hp, Hp), R.nchw(out, B, Hp, Hp), ref.code, H, H)
    assert torch.equal(dY, R.nhwc(dy).to(torch.bfloat16))
    # dgrad into layer l - 1
    assert R.max_abs_sum_ok(R.dgrad_abs(dy, w))

    def dgrad():
        dX = _nan(P, Ci)
        ops.conv_dgrad(dY, lay.Wd[l], dX, B, H, H, Co, Ci)
        return dX
    dX, names = kernels_run(dgrad)
    if B == 32:
        assert ran(names, DGRAD[l]), sorted(names)
    assert torch.equal(dX, R.nhwc(R.bf16_rn(R.dgrad(dy, w))))
    # weight gradient
    assert R.max_abs_sum_ok(R.wgrad_abs(xr, dy, CK))
    dW, names = kernels_run(lambda: _wgrad(X, dY, B, H, CK, Co))
    if B == 32:
        assert ran(names, WGRAD[l]), sorted(names)
    exact = R.wgrad(xr, dy, CK)
    assert torch.equal(dW.double().view(-1, Co), exact)
    # the data reach the last row unit: omitting it changes the exact result
    assert not torch.equal(R.wgrad(xr, R.omit_unit(dy, R.wgrad_last_unit(B, H, H)), CK), exact)


# ---------------------------------------------------------------------------------------------- (b, c) real data
def _check_fwd(out, am, ref, n, x, w, bias, B, Hp, tag):
    got = R.nchw(out, B, Hp, Hp)
    assert R.within(got, ref.out, R.fwd_bound(ref.out, ref.S, n)), tag
    ok, checked = R.codes_agree(R.nchw(am, B, Hp, Hp), ref, n)
    assert ok and checked > 0.5 * ref.code.numel(), (tag, checked)
    # teeth: one input channel's tap zeroed, the last conv column of each row ignored by the pool
    for bad in (R.fwd_pool(x, R.drop_tap(w, w.shape[1] - 1, 1, 1), bias), R.fwd_pool(x, w, bias, drop_last_col=True)):
        assert not R.within(got, bad.out, R.fwd_bound(bad.out, bad.S, n)), tag


def _check_wgrad(dW, ref, S, CK, Co, tag, rows=None):
    """Weight gradient (dW32 layout) within the sanity bound 2^-14 S per element, S = sum of |terms|: chains of up to
    ~500k terms make the worst-case bound useless, and the integer tests are what give wgrad its teeth. Measured on
    an H100 80GB HBM3 at a 400 W power limit: the largest err / S was 2.9e-8 for the layer-1 kernels, 1.1e-7 for
    layers 2-6 and 9.7e-8 in the engine step, against 6.1e-5 allowed. `rows`: the dW32 rows the kernel defines."""
    got = dW.double().view(-1, Co)
    bad = ref.clone()
    bad[4 * CK] = 0                                  # the centre tap of input channel 0 not written
    if rows is not None:
        got, ref, S, bad = got[rows], ref[rows], S[rows], bad[rows]
    err = ((got - ref).abs() / S.clamp_min(1e-30))
    ratio = float(err[S > 0].max())
    print(f"{tag}: max |wgrad err| / S = {ratio:.3e}")
    assert R.within(got, ref, 2.0 ** -14 * S), (tag, ratio)
    assert not R.within(got, bad, 2.0 ** -14 * S), tag


@pytest.mark.parametrize("ch", [3, 1])
def test_layer1_real_data_within_derived_bounds(ch):
    B, H, Co = 32, 256, 32
    Hp = (H - 2) // 2
    g = _gen(20 + ch)
    img = R.bf16_rn(torch.rand((B, H, H, ch), generator=g, device="cuda"))
    ws = _weights(ch, g, False)
    bias = _bias(Co, g, False)
    gp = _randn((B * Hp * Hp, Co), g)
    xr = img.permute(0, 3, 1, 2).double()
    ref = R.fwd_pool(xr, ws[0], bias)
    out, am, out_eval, grads = _run_layer1(ch, img, ws, bias, gp, B, H)
    _check_fwd(out, am, ref, 9 * ch, xr, ws[0].double(), bias, B, Hp, f"layer 1 ({ch} ch)")
    assert torch.equal(out_eval, out)
    gpr = R.nchw(gp, B, Hp, Hp)
    code = R.nchw(am, B, Hp, Hp)              # the kernel's own decisions: ties cannot differ
    rW, sW = R.wgrad0(xr, gpr, code), R.wgrad0_abs(xr, gpr, code)
    for kern, dW in grads.items():
        _check_wgrad(dW, rW, sW, 16, Co, f"layer 1 {kern}", _gradient_rows(kern, ch))


@pytest.mark.parametrize("l", [1, 2, 3, 4, 5])
def test_layer_real_data_within_derived_bounds(l):
    B, H, CK, Co = 32, H_OF[l], CK_OF[l], R.MEDCNN_CO[l]
    Ci, Hp, P = CK, (H - 2) // 2, B * H * H
    g = _gen(200 + l)
    ws = _weights(3, g, False)
    lay = R.weight_layouts(ops, ws)
    w = ws[l].double()
    X = _randn((P, CK), g)
    bias = _bias(Co, g, False)
    xr = R.nchw(X, B, H, H)
    ref = R.fwd_pool(xr, w, bias)
    out, am = _fwd(X, lay.Wf[l], bias, B, H, CK, Co)
    _check_fwd(out, am, ref, 9 * CK, xr, w, bias, B, Hp, f"layer {l + 1}")
    gp = _randn((B * Hp * Hp, Co), g)
    dY = _nan(P, Co)
    ops.unpool_relu(gp, am, out, dY, B, H, H, Co)
    dy = R.unpool(R.nchw(gp, B, Hp, Hp), R.nchw(out, B, Hp, Hp), R.nchw(am, B, Hp, Hp), H, H)
    assert torch.equal(dY, R.nhwc(dy).to(torch.bfloat16))
    dX = _nan(P, Ci)
    ops.conv_dgrad(dY, lay.Wd[l], dX, B, H, H, Co, Ci)
    nd = 9 * Co
    rd, sd = R.dgrad(dy, w), R.dgrad_abs(dy, w)
    got = R.nchw(dX, B, H, H)
    assert R.within(got, rd, R.fwd_bound(rd, sd, nd))
    w_bad = R.drop_tap(w, None, 2, 0)
    assert not R.within(got, R.dgrad(dy, w_bad), R.fwd_bound(R.dgrad(dy, w_bad), R.dgrad_abs(dy, w_bad), nd))
    dW = _wgrad(X, dY, B, H, CK, Co)
    _check_wgrad(dW, R.wgrad(xr, dy, CK), R.wgrad_abs(xr, dy, CK), CK, Co, f"layer {l + 1} wgrad")


# ---------------------------------------------------------------------------------------------- (e) one engine step
@pytest.mark.parametrize("ch", [3, 1])
def test_engine_step_stage_by_stage(ch, monkeypatch):
    """One default training step (B = 32, 256 x 256) and the evaluation forward on the same batch, every stage
    checked against float64 computed from the engine's own bf16 input to that stage (teacher-forced)."""
    from hefl_b200.config import FLConfig
    from hefl_b200.models import ParamPack, create_model
    from hefl_b200.ops.conv_engine import MedCNNEngine

    for k in list(os.environ):
        if k.startswith("HEFL_"):
            monkeypatch.delenv(k)
    torch.manual_seed(3)
    cfg = FLConfig(in_channels=ch)
    B, S = cfg.batch_size, cfg.image_size
    assert (B, S) == (32, 256)
    dev = torch.device("cuda")
    model = create_model("medcnn", in_channels=ch).to(dev)
    pack = ParamPack(model)
    eng = MedCNNEngine(model, pack, cfg, dev)
    assert eng.compact0 == (ch == 3) and eng.spack0 and eng.gather_wgrad0
    g = _gen(30 + ch)
    x = torch.randint(0, 256, (B, S, S, ch), dtype=torch.uint8, device="cuda", generator=g)
    y = torch.randint(0, 2, (B,), device="cuda", generator=g)
    out = torch.zeros(2, device="cuda")

    def step():
        pack.grad.zero_()
        eng.train_step(x, y, out, augment=False, opt=None)
    _, names = kernels_run(step)
    expect = ["pair_fwd_compact_kernel" if ch == 3 else "pair_fwd_rs_kernel",
              "wgrad0_mma_compact_kernel" if ch == 3 else "wgrad0_mma_rs_kernel", "unpool_relu_kernel",
              "head_cluster_kernel"] + sorted(set(FWD.values()) | set(DGRAD.values()) | set(WGRAD.values()))
    for k in expect:
        assert ran(names, k), (k, sorted(names))
    n = eng.n
    acts = [t.clone() for t in eng.X[1:]]
    img = eng.x0(0)[:, :3] if ch == 3 else eng.x0(0)[: B * S * S, :1]
    xin = [R.nchw(img, B, S, S)] + [R.nchw(acts[l - 1], B, eng.H[l], eng.H[l]) for l in range(1, n)]
    convs = list(model.convs)
    ws = [c.weight.detach().to(torch.bfloat16).double() for c in convs]
    refs = []
    for l in range(n):
        Hp = eng.H[l + 1]
        ref = R.fwd_pool(xin[l], ws[l], convs[l].bias.detach())
        _check_fwd_engine(acts[l], eng.amax[l], ref, 9 * eng.Ci[l], B, Hp, l)
        refs.append(ref)
    # dense head: fp64 autograd on the engine's X[6]
    feat = acts[-1].view(B, -1).double().requires_grad_(True)
    fcs = copy.deepcopy(model.fcs).double()
    fcs.zero_grad(set_to_none=True)
    h = feat
    for fc in fcs[:-1]:
        h = F.relu(fc(h))
    loss = F.cross_entropy(fcs[-1](h), y)
    loss.backward()
    loss = float(loss.detach())
    assert abs(float(out[0]) - loss) < 1e-4 * max(1.0, loss)
    d_ref = feat.grad
    d_got = eng.dfeat.view(B, -1).double()
    assert R.within(d_got, d_ref, R.BF16_EPS * d_ref.abs() + 2.0 ** -16 * d_ref.abs().max())
    for p64, p in zip(fcs.parameters(), model.fcs.parameters()):
        assert (p.grad.double() - p64.grad).abs().max() <= 1e-4 * p64.grad.abs().max() + 1e-7
    # backward, layer by layer from the engine's own pooled gradients
    ratios = {}
    for l in range(n - 1, -1, -1):
        H, Hp = eng.H[l], eng.H[l + 1]
        gl = eng.dfeat if l == n - 1 else eng.gX[l + 1]
        gpr = R.nchw(gl.view(-1, eng.Co[l]), B, Hp, Hp)
        code = R.nchw(eng.amax[l], B, Hp, Hp)
        wgot = convs[l].weight.grad.double()
        bgot = convs[l].bias.grad.double()
        if l == 0:
            rW, sW = R.wgrad0(xin[0], gpr, code), R.wgrad0_abs(xin[0], gpr, code)
        else:
            dy = R.unpool(gpr, R.nchw(acts[l], B, Hp, Hp), code, H, H)
            assert torch.equal(eng.dY[l], R.nhwc(dy).to(torch.bfloat16)), l
            rd, sd = R.dgrad(dy, ws[l]), R.dgrad_abs(dy, ws[l])
            assert R.within(R.nchw(eng.gX[l], B, H, H), rd, R.fwd_bound(rd, sd, 9 * eng.Co[l])), l
            rW, sW = R.wgrad(xin[l], dy, eng.CK[l]), R.wgrad_abs(xin[l], dy, eng.CK[l])
        rw, rb = R.wgrad_to_oihw(rW, eng.Ci[l], eng.CK[l], eng.Co[l])
        sw, sb = R.wgrad_to_oihw(sW, eng.Ci[l], eng.CK[l], eng.Co[l])
        got, ref, S_ = torch.cat([wgot.reshape(-1), bgot]), torch.cat([rw.reshape(-1), rb]), torch.cat([sw.reshape(-1), sb])
        ratios[l + 1] = float(((got - ref).abs() / S_.clamp_min(1e-30))[S_ > 0].max())
        assert R.within(got, ref, 2.0 ** -14 * S_), (l, ratios)
    print(f"engine step ({ch} ch): max |wgrad err| / S per layer {ratios}")
    # evaluation forward on the same batch: the same activations, bit for bit
    eng.eval_step(x, y, out)
    torch.cuda.synchronize()
    for l in range(n):
        assert torch.equal(eng.X[l + 1], acts[l]), l


def _check_fwd_engine(out, am, ref, n, B, Hp, l):
    got = R.nchw(out, B, Hp, Hp)
    assert R.within(got, ref.out, R.fwd_bound(ref.out, ref.S, n)), l
    ok, _ = R.codes_agree(R.nchw(am, B, Hp, Hp), ref, n)
    assert ok, l

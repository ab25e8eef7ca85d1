"""The ResNet kernels at the shapes of the ResNet-18 / ResNet-50 training step (batch 32, 224 x 224), against the
float64 references of tests/resnet_ref.py.

The shape table is recorded from the models themselves: one train-mode forward of ResNet-18, ResNet-50 and ResNet-50
with block-scaled e4m3 (MX) 1x1 convolutions logs every call that reaches the hand-written convolutions, BatchNorm and
average pool. Every test below iterates over that table.

Integer tests: small-integer operands keep every output's sum of |terms| below 2^24 (bf16 operands, fp32
accumulation) or 2^12 (e4m3 operands, whose tensor-core accumulation may keep fewer bits), asserted on the data, so the
kernels must equal the exactly rounded float64 result bit for bit (bf16 results are compared as int16 bit patterns;
only where the reference is zero may the kernel's zero carry either sign). Real-data tests hold randn operands, rows
scaled by powers of two, to the per-element bounds of resnet_ref (each shown to reject a defect in
test_resnet_ref_cpu.py).
Outputs written by the bindings live inside NaN-filled buffers, and the margins must come back untouched. The host
formulas of gemm_tcgen05.cu tell which regime (tiles per CTA, partial tiles, pixel splits) each case is in, with the
device's SM count; the profiler confirms which kernel instantiations ran, tracing again (a bounded number of times)
when a trace does not show them, and every result check is made on an untraced run or outside the trace."""
import math
import time

import pytest
import torch

import resnet_ref as R
from kernel_trace import kernels_run, ran

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from hefl_b200 import _ext
    ops = _ext.ops()
    SMS = torch.cuda.get_device_properties(0).multi_processor_count

B, IMG = 32, 224
NAN = float("nan")
MARGIN = 4096                      # poisoned elements before and after every output slice
RECORDED = {}                      # filled by the table fixture: kind -> set of keys
COVERAGE = {"kmajor": [], "wgrad": [], "names": set(), "fp8_err": []}


# ---------------------------------------------------------------------------------------------- helpers
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _ints(shape, lo, hi, g, dtype=torch.bfloat16):
    return torch.randint(lo, hi + 1, shape, generator=g, device="cuda").to(dtype)


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def _poisoned(n, dtype=torch.bfloat16):
    """(buffer, its middle n elements): an output slice with NaN margins on both sides."""
    buf = torch.full((n + 2 * MARGIN,), NAN, dtype=dtype, device="cuda")
    return buf, buf[MARGIN: MARGIN + n]


def _margins_untouched(buf):
    return bool(torch.isnan(buf[:MARGIN].float()).all()) and bool(torch.isnan(buf[-MARGIN:].float()).all())


def _bits_equal(got, want):
    """bf16 tensors equal bit for bit; only where `want` is zero may `got` be a zero of either sign (a float64
    reference has no signed zero)."""
    same = got.view(torch.int16) == want.view(torch.int16)
    zeros = (want.float() == 0) & (got.float() == 0)
    return bool((same | zeros).all())


def _confirm(fn, kernels, tries=4):
    """(last result of fn, the subset of `kernels` seen): fn runs under the profiler until every kernel has appeared in
    a trace, at most `tries` times. A trace can come back empty or without a kernel although it ran; in a long test
    process the earliest kernels of a trace are the ones it loses. So one trace is not final, and each traced body runs
    fn twice, so that every kernel of fn also launches after others. fn must be repeatable; the checks of its results
    are made outside the profiler."""
    seen, out = set(), None
    for _ in range(tries):
        out, names = kernels_run(lambda: (fn(), fn())[1])
        COVERAGE["names"] |= names
        seen |= {k for k in kernels if ran(names, k)}
        if seen == set(kernels):
            break
    return out, seen


def _check(ok_msg, what):
    ok, msg = ok_msg
    assert ok, f"{what}: {msg}"


# ---------------------------------------------------------------------------------------------- host formulas
def kmajor_regime(a_rows, N):
    """gemm_taps / launch_kmajor: (BN, tiles, tiles per CTA, partial last M tile)."""
    bn = 128 if N % 128 == 0 else 64
    tiles = (a_rows + 127) // 128 * (N // bn)
    grid = min(tiles, SMS)
    return bn, tiles, (tiles + grid - 1) // grid, a_rows % 128 != 0


def wgrad_regime(rows, Co, Ci, taps):
    """wgrad_taps: (CT, ksplit, chunks per split, last split empty)."""
    ct = 128 if Ci % 128 == 0 else 64
    base = (Co + 127) // 128 * (Ci // ct) * (9 if taps == 9 else 1)
    kchunks = (rows + 63) // 64
    ks = min(max((SMS + base - 1) // base, 1), kchunks)
    per = (kchunks + ks - 1) // ks
    return ct, ks, per, (ks - 1) * per >= kchunks


# ---------------------------------------------------------------------------------------------- the shape table
@pytest.fixture(scope="module", autouse=True)
def _budget(request):
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    tr = request.config.pluginmanager.get_plugin("terminalreporter")
    line = (f"test_gpu_resnet_step_shapes: wall {time.time() - t0:.1f} s, peak allocated "
            f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB on {torch.cuda.get_device_name(0)} ({SMS} SMs)")
    if COVERAGE["fp8_err"]:
        line += f"; largest e4m3 real-data error / sum|terms|: {max(COVERAGE['fp8_err']):.3e}"
    print(line)
    if tr is not None:
        tr.write_line(line)


@pytest.fixture(scope="module")
def table():
    """Every call that reaches _Conv1x1TC, _Conv3x3TC, _BNActFn and _AvgPoolFn in one train-mode forward at B = 32,
    224 x 224 (channels_last, bf16 autocast, no grad): ("1x1", Cin, Cout, H, W, stride, mx) with H, W the map before
    the stride, ("3x3", Cin, Cout, H, W), ("bn", C, P, residual, relu), ("pool", B, HW, C)."""
    from hefl_b200.models import create_model
    from hefl_b200.ops import fp8, resnet_ops, tc_conv

    rec = {"1x1": set(), "3x3": set(), "bn": set(), "pool": set()}
    per_model = {}
    pending = []
    orig = {"c1": tc_conv._Conv1x1TC.apply, "c3": tc_conv._Conv3x3TC.apply, "bn": resnet_ops._BNActFn.apply,
            "pool": resnet_ops._AvgPoolFn.apply, "conv1x1": tc_conv.conv1x1}

    def conv1x1(x, w, stride=1, fp8_state=None):
        pending.append((x.shape[2], x.shape[3], stride))
        return orig["conv1x1"](x, w, stride, fp8_state)

    def c1(x, w, fp8_state):
        H, W, stride = pending.pop()
        Cout, Cin = w.shape[:2]
        mx = fp8_state == "mx" and Cin % 128 == 0 and Cout % 128 == 0
        cur.add(("1x1", Cin, Cout, H, W, stride, mx))
        return orig["c1"](x, w, fp8_state)

    def c3(x, w):
        cur.add(("3x3", x.shape[1], w.shape[0], x.shape[2], x.shape[3]))
        return orig["c3"](x, w)

    def bn(x, res, *a):
        cur.add(("bn", x.shape[1], x.numel() // x.shape[1], res is not None, bool(a[-1])))
        return orig["bn"](x, res, *a)

    def pool(x):
        cur.add(("pool", x.shape[0], x.shape[2] * x.shape[3], x.shape[1]))
        return orig["pool"](x)

    mp = pytest.MonkeyPatch()
    mp.setattr(tc_conv, "conv1x1", conv1x1)
    mp.setattr(tc_conv._Conv1x1TC, "apply", c1)
    mp.setattr(tc_conv._Conv3x3TC, "apply", c3)
    mp.setattr(resnet_ops._BNActFn, "apply", bn)
    mp.setattr(resnet_ops._AvgPoolFn, "apply", pool)
    try:
        x = _cl(torch.randn(B, 3, IMG, IMG, device="cuda", generator=_gen(0)))
        for name, use_fp8 in (("resnet18", False), ("resnet50", False), ("resnet50", True)):
            torch.manual_seed(0)
            m = create_model(name, 3, 1000, IMG).cuda().to(memory_format=torch.channels_last).train()
            tc_conv.set_model_tc(m, True)
            fp8.set_model_fp8(m, use_fp8)
            cur = set()
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                m(x)
            torch.cuda.synchronize()
            per_model[name + ("-mx" if use_fp8 else "")] = cur
            for k in cur:
                rec[k[0]].add(k)
            del m
    finally:
        mp.undo()
    assert not pending
    for name, keys in per_model.items():
        counts = {k: sum(1 for e in keys if e[0] == k) for k in rec}
        counts["mx"] = sum(1 for e in keys if e[0] == "1x1" and e[6])
        print(f"{name}: {counts}")
    RECORDED.update(rec)
    torch.cuda.empty_cache()
    return rec


def test_recorded_table_has_the_step_shapes(table):
    """The hand-written paths see what the step runs: the 56..7 pyramid of both models, the stem BatchNorm at
    P = 32 * 112^2, C = 2048 at P = 1568, and the pool at 7 x 7."""
    for k in sorted(table["3x3"]):
        print(k)
    assert {k[1:4] for k in table["3x3"]} == {(64, 64, 56), (128, 128, 28), (256, 256, 14), (512, 512, 7)}
    assert ("bn", 64, B * 112 * 112, False, True) in table["bn"]
    assert any(k[1] == 2048 and k[2] == B * 49 for k in table["bn"])
    assert table["pool"] == {("pool", B, 49, 512), ("pool", B, 49, 2048)}
    mx = {k for k in table["1x1"] if k[6]}
    assert mx and any(k[3] // k[5] == 7 for k in mx)                      # M = 1568 on the MX path
    assert any(not k[6] and k[3] // k[5] == 7 for k in table["1x1"])    # and on the bf16 path


# ---------------------------------------------------------------------------------------------- GEMM cases
def _conv_case(key, seed, integer, trace=()):
    """Runs one table convolution through tc_conv (forward + autograd backward) and the bindings directly into
    poisoned buffers; returns (x, w, gy, results of autograd, kernel names)."""
    from hefl_b200.ops import tc_conv

    kind = key[0]
    Cin, Cout, H, W = key[1:5]
    stride = key[5] if kind == "1x1" else 1
    mx = kind == "1x1" and key[6]
    Ho, Wo = (H + stride - 1) // stride, (W + stride - 1) // stride
    g = _gen(seed)
    k = 1 if kind == "1x1" else 3
    if integer:
        x = _cl(_ints((B, Cin, H, W), -2, 2, g))
        w = _ints((Cout, Cin, k, k), -1 if mx else -2, 1 if mx else 2, g, torch.float32)
        gy = _cl(_ints((B, Cout, Ho, Wo), -2, 2, g))
    else:
        rows = torch.exp2((torch.arange(B * H * W, device="cuda") % 9).float() - 4).view(B, 1, H, W)
        x = _cl((torch.randn(B, Cin, H, W, device="cuda", generator=g) * rows).to(torch.bfloat16))
        w = (torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / math.sqrt(Cin * k * k)).to(torch.bfloat16).float()
        gy = _cl(torch.randn(B, Cout, Ho, Wo, device="cuda", generator=g).to(torch.bfloat16))

    def run():
        xt, wt = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
        y = tc_conv.conv1x1(xt, wt, stride, "mx" if mx else None) if kind == "1x1" else tc_conv.conv3x3(xt, wt)
        y.backward(gy)
        return y.detach(), xt.grad, wt.grad

    if trace:
        (y, dx, dw), names = _confirm(run, trace, tries=2)
    else:
        (y, dx, dw), names = run(), set()
    return x, w, gy, (y, dx, dw), names


def _direct_1x1(key, x, w, gy, y, dx, dw):
    """The bindings the 1x1 step calls, into NaN-poisoned outputs: they must equal the autograd results."""
    _, Cin, Cout, H, W, stride, mx = key
    xs = R.subsample(R.nhwc(x), B, H, W, stride).contiguous()
    M = xs.shape[0]
    wb, wT = ops.conv_weight_prep(w.contiguous())
    g2 = R.nhwc(gy)
    buf, out = _poisoned(M * Cout)
    if mx:
        (xq, xsf), (wq, wsf) = ops.mxfp8_quantize(xs), ops.mxfp8_quantize(wb)
        ops.gemm_mxfp8(xq, wq, xsf, wsf, out.view(M, Cout))
    else:
        ops.gemm_taps(xs, wb, out.view(M, Cout), Cout, Cin, [], 0, 0, 0, 0, None, None)
    assert _margins_untouched(buf) and _bits_equal(out.view(M, Cout), R.nhwc(y)), key
    buf, out = _poisoned(M * Cin)
    if mx:
        (gq, gsf), (tq, tsf) = ops.mxfp8_quantize(g2), ops.mxfp8_quantize(wT)
        ops.gemm_mxfp8(gq, tq, gsf, tsf, out.view(M, Cin))
    else:
        ops.gemm_taps(g2, wT, out.view(M, Cin), Cin, Cout, [], 0, 0, 0, 0, None, None)
    assert _margins_untouched(buf) and _bits_equal(out.view(M, Cin), R.subsample(R.nhwc(dx), B, H, W, stride)), key
    buf, out = _poisoned(Cout * Cin, torch.float32)
    ops.wgrad_taps(g2, xs, out.view(1, Cout, Cin), 1, 0)           # the buffer starts as NaN: the binding zeroes it
    assert _margins_untouched(buf) and torch.equal(out.view(Cout, Cin), dw.view(Cout, Cin)), key


def _direct_3x3(key, x, w, gy, y, dx, dw):
    _, Cin, Cout, H, W = key
    xp = ops.pad_nhwc(x)
    assert torch.equal(xp.view(-1, Cin), R.pad_grid(R.nhwc(x), B, H, W))
    wt, wd = ops.conv_weight_prep(w.contiguous())
    gp = ops.pad_nhwc(gy)
    sh = R.shifts(W + 2)
    P = B * H * W
    buf, out = _poisoned(P * Cout)
    ops.gemm_taps(xp.view(-1, Cin), wt, out.view(P, Cout), Cout, Cin, sh, 1, B, H, W, None, None)
    assert _margins_untouched(buf) and _bits_equal(out.view(P, Cout), R.nhwc(y)), key
    buf, out = _poisoned(P * Cin)
    ops.gemm_taps(gp.view(-1, Cout), wd, out.view(P, Cin), Cin, Cout, sh, 1, B, H, W, None, None)
    assert _margins_untouched(buf) and _bits_equal(out.view(P, Cin), R.nhwc(dx)), key
    buf, out = _poisoned(9 * Cout * Cin, torch.float32)
    ops.wgrad_taps(gp.view(-1, Cout), xp.view(-1, Cin), out.view(9, Cout, Cin), 9, W + 2)
    assert _margins_untouched(buf) and torch.equal(out.view(9, Cout, Cin).permute(1, 2, 0), dw.view(Cout, Cin, 9)), key


def _refs(key, x, w, gy):
    """Generators of (name, float64 reference, sum of |terms|, accumulation length) for forward, dgrad, wgrad;
    one float64 layer alive at a time."""
    kind, Cin, Cout, H, W = key[:5]
    x2, dy2 = R.nhwc(x), R.nhwc(gy)
    if kind == "1x1":
        stride = key[5]
        xs = R.subsample(x2, B, H, W, stride)
        w2 = w.view(Cout, Cin)
        yield "fwd", R.conv1x1_fwd(xs, w2), R.conv1x1_fwd_abs(xs, w2), Cin
        yield "dgrad", R.conv1x1_dgrad(dy2, w2), R.conv1x1_dgrad_abs(dy2, w2), Cout
        yield "wgrad", R.conv1x1_wgrad(dy2, xs), R.conv1x1_wgrad_abs(dy2, xs), xs.shape[0]
    else:
        yield "fwd", R.conv3x3_fwd(x2, w, B, H, W), R.conv3x3_fwd_abs(x2, w, B, H, W), 9 * Cin
        yield "dgrad", R.conv3x3_dgrad(dy2, w, B, H, W), R.conv3x3_dgrad_abs(dy2, w, B, H, W), 9 * Cout
        yield "wgrad", R.conv3x3_wgrad(dy2, x2, B, H, W), R.conv3x3_wgrad_abs(dy2, x2, B, H, W), B * (H + 2) * (W + 2)


def _got(key, name, y, dx, dw):
    """The kernel result matching a reference of _refs (the strided dgrad at the sampled pixels)."""
    kind, Cin, Cout, H, W = key[:5]
    if name == "fwd":
        return R.nhwc(y)
    if name == "dgrad":
        d = R.nhwc(dx)
        return R.subsample(d, B, H, W, key[5]) if kind == "1x1" else d
    return dw.view(Cout, Cin) if kind == "1x1" else dw


def _expected_kernels(key):
    kind, Cin, Cout, H, W = key[:5]
    mx = kind == "1x1" and key[6]
    ct, *_ = wgrad_regime(1, Cout, Cin, 1)
    names = ["conv_weight_prep_kernel", f"wgrad_mn_kernel<{ct}>"]
    if mx:
        names += ["mx_gemm_kernel", "mxfp8_quantize_kernel"]
    else:
        names += [f"kmajor_gemm_kernel<{kmajor_regime(128, Cout)[0]}, false>",
                  f"kmajor_gemm_kernel<{kmajor_regime(128, Cin)[0]}, false>"]
    if kind == "3x3":
        names += ["pad_nhwc_kernel", "conv_wgrad_unpack_kernel"]
    return names


def _record_regimes(key):
    kind, Cin, Cout, H, W = key[:5]
    if kind == "1x1":
        stride = key[5]
        M = B * ((H + stride - 1) // stride) * ((W + stride - 1) // stride)
        rows, padded, taps = M, False, 1
    else:
        rows, padded, taps = B * (H + 2) * (W + 2), True, 9
    if not (kind == "1x1" and key[6]):
        for N in (Cout, Cin):
            COVERAGE["kmajor"].append((key, N, padded) + kmajor_regime(rows, N))
    COVERAGE["wgrad"].append((key, Cout) + wgrad_regime(rows, Cout, Cin, taps))


def _gemm_keys(table):
    return sorted(table["1x1"] | {k + (1, False) for k in table["3x3"]}, key=str)


def test_every_table_gemm_is_exact_on_integer_data(table):
    """Forward, dgrad (autograd through tc_conv, stride-2 scatter included) and the fp32 weight gradient of every
    table convolution equal the exact result on integers, bf16 and MX alike; the bindings write nothing outside
    their outputs; the profiler confirms every instantiation the host formulas select (cases run under it, up to
    twice each, until all of their instantiations have been seen; the results are checked the same way either way)."""
    expected, confirmed = set(), set()
    for i, key in enumerate(_gemm_keys(table)):
        mx = key[0] == "1x1" and key[6]
        k3 = key[:5] if key[0] == "3x3" else key
        want = set(_expected_kernels(k3))
        expected |= want
        x, w, gy, (y, dx, dw), seen = _conv_case(k3, 100 + i, True, trace=sorted(want - confirmed))
        confirmed |= seen
        _record_regimes(k3)
        for name, ref, S, n in _refs(k3, x, w, gy):
            limit = R.FP8_INT_LIMIT if mx and name != "wgrad" else 2 ** 24
            R.assert_exact_premise(S, limit)
            got = _got(k3, name, y, dx, dw)
            if name == "wgrad":
                assert torch.equal(got.double(), ref), (key, name)
            else:
                assert _bits_equal(got, R.bf16_rn(ref)), (key, name)
            del ref, S
        if key[0] == "1x1" and key[5] > 1:      # the unsampled pixels get no gradient
            d = R.nhwc(dx).view(B, key[3], key[4], -1)
            assert not bool((d[:, 1::2] != 0).any()) and not bool((d[:, :, 1::2] != 0).any()), key
        (_direct_1x1 if key[0] == "1x1" else _direct_3x3)(k3, x, w, gy, y, dx, dw)
        del x, w, gy, y, dx, dw
    torch.cuda.empty_cache()
    print("confirmed by the profiler:", sorted(confirmed))
    assert expected == confirmed, sorted(expected - confirmed)


def test_every_table_gemm_is_within_bounds_on_real_data(table):
    """randn operands, pixel rows scaled by 2^-4 ... 2^4 so that rows of very different magnitude share a tile:
    bf16 results within the accumulation bound, MX results within the e4m3 bound against the product of the
    operands as the kernels quantised them."""
    for i, key in enumerate(_gemm_keys(table)):
        mx = key[0] == "1x1" and key[6]
        k3 = key[:5] if key[0] == "3x3" else key
        x, w, gy, (y, dx, dw), _ = _conv_case(k3, 200 + i, False)
        if mx:
            _, Cin, Cout, H, W, stride, _ = key
            xs = R.subsample(R.nhwc(x), B, H, W, stride).contiguous()
            wb, wT = ops.conv_weight_prep(w.contiguous())
            for name, a, bm, got in (("fwd", xs, wb, R.nhwc(y)),
                                     ("dgrad", R.nhwc(gy), wT, R.subsample(R.nhwc(dx), B, H, W, stride))):
                qa, sa, _ = R.mx_quantize(a)
                qb, sb, _ = R.mx_quantize(bm)
                ka, kb = ops.mxfp8_quantize(a), ops.mxfp8_quantize(bm)
                assert torch.equal(ka[0], qa) and torch.equal(ka[1], sa) and torch.equal(kb[0], qb) and torch.equal(kb[1], sb)
                da, db = R.mx_dequantize(qa, sa, *a.shape), R.mx_dequantize(qb, sb, *bm.shape)
                K = a.shape[1]
                ref, S = da @ db.t(), da.abs() @ db.abs().t()
                _check(R.within(got, ref, R.gemm_bound(ref, S, K, R.FP8_STEP_EPS, K // 32)), f"{key} {name}")
                COVERAGE["fp8_err"].append(float(((got.double() - ref).abs() / S.clamp_min(1e-30)).max()))
                del da, db, ref, S
            refs = (r for r in _refs(k3, x, w, gy) if r[0] == "wgrad")
        else:
            refs = _refs(k3, x, w, gy)
        for name, ref, S, n in refs:
            got = _got(k3, name, y, dx, dw)
            if name == "wgrad":
                ks = wgrad_regime(n, key[2], key[1], 1 if key[0] == "1x1" else 9)[1]
                bound = R.acc_bound(S, n + ks)
            else:
                bound = R.gemm_bound(ref, S, n)
            _check(R.within(got, ref, bound), f"{key} {name}")
            del ref, S
        del x, w, gy, y, dx, dw
    torch.cuda.empty_cache()


def test_the_table_reaches_every_gemm_regime(table):
    """Coverage, from the host formulas at this device's SM count: more than one tile per CTA, padded mode (whose
    first tiles read negative tap rows, zero-filled by TMA), partial last M tiles dense and padded, BN = 64 and 128,
    CT = 64 and 128, Co = 64 (the zero-filled second dY atom), ksplit == 1, ksplit > 1 and an empty last split (a
    synthetic weight gradient when no table shape has one)."""
    if not COVERAGE["kmajor"]:
        for key in _gemm_keys(table):
            _record_regimes(key[:5] if key[0] == "3x3" else key)
    km, wg = COVERAGE["kmajor"], COVERAGE["wgrad"]
    for key, N, padded, bn, tiles, per_cta, partial in km:
        print(f"kmajor {key} N={N}: BN={bn} tiles={tiles} tiles/CTA={per_cta} partial={partial} padded={padded}")
    for key, Co, ct, ks, per, empty in wg:
        print(f"wgrad {key}: CT={ct} ksplit={ks} chunks/split={per} empty last split={empty}")
    assert any(r[5] > 1 for r in km) and any(r[2] for r in km)
    assert any(r[6] and not r[2] for r in km) and any(r[6] and r[2] for r in km)
    assert {r[3] for r in km} == {64, 128}
    assert {r[2] for r in wg} == {64, 128} and any(r[1] == 64 for r in wg)
    assert any(r[3] == 1 for r in wg) and any(r[3] > 1 for r in wg)
    if not any(r[5] for r in wg):
        # smallest 64 x 64 weight gradient whose pixel chunks leave the last split empty on this device
        kchunks = next(c for c in range(SMS, 64 * SMS) if wgrad_regime(64 * c, 64, 64, 1)[3])
        g = _gen(7)
        dy, x = _ints((64 * kchunks, 64), -2, 2, g), _ints((64 * kchunks, 64), -2, 2, g)
        buf, out = _poisoned(64 * 64, torch.float32)
        ops.wgrad_taps(dy, x, out.view(1, 64, 64), 1, 0)
        assert _margins_untouched(buf) and torch.equal(out.view(64, 64).double(), R.conv1x1_wgrad(dy, x))
        print(f"synthetic wgrad with an empty last split: {64 * kchunks} rows")


# ---------------------------------------------------------------------------------------------- e4m3 paths
@pytest.mark.parametrize("M,N,K", [(1568, 64, 256), (25088, 128, 512)])
def test_per_tensor_e4m3_gemm_is_exact_with_power_of_two_scales(M, N, K):
    """kmajor_gemm_kernel<BN, true> (BN = 64 and 128): e4m3 integer operands, scale_a * scale_b a power of two, so
    the result is bf16_rn(alpha * A B^T) exactly, on each of three launches into separate poisoned outputs (a race
    would have to hit none of them); then randn operands through fp8_quantize within the e4m3 bound."""
    g = _gen(11)
    a, b = _ints((M, K), -2, 2, g, torch.float32), _ints((N, K), -2, 2, g, torch.float32)
    qa, qb = a.to(torch.float8_e4m3fn).view(torch.uint8), b.to(torch.float8_e4m3fn).view(torch.uint8)
    sa, sb = torch.tensor([0.125], device="cuda"), torch.tensor([4.0], device="cuda")
    S = a.double().abs() @ b.double().abs().t()
    R.assert_exact_premise(S, R.FP8_INT_LIMIT)
    ref = R.bf16_rn(0.5 * (a.double() @ b.double().t()))
    for _ in range(3):
        buf, out = _poisoned(M * N)
        ops.gemm_taps(qa, qb, out.view(M, N), N, K, [], 0, 0, 0, 0, sa, sb)
        assert _margins_untouched(buf) and _bits_equal(out.view(M, N), ref)
    kern = f"kmajor_gemm_kernel<{kmajor_regime(M, N)[0]}, true>"
    scratch = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    _, seen = _confirm(lambda: [ops.gemm_taps(qa, qb, scratch, N, K, [], 0, 0, 0, 0, sa, sb) for _ in range(4)], [kern])
    assert seen == {kern}, f"the profiler never showed {kern} in 4 traces"
    # real data: the per-tensor quantiser then the same GEMM with the de-quantisation factors
    x = (torch.randn(M, K, device="cuda", generator=g) * 3).to(torch.bfloat16)
    wv = torch.randn(N, K, device="cuda", generator=g).to(torch.bfloat16)
    qs = []
    for t in (x, wv):
        scale = torch.tensor([224.0 / float(t.float().abs().max())], device="cuda")
        amax = torch.zeros(1, device="cuda")
        q = torch.empty(t.shape, dtype=torch.uint8, device="cuda")
        ops.fp8_quantize(t, q, scale, amax)
        rq, ramax = R.fp8_quantize(t, float(scale))
        assert torch.equal(q, rq) and float(amax) == ramax
        qs.append((q, 1.0 / scale))
    (q1, i1), (q2, i2) = qs
    ops.gemm_taps(q1, q2, out.view(M, N), N, K, [], 0, 0, 0, 0, i1, i2)
    d1 = q1.view(torch.float8_e4m3fn).double() * float(i1)
    d2 = q2.view(torch.float8_e4m3fn).double() * float(i2)
    ref, S = d1 @ d2.t(), d1.abs() @ d2.abs().t()
    # alpha = fl(i1 * i2) is one more fp32 rounding of the whole sum
    bound = R.gemm_bound(ref, S, K + 1, R.FP8_STEP_EPS, K // 32)
    _check(R.within(out.view(M, N), ref, bound), f"per-tensor e4m3 {M}x{N}x{K}")
    COVERAGE["fp8_err"].append(float(((out.view(M, N).double() - ref).abs() / S.clamp_min(1e-30)).max()))


def test_gemm_binding_works_as_the_first_cuda_work_of_a_new_thread():
    """A thread that has made no CUDA runtime call has no current context (autograd's device thread can be one when
    a tc_conv backward comes first). The GEMM bindings encode their tensor maps through the driver, which needs one:
    gemm_taps as the very first CUDA work of a new Python thread must run, and run exactly."""
    import threading

    M, N, K = 1568, 64, 128
    g = _gen(13)
    a, b = _ints((M, K), -2, 2, g), _ints((N, K), -2, 2, g)
    buf, out = _poisoned(M * N)
    torch.cuda.synchronize()
    errors = []

    def work():
        try:
            ops.gemm_taps(a, b, out.view(M, N), N, K, [], 0, 0, 0, 0, None, None)
        except Exception as e:  # noqa: BLE001 (re-raised in the test's thread)
            errors.append(e)

    t = threading.Thread(target=work)
    t.start()
    t.join()
    assert not errors, errors[0]
    torch.cuda.synchronize()
    assert _margins_untouched(buf) and _bits_equal(out.view(M, N), R.bf16_rn(a.double() @ b.double().t()))


def test_quantisers_match_the_reference_bytes_on_boundary_cases():
    """mxfp8_quantize on hand-built blocks (all zero, amax = 448 * 2^k and one ulp above, bf16 subnormals, 130 rows:
    a partial row block whose padding bytes stay 127) and fp8_quantize on values past +-448, both byte for byte."""
    x = torch.zeros(130, 256, dtype=torch.bfloat16, device="cuda")
    x[0, 32:64] = 448.0 * 4
    x[0, 64] = 448.0 * 4 + 8
    x[1, :32] = torch.tensor([2.0 ** -133 * (i % 16 + 1) for i in range(32)]).to(torch.bfloat16)
    x[2, 96:128] = 448.0 * 2 ** -20
    x[3, 128:160] = -(448.0 * 2 ** 20)
    x[129, 224:] = -3.0
    x[64:100, 160:] = torch.randn(36, 96, device="cuda", generator=_gen(3)).to(torch.bfloat16) * 1e-3
    q, sf = ops.mxfp8_quantize(x)
    rq, rsf, _ = R.mx_quantize(x)
    assert torch.equal(q, rq) and torch.equal(sf, rsf)
    v = torch.tensor([0.0, 1.0, -1.0, 500.0, -1e4, 448.0, 449.0, 2.0 ** -12, 3.0, -0.0, 2.0 ** -133, 1e30, -1e30, 7.0,
                      0.3, -0.3], dtype=torch.bfloat16, device="cuda")
    for scale in (1.0, 0.25, 64.0, 0.3):
        for prev in (0.0, 2e30):
            amax = torch.tensor([prev], device="cuda")
            qq = torch.empty(16, dtype=torch.uint8, device="cuda")
            ops.fp8_quantize(v, qq, torch.tensor([scale], device="cuda"), amax)
            rq, ramax = R.fp8_quantize(v, scale, prev)
            assert torch.equal(qq, rq), (scale, qq.tolist(), rq.tolist())
            assert float(amax) == float(torch.tensor(ramax, dtype=torch.float32)), (scale, prev)


def test_fp8_scale_update_matches_target_over_amax():
    target = 224.0
    for a, s in ((3.0, 1.0), (1e-3, 5.0), (448.0 * 7, 0.5), (0.0, 3.0)):
        amax, scale, inv = (torch.tensor([v], device="cuda") for v in (a, s, 0.0))
        ops.fp8_scale_update(amax, scale, inv, target)
        rs, rinv, ramax = R.fp8_scale_update(a, s, target)
        assert float(scale) == rs and float(inv) == rinv and float(amax) == ramax, (a, s)


def test_mx_quantiser_matches_on_the_step_tensors(table):
    """mxfp8_quantize byte for byte on the MX operands of every table 1x1: activations (rows scaled by powers of two),
    weights, the gradient and the transposed weights of the dgrad."""
    for i, key in enumerate(sorted(k for k in table["1x1"] if k[6])):
        _, Cin, Cout, H, W, stride, _ = key
        M = B * ((H + stride - 1) // stride) * ((W + stride - 1) // stride)
        g = _gen(300 + i)
        rows = torch.exp2((torch.arange(M, device="cuda") % 13).float() - 6).unsqueeze(1)
        for t in ((torch.randn(M, Cin, device="cuda", generator=g) * rows).to(torch.bfloat16),
                  torch.randn(M, Cout, device="cuda", generator=g).to(torch.bfloat16),
                  (torch.randn(Cout, Cin, device="cuda", generator=g) * 0.05).to(torch.bfloat16),
                  (torch.randn(Cin, Cout, device="cuda", generator=g) * 0.05).to(torch.bfloat16)):
            q, sf = ops.mxfp8_quantize(t)
            rq, rsf, _ = R.mx_quantize(t)
            assert torch.equal(q, rq) and torch.equal(sf, rsf), key


# ---------------------------------------------------------------------------------------------- BatchNorm, pool
def test_batchnorm_at_every_table_shape(table):
    """Every (C, P, residual, ReLU) of the table, channels 0-7 with mean / std = 16: forward output, mean, invstd,
    running statistics, dgamma, dbeta, dx within the bounds derived from the fp32 statistics path; dres and the ReLU
    mask exact against the kernel's own bf16 output."""
    eps, mom = 1e-5, 0.1
    for i, (_, C, P, has_res, relu) in enumerate(sorted(table["bn"])):
        g = _gen(400 + i)
        x = torch.randn(P, C, device="cuda", generator=g)
        x[:, :8] += 16.0
        x = x.to(torch.bfloat16)
        res = torch.randn(P, C, device="cuda", generator=g).to(torch.bfloat16) if has_res else None
        gamma = 1 + 0.2 * torch.randn(C, device="cuda", generator=g)
        beta = 0.1 * torch.randn(C, device="cuda", generator=g)
        rm0, rv0 = 0.1 * torch.randn(C, device="cuda", generator=g), 1 + torch.rand(C, device="cuda", generator=g)
        rm, rv = rm0.clone(), rv0.clone()
        sbuf, stats = _poisoned(4 * C, torch.float32)
        ybuf, y = _poisoned(P * C)
        y = y.view(P, C)
        ops.bn_forward(x, res, gamma, beta, rm, rv, stats[:C], stats[C:2 * C], stats[2 * C:], y, mom, eps, relu)
        assert _margins_untouched(sbuf) and _margins_untouched(ybuf)
        ref = R.bn_forward(x, res, gamma, beta, eps, relu)
        bb = R.BNBounds(x, gamma, beta, eps, SMS, ref)
        what = f"bn C={C} P={P} res={has_res} relu={relu}"
        fb, e = bb.forward(x, res, ref[1])
        _check(R.within(y, ref[0], fb), what + " y")
        if relu:
            sure = ref[1].abs() > e
            assert bool(((y.float() > 0) == (ref[1] > 0))[sure].all()), what + " mask"
        _check(R.within(stats[:C], ref[2], bb.mean_bound()), what + " mean")
        _check(R.within(stats[C:2 * C], ref[4], bb.invstd_bound()), what + " invstd")
        m2, v2 = R.bn_running(rm0, rv0, ref[2], ref[3], P, mom)
        dm, dv = bb.running(rm0, rv0, mom)
        _check(R.within(rm, m2, dm), what + " running mean")
        _check(R.within(rv, v2, dv), what + " running var")
        # the statistics against the statistical bound, per channel; the batch variance the kernel used is read back
        # from the running variance it wrote, rv = (1 - m) rv0 + m k var (m = momentum in fp32, k = P / (P - 1))
        m32, k = float(torch.tensor(mom, dtype=torch.float32)), P / (P - 1)
        var_k = (rv.double() - (1 - m32) * rv0.double()) / (m32 * k)
        rec = 4 * R.U32 * (rv.double().abs() + (1 - m32) * rv0.double() + m32 * k * ref[3]) / (m32 * k)
        dm_s, dv_s, dis_s = bb.statistical()
        for name, got, want, bnd in (("mean", stats[:C], ref[2], dm_s), ("var", var_k, ref[3], dv_s + rec),
                                     ("invstd", stats[C:2 * C], ref[4], dis_s)):
            for chans, label in ((slice(0, 8), "mean/std = 16"), (slice(8, C), "mean 0")):
                ok, msg = R.within(got[chans], want[chans], bnd[chans])
                print(f"{what} {name}, channels with {label}, statistical bound: {msg}")
                assert ok, f"{what} {name} ({label}): {msg}"
        del fb, e
        dy = torch.randn(P, C, device="cuda", generator=g).to(torch.bfloat16)
        s2buf, sums = _poisoned(2 * C, torch.float32)
        dxbuf, dx = _poisoned(P * C)
        drbuf, dres = _poisoned(P * C)
        dx, dres = dx.view(P, C), dres.view(P, C)
        ops.bn_backward(dy, x, y, stats[:C], stats[C:2 * C], gamma, sums, dx, dres if has_res else None, relu)
        assert _margins_untouched(s2buf) and _margins_untouched(dxbuf) and _margins_untouched(drbuf)
        mask = R.relu_mask(y, relu)
        rdx, d, dgamma, dbeta = R.bn_backward(dy, x, mask, gamma, ref[2], ref[4])
        ddg, ddb, dxb = bb.backward(x, d, dgamma, dbeta, rdx)
        _check(R.within(sums[C:], dgamma, ddg), what + " dgamma")
        _check(R.within(sums[:C], dbeta, ddb), what + " dbeta")
        _check(R.within(dx, rdx, dxb), what + " dx")
        if has_res:
            want = torch.where(mask, dy, torch.zeros_like(dy))
            assert torch.equal(dres.view(torch.int16), want.view(torch.int16)), what + " dres"
        del ref, bb, rdx, d, dxb, mask
    torch.cuda.empty_cache()


def test_avgpool_at_the_table_shapes(table):
    for i, (_, Bn, HW, C) in enumerate(sorted(table["pool"])):
        g = _gen(500 + i)
        x = (torch.randn(Bn, HW, C, device="cuda", generator=g) + 2).to(torch.bfloat16)
        buf, out = _poisoned(Bn * C, torch.float32)
        ops.avgpool_forward(x, out, Bn, HW, C)
        ref = R.avgpool_fwd(x)
        assert _margins_untouched(buf)
        _check(R.within(out.view(Bn, C), ref, R.avgpool_fwd_bound(x)), f"avgpool fwd {Bn, HW, C}")
        dout = torch.randn(Bn, C, device="cuda", generator=g)
        buf, dx = _poisoned(Bn * HW * C)
        ops.avgpool_backward(dout, dx, Bn, HW, C)
        assert _margins_untouched(buf)
        rdx = R.avgpool_bwd(dout, HW)
        e = 2 * R.U32 * rdx.abs()
        _check(R.within(dx.view(Bn, HW, C), rdx, R.half_ulp_bf16(rdx.abs() + e) + e), f"avgpool bwd {Bn, HW, C}")

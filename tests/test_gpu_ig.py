"""Integrated Gradients on the H100 (DESIGN.md §12): the input_grad0 kernel against float64, one path point of the
engine teacher-forced on its own activations, the whole ``attribute`` against float64 ``integrated_gradients_torch``,
batch independence, and that attributing leaves a training run bit for bit as it was."""
import copy
import os

import pytest
import torch

import medcnn_ref as R
from hefl_b200 import _ext
from hefl_b200.config import FLConfig
from hefl_b200.fl import FederatedRunner
from hefl_b200.fl.data import SyntheticImageDataset
from hefl_b200.fl.explain import integrated_gradients_torch
from hefl_b200.models import ParamPack, create_model

ops = _ext.ops()
pytestmark = pytest.mark.gpu
CUDA = torch.device("cuda")
# calibrated on the H100: test_attribute_matches_float64_integrated_gradients
REL_L2, GAP_RATIO = 0.35, 0.03
TERMS = 4 * 32 + 1          # products per pixel (<= 4 windows x 32 channels) and the add into the accumulator


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _inputs(B, S, ci, seed):
    Hp = (S - 2) // 2
    g = _gen(seed)
    grad = (torch.randn(B * Hp * Hp, 32, device="cuda", generator=g) * 0.1).to(torch.bfloat16)
    code = torch.randint(0, 8, (B * Hp * Hp, 32), device="cuda", generator=g, dtype=torch.uint8)
    w = (torch.randn(32, ci, 3, 3, device="cuda", generator=g) * 0.2).to(torch.bfloat16)
    return Hp, grad, code, w


def _ref(grad, code, w, B, S, Hp):
    """(dx, sum of |terms|) in float64, [B, S, S, Ci]."""
    gp, cp = R.nchw(grad, B, Hp, Hp), R.nchw(code, B, Hp, Hp)
    dy = R.conv_grid_grad(gp, cp, S, S)
    wd = w.double()
    return (R.dgrad(dy, wd).permute(0, 2, 3, 1), R.dgrad_abs(dy, wd).permute(0, 2, 3, 1))


# ------------------------------------------------------------------ the kernel
# RGB and grayscale at the engine's batch 32 and 256 x 256, odd sizes (an odd conv grid: the floor-pool edge is
# dropped), and a single scan
SHAPES = [(32, 256, 3), (32, 256, 1), (3, 129, 3), (2, 127, 1), (1, 64, 3), (1, 5, 1)]


@pytest.mark.parametrize("B,S,ci", SHAPES)
def test_input_grad0_matches_float64(B, S, ci):
    Hp, grad, code, w = _inputs(B, S, ci, seed=S * 10 + ci)
    ref, ab = _ref(grad, code, w, B, S, Hp)
    acc = torch.zeros(B, S, S, ci, device="cuda")
    n0 = int(ops.launch_count())
    ops.input_grad0(grad, code, w.view(-1), acc, B, S, ci, B)
    torch.cuda.synchronize()
    assert int(ops.launch_count()) - n0 == 1
    assert R.within(acc, ref, TERMS * R.ACC_EPS * ab), float((acc.double() - ref).abs().max())
    # the 2-pixel border and the dropped floor-pool edge get no gradient
    edge = 2 * Hp + 2
    assert (acc[:, edge:] == 0).all() and (acc[:, :, edge:] == 0).all()
    # a second call accumulates; a repeat gives the same bits
    first = acc.clone()
    ops.input_grad0(grad, code, w.view(-1), acc, B, S, ci, B)
    assert R.within(acc, 2 * ref, 2 * TERMS * R.ACC_EPS * ab)
    again = first.clone()
    ops.input_grad0(grad, code, w.view(-1), again, B, S, ci, B)
    assert torch.equal(again, acc)


@pytest.mark.parametrize("ci", [3, 1])
def test_input_grad0_leaves_scans_past_nvalid_alone(ci):
    """Scans >= nvalid are neither read (their gradient is NaN) nor written (their accumulator stays NaN), and the
    valid scans' bits do not depend on the batch size."""
    B, S, nv = 8, 130, 5
    Hp, grad, code, w = _inputs(B, S, ci, seed=77 + ci)
    poisoned = grad.clone().view(B, -1)
    poisoned[nv:] = float("nan")
    acc = torch.full((B, S, S, ci), float("nan"), device="cuda")
    acc[:nv] = 0
    ops.input_grad0(poisoned.view_as(grad), code, w.view(-1), acc, B, S, ci, nv)
    torch.cuda.synchronize()
    assert torch.isnan(acc[nv:]).all()
    assert not torch.isnan(acc[:nv]).any()
    full = torch.zeros(B, S, S, ci, device="cuda")
    ops.input_grad0(grad, code, w.view(-1), full, B, S, ci, B)
    assert torch.equal(acc[:nv], full[:nv])
    # the same scans placed last in a batch
    order = torch.arange(B - 1, -1, -1, device="cuda")
    rev = torch.zeros_like(full)
    ops.input_grad0(grad.view(B, -1)[order].contiguous().view_as(grad), code.view(B, -1)[order].contiguous()
                    .view_as(code), w.view(-1), rev, B, S, ci, B)
    assert torch.equal(rev[order], full)


def test_input_grad0_rejects_bad_arguments():
    Hp, grad, code, w = _inputs(1, 64, 3, seed=5)
    acc = torch.zeros(1, 64, 64, 3, device="cuda")
    with pytest.raises(RuntimeError, match="in_channels"):
        ops.input_grad0(grad, code, w.view(-1), acc, 1, 64, 2, 1)
    with pytest.raises(RuntimeError, match="Hp"):
        ops.input_grad0(grad, code, w.view(-1), acc, 1, 66, 3, 1)
    with pytest.raises(RuntimeError, match="nvalid"):
        ops.input_grad0(grad, code, w.view(-1), acc, 1, 64, 3, 2)


# ------------------------------------------------------------------ one path point of the engine
@pytest.mark.parametrize("ch", [3, 1])
def test_path_point_matches_the_reference_chain(ch, monkeypatch):
    """One path point (steps = 1, alpha = 1/2): slot 0 is bf16(alpha x) of slot 1, the chain from dfeat down to X[1]
    and the accumulator are medcnn_ref applied to the engine's own X, codes and dfeat, to the training step's dgrad
    bounds; the attribution is x * acc summed over channels; only scratch buffers change."""
    from hefl_b200.ops.conv_engine import MedCNNEngine

    for k in list(os.environ):
        if k.startswith("HEFL_"):
            monkeypatch.delenv(k)
    torch.manual_seed(3)
    cfg = FLConfig(in_channels=ch)
    model = create_model("medcnn", in_channels=ch).to(CUDA)
    pack = ParamPack(model)
    eng = MedCNNEngine(model, pack, cfg, CUDA)
    B, S, n = eng.B, eng.H[0], eng.n
    g = _gen(60 + ch)
    x = torch.randint(0, 256, (B, S, S, ch), dtype=torch.uint8, device="cuda", generator=g)
    target = torch.randint(-1, 2, (B,), device="cuda", generator=g)
    pack.grad.copy_(torch.randn(pack.grad.shape, device="cuda", generator=g))
    eng.dW32.copy_(torch.randn(eng.dW32.shape, device="cuda", generator=g))
    keep = [t.clone() for t in (pack.flat, pack.grad, eng.dW32, eng.Wf, eng.Wd, eng.shadow)]
    prep = eng.prep_count
    logits, base = torch.zeros(B, 2, device="cuda"), torch.zeros(B, 2, device="cuda")
    attr = torch.full((B, S, S), float("nan"), device="cuda")
    eng.preprocess(x, 1, False, False)
    t = eng.ig_staged(1, target, logits, base, attr, B)
    torch.cuda.synchronize()
    x1, x0 = eng.x0(1), eng.x0(0)
    assert torch.equal(x0, (x1.float() * 0.5).to(torch.bfloat16))
    assert torch.equal(t, torch.where(target < 0, logits.argmax(1), target))
    ws = [c.weight.detach().to(torch.bfloat16).double() for c in model.convs]
    for l in range(n - 1, 0, -1):
        H, Hp = eng.H[l], eng.H[l + 1]
        gl = eng.dfeat if l == n - 1 else eng.gX[l + 1]
        gpr = R.nchw(gl.view(-1, eng.Co[l]), B, Hp, Hp)
        dy = R.unpool(gpr, R.nchw(eng.X[l + 1], B, Hp, Hp), R.nchw(eng.amax[l], B, Hp, Hp), H, H)
        assert torch.equal(eng.dY[l], R.nhwc(dy).to(torch.bfloat16)), l
        rd, sd = R.dgrad(dy, ws[l]), R.dgrad_abs(dy, ws[l])
        assert R.within(R.nchw(eng.gX[l], B, H, H), rd, R.fwd_bound(rd, sd, 9 * eng.Co[l])), l
    ref, ab = _ref(eng.gX[1], eng.amax[0], ws[0], B, S, eng.H[1])
    assert R.within(eng.ig_acc, ref, TERMS * R.ACC_EPS * ab), float((eng.ig_acc.double() - ref).abs().max())
    assert float(ref.abs().max()) > 0, "the path point must carry a gradient"
    xh = x1[: B * S * S, :ch].view(B, S, S, ch).float()
    assert torch.equal(attr, (xh * eng.ig_acc).sum(-1) / 1)
    for a, b in zip(keep, (pack.flat, pack.grad, eng.dW32, eng.Wf, eng.Wd, eng.shadow)):
        assert torch.equal(a, b), "ig_staged changed a parameter, gradient or weight layout"
    assert eng.prep_count == prep


# ------------------------------------------------------------------ attribute on the engine
def _cfg(**kw):
    return FLConfig(model="medcnn", local_epochs=1, steps_per_epoch=2, val_steps=1, deterministic_crypto=True, **kw)


def _train(run, steps, seed):
    ds = SyntheticImageDataset(run.cfg.batch_size * steps, 256, run.cfg.in_channels, 2, seed=seed, pin=False)
    losses = []
    B = run.cfg.batch_size
    for i in range(steps):
        out = run.trainer.train_step(ds.images[i * B:(i + 1) * B].to(CUDA), ds.labels[i * B:(i + 1) * B].to(CUDA))
        losses.append(out.clone())
    torch.cuda.synchronize()
    return losses


@pytest.fixture(scope="module")
def trained():
    run = FederatedRunner(_cfg(), device=CUDA)
    assert run.trainer.engine is not None and run.trainer.engine.fused_head
    _train(run, 4, seed=12)
    x = SyntheticImageDataset(37, 256, 3, 2, seed=9, pin=False).images
    return run, x


def test_attribute_matches_float64_integrated_gradients(trained):
    """The engine (bf16 path points and activations, fp32 sums) against float64 autograd (no bf16 rounding) on the same
    weights and scans, for the float64 predicted class, m = 16; and the engine's completeness gap at m = 64. Observed on
    an H100 80GB HBM3 (700 W) after 4 training steps: per-scan relative L2 error of attr 0.13 to 0.23 (median 0.18),
    |p - p64| <= 3.6e-4, |gap| / |score - baseline score| at m = 64 at most 0.012 (median 0.0027; float64 at m = 16:
    0.019). The pixel-level error is that of bf16 activations and gradients through six layers, where a pooling
    window whose two largest conv outputs are within rounding moves its gradient to the neighbouring pixel; the
    teacher-forced path-point test pins the arithmetic. Asserted with margin: REL_L2 = 0.35 and GAP_RATIO = 0.03."""
    run, x = trained
    x = x[:32]
    ref_model = copy.deepcopy(run.model).double()
    p64, a64, g64 = integrated_gradients_torch(ref_model, x, 16)
    t = p64.argmax(1).cpu()
    probs, attr, gap = run.attribute(x, steps=16, target=t)
    a64, g64 = a64.cpu(), g64.cpu()
    rel = (attr.double() - a64).norm(dim=(1, 2)) / a64.norm(dim=(1, 2))
    _, _, gap_m, _, score, base = run._attribute(x, 64, t, None)
    ratio = gap_m.double().abs() / (score.double() - base.double()).abs()
    print(f"attribute vs float64 (m = 16): rel L2 max {float(rel.max()):.3e} median {float(rel.median()):.3e}, "
          f"|dp| max {float((probs.double() - p64.cpu()).abs().max()):.2e}; float64 |gap| / |ds| at m = 16 max "
          f"{float((g64.abs() / (a64.sum((1, 2)) - g64).abs()).max()):.3e}; engine |gap| / |ds| at m = 64 max "
          f"{float(ratio.max()):.3e} median {float(ratio.median()):.3e}")
    assert (probs.double() - p64.cpu()).abs().max() <= 1e-3
    assert float(rel.max()) <= REL_L2
    assert float(ratio.max()) <= GAP_RATIO


def test_attribute_is_batch_independent(trained):
    """37 scans at B = 32 (a full batch and a padded one), the same scans permuted, and the last 5 inside a full batch:
    per-scan probabilities, attributions and gaps are bit-identical."""
    run, x = trained
    r = run.attribute(x, steps=4)
    perm = torch.randperm(37, generator=torch.Generator().manual_seed(4))
    rp = run.attribute(x[perm], steps=4)
    inv = torch.argsort(perm)
    assert all(torch.equal(a[inv], b) for a, b in zip(rp, r))
    rf = run.attribute(x[5:37], steps=4)
    assert all(torch.equal(a, b[5:37]) for a, b in zip(rf, r))


def _state(run):
    tr = run.trainer
    return [run.pack.flat.clone(), tr.m.clone(), tr.v.clone(), tr.step_t.clone(), tr.lr_scale.clone()]


@pytest.mark.parametrize("personal", [False, True])
def test_attribute_leaves_training_bit_identical(personal):
    """Graph-replayed training: 3 steps, attribute, 3 steps equals 6 steps without it (weights, loss, Adam state,
    gradients, augmentation position, torch RNG); with personal layers, attribute runs with the other client's head."""
    kw = dict(personal_layers=1, clients_per_rank=2) if personal else {}
    x = SyntheticImageDataset(5, 256, 3, 2, seed=3, pin=False).images
    results = []
    for attribute in (True, False):
        run = FederatedRunner(_cfg(**kw), device=CUDA)
        assert run.trainer.use_graph and run.trainer.engine is not None
        if personal:
            run._c_head[1].add_(0.01)
        losses = _train(run, 3, seed=5)
        if attribute:
            run.attribute(x, steps=3, client=1 if personal else None)
        losses += _train(run, 3, seed=6)
        eng = run.trainer.engine
        results.append((_state(run) + [run.pack.grad.clone(), eng.dW32.clone()], torch.stack(losses).cpu(),
                        eng.prep_count, torch.get_rng_state(), torch.cuda.get_rng_state()))
    (s1, l1, c1, r1, g1), (s2, l2, c2, r2, g2) = results
    assert all(torch.equal(a, b) for a, b in zip(s1, s2))
    assert torch.equal(l1, l2) and c1 == c2 and c1 > 0
    assert torch.equal(r1, r2) and torch.equal(g1, g2)

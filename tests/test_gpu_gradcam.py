"""Grad-CAM on the H100 (DESIGN.md §11): the gradcam kernel at every stage shape of the medical CNN against float64,
the head's saliency mode (cluster kernel and four-kernel fallback) against float64 autograd, the engine's un-pool /
dgrad chain down to every stage, the whole explain step against ``gradcam_torch`` in float64, batch independence, and
that explaining leaves a training run bit for bit as it was."""
import copy
import os

import pytest
import torch
import torch.nn.functional as F

import medcnn_ref as R
from hefl_b200 import _ext
from hefl_b200.config import FLConfig
from hefl_b200.fl import FederatedRunner
from hefl_b200.fl.data import SyntheticImageDataset
from hefl_b200.fl.explain import gradcam_torch
from hefl_b200.models import ParamPack, create_model

ops = _ext.ops()
pytestmark = pytest.mark.gpu
CUDA = torch.device("cuda")
SENTINEL = 7.5
MARGIN, PEARSON, MIN_MAPS = 0.05, 0.9, 36         # calibrated on the H100: test_explain_matches_float64_gradcam_torch


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _cam_ref(X, G, B, Hp, C, S):
    """Steps 3-6 of the definition in float64 on the kernel's own bf16 inputs: [B, S, S], and per scan the ratio of the
    largest sum of |alpha_c X_c| over the map's maximum (how much cancellation the fp32 sums faced)."""
    X = X.double().view(B, Hp * Hp, C)
    G = G.double().view(B, Hp * Hp, C)
    alpha = G.mean(1)
    cam = torch.relu((X * alpha[:, None, :]).sum(-1)).view(B, Hp, Hp)
    absum = (X * alpha[:, None, :]).abs().sum(-1).amax(1)
    up = F.interpolate(cam[:, None], (S, S), mode="bilinear", align_corners=False)[:, 0]
    mx = cam.amax((1, 2))
    out = torch.where(mx[:, None, None] > 0, up / torch.where(mx > 0, mx, 1)[:, None, None], torch.zeros_like(up))
    return out, absum / torch.where(mx > 0, mx, 1)


# ------------------------------------------------------------------ the gradcam kernel
# the six stages of the medical CNN at 256 x 256, an odd map with an odd channel count and an odd output size (the
# scalar-store path), and a 1 x 1 map
SHAPES = [(127, 32, 256), (62, 32, 256), (30, 32, 256), (14, 64, 256), (6, 64, 256), (2, 128, 256), (63, 24, 129),
          (1, 8, 256)]


@pytest.mark.parametrize("Hp,C,S", SHAPES)
def test_gradcam_kernel_matches_float64(Hp, C, S):
    """X ~ U[0, 1) (a post-ReLU stage output) and G = 0.02 + 0.01 N(0, 1): alpha_c ~ 0.02 > 0 for every channel, so
    the map is a sum of positive terms and its maximum is not the result of cancellation."""
    B = 32
    g = _gen(Hp * 1000 + C)
    X = torch.rand(B * Hp * Hp, C, device="cuda", generator=g).to(torch.bfloat16)
    G = (0.02 + 0.01 * torch.randn(B * Hp * Hp, C, device="cuda", generator=g)).to(torch.bfloat16)
    ref, _ = _cam_ref(X, G, B, Hp, C, S)
    out = torch.full((B + 3, S, S), SENTINEL, device="cuda")
    n0 = int(ops.launch_count())
    ops.gradcam(X, G, out, B, Hp, C, S, B)
    torch.cuda.synchronize()
    assert int(ops.launch_count()) - n0 == 1
    err = (out[:B].double() - ref).abs().max().item()
    assert err <= 1e-4, err
    assert (out[B:] == SENTINEL).all()
    again = torch.full_like(out, SENTINEL)
    ops.gradcam(X, G, again, B, Hp, C, S, B)
    assert torch.equal(out, again), "two launches differ"
    # rows >= nvalid of a larger buffer are neither computed nor written
    part = torch.full((B, S, S), SENTINEL, device="cuda")
    ops.gradcam(X, G, part, B, Hp, C, S, B - 5)
    assert torch.equal(part[:B - 5], out[:B - 5]) and (part[B - 5:] == SENTINEL).all()
    # an all-negative map: exact zeros, never NaN
    neg = torch.full_like(out, SENTINEL)
    ops.gradcam(X, (-G.float()).to(torch.bfloat16), neg, B, Hp, C, S, B)
    torch.cuda.synchronize()
    assert torch.equal(neg[:B], torch.zeros_like(neg[:B]))


def test_gradcam_rejects_unsupported_shapes():
    X = torch.zeros(4 * 4, 12, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="multiple of 8"):
        ops.gradcam(X, X, torch.zeros(1, 8, 8, device="cuda"), 1, 4, 12, 8, 1)
    X = torch.zeros(300 * 300, 8, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="shared memory"):
        ops.gradcam(X, X, torch.zeros(1, 8, 8, device="cuda"), 1, 300, 8, 8, 1)


# ------------------------------------------------------------------ the head's saliency mode
@pytest.mark.parametrize("explicit", [True, False])
@pytest.mark.parametrize("C", [2, 3])
@pytest.mark.parametrize("B", [8, 32])
@pytest.mark.parametrize("Fdim", [512, 256])
def test_head_saliency_matches_float64_autograd(Fdim, B, C, explicit):
    """F = 512 runs the cluster kernel (1 launch), F = 256 the four-kernel fallback (4 launches)."""
    H1, H2 = 128, 64
    g = _gen(Fdim + 7 * B + C)
    sizes = [H1 * Fdim, H1, H2 * H1, H2, C * H2, C]
    offs = [0]
    for n in sizes[:-1]:
        offs.append(offs[-1] + n)
    flat = torch.randn(sum(sizes), device="cuda", generator=g) * 0.05
    grad = torch.randn(sum(sizes), device="cuda", generator=g)
    grad0 = grad.clone()
    feat = torch.rand(B, Fdim, device="cuda", generator=g).to(torch.bfloat16)
    target = (torch.randint(0, C, (B,), device="cuda", generator=g) if explicit
              else torch.full((B,), -1, dtype=torch.int64, device="cuda"))
    dfeat = torch.full((B, Fdim), SENTINEL, dtype=torch.bfloat16, device="cuda")
    h1_buf = torch.zeros(B * H1, device="cuda")
    dh1_buf = torch.zeros(B * (H1 + H2), device="cuda")
    logits = torch.full((B, C), SENTINEL, device="cuda")
    n0 = int(ops.launch_count())
    ops.head_saliency(feat, flat, offs, target, dfeat, h1_buf, dh1_buf, logits, B, Fdim, H1, H2, C)
    torch.cuda.synchronize()
    assert int(ops.launch_count()) - n0 == (1 if Fdim == 512 else 4)
    assert torch.equal(grad, grad0), "the saliency mode wrote a parameter gradient"
    ps = [flat[o:o + n].double().view(-1) for o, n in zip(offs, sizes)]
    x = feat.double().requires_grad_(True)
    h = F.relu(F.linear(x, ps[0].view(H1, Fdim), ps[1]))
    h = F.relu(F.linear(h, ps[2].view(H2, H1), ps[3]))
    ref_logits = F.linear(h, ps[4].view(C, H2), ps[5])
    assert (logits.double() - ref_logits).abs().max() <= 1e-4
    t = target if explicit else logits.argmax(1)
    if not explicit:                 # -1 resolves to the arg-max, the float64 one wherever the margin is clear
        top2 = ref_logits.detach().topk(2, 1).values
        clear = (top2[:, 0] - top2[:, 1]) > 1e-3
        assert torch.equal(t[clear], ref_logits.argmax(1)[clear])
    ref_logits.gather(1, t[:, None]).sum().backward()
    assert (dfeat.double() - x.grad).abs().max() <= 1e-2 * x.grad.abs().max() + 1e-7


# ------------------------------------------------------------------ the engine
def _engine(ch, seed=3):
    from hefl_b200.ops.conv_engine import MedCNNEngine

    torch.manual_seed(seed)
    cfg = FLConfig(in_channels=ch)
    assert (cfg.batch_size, cfg.image_size) == (32, 256)
    model = create_model("medcnn", in_channels=ch).to(CUDA)
    pack = ParamPack(model)
    return model, pack, MedCNNEngine(model, pack, cfg, CUDA)


@pytest.mark.parametrize("ch", [3, 1])
def test_engine_chain_matches_the_reference_at_every_stage(ch, monkeypatch):
    """G at X[s] is medcnn_ref's unpool / dgrad chain applied to the engine's own X, codes and dfeat, layer by layer,
    to the bounds of the training step's dgrad chain; the map is steps 3-6 on the engine's X[s] and G; only scratch
    buffers change."""
    for k in list(os.environ):
        if k.startswith("HEFL_"):
            monkeypatch.delenv(k)
    model, pack, eng = _engine(ch)
    B, S, n = eng.B, eng.H[0], eng.n
    g = _gen(40 + ch)
    x = torch.randint(0, 256, (B, S, S, ch), dtype=torch.uint8, device="cuda", generator=g)
    target = torch.randint(-1, 2, (B,), device="cuda", generator=g)
    logits = torch.zeros(B, 2, device="cuda")
    cam = torch.full((B, S, S), SENTINEL, device="cuda")
    pack.grad.copy_(torch.randn(pack.grad.shape, device="cuda", generator=g))
    eng.dW32.copy_(torch.randn(eng.dW32.shape, device="cuda", generator=g))
    keep = [t.clone() for t in (pack.flat, pack.grad, eng.dW32, eng.Wf, eng.Wd, eng.shadow)]
    prep = eng.prep_count
    ws = [c.weight.detach().to(torch.bfloat16).double() for c in model.convs]
    fcs = copy.deepcopy(model.fcs).double()
    for s in range(1, n + 1):
        eng.preprocess(x, 0, False, False)
        eng.gradcam_staged(0, s, target, logits, cam, B)
        torch.cuda.synchronize()
        feat = eng.X[n].view(B, -1).double().requires_grad_(True)
        h = feat
        for fc in fcs[:-1]:
            h = F.relu(fc(h))
        ref_logits = fcs[-1](h)
        assert (logits.double() - ref_logits).abs().max() <= 1e-4, s
        t = torch.where(target < 0, logits.argmax(1), target)
        d_ref, = torch.autograd.grad(ref_logits.gather(1, t[:, None]).sum(), feat)
        d_got = eng.dfeat.view(B, -1).double()
        assert R.within(d_got, d_ref, R.BF16_EPS * d_ref.abs() + 2.0 ** -16 * d_ref.abs().max()), s
        for l in range(n - 1, s - 1, -1):
            H, Hp = eng.H[l], eng.H[l + 1]
            gl = eng.dfeat if l == n - 1 else eng.gX[l + 1]
            gpr = R.nchw(gl.view(-1, eng.Co[l]), B, Hp, Hp)
            dy = R.unpool(gpr, R.nchw(eng.X[l + 1], B, Hp, Hp), R.nchw(eng.amax[l], B, Hp, Hp), H, H)
            assert torch.equal(eng.dY[l], R.nhwc(dy).to(torch.bfloat16)), (s, l)
            rd, sd = R.dgrad(dy, ws[l]), R.dgrad_abs(dy, ws[l])
            assert R.within(R.nchw(eng.gX[l], B, H, H), rd, R.fwd_bound(rd, sd, 9 * eng.Co[l])), (s, l)
        G = eng.dfeat.view(-1, eng.Co[n - 1]) if s == n else eng.gX[s]
        ref, cond = _cam_ref(eng.X[s], G, B, eng.H[s], eng.Co[s - 1], S)
        err = (cam.double() - ref).abs().amax((1, 2))
        print(f"engine chain ({ch} ch) stage {s}: {int((ref.amax((1, 2)) > 0).sum())} of {B} maps non-zero, "
              f"max err {float(err.max()):.2e}, max cancellation ratio {float(cond.max()):.1f}")
        assert (err <= 1e-4 * cond.clamp_min(1.0)).all(), (s, float(err.max()), float(cond.max()))
    for a, b in zip(keep, (pack.flat, pack.grad, eng.dW32, eng.Wf, eng.Wd, eng.shadow)):
        assert torch.equal(a, b), "gradcam_staged changed a parameter, gradient or weight layout"
    assert eng.prep_count == prep


# ------------------------------------------------------------------ explain on the engine
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
def seeded():
    """The seeded medical CNN on the engine. Its stage-4 maps are live: a few training steps on the synthetic set
    leave stage 4 with no positive evidence for most scans, and a map that is zero on both paths compares nothing."""
    run = FederatedRunner(_cfg(), device=CUDA)
    assert run.trainer.engine is not None and run.trainer.engine.fused_head
    x = SyntheticImageDataset(37, 256, 3, 2, seed=9, pin=False).images
    return run, x


def test_explain_matches_float64_gradcam_torch(seeded):
    """The engine (bf16 activations, fp32 sums) against float64 autograd on the same weights and scans, at stage 4, for
    the predicted class and for each class. Observed on an H100 80GB HBM3 (700 W) in three runs, identical up to the
    float64 reference's last bits: the predicted class agreed on all 32 scans, |p - p64| <= 1.2e-4; Pearson
    correlation of the 256 x 256 maps min 0.959, median 0.995 over the 32 live maps of the predicted class (class 0
    for every scan), min 0.997 over the 4 live maps of class 1, where one more map was zero on one path only (its
    maximum is within rounding of 0). Asserted with margin: agreement wherever the float64 logit margin exceeds 0.05,
    Pearson > 0.9 on every map that is live on both paths, at most 2 maps zero on one path only per class, and at
    least 36 live maps over the three targets."""
    run, x = seeded
    x = x[:32]
    ref_model = copy.deepcopy(run.model).double()
    stats = {}
    for t in (None, 0, 1):
        probs, cams = run.explain(x, stage=4, target=t)
        p64, c64 = gradcam_torch(ref_model, x, stage=4, target=t)
        p64, c64 = p64.cpu(), c64.cpu()
        if t is None:
            top2 = p64.log().topk(2, 1).values
            margin = top2[:, 0] - top2[:, 1]
            clear = margin > MARGIN
            assert torch.equal(probs.argmax(1)[clear], p64.argmax(1)[clear])
            stats["min_margin_of_disagreement"] = float(margin[probs.argmax(1) != p64.argmax(1)].min()) \
                if bool((probs.argmax(1) != p64.argmax(1)).any()) else None
            stats["max_abs_dp"] = float((probs.double() - p64).abs().max())
        live = (cams.amax((1, 2)) > 0) & (c64.amax((1, 2)) > 0)
        a, b = cams.double().view(32, -1)[live], c64.view(32, -1)[live]
        a, b = a - a.mean(1, keepdim=True), b - b.mean(1, keepdim=True)
        r = (a * b).sum(1) / (a.norm(dim=1) * b.norm(dim=1))
        stats[f"target {t}"] = {"maps": int(live.sum()), "one_side_zero": int(((cams.amax((1, 2)) > 0) ^
                                                                             (c64.amax((1, 2)) > 0)).sum()),
                                "pearson_min": float(r.min()) if r.numel() else None,
                                "pearson_median": float(r.median()) if r.numel() else None}
    print("explain vs float64 at stage 4:", stats)
    for t in (None, 0, 1):
        st = stats[f"target {t}"]
        assert st["one_side_zero"] <= 2 and (not st["maps"] or st["pearson_min"] > PEARSON), (t, st)
    assert sum(stats[f"target {t}"]["maps"] for t in (None, 0, 1)) >= MIN_MAPS, stats


def test_explain_is_batch_independent(seeded):
    """37 scans at B = 32 (a full batch and a padded one), the same scans permuted, and the last 5 inside a full batch:
    per-scan probabilities and maps are bit-identical."""
    run, x = seeded
    p, c = run.explain(x, stage=4)
    perm = torch.randperm(37, generator=torch.Generator().manual_seed(4))
    pp, cp = run.explain(x[perm], stage=4)
    inv = torch.argsort(perm)
    assert torch.equal(pp[inv], p) and torch.equal(cp[inv], c)
    pf, cf = run.explain(x[5:37], stage=4)
    assert torch.equal(pf, p[5:37]) and torch.equal(cf, c[5:37])
    t = torch.arange(37) % 2
    pt, ct = run.explain(x, stage=2, target=t)
    ptp, ctp = run.explain(x[perm], stage=2, target=t[perm])
    assert torch.equal(ptp[inv], pt) and torch.equal(ctp[inv], ct)


def _state(run):
    tr = run.trainer
    return [run.pack.flat.clone(), tr.m.clone(), tr.v.clone(), tr.step_t.clone(), tr.lr_scale.clone()]


@pytest.mark.parametrize("personal", [False, True])
def test_explain_leaves_training_bit_identical(personal):
    """Graph-replayed training: 3 steps, explain, 3 steps equals 6 steps without explain (weights, loss, Adam state,
    augmentation position, torch RNG); with personal layers, explain runs with the other client's head."""
    kw = dict(personal_layers=1, clients_per_rank=2) if personal else {}
    x = SyntheticImageDataset(5, 256, 3, 2, seed=3, pin=False).images
    results = []
    for explain in (True, False):
        run = FederatedRunner(_cfg(**kw), device=CUDA)
        assert run.trainer.use_graph and run.trainer.engine is not None
        if personal:
            run._c_head[1].add_(0.01)
        losses = _train(run, 3, seed=5)
        if explain:
            run.explain(x, stage=3, client=1 if personal else None)
        losses += _train(run, 3, seed=6)
        results.append((_state(run), torch.stack(losses).cpu(), run.trainer.engine.prep_count,
                        torch.get_rng_state(), torch.cuda.get_rng_state()))
    (s1, l1, c1, r1, g1), (s2, l2, c2, r2, g2) = results
    assert all(torch.equal(a, b) for a, b in zip(s1, s2))
    assert torch.equal(l1, l2) and c1 == c2 and c1 > 0
    assert torch.equal(r1, r2) and torch.equal(g1, g2)

"""Compact RGB layer-1 input ([P, 4] = R, G, B, 0; 8 bytes per pixel instead of the 32 of the s-packed layout):
pre-processing, the pair-row forward and the masked-GEMM weight gradient on it, and the engine that selects it."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from hefl_b200 import _ext
    ops = _ext.ops()


def _bf(t):
    return t.to(torch.bfloat16)


def _spacked_and_compact(x, seed):
    B, H, W, _ = x.shape
    P = B * H * W
    Xs = torch.zeros(P + 8, 16, dtype=torch.bfloat16, device="cuda")
    Xc = torch.full((P, 4), float("nan"), dtype=torch.bfloat16, device="cuda")
    ops.preprocess_u8(x, None, Xs[:P], seed, None, True)
    ops.preprocess_u8(x, None, Xc, seed, None, True, True)
    return Xs, Xc


def _weights(w):
    """s-packed [3 r][Co][16] (k = 3 s + ci) and compact [3 r][2 dx][Co][16] (k = 4 (s + dx) + ci) layer-1 weights."""
    Co = w.shape[0]
    Ws = torch.zeros(3, Co, 16, dtype=torch.bfloat16, device="cuda")
    Ws[:, :, :9] = w.permute(2, 0, 3, 1).reshape(3, Co, 9).to(torch.bfloat16)
    Wc = torch.zeros(3, 2, Co, 4, 4, dtype=torch.bfloat16, device="cuda")
    for dx in range(2):
        Wc[:, dx, :, dx:dx + 3, :3] = w.permute(2, 0, 3, 1).to(torch.bfloat16)
    return Ws, Wc.view(3, 2, Co, 16)


@pytest.mark.parametrize("H,W", [(256, 256), (64, 70)])
@pytest.mark.parametrize("seed", [0, 12345, 987654321])
def test_compact_preprocess_is_channels_0_to_2_of_the_spacked_one(H, W, seed):
    """Same sampling, Philox keying and bf16 rounding: R, G, B bit-identical to channels 0-2 of the s-packed output,
    channel 3 zero (seed 0 = no augmentation; W = 70 is a multiple of neither warp run, 30 or 32)."""
    B = 4
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randint(0, 256, (B, H, W, 3), dtype=torch.uint8, device="cuda", generator=g)
    Xs, Xc = _spacked_and_compact(x, seed)
    P = B * H * W
    assert torch.equal(Xc[:, :3].view(torch.int16), Xs[:P, :3].view(torch.int16))
    assert torch.equal(Xc[:, 3].view(torch.int16), torch.zeros(P, dtype=torch.int16, device="cuda"))


def test_compact_weight_relayout_matches_the_reference_layout():
    """conv_weight_relayout(compact0): s-packed [3][32][16] and then compact [3][2][32][16] in layer 1's Wf slot."""
    from hefl_b200.config import FLConfig
    from hefl_b200.models import ParamPack, create_model
    from hefl_b200.ops.conv_engine import MedCNNEngine

    torch.manual_seed(2)
    dev = torch.device("cuda")
    model = create_model("medcnn").to(dev)
    pack = ParamPack(model)
    eng = MedCNNEngine(model, pack, FLConfig(model="medcnn", batch_size=8, image_size=256), dev)
    assert eng.compact0
    w = model.convs[0].weight.detach().to(torch.bfloat16).float()
    Ws, Wc = _weights(w)
    wf0 = eng.Wf[eng.wf_off[0]: eng.wf_off[1]]
    assert torch.equal(wf0[: Ws.numel()], Ws.view(-1))
    assert torch.equal(eng._wf0c(), Wc.view(-1))


@pytest.mark.parametrize("B,H", [(32, 256), (3, 70), (1, 20)])
def test_compact_pair_forward_matches_the_spacked_one(B, H):
    """Pair-row forward on the compact input (overlapping 32-byte A rows, dx in the weights) vs the s-packed one:
    the same nonzero products in the same filter-row order, so pooled values and arg-max codes are expected bit for
    bit; both against PyTorch conv -> ReLU -> max-pool at the existing tolerance."""
    Ci, Co = 3, 32
    g = torch.Generator(device="cuda").manual_seed(41)
    x = torch.randint(0, 256, (B, H, H, 3), dtype=torch.uint8, device="cuda", generator=g)
    w = _bf(torch.randn(Co, Ci, 3, 3, device="cuda", generator=g) * 0.3)
    bias = torch.randn(Co, device="cuda", generator=g) * 0.1
    Xs, Xc = _spacked_and_compact(x, 0)
    Ws, Wc = _weights(w.float())
    Hp = (H - 2) // 2
    out0 = torch.zeros(B * Hp * Hp, Co, dtype=torch.bfloat16, device="cuda")
    am0 = torch.zeros(B * Hp * Hp, Co, dtype=torch.uint8, device="cuda")
    out1 = torch.full_like(out0, float("nan")); am1 = torch.full_like(am0, 255)
    ops.conv_fwd_pool_pair(Xs, Ws.view(-1), bias, out0, am0, B, H, H, 16, Co, True)
    ops.conv_fwd_pool_pair(Xc, Wc.view(-1), bias, out1, am1, B, H, H, 16, Co, True, 3, True)
    torch.cuda.synchronize()
    diff = (out0.float() - out1.float()).abs().max().item()
    flipped = int((am0 != am1).sum())
    print(f"compact vs s-packed forward B={B} H={H}: max |diff| {diff}, flipped codes {flipped}")
    ref = F.max_pool2d(F.relu(F.conv2d(_bf(x.float() / 255.0).float().permute(0, 3, 1, 2), w.float(), bias)), 2)
    for out in (out0, out1):
        got = out.view(B, Hp, Hp, Co).permute(0, 3, 1, 2).float()
        assert (got - ref).abs().max() <= 2.0 ** -7 * ref.abs().max() + 1e-3
    assert torch.equal(out0, out1) and torch.equal(am0, am1)


@pytest.mark.parametrize("B,H", [(4, 256), (3, 66), (2, 20), (5, 130)])
def test_compact_wgrad0_matches_spacked_gather_and_autograd(B, H):
    """Masked GEMMs on the compact input == the s-packed masked GEMMs == the FP32 gather == autograd through
    conv -> ReLU -> max-pool (with the forward kernel's own arg-max / activity decisions)."""
    Ci, Co = 3, 32
    g = torch.Generator(device="cuda").manual_seed(23)
    x = torch.randint(0, 256, (B, H, H, 3), dtype=torch.uint8, device="cuda", generator=g)
    w = _bf(torch.randn(Co, Ci, 3, 3, device="cuda", generator=g) * 0.3).float().requires_grad_(True)
    bias = (torch.randn(Co, device="cuda", generator=g) * 0.1).requires_grad_(True)
    Xs, Xc = _spacked_and_compact(x, 0)
    Ws, _ = _weights(w.detach())
    P = B * H * H
    Hp = (H - 2) // 2
    out = torch.zeros(B * Hp * Hp, Co, dtype=torch.bfloat16, device="cuda")
    amax = torch.zeros(B * Hp * Hp, Co, dtype=torch.uint8, device="cuda")
    ops.conv_fwd_pool(Xs[:P], Ws.view(-1), bias.detach(), out, amax, B, H, H, 16, Co, True)
    gp = _bf(torch.randn(B, Co, Hp, Hp, device="cuda", generator=g))
    gflat = gp.permute(0, 2, 3, 1).contiguous().view(-1, Co)
    d_cpt = torch.zeros(9 * 16 + 1, Co, dtype=torch.float32, device="cuda")
    d_mma = torch.zeros_like(d_cpt)
    d_gat = torch.zeros_like(d_cpt)
    ops.wgrad0_gather(Xc, gflat, amax, d_cpt.view(-1), B, H, H, True, 3, True)
    ops.wgrad0_gather(Xs, gflat, amax, d_mma.view(-1), B, H, H, True)
    ops.wgrad0_gather(Xs, gflat, amax, d_gat.view(-1), B, H, H, False)
    torch.cuda.synchronize()
    scale = d_gat.abs().max()
    # same products, fp32 sums in another order (the two column parities are added when the warp tiles are parked)
    assert (d_cpt - d_mma).abs().max() <= 2e-5 * scale + 1e-5
    assert (d_cpt - d_gat).abs().max() <= 2e-5 * scale + 1e-5
    assert float(d_cpt[:144].view(9, 16, Co)[:, Ci:, :].abs().max()) == 0.0
    xin = _bf(x.float() / 255.0).float().permute(0, 3, 1, 2)
    conv = F.conv2d(xin, w, bias)
    am = amax.view(B, Hp, Hp, Co).permute(0, 3, 1, 2).long()
    dy, dx, act = (am >> 1) & 1, am & 1, (am & 4) != 0
    idx = (2 * torch.arange(Hp, device="cuda").view(1, 1, Hp, 1) + dy) * (H - 2) + 2 * torch.arange(Hp, device="cuda").view(1, 1, 1, Hp) + dx
    pooled = conv.flatten(2).gather(2, idx.flatten(2)).view(B, Co, Hp, Hp) * act
    pooled.backward(gp.float())
    got_w = d_cpt[:144].view(9, 16, Co)[:, :Ci, :].permute(2, 1, 0).reshape(Co, Ci, 3, 3)
    assert (got_w - w.grad).abs().max() <= 2e-3 * w.grad.abs().max() + 1e-3
    assert (d_cpt[144] - bias.grad).abs().max() <= 2e-3 * bias.grad.abs().max() + 1e-3


def test_engine_gradients_match_autograd_on_the_compact_layout():
    """Whole medical CNN with the compact layer-1 input selected (the RGB default): engine forward/backward vs
    PyTorch autograd on the same weights, with the limits of the 16-channel engine test."""
    from hefl_b200.config import FLConfig
    from hefl_b200.models import ParamPack, create_model
    from hefl_b200.ops.conv_engine import MedCNNEngine

    torch.manual_seed(0)
    cfg = FLConfig(model="medcnn", batch_size=8, image_size=256)
    dev = torch.device("cuda")
    model = create_model("medcnn").to(dev)
    pack = ParamPack(model)
    pack.flat.copy_(pack.flat.to(torch.bfloat16).float())
    eng = MedCNNEngine(model, pack, cfg, dev)
    assert eng.compact0
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randint(0, 256, (8, 256, 256, 3), dtype=torch.uint8, device="cuda", generator=g)
    y = torch.randint(0, 2, (8,), device="cuda", generator=g)
    out = torch.zeros(2, device="cuda")
    eng.train_step(x, y, out, augment=False)
    torch.cuda.synchronize()
    g_eng = pack.grad.clone()
    pack.grad.zero_()

    class RoundBF(torch.autograd.Function):
        @staticmethod
        def forward(ctx, t):
            return t.to(torch.bfloat16).float()

        @staticmethod
        def backward(ctx, gr):
            return gr.to(torch.bfloat16).float()

    h = (x.float() / 255.0).to(torch.bfloat16).float().permute(0, 3, 1, 2)
    for l, conv in enumerate(model.convs):
        h = RoundBF.apply(F.max_pool2d(F.relu(conv(h)), 2))
        e = eng.X[l + 1].view(8, h.shape[2], h.shape[3], h.shape[1]).permute(0, 3, 1, 2).float()
        assert (e - h).abs().max() <= 2.0 ** -7 * h.abs().max()
    h = h.permute(0, 2, 3, 1).flatten(1)
    for fc in model.fcs[:-1]:
        h = F.relu(fc(h))
    loss = F.cross_entropy(model.fcs[-1](h), y)
    loss.backward()
    assert abs(float(out[0]) - float(loss.detach())) < 2e-3
    for key, shape, off, n in pack.entries:
        a, b = g_eng[off:off + n], pack.grad[off:off + n]
        rel = (a - b).abs().max().item() / (b.abs().max().item() + 1e-6)
        cos = F.cosine_similarity(a, b, dim=0).item() if b.norm() > 0 else 1.0
        lim = 0.16 if key.startswith("c_0_") else (0.10 if key.startswith(("c_2_", "c_4_", "c_13_")) else 0.06)
        assert cos > 0.995 and rel < lim, (key, rel, cos)
    assert float(eng.dW32.abs().max()) == 0.0


def _trainer_run(use_graph, compact, steps=4):
    from hefl_b200.config import FLConfig
    from hefl_b200.fl.trainer import LocalTrainer
    from hefl_b200.models import ParamPack, create_model

    torch.manual_seed(1)
    cfg = FLConfig(model="medcnn", batch_size=8, nn_backend="tcgen05")
    dev = torch.device("cuda")
    model = create_model("medcnn").to(dev)
    pack = ParamPack(model)
    tr = LocalTrainer(model, pack, cfg, dev, backend="tcgen05", use_graph=use_graph, augment=True)
    if not compact:
        tr.engine._wgrad0_mma = False        # -> the s-packed 16-channel layer 1 (same kernels, 32 bytes per pixel)
        tr.engine.after_restore()
    assert tr.engine.compact0 == compact
    g = torch.Generator(device="cuda").manual_seed(3)
    losses = []
    for _ in range(steps):
        x = torch.randint(0, 256, (8, 256, 256, 3), dtype=torch.uint8, device="cuda", generator=g)
        y = torch.randint(0, 2, (8,), device="cuda", generator=g)
        losses.append(tr.train_step(x, y).clone())
    torch.cuda.synchronize()
    return pack.flat.clone(), torch.stack(losses)


def test_compact_graph_replay_equals_eager_and_tracks_the_16_channel_layout():
    """Several augmented steps: the captured graph and the eager step give the same bits on the compact layout; the
    16-channel layout differs only by the order of the layer-1 weight-gradient sums."""
    flat_g, loss_g = _trainer_run(True, True)
    flat_e, loss_e = _trainer_run(False, True)
    assert torch.equal(flat_g, flat_e) and torch.equal(loss_g, loss_e)
    flat_s, loss_s = _trainer_run(True, False)
    assert (flat_g - flat_s).abs().max() < 2e-3
    assert (loss_g - loss_s).abs().max() < 5e-3

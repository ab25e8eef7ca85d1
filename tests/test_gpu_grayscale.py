"""GPU tests of grayscale (one-channel) input on the hand-written engine: the rs-packed layer-1 layout (channel
3r + s = pixel (h + r, w + s)), its pre-processing, forward kernels (pair-row and tap-GEMM), masked-GEMM weight
gradient and weight re-layout, then the whole engine, training and one encrypted FedAvg round."""
import pytest
import torch
import torch.nn.functional as F

from hefl_b200 import _ext

pytestmark = pytest.mark.gpu
ops = _ext.ops()
Co = 32


def _bf(x):
    return x.to(torch.bfloat16)


def _gray(B, H, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, (B, H, H, 1), dtype=torch.uint8, device="cuda", generator=g), g


def _prep(x, spack, seed=0, theta=None):
    """layer-1 input with 8 pixels of slack (as the engine allocates it)"""
    B, H, W, _ = x.shape
    P = B * H * W
    X = torch.zeros(P + 8, 16, dtype=torch.bfloat16, device="cuda")
    ops.preprocess_u8(x, theta, X[:P], seed, None, spack)
    return X


def _w_rs(w):
    """[Co,1,3,3] -> rs-packed forward weights [1][Co][16], k = 3r + s"""
    Wp = torch.zeros(1, w.shape[0], 16, dtype=torch.bfloat16, device="cuda")
    Wp[0, :, :9] = w.reshape(w.shape[0], 9).to(torch.bfloat16)
    return Wp


def _w_plain(w):
    """[Co,1,3,3] -> plain 9-tap forward weights [9][Co][16], channel 0 only"""
    W9 = torch.zeros(9, w.shape[0], 16, dtype=torch.bfloat16, device="cuda")
    W9[:, :, :1] = w.permute(2, 3, 0, 1).reshape(9, w.shape[0], 1).to(torch.bfloat16)
    return W9


def _check_rs_neighbours(xv, H):
    """channel 3r + s of pixel (h, w) == channel 0 of pixel (h + r, w + s), exact zeros past the edges"""
    for r in range(3):
        for s in range(3):
            k = 3 * r + s
            assert torch.equal(xv[:, : H - r, : H - s, k], xv[:, r:, s:, 0]), (r, s)
            assert not xv[:, H - r:, :, k].any() and not xv[:, :, H - s:, k].any(), (r, s)
    assert float(xv[..., 9:].abs().max()) == 0.0


# ------------------------------------------------------------------ 1. pre-processing
@pytest.mark.parametrize("H", [256, 70])
def test_preprocess_gray_rs_and_plain_layouts(H):
    B = 2
    x, _ = _gray(B, H, 51)
    P = B * H * H
    ref = _bf(x[..., 0].float() / 255.0).float()                     # [B,H,H]
    xv = _prep(x, True)[:P].view(B, H, H, 16).float()
    for r in range(3):
        for s in range(3):
            exp = torch.zeros(B, H, H, device="cuda")
            exp[:, : H - r, : H - s] = ref[:, r:, s:]
            assert torch.equal(xv[..., 3 * r + s], exp), (r, s)
    _check_rs_neighbours(xv, H)
    pv = _prep(x, False)[:P].view(B, H, H, 16).float()
    assert torch.equal(pv[..., 0], ref)
    assert float(pv[..., 1:].abs().max()) == 0.0


def test_preprocess_gray_augmented_matches_grid_sample_and_rgb_keying():
    B, H = 4, 64
    x, _ = _gray(B, H, 52)
    P = B * H * H
    theta = torch.tensor([[[0.9, 0.05, 0.0], [0.0, 1.1, 0.0]]], device="cuda").repeat(B, 1, 1)
    theta[1, 0, 0] *= -1
    xv = _prep(x, True, theta=theta.contiguous())[:P].view(B, H, H, 16).float()
    xr = (x.float() / 255.0).permute(0, 3, 1, 2)
    grid = F.affine_grid(theta, list(xr.shape), align_corners=False)
    ref = F.grid_sample(xr, grid, mode="bilinear", padding_mode="border", align_corners=False)[:, 0]
    assert (xv[..., 0] - ref).abs().max() < 1e-2                      # as test_preprocess_matches_grid_sample
    _check_rs_neighbours(xv, H)
    # in-kernel Philox augmentation: the packed and plain layouts agree on channel 0 bit for bit, and the draw is keyed
    # as for RGB: the same image stored as RGB is warped the same way (the two kernels may round the bilinear weights
    # differently in the last fp32 bit, so a rare pixel lands on the neighbouring bf16 value)
    seed = 0x1234567
    gv = _prep(x, True, seed=seed)[:P].view(B, H, H, 16).float()
    _check_rs_neighbours(gv, H)
    pv = _prep(x, False, seed=seed)[:P].view(B, H, H, 16).float()
    assert torch.equal(gv[..., 0], pv[..., 0])
    rgb = _prep(x.repeat(1, 1, 1, 3).contiguous(), False, seed=seed)[:P].view(B, H, H, 16).float()
    d = (pv[..., 0] - rgb[..., 0]).abs()
    print("gray vs RGB keyed augmentation: max diff", float(d.max()), "share of differing pixels", float((d > 0).float().mean()))
    assert float(d.max()) < 1e-2 and float((d > 0).float().mean()) < 0.05
    assert not torch.equal(gv[..., 0], _prep(x, True)[:P].view(B, H, H, 16).float()[..., 0])   # it did warp


# ------------------------------------------------------------------ 2. forward
@pytest.mark.parametrize("B,H", [(2, 256), (3, 70), (1, 66), (2, 191), (3, 62), (2, 20)])
def test_rs_forward_pair_and_tap_gemm_match_torch_and_the_plain_layout(B, H):
    """rs-packed layer 1: one GEMM per accumulator. H = 191 (odd) only runs on the tap-GEMM column tiles, H <= 64 on
    its row-packed tiles; wherever the pair-row kernel applies too, both agree bit for bit."""
    x, g = _gray(B, H, 61)
    w = _bf(torch.randn(Co, 1, 3, 3, device="cuda", generator=g) * 0.5)
    bias = torch.randn(Co, device="cuda", generator=g) * 0.1
    P, Hp = B * H * H, (H - 2) // 2
    X = _prep(x, True)
    out = torch.zeros(B * Hp * Hp, Co, dtype=torch.bfloat16, device="cuda")
    am = torch.zeros(B * Hp * Hp, Co, dtype=torch.uint8, device="cuda")
    ops.conv_fwd_pool(X[:P], _w_rs(w).view(-1), bias, out, am, B, H, H, 16, Co, True, 1)
    ref = F.max_pool2d(F.relu(F.conv2d(_bf(x.float() / 255.0).float().permute(0, 3, 1, 2), w.float(), bias)), 2)
    got = out.view(B, Hp, Hp, Co).permute(0, 3, 1, 2).float()
    bound = 2.0 ** -7 * ref.abs().max() + 1e-3
    assert (got - ref).abs().max() <= bound
    if H % 2 == 0 and Hp <= 128:
        out_p, am_p = torch.zeros_like(out), torch.zeros_like(am)
        ops.conv_fwd_pool_pair(X, _w_rs(w).view(-1), bias, out_p, am_p, B, H, H, 16, Co, True, 1)
        torch.cuda.synchronize()
        assert torch.equal(out, out_p)
        assert torch.equal(am, am_p)
    # the 9-tap kernel on the plain one-channel layout
    X9 = _prep(x, False)
    out9, am9 = torch.zeros_like(out), torch.zeros_like(am)
    ops.conv_fwd_pool(X9[:P], _w_plain(w).view(-1), bias, out9, am9, B, H, H, 16, Co, False, 1)
    torch.cuda.synchronize()
    assert (out.float() - out9.float()).abs().max() <= bound
    assert ((am & 4) == (am9 & 4)).float().mean() > 0.999


def test_unsupported_channel_counts_are_refused():
    x, _ = _gray(1, 20, 1)
    X = _prep(x, True)
    out = torch.zeros(81, Co, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="in_channels"):
        ops.conv_fwd_pool(X[:400], torch.zeros(9 * Co * 16, dtype=torch.bfloat16, device="cuda"),
                          torch.zeros(Co, device="cuda"), out, None, 1, 20, 20, 16, Co, True, 2)
    with pytest.raises(RuntimeError, match=r"\[B,H,W,3\] or \[B,H,W,1\]"):
        ops.preprocess_u8(torch.zeros(1, 20, 20, 2, dtype=torch.uint8, device="cuda"), None, X[:400], 0, None, True)


# ------------------------------------------------------------------ 3. layer-1 weight gradient
@pytest.mark.parametrize("B,H", [(4, 256), (3, 66), (2, 20), (5, 130)])
def test_rs_wgrad0_masked_gemm_matches_gather_and_autograd(B, H):
    """Masked GEMMs with M = 16 on the rs-packed input == the FP32-pipe gather on the same buffers (which reads
    channel 0 of the shifted pixels) == autograd with the forward kernel's own arg-max and activity decisions."""
    x, g = _gray(B, H, 71)
    w = _bf(torch.randn(Co, 1, 3, 3, device="cuda", generator=g) * 0.5).float().requires_grad_(True)
    bias = (torch.randn(Co, device="cuda", generator=g) * 0.1).requires_grad_(True)
    P, Hp = B * H * H, (H - 2) // 2
    X = _prep(x, True)
    out = torch.zeros(B * Hp * Hp, Co, dtype=torch.bfloat16, device="cuda")
    amax = torch.zeros(B * Hp * Hp, Co, dtype=torch.uint8, device="cuda")
    ops.conv_fwd_pool(X[:P], _w_rs(w.detach()).view(-1), bias.detach(), out, amax, B, H, H, 16, Co, True, 1)
    gp = _bf(torch.randn(B, Co, Hp, Hp, device="cuda", generator=g))
    gflat = gp.permute(0, 2, 3, 1).contiguous().view(-1, Co)
    d_mma = torch.zeros(9 * 16 + 1, Co, dtype=torch.float32, device="cuda")
    d_gat = torch.zeros_like(d_mma)
    ops.wgrad0_gather(X, gflat, amax, d_mma.view(-1), B, H, H, True, 1)
    ops.wgrad0_gather(X, gflat, amax, d_gat.view(-1), B, H, H, False, 1)
    torch.cuda.synchronize()
    used = torch.zeros(9 * 16 + 1, dtype=torch.bool, device="cuda")
    used[0:144:16] = True
    used[144] = True                                                   # bias row
    scale = d_gat[used].abs().max()
    assert (d_mma[used] - d_gat[used]).abs().max() <= 2e-5 * scale + 1e-5
    assert float(d_mma[~used].abs().max()) == 0.0                     # rows tap*16 + 1..15 stay zero
    xin = _bf(x.float() / 255.0).float().permute(0, 3, 1, 2)
    conv = F.conv2d(xin, w, bias)
    am = amax.view(B, Hp, Hp, Co).permute(0, 3, 1, 2).long()
    dy, dx, act = (am >> 1) & 1, am & 1, (am & 4) != 0
    idx = (2 * torch.arange(Hp, device="cuda").view(1, 1, Hp, 1) + dy) * (H - 2) + 2 * torch.arange(Hp, device="cuda").view(1, 1, 1, Hp) + dx
    pooled = conv.flatten(2).gather(2, idx.flatten(2)).view(B, Co, Hp, Hp) * act
    pooled.backward(gp.float())
    got_w = d_mma[:144].view(9, 16, Co)[:, 0, :].permute(1, 0).reshape(Co, 1, 3, 3)
    assert (got_w - w.grad).abs().max() <= 2e-3 * w.grad.abs().max() + 1e-3
    assert (d_mma[144] - bias.grad).abs().max() <= 2e-3 * bias.grad.abs().max() + 1e-3


# ------------------------------------------------------------------ 4. whole engine
def _gray_engine(batch):
    from hefl_b200.config import FLConfig
    from hefl_b200.models import ParamPack, create_model
    from hefl_b200.ops.conv_engine import MedCNNEngine

    torch.manual_seed(0)
    cfg = FLConfig(model="medcnn", batch_size=batch, image_size=256, in_channels=1)
    dev = torch.device("cuda")
    model = create_model("medcnn", in_channels=1).to(dev)
    pack = ParamPack(model)
    pack.flat.copy_(pack.flat.to(torch.bfloat16).float())
    return model, pack, MedCNNEngine(model, pack, cfg, dev)


@pytest.mark.parametrize("packed,gather", [(True, True), (True, False), (False, True), (False, False)])
def test_gray_engine_gradients_match_autograd(packed, gather):
    """MedCNN(in_channels=1) on the engine (rs-packed or plain layer 1, masked-GEMM / gather or un-pool + wgrad
    layer-1 weight gradient) vs PyTorch autograd on the same bf16-rounded weights."""
    model, pack, eng = _gray_engine(8)
    assert eng.spack0 and eng.p0 == 320
    eng.gather_wgrad0 = gather
    if not packed:
        eng.spack0 = False
        eng.after_restore()
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randint(0, 256, (8, 256, 256, 1), dtype=torch.uint8, device="cuda", generator=g)
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
    g_ref = pack.grad.clone()
    assert abs(float(out[0]) - float(loss.detach())) < 2e-3
    rels = {}
    for key, shape, off, n in pack.entries:
        a, b = g_eng[off:off + n], g_ref[off:off + n]
        rel = (a - b).abs().max().item() / (b.abs().max().item() + 1e-6)
        cos = F.cosine_similarity(a, b, dim=0).item() if b.norm() > 0 else 1.0
        rels[key] = (round(rel, 4), round(cos, 5))
    print("gray engine vs autograd, (max rel err, cosine) per tensor:", rels)
    # the bounds of test_engine_gradients_match_autograd (RGB). Measured on an H100, the same for all four variants to
    # the digits shown: max-norm relative error 0.056 / 0.062 (first convolution, weights / bias), 0.045 / 0.040,
    # 0.021 / 0.021, 0.015 / 0.015, 0.026 / 0.016, 0.023 for the six convolutions, < 0.002 for the dense layers;
    # cosine 0.9983 (first convolution) ... 1.0000
    for key, (rel, cos) in rels.items():
        lim = 0.16 if key.startswith("c_0_") else (0.10 if key.startswith(("c_2_", "c_4_", "c_13_")) else 0.06)
        assert cos > 0.995 and rel < lim, (key, rel, cos, rels)
    assert float(eng.dW32.abs().max()) == 0.0


def test_gray_engine_rejects_other_channel_counts():
    from hefl_b200.config import FLConfig
    from hefl_b200.models import ParamPack, create_model
    from hefl_b200.ops.conv_engine import MedCNNEngine

    model = create_model("medcnn", in_channels=2).cuda()
    with pytest.raises(ValueError, match="1- or 3-channel"):
        MedCNNEngine(model, ParamPack(model), FLConfig(model="medcnn", batch_size=8, in_channels=2), torch.device("cuda"))


# ------------------------------------------------------------------ 5. training
def _setup(backend, dtype, use_graph, n_img=256, seed=5):
    from hefl_b200.config import FLConfig
    from hefl_b200.fl.data import BatchFeeder, SyntheticImageDataset
    from hefl_b200.fl.trainer import LocalTrainer
    from hefl_b200.models import ParamPack, create_model

    dev = torch.device("cuda")
    torch.manual_seed(seed)
    cfg = FLConfig(model="medcnn", batch_size=32, nn_backend=backend, dtype=dtype, lr=1e-3, in_channels=1)
    model = create_model("medcnn", in_channels=1).to(dev)
    pack = ParamPack(model)
    tr = LocalTrainer(model, pack, cfg, dev, backend=backend, use_graph=use_graph, augment=False)
    ds = SyntheticImageDataset(n_img, 256, 1, 2, seed=11)
    feed = BatchFeeder(ds, range(0, n_img), 32, dev, shuffle=True, seed=3)
    return tr, pack, feed


def _layouts_follow_weights(tr):
    """After the update (the layers above layer 1 on the side stream, layer 1 in the tail), the bf16 shadow and both
    tensor-core weight layouts hold exactly the fp32 weights."""
    eng = tr.engine
    assert torch.equal(eng.shadow, tr.pack.trainable().to(torch.bfloat16))
    Wf, Wd = torch.zeros_like(eng.Wf), torch.zeros_like(eng.Wd)
    tr.ops.conv_weight_relayout(eng.shadow, eng.table, Wf, Wd, 0, -1, eng.spack0, eng.compact0)
    assert torch.equal(eng.Wf, Wf) and torch.equal(eng.Wd, Wd)


def test_three_gray_epochs_of_the_bf16_engine_track_fp32_pytorch():
    eng, pack_e, feed_e = _setup("tcgen05", "bf16", True)
    assert eng.engine.spack0
    ref, pack_r, feed_r = _setup("cudnn", "fp32", False)
    assert torch.equal(pack_e.flat, pack_r.flat)
    h_e = eng.fit(feed_e, None, 3, early_stopping=None, reduce_lr_patience=None)
    h_r = ref.fit(feed_r, None, 3, early_stopping=None, reduce_lr_patience=None)
    print("gray engine :", [(round(s.loss, 4), round(s.accuracy, 3)) for s in h_e])
    print("gray fp32   :", [(round(s.loss, 4), round(s.accuracy, 3)) for s in h_r])
    assert h_r[-1].loss < h_r[0].loss
    assert h_e[-1].loss < h_e[0].loss
    assert abs(h_e[-1].loss - h_r[-1].loss) <= max(0.05 * h_r[-1].loss, 0.02)
    assert abs(h_e[-1].accuracy - h_r[-1].accuracy) <= 0.02
    assert abs(h_e[0].loss - h_r[0].loss) <= 0.05 * h_r[0].loss
    assert abs(h_e[0].accuracy - h_r[0].accuracy) <= 0.15
    # measured on an H100: losses (0.6471, 0.1968, 0.0001) vs fp32 (0.6432, 0.1753, 0.0006), accuracy 1.0 / 1.0 from
    # epoch 2 on both, trained weights cosine 0.9984
    cos = F.cosine_similarity(pack_e.flat, pack_r.flat, dim=0).item()
    print("gray trained weights cosine:", cos)
    assert cos > 0.99


def test_gray_graph_and_pipeline_path_equals_the_eager_path_over_eight_steps():
    a, pack_a, feed_a = _setup("tcgen05", "bf16", True)
    b, pack_b, feed_b = _setup("tcgen05", "bf16", False)
    a.fit(feed_a, None, 1, early_stopping=None, reduce_lr_patience=None)
    b.fit(feed_b, None, 1, early_stopping=None, reduce_lr_patience=None)
    torch.cuda.synchronize()
    assert int(a.step_t.item()) == int(b.step_t.item()) == 8
    _layouts_follow_weights(a)
    _layouts_follow_weights(b)
    d = (pack_a.flat - pack_b.flat).abs()
    print("gray graph vs eager: max", float(d.max()), "mean", float(d.mean()))
    assert float(d.max()) <= 2 * 8 * 1e-3
    assert float(d.mean()) < 6e-4
    assert F.cosine_similarity(pack_a.flat, pack_b.flat, dim=0).item() > 0.9995


# ------------------------------------------------------------------ 6. end to end
def test_gray_encrypted_fedavg_round():
    """One client, one round: train on the engine, encrypt, aggregate, decrypt; CKKS error as for RGB input."""
    from hefl_b200.config import FLConfig
    from hefl_b200.fl import FederatedRunner

    errs = {}
    for c in (1, 3):
        cfg = FLConfig(model="medcnn", local_epochs=1, steps_per_epoch=2, val_steps=1, batch_size=32, in_channels=c,
                       nn_backend="tcgen05", transport="fused", device="cuda", debug_precision=True)
        run = FederatedRunner(cfg, device=torch.device("cuda"))
        assert run.trainer.engine is not None and run.trainer.engine.Ci[0] == c
        w0 = run.pack.flat.clone()
        rec = run.run_round(check=True)
        torch.cuda.synchronize()
        assert rec["loss"] is not None and rec["loss"] == rec["loss"]
        assert not torch.equal(run.pack.flat, w0)                       # it trained
        errs[c] = rec["ckks_max_abs_err"]
    print("ckks_max_abs_err gray / rgb:", errs)          # measured on an H100: 7.5e-8 / 6.7e-8
    assert errs[1] < 1e-3 and errs[1] <= 10 * errs[3] + 1e-9

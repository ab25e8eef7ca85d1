"""Non-IID clients on the H100: the FedProx term of the Adam kernels (adam_kernel<true>, fused_update_kernel<true>),
the engine trained with it, its pull towards the round's global model, sample-weighted encrypted FedAvg on CUDA,
and the multi-GPU round on the fused transport."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEDCNN_PARAMS = 222722


def _ops():
    from hefl_b200 import _ext
    return _ext.ops()


def _adam64(p, g, m, v, anchor, mu, t, lr=1e-3, decay=1e-4, b1=0.9, b2=0.999, eps=1e-7):
    p, g, m, v, a = (x.double().cpu() for x in (p, g, m, v, anchor))
    g = g + mu * (p - a)
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    alpha = lr / (1 + decay * (t - 1)) * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
    return p - alpha * m / (v.sqrt() + eps)


# ------------------------------------------------------------------ 1. adam_step_ with the anchor
@pytest.mark.parametrize("n", [MEDCNN_PARAMS, 1001])
def test_prox_adam_kernel_matches_cpu_twin_and_float64(n):
    ops = _ops()
    gen = torch.Generator().manual_seed(n)
    p0, g0 = torch.randn(n, generator=gen), torch.randn(n, generator=gen) * 1e-2
    m0, v0 = torch.randn(n, generator=gen) * 1e-3, torch.rand(n, generator=gen) * 1e-4
    anchor = p0 + torch.randn(n, generator=gen) * 0.05
    mu, t = 0.05, 4

    def run(dev, anc, mu_):
        p, g, m, v = (x.clone().to(dev) for x in (p0, g0, m0, v0))
        sh = torch.zeros(n, dtype=torch.bfloat16, device=dev)
        step = torch.tensor([t], dtype=torch.int64, device=dev)
        ops.adam_step_(p, g, m, v, sh, step, None, 1e-3, 1e-4, 0.9, 0.999, 1e-7,
                       anc.to(dev) if anc is not None else None, mu_)
        torch.cuda.synchronize()
        assert float(g.abs().max()) == 0.0
        return p.cpu(), m.cpu(), v.cpu(), sh.cpu()

    gpu = run("cuda", anchor, mu)
    cpu = run("cpu", anchor, mu)
    ref = _adam64(p0, g0, m0, v0, anchor, mu, t)
    e_cpu = float((gpu[0] - cpu[0]).abs().max())
    e_ref = float((gpu[0].double() - ref).abs().max())
    # measured on an H100: 1.2e-7 / 2.2e-7 at 222,722 elements, 0 / 1.2e-7 at 1001 (unit-scale weights)
    print(f"n={n}: PROX adam |gpu - cpu twin| {e_cpu:.3g}, |gpu - float64| {e_ref:.3g}")
    assert e_cpu < 1e-6 and e_ref < 1e-6
    assert torch.equal(gpu[3], gpu[0].to(torch.bfloat16))               # shadow of the new weights
    # mu = 0 with an anchor runs adam_kernel<false>: bit-identical to no anchor
    a, b = run("cuda", anchor, 0.0), run("cuda", None, 0.0)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert not torch.equal(gpu[0], b[0])


# ------------------------------------------------------------------ 2. fused_update with the anchor
def test_prox_fused_update_matches_finalize_adam_relayout():
    """fused_update(anchor) == conv_grad_finalize -> adam_step_(anchor) -> conv_weight_relayout on the same
    gradients, to the last fp32 bits (the op-level twin of test_fused_update_matches_separate_path)."""
    from hefl_b200.config import FLConfig
    from hefl_b200.fl.trainer import LocalTrainer
    from hefl_b200.models import ParamPack, create_model

    ops = _ops()
    torch.manual_seed(1)
    dev = torch.device("cuda")
    cfg = FLConfig(model="medcnn", batch_size=8, nn_backend="tcgen05")
    model = create_model("medcnn").to(dev)
    pack = ParamPack(model)
    tr = LocalTrainer(model, pack, cfg, dev, backend="tcgen05", use_graph=False, augment=False)
    eng = tr.engine
    eng.spack0 = False                     # the one-launch update writes the plain 9-tap layer-1 layout
    eng.after_restore()
    g = torch.Generator(device="cuda").manual_seed(7)
    nt = pack.n_trainable
    dW = torch.randn(eng.dW32.shape, device=dev, generator=g) * 1e-2
    grad = torch.randn(nt, device=dev, generator=g) * 1e-2
    m0 = torch.randn(nt, device=dev, generator=g) * 1e-3
    v0 = torch.rand(nt, device=dev, generator=g) * 1e-4
    anchor = pack.trainable() + torch.randn(nt, device=dev, generator=g) * 0.05
    step = torch.tensor([5], dtype=torch.int64, device=dev)
    lr_scale = torch.ones(1, device=dev)
    flat0 = pack.flat.clone()

    def state(m, v):    # the one-launch update reads the conv gradients from dW32 and clears only the dense tail
        return [pack.flat.clone(), m.clone(), v.clone(), eng.shadow.clone(), eng.Wf.clone(), eng.Wd.clone(),
                pack.grad[eng.dense_off:].clone(), eng.dW32.clone()]

    def fused(mu):
        pack.flat.copy_(flat0); eng.after_restore(); eng.dW32.copy_(dW); pack.grad.copy_(grad)
        m, v = m0.clone(), v0.clone()
        ops.fused_update(eng.dW32, eng.table, pack.flat, pack.grad, m, v, eng.shadow, eng.Wf, eng.Wd, step, lr_scale,
                         1e-3, 1e-4, 0.9, 0.999, 1e-7, eng.dense_off, nt, anchor, mu)
        torch.cuda.synchronize()
        return state(m, v)

    def separate(mu):
        pack.flat.copy_(flat0); eng.after_restore(); eng.dW32.copy_(dW); pack.grad.copy_(grad)
        m, v = m0.clone(), v0.clone()
        ops.conv_grad_finalize(eng.dW32, eng.table, pack.grad)
        ops.adam_step_(pack.trainable(), pack.grad, m, v, eng.shadow, step, lr_scale, 1e-3, 1e-4, 0.9, 0.999, 1e-7,
                       anchor, mu)
        ops.conv_weight_relayout(eng.shadow, eng.table, eng.Wf, eng.Wd, 0, -1, False)
        torch.cuda.synchronize()
        return state(m, v)

    # The two kernels evaluate the same Adam expressions, but nvcc contracts them into FMAs differently (m and v of
    # adam_kernel<false> and fused_update_kernel<false> already differ that way, unchanged by the FedProx template),
    # so the fp32 results may differ in the last bit or two and a bf16 copy may round to the neighbouring value.
    # An m that cancels (beta1*m ~ -(1-beta1)*g) keeps the absolute error of its ~1e-3 terms, hence the floors.
    # Measured on H100s: max |diff| 0 or flat 7.5e-9, m 4.7e-10, v 7.3e-12, bf16 copies 0, with mu = 0.05 and 0.
    names = ["flat", "m", "v", "shadow", "Wf", "Wd", "grad", "dW32"]
    for mu in (0.05, 0.0):
        a, b = fused(mu), separate(mu)
        diffs = {k: float((x.float() - y.float()).abs().max()) for k, x, y in zip(names, a, b)}
        print(f"mu={mu}: fused vs separate max |diff|", diffs)
        # one bf16 ulp, or a few fp32 ulps; floors: 1e-6 of an Adam step (~lr) for the weights, ~8 ulps of the
        # terms of m and v
        floor = {"flat": 1e-9, "m": 1e-9, "v": 1e-13}
        for k, x, y in zip(names, a, b):
            x, y = x.float(), y.float()
            ulps = 2.0 ** -7 if k in ("shadow", "Wf", "Wd") else 2.0 ** -21
            tol = ulps * torch.maximum(x.abs(), y.abs()) + floor.get(k, 0.0)
            assert bool(((x - y).abs() <= tol).all()), (k, diffs)
    moved = (fused(0.05)[0] - fused(0.0)[0]).abs().max()
    assert float(moved) > 1e-6                         # the proximal term itself is far above that rounding


# ------------------------------------------------------------------ 3. the engine with FedProx
def _setup(backend, dtype, use_graph, mu, n_img=256, seed=5):
    from hefl_b200.config import FLConfig
    from hefl_b200.fl.data import BatchFeeder, SyntheticImageDataset
    from hefl_b200.fl.trainer import LocalTrainer
    from hefl_b200.models import ParamPack, create_model

    dev = torch.device("cuda")
    torch.manual_seed(seed)
    cfg = FLConfig(model="medcnn", batch_size=32, nn_backend=backend, dtype=dtype, lr=1e-3, fedprox_mu=mu)
    model = create_model("medcnn").to(dev)
    pack = ParamPack(model)
    tr = LocalTrainer(model, pack, cfg, dev, backend=backend, use_graph=use_graph, augment=False)
    ds = SyntheticImageDataset(n_img, 256, 3, 2, seed=11)
    feed = BatchFeeder(ds, range(0, n_img), 32, dev, shuffle=True, seed=3)
    return tr, pack, feed


def test_three_prox_epochs_of_the_bf16_engine_track_fp32_pytorch():
    eng, pack_e, feed_e = _setup("tcgen05", "bf16", True, 0.05)
    ref, pack_r, feed_r = _setup("cudnn", "fp32", False, 0.05)
    assert eng.anchor is not None and ref.anchor is not None
    assert torch.equal(pack_e.flat, pack_r.flat)
    h_e = eng.fit(feed_e, None, 3, early_stopping=None, reduce_lr_patience=None)
    h_r = ref.fit(feed_r, None, 3, early_stopping=None, reduce_lr_patience=None)
    print("prox engine:", [(round(s.loss, 4), round(s.accuracy, 3)) for s in h_e])
    print("prox fp32  :", [(round(s.loss, 4), round(s.accuracy, 3)) for s in h_r])
    assert h_r[-1].loss < h_r[0].loss
    assert h_e[-1].loss < h_e[0].loss
    assert abs(h_e[-1].loss - h_r[-1].loss) <= max(0.05 * h_r[-1].loss, 0.02)
    assert abs(h_e[-1].accuracy - h_r[-1].accuracy) <= 0.02
    assert abs(h_e[0].loss - h_r[0].loss) <= 0.05 * h_r[0].loss
    assert abs(h_e[0].accuracy - h_r[0].accuracy) <= 0.15
    # measured on an H100: losses (0.648, 0.1975, 0.0002) vs fp32 (0.652, 0.205, 0.0003), accuracy 1.0 / 1.0 from
    # epoch 2 on both, trained weights cosine 0.9984
    cos = F.cosine_similarity(pack_e.flat, pack_r.flat, dim=0).item()
    print("prox trained weights cosine:", cos)
    assert cos > 0.99


def test_prox_graph_and_pipeline_path_equals_the_eager_path_over_eight_steps():
    a, pack_a, feed_a = _setup("tcgen05", "bf16", True, 0.05)
    b, pack_b, feed_b = _setup("tcgen05", "bf16", False, 0.05)
    a.fit(feed_a, None, 1, early_stopping=None, reduce_lr_patience=None)
    b.fit(feed_b, None, 1, early_stopping=None, reduce_lr_patience=None)
    torch.cuda.synchronize()
    assert int(a.step_t.item()) == int(b.step_t.item()) == 8
    assert torch.equal(a.anchor, b.anchor)
    # same bound as the plain engine's graph-vs-eager test, whose only source of difference is the order of fp32
    # atomics in the weight gradients (measured on an H100 with mu = 0.05: max 0.0, the two paths were bit-identical)
    d = (pack_a.flat - pack_b.flat).abs()
    print("prox graph vs eager: max", float(d.max()), "mean", float(d.mean()))
    assert float(d.max()) <= 2 * 8 * 1e-3
    assert float(d.mean()) < 6e-4
    assert F.cosine_similarity(pack_a.flat, pack_b.flat, dim=0).item() > 0.9995


def test_proximal_term_pulls_towards_the_anchor():
    dist = {}
    for mu in (0.0, 1.0):
        tr, pack, feed = _setup("tcgen05", "bf16", True, mu)
        w0 = pack.trainable().clone()
        h = tr.fit(feed, None, 1, early_stopping=None, reduce_lr_patience=None)
        torch.cuda.synchronize()
        if mu > 0:
            assert torch.equal(tr.anchor, w0)
        dist[mu] = float((pack.trainable() - w0).norm())
        assert h[0].loss == h[0].loss
    print("||w - anchor|| after one epoch, mu=0 / mu=1:", dist)      # measured on an H100: 1.18 / 0.31
    assert dist[1.0] < dist[0.0]


# ------------------------------------------------------------------ 4. sample-weighted encrypted FedAvg on CUDA
def test_simulated_noniid_clients_on_cuda():
    from hefl_b200.config import FLConfig
    from hefl_b200.fl import simulate_clients

    cfg = FLConfig(model="cnn2", image_size=28, in_channels=1, num_classes=10, batch_size=8, local_epochs=1,
                   steps_per_epoch=4, val_steps=1, clients=3, he_preset="n4096_l3", device="cuda", transport="loopback",
                   dtype="fp32", nn_backend="cudnn", dirichlet_alpha=0.3, fedavg_weighting="samples", fedprox_mu=0.01)
    r = simulate_clients(cfg, device=torch.device("cuda"), rounds=1)
    print("n_train", r["n_train"], "weights", r["fedavg_weights"], "max_abs_err", r["max_abs_err"])
    assert len(set(r["n_train"])) > 1
    # measured on an H100: n_train [41, 27, 41], weights 1.128 / 0.743 / 1.128, max_abs_err 3.0e-8
    assert r["max_abs_err"] < 1e-6


# ------------------------------------------------------------------ 5. two GPUs
@pytest.mark.multigpu
def test_noniid_round_across_two_gpus():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29691", os.path.join(ROOT, "tests", "mp_noniid_worker.py"),
           "--backend", "nccl", "--model", "medcnn", "--mu", "0.05"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, OMP_NUM_THREADS="2"),
                       cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    rep = json.loads([l for l in r.stdout.splitlines() if l.startswith("MP_REPORT ")][-1][len("MP_REPORT "):])
    assert rep["transport"] == "fused"
    assert rep["max_abs_err"] < 1e-5 and rep["debug_precision_err"] < 1e-5

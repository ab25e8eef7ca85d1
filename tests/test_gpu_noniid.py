"""Non-IID clients on the H100: the FedProx term of the Adam kernel (adam_kernel<true>), the engine trained with it,
its pull towards the round's global model, sample-weighted encrypted FedAvg on CUDA, and the multi-GPU round on the
fused transport."""
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


# ------------------------------------------------------------------ 2. the engine with FedProx
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


# ------------------------------------------------------------------ 3. sample-weighted encrypted FedAvg on CUDA
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


# ------------------------------------------------------------------ 4. two GPUs
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

"""Non-IID clients on CPU: Dirichlet label-skew shards, sample-weighted encrypted FedAvg (the client weight folded
into the CKKS encode scale) and the FedProx term of the CPU Adam twin; gloo world-2 runs; CLI and environment."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from hefl_b200.config import FLConfig
from hefl_b200.fl import FederatedRunner, simulate_clients
from hefl_b200.fl.data import ImageFolderDataset, dirichlet_partition

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _labels(n=3000, classes=4, seed=0):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, classes, n))


# ------------------------------------------------------------------ partition
def test_dirichlet_partition_is_a_deterministic_disjoint_cover():
    y = _labels()
    parts = dirichlet_partition(y, 5, 0.5, seed=7, min_train=32)
    allidx = torch.cat(parts)
    assert allidx.numel() == y.numel() and torch.equal(allidx.sort().values, torch.arange(y.numel()))
    assert all(p.numel() - int(p.numel() * 0.1) >= 32 for p in parts)
    again = dirichlet_partition(y, 5, 0.5, seed=7, min_train=32)
    assert all(torch.equal(a, b) for a, b in zip(parts, again))
    other = dirichlet_partition(y, 5, 0.5, seed=8, min_train=32)
    assert not all(torch.equal(a, b) for a, b in zip(parts, other))


def test_dirichlet_alpha_controls_label_skew():
    y = _labels(4000, 4)
    pool = torch.bincount(y, minlength=4).double() / y.numel()

    def worst_tv(alpha):
        parts = dirichlet_partition(y, 4, alpha, seed=1, min_train=8)
        return max(0.5 * float((torch.bincount(y[p], minlength=4).double() / p.numel() - pool).abs().sum())
                   for p in parts)

    assert worst_tv(1e4) < 0.03              # near the pool's class mix
    assert worst_tv(0.1) > 0.3               # clearly skewed


def test_dirichlet_partition_fails_with_the_client_sizes():
    with pytest.raises(ValueError, match="client sizes"):
        dirichlet_partition(_labels(40, 2), 8, 0.05, seed=0, min_train=32)


def test_image_folder_dirichlet_clients_are_disjoint_and_cover_the_folder(tmp_path):
    rng = np.random.default_rng(0)
    for label in ("a", "b", "c"):
        d = tmp_path / label
        d.mkdir()
        for i in range(30):
            np.save(d / f"{i:02d}.npy", rng.integers(0, 255, (8, 8, 3), dtype=np.uint8))
    K = 3
    parts = [ImageFolderDataset(str(tmp_path), image_size=8, index=i, num_clients=K, shuffle_seed=5, pin=False,
                                dirichlet_alpha=0.5, min_train=4) for i in range(K)]
    names = [set(p.filenames) for p in parts]
    assert sum(len(n) for n in names) == 90 and len(set.union(*names)) == 90
    assert all(len(p) - int(len(p) * 0.1) >= 4 for p in parts)
    for p in parts:                                   # labels follow the files, class ids are the folder's
        for f, l in zip(p.filenames, p.labels.tolist()):
            assert p.class_indices[os.path.basename(os.path.dirname(f))] == l


# ------------------------------------------------------------------ encrypt weight
def test_encrypt_weight_one_is_bit_identical_and_weight_scales_the_values():
    from hefl_b200.he.context import CKKSContext
    ctx = CKKSContext(4096, prime_bits=(36, 36, 37), scale_bits=40, device="cpu")
    sk, pk = ctx.keygen(seed=3)
    x = torch.randn(5000, generator=torch.Generator().manual_seed(0)) * 0.1
    a = ctx.encrypt(x, pk, seed=9)
    b = ctx.encrypt(x, pk, seed=9, weight=1.0)
    assert torch.equal(a.data, b.data) and a.scale == b.scale == ctx.scale
    for w in (0.37, 1.8):
        c = ctx.encrypt(x, pk, seed=9, weight=w)
        assert c.scale == ctx.scale
        assert float((ctx.decrypt(c, sk) - w * x).abs().max()) < 1e-6


# ------------------------------------------------------------------ simulation
def _cfg(**kw):
    base = dict(model="cnn2", image_size=28, in_channels=1, num_classes=10, batch_size=8, local_epochs=1,
                steps_per_epoch=4, val_steps=1, clients=3, he_preset="n4096_l3", device="cpu", transport="loopback",
                dtype="fp32", nn_backend="cudnn")
    base.update(kw)
    return FLConfig(**base)


def test_simulated_dirichlet_clients_with_sample_weights():
    r = simulate_clients(_cfg(dirichlet_alpha=0.3, fedavg_weighting="samples"), rounds=1)
    assert len(set(r["n_train"])) > 1                           # unequal shards
    assert abs(sum(r["fedavg_weights"]) - 3.0) < 1e-12
    assert r["max_abs_err"] < 1e-5                              # against sum(n_k x_k) / N
    # the weights took effect: the unweighted mean of the same client models is further away than the CKKS error
    # (the cross-check re-runs the clients with uniform weighting on the same shards)
    u = simulate_clients(_cfg(dirichlet_alpha=0.3, fedavg_weighting="uniform"), rounds=1)
    assert float((r["encrypted_avg"] - u["plain_avg"]).abs().max()) > 10 * max(r["max_abs_err"], 1e-7)


def test_iid_shards_with_sample_weights_are_bit_identical_to_uniform():
    a = simulate_clients(_cfg(fedavg_weighting="samples"), rounds=1)
    b = simulate_clients(_cfg(), rounds=1)
    assert a["fedavg_weights"] == [1.0, 1.0, 1.0]
    assert torch.equal(a["encrypted_avg"], b["encrypted_avg"])


def test_fedprox_changes_local_training_and_keeps_the_oracle():
    a = simulate_clients(_cfg(clients=2, fedprox_mu=0.5), rounds=1)
    b = simulate_clients(_cfg(clients=2), rounds=1)
    assert a["max_abs_err"] < 1e-5
    assert float((a["encrypted_avg"] - b["encrypted_avg"]).abs().max()) > 1e-6


# ------------------------------------------------------------------ CPU Adam twin
def _adam64(p, g, m, v, anchor, mu, t, lr=1e-3, decay=1e-4, b1=0.9, b2=0.999, eps=1e-7):
    p, g, m, v, a = (x.double() for x in (p, g, m, v, anchor))
    g = g + mu * (p - a)
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    lr_t = lr / (1 + decay * (t - 1))
    alpha = lr_t * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
    return p - alpha * m / (v.sqrt() + eps), m, v


def test_cpu_adam_twin_with_anchor():
    from hefl_b200 import _ext
    ops = _ext.ops()
    gen = torch.Generator().manual_seed(0)
    n = 1001
    p0, g0 = torch.randn(n, generator=gen), torch.randn(n, generator=gen) * 1e-2
    m0, v0 = torch.randn(n, generator=gen) * 1e-3, torch.rand(n, generator=gen) * 1e-4
    anchor = p0 + torch.randn(n, generator=gen) * 0.05
    step = torch.tensor([3], dtype=torch.int64)

    def run(anc, mu):
        p, g, m, v = p0.clone(), g0.clone(), m0.clone(), v0.clone()
        ops.adam_step_(p, g, m, v, None, step, None, 1e-3, 1e-4, 0.9, 0.999, 1e-7, anc, mu)
        assert float(g.abs().max()) == 0.0
        return p, m, v

    p, m, v = run(anchor, 0.3)
    rp, rm, rv = _adam64(p0, g0, m0, v0, anchor, 0.3, 3)
    assert float((p.double() - rp).abs().max()) < 1e-6
    assert float((m.double() - rm).abs().max()) < 1e-8 and float((v.double() - rv).abs().max()) < 1e-9
    plain = run(None, 0.0)
    for x, y in zip(run(anchor, 0.0), plain):          # mu = 0 with an anchor: today's update, bit for bit
        assert torch.equal(x, y)
    assert not torch.equal(p, plain[0])


# ------------------------------------------------------------------ runner validation and records
def test_runner_rejects_bad_noniid_options():
    for kw, msg in ((dict(dirichlet_alpha=-0.1), "dirichlet_alpha"), (dict(fedprox_mu=-1.0), "fedprox_mu"),
                    (dict(fedavg_weighting="size"), "fedavg_weighting")):
        with pytest.raises(ValueError, match=msg):
            FederatedRunner(_cfg(clients=1, **kw), device=torch.device("cpu"))


def test_runner_round_record_reports_shard_and_weight():
    cfg = _cfg(clients=1, dirichlet_alpha=0.5, fedavg_weighting="samples", fedprox_mu=0.01, transport="gloo",
               debug_precision=True)
    r = FederatedRunner(cfg, device=torch.device("cpu"))
    rec = r.run_round(check=True)
    assert rec["n_train"] == r.n_train == len(r.train_feed.indices)
    assert sum(rec["label_counts"]) == rec["n_train"] and len(rec["label_counts"]) == 10
    assert rec["fedavg_weight"] == 1.0 and rec["ckks_max_abs_err"] < 1e-6


# ------------------------------------------------------------------ gloo world 2
def _mp(port, extra=()):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "mp_noniid_worker.py"), "--backend", "gloo", *extra]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=dict(os.environ, OMP_NUM_THREADS="2"),
                       cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("MP_REPORT ")][-1]
    return json.loads(line[len("MP_REPORT "):])


def test_noniid_federated_rounds_gloo_world2():
    rep = _mp(29681)
    assert rep["world"] == 2 and rep["n_train"][0] != rep["n_train"][1]
    assert rep["weights_rank0"][0] != 1.0
    assert rep["max_abs_err"] < 1e-5 and rep["debug_precision_err"] < 1e-5


def test_noniid_federated_rounds_with_a_dropped_client_gloo():
    rep = _mp(29685, ["--drop-rank", "1"])
    assert rep["weights_rank0"] == [1.0, 1.0] and rep["max_abs_err"] < 1e-5 and rep["debug_precision_err"] < 1e-5


# ------------------------------------------------------------------ CLI and environment
def test_noniid_flags_parse_from_cli_and_environment(monkeypatch):
    cfg = FLConfig.from_args(["--dirichlet-alpha", "0.3", "--fedavg-weighting", "samples", "--fedprox-mu", "0.01"])
    assert (cfg.dirichlet_alpha, cfg.fedavg_weighting, cfg.fedprox_mu) == (0.3, "samples", 0.01)
    monkeypatch.setenv("HEFL_DIRICHLET_ALPHA", "2")
    monkeypatch.setenv("HEFL_FEDAVG_WEIGHTING", "samples")
    monkeypatch.setenv("HEFL_FEDPROX_MU", "0.5")
    cfg = FLConfig.from_args([])
    assert (cfg.dirichlet_alpha, cfg.fedavg_weighting, cfg.fedprox_mu) == (2.0, "samples", 0.5)
    d = FLConfig()
    assert (d.dirichlet_alpha, d.fedavg_weighting, d.fedprox_mu) == (0.0, "uniform", 0.0)


def test_cli_simulation_with_noniid_flags():
    env = dict(os.environ, PYTHONPATH=ROOT)
    env.pop("RANK", None); env.pop("WORLD_SIZE", None)
    args = ["--device", "cpu", "--model", "cnn2", "--image-size", "28", "--in-channels", "1", "--num-classes", "10",
            "--batch-size", "8", "--local-epochs", "1", "--steps-per-epoch", "4", "--val-steps", "1",
            "--he-preset", "n2048_l1", "--nn-backend", "cudnn", "--dtype", "fp32", "--simulate", "--clients", "3",
            "--dirichlet-alpha", "0.3", "--fedavg-weighting", "samples", "--fedprox-mu", "0.01"]
    r = subprocess.run([sys.executable, "-m", "hefl_b200", *args], capture_output=True, text=True, cwd=ROOT, env=env,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    d = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    assert d["mode"] == "simulate" and d["clients"] == 3 and d["max_abs_err_vs_plaintext"] < 1e-4

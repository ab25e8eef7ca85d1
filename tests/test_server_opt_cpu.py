"""Server optimizers of encrypted FedAvg on CPU (DESIGN.md §8): the host twin of the fused decode + step against an
independent float64 reference, option checks, the loopback simulation against its float64 oracle, the runner's
checkpoints / dropouts / debug_precision / records, gloo world-2 runs and the CLI."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from hefl_b200.config import FLConfig
from hefl_b200.fl import FederatedRunner, simulate_clients
from hefl_b200.fl.server_opt import SERVER_OPTS, ServerOptimizer, check_server_options, lipschitz
from hefl_b200.he.context import CKKSContext

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPTS = ("fedavgm", "fedadagrad", "fedyogi", "fedadam")


# ------------------------------------------------------------------ float64 reference of the update
def ref_step(name, lr, b1, b2, tau, x, a, m, v):
    """DESIGN.md §8 in float64 numpy on one slice of trainable values; m and v are updated in place."""
    d = a - x
    if name == "fedavgm":
        m[:] = b1 * m + d
        return x + lr * m
    m[:] = b1 * m + (1 - b1) * d
    if name == "fedadagrad":
        v[:] = v + d * d
    elif name == "fedyogi":
        v[:] = v - (1 - b2) * d * d * np.sign(v - d * d)
    else:
        v[:] = b2 * v + (1 - b2) * d * d
    return x + lr * m / (np.sqrt(v) + tau)


HP = {"fedavgm": dict(lr=1.0, beta1=0.9, beta2=0.99, tau=1e-3)}
for _o in OPTS[1:]:
    HP[_o] = dict(lr=0.1, beta1=0.9, beta2=0.99, tau=1e-3)


def run_twin_vs_reference(ctx, name, device, steps=3, seed=0):
    """Three consecutive fused steps on a batch whose values start at flat index g0 > 0, end partway through a
    ciphertext and cross the n_trainable boundary inside a ciphertext; the reference is fed each step's own fp64
    average and x_t, and carries its own float64 m and v. Returns the worst |x_new|, |m|, |v| differences."""
    sk, pk = ctx.keygen(seed=seed + 1)
    slots = ctx.slots
    g0 = 37
    nvals = 2 * slots + slots // 2 + 11
    end = g0 + nvals
    nt = g0 + slots + slots // 3                    # inside the second ciphertext
    hp = HP[name]
    gen = torch.Generator().manual_seed(seed)
    x = (torch.rand(end, generator=gen) * 2 - 1).to(device)
    opt = ServerOptimizer(name, nt, device, lr=hp["lr"], beta1=hp["beta1"], beta2=hp["beta2"], tau=hp["tau"])
    rm = np.zeros(nt)
    rv = np.full(nt, hp["tau"] ** 2)
    worst = {"x": 0.0, "m": 0.0, "v": 0.0}
    for s in range(steps):
        vals = x[g0:].cpu() + torch.randn(nvals, generator=gen) * 0.02
        ct = ctx.encrypt(vals.to(device), pk, seed=100 + s)
        out = torch.full((end,), 7.0, device=device)
        avg = torch.zeros(end, dtype=torch.float64, device=device)
        opt.step(ctx, ct, sk, 1.0, x, out, offset=g0, avg_out=avg)
        o, a, xs = out.cpu().double().numpy(), avg.cpu().numpy(), x.cpu().double().numpy()
        assert np.all(o[:g0] == 7.0) and np.all(a[:g0] == 0.0)          # nothing outside the batch is written
        want = a.copy()
        want[g0:nt] = ref_step(name, hp["lr"], hp["beta1"], hp["beta2"], hp["tau"], xs[g0:nt], a[g0:nt],
                               rm[g0:nt], rv[g0:nt])
        want[nt:] = a[nt:]                                               # the tail: plain FedAvg
        worst["x"] = max(worst["x"], float(np.abs(o[g0:] - want[g0:]).max()))
        worst["m"] = max(worst["m"], float(np.abs(opt.m.cpu().double().numpy() - rm).max()))
        worst["v"] = max(worst["v"], float(np.abs(opt.v.cpu().double().numpy() - rv).max()))
        assert np.all(o[nt:] == a[nt:].astype(np.float32))               # the tail is the fp32 average, bit for bit
        assert torch.equal(opt.m[:g0].cpu(), torch.zeros(g0))            # state below g0 untouched
        x = out
    return worst


@pytest.mark.parametrize("name", OPTS)
@pytest.mark.parametrize("n,bits", [(2048, (54,)), (2048, (36, 36, 37)), (4096, (54,)), (4096, (36, 36, 37))])
def test_host_twin_matches_float64_reference(name, n, bits):
    ctx = CKKSContext(n, prime_bits=bits, scale_bits=40, device="cpu", enforce_security=False)
    w = run_twin_vs_reference(ctx, name, "cpu")
    print(f"{name} n={n} k={min(len(bits), 2)}: max |x| {w['x']:.3g} |m| {w['m']:.3g} |v| {w['v']:.3g}")
    assert w["x"] <= 1e-6 and w["m"] <= 1e-7 and w["v"] <= 1e-8


def test_fedavgm_without_momentum_is_fedavg_within_one_ulp():
    ctx = CKKSContext(4096, prime_bits=(36, 36, 37), scale_bits=40, device="cpu")
    sk, pk = ctx.keygen(seed=2)
    gen = torch.Generator().manual_seed(1)
    x = torch.rand(5000, generator=gen) * 2 - 1
    ct = ctx.encrypt(x + torch.randn(5000, generator=gen) * 0.05, pk, seed=3)
    plain = ctx.decrypt(ct, sk, divide_by=1.0)
    opt = ServerOptimizer("fedavgm", x.numel(), "cpu", lr=1.0, beta1=0.0)
    out = torch.empty_like(x)
    opt.step(ctx, ct, sk, 1.0, x, out)
    # x + (float)(a - x) rounds once more, at the scale of the larger of |x| and |a|: one ulp there
    ulp = np.spacing(np.maximum(np.abs(plain.numpy()), np.abs(x.numpy())))
    diff = np.abs(out.numpy() - plain.numpy())
    print(f"fedavgm(beta1=0, eta=1) vs decrypt: {int((diff > 0).sum())} of {diff.size} values differ, "
          f"max {float((diff / ulp).max()):.2f} ulp")
    assert np.all(diff <= ulp)


# ------------------------------------------------------------------ options
def test_server_flags_parse_from_cli_and_environment(monkeypatch):
    cfg = FLConfig.from_args(["--server-opt", "fedadam", "--server-lr", "0.3", "--server-momentum", "0.5",
                              "--server-beta2", "0.9", "--server-tau", "0.01"])
    assert (cfg.server_opt, cfg.server_lr, cfg.server_momentum, cfg.server_beta2, cfg.server_tau) == \
        ("fedadam", 0.3, 0.5, 0.9, 0.01)
    for k, v in (("OPT", "fedyogi"), ("LR", "0.2"), ("MOMENTUM", "0"), ("BETA2", "0.5"), ("TAU", "0.1")):
        monkeypatch.setenv("HEFL_SERVER_" + k, v)
    cfg = FLConfig.from_args([])
    assert (cfg.server_opt, cfg.server_lr, cfg.server_momentum, cfg.server_beta2, cfg.server_tau) == \
        ("fedyogi", 0.2, 0.0, 0.5, 0.1)
    d = FLConfig()
    assert (d.server_opt, d.server_lr, d.server_momentum, d.server_beta2, d.server_tau) == \
        ("fedavg", 1.0, 0.9, 0.99, 1e-3)
    for name in SERVER_OPTS:
        check_server_options(FLConfig(server_opt=name))


@pytest.mark.parametrize("kw,msg", [
    (dict(server_opt="fedsgd"), "server_opt"),
    (dict(server_opt="fedadam", server_lr=0.0), "server_lr"),
    (dict(server_opt="fedadam", server_lr=-1.0), "server_lr"),
    (dict(server_momentum=1.0), "server_momentum"),
    (dict(server_momentum=-0.1), "server_momentum"),
    (dict(server_beta2=1.0), "server_beta2"),
    (dict(server_beta2=-0.5), "server_beta2"),
    (dict(server_tau=0.0), "server_tau"),
    (dict(server_opt="fedavgm", packing="coeff"), "coefficient packing"),
])
def test_bad_server_options_raise(kw, msg):
    with pytest.raises(ValueError, match=msg):
        check_server_options(FLConfig(**kw))
    with pytest.raises(ValueError, match=msg):
        FederatedRunner(_cfg(clients=1, **kw), device=torch.device("cpu"))
    with pytest.raises(ValueError, match=msg):
        simulate_clients(_cfg(**kw))
    check_server_options(FLConfig(packing="coeff"))                # coefficient packing with plain FedAvg is fine


def test_the_op_rejects_bad_arguments():
    ctx = CKKSContext(2048, prime_bits=(54,), scale_bits=40, device="cpu")
    sk, pk = ctx.keygen(seed=1)
    ct = ctx.encrypt(torch.zeros(100), pk, seed=1)
    x, out = torch.zeros(100), torch.zeros(100)
    m, v = torch.zeros(100), torch.ones(100)
    hp = dict(lr=1.0, beta1=0.9, beta2=0.99, tau=1e-3)
    with pytest.raises(RuntimeError, match="opt must be"):
        ctx.decrypt_server_step(ct, sk, 1.0, x, out, m, v, 0, hp, 100)
    with pytest.raises(RuntimeError, match="x_t has 100 elements, needs 101"):
        ctx.decrypt_server_step(ct, sk, 1.0, x, out, m, v, 4, hp, 100, offset=1)
    with pytest.raises(RuntimeError, match="float32"):
        ctx.decrypt_server_step(ct, sk, 1.0, x.double(), out, m, v, 4, hp, 100)
    with pytest.raises(RuntimeError, match="m has"):
        ctx.decrypt_server_step(ct, sk, 1.0, x, out, m[:50], v, 4, hp, 100)
    ctx.decrypt_server_step(ct, sk, 1.0, x, out, m[:50], v[:50], 4, hp, 50)   # state covers n_trainable only
    ctc = ctx.encrypt(torch.zeros(100), pk, seed=1, packing="coeff")
    with pytest.raises(ValueError, match="coefficient packing"):
        ctx.decrypt_server_step(ctc, sk, 1.0, x, out, m, v, 4, hp, 100)


# ------------------------------------------------------------------ simulation
def _cfg(**kw):
    base = dict(model="cnn2", image_size=28, in_channels=1, num_classes=10, batch_size=8, local_epochs=1,
                steps_per_epoch=4, val_steps=1, clients=3, he_preset="n4096_l3", device="cpu", transport="loopback",
                dtype="fp32", nn_backend="cudnn")
    base.update(kw)
    return FLConfig(**base)


def check_simulation(r, cfg):
    """The step moves the model away from the average, and the fused step of the encrypted average lies within
    (its error) x (the step's Lipschitz constant in d) of the float64 step of the plaintext average, plus a few
    fp32 roundings of the new weights."""
    L = max(1.0, lipschitz(cfg.server_opt, cfg.server_lr, cfg.server_momentum, cfg.server_tau))
    g, go = r["global"].double(), r["global_oracle"].double()
    bound = L * r["max_abs_err"] + 8 * 2.0 ** -24 * max(1.0, float(go.abs().max()))
    err = float((g - go).abs().max())
    moved = float((g - r["encrypted_avg"].double()).abs().max())
    print(f"{cfg.server_opt}: |global - oracle| {err:.3g} (bound {bound:.3g}), avg err {r['max_abs_err']:.3g}, "
          f"step moved the model {moved:.3g} from the average")
    assert err <= bound
    assert moved > 10 * bound
    assert r["max_abs_err"] < 1e-5


@pytest.mark.parametrize("name,lr", [("fedadam", 1.0), ("fedavgm", 0.5)])   # (the first FedAvgM step at eta = 1 is FedAvg)
def test_simulated_server_step_matches_its_float64_oracle(name, lr):
    cfg = _cfg(dirichlet_alpha=0.3, fedavg_weighting="samples", server_opt=name, server_lr=lr)
    r = simulate_clients(cfg, rounds=1)
    check_simulation(r, cfg)
    assert len(set(r["n_train"])) > 1
    # the average itself is unchanged by the step: the same as plain FedAvg's
    b = simulate_clients(_cfg(dirichlet_alpha=0.3, fedavg_weighting="samples"), rounds=1)
    assert torch.equal(r["encrypted_avg"], b["encrypted_avg"]) and "global" not in b


# ------------------------------------------------------------------ runner
def _runner(**kw):
    cfg = _cfg(clients=1, transport="gloo", deterministic_crypto=True, server_opt="fedadam", server_lr=0.1, **kw)
    r = FederatedRunner(cfg, device=torch.device("cpu"))
    # the data order is fixed here, so that only the server state can differ
    r.train_feed.shuffle = False
    if r.val_feed is not None:
        r.val_feed.shuffle = False
    return r


def test_resumed_run_equals_uninterrupted_run(tmp_path):
    a = _runner()
    for _ in range(3):
        a.run_round(check=True)
    b = _runner()
    for _ in range(2):
        b.run_round(check=True)
    ck = str(tmp_path / "ck.pt")
    b.save_checkpoint(ck)
    c = _runner()
    c.load_checkpoint(ck)
    assert c.round == 2 and torch.equal(c.server_opt.m, b.server_opt.m)
    c.run_round(check=True)
    assert torch.equal(a.pack.flat, c.pack.flat)
    assert torch.equal(a.server_opt.m, c.server_opt.m) and torch.equal(a.server_opt.v, c.server_opt.v)
    # without the server state in the rank file the step starts fresh, as the local optimizer does
    os.remove(ck + ".rank0")
    d = _runner()
    d.load_checkpoint(ck)
    assert d.server_opt.m is None


def test_no_contributor_keeps_the_model_and_the_state():
    r = _runner(allow_dropouts=True)
    r.run_round(check=True)
    m, v = r.server_opt.m.clone(), r.server_opt.v.clone()
    r.participating = False
    r.global_flat.copy_(r.pack.flat)
    r.local_train()
    before = r.pack.flat.clone()
    r.decrypt_apply(r.aggregate(r.encrypt_update()))
    assert r._contributors() == 0
    assert torch.equal(r.pack.flat, before)
    assert torch.equal(r.server_opt.m, m) and torch.equal(r.server_opt.v, v)


def test_debug_precision_records_the_average_error_and_the_record_names_the_optimizer():
    r = _runner(debug_precision=True)
    x0 = r.pack.flat.clone()
    rec = r.run_round(check=True)
    assert rec["server_opt"] == "fedadam"
    assert rec["ckks_max_abs_err"] < 1e-6
    # the stepped model is far from the average that was checked
    assert float((r.pack.flat - r._avg_out).abs().max()) > 1e-3
    assert not torch.equal(r.pack.flat, x0)
    plain = FederatedRunner(_cfg(clients=1, transport="gloo", deterministic_crypto=True), device=torch.device("cpu"))
    assert plain.server_opt is None and plain.run_round()["server_opt"] == "fedavg"


# ------------------------------------------------------------------ gloo world 2
def _mp(port, extra=()):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "mp_server_opt_worker.py"), "--backend", "gloo", *extra]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=dict(os.environ, OMP_NUM_THREADS="2"),
                       cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("MP_REPORT ")][-1]
    return json.loads(line[len("MP_REPORT "):])


def test_key_holder_steps_and_broadcasts_gloo_world2():
    rep = _mp(29701, ["--key-holder", "0", "--opt", "fedadam"])
    assert rep["world"] == 2 and rep["rounds_equal"] == rep["rounds"] == 3
    assert rep["state_on"] == [True, False]
    assert rep["debug_precision_err"] < 1e-5


def test_every_rank_steps_alike_without_a_key_holder_gloo():
    rep = _mp(29705, ["--key-holder", "-1", "--opt", "fedyogi"])
    assert rep["rounds_equal"] == rep["rounds"] == 3 and rep["state_equal"] == 3
    assert rep["state_on"] == [True, True]


# ------------------------------------------------------------------ CLI
def test_cli_simulation_with_a_server_optimizer():
    env = dict(os.environ, PYTHONPATH=ROOT)
    env.pop("RANK", None); env.pop("WORLD_SIZE", None)
    args = ["--device", "cpu", "--model", "cnn2", "--image-size", "28", "--in-channels", "1", "--num-classes", "10",
            "--batch-size", "8", "--local-epochs", "1", "--steps-per-epoch", "4", "--val-steps", "1",
            "--he-preset", "n2048_l1", "--nn-backend", "cudnn", "--dtype", "fp32", "--simulate", "--clients", "3",
            "--server-opt", "fedyogi", "--server-lr", "0.1"]
    r = subprocess.run([sys.executable, "-m", "hefl_b200", *args], capture_output=True, text=True, cwd=ROOT, env=env,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    d = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    assert d["mode"] == "simulate" and d["server_opt"] == "fedyogi" and d["max_abs_err_vs_plaintext"] < 1e-4
    assert d["max_abs_err_global_vs_oracle"] < 1e-3

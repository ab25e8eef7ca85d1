"""Server optimizers on the H100 (DESIGN.md §8): the decode kernel's OPT = 1..4 instantiations against the host twin
and an independent float64 reference at logn 12-15, one launch per op, the pipelined FedAvg against the unchunked
path, the CUDA simulation against its float64 oracle, and the two-GPU round with a key holder."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from hefl_b200.fl.server_opt import ServerOptimizer, lipschitz
from hefl_b200.he.context import CKKSContext, CtBatch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPTS = ("fedavgm", "fedadagrad", "fedyogi", "fedadam")
CODES = {"fedavgm": 1, "fedadagrad": 2, "fedyogi": 3, "fedadam": 4}


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


def _hp(name):
    return dict(lr=1.0 if name == "fedavgm" else 0.1, beta1=0.9, beta2=0.99, tau=1e-3)


# ------------------------------------------------------------------ 1. the fused kernel
@pytest.mark.parametrize("name", OPTS)
@pytest.mark.parametrize("k", [1, 2])
@pytest.mark.parametrize("logn", [12, 13, 14, 15])
def test_fused_step_matches_host_twin_and_float64_reference(name, k, logn):
    n = 1 << logn
    c = CKKSContext(n, prime_bits=(54,) if k == 1 else (54, 50), scale_bits=40, enforce_security=False)
    g = CKKSContext(n, primes=c.primes, scale_bits=40, enforce_security=False, device="cuda")
    sk, pk = c.keygen(seed=logn + k)
    skg = sk.cuda()
    slots = c.slots
    g0 = 29
    nvals = 2 * slots + slots // 2 + 5                # ends partway through the third ciphertext
    end = g0 + nvals
    nt = g0 + slots + slots // 3                     # the trainable boundary inside the second ciphertext
    hp = _hp(name)
    gen = torch.Generator().manual_seed(logn * 10 + k)
    x = torch.rand(end, generator=gen) * 2 - 1
    dev = ServerOptimizer(name, nt, "cuda", **hp)
    twin = ServerOptimizer(name, nt, "cpu", **hp)
    rm, rv = np.zeros(nt), np.full(nt, hp["tau"] ** 2)
    xg, xc = x.cuda(), x.clone()
    worst = {"twin_x": 0.0, "twin_m": 0.0, "twin_v": 0.0, "ref_x": 0.0, "ref_m": 0.0, "ref_v": 0.0}
    for s in range(3):
        vals = xg[g0:].cpu() + torch.randn(nvals, generator=gen) * 0.02
        ct = c.encrypt(vals, pk, seed=50 + s)
        ctg = CtBatch(ct.data.cuda(), ct.scale, ct.nvals, ct.packing)
        out_g = torch.full((end,), 7.0, device="cuda")
        avg_g = torch.zeros(end, dtype=torch.float64, device="cuda")
        dev.step(g, ctg, skg, 1.0, xg, out_g, offset=g0, avg_out=avg_g)
        out_c = torch.full((end,), 7.0)
        twin.step(c, ct, sk, 1.0, xc, out_c, offset=g0)
        o, a, xs = out_g.cpu().double().numpy(), avg_g.cpu().numpy(), xg.cpu().double().numpy()
        assert np.all(o[:g0] == 7.0) and np.all(a[:g0] == 0.0)
        want = a.copy()
        want[g0:nt] = ref_step(name, hp["lr"], hp["beta1"], hp["beta2"], hp["tau"], xs[g0:nt], a[g0:nt],
                               rm[g0:nt], rv[g0:nt])
        assert np.all(o[nt:] == a[nt:].astype(np.float32))          # the tail is the fp32 average
        worst["ref_x"] = max(worst["ref_x"], float(np.abs(o[g0:] - want[g0:]).max()))
        worst["twin_x"] = max(worst["twin_x"], float((out_g.cpu() - out_c)[g0:].abs().max()))
        for key, t, tc, r in (("m", dev.m, twin.m, rm), ("v", dev.v, twin.v, rv)):
            worst["twin_" + key] = max(worst["twin_" + key], float((t.cpu() - tc).abs().max()))
            worst["ref_" + key] = max(worst["ref_" + key], float(np.abs(t.cpu().double().numpy() - r).max()))
        if s == 0:
            # the fp32 average of the fused op is ctx.decrypt's output, bit for bit
            avg32 = torch.zeros(end, device="cuda")
            m0, v0 = torch.zeros(nt, device="cuda"), torch.full((nt,), 1e-6, device="cuda")
            g.decrypt_server_step(ctg, skg, 1.0, xg, torch.empty(end, device="cuda"), m0, v0, CODES[name], hp, nt,
                                  offset=g0, avg_out=avg32)
            assert torch.equal(avg32[g0:], g.decrypt(ctg, skg))
        xg, xc = out_g, out_c
    print(f"{name} logn={logn} k={k}: " + ", ".join(f"{kk} {vv:.3g}" for kk, vv in worst.items()))
    assert worst["ref_x"] <= 1e-6 and worst["twin_x"] <= 1e-6
    assert worst["ref_m"] <= 1e-7 and worst["twin_m"] <= 1e-7
    assert worst["ref_v"] <= 1e-8 and worst["twin_v"] <= 1e-8


ONE_LAUNCH = r"""
import json, sys, torch
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, sys.argv[1])
from hefl_b200.he.context import CKKSContext
g = CKKSContext(4096, prime_bits=(36, 36, 37), scale_bits=40, device="cuda")
sk, pk = g.keygen(seed=1)
nv = 109 * g.slots - 100
x = torch.rand(nv, device="cuda")
ct = g.encrypt(x + 0.01, pk, seed=2)
res = g.decrypt_residues(ct, sk)
out, m = torch.empty_like(x), torch.zeros(nv, device="cuda")
v = torch.full_like(m, 1e-6)
torch.cuda.synchronize()
l0 = int(g.ops.launch_count())
with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    g.ops.ckks_decode_server_step_(res, g.consts_cpu, g.q0_inv_q1, g.logn, 1.0 / ct.scale, g.rot, g.ksi, nv, 0, nv,
                                   x, out, m, v, 4, 0.1, 0.9, 0.99, 1e-3, None)
    torch.cuda.synchronize()
kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
           and "Memcpy" not in e.name and "Memset" not in e.name]
print("ONE_LAUNCH " + json.dumps({"launches": int(g.ops.launch_count()) - l0, "kernels": kernels,
                                  "moved": float((out - (x + 0.01)).abs().max())}))
"""


def test_the_op_is_one_launch_of_the_stepping_decode():
    # in a fresh process: late in a long pytest session the profiler has returned empty traces
    r = subprocess.run([sys.executable, "-c", ONE_LAUNCH, ROOT], capture_output=True, text=True, timeout=300,
                       cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    rep = json.loads([l for l in r.stdout.splitlines() if l.startswith("ONE_LAUNCH ")][-1][len("ONE_LAUNCH "):])
    print("kernels of the op:", rep["kernels"])
    assert rep["launches"] == 1
    assert len(rep["kernels"]) == 1 and "ckks_decode_step_kernel<4>" in rep["kernels"][0]
    assert rep["moved"] > 1e-3                                       # it stepped: FedAdam moves by ~eta


# ------------------------------------------------------------------ 2. the runner
def test_pipelined_server_step_matches_unchunked():
    """fedavg_pipelined (one fused step per 20-ciphertext chunk, on the decrypt stream) == encrypt_update ->
    aggregate -> decrypt_apply on the same weights: the same model and the same server state, bit for bit."""
    from hefl_b200.config import FLConfig
    from hefl_b200.fl import FederatedRunner

    cfg = FLConfig(model="medcnn", local_epochs=1, steps_per_epoch=1, val_steps=0, nn_backend="cudnn",
                   transport="fused", device="cuda", deterministic_crypto=True, server_opt="fedadam", server_lr=0.1)
    run = FederatedRunner(cfg, device=torch.device("cuda"))
    gen = torch.Generator(device="cuda").manual_seed(3)
    for step in range(2):
        run.global_flat.copy_(run.pack.flat)
        w = run.pack.flat + torch.randn(run.pack.numel, device="cuda", generator=gen) * 0.01   # "trained" weights
        run.pack.load_flat(w)
        run.server_opt.ensure_state()
        m0, v0 = run.server_opt.m.clone(), run.server_opt.v.clone()
        run.fedavg_pipelined(chunk_cts=20)
        torch.cuda.synchronize()
        flat_p, m_p, v_p = run.pack.flat.clone(), run.server_opt.m.clone(), run.server_opt.v.clone()
        run.pack.load_flat(w)
        run.server_opt.m.copy_(m0)
        run.server_opt.v.copy_(v0)
        run.decrypt_apply(run.aggregate(run.encrypt_update()))
        torch.cuda.synchronize()
        assert torch.equal(run.pack.flat, flat_p)
        assert torch.equal(run.server_opt.m, m_p) and torch.equal(run.server_opt.v, v_p)
        assert float((flat_p - w).abs().max()) > 1e-3                 # the step, not the average
        run.round += 1


def test_simulated_fedyogi_on_cuda_matches_its_float64_oracle():
    from hefl_b200.config import FLConfig
    from hefl_b200.fl import simulate_clients

    cfg = FLConfig(model="cnn2", image_size=28, in_channels=1, num_classes=10, batch_size=8, local_epochs=1,
                   steps_per_epoch=4, val_steps=1, clients=3, he_preset="n4096_l3", device="cuda", transport="loopback",
                   dtype="fp32", nn_backend="cudnn", dirichlet_alpha=0.3, fedavg_weighting="samples",
                   server_opt="fedyogi")
    r = simulate_clients(cfg, device=torch.device("cuda"), rounds=1)
    L = max(1.0, lipschitz(cfg.server_opt, cfg.server_lr, cfg.server_momentum, cfg.server_tau))
    go = r["global_oracle"].double()
    bound = L * r["max_abs_err"] + 8 * 2.0 ** -24 * max(1.0, float(go.abs().max()))
    err = float((r["global"].double() - go).abs().max())
    print(f"fedyogi on cuda: |global - oracle| {err:.3g} (bound {bound:.3g}), avg err {r['max_abs_err']:.3g}")
    assert err <= bound and r["max_abs_err"] < 1e-6
    assert float((r["global"] - r["encrypted_avg"]).abs().max()) > 10 * bound


# ------------------------------------------------------------------ 3. two GPUs
@pytest.mark.multigpu
def test_server_step_round_across_two_gpus():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29711", os.path.join(ROOT, "tests", "mp_server_opt_worker.py"),
           "--backend", "nccl", "--model", "medcnn", "--key-holder", "0", "--opt", "fedadam"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, OMP_NUM_THREADS="2"),
                       cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    rep = json.loads([l for l in r.stdout.splitlines() if l.startswith("MP_REPORT ")][-1][len("MP_REPORT "):])
    assert rep["transport"] == "fused" and rep["rounds_equal"] == rep["rounds"]
    assert rep["state_on"] == [True, False] and rep["debug_precision_err"] < 1e-5

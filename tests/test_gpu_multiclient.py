"""Several federated clients per GPU: encrypt-accumulate on every device path of the encryption, bit for bit against
the host twin; placement and order independence of the medical CNN on the tcgen05 engine with CUDA graphs (batch 32,
256 x 256); graphs captured once per rank; the pipelined round with several clients; two GPUs x two clients."""
import os
import subprocess
import sys

import pytest
import torch

from hefl_b200 import _ext
from hefl_b200.fl import FederatedRunner
from hefl_b200.he.context import CKKSContext
from kernel_trace import kernels_run, ran
from mp_multiclient_worker import config as worker_config
from test_multiclient_cpu import Placement

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ops = _ext.ops()
pytestmark = pytest.mark.gpu


def _workers(L):
    """CTAs of the busiest limb of a whole-chip persistent encrypt (clusters of two dealt round-robin to limbs)."""
    g = torch.cuda.get_device_properties(0).multi_processor_count & ~1
    return 2 * -(-(g // 2) // L)


def _cases():
    """(n, prime bits, ciphertexts, kernel that must run): every device path of the encryption."""
    return [(4096, (36, 36, 37), 109, "encrypt_kernel<true>"),                       # the medical CNN's round
            (8192, (54, 54, 54, 55), 2 * _workers(4) + 1, "encrypt2_kernel<13>"),
            (16384, (54,) * 4, 5, "encrypt_kernel<false>"),                          # K6, one shared buffer
            (16384, (54,) * 4, 2 * _workers(4) + 1, "encrypt2_kernel<14>"),          # USCR: u_hat in global scratch
            (32768, (54,) * 4, 3, "enc_combine_kernel")]


@pytest.mark.parametrize("case", range(5))
@pytest.mark.parametrize("scaled", [False, True])
def test_encrypt_accumulate_is_encrypt_plus_modular_add_on_every_path(case, scaled):
    n, bits, C, kernel = _cases()[case]
    c = CKKSContext(n, prime_bits=bits, scale_bits=40, enforce_security=False)
    g = CKKSContext(n, primes=c.primes, scale_bits=40, enforce_security=False, device="cuda")
    L, logn = c.L, c.logn
    _, pk = c.keygen(seed=7 + case)
    pk_g = pk.cuda()
    gen = torch.Generator().manual_seed(n + C)
    msg = torch.randint(-2**40, 2**40, (C, n), generator=gen, dtype=torch.int64)
    sc = torch.tensor([3, 5, 7, 11][:L], dtype=torch.int64) if scaled else None
    sc_g = sc.cuda() if scaled else None
    # the accumulator: a ciphertext batch already in the buffer (uniform words below each prime)
    before = torch.stack([torch.randint(0, q, (C, 2, n), generator=gen, dtype=torch.int64) for q in c.primes],
                         dim=2).contiguous()
    for m, seed, off in ((msg, 41, 1000 + C), (None, 42, 0)):
        fresh = ops.encrypt(m, pk, C, L, logn, c.tables, c.consts, sc, seed, off)
        want = before.clone()
        ops.pointwise_(want, want, fresh, L, c.consts, 0)
        host = before.clone()
        ops.encrypt_out(m, pk, C, L, logn, c.tables, c.consts, sc, seed, off, host, True)
        assert torch.equal(host, want)
        acc = before.cuda()
        m_g = m.cuda() if m is not None else None
        _, names = kernels_run(lambda: ops.encrypt_out(m_g, pk_g, C, L, logn, g.tables, g.consts, sc_g, seed, off,
                                                       acc, True), attempts=1)
        assert ran(names, kernel), (n, C, sorted(names))
        assert torch.equal(acc.cpu(), want), f"n={n} C={C}: accumulated words differ"
        # and without accumulate the buffer's old words play no part
        out = before.cuda()
        ops.encrypt_out(m_g, pk_g, C, L, logn, g.tables, g.consts, sc_g, seed, off, out)
        assert torch.equal(out.cpu(), fresh)


def test_encrypt_accumulate_into_chunk_views_of_one_buffer():
    """Chunk by chunk into views of a larger buffer (the pipelined round), with the chunk's ciphertext offset and a
    FedAvg weight: the same words as the whole vector encrypted into a fresh buffer and added mod q."""
    g = CKKSContext(4096, prime_bits=(36, 36, 37), scale_bits=40, device="cuda")
    _, pk = g.keygen(seed=51)
    n_ct, chunk = 109, 16
    per = 2 * g.L * g.n
    x = torch.randn(n_ct * g.slots - 123, generator=torch.Generator().manual_seed(5)).cuda() * 0.05
    y = torch.randn(n_ct * g.slots - 123, generator=torch.Generator().manual_seed(6)).cuda() * 0.05
    buf = torch.zeros(n_ct * per + per, dtype=torch.int64, device="cuda")
    body = buf[:n_ct * per]
    g.encrypt(x, pk, seed=3, out=body, weight=0.8)
    for c0 in range(0, n_ct, chunk):
        c1 = min(n_ct, c0 + chunk)
        g.encrypt(y[c0 * g.slots: c1 * g.slots], pk, seed=9, out=body[c0 * per: c1 * per], ct_offset=c0, weight=1.3,
                  accumulate=True)
    want = g.encrypt(x, pk, seed=3, weight=0.8).data.clone()
    ops.pointwise_(want, want, g.encrypt(y, pk, seed=9, weight=1.3).data, g.L, g.consts, 0)
    assert torch.equal(body.view_as(want), want)
    assert int(buf[n_ct * per:].abs().sum()) == 0


# ------------------------------------------------------------------ the medical CNN, several clients per GPU
def _med(**kw):
    from hefl_b200.config import FLConfig

    base = dict(model="medcnn", local_epochs=1, steps_per_epoch=3, val_steps=1, nn_backend="tcgen05", device="cuda",
                transport="loopback", deterministic_crypto=True, key_holder=-1)
    base.update(kw)
    return FLConfig(**base)


def _placement_rounds(world, per, order=None, rounds=2):
    p = Placement(world, per, make_cfg=_med, device=torch.device("cuda"))
    cts, models = [], []
    for _ in range(rounds):
        ct = p.round_ciphertext(order=order)
        cts.append(ct)
        models.append(p.finish_round(ct, p.K).clone())
    return p, cts, models


def test_medcnn_placement_and_order_do_not_change_the_ciphertext_or_the_model():
    _, cts_a, mod_a = _placement_rounds(1, 3)
    _, cts_b, mod_b = _placement_rounds(3, 1)
    _, cts_c, mod_c = _placement_rounds(1, 3, order=[2, 0, 1])
    for rnd in range(2):
        assert torch.equal(cts_a[rnd], cts_b[rnd]), f"round {rnd}: 1 x 3 and 3 x 1 ciphertexts differ"
        assert torch.equal(mod_a[rnd], mod_b[rnd]), f"round {rnd}: 1 x 3 and 3 x 1 models differ"
        assert torch.equal(cts_a[rnd], cts_c[rnd]), f"round {rnd}: the training order changed the ciphertext"
        assert torch.equal(mod_a[rnd], mod_c[rnd])
    assert not torch.equal(mod_a[0], mod_a[1])


def test_graphs_are_captured_once_per_rank_across_clients_and_rounds():
    run = FederatedRunner(_med(clients_per_rank=3, client_fraction=0.67), device=torch.device("cuda"))
    tr = run.trainer
    calls = []
    orig = tr._capture
    tr._capture = lambda: (calls.append(1), orig())[1]
    l0 = tr.replayed_launches
    run.run_round(check=True)
    graphs = dict(tr._graphs)
    for _ in range(2):
        rec = run.run_round(check=True)
    assert len(calls) == 1, f"{len(calls)} captures"
    assert all(tr._graphs[k] is graphs[k] for k in graphs) and tr.replayed_launches > l0
    assert len(rec["clients"]) == 2 and len(rec["selected"]) == 2


def test_pipelined_round_with_several_clients_equals_the_unchunked_round():
    a = FederatedRunner(_med(clients_per_rank=3), device=torch.device("cuda"))
    b = FederatedRunner(_med(clients_per_rank=3), device=torch.device("cuda"))
    for _ in range(2):
        a.local_train()
        a.decrypt_apply(a.aggregate(a.encrypt_update()))
        a.round += 1
        b.local_train()
        b.fedavg_pipelined(chunk_cts=16)
        b.trainer.engine.after_restore()
        b.round += 1
        assert torch.equal(a.pack.flat, b.pack.flat)


@pytest.mark.multigpu
def test_two_gpus_of_two_clients_equal_one_gpu_of_four(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = str(tmp_path / "model_2x2.pt")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29691", os.path.join(ROOT, "tests", "mp_multiclient_worker.py"),
           "--backend", "nccl", "--clients-per-rank", "2", "--client-fraction", "0.75", "--rounds", "2", "--out", out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    run = FederatedRunner(worker_config(True, 4, 0.75, "fused"), device=torch.device("cuda"))
    for _ in range(2):
        run.run_round(check=True)
    assert torch.equal(torch.load(out).cuda(), run.pack.flat)

"""Several federated clients per rank on CPU (cnn2 28x28, n = 2048 / one prime, cuDNN backend on CPU): placement
independence of the aggregate ciphertext and the global model, order independence inside a rank, per-round client
sampling, checkpoint / resume of every client's state, the host twin of encrypt-accumulate, option validation and a
two-process gloo federation."""
import os
import subprocess
import sys

import pytest
import torch

from hefl_b200.config import FLConfig
from hefl_b200.fl import FederatedRunner
from hefl_b200.fl.runner import check_client_options, select_clients
from hefl_b200.he.context import CKKSContext

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from mp_multiclient_worker import config as worker_config  # noqa: E402

CPU = torch.device("cpu")


def _cfg(**kw):
    base = dict(model="cnn2", image_size=28, in_channels=1, num_classes=10, batch_size=8, local_epochs=1,
                steps_per_epoch=2, val_steps=1, he_preset="n2048_l1", nn_backend="cudnn", dtype="fp32", device="cpu",
                transport="loopback", deterministic_crypto=True, key_holder=-1)
    base.update(kw)
    return FLConfig(**base)


class Placement:
    """W runners of one federation in this process, each in the state a rank of its own process would hold: the
    global torch RNG (CPU and CUDA) is saved and restored around every call, as a separate process would keep it."""

    def __init__(self, world, per_rank, make_cfg=None, device=CPU, **kw):
        self.device = device
        self.runners, self.rng = [], []
        for r in range(world):
            cfg = (make_cfg or _cfg)(clients_per_rank=per_rank, **kw)
            self.runners.append(FederatedRunner(cfg, rank=r, world=world, device=device))
            self.rng.append(self._state())
        self.K = world * per_rank

    def _state(self):
        return torch.get_rng_state(), torch.cuda.get_rng_state(self.device) if self.device.type == "cuda" else None

    def _call(self, r, fn):
        torch.set_rng_state(self.rng[r][0])
        if self.rng[r][1] is not None:
            torch.cuda.set_rng_state(self.rng[r][1], self.device)
        out = fn(self.runners[r])
        self.rng[r] = self._state()
        return out

    def round_ciphertext(self, order=None):
        """local_train + encrypt_update on every rank; the rank buffers summed mod q (what the all-reduce computes)."""
        cts = []
        for r in range(len(self.runners)):
            self._call(r, lambda run: run.local_train(order=order))
            cts.append(self._call(r, lambda run: run.encrypt_update()))
        r0 = self.runners[0]
        if len(cts) == 1:
            return cts[0].data.clone()
        out = torch.empty_like(cts[0].data)
        r0.ctx.ops.local_sum_modq([c.data.contiguous() for c in cts], out, r0.ctx.L, r0.ctx.logn, r0.ctx.consts)
        return out

    def finish_round(self, agg, k):
        """Decrypt the aggregate with the clients' count and install it on every rank (the decode of decrypt_apply)."""
        from hefl_b200.he.context import CtBatch

        r0 = self.runners[0]
        avg = r0.ctx.decrypt(CtBatch(agg, r0.ctx.scale, r0.pack.numel, r0.cfg.packing), r0.sk, divide_by=float(k))
        for run in self.runners:
            run.pack.load_flat(avg)
            if run.trainer.engine is not None:
                run.trainer.engine.after_restore()
            run.round += 1
        return avg


@pytest.fixture(scope="module")
def placements():
    """Two rounds of the same 4-client federation placed as 1 x 4, 2 x 2 and 4 x 1."""
    out = {}
    for world, per in ((1, 4), (2, 2), (4, 1)):
        p = Placement(world, per)
        cts, models = [], []
        for _ in range(2):
            ct = p.round_ciphertext()
            cts.append(ct)
            models.append(p.finish_round(ct, p.K).clone())
        out[(world, per)] = (cts, models)
    return out


@pytest.mark.parametrize("placement", [(2, 2), (4, 1)])
def test_placement_does_not_change_the_ciphertext_or_the_model(placements, placement):
    ref_cts, ref_models = placements[(1, 4)]
    cts, models = placements[placement]
    for rnd in range(2):
        assert torch.equal(cts[rnd], ref_cts[rnd]), f"round {rnd}: aggregate ciphertext words differ"
        assert torch.equal(models[rnd], ref_models[rnd]), f"round {rnd}: global model differs"
    assert not torch.equal(ref_models[0], ref_models[1])


def test_training_order_inside_a_rank_does_not_matter():
    a, b = Placement(1, 4), Placement(1, 4)
    ct_a = a.round_ciphertext()
    ct_b = b.round_ciphertext(order=[2, 0, 3, 1])
    assert torch.equal(ct_a, ct_b)
    ra, rb = a.runners[0], b.runners[0]
    for t in ("_c_m", "_c_v", "_c_step", "_c_lr"):
        assert torch.equal(getattr(ra, t), getattr(rb, t)), t
    assert all(torch.equal(x[0], y[0]) for x, y in zip(ra._c_rng, rb._c_rng))


def test_client_sampling_is_shared_and_leaves_unselected_clients_untouched():
    cfg = _cfg(client_fraction=0.4)
    for rnd in range(4):
        ids = select_clients(cfg, 8, rnd)
        assert len(ids) == 3 and ids == sorted(set(ids)) and all(0 <= i < 8 for i in ids)      # round(3.2) = 3
    assert select_clients(_cfg(client_fraction=0.01), 8, 0).__len__() == 1
    assert len({tuple(select_clients(cfg, 8, r)) for r in range(6)}) > 1
    # every rank of a 2 x 4 federation draws the same ids without communicating
    p = Placement(2, 4, client_fraction=0.4, fedavg_weighting="samples", dirichlet_alpha=0.5)
    for r in range(2):
        p._call(r, lambda run: run.local_train())
    sel = [run._selected for run in p.runners]
    assert sel[0] == sel[1] == select_clients(p.runners[0].cfg, 8, 0)
    # K and N of the decode count the sampled clients only (one rank holding all of them agrees locally)
    one = FederatedRunner(_cfg(clients_per_rank=8, client_fraction=0.4, fedavg_weighting="samples",
                               dirichlet_alpha=0.5), device=CPU)
    rng0 = torch.get_rng_state()                    # what every client starts from (no graphs on CPU)
    before = {k: getattr(one, k).clone() for k in ("_c_m", "_c_v", "_c_step", "_c_lr")}
    gens = [[g.get_state() for g in pair] for pair in one._c_gen]
    rec = one.run_round(check=True)
    chosen = select_clients(one.cfg, 8, 0)
    assert rec["selected"] == chosen and [c["id"] for c in rec["clients"]] == chosen
    assert one._contributors() == len(chosen)
    assert one._n_total == sum(one.clients[i]["n_train"] for i in chosen)
    assert abs(sum(c["fedavg_weight"] for c in rec["clients"]) - len(chosen)) < 1e-9
    for i in range(8):
        same = all(torch.equal(before[k][i], getattr(one, k)[i]) for k in before)
        same_gen = all(torch.equal(a, g.get_state()) for a, g in zip(gens[i], one._c_gen[i]))
        if i in chosen:
            assert not same and not same_gen
        else:
            assert same and same_gen, f"client {i} was not sampled but its state changed"
            assert torch.equal(one._c_rng[i][0], rng0) and one._c_prep[i] == 0


def test_round_record_is_the_sample_weighted_mean_of_the_clients():
    run = FederatedRunner(_cfg(clients_per_rank=3, dirichlet_alpha=0.5), device=CPU)
    rec = run.run_round(check=True)
    cl = rec["clients"]
    assert [c["id"] for c in cl] == [0, 1, 2] and rec["selected"] == [0, 1, 2]
    n = [c["n_train"] for c in cl]
    assert rec["n_train"] == sum(n)
    assert abs(rec["loss"] - sum(a * c["loss"] for a, c in zip(n, cl)) / sum(n)) < 1e-12
    assert rec["label_counts"] == [sum(c["label_counts"][k] for c in cl) for k in range(10)]


def _debug_precision_error(per_rank):
    run = FederatedRunner(_cfg(clients_per_rank=per_rank, debug_precision=True, fedavg_weighting="samples",
                               dirichlet_alpha=0.5), device=CPU)
    return run.run_round(check=True)["ckks_max_abs_err"]


def test_debug_precision_oracle_sums_the_clients():
    assert _debug_precision_error(3) < 1e-6


def test_debug_precision_oracle_of_a_single_one_client_process():
    assert _debug_precision_error(1) < 1e-6


def test_one_client_rank_encrypts_its_installed_model_without_training():
    run = FederatedRunner(_cfg(), device=CPU)
    run.run_round(check=True)
    ct = run.encrypt_update()
    assert float((run.ctx.decrypt(ct, run.sk) - run.pack.flat).abs().max()) < 1e-6


def _resume_at_round_2(tmp_path, per_rank, fraction):
    """The uninterrupted runner after three rounds and one saved after two, resumed and run for the third; their
    global models must be equal."""
    kw = dict(clients_per_rank=per_rank, client_fraction=fraction)
    a = FederatedRunner(_cfg(**kw), device=CPU)
    for _ in range(3):
        a.run_round(check=True)
    b = FederatedRunner(_cfg(**kw), device=CPU)
    for _ in range(2):
        b.run_round(check=True)
    ck = str(tmp_path / "ck.pt")
    b.save_checkpoint(ck)
    c = FederatedRunner(_cfg(**kw), device=CPU)
    c.load_checkpoint(ck)
    assert c.round == 2
    c.run_round(check=True)
    assert torch.equal(a.pack.flat, c.pack.flat)
    return a, c


def test_resumed_run_equals_uninterrupted_run(tmp_path):
    a, c = _resume_at_round_2(tmp_path, 3, 0.67)
    assert torch.equal(a._c_m, c._c_m) and torch.equal(a._c_step, c._c_step)


def test_resumed_one_client_run_with_sampling_equals_uninterrupted_run(tmp_path):
    a, c = _resume_at_round_2(tmp_path, 1, 0.5)
    assert torch.equal(a.trainer.m, c.trainer.m) and torch.equal(a.trainer.step_t, c.trainer.step_t)


def test_dataset_list_must_have_one_dataset_per_client():
    from hefl_b200.fl.data import SyntheticImageDataset

    ds = SyntheticImageDataset(40, 28, 1, 10, seed=0, pin=False)
    with pytest.raises(ValueError, match="one per client"):
        FederatedRunner(_cfg(clients_per_rank=2), device=CPU, dataset=[ds])
    run = FederatedRunner(_cfg(clients_per_rank=2), device=CPU, dataset=[ds, ds])
    assert [c["n_train"] for c in run.clients] == [36, 36]


# ------------------------------------------------------------------ encrypt-accumulate (host twin)
def test_encrypt_accumulate_equals_encrypt_plus_modular_add():
    ctx = CKKSContext(4096, prime_bits=(36, 36, 37), scale_bits=30)
    sk, pk = ctx.keygen(seed=3)
    ops = ctx.ops
    x = torch.randn(3 * 2048 + 17)
    # a larger buffer: the accumulation goes into a chunk view of it at ciphertext offset 2
    C = ctx.num_ct(x.numel())
    per_ct = 2 * ctx.L * ctx.n
    big = ctx.encrypt(torch.randn((C + 3) * 2048), pk, seed=11).data.reshape(-1).clone()
    view = big[2 * per_ct: (2 + C) * per_ct]
    before = view.clone().view(C, 2, ctx.L, ctx.n)
    ctx.encrypt(x, pk, seed=5, out=view, ct_offset=2, weight=0.37, accumulate=True)
    fresh = ctx.encrypt(x, pk, seed=5, ct_offset=2, weight=0.37).data
    ref = before.clone()
    ops.pointwise_(ref, ref, fresh, ctx.L, ctx.consts, 0)
    assert torch.equal(view.view(C, 2, ctx.L, ctx.n), ref)
    # msg=None (an encryption of zero) through the op itself
    acc = fresh.clone()
    ops.encrypt_out(None, pk, C, ctx.L, ctx.logn, ctx.tables, ctx.consts, None, 9, 4, acc, True)
    zero = ops.encrypt(None, pk, C, ctx.L, ctx.logn, ctx.tables, ctx.consts, None, 9, 4)
    ref = fresh.clone()
    ops.pointwise_(ref, ref, zero, ctx.L, ctx.consts, 0)
    assert torch.equal(acc, ref)
    # accumulate=False is the plain encryption, whatever the buffer held
    junk = torch.full_like(fresh, 7)
    ops.encrypt_out(None, pk, C, ctx.L, ctx.logn, ctx.tables, ctx.consts, None, 9, 4, junk)
    assert torch.equal(junk, zero)
    # the decoded sum is the sum of the messages
    two = ctx.encrypt(x, pk, seed=1)
    ctx.encrypt(2 * x, pk, seed=2, out=two.data, accumulate=True)
    assert float((ctx.decrypt(two, sk) - 3 * x).abs().max()) < 1e-4


def test_encrypt_accumulate_needs_an_output_buffer():
    ctx = CKKSContext(2048, prime_bits=(54,), scale_bits=40)
    _, pk = ctx.keygen(seed=1)
    with pytest.raises(ValueError, match="out="):
        ctx.encrypt(torch.randn(10), pk, seed=1, accumulate=True)


# ------------------------------------------------------------------ options
def test_client_options_are_validated_from_flags_and_environment(monkeypatch):
    for argv in (["--clients-per-rank", "0"], ["--client-fraction", "0"], ["--client-fraction", "1.5"],
                 ["--client-fraction", "nan"]):
        cfg = FLConfig.from_args(argv)
        with pytest.raises(ValueError, match="clients_per_rank|client_fraction"):
            check_client_options(cfg)
        with pytest.raises(ValueError, match="clients_per_rank|client_fraction"):
            FederatedRunner(_cfg(clients_per_rank=cfg.clients_per_rank, client_fraction=cfg.client_fraction),
                            device=CPU)
    monkeypatch.setenv("HEFL_CLIENTS_PER_RANK", "4")
    monkeypatch.setenv("HEFL_CLIENT_FRACTION", "0.5")
    cfg = FLConfig.from_args([])
    assert cfg.clients_per_rank == 4 and cfg.client_fraction == 0.5
    check_client_options(cfg)
    monkeypatch.setenv("HEFL_CLIENT_FRACTION", "-0.5")
    with pytest.raises(ValueError, match="client_fraction"):
        check_client_options(FLConfig.from_args([]))
    cfg = FLConfig.from_args(["--client-fraction", "0.25"])      # the flag wins over the environment
    assert cfg.client_fraction == 0.25 and cfg.clients_per_rank == 4


def test_cli_rejects_and_runs_several_clients_per_rank(tmp_path):
    env = dict(os.environ, OMP_NUM_THREADS="2")
    common = [sys.executable, "-m", "hefl_b200", "--device", "cpu", "--model", "cnn2", "--image-size", "28",
              "--in-channels", "1", "--num-classes", "10", "--he-preset", "n2048_l1", "--nn-backend", "cudnn",
              "--dtype", "fp32", "--batch-size", "8", "--local-epochs", "1", "--steps-per-epoch", "2",
              "--val-steps", "1"]
    bad = subprocess.run(common + ["--clients-per-rank", "0"], capture_output=True, text=True, cwd=ROOT, env=env,
                         timeout=600)
    assert bad.returncode != 0 and "clients_per_rank" in bad.stderr
    ok = subprocess.run(common + ["--clients-per-rank", "4", "--client-fraction", "0.5", "--rounds", "2"],
                        capture_output=True, text=True, cwd=ROOT, env=env, timeout=600)
    assert ok.returncode == 0, ok.stderr[-3000:]
    import json

    lines = [json.loads(l) for l in ok.stdout.splitlines() if l.startswith("{")]
    assert [l["round"] for l in lines] == [0, 1]
    for l in lines:
        assert l["clients"] == 4 and len(l["selected"]) == 2
        assert [c["id"] for c in l["rank0_clients"]] == l["selected"]


# ------------------------------------------------------------------ two processes
def test_two_ranks_of_two_clients_equal_one_rank_of_four_gloo(tmp_path):
    out = str(tmp_path / "model.pt")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29681", os.path.join(ROOT, "tests", "mp_multiclient_worker.py"),
           "--backend", "gloo", "--clients-per-rank", "2", "--rounds", "2", "--out", out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT,
                       env=dict(os.environ, OMP_NUM_THREADS="2"))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    # CPU convolutions reduce in an order that depends on the thread count: the reference runs with the workers' 2
    threads = torch.get_num_threads()
    torch.set_num_threads(2)
    try:
        run = FederatedRunner(worker_config(False, 4, 1.0, "loopback"), device=CPU)
        for _ in range(2):
            run.run_round(check=True)
    finally:
        torch.set_num_threads(threads)
    assert torch.equal(torch.load(out), run.pack.flat)

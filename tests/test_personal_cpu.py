"""Personalised federated learning on CPU (cnn2 28x28, n = 2048 / one prime, cuDNN backend on CPU; the medical CNN for
the ciphertext counts): option validation, the shared / personal split of the ciphertext, per-client personal layers
across placements, client sampling and resume, head-only epochs, and the feature switched off."""
import math
import os
import subprocess
import sys

import pytest
import torch

from hefl_b200.config import FLConfig
from hefl_b200.fl import FederatedRunner, simulate_clients
from hefl_b200.fl.runner import check_personal_options, select_clients
from hefl_b200.he.context import CtBatch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from mp_personal_worker import config as worker_config  # noqa: E402

CPU = torch.device("cpu")
SENTINEL = 1e4


def _cfg(**kw):
    base = dict(model="cnn2", image_size=28, in_channels=1, num_classes=10, batch_size=8, local_epochs=1,
                steps_per_epoch=2, val_steps=1, he_preset="n2048_l1", nn_backend="cudnn", dtype="fp32", device="cpu",
                transport="loopback", deterministic_crypto=True, key_holder=-1)
    base.update(kw)
    return FLConfig(**base)


def _pcfg(**kw):
    return _cfg(**{"personal_layers": 1, "personal_head_epochs": 1, **kw})


# ------------------------------------------------------------------ options
@pytest.mark.parametrize("argv,match", [
    (["--personal-layers", "-1"], "personal_layers"),
    (["--personal-layers", "4"], "at most 3"),
    (["--model", "cnn2", "--personal-layers", "2"], "at most 1"),
    (["--model", "resnet18", "--personal-layers", "1"], "sequential CNNs"),
    (["--model", "resnet50", "--personal-layers", "1"], "sequential CNNs"),
    (["--personal-head-epochs", "2"], "needs personal_layers > 0"),
    (["--personal-layers", "1", "--personal-head-epochs", "-1"], "personal_head_epochs"),
    (["--personal-layers", "1", "--compat-sequential-clients", "1"], "compat_sequential_clients"),
])
def test_personal_options_are_rejected_from_flags(argv, match):
    cfg = FLConfig.from_args(argv)
    with pytest.raises(ValueError, match=match):
        check_personal_options(cfg)


def test_personal_options_from_environment_and_the_runner(monkeypatch):
    monkeypatch.setenv("HEFL_PERSONAL_LAYERS", "3")
    monkeypatch.setenv("HEFL_PERSONAL_HEAD_EPOCHS", "2")
    cfg = FLConfig.from_args([])
    assert cfg.personal_layers == 3 and cfg.personal_head_epochs == 2
    check_personal_options(cfg)                                  # medcnn has three Dense layers
    assert FLConfig.from_args(["--personal-layers", "1"]).personal_layers == 1     # the flag wins
    monkeypatch.setenv("HEFL_PERSONAL_LAYERS", "0")
    with pytest.raises(ValueError, match="needs personal_layers > 0"):
        check_personal_options(FLConfig.from_args([]))
    with pytest.raises(ValueError, match="at most 1"):
        FederatedRunner(_cfg(personal_layers=2), device=CPU)
    with pytest.raises(ValueError, match="compat_sequential_clients"):
        FederatedRunner(_cfg(personal_layers=1, compat_sequential_clients=True), device=CPU)
    with pytest.raises(ValueError, match="FederatedRunner"):
        simulate_clients(_cfg(personal_layers=1))


def test_cli_rejects_personal_layers_of_a_resnet():
    r = subprocess.run([sys.executable, "-m", "hefl_b200", "--device", "cpu", "--model", "resnet18",
                        "--personal-layers", "1"], capture_output=True, text=True, cwd=ROOT, timeout=600,
                       env=dict(os.environ, OMP_NUM_THREADS="2"))
    assert r.returncode != 0 and "sequential CNNs" in r.stderr


# ------------------------------------------------------------------ ciphertext counts
@pytest.mark.parametrize("packing", ["slots", "coeff"])
def test_ciphertext_count_covers_the_shared_base(packing):
    personal = {0: 0, 1: 130, 2: 8_386, 3: 74_050}
    slots_ct = {0: 109, 1: 109, 2: 105, 3: 73}
    for p, n_personal in personal.items():
        run = FederatedRunner(_cfg(model="medcnn", image_size=256, in_channels=3, num_classes=2, batch_size=2,
                                   steps_per_epoch=1, val_steps=1, he_preset="n4096_l3", packing=packing,
                                   personal_layers=p), device=CPU)
        assert run.pack.numel == 222_722 and run.n_personal == n_personal
        assert run.n_shared == 222_722 - n_personal
        assert run.n_ct == math.ceil(run.n_shared / run.ctx.values_per_ct(packing))
        if packing == "slots":
            assert run.n_ct == slots_ct[p]


# ------------------------------------------------------------------ the round
def _record_heads(run):
    """Wrap the trainer's fit so that the personal layers each client ends its round with are recorded."""
    trained, fit = {}, run.trainer.fit

    def wrapped(*a, **kw):
        hist = fit(*a, **kw)
        if not kw.get("head_only"):
            trained[len(trained)] = run.pack.flat[run.n_shared:].clone()
        return hist

    run.trainer.fit = wrapped
    return trained


def test_personal_layers_never_enter_the_ciphertext():
    run = FederatedRunner(_pcfg(clients_per_rank=2), device=CPU)
    run._c_head.fill_(SENTINEL)
    run.pack.flat[run.n_shared:].fill_(SENTINEL)
    trained = _record_heads(run)
    run.local_train()
    ct = run.encrypt_update()
    assert ct.nvals == run.n_shared and ct.data.shape[0] == run.n_ct
    agg = run.aggregate(ct)
    avg = run.ctx.decrypt(agg, run.sk, divide_by=2.0)
    assert avg.numel() == run.n_shared
    assert float(avg.abs().max()) < 10.0, "a personal layer leaked into the aggregate"
    run.decrypt_apply(agg)
    assert torch.equal(run.shared(), avg)
    for i in range(2):
        assert torch.equal(run._c_head[i], trained[i]), f"client {i}: personal layers differ from the trained ones"
        assert float((trained[i] - SENTINEL).abs().max()) < 1.0          # trained from the sentinel, a few Adam steps
    assert torch.equal(run.pack.flat[run.n_shared:], trained[1])      # the last trained client's stay installed


@pytest.mark.parametrize("per_rank", [1, 3])
def test_debug_precision_error_covers_the_shared_base(per_rank):
    run = FederatedRunner(_pcfg(clients_per_rank=per_rank, debug_precision=True, dirichlet_alpha=0.5,
                                fedavg_weighting="samples"), device=CPU)
    run._heads().fill_(SENTINEL)
    rec = run.run_round(check=True)
    assert rec["ckks_max_abs_err"] < 1e-6
    assert "val_accuracy" in rec
    if per_rank > 1:
        assert all("val_accuracy" in c for c in rec["clients"])


class Placement:
    """W runners of one federation in this process, each with the torch RNG state its own process would keep."""

    def __init__(self, world, per_rank, make_cfg=None, device=CPU, **kw):
        self.device = device
        self.runners, self.rng = [], []
        for r in range(world):
            self.runners.append(FederatedRunner((make_cfg or _pcfg)(clients_per_rank=per_rank, **kw), rank=r,
                                                world=world, device=device))
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

    def round(self):
        """One round: every rank's ciphertext, their sum mod q, its decryption installed everywhere."""
        cts = []
        for r in range(len(self.runners)):
            self._call(r, lambda run: run.local_train())
            cts.append(self._call(r, lambda run: run.encrypt_update()).data.clone())
        r0 = self.runners[0]
        agg = cts[0]
        if len(cts) > 1:
            agg = torch.empty_like(cts[0])
            r0.ctx.ops.local_sum_modq([c.contiguous() for c in cts], agg, r0.ctx.L, r0.ctx.logn, r0.ctx.consts)
        avg = r0.ctx.decrypt(CtBatch(agg, r0.ctx.scale, r0.n_shared, r0.cfg.packing), r0.sk, divide_by=float(self.K))
        for run in self.runners:
            run._install_shared(avg)
            if run.trainer.engine is not None:
                run.trainer.engine.after_restore()
            run.round += 1
        return agg, avg.clone(), torch.cat([run._heads() for run in self.runners]).clone()


@pytest.fixture(scope="module")
def placements():
    out = {}
    for world, per in ((1, 4), (2, 2), (4, 1)):
        p = Placement(world, per)
        out[(world, per)] = [p.round() for _ in range(2)]
    return out


@pytest.mark.parametrize("placement", [(2, 2), (4, 1)])
def test_placement_does_not_change_ciphertexts_bases_or_heads(placements, placement):
    ref, got = placements[(1, 4)], placements[placement]
    for rnd in range(2):
        for name, a, b in zip(("ciphertext", "base", "heads"), ref[rnd], got[rnd]):
            assert torch.equal(a, b), f"round {rnd}: {name} differs"
    heads = ref[1][2]
    assert not torch.equal(heads[0], heads[1]), "two clients ended with the same personal layers"


def test_two_gloo_ranks_of_two_clients_equal_one_rank_of_four(tmp_path):
    out = str(tmp_path / "personal.pt")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29683", os.path.join(ROOT, "tests", "mp_personal_worker.py"),
           "--clients-per-rank", "2", "--rounds", "2", "--out", out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT,
                       env=dict(os.environ, OMP_NUM_THREADS="2"))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    threads = torch.get_num_threads()
    torch.set_num_threads(2)                       # CPU convolutions reduce in a thread-count dependent order
    try:
        run = FederatedRunner(worker_config(4, "loopback"), device=CPU)
        for _ in range(2):
            run.run_round(check=True)
    finally:
        torch.set_num_threads(threads)
    for rank in range(2):
        st = torch.load(f"{out}.rank{rank}")
        assert st["ids"] == [2 * rank, 2 * rank + 1]
        assert torch.equal(st["base"], run.shared())
        assert torch.equal(st["heads"], run._c_head[2 * rank: 2 * rank + 2])


def test_unselected_clients_keep_their_personal_layers():
    run = FederatedRunner(_pcfg(clients_per_rank=6, client_fraction=0.5), device=CPU)
    for rnd in range(2):
        before = run._c_head.clone()
        run.run_round(check=True)
        chosen = select_clients(run.cfg, 6, rnd)
        for i in range(6):
            same = torch.equal(before[i], run._c_head[i])
            assert same == (i not in chosen), f"round {rnd}, client {i}"
    never = set(range(6)) - set(select_clients(run.cfg, 6, 0)) - set(select_clients(run.cfg, 6, 1))
    for i in never:
        assert torch.equal(run._c_head[i], run.head0)


def test_resumed_run_with_personal_layers_equals_uninterrupted_run(tmp_path):
    kw = dict(clients_per_rank=2)
    a = FederatedRunner(_pcfg(**kw), device=CPU)
    for _ in range(3):
        a.run_round(check=True)
    b = FederatedRunner(_pcfg(**kw), device=CPU)
    for _ in range(2):
        b.run_round(check=True)
    ck = str(tmp_path / "ck.pt")
    b.save_checkpoint(ck)
    assert torch.equal(torch.load(ck)["flat"][b.n_shared:], b.head0), "the global file holds a client's head"
    c = FederatedRunner(_pcfg(**kw), device=CPU)
    c.load_checkpoint(ck)
    assert torch.equal(c._c_head, b._c_head)
    c.run_round(check=True)
    assert torch.equal(a.pack.flat, c.pack.flat) and torch.equal(a._c_head, c._c_head)
    assert torch.equal(a._c_m, c._c_m) and torch.equal(a._c_step, c._c_step)
    # a rank without a state file restarts its clients from head0
    os.remove(f"{ck}.rank0")
    d = FederatedRunner(_pcfg(**kw), device=CPU)
    d._c_head.fill_(SENTINEL)
    d.load_checkpoint(ck)
    assert torch.equal(d._c_head, d.head0.expand(2, -1))


def test_evaluate_installs_the_clients_head_and_restores_the_installed_one():
    from hefl_b200.fl.data import SyntheticImageDataset

    run = FederatedRunner(_pcfg(clients_per_rank=2), device=CPU)
    run.run_round(check=True)
    test = SyntheticImageDataset(32, 28, 1, 10, seed=5, pin=False)
    installed = run.pack.flat.clone()
    scores = [run.evaluate(test, client=i) for i in range(2)]
    assert torch.equal(run.pack.flat, installed)
    run.pack.flat[run.n_shared:].copy_(run._c_head[0])
    assert run.evaluate(test) == scores[0]
    with pytest.raises(ValueError, match="slot"):
        run.evaluate(test, client=2)


# ------------------------------------------------------------------ the feature switched off
def test_personal_layers_zero_is_todays_round():
    def two_rounds(cfg):                          # one runner after the other: they share the global torch RNG
        run = FederatedRunner(cfg, device=CPU)
        recs = [run.run_round(check=True) for _ in range(2)]
        for r in recs:
            r.pop("stage_ms")
        return run, recs, run.encrypt_update()

    a, ra, ca = two_rounds(_cfg(clients_per_rank=2))
    b, rb, cb = two_rounds(_cfg(clients_per_rank=2, personal_layers=0, personal_head_epochs=0))
    assert b.n_shared == b.pack.numel and b.head0 is None
    assert torch.equal(a.pack.flat, b.pack.flat)
    assert ra == rb and all("val_accuracy" not in r and "val_accuracy" not in r["clients"][0] for r in ra)
    assert torch.equal(ca.data, cb.data) and ca.nvals == cb.nvals == a.pack.numel


# ------------------------------------------------------------------ head-only epochs (the CPU reference)
def test_head_only_epochs_leave_the_shared_base_and_its_adam_state():
    run = FederatedRunner(_pcfg(personal_head_epochs=0, fedprox_mu=0.01), device=CPU)
    tr = run.trainer
    run.trainer.fit(run.train_feed, run.val_feed, 1)                    # non-zero Adam state everywhere
    base, m, v = run.shared().clone(), tr.m.clone(), tr.v.clone()
    head, step = run.pack.flat[run.n_shared:].clone(), int(tr.step_t)
    hist = tr.fit(run.train_feed, run.val_feed, 2, head_only=True)
    lo = run.n_shared
    assert len(hist) == 2 and all(math.isfinite(h.loss) and 0 <= h.accuracy <= 1 for h in hist)
    assert torch.equal(run.shared(), base)
    assert torch.equal(tr.m[:lo], m[:lo]) and torch.equal(tr.v[:lo], v[:lo])
    assert not torch.equal(run.pack.flat[lo:], head) and not torch.equal(tr.m[lo:], m[lo:])
    assert int(tr.step_t) == step + 2 * run.cfg.steps_per_epoch
    assert float(tr.pack.grad.abs().max()) == 0.0

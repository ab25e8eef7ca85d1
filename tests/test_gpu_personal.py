"""Personalised federated learning on the H100: the head kernels' backward depths against the full backward (cluster
kernel and four-kernel fallback), the engine's head-only step against a full training step, graph-replayed against
eager, and the medical CNN federation with personal Dense layers on the tcgen05 engine with CUDA graphs."""
import pytest
import torch

from hefl_b200 import _ext
from hefl_b200.config import FLConfig
from hefl_b200.fl import FederatedRunner
from hefl_b200.fl.trainer import LocalTrainer
from hefl_b200.models import ParamPack, create_model
from test_personal_cpu import Placement

ops = _ext.ops()
pytestmark = pytest.mark.gpu
SENTINEL = 12345.0
CUDA = torch.device("cuda")


# ------------------------------------------------------------------ head kernel depths
def _head_case(Fdim, B, C=2, H1=128, H2=64):
    g = torch.Generator(device="cuda").manual_seed(Fdim + B)
    sizes = [H1 * Fdim, H1, H2 * H1, H2, C * H2, C]
    offs = [0]
    for n in sizes[:-1]:
        offs.append(offs[-1] + n)
    flat = torch.randn(sum(sizes), device="cuda", generator=g) * 0.05
    feat = (torch.rand(B, Fdim, device="cuda", generator=g)).to(torch.bfloat16)
    y = torch.randint(0, C, (B,), device="cuda", generator=g)
    return flat, feat, y, offs, sizes, (B, Fdim, H1, H2, C)


def _run_head(flat, feat, y, offs, dims, depth):
    B, Fdim, H1, H2, C = dims
    grad = torch.full_like(flat, SENTINEL)
    dfeat = torch.full((B, Fdim), SENTINEL, dtype=torch.bfloat16, device="cuda")
    h1_buf = torch.zeros(B * H1, device="cuda")
    dh1_buf = torch.zeros(B * (H1 + H2), device="cuda")
    out = torch.zeros(2, device="cuda")
    ops.head_forward_backward(feat, flat, grad, offs, y, dfeat, h1_buf, dh1_buf, out, B, Fdim, H1, H2, C, depth)
    torch.cuda.synchronize()
    return grad, dfeat, out


@pytest.mark.parametrize("Fdim", [512, 256])          # 512: the cluster kernel; 256: the four-kernel fallback
@pytest.mark.parametrize("B", [32, 2])
@pytest.mark.parametrize("depth", [2, 3, 4])
def test_head_depth_gradients_equal_the_full_backward(Fdim, B, depth):
    flat, feat, y, offs, sizes, dims = _head_case(Fdim, B)
    g1, d1, o1 = _run_head(flat, feat, y, offs, dims, 1)
    gd, dd, od = _run_head(flat, feat, y, offs, dims, depth)
    assert torch.equal(o1, od)
    assert not torch.equal(d1, torch.full_like(d1, SENTINEL))
    assert torch.equal(dd, torch.full_like(dd, SENTINEL)), "dfeat was written"
    first = 2 * (depth - 2)                   # depth 2: W1 on, depth 3: W2 on, depth 4: W3 on
    for t, (o, n) in enumerate(zip(offs, sizes)):
        if t >= first:
            assert torch.equal(gd[o:o + n], g1[o:o + n]), f"depth {depth}: gradient tensor {t} differs"
        else:
            assert torch.equal(gd[o:o + n], torch.full_like(gd[o:o + n], SENTINEL)), f"tensor {t} was written"


# ------------------------------------------------------------------ the engine's head-only step
class _Hooks:
    """An ``opt`` that updates nothing and records the range it was asked to update."""

    def __init__(self):
        self.bumps, self.ranges = 0, []

    def bump(self):
        self.bumps += 1

    def apply(self, lo, hi):
        self.ranges.append((lo, hi))


def _medcnn_cfg(**kw):
    return FLConfig(**{"model": "medcnn", "batch_size": 32, "nn_backend": "tcgen05", "device": "cuda", **kw})


def _trainer(p, use_graph, seed=3):
    cfg = _medcnn_cfg(personal_layers=p, personal_head_epochs=1)
    torch.manual_seed(seed)
    model = create_model("medcnn", 3, 2, 256).to(CUDA)
    pack = ParamPack(model)
    return LocalTrainer(model, pack, cfg, CUDA, use_graph=use_graph)


def _batch(seed=7):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randint(0, 256, (32, 256, 256, 3), device="cuda", generator=g, dtype=torch.int64).to(torch.uint8)
    y = torch.randint(0, 2, (32,), device="cuda", generator=g)
    return x, y


@pytest.mark.parametrize("p", [1, 2, 3])
def test_engine_head_step_gradients_equal_the_full_step(p):
    tr = _trainer(p, use_graph=False)
    eng, pack = tr.engine, tr.pack
    x, y = _batch()
    eng.preprocess(x, 0, True, True)
    out_full = torch.zeros(2, device="cuda")
    eng.train_step_staged(0, y, out_full)                   # no opt: every gradient, nothing updated
    full = pack.grad.clone()
    pack.grad.zero_()
    wf, wd, flat = eng.Wf.clone(), eng.Wd.clone(), pack.flat.clone()
    hooks, out = _Hooks(), torch.zeros(2, device="cuda")
    eng.head_step_staged(0, y, out, hooks)
    torch.cuda.synchronize()
    lo = eng.head_lo
    assert hooks.bumps == 1 and hooks.ranges == [(lo, pack.n_trainable)]
    assert lo == pack.n_trainable - {1: 130, 2: 8_386, 3: 74_050}[p]
    assert torch.equal(pack.grad[lo:], full[lo:]), "head gradients differ from the full step's"
    assert float(pack.grad[:lo].abs().max()) == 0.0
    assert torch.equal(out, out_full)
    assert torch.equal(eng.Wf, wf) and torch.equal(eng.Wd, wd) and torch.equal(pack.flat, flat)


@pytest.mark.parametrize("p", [1, 3])
def test_head_step_updates_only_the_personal_layers_and_replays_as_it_runs_eagerly(p):
    x, y = _batch(11)
    res = []
    for use_graph in (False, True):
        tr = _trainer(p, use_graph)
        eng, pack = tr.engine, tr.pack
        lo = tr.head_lo
        wf, wd, base = eng.Wf.clone(), eng.Wd.clone(), pack.flat[:lo].clone()
        head = pack.flat[lo:].clone()
        losses = [float(tr.head_step(x, y)[0]) for _ in range(3)]
        torch.cuda.synchronize()
        assert torch.equal(eng.Wf, wf) and torch.equal(eng.Wd, wd) and torch.equal(pack.flat[:lo], base)
        assert float(tr.m[:lo].abs().max()) == 0.0 and float(tr.v[:lo].abs().max()) == 0.0
        assert not torch.equal(pack.flat[lo:], head) and int(tr.step_t) == 3
        res.append((pack.flat.clone(), tr.m.clone(), tr.v.clone(), losses))
        if use_graph:
            assert ("head", 0) in tr._graphs and tr.head_launches > 0
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1]) and torch.equal(res[0][2], res[1][2])
    assert res[0][3] == res[1][3]


# ------------------------------------------------------------------ the federation
def _med(**kw):
    base = dict(model="medcnn", local_epochs=1, steps_per_epoch=2, val_steps=1, nn_backend="tcgen05", device="cuda",
                transport="loopback", deterministic_crypto=True, key_holder=-1, personal_layers=3,
                personal_head_epochs=1)
    base.update(kw)
    return FLConfig(**base)


def test_medcnn_placement_does_not_change_ciphertexts_bases_or_heads():
    a = Placement(1, 3, make_cfg=_med, device=CUDA)
    b = Placement(3, 1, make_cfg=_med, device=CUDA)
    assert a.runners[0].n_ct == 73
    for rnd in range(2):
        ra, rb = a.round(), b.round()
        for name, u, v in zip(("ciphertext", "base", "heads"), ra, rb):
            assert torch.equal(u, v), f"round {rnd}: 1 x 3 and 3 x 1 {name} differ"
    heads = ra[2]
    assert not torch.equal(heads[0], heads[1]) and not torch.equal(heads[0], a.runners[0].head0)


def test_medcnn_pipelined_round_equals_the_unchunked_round():
    a = FederatedRunner(_med(clients_per_rank=3), device=CUDA)
    b = FederatedRunner(_med(clients_per_rank=3), device=CUDA)
    for _ in range(2):
        a.run_round(pipelined=False)
        b.run_round(pipelined=True)
        assert torch.equal(a.pack.flat, b.pack.flat) and torch.equal(a._c_head, b._c_head)
    b.local_train()
    b.fedavg_pipelined(chunk_cts=16)                         # several chunks of the 73 ciphertexts
    a.local_train()
    a.decrypt_apply(a.aggregate(a.encrypt_update()))
    assert torch.equal(a.pack.flat, b.pack.flat)


def test_medcnn_graphs_are_captured_once_per_rank():
    run = FederatedRunner(_med(clients_per_rank=3, client_fraction=0.67), device=CUDA)
    tr = run.trainer
    calls = []
    orig, orig_head = tr._capture, tr._capture_head
    tr._capture = lambda: (calls.append("train"), orig())[1]
    tr._capture_head = lambda: (calls.append("head"), orig_head())[1]
    rec = run.run_round(check=True)
    graphs = dict(tr._graphs)
    for _ in range(2):
        rec = run.run_round(check=True)
    assert sorted(calls) == ["head", "train"], calls
    assert len(graphs) == 6 and all(tr._graphs[k] is graphs[k] for k in graphs)
    assert all(0 <= c["val_accuracy"] <= 1 for c in rec["clients"])


def test_default_run_captures_no_head_graphs():
    run = FederatedRunner(_med(personal_layers=0, personal_head_epochs=0), device=CUDA)
    run.run_round(check=True)
    assert sorted(k for k in run.trainer._graphs if k[0] == "head") == [] and run.trainer.head_launches == 0

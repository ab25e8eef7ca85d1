"""Federated evaluation on the H100 (DESIGN.md §13): the head_logits op against float64 on both head paths, the
score_stats kernel against score_counts_torch on its own logits and probs, LocalTrainer.score graph-replayed and eager
against each other and against the float64 model, training left bit-identical around evaluate_federated, and a
medical-CNN round on the fused transport that decodes exact counts."""
import copy

import pytest
import torch
import torch.nn.functional as F

from hefl_b200 import _ext
from hefl_b200.config import FLConfig
from hefl_b200.fl import FederatedRunner
from hefl_b200.fl.data import BatchFeeder, SyntheticImageDataset
from hefl_b200.fl.fedeval import count_len, metrics_from_counts, score_counts_torch

ops = _ext.ops()
pytestmark = pytest.mark.gpu
CUDA = torch.device("cuda")
SENTINEL = -12345.0
# calibrated on the H100 (test_score_pass_graph_equals_eager_and_float64): the engine's bf16 logits of the seeded
# medical CNN differed from the float64 model's by at most 2.7e-4; scans whose float64 top-2 margin is below this may
# change class
MARGIN = 1e-2


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _head_case(Fdim, B, C, seed):
    H1, H2 = 128, 64
    g = _gen(seed)
    sizes = [H1 * Fdim, H1, H2 * H1, H2, C * H2, C]
    offs = [0]
    for n in sizes[:-1]:
        offs.append(offs[-1] + n)
    flat = torch.randn(sum(sizes), device="cuda", generator=g) * 0.05
    feat = torch.rand(B, Fdim, device="cuda", generator=g).to(torch.bfloat16)
    ps = [flat[o:o + n].double().view(-1) for o, n in zip(offs, sizes)]
    h = F.relu(F.linear(feat.double(), ps[0].view(H1, Fdim), ps[1]))
    h = F.relu(F.linear(h, ps[2].view(H2, H1), ps[3]))
    return flat, offs, feat, F.linear(h, ps[4].view(C, H2), ps[5]), H1, H2


@pytest.mark.parametrize("Fdim,B,C", [(512, 32, 2), (512, 7, 3), (512, 1, 4), (256, 32, 2), (256, 6, 3)])
def test_head_logits_matches_float64(Fdim, B, C):
    """F = 512 runs the cluster kernel (one launch, any B), F = 256 the fallback (k1 and k2 only, even B)."""
    flat, offs, feat, ref, H1, H2 = _head_case(Fdim, B, C, seed=Fdim + 7 * B + C)
    h1_buf = torch.zeros(B * H1, device="cuda")
    dh1_buf = torch.full((B * (H1 + H2),), SENTINEL, device="cuda")
    logits = torch.full((B, C), SENTINEL, device="cuda")
    flat0 = flat.clone()
    n0 = int(ops.launch_count())
    ops.head_logits(feat, flat, offs, h1_buf, dh1_buf, logits, B, Fdim, H1, H2, C)
    torch.cuda.synchronize()
    assert int(ops.launch_count()) - n0 == (1 if Fdim == 512 else 2)
    assert (logits.double() - ref).abs().max() <= 1e-4
    assert torch.equal(flat, flat0)
    assert bool((dh1_buf == SENTINEL).all()), "the forward-only head wrote backward scratch"


def _score_inputs(B, C, seed, nan_from=None):
    g = _gen(seed)
    logits = torch.randn(B, C, device="cuda", generator=g) * 3
    logits[: B // 4, 0] = logits[: B // 4, 1]                 # ties: the lowest index wins
    labels = torch.randint(0, C, (B,), device="cuda", generator=g)
    if nan_from is not None:
        logits[nan_from:] = float("nan")
        labels[nan_from:] = 10 ** 6                           # would raise the flag if it were read
    return logits, labels


def _score_bufs(B, C, nbins):
    return (torch.zeros(C * C * (nbins + 1), dtype=torch.int32, device="cuda"),
            torch.zeros(1, dtype=torch.float64, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda"),
            torch.full((B, C), SENTINEL, device="cuda"))


@pytest.mark.parametrize("B,C,nbins", [(32, 2, 100), (37, 5, 7), (300, 32, 1024), (1, 3, 2)])
def test_score_stats_matches_score_counts_torch(B, C, nbins):
    logits, labels = _score_inputs(B, C, seed=B * 31 + C)
    counts, loss, err, probs = _score_bufs(B, C, nbins)
    nv = torch.tensor([B], dtype=torch.int32, device="cuda")
    n0 = int(ops.launch_count())
    ops.score_stats(logits, labels, nv, probs, counts, loss, err, nbins)
    torch.cuda.synchronize()
    assert int(ops.launch_count()) - n0 == 1 and int(err) == 0
    assert (probs.double() - torch.softmax(logits.double(), 1)).abs().max() <= 1e-6
    ref = score_counts_torch(logits.cpu(), labels.cpu(), nbins, probs=probs.cpu())
    assert torch.equal(counts.cpu().double(), ref[:-1])
    assert abs(float(loss) - float(ref[-1])) <= 1e-9 * max(1.0, abs(float(ref[-1])))
    assert int(counts[: C * C].sum()) == B and int(counts[C * C:].sum()) == B * C


def test_score_stats_nvalid_accumulation_and_determinism():
    """Rows >= nvalid hold NaN logits and out-of-range labels: neither read nor written. Two launches add up, and the
    loss sum has the same bits on every run."""
    B, C, nb, nvalid = 32, 3, 50, 19
    logits, labels = _score_inputs(B, C, seed=5, nan_from=nvalid)
    counts, loss, err, probs = _score_bufs(B, C, nb)
    nv = torch.tensor([nvalid], dtype=torch.int32, device="cuda")
    ops.score_stats(logits, labels, nv, probs, counts, loss, err, nb)
    torch.cuda.synchronize()
    assert int(err) == 0
    assert bool((probs[nvalid:] == SENTINEL).all())
    ref = score_counts_torch(logits[:nvalid].cpu(), labels[:nvalid].cpu(), nb, probs=probs[:nvalid].cpu())
    assert torch.equal(counts.cpu().double(), ref[:-1])
    first = loss.clone()
    ops.score_stats(logits, labels, nv, probs, counts, loss, err, nb)
    assert torch.equal(counts.cpu().double(), 2 * ref[:-1])
    for _ in range(5):
        c2, l2, e2, p2 = _score_bufs(B, C, nb)
        ops.score_stats(logits, labels, nv, p2, c2, l2, e2, nb)
        assert torch.equal(l2, first) and torch.equal(c2.double(), ref[:-1].cuda())
    nv.fill_(0)
    before = counts.clone()
    ops.score_stats(logits, labels, nv, probs, counts, loss, err, nb)
    assert torch.equal(counts, before)


def test_score_stats_flags_bad_labels():
    B, C, nb = 8, 2, 10
    logits, labels = _score_inputs(B, C, seed=9)
    labels[3] = 2
    counts, loss, err, probs = _score_bufs(B, C, nb)
    ops.score_stats(logits, labels, torch.tensor([B], dtype=torch.int32, device="cuda"), probs, counts, loss, err, nb)
    torch.cuda.synchronize()
    assert int(err) == 1 and int(counts.sum()) == (B - 1) * (1 + C)
    with pytest.raises(RuntimeError, match="classes"):
        ops.score_stats(torch.zeros(2, 33, device="cuda"), labels[:2], torch.tensor([2], dtype=torch.int32, device="cuda"),
                        torch.zeros(2, 33, device="cuda"), torch.zeros(33 * 33 * 11, dtype=torch.int32, device="cuda"),
                        loss, err, 10)
    with pytest.raises(RuntimeError, match="nbins"):
        ops.score_stats(logits, labels, torch.tensor([B], dtype=torch.int32, device="cuda"), probs,
                        torch.zeros(C * C * 1026, dtype=torch.int32, device="cuda"), loss, err, 1025)


# ------------------------------------------------------------------ the trainer and the runner
def _cfg(**kw):
    return FLConfig(model="medcnn", local_epochs=1, steps_per_epoch=2, val_steps=1, deterministic_crypto=True, **kw)


def test_score_pass_graph_equals_eager_and_float64():
    """100 scans: three full batches and a wrapped fourth. The graph-replayed pass and the eager pass give the same
    counts bit for bit, n = 100, and the predictions differ from the float64 model's only where its margin is small."""
    ds = SyntheticImageDataset(100, 256, 3, 2, seed=11, pin=True)
    run = FederatedRunner(_cfg(), device=CUDA)
    tr = run.trainer
    assert tr.use_graph and tr.engine is not None and not tr._score_graphs
    V = count_len(2, 100)
    feed = BatchFeeder(ds, range(100), 32, CUDA, shuffle=False)
    row_g = torch.zeros(V, dtype=torch.float64, device=CUDA)
    l0 = tr.replayed_launches
    tr.score(feed, row_g)
    assert len(tr._score_graphs) == 2 and tr.replayed_launches - l0 == 4 * tr.score_launches
    assert tr.score_launches == 9, "pre-processing, six forward convs, head_logits and score_stats"
    tr.use_graph = False
    row_e = torch.zeros(V, dtype=torch.float64, device=CUDA)
    tr.score(feed, row_e)
    tr.use_graph = True
    assert torch.equal(row_g, row_e)
    m = metrics_from_counts(row_g.cpu(), 2, 100)
    assert m["n"] == 100
    ref = copy.deepcopy(run.model).double().eval()
    with torch.no_grad():
        logits = ref(ds.images.to(CUDA).permute(0, 3, 1, 2).double() / 255.0)
    conf = torch.zeros(2, 2, dtype=torch.int64)
    for t, p in zip(ds.labels.tolist(), logits.argmax(1).tolist()):
        conf[t, p] += 1
    top2 = logits.topk(2, 1).values
    close = int(((top2[:, 0] - top2[:, 1]) < MARGIN).sum())
    assert int((torch.tensor(m["confusion"]) - conf).abs().sum()) <= 2 * close
    eng_last = tr.engine.score_logits[:4].double()               # rows 96..99 of the last batch
    diff = float((eng_last - logits[96:]).abs().max())
    print(f"engine vs float64 logits, last batch: max |diff| = {diff:.3g}; scans within the margin: {close}")
    assert diff <= MARGIN / 2


def _state(run):
    tr = run.trainer
    return [run.pack.flat.clone(), tr.m.clone(), tr.v.clone(), tr.step_t.clone(), tr.lr_scale.clone(), tr.engine.dW32.clone()]


def _train(run, steps, seed):
    ds = SyntheticImageDataset(run.cfg.batch_size * steps, 256, 3, 2, seed=seed, pin=False)
    losses = []
    B = run.cfg.batch_size
    for i in range(steps):
        out = run.trainer.train_step(ds.images[i * B:(i + 1) * B].to(CUDA), ds.labels[i * B:(i + 1) * B].to(CUDA))
        losses.append(out.clone())
    torch.cuda.synchronize()
    return losses


@pytest.mark.parametrize("personal", [False, True])
def test_evaluate_federated_leaves_training_bit_identical(personal):
    """3 steps, evaluate_federated, 3 steps equals 6 steps without it: weights, gradient accumulator, loss, Adam state,
    augmentation position, the torch RNG and the graphs' launch counts; with personal layers every client scores with
    its own head. A run that never scores captures no score graph."""
    kw = dict(personal_layers=1, clients_per_rank=2) if personal else {}
    tests = [SyntheticImageDataset(n, 256, 3, 2, seed=20 + n, pin=True) for n in ((45, 7) if personal else (45,))]
    results = []
    for ev in (True, False):
        run = FederatedRunner(_cfg(**kw), device=CUDA, test_dataset=tests)
        if personal:
            run._c_head[1].add_(0.01)
        losses = _train(run, 3, seed=5)
        if ev:
            fed = run.evaluate_federated()
            assert fed["n"] == sum(len(t) for t in tests)
        losses += _train(run, 3, seed=6)
        results.append((_state(run), torch.stack(losses).cpu(), run.trainer.engine.prep_count,
                        torch.get_rng_state(), torch.cuda.get_rng_state(), list(run.trainer.graph_launches)))
        if not ev:
            assert not run.trainer._score_graphs, "a run that never scores captured score graphs"
    (s1, l1, c1, r1, g1, n1), (s2, l2, c2, r2, g2, n2) = results
    assert all(torch.equal(a, b) for a, b in zip(s1, s2))
    assert torch.equal(l1, l2) and c1 == c2
    assert torch.equal(r1, r2) and torch.equal(g1, g2)
    assert n1 == n2


def test_medcnn_round_decodes_exact_counts():
    """One round on the fused transport with fed_eval_every = 1 and two clients, one without scans: the decoded counts
    are the sum of the clients' plaintext counts, exactly."""
    tests = [SyntheticImageDataset(n, 256, 3, 2, seed=40 + n, pin=True) for n in (33, 0)]
    run = FederatedRunner(_cfg(fed_eval_every=1, clients_per_rank=2), device=CUDA, test_dataset=tests)
    assert run.transport.name == "fused"
    rec = run.run_round(check=True)
    fed = rec["fed_eval"]
    assert "fed_eval" in rec["stage_ms"]
    assert fed["n"] == 33 and fed["local"][1]["n"] == 0
    conf = [[sum(c["confusion"][t][p] for c in fed["local"]) for p in range(2)] for t in range(2)]
    assert fed["confusion"] == conf
    assert abs(fed["loss"] - fed["local"][0]["loss"]) <= 1e-5 * abs(fed["loss"])
    assert fed["auc"] == fed["local"][0]["auc"]

"""Federated evaluation on the CPU (DESIGN.md §13): the count layout and the metrics derived from it against
classification_metrics and an exact Mann–Whitney AUC, score_counts_torch against a loop, evaluate_federated of a cnn2
federation over loopback against plaintext sums and against evaluate on the union of the test sets, personal heads,
an empty client, the rejections, training left unchanged, and the --fed-test-dir command line."""
import json
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

from hefl_b200.config import FLConfig
from hefl_b200.fl import FederatedRunner
from hefl_b200.fl.data import SyntheticImageDataset
from hefl_b200.fl.fedeval import (binned_auc, check_fedeval_options, count_len, metrics_from_counts,
                                  score_counts_torch)
from hefl_b200.fl.runner import classification_metrics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPU = torch.device("cpu")
NB = 20                                   # cnn2 at n2048_l1 holds 6,144 values: 10 classes x 20 bins fit


def _cfg(**kw):
    base = dict(model="cnn2", image_size=28, in_channels=1, num_classes=10, batch_size=8, local_epochs=1,
                steps_per_epoch=2, val_steps=1, he_preset="n2048_l1", nn_backend="cudnn", dtype="fp32", device="cpu",
                transport="loopback", deterministic_crypto=True, key_holder=-1, fed_eval_bins=NB)
    base.update(kw)
    return FLConfig(**base)


def _counts_of(y, pred, C, nbins):
    v = torch.zeros(count_len(C, nbins), dtype=torch.float64)
    for t, p in zip(y.tolist(), pred.tolist()):
        v[t * C + p] += 1
    return v


@pytest.mark.parametrize("seed", range(6))
def test_metrics_from_counts_equal_classification_metrics(seed):
    g = torch.Generator().manual_seed(seed)
    C = 2 + seed
    n = int(torch.randint(1, 60, (1,), generator=g))
    y = torch.randint(0, C - 1, (n,), generator=g)          # class C-1 never occurs as a label
    pred = torch.randint(0, C, (n,), generator=g)
    pred[pred == 1] = 0                                      # class 1 is never predicted
    m = metrics_from_counts(_counts_of(y, pred, C, 4), C, 4)
    ref = classification_metrics(y, pred, C)
    for k in ("precision", "recall", "f1", "accuracy"):
        assert m[k] == ref[k], k
    assert m["n"] == n


def _mw_auc(pos_scores, neg_scores):
    num = sum(Fraction(1) if p > q else Fraction(1, 2) if p == q else Fraction(0)
              for p in pos_scores for q in neg_scores)
    return num / (len(pos_scores) * len(neg_scores))


@pytest.mark.parametrize("seed", range(4))
def test_binned_auc_is_the_exact_mann_whitney_auc_of_the_bins(seed):
    rng = np.random.default_rng(seed)
    nbins = int(rng.integers(2, 12))
    pos = rng.integers(0, nbins, int(rng.integers(1, 30))).tolist()
    neg = rng.integers(0, nbins, int(rng.integers(1, 30))).tolist()
    hp, hn = np.bincount(pos, minlength=nbins).tolist(), np.bincount(neg, minlength=nbins).tolist()
    assert binned_auc(hp, hn) == float(_mw_auc(pos, neg))
    assert binned_auc(hp, [0] * nbins) is None and binned_auc([0] * nbins, hn) is None


def test_score_counts_torch_matches_a_loop():
    g = torch.Generator().manual_seed(3)
    B, C, nbins = 41, 4, 9
    logits = torch.randn(B, C, generator=g) * 2
    logits[:5, 2] = logits[:5, 3]
    y = torch.randint(0, C, (B,), generator=g)
    v = score_counts_torch(logits, y, nbins)
    ref = torch.zeros(count_len(C, nbins), dtype=torch.float64)
    p = torch.softmax(logits, 1)
    loss = 0.0
    for i in range(B):
        row = logits[i].tolist()
        pred = row.index(max(row))
        ref[y[i] * C + pred] += 1
        for c in range(C):
            b = min(nbins - 1, int(np.floor(np.float32(p[i, c]) * np.float32(nbins))))
            ref[C * C + (int(y[i]) * C + c) * nbins + b] += 1
        loss += -float(torch.log_softmax(logits[i].double(), 0)[y[i]])
    assert torch.equal(v[:-1], ref[:-1])
    assert abs(float(v[-1]) - loss) <= 1e-9 * loss
    m = metrics_from_counts(v, C, nbins)
    assert m["n"] == B and abs(m["loss"] - loss / B) <= 1e-12


class _Union:
    def __init__(self, sets):
        self.images = torch.cat([s.images for s in sets])
        self.labels = torch.cat([s.labels for s in sets])
        self.classes = sets[0].classes

    def __len__(self):
        return len(self.labels)


def _tests(sizes, seed=50):
    return [SyntheticImageDataset(n, 28, 1, 10, seed=seed + n, pin=False) for n in sizes]


def test_loopback_federation_sums_exact_counts_and_matches_evaluate():
    """Three clients on one rank, one of them without scans: the decoded counts are the plaintext sum exactly, and the
    metrics are evaluate's on the union of the test sets."""
    tests = _tests((13, 0, 21))
    run = FederatedRunner(_cfg(clients_per_rank=3), device=CPU, test_dataset=tests)
    run.run_round()
    flat = run.pack.flat.clone()
    fed = run.evaluate_federated()
    assert torch.equal(run.pack.flat, flat)
    assert fed["n"] == 34 and fed["local"][1]["n"] == 0
    conf = [[sum(c["confusion"][t][p] for c in fed["local"]) for p in range(10)] for t in range(10)]
    assert fed["confusion"] == conf
    rows = torch.zeros(count_len(10, NB), dtype=torch.float64)
    for i, t in enumerate(tests):
        if len(t):
            from hefl_b200.fl.data import BatchFeeder

            run.trainer.score(BatchFeeder(t, range(len(t)), 8, CPU, shuffle=False), rows)
    assert fed["auc"] == metrics_from_counts(rows, 10, NB)["auc"]
    ref = run.evaluate(_Union([t for t in tests if len(t)]))
    for k in ("precision", "recall", "f1", "accuracy"):
        assert fed[k] == ref[k], k


def test_personal_heads_show_up_per_client_and_are_restored():
    """Sentinel heads: client k's Dense layer maps everything to class k, so every scan of client k lands in column k.
    The installed personal layers are the same afterwards."""
    tests = _tests((9, 11, 5), seed=70)
    run = FederatedRunner(_cfg(clients_per_rank=3, personal_layers=1, fed_eval_bins=10), device=CPU,
                          test_dataset=tests)
    for k in range(3):
        head = run._c_head[k]
        head.zero_()
        head[-10 + k] = 100.0                      # the bias of the last Dense layer
    installed = run.pack.flat.clone()
    fed = run.evaluate_federated()
    assert torch.equal(run.pack.flat, installed)
    cols = [sum(fed["confusion"][t][k] for t in range(10)) for k in range(10)]
    assert cols == [9, 11, 5] + [0] * 7


def test_rejections():
    with pytest.raises(ValueError, match="fed_eval_every"):
        FederatedRunner(_cfg(fed_eval_every=-1), device=CPU)
    for nb in (1, 1025):
        with pytest.raises(ValueError, match="fed_eval_bins"):
            FederatedRunner(_cfg(fed_eval_bins=nb), device=CPU)
    with pytest.raises(ValueError, match="does not fit"):
        FederatedRunner(_cfg(fed_eval_every=1, fed_eval_bins=100), device=CPU)
    with pytest.raises(ValueError, match="compat_sequential_clients"):
        FederatedRunner(_cfg(fed_eval_every=1, compat_sequential_clients=True), device=CPU)
    bad = _tests((6,))[0]
    bad.labels[2] = 10
    with pytest.raises(ValueError, match="labels"):
        FederatedRunner(_cfg(), device=CPU, test_dataset=[bad])
    run = FederatedRunner(_cfg(), device=CPU)
    with pytest.raises(ValueError, match="class names"):
        check_fedeval_options(run.cfg, 10, None, [type("D", (), {"labels": torch.zeros(1, dtype=torch.long),
                                                                 "class_indices": {"b": 0}, "__len__": lambda s: 1})()],
                              {"a": 0})


def test_fed_eval_every_round_leaves_the_global_models_unchanged():
    models = []
    for every in (1, 0):
        run = FederatedRunner(_cfg(clients_per_rank=2, fed_eval_every=every), device=CPU, test_dataset=_tests((7, 12)))
        got = []
        for _ in range(2):
            rec = run.run_round()
            assert ("fed_eval" in rec) == bool(every)
            got.append(run.pack.flat.clone())
        models.append(got)
    assert all(torch.equal(a, b) for a, b in zip(*models))


def _png_folder(root, n_per_class, seed):
    from PIL import Image

    rng = np.random.default_rng(seed)
    for c in ("benign", "malignant"):
        os.makedirs(os.path.join(root, c), exist_ok=True)
        for i in range(n_per_class):
            a = rng.integers(0, 255, (20, 20), dtype=np.uint8)
            Image.fromarray(a, "L").save(os.path.join(root, c, f"{i}.png"))


def test_cli_fed_test_dir(tmp_path):
    train, test = tmp_path / "train", tmp_path / "test"
    _png_folder(str(train), 24, 1)
    _png_folder(str(test), 9, 2)
    cmd = [sys.executable, "-m", "hefl_b200", "--device", "cpu", "--model", "cnn2", "--image-size", "28",
           "--in-channels", "1", "--he-preset", "n2048_l1", "--nn-backend", "cudnn", "--dtype", "fp32",
           "--transport", "loopback", "--rounds", "2", "--local-epochs", "1", "--batch-size", "8",
           "--deterministic-crypto", "1", "--data-dir", str(train), "--fed-test-dir", str(test),
           "--clients-per-rank", "2", "--personal-layers", "1", "--fed-eval-every", "1"]
    env = {**os.environ, "PYTHONPATH": ROOT}
    out = subprocess.run(cmd, capture_output=True, text=True, cwd=str(tmp_path), env=env, timeout=600)
    assert out.returncode == 0, out.stderr
    lines = [json.loads(l) for l in out.stdout.splitlines() if l.startswith("{")]
    fed = [l for l in lines if "fed_eval" in l]
    assert [l["round"] for l in fed] == [0, 1]
    for l in fed:
        assert l["fed_eval"]["n"] == 18 and "local" not in l["fed_eval"]
        assert sum(map(sum, l["fed_eval"]["confusion"])) == 18
    assert len([l for l in lines if "loss" in l and "fed_eval" not in l]) == 2


def test_two_gloo_ranks_of_two_clients_equal_one_rank_of_four(tmp_path):
    """A key holder, pairwise masks and the ciphertext sum over gloo give every rank the fed_eval of the same four
    clients in one process."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from mp_fedeval_worker import config as worker_config, test_sets

    out = str(tmp_path / "fedeval.pt")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29687", os.path.join(ROOT, "tests", "mp_fedeval_worker.py"),
           "--clients-per-rank", "2", "--out", out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT,
                       env=dict(os.environ, OMP_NUM_THREADS="2"))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    threads = torch.get_num_threads()
    torch.set_num_threads(2)                       # CPU convolutions reduce in a thread-count dependent order
    try:
        run = FederatedRunner(worker_config(4, "loopback", -1), device=CPU, test_dataset=test_sets(range(4)))
        ref = run.run_round(check=True)["fed_eval"]
    finally:
        torch.set_num_threads(threads)
    for rank in range(2):
        got = torch.load(f"{out}.rank{rank}")
        assert got["n"] == 34
        for k in ("n", "confusion", "auc", "macro_auc", "precision", "recall", "f1", "accuracy"):
            assert got[k] == ref[k], k
        assert abs(got["loss"] - ref["loss"]) <= 1e-5 * abs(ref["loss"])

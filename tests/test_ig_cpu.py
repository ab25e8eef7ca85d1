"""Integrated Gradients on the CPU (DESIGN.md §12): ``integrated_gradients_torch`` against the closed form of a
positively homogeneous network, the rejections, ``attribute`` on the PyTorch path (batching, the personal head of
another client) and the ``--ig-dir`` command line on a 28 x 28 image folder."""
import csv
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from hefl_b200.config import FLConfig
from hefl_b200.fl import FederatedRunner
from hefl_b200.fl.data import ImageFolderDataset, SyntheticImageDataset
from hefl_b200.fl.explain import integrated_gradients_torch
from hefl_b200.models import create_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPU = torch.device("cpu")


def _cfg(**kw):
    base = dict(model="cnn2", image_size=28, in_channels=1, num_classes=10, batch_size=8, local_epochs=1,
                steps_per_epoch=2, val_steps=1, he_preset="n2048_l1", nn_backend="cudnn", dtype="fp32", device="cpu",
                transport="loopback", deterministic_crypto=True, key_holder=-1)
    base.update(kw)
    return FLConfig(**base)


@pytest.mark.parametrize("target", [None, 4])
@pytest.mark.parametrize("steps", [1, 7])
def test_homogeneous_network_matches_the_closed_form(steps, target):
    """With every bias zero, cnn2 (conv, ReLU, max-pool, Dense) is positively homogeneous of degree 1: the gradient is
    the same at every point alpha x of the path, so for any number of steps attr = sum_c x * grad logit_t(x), and
    Euler's identity makes the attributions add up to logit_t(x) - logit_t(0) = logit_t(x) exactly."""
    torch.manual_seed(1)
    model = create_model("cnn2", 1, 10, 28).double()
    with torch.no_grad():
        for m in [*model.convs, *model.fcs]:
            m.bias.zero_()
    x = SyntheticImageDataset(5, 28, 1, 10, seed=2, pin=False).images
    probs, attr, gap = integrated_gradients_torch(model, x, steps, target)
    xh = (x.permute(0, 3, 1, 2).double() / 255.0).requires_grad_(True)
    logits = model(xh)
    t = logits.argmax(1) if target is None else torch.full((5,), target)
    grad, = torch.autograd.grad(logits.gather(1, t[:, None]).sum(), xh)
    ref = (xh * grad).sum(1).detach()
    assert attr.dtype == torch.float64 and attr.shape == (5, 28, 28)
    assert (attr - ref).abs().max() <= 1e-12
    assert gap.abs().max() <= 1e-12
    assert (probs - torch.softmax(logits.detach(), 1)).abs().max() <= 1e-12
    assert float(ref.abs().sum()) > 0, "the draw must give non-zero attributions"


@pytest.mark.parametrize("name", ["resnet18", "resnet50"])
def test_resnets_are_rejected(name):
    with pytest.raises(ValueError, match="ResNet"):
        integrated_gradients_torch(create_model(name, 3, 2, 32), torch.zeros(1, 32, 32, 3, dtype=torch.uint8), 4)


@pytest.mark.parametrize("steps", [0, 1025, -3, 2.0, True])
def test_steps_out_of_range_are_rejected(steps):
    with pytest.raises(ValueError, match="steps"):
        integrated_gradients_torch(create_model("cnn2", 1, 10, 28), torch.zeros(1, 28, 28, 1, dtype=torch.uint8),
                                   steps)


@pytest.mark.parametrize("target", [10, torch.tensor([0, 12]), -2, torch.tensor([1, 2, 3])])
def test_target_out_of_range_is_rejected(target):
    with pytest.raises(ValueError, match="target"):
        integrated_gradients_torch(create_model("cnn2", 1, 10, 28), torch.zeros(2, 28, 28, 1, dtype=torch.uint8), 2,
                                   target)


def test_attribute_rejects_bad_images():
    run = FederatedRunner(_cfg(), device=CPU)
    with pytest.raises(ValueError, match="uint8"):
        run.attribute(torch.zeros(2, 27, 27, 1, dtype=torch.uint8), 2)
    with pytest.raises(ValueError, match="steps"):
        run.attribute(torch.zeros(2, 28, 28, 1, dtype=torch.uint8), 0)


def test_attribute_batches_equal_scan_by_scan():
    """11 scans in batches of 8 (the last one short) give each scan's own result."""
    run = FederatedRunner(_cfg(), device=CPU)
    x = SyntheticImageDataset(11, 28, 1, 10, seed=5, pin=False).images
    tgt = torch.tensor([-1, 2, 5, -1, 0, 9, -1, 1, 3, -1, 7])
    probs, attr, gap = run.attribute(x, steps=4, target=tgt, batch_size=8)
    assert probs.dtype == attr.dtype == gap.dtype == torch.float32
    assert probs.shape == (11, 10) and attr.shape == (11, 28, 28) and gap.shape == (11,)
    for i in range(11):
        p, a, g = run.attribute(x[i:i + 1], steps=4, target=tgt[i:i + 1])
        assert torch.allclose(p[0], probs[i], rtol=0, atol=1e-6)
        assert torch.allclose(a[0], attr[i], rtol=0, atol=1e-6 * float(attr[i].abs().max()) + 1e-9)
        assert abs(float(g[0]) - float(gap[i])) <= 1e-5 * float(attr[i].abs().sum()) + 1e-6
    p_pred = run.attribute(x, steps=2, batch_size=8)
    p_m1 = run.attribute(x, steps=2, target=-1, batch_size=8)
    assert all(torch.equal(a, b) for a, b in zip(p_pred, p_m1))


def test_attribute_installs_another_clients_head_and_restores_the_installed_one():
    run = FederatedRunner(_cfg(personal_layers=1, clients_per_rank=2), device=CPU)
    g = torch.Generator().manual_seed(11)
    run._c_head[1].add_(torch.randn(run._c_head[1].shape, generator=g) * 0.5)
    installed = run.pack.flat[run.n_shared:].clone()
    x = SyntheticImageDataset(5, 28, 1, 10, seed=7, pin=False).images
    r1 = run.attribute(x, steps=3, client=1)
    assert torch.equal(run.pack.flat[run.n_shared:], installed)
    run.pack.flat[run.n_shared:].copy_(run._c_head[1])
    r_ref = run.attribute(x, steps=3)
    run.pack.flat[run.n_shared:].copy_(installed)
    assert all(torch.equal(a, b) for a, b in zip(r1, r_ref))
    r0 = run.attribute(x, steps=3, client=0)
    assert not torch.equal(r0[0], r1[0]), "the two clients' heads gave the same probabilities"
    with pytest.raises(ValueError, match="client slot"):
        run.attribute(x, steps=3, client=2)


def test_cli_rejects_ig_dir_without_test_dir(tmp_path):
    r = subprocess.run([sys.executable, "-m", "hefl_b200", "--device", "cpu", "--model", "cnn2", "--ig-dir",
                        str(tmp_path / "ig")], capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode != 0 and "--test-dir" in r.stderr
    assert not (tmp_path / "ig").exists()


def _image_folder(root, per_class=3, classes=2):
    from PIL import Image

    rng = np.random.default_rng(0)
    for c in range(classes):
        os.makedirs(os.path.join(root, f"class{c}"))
        for k in range(per_class):
            Image.fromarray(rng.integers(0, 256, (28, 28), dtype=np.uint8), mode="L").save(
                os.path.join(root, f"class{c}", f"scan{k}.png"))
    return per_class * classes


def _cli(tmp_path, name, extra):
    args = [sys.executable, "-m", "hefl_b200", "--device", "cpu", "--model", "cnn2", "--image-size", "28",
            "--in-channels", "1", "--num-classes", "10", "--he-preset", "n2048_l1", "--nn-backend", "cudnn", "--dtype",
            "fp32", "--rounds", "1", "--local-epochs", "1", "--steps-per-epoch", "2", "--val-steps", "1",
            "--batch-size", "8", "--deterministic-crypto", "1", "--checkpoint", str(tmp_path / f"{name}.pt"), *extra]
    r = subprocess.run(args, capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout.splitlines()


def test_cli_writes_attributions_and_heatmaps(tmp_path):
    test_dir, out = str(tmp_path / "test"), str(tmp_path / "ig")
    n = _image_folder(test_dir)
    with_ig = _cli(tmp_path, "a", ["--test-dir", test_dir, "--ig-dir", out, "--ig-steps", "5", "--ig-class", "3"])
    plain = _cli(tmp_path, "b", ["--test-dir", test_dir])
    metrics = [l for l in plain if '"test_images"' in l]
    assert len(metrics) == 1 and metrics[0] in with_ig
    assert json.loads(with_ig[-1]) == {"ig_dir": out, "images": n, "steps": 5}
    with open(os.path.join(out, "attributions.csv")) as fh:
        rows = list(csv.reader(fh))
    assert rows[0] == ["file", "label", "target", "p_target", "score", "baseline_score", "attribution_sum", "gap"]
    assert len(rows) == n + 1
    from PIL import Image

    pngs = sorted(f for f in os.listdir(out) if f.endswith(".png"))
    assert len(pngs) == n
    for f in pngs:
        assert Image.open(os.path.join(out, f)).size == (28, 28)
    # the rows are attribute's on the trained model (the checkpoint of the run)
    run = FederatedRunner(_cfg(), device=CPU)
    run.load_checkpoint(str(tmp_path / "a.pt"))
    ds = ImageFolderDataset(test_dir, 28, 1, shuffle_seed=None, pin=False)
    probs, attr, gap = run.attribute(ds.images, steps=5, target=3)
    assert [r[0] for r in rows[1:]] == [os.path.relpath(f, test_dir) for f in ds.filenames]
    assert [int(r[1]) for r in rows[1:]] == ds.labels.tolist()
    assert all(int(r[2]) == 3 for r in rows[1:])
    vals = torch.tensor([[float(v) for v in r[3:]] for r in rows[1:]], dtype=torch.float64)
    assert torch.allclose(vals[:, 0], probs[:, 3].double(), rtol=0, atol=1e-6)
    assert torch.allclose(vals[:, 3], attr.double().sum((1, 2)), rtol=1e-5, atol=1e-6)
    assert torch.allclose(vals[:, 4], gap.double(), rtol=1e-5, atol=1e-6)
    # gap = attribution_sum - (score - baseline_score)
    assert torch.allclose(vals[:, 4], vals[:, 3] - (vals[:, 1] - vals[:, 2]), rtol=0, atol=1e-5)

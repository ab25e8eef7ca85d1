"""Grad-CAM on the CPU (DESIGN.md §11): ``gradcam_torch`` against a numpy closed form, the rejections, ``explain`` on
the PyTorch path (batching, the personal head of another client) and the ``--gradcam-dir`` command line on a 28 x 28
image folder."""
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
from hefl_b200.fl.explain import gradcam_torch
from hefl_b200.models import create_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPU = torch.device("cpu")


def _cfg(**kw):
    base = dict(model="cnn2", image_size=28, in_channels=1, num_classes=10, batch_size=8, local_epochs=1,
                steps_per_epoch=2, val_steps=1, he_preset="n2048_l1", nn_backend="cudnn", dtype="fp32", device="cpu",
                transport="loopback", deterministic_crypto=True, key_holder=-1)
    base.update(kw)
    return FLConfig(**base)


def _bilinear(cam, S):
    """F.interpolate(bilinear, align_corners=False) of [N, Hp, Hp] to S x S, written out in numpy."""
    Hp = cam.shape[-1]
    src = np.maximum((np.arange(S) + 0.5) * (Hp / S) - 0.5, 0.0)
    i0 = np.minimum(np.floor(src).astype(np.int64), Hp - 1)
    i1 = np.minimum(i0 + 1, Hp - 1)
    l1 = src - i0
    l0 = 1.0 - l1
    rows = cam[:, i0, :] * l0[None, :, None] + cam[:, i1, :] * l1[None, :, None]
    return rows[:, :, i0] * l0[None, None, :] + rows[:, :, i1] * l1[None, None, :]


@pytest.mark.parametrize("target", [3, None])
def test_cnn2_last_stage_matches_the_closed_form(target):
    """cnn2's head is one Dense layer, so at its last stage G[b, h, w, c] = W[t_b, (h Hp + w) C + c] for every scan."""
    torch.manual_seed(0)
    model = create_model("cnn2", 1, 10, 28).double()
    x = SyntheticImageDataset(6, 28, 1, 10, seed=3, pin=False).images
    probs, cams = gradcam_torch(model, x, stage=2, target=target)
    with torch.no_grad():
        A = model.features(x.permute(0, 3, 1, 2).double() / 255.0).permute(0, 2, 3, 1).numpy()    # [N, Hp, Hp, C]
    N, Hp, _, C = A.shape
    W, b = model.fcs[0].weight.detach().numpy(), model.fcs[0].bias.detach().numpy()
    logits = A.reshape(N, -1) @ W.T + b
    t = logits.argmax(1) if target is None else np.full(N, target)
    G = W[t].reshape(N, Hp, Hp, C)
    alpha = G.mean(axis=(1, 2))
    cam = np.maximum((A * alpha[:, None, None, :]).sum(-1), 0.0)
    mx = cam.max(axis=(1, 2))
    assert (mx > 0).all(), "the draw must give non-empty maps"
    ref = _bilinear(cam, 28) / mx[:, None, None]
    p = np.exp(logits - logits.max(1, keepdims=True))
    p /= p.sum(1, keepdims=True)
    assert cams.dtype == torch.float64 and cams.shape == (N, 28, 28)
    assert np.abs(cams.numpy() - ref).max() <= 1e-12
    assert np.abs(probs.numpy() - p).max() <= 1e-12
    assert float(cams.min()) >= 0.0 and float(cams.max()) <= 1.0 + 1e-12


def test_a_map_without_positive_evidence_is_all_zero():
    model = create_model("cnn2", 1, 10, 28).double()
    with torch.no_grad():
        model.fcs[0].weight.fill_(-1.0)              # G < 0 everywhere and X[s] >= 0: relu leaves nothing
    _, cams = gradcam_torch(model, SyntheticImageDataset(2, 28, 1, 10, seed=1, pin=False).images, 2, 0)
    assert torch.equal(cams, torch.zeros_like(cams))


@pytest.mark.parametrize("name", ["resnet18", "resnet50"])
def test_resnets_are_rejected(name):
    model = create_model(name, 3, 2, 32)
    with pytest.raises(ValueError, match="ResNet"):
        gradcam_torch(model, torch.zeros(1, 32, 32, 3, dtype=torch.uint8), 1)


@pytest.mark.parametrize("stage", [0, 3, -1])
def test_stage_out_of_range_is_rejected(stage):
    with pytest.raises(ValueError, match="stage"):
        gradcam_torch(create_model("cnn2", 1, 10, 28), torch.zeros(1, 28, 28, 1, dtype=torch.uint8), stage)


@pytest.mark.parametrize("target", [10, torch.tensor([0, 12]), -2])
def test_target_out_of_range_is_rejected(target):
    with pytest.raises(ValueError, match="target"):
        gradcam_torch(create_model("cnn2", 1, 10, 28), torch.zeros(2, 28, 28, 1, dtype=torch.uint8), 2, target)


def test_cli_rejects_gradcam_dir_without_test_dir(tmp_path):
    r = subprocess.run([sys.executable, "-m", "hefl_b200", "--device", "cpu", "--model", "cnn2", "--gradcam-dir",
                        str(tmp_path / "cams")], capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode != 0 and "--test-dir" in r.stderr
    assert not (tmp_path / "cams").exists()


def test_explain_batches_equal_scan_by_scan():
    run = FederatedRunner(_cfg(), device=CPU)
    x = SyntheticImageDataset(11, 28, 1, 10, seed=5, pin=False).images
    tgt = torch.tensor([-1, 2, 5, -1, 0, 9, -1, 1, 3, -1, 7])
    probs, cams = run.explain(x, stage=2, target=tgt, batch_size=8)
    assert probs.dtype == cams.dtype == torch.float32 and probs.shape == (11, 10) and cams.shape == (11, 28, 28)
    for i in range(11):
        p, c = run.explain(x[i:i + 1], stage=2, target=tgt[i:i + 1])
        assert torch.allclose(p[0], probs[i], rtol=0, atol=1e-6) and torch.allclose(c[0], cams[i], rtol=0, atol=1e-5)
    p_pred, _ = run.explain(x, stage=1, batch_size=8)
    assert torch.equal(p_pred, run.explain(x, stage=1, target=-1, batch_size=8)[0])
    assert 0.0 <= float(cams.min()) and float(cams.max()) <= 1.0


def test_explain_installs_another_clients_head_and_restores_the_installed_one():
    run = FederatedRunner(_cfg(personal_layers=1, clients_per_rank=2), device=CPU)
    g = torch.Generator().manual_seed(11)
    run._c_head[1].add_(torch.randn(run._c_head[1].shape, generator=g) * 0.5)
    installed = run.pack.flat[run.n_shared:].clone()
    x = SyntheticImageDataset(5, 28, 1, 10, seed=7, pin=False).images
    p1, c1 = run.explain(x, stage=2, client=1)
    assert torch.equal(run.pack.flat[run.n_shared:], installed)
    run.pack.flat[run.n_shared:].copy_(run._c_head[1])
    p_ref, c_ref = run.explain(x, stage=2)
    run.pack.flat[run.n_shared:].copy_(installed)
    assert torch.equal(p1, p_ref) and torch.equal(c1, c_ref)
    p0, _ = run.explain(x, stage=2, client=0)
    assert not torch.equal(p0, p1), "the two clients' heads gave the same probabilities"
    with pytest.raises(ValueError, match="client slot"):
        run.explain(x, stage=2, client=2)


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


def test_cli_writes_predictions_and_heatmaps(tmp_path):
    test_dir, out = str(tmp_path / "test"), str(tmp_path / "cams")
    n = _image_folder(test_dir)
    with_cam = _cli(tmp_path, "a", ["--test-dir", test_dir, "--gradcam-dir", out, "--gradcam-stage", "2"])
    plain = _cli(tmp_path, "b", ["--test-dir", test_dir])
    metrics = [l for l in plain if '"test_images"' in l]
    assert len(metrics) == 1 and metrics[0] in with_cam
    summary = json.loads(with_cam[-1])
    assert summary == {"gradcam_dir": out, "images": n, "stage": 2}
    with open(os.path.join(out, "predictions.csv")) as fh:
        rows = list(csv.reader(fh))
    assert rows[0] == ["file", "label", "predicted", *[f"p_{c}" for c in range(10)]]
    assert len(rows) == n + 1
    from PIL import Image

    pngs = sorted(f for f in os.listdir(out) if f.endswith(".png"))
    assert len(pngs) == n
    for f in pngs:
        assert Image.open(os.path.join(out, f)).size == (28, 28)
    # the probabilities are explain's on the trained model (the checkpoint of the run)
    cfg = _cfg(deterministic_crypto=True)
    run = FederatedRunner(cfg, device=CPU)
    run.load_checkpoint(str(tmp_path / "a.pt"))
    ds = ImageFolderDataset(test_dir, 28, 1, shuffle_seed=None, pin=False)
    probs, _ = run.explain(ds.images, stage=2)
    csv_p = torch.tensor([[float(v) for v in r[3:]] for r in rows[1:]], dtype=torch.float32)
    assert torch.allclose(csv_p, probs, rtol=0, atol=1e-6)
    assert [int(r[2]) for r in rows[1:]] == probs.argmax(1).tolist()
    assert [int(r[1]) for r in rows[1:]] == ds.labels.tolist()
    assert [r[0] for r in rows[1:]] == [os.path.relpath(f, test_dir) for f in ds.filenames]

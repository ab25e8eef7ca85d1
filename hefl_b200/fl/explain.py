"""Grad-CAM (Selvaraju et al. 2017) for the sequential CNNs: class probabilities and a heatmap of where the model
looked, per scan (DESIGN.md §11); and pixel-level Integrated Gradients (Sundararajan et al. 2017, DESIGN.md §12).

For stage s (the output X[s] of the s-th [Conv 3x3 + ReLU -> MaxPool 2x2] block, [N, C, Hp, Hp]) and a target class
t_b per scan (-1: the predicted class, the arg-max of the logits with the lowest index on ties):

    G        = d logits[b, t_b] / d X[s]                 (the class score, not the loss)
    alpha    = mean over (h, w) of G                      [N, C]
    cam      = relu(sum_c alpha[:, c] X[s][:, c])         [N, Hp, Hp]
    out      = F.interpolate(cam, (S, S), bilinear, align_corners=False) / max_hw cam   (0 where that max is 0)

``gradcam_torch`` is that definition with autograd, in the dtype of the model: in float64 it is the tests' reference,
and it is the path of the CPU, of the cuDNN backend and of ``cnn2``. The hand-written engine computes the same in
``MedCNNEngine.gradcam_staged``. Nothing computed here ever enters a ciphertext.
"""
from __future__ import annotations

from typing import Optional, Tuple, Union

import torch
import torch.nn.functional as F

from ..models.cnn import _SeqCNN

Target = Optional[Union[int, torch.Tensor]]
MAX_IG_STEPS = 1024


def _check_model(model, what: str) -> None:
    if not isinstance(model, _SeqCNN):
        raise ValueError(f"{what} supports the sequential CNNs (medcnn, cnn2), not {type(model).__name__}: the "
                         "ResNets (resnet18, resnet50) would need a BatchNorm backward without statistics updates")


def check_target(model, target: Target, n: int) -> torch.Tensor:
    """The explained class of each of ``n`` scans as int64 [n] (-1 = the predicted class); rejects classes >= C."""
    C = model.num_classes
    if target is None:
        t = torch.full((n,), -1, dtype=torch.int64)
    elif isinstance(target, torch.Tensor):
        t = target.detach().to("cpu", torch.int64).reshape(-1)
        if t.numel() != n:
            raise ValueError(f"target has {t.numel()} entries for {n} scans")
    else:
        t = torch.full((n,), int(target), dtype=torch.int64)
    if t.numel() and (int(t.max()) >= C or int(t.min()) < -1):
        raise ValueError(f"target classes must be in 0..{C - 1} (or -1 for the predicted class), got "
                         f"{int(t.min())}..{int(t.max())}")
    return t


def check_gradcam(model, stage: int, target: Target, n: int) -> torch.Tensor:
    """Reject what Grad-CAM cannot explain and return the targets of ``n`` scans as int64 [n] (-1 = predicted class)."""
    _check_model(model, "Grad-CAM")
    stages = len(model.convs)
    if isinstance(stage, bool) or not isinstance(stage, int) or not 1 <= stage <= stages:
        raise ValueError(f"stage must be an integer in 1..{stages} for this model, got {stage!r}")
    return check_target(model, target, n)


def gradcam_torch(model, x_u8: torch.Tensor, stage: int = 4, target: Target = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """(probs [N, C], cams [N, S, S]) of the uint8 NHWC scans ``x_u8`` at ``stage``, in the dtype of the model and on
    its device. ``target``: None (each scan's predicted class), an int, or N ints (-1 = predicted)."""
    N = x_u8.shape[0]
    t = check_gradcam(model, stage, target, N)
    p = next(model.parameters())
    dtype, dev = p.dtype, p.device
    x = x_u8.to(dev).permute(0, 3, 1, 2).to(dtype) * (1.0 / 255.0)
    S = x.shape[-1]
    with torch.enable_grad():
        for i, conv in enumerate(model.convs):
            x = F.max_pool2d(F.relu(conv(x)), 2)
            if i + 1 == stage:
                x = x.detach().requires_grad_(True)    # the stage output: the leaf the score is differentiated by
                A = x
        h = x.permute(0, 2, 3, 1).flatten(1)           # Keras Flatten: H, W, C order
        for fc in model.fcs[:-1]:
            h = F.relu(fc(h))
        logits = model.fcs[-1](h)
        t = t.to(dev)
        t = torch.where(t < 0, logits.argmax(1), t)
        G, = torch.autograd.grad(logits.gather(1, t[:, None]).sum(), A)
    A = A.detach()
    alpha = G.mean(dim=(2, 3))                                          # [N, C]
    cam = torch.relu((alpha[:, :, None, None] * A).sum(1))              # [N, Hp, Hp]
    up = F.interpolate(cam[:, None], (S, S), mode="bilinear", align_corners=False)[:, 0]
    mx = cam.amax(dim=(1, 2))
    cams = torch.where(mx[:, None, None] > 0, up / torch.where(mx > 0, mx, 1)[:, None, None], torch.zeros_like(up))
    return torch.softmax(logits.detach(), dim=1), cams


def check_ig(model, steps: int, target: Target, n: int) -> torch.Tensor:
    """Reject what Integrated Gradients cannot explain and return the targets of ``n`` scans as int64 [n]."""
    _check_model(model, "Integrated Gradients")
    if isinstance(steps, bool) or not isinstance(steps, int) or not 1 <= steps <= MAX_IG_STEPS:
        raise ValueError(f"steps must be an integer in 1..{MAX_IG_STEPS}, got {steps!r}")
    return check_target(model, target, n)


def _ig_torch(model, x_u8: torch.Tensor, steps: int, t: torch.Tensor):
    """(probs, attr, score, baseline score, resolved targets) of the definition in ``integrated_gradients_torch``."""
    p = next(model.parameters())
    dtype, dev = p.dtype, p.device
    xh = x_u8.to(dev).permute(0, 3, 1, 2).to(dtype) * (1.0 / 255.0)
    with torch.no_grad():
        logits = model(xh)
        base = model(torch.zeros_like(xh))
    t = t.to(dev)
    t = torch.where(t < 0, logits.argmax(1), t)
    total = torch.zeros_like(xh)
    with torch.enable_grad():
        for k in range(1, steps + 1):
            xk = (xh * ((k - 0.5) / steps)).requires_grad_(True)
            gk, = torch.autograd.grad(model(xk).gather(1, t[:, None]).sum(), xk)
            total += gk
    attr = (xh * total).sum(1) / steps
    return (torch.softmax(logits, dim=1), attr, logits.gather(1, t[:, None])[:, 0],
            base.gather(1, t[:, None])[:, 0], t)


def integrated_gradients_torch(model, x_u8: torch.Tensor, steps: int = 32,
                               target: Target = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(probs [N, C], attr [N, S, S], gap [N]) of the uint8 NHWC scans ``x_u8``, in the dtype of the model and on its
    device: Integrated Gradients against the black image with ``steps`` midpoint-rule path points. ``target``: None
    (each scan's predicted class), an int, or N ints (-1 = predicted)."""
    t = check_ig(model, steps, target, x_u8.shape[0])
    probs, attr, score, base, _ = _ig_torch(model, x_u8, steps, t)
    return probs, attr, attr.sum((1, 2)) - (score - base)


def heat_overlay(img_u8, cam, weight: float = 0.5):
    """uint8 [S, S, 3]: the scan (grey or RGB, uint8 [S, S, C]) blended with a blue-green-red ramp of ``cam`` [S, S]
    in [0, 1]."""
    import numpy as np

    v = np.clip(np.asarray(cam, dtype=np.float32), 0.0, 1.0)[..., None]
    heat = np.clip(1.5 - np.abs(4.0 * v - np.array([3.0, 2.0, 1.0], dtype=np.float32)), 0.0, 1.0) * 255.0
    img = np.asarray(img_u8, dtype=np.float32)
    if img.shape[-1] == 1:
        img = np.repeat(img, 3, axis=-1)
    return np.clip((1.0 - weight) * img + weight * heat, 0, 255).round().astype(np.uint8)


def write_explanations(run, test_dir: str, out_dir: str, stage: int, target: Optional[int] = None,
                       client: Optional[int] = None, chunk: int = 256) -> dict:
    """``out_dir/predictions.csv`` (file, label, predicted, p_0 .. p_{C-1}) and one PNG per scan of the image folder
    ``test_dir`` (``<label>/<file>``): the scan blended with a heat ramp of its Grad-CAM map at ``stage``. The folder is
    decoded ``chunk`` scans at a time, so memory does not grow with its size. Returns the JSON summary."""
    import csv
    import os

    from PIL import Image

    from .data import ImageFolderDataset

    cfg = run.cfg
    ds = ImageFolderDataset(test_dir, cfg.image_size, cfg.in_channels, shuffle_seed=None, pin=False, stream=True)
    os.makedirs(out_dir, exist_ok=True)
    C = run.model.num_classes
    root = os.path.abspath(test_dir)
    buf = torch.empty(min(chunk, len(ds)), cfg.image_size, cfg.image_size, cfg.in_channels, dtype=torch.uint8)
    with open(os.path.join(out_dir, "predictions.csv"), "w", newline="") as fh:
        w = csv.writer(fh)
        w.writerow(["file", "label", "predicted", *[f"p_{c}" for c in range(C)]])
        for i in range(0, len(ds), chunk):
            n = min(chunk, len(ds) - i)
            x = buf[:n]
            ds.load_batch(torch.arange(i, i + n), x)
            probs, cams = run.explain(x, stage, target, client=client)
            pred = probs.argmax(1)
            for k in range(n):
                name = os.path.relpath(ds.filenames[i + k], root)
                w.writerow([name, int(ds.labels[i + k]), int(pred[k]), *[repr(float(p)) for p in probs[k]]])
                png = f"{i + k:06d}_{os.path.splitext(os.path.basename(name))[0]}.png"
                Image.fromarray(heat_overlay(x[k].numpy(), cams[k].numpy())).save(os.path.join(out_dir, png))
    return {"gradcam_dir": out_dir, "images": len(ds), "stage": stage}


def write_attributions(run, test_dir: str, out_dir: str, steps: int, target: Optional[int] = None,
                       client: Optional[int] = None, chunk: int = 256) -> dict:
    """``out_dir/attributions.csv`` (file, label, target, p_target, score, baseline_score, attribution_sum, gap) and
    one PNG per scan of the image folder ``test_dir`` (``<label>/<file>``): the scan blended with a heat ramp of its
    positive Integrated Gradients attributions over their 99th percentile, clipped to [0, 1] (0 for a scan with no
    positive attribution). The folder is decoded ``chunk`` scans at a time. Returns the JSON summary."""
    import csv
    import os

    from PIL import Image

    from .data import ImageFolderDataset

    cfg = run.cfg
    ds = ImageFolderDataset(test_dir, cfg.image_size, cfg.in_channels, shuffle_seed=None, pin=False, stream=True)
    os.makedirs(out_dir, exist_ok=True)
    root = os.path.abspath(test_dir)
    buf = torch.empty(min(chunk, len(ds)), cfg.image_size, cfg.image_size, cfg.in_channels, dtype=torch.uint8)
    with open(os.path.join(out_dir, "attributions.csv"), "w", newline="") as fh:
        w = csv.writer(fh)
        w.writerow(["file", "label", "target", "p_target", "score", "baseline_score", "attribution_sum", "gap"])
        for i in range(0, len(ds), chunk):
            n = min(chunk, len(ds) - i)
            x = buf[:n]
            ds.load_batch(torch.arange(i, i + n), x)
            probs, attr, gap, t, score, base = run._attribute(x, steps, target, client)
            for k in range(n):
                name = os.path.relpath(ds.filenames[i + k], root)
                tk = int(t[k])
                w.writerow([name, int(ds.labels[i + k]), tk, repr(float(probs[k, tk])), repr(float(score[k])),
                            repr(float(base[k])), repr(float(attr[k].double().sum())), repr(float(gap[k]))])
                pos = attr[k].clamp_min(0)
                q = float(torch.quantile(pos[pos > 0], 0.99)) if bool((pos > 0).any()) else 0.0
                heat = (pos / q).clamp(0, 1) if q > 0 else torch.zeros_like(pos)
                png = f"{i + k:06d}_{os.path.splitext(os.path.basename(name))[0]}.png"
                Image.fromarray(heat_overlay(x[k].numpy(), heat.numpy())).save(os.path.join(out_dir, png))
    return {"ig_dir": out_dir, "images": len(ds), "steps": steps}

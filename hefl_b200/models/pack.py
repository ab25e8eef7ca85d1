"""Flat parameter packing.

All federated state of a model (trainable weights in Keras ``get_weights`` order, then
BatchNorm running statistics) lives in ONE contiguous fp32 buffer; the module's parameters
are views into it. The buffer is what gets CKKS-encoded (no gather), what the fused Adam
kernel updates, and what the decrypted average is copied back into — each one launch.

``to_keras_dict`` / ``from_keras_dict`` convert to the reference's ``c_{layer}_{tensor}``
dictionary with Keras layouts (FLPyfhelin.py:205-221, :271-278; SURVEY.md Appendix B).
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np
import torch
import torch.nn as nn


class ParamPack:
    def __init__(self, model: nn.Module):
        self.model = model
        self.entries: List[Tuple[str, torch.Size, int, int]] = []  # key, shape, offset, numel
        tensors: List[Tuple[str, torch.Tensor, bool]] = []
        for li, (kind, mod) in enumerate(model.keras_layers()):
            if mod is None:
                continue
            if kind in ("conv", "dense"):
                tensors.append((f"c_{li}_0", mod.weight, True))
                if mod.bias is not None:
                    tensors.append((f"c_{li}_1", mod.bias, True))
            elif kind == "bn":
                tensors.append((f"c_{li}_0", mod.weight, True))
                tensors.append((f"c_{li}_1", mod.bias, True))
                tensors.append((f"c_{li}_2", mod.running_mean, False))
                tensors.append((f"c_{li}_3", mod.running_var, False))
        self._kinds = {f"c_{li}": kind for li, (kind, mod) in enumerate(model.keras_layers()) if mod is not None}
        # trainable first so the optimiser touches one contiguous prefix
        ordered = [t for t in tensors if t[2]] + [t for t in tensors if not t[2]]
        total = sum(t[1].numel() for t in ordered)
        self.n_trainable = sum(t[1].numel() for t in ordered if t[2])
        dev = next(model.parameters()).device
        self.flat = torch.zeros(total, dtype=torch.float32, device=dev)
        self.grad = torch.zeros(self.n_trainable, dtype=torch.float32, device=dev)
        off = 0
        self._tensors: Dict[str, torch.Tensor] = {}
        for key, t, trainable in ordered:
            n = t.numel()
            view = self.flat[off:off + n].view(t.shape)
            view.copy_(t.detach().float())
            t.data = view
            if trainable:
                t.grad = self.grad[off:off + n].view(t.shape)
            self.entries.append((key, t.shape, off, n))
            self._tensors[key] = t
            off += n
        self.numel = total

    # ------------------------------------------------------------------ flat access
    def trainable(self) -> torch.Tensor:
        return self.flat[: self.n_trainable]

    def dense_tail_start(self, layers: int) -> int:
        """Offset of the last ``layers`` Dense layers, which must be the tail of the trainable prefix (the sequential
        CNNs): [0, offset) is everything before them. ``layers = 0`` gives ``n_trainable``."""
        dense = sorted({int(k.split("_")[1]) for k, *_ in self.entries if self._kind(k) == "dense"})
        if not 0 <= layers <= len(dense):
            raise ValueError(f"the model has {len(dense)} Dense layers, cannot keep the last {layers}")
        if layers == 0:
            return self.n_trainable
        tail = {f"c_{li}" for li in dense[-layers:]}
        lo = min(off for k, _, off, _ in self.entries if k.rsplit("_", 1)[0] in tail)
        if any((k.rsplit("_", 1)[0] in tail) != (off >= lo) for k, _, off, _ in self.entries) or self.numel != self.n_trainable:
            raise ValueError("the last Dense layers are not the tail of the parameter vector")
        return lo

    def load_flat(self, vec: torch.Tensor) -> None:
        self.flat.copy_(vec.to(self.flat.device, torch.float32).reshape(-1)[: self.numel])

    def rebind_grads(self) -> None:
        """Re-point ``.grad`` at the flat gradient buffer (after ``zero_grad(set_to_none)``)."""
        for key, shape, off, n in self.entries:
            t = self._tensors[key]
            if isinstance(t, nn.Parameter) and off < self.n_trainable:
                t.grad = self.grad[off:off + n].view(shape)

    # ------------------------------------------------------------------ Keras dictionary
    def to_keras_dict(self) -> Dict[str, np.ndarray]:
        out: Dict[str, np.ndarray] = {}
        for key, shape, off, n in self.entries:
            t = self.flat[off:off + n].view(shape).detach().cpu()
            out[key] = self._to_keras_layout(key, t).numpy().copy()
        return self._sorted(out)

    def from_keras_dict(self, d: Dict[str, np.ndarray]) -> None:
        for key, shape, off, n in self.entries:
            arr = torch.as_tensor(np.asarray(d[key], dtype=np.float32))
            t = self._from_keras_layout(key, arr, shape)
            self.flat[off:off + n].copy_(t.reshape(-1))

    def keras_order_keys(self) -> List[str]:
        return list(self._sorted({k: None for k, *_ in self.entries}).keys())

    def _kind(self, key: str) -> str:
        return self._kinds[key.rsplit("_", 1)[0]]

    def _to_keras_layout(self, key: str, t: torch.Tensor) -> torch.Tensor:
        kind = self._kind(key)
        if key.endswith("_0") and kind == "conv":
            return t.permute(2, 3, 1, 0).contiguous()      # OIHW -> HWIO
        if key.endswith("_0") and kind == "dense":
            return t.t().contiguous()                       # [out,in] -> [in,out]
        return t.contiguous()

    def _from_keras_layout(self, key: str, a: torch.Tensor, shape: torch.Size) -> torch.Tensor:
        kind = self._kind(key)
        if key.endswith("_0") and kind == "conv":
            return a.permute(3, 2, 0, 1).contiguous()
        if key.endswith("_0") and kind == "dense":
            return a.t().contiguous()
        return a.reshape(shape)

    @staticmethod
    def _sorted(d):
        def k(key):
            _, li, ti = key.split("_")
            return (int(li), int(ti))

        return {key: d[key] for key in sorted(d, key=k)}

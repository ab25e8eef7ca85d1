"""Server optimizers of encrypted FedAvg (DESIGN.md §8): FedAvgM (Hsu et al. 2019) and FedAdagrad, FedYogi,
FedAdam (Reddi et al. 2021, Algorithm 2, no bias correction).

The decrypted average ``a`` of a round and the round's starting global model ``x`` give the pseudo-gradient
``d = a - x``; the key holder keeps the fp32 moments ``m`` and ``v`` and broadcasts ``x'`` instead of ``a``. The
step is fused into the CKKS decode (``torch.ops.hefl.ckks_decode_server_step_``), so the average never goes to
memory. Only the first ``n_trainable`` values are stepped; the flat tail (BatchNorm running statistics,
``models/pack.py``) takes the average as plain FedAvg does.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

# name -> opt code of the fused decode (csrc/he/server_step.h)
SERVER_OPTS = {"fedavg": 0, "fedavgm": 1, "fedadagrad": 2, "fedyogi": 3, "fedadam": 4}


def check_server_options(cfg) -> None:
    """Reject unknown or out-of-range server-optimizer settings (they arrive from flags and environment
    variables)."""
    if cfg.server_opt not in SERVER_OPTS:
        raise ValueError(f"server_opt must be one of {tuple(SERVER_OPTS)}, got {cfg.server_opt!r}")
    if not cfg.server_lr > 0:
        raise ValueError(f"server_lr must be > 0, got {cfg.server_lr}")
    if not 0 <= cfg.server_momentum < 1:
        raise ValueError(f"server_momentum (beta1) must lie in [0, 1), got {cfg.server_momentum}")
    if not 0 <= cfg.server_beta2 < 1:
        raise ValueError(f"server_beta2 must lie in [0, 1), got {cfg.server_beta2}")
    if not cfg.server_tau > 0:
        raise ValueError(f"server_tau must be > 0, got {cfg.server_tau}")
    if cfg.packing == "coeff" and cfg.server_opt != "fedavg":
        raise ValueError(f"server_opt={cfg.server_opt!r} needs slot packing: the step is fused into the slot decode, "
                         "coefficient packing supports server_opt='fedavg' only")


def lipschitz(name: str, lr: float, beta1: float, tau: float) -> float:
    """Bound on |dx'/dd| of one step: how far an error in the decoded average can move the new model."""
    if name == "fedavgm":
        return lr / (1.0 - beta1)
    return lr * (1.0 - beta1) / tau


def reference_step(name: str, hp: Dict[str, float], x: torch.Tensor, a: torch.Tensor, m: torch.Tensor,
                   v: torch.Tensor, n_trainable: int) -> torch.Tensor:
    """The update of DESIGN.md §8 in float64 on plain tensors (the oracle of ``simulate_clients``). ``m`` and
    ``v`` (float64, ``n_trainable`` entries) are updated in place; returns x' (float64)."""
    lr, b1, b2, tau = hp["lr"], hp["beta1"], hp["beta2"], hp["tau"]
    x, a = x.double(), a.double()
    nt = n_trainable
    d = a[:nt] - x[:nt]
    out = a.clone()
    if name == "fedavgm":
        m.mul_(b1).add_(d)
        out[:nt] = x[:nt] + lr * m
        return out
    m.mul_(b1).add_((1 - b1) * d)
    d2 = d * d
    if name == "fedadagrad":
        v.add_(d2)
    elif name == "fedyogi":
        v.sub_((1 - b2) * d2 * torch.sign(v - d2))
    elif name == "fedadam":
        v.mul_(b2).add_((1 - b2) * d2)
    else:
        raise ValueError(f"no server step for {name!r}")
    out[:nt] = x[:nt] + lr * m / (v.sqrt() + tau)
    return out


class ServerOptimizer:
    """Optimizer state of the key holder: fp32 ``m`` and ``v`` of ``n_trainable`` entries on the context device,
    allocated on the first step (m = 0, v = tau^2)."""

    def __init__(self, name: str, n_trainable: int, device, lr: float = 1.0, beta1: float = 0.9,
                 beta2: float = 0.99, tau: float = 1e-3):
        if name not in SERVER_OPTS or SERVER_OPTS[name] == 0:
            raise ValueError(f"ServerOptimizer needs one of fedavgm, fedadagrad, fedyogi, fedadam, got {name!r}")
        self.name = name
        self.code = SERVER_OPTS[name]
        self.n_trainable = int(n_trainable)
        self.device = torch.device(device)
        self.hp = {"lr": float(lr), "beta1": float(beta1), "beta2": float(beta2), "tau": float(tau)}
        self.m: Optional[torch.Tensor] = None
        self.v: Optional[torch.Tensor] = None

    @classmethod
    def from_config(cls, cfg, n_trainable: int, device) -> "ServerOptimizer":
        return cls(cfg.server_opt, n_trainable, device, lr=cfg.server_lr, beta1=cfg.server_momentum,
                   beta2=cfg.server_beta2, tau=cfg.server_tau)

    def ensure_state(self) -> None:
        if self.m is None:
            self.m = torch.zeros(self.n_trainable, dtype=torch.float32, device=self.device)
            tau = torch.tensor(self.hp["tau"], dtype=torch.float32)
            self.v = torch.full((self.n_trainable,), float(tau * tau), dtype=torch.float32, device=self.device)

    def step(self, ctx, agg, sk: torch.Tensor, divide_by: float, x_t: torch.Tensor, out: torch.Tensor,
             offset: int = 0, avg_out: Optional[torch.Tensor] = None) -> None:
        """Decrypt ``agg`` (flat values ``offset .. offset + agg.nvals - 1`` of the model), divide by
        ``divide_by`` and write the stepped model into ``out`` at the same indices; one decode launch."""
        self.ensure_state()
        ctx.decrypt_server_step(agg, sk, divide_by, x_t, out, self.m, self.v, self.code, self.hp, self.n_trainable,
                                offset=offset, avg_out=avg_out)

    def reset(self) -> None:
        """Start fresh: the next step allocates m = 0, v = tau^2."""
        self.m = self.v = None

    def state_dict(self) -> Dict:
        return {"name": self.name, "hp": dict(self.hp), "n_trainable": self.n_trainable,
                "m": None if self.m is None else self.m.detach().cpu().clone(),
                "v": None if self.v is None else self.v.detach().cpu().clone()}

    def load_state_dict(self, st: Dict) -> None:
        if st["name"] != self.name or int(st["n_trainable"]) != self.n_trainable:
            raise ValueError(f"server state of {st['name']} over {st['n_trainable']} values does not fit "
                             f"{self.name} over {self.n_trainable}")
        if st["m"] is None:
            self.m = self.v = None
            return
        self.m = st["m"].to(self.device, torch.float32).contiguous()
        self.v = st["v"].to(self.device, torch.float32).contiguous()

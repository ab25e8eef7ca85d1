"""Ciphertext all-reduce transports.

FedAvg's server loop (FLPyfhelin.py:372-381: import each client's pickle, ``enc + dct`` per
scalar ciphertext) is a coefficient-wise modular sum over clients. Three interchangeable
transports implement it behind one interface:

* ``FusedTransport``   — the product: one sm_90a kernel that pulls peer tiles over NVLink,
  adds, reduces mod q_l and pushes/broadcasts the result (csrc/comm/allreduce_modq.cu).
* ``CollectiveTransport`` — the baseline the product must beat: ``all_reduce(int64, SUM)``
  through NCCL (or gloo on CPU) followed by a separate mod-q kernel (SURVEY.md K2).
* ``LoopbackTransport`` — in-process fake backend for tests and the single-process
  simulation (the reference's loop-over-clients pattern, SURVEY.md §4.3).
"""
from __future__ import annotations

import os
from typing import List, Optional

import torch
import torch.distributed as dist

from .. import _ext
from ..he.context import CKKSContext
from .symm import SymmetricBuffer

ALGOS = {"two_shot": 0, "one_shot": 1, "multimem": 2}


class Transport:
    name = "abstract"
    world = 1
    rank = 0

    def buffer(self, numel: int) -> torch.Tensor:
        """Where a rank should write its ciphertext words before ``allreduce``."""
        raise NotImplementedError

    def allreduce(self, data: torch.Tensor) -> torch.Tensor:
        """Sum ``data`` ([C,2,L,N] int64 words) over ranks modulo each limb prime."""
        raise NotImplementedError

    def contributors(self) -> int:
        return self.world


class FusedTransport(Transport):
    name = "fused"

    def __init__(self, ctx: CKKSContext, max_numel: int, group: Optional[dist.ProcessGroup] = None,
                 algo: str = "auto", blocks: int = 0, threads: int = 512, timeout_s: float = 20.0,
                 backend: str = "auto", no_owner: int = -1):
        self.ops = _ext.ops()
        self.ctx = ctx
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.max_numel = int((max_numel + 3) // 4 * 4)
        self.threads = threads
        # one CTA per SM: the kernel is a copy engine, a second CTA per SM only adds flag traffic
        self.max_blocks = (torch.cuda.get_device_properties(ctx.device).multi_processor_count
                           if ctx.device.type == "cuda" else 128)
        self.blocks = blocks
        # rank that must never read un-aggregated ciphertext (the secret-key holder): it owns no chunk
        self.no_owner = int(no_owner) if self.world > 1 else -1
        self.stats = torch.zeros(1, dtype=torch.int32, device=ctx.device)
        self.timeout_ms = int(timeout_s * 1000)
        self.sym = SymmetricBuffer(self.max_numel, torch.int64, ctx.device, group, backend)
        self.sig = SymmetricBuffer(2 * self.max_blocks * max(self.world, 1) + 64, torch.int32,
                                   ctx.device, group, backend)
        self.out = torch.empty(self.max_numel, dtype=torch.int64, device=ctx.device)
        self.status = torch.zeros(1, dtype=torch.int32, device=ctx.device)
        self.algo = os.environ.get("HEFL_ALLREDUCE_ALGO", algo)
        self.last_algo = None

    def buffer(self, numel: int) -> torch.Tensor:
        if numel > self.max_numel:
            raise ValueError(f"symmetric buffer too small: {numel} > {self.max_numel}")
        return self.sym.tensor[:numel]

    def pick_algo(self, nbytes: int) -> str:
        if self.algo != "auto":
            # one_shot has every rank load every peer's whole ciphertext, so a key holder turns a forced one_shot
            # into two_shot (where it owns no chunk); multimem honours the key holder and is kept
            return "two_shot" if self.algo == "one_shot" and self.no_owner >= 0 else self.algo
        if self.world == 1:
            return "two_shot"
        if nbytes <= 256 * 1024 and self.no_owner < 0:
            return "one_shot"          # every rank reads everything: never with a key holder
        if self.sym.mc_ptr and os.environ.get("HEFL_USE_MULTIMEM", "0") == "1":
            return "multimem"
        return "two_shot"

    def pick_blocks(self, numel: int, algo: str) -> int:
        if self.blocks:
            return min(self.blocks, self.max_blocks)
        owners = self.world - (1 if self.no_owner >= 0 else 0)
        work = numel // 4 if algo == "one_shot" else max(1, numel // 4 // max(1, owners))   # 32-byte quads
        return max(1, min(self.max_blocks, (work + self.threads - 1) // self.threads))

    def allreduce(self, data: torch.Tensor) -> torch.Tensor:
        numel = data.numel()
        base = self.sym.tensor
        off = data.data_ptr() - base.data_ptr()
        if numel % 4:
            raise ValueError("ciphertext word count must be a multiple of 4")
        inside = 0 <= off and off + numel * 8 <= self.max_numel * 8 and off % 32 == 0
        if not inside:
            # caller did not encrypt in place: stage into the symmetric buffer
            self.buffer(numel).copy_(data.reshape(-1))
            off = 0
        algo = self.pick_algo(numel * 8)
        self.last_algo = algo
        blocks = self.pick_blocks(numel, algo)
        e0 = off // 8                              # a view of the symmetric buffer (chunked pipelines)
        out = self.out[e0:e0 + numel] if algo == "one_shot" else None
        self.ops.allreduce_modq([p + off for p in self.sym.ptrs], self.sig.ptrs,
                                self.sym.mc_ptr + off if self.sym.mc_ptr else 0, out, self.status,
                                self.ctx.consts_cpu, numel, data.shape[-2], self.ctx.logn,
                                self.rank, self.world, ALGOS[algo], blocks, self.threads,
                                self.timeout_ms, self.no_owner, self.stats)
        src = self.out if algo == "one_shot" else base
        return src[e0:e0 + numel].view(data.shape)

    def peer_load_steps(self) -> int:
        """32-byte peer-load steps this rank has issued since the last call (0 for a key holder)."""
        n = int(self.stats.item())
        self.stats.zero_()
        return n

    def check_status(self) -> None:
        """Raises if a bounded spin-wait timed out in a previous launch (failure detection)."""
        code = int(self.status.item())
        if code:
            self.status.zero_()
            peer = (code & 0xFF) - 1
            raise TimeoutError(
                f"fused all-reduce: rank {self.rank} block {(code >> 16)} timed out waiting for "
                f"rank {peer} at barrier {(code >> 8) & 0xFF} after {self.timeout_ms} ms")


class CollectiveTransport(Transport):
    """NCCL (GPU) / gloo (CPU) all-reduce + separate mod kernel: the baseline (K2)."""

    name = "nccl"

    def __init__(self, ctx: CKKSContext, max_numel: int, group: Optional[dist.ProcessGroup] = None):
        self.ops = _ext.ops()
        self.ctx = ctx
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.buf = torch.empty(int(max_numel), dtype=torch.int64, device=ctx.device)
        if dist.is_initialized():
            self.name = str(dist.get_backend(group))          # "nccl" on GPUs, "gloo" on CPU

    def buffer(self, numel: int) -> torch.Tensor:
        return self.buf[:numel]

    def allreduce(self, data: torch.Tensor) -> torch.Tensor:
        if self.world > 1:
            dist.all_reduce(data, op=dist.ReduceOp.SUM, group=self.group)
        self.ops.reduce_mod_(data, data.shape[-2], self.ctx.consts)
        return data


class LoopbackTransport(Transport):
    """All clients live in this process; ``contribute`` then ``reduce``."""

    name = "loopback"

    def __init__(self, ctx: CKKSContext, world: int):
        self.ops = _ext.ops()
        self.ctx = ctx
        self.world = int(world)
        self.rank = 0
        self.slots: List[Optional[torch.Tensor]] = [None] * self.world
        self.mask = [True] * self.world

    def buffer(self, numel: int) -> torch.Tensor:
        return torch.empty(numel, dtype=torch.int64, device=self.ctx.device)

    def contribute(self, client: int, data: torch.Tensor) -> None:
        self.slots[client] = data

    def drop(self, client: int) -> None:
        """Fault-injection hook: exclude a client from this round (participation mask)."""
        self.mask[client] = False
        self.slots[client] = None

    def contributors(self) -> int:
        return sum(1 for s, m in zip(self.slots, self.mask) if m and s is not None)

    def reduce(self) -> torch.Tensor:
        srcs = [s.contiguous() for s, m in zip(self.slots, self.mask) if m and s is not None]
        if not srcs:
            raise RuntimeError("no client contributed to this round")
        out = torch.empty_like(srcs[0])
        self.ops.local_sum_modq(srcs, out, srcs[0].shape[-2], self.ctx.logn, self.ctx.consts)
        return out

    def allreduce(self, data: torch.Tensor) -> torch.Tensor:
        self.contribute(0, data)
        return self.reduce()

    def reset(self) -> None:
        self.slots = [None] * self.world
        self.mask = [True] * self.world


def make_transport(kind: str, ctx: CKKSContext, max_numel: int, world: int = 1,
                   group: Optional[dist.ProcessGroup] = None, **kw) -> Transport:
    if kind == "fused":
        return FusedTransport(ctx, max_numel, group, **kw)
    kw.pop("no_owner", None)
    if kind in ("nccl", "gloo", "collective"):
        return CollectiveTransport(ctx, max_numel, group)
    if kind == "loopback":
        return LoopbackTransport(ctx, world)
    raise ValueError(f"unknown transport {kind}")

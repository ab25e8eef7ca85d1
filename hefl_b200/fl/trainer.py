"""Local (per-client) training: the PyTorch replacement of ``model.fit`` in the reference
(FLPyfhelin.py:161-198).

Recipe kept from the reference: Adam(lr=1e-3) with Keras' legacy time-based decay 1e-4 (:140),
categorical cross-entropy + accuracy (:141), batch 32 (:33), EarlyStopping on training loss
(patience 5, restore best weights, :186), ReduceLROnPlateau on training loss (patience 2,
factor 0.3, floor 1e-6, :187), ModelCheckpoint on best training accuracy (:189-191),
augmentation shear/zoom/flip and 1/255 rescale (:80-86).

Design: parameters, gradients and Adam moments are flat fp32 buffers (``ParamPack``),
the optimiser is one fused kernel, the step (forward -> backward -> Adam) is captured in a CUDA
graph and replayed, the learning-rate scale and step counter live on the device, and losses are
read back asynchronously (one sync per epoch, not per step). With the tcgen05 engine an epoch is
a four-stream software pipeline: H2D / gather + pre-processing of batch i+1 (prep stream), the
graph of step i (main + the engine's side stream), the loss read-back of step i-1 (stats stream);
the first batch of the next pass (validation, next epoch) is staged under the last step.
Two NN backends: ``cudnn`` (PyTorch autograd + cuDNN/cuBLAS in bf16 autocast, fused BN kernels and
optional fp8 1x1 convolutions for the ResNets — also the baseline arm) and ``tcgen05``
(hand-written kernels, ``hefl_b200.ops.conv_engine``).
"""
from __future__ import annotations

import dataclasses
import os
from typing import Callable, Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

from .. import _ext
from ..config import FLConfig
from ..models.pack import ParamPack
from .data import BatchFeeder, augment_batch


@dataclasses.dataclass
class EpochStats:
    loss: float
    accuracy: float
    val_loss: float
    val_accuracy: float
    lr_scale: float


class LocalTrainer:
    def __init__(self, model: torch.nn.Module, pack: ParamPack, cfg: FLConfig, device: torch.device,
                 backend: Optional[str] = None, augment: bool = True, use_graph: Optional[bool] = None):
        self.ops = _ext.ops()
        self.model = model
        self.pack = pack
        self.cfg = cfg
        self.device = device
        self.backend = backend or cfg.nn_backend
        self.augment = augment
        self.cuda = device.type == "cuda"
        self.use_graph = self.cuda if use_graph is None else (use_graph and self.cuda)
        n = pack.n_trainable
        self.m = torch.zeros(n, dtype=torch.float32, device=device)
        self.v = torch.zeros(n, dtype=torch.float32, device=device)
        self.step_t = torch.zeros(1, dtype=torch.int64, device=device)
        self.lr_scale = torch.ones(1, dtype=torch.float32, device=device)
        # FedProx: the model at the start of fit() (the round's global model); the Adam kernels add mu*(w - anchor)
        # to the gradient. Allocated once, so captured graphs keep a valid pointer to it.
        self.mu = float(cfg.fedprox_mu)
        self.anchor = torch.zeros(n, dtype=torch.float32, device=device) if self.mu > 0 else None
        # personal layers (DESIGN.md §10): a head-only step updates flat[head_lo:n]
        self.head_lo = pack.dense_tail_start(cfg.personal_layers) if cfg.personal_layers else n
        # "fp8": bf16 autocast + e4m3 GEMMs for the 1x1 convolutions of the ResNets (ops/fp8.py)
        self.amp_dtype = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32,
                          "fp8": torch.bfloat16}[cfg.dtype]
        from ..ops import fp8 as _fp8

        _fp8.set_model_fp8(model, cfg.dtype == "fp8" and self.cuda)      # per model, not process-wide
        B, S, C = cfg.batch_size, cfg.image_size, cfg.in_channels
        self.static_x = torch.zeros(B, S, S, C, dtype=torch.uint8, device=device)
        self.static_y = torch.zeros(B, dtype=torch.int64, device=device)
        self.out_train = torch.zeros(2, dtype=torch.float32, device=device)   # loss, ncorrect
        self.out_eval = torch.zeros(2, dtype=torch.float32, device=device)
        self._graph_train: Optional[torch.cuda.CUDAGraph] = None
        self._graph_eval: Optional[torch.cuda.CUDAGraph] = None
        self.graph_launches = [0, 0]      # our kernels inside one train / eval graph
        self.head_launches = 0            # ... inside one head-only graph (captured by the first head-only fit)
        self.replayed_launches = 0        # ... summed over replays (bench.py gpu_launches)
        self.engine = None
        if self.backend == "cudnn" and self.cuda:
            # the library arm gets what a tuned PyTorch script gets: cuDNN's algorithm search (input is already
            # NHWC storage viewed as NCHW, i.e. channels_last activations), bf16 autocast, CUDA graphs
            torch.backends.cudnn.benchmark = True
        if self.backend == "tcgen05" and not hasattr(model, "convs"):
            # the ResNets: same autograd / CUDA-graph step as the library arm, with every eligible convolution
            # (1x1, 3x3 stride 1) on the tcgen05 GEMM kernels of ops/tc_conv.py
            from ..ops import tc_conv

            tc_conv.set_model_tc(model, self.cuda)
            torch.backends.cudnn.benchmark = True        # the stem and the three stride-2 3x3 layers stay on cuDNN
            self.backend = "tcgen05-gemm"
        if self.backend == "tcgen05":
            from ..ops.conv_engine import MedCNNEngine

            self.engine = MedCNNEngine(model, pack, cfg, device)
            # staged input pipeline: batch i+1 is pre-processed into the other X0 slot on `prep_stream`
            # while the graph of step i runs; one captured graph per (train/eval, slot)
            self.static_y2 = [torch.zeros(B, dtype=torch.int64, device=device) for _ in range(2)]
            # per-slot result buffers: the D2H read of step i runs on `stats_stream` under step i+1
            self.out_train2 = [self.out_train, torch.zeros(2, dtype=torch.float32, device=device)]
            self.out_eval2 = [self.out_eval, torch.zeros(2, dtype=torch.float32, device=device)]
            self.stats_stream = torch.cuda.Stream(device)
            self._stats_done = [torch.cuda.Event() for _ in range(2)]
            self._graphs: Dict[Tuple[bool, int], torch.cuda.CUDAGraph] = {}
            self.prep_stream = torch.cuda.Stream(device)
            self._slot_ready = [torch.cuda.Event() for _ in range(2)]
            self._slot_free = [torch.cuda.Event() for _ in range(2)]
            self._pre = None         # (feeder, train, iterator, slot) of a first batch staged ahead of its pass
            self._score_graphs: Dict[int, torch.cuda.CUDAGraph] = {}     # captured by the first score() only
            self._score_bufs = None  # (counts, loss, err), nvalid per slot, probs of the captured score graphs
        self.score_launches = 0           # our kernels inside one score graph (+ the pre-process launch)

    # ------------------------------------------------------------------ one step (eager)
    def _prep(self, x_u8: torch.Tensor, train: bool) -> torch.Tensor:
        x = x_u8.permute(0, 3, 1, 2).to(torch.float32) * (1.0 / 255.0)   # NHWC storage, NCHW view
        if train and self.augment:
            x = augment_batch(x, None)
        return x

    def _forward(self, x_u8: torch.Tensor, train: bool) -> torch.Tensor:
        x = self._prep(x_u8, train)
        if self.amp_dtype != torch.float32 and self.cuda:
            with torch.autocast("cuda", dtype=self.amp_dtype):
                return self.model(x).float()
        return self.model(x)

    def _train_eager(self, x_u8: torch.Tensor, y: torch.Tensor) -> None:
        if self.engine is not None:
            self.engine.train_step(x_u8, y, self.out_train, augment=self.augment, opt=self)
            return
        logits = self._forward(x_u8, True)
        loss = F.cross_entropy(logits, y)
        loss.backward()
        self.out_train[0] = loss.detach()
        self.out_train[1] = (logits.argmax(1) == y).sum()
        self._optimizer_step()

    def _head_eager(self, x_u8: torch.Tensor, y: torch.Tensor) -> None:
        """Head-only step: the same augmented batch as a train step, the frozen layers under no_grad, Adam over the
        personal layers alone."""
        if self.engine is not None:
            self.engine.preprocess(x_u8, 0, True, self.augment)
            self.engine.head_step_staged(0, y, self.out_train, opt=self)
            return
        fcs = self.model.fcs
        shared = len(fcs) - self.cfg.personal_layers
        amp = self.amp_dtype != torch.float32 and self.cuda
        with torch.autocast("cuda", dtype=self.amp_dtype, enabled=amp):
            with torch.no_grad():
                x = self.model.features(self._prep(x_u8, True)).permute(0, 2, 3, 1).flatten(1)   # Keras Flatten
                for fc in fcs[:shared]:
                    x = F.relu(fc(x))
            for j in range(shared, len(fcs)):
                x = fcs[j](x)
                if j + 1 < len(fcs):
                    x = F.relu(x)
        logits = x.float()
        loss = F.cross_entropy(logits, y)
        loss.backward()
        self.out_train[0] = loss.detach()
        self.out_train[1] = (logits.argmax(1) == y).sum()
        c = self.cfg
        lo, hi = self.head_lo, self.pack.n_trainable
        self.step_t += 1
        self.ops.adam_step_(self.pack.trainable()[lo:hi], self.pack.grad[lo:hi], self.m[lo:hi], self.v[lo:hi], None,
                            self.step_t, self.lr_scale, c.lr, c.lr_decay, 0.9, 0.999, 1e-7,
                            self.anchor[lo:hi] if self.anchor is not None else None, self.mu)

    def _head_staged(self, slot: int) -> None:
        self.engine.head_step_staged(slot, self.static_y2[slot], self.out_train2[slot], opt=self)

    def _train_staged(self, slot: int) -> None:
        """Graph body of the tcgen05 engine: forward/backward on the pre-processed batch of ``slot`` + update."""
        self.engine.train_step_staged(slot, self.static_y2[slot], self.out_train2[slot], opt=self)

    # update hooks driven by the engine (it knows when each layer's gradient is final)
    def bump(self) -> None:
        self.step_t += 1

    def apply(self, lo: int, hi: int) -> None:
        c = self.cfg
        if hi <= lo:
            return
        self.ops.adam_step_(self.pack.trainable()[lo:hi], self.pack.grad[lo:hi], self.m[lo:hi], self.v[lo:hi],
                            self.engine.shadow[lo:hi], self.step_t, self.lr_scale, c.lr, c.lr_decay, 0.9, 0.999, 1e-7,
                            self.anchor[lo:hi] if self.anchor is not None else None, self.mu)

    def _optimizer_step(self) -> None:
        """Adam over every parameter after an autograd step (the cudnn and ResNet backends)."""
        c = self.cfg
        self.step_t += 1
        self.ops.adam_step_(self.pack.trainable(), self.pack.grad, self.m, self.v, None,
                            self.step_t, self.lr_scale, c.lr, c.lr_decay, 0.9, 0.999, 1e-7, self.anchor, self.mu)

    def _eval_eager(self, x_u8: torch.Tensor, y: torch.Tensor) -> None:
        with torch.no_grad():
            if self.engine is not None:
                self.engine.eval_step(x_u8, y, self.out_eval)
                return
            logits = self._forward(x_u8, False)
            self.out_eval[0] = F.cross_entropy(logits, y)
            self.out_eval[1] = (logits.argmax(1) == y).sum()

    # ------------------------------------------------------------------ graph capture
    def _capture(self) -> None:
        self.model.train()
        snap = (self.pack.flat.clone(), self.m.clone(), self.v.clone(), self.step_t.clone())
        side = torch.cuda.Stream(self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        eng = self.engine
        with torch.cuda.stream(side):
            if eng is not None:
                for slot in range(2):
                    eng.preprocess(self.static_x, slot, False, False)
            for _ in range(3):
                if eng is not None:
                    for slot in range(2):
                        self._train_staged(slot)
                        eng.eval_step_staged(slot, self.static_y2[slot], self.out_eval2[slot])
                else:
                    self._train_eager(self.static_x, self.static_y)
                    self._eval_eager(self.static_x, self.static_y)
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        l0 = int(self.ops.launch_count())
        if eng is not None:
            counts = {}
            for slot in range(2):
                for train in (True, False):
                    a = int(self.ops.launch_count())
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        if train:
                            self._train_staged(slot)
                        else:
                            with torch.no_grad():
                                eng.eval_step_staged(slot, self.static_y2[slot], self.out_eval2[slot])
                    self._graphs[(train, slot)] = g
                    counts[(train, slot)] = int(self.ops.launch_count()) - a
            self._graph_train, self._graph_eval = self._graphs[(True, 0)], self._graphs[(False, 0)]
            self.graph_launches = [counts[(True, 0)] + 1, counts[(False, 0)] + 1]     # + the pre-process launch
        else:
            self._graph_train = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self._graph_train):
                self._train_eager(self.static_x, self.static_y)
            l1 = int(self.ops.launch_count())
            self._graph_eval = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self._graph_eval):
                self._eval_eager(self.static_x, self.static_y)
            self.graph_launches = [l1 - l0, int(self.ops.launch_count()) - l1]
        # undo the warm-up updates
        self.pack.flat.copy_(snap[0]); self.m.copy_(snap[1]); self.v.copy_(snap[2]); self.step_t.copy_(snap[3])
        self.pack.grad.zero_()
        if self.engine is not None:
            self.engine.after_restore()
        torch.cuda.synchronize(self.device)

    def _capture_head(self) -> None:
        """Head-only graphs of the tcgen05 engine, one per input slot, captured by the first head-only fit only, so a
        run without head epochs captures exactly the train / eval graphs."""
        if not self._graphs:
            self._capture()
        eng, cur = self.engine, torch.cuda.current_stream(self.device)
        snap = (self.pack.flat.clone(), self.m.clone(), self.v.clone(), self.step_t.clone())
        side = torch.cuda.Stream(self.device)
        side.wait_stream(cur)
        side.wait_stream(self.prep_stream)
        with torch.cuda.stream(side):
            for slot in range(2):
                eng.preprocess(self.static_x, slot, False, False)
            for _ in range(3):
                for slot in range(2):
                    self._head_staged(slot)
        cur.wait_stream(side)
        torch.cuda.synchronize(self.device)
        for slot in range(2):
            a = int(self.ops.launch_count())
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._head_staged(slot)
            self._graphs[("head", slot)] = g
            if slot == 0:
                self.head_launches = int(self.ops.launch_count()) - a + 1       # + the pre-process launch
        self.pack.flat.copy_(snap[0]); self.m.copy_(snap[1]); self.v.copy_(snap[2]); self.step_t.copy_(snap[3])
        self.pack.grad.zero_()
        eng.after_restore()
        torch.cuda.synchronize(self.device)

    def _alloc_score_bufs(self, nbins: int) -> None:
        """(int32 counts, float64 loss sum, int32 error flag), the valid row count of each input slot, and probs."""
        C, dev = self.model.fcs[-1].out_features, self.device
        self._score_bufs = ((torch.zeros(C * C * (nbins + 1), dtype=torch.int32, device=dev),
                             torch.zeros(1, dtype=torch.float64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)),
                            [torch.zeros(1, dtype=torch.int32, device=dev) for _ in range(2)],
                            torch.zeros(self.cfg.batch_size, C, dtype=torch.float32, device=dev))

    def _score_step(self, slot: int, y: Optional[torch.Tensor] = None) -> None:
        bufs, nv, probs = self._score_bufs
        self.engine.score_staged(slot, self.static_y2[slot] if y is None else y, nv[slot], bufs, probs)

    def _capture_score(self, nbins: int) -> None:
        """Score graphs of the tcgen05 engine, one per input slot, captured by the first ``score`` only (and again if
        the bin count changes), so a run that never scores captures exactly the graphs it captured before. Scoring
        writes no parameter, gradient, optimiser state or augmentation position, so nothing needs restoring."""
        eng, cur = self.engine, torch.cuda.current_stream(self.device)
        self._alloc_score_bufs(nbins)
        side = torch.cuda.Stream(self.device)
        side.wait_stream(cur)
        side.wait_stream(self.prep_stream)
        with torch.cuda.stream(side):
            for slot in range(2):
                eng.preprocess(self.static_x, slot, False, False)
            for _ in range(3):
                for slot in range(2):
                    self._score_step(slot)
        cur.wait_stream(side)
        torch.cuda.synchronize(self.device)
        self._score_graphs = {}
        for slot in range(2):
            a = int(self.ops.launch_count())
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._score_step(slot)
            self._score_graphs[slot] = g
            if slot == 0:
                self.score_launches = int(self.ops.launch_count()) - a + 1       # + the pre-process launch
        torch.cuda.synchronize(self.device)

    @torch.no_grad()
    def score(self, feeder: BatchFeeder, counts_row: torch.Tensor) -> None:
        """Federated-evaluation counts of the installed model (DESIGN.md §13) over one pass of the non-shuffled
        ``feeder``, added into ``counts_row`` (float64 [V], ``fedeval`` layout) on the trainer's device. The tcgen05
        engine scores on its own kernels -- graph-replayed in the ``_run_epoch`` pipeline, or eagerly without graphs;
        the other backends run the model's forward in its dtype and ``score_counts_torch``. Weights, gradients,
        optimiser state, the augmentation position and the RNG are left as they were. Raises ValueError if a label is
        outside 0..C-1."""
        from .fedeval import score_counts_torch

        if feeder.shuffle:
            raise ValueError("score needs a non-shuffled feeder (the wrapped rows of its last batch are skipped)")
        C = self.model.fcs[-1].out_features if hasattr(self.model, "fcs") else None
        rows, B = len(feeder.indices), feeder.bs
        if rows == 0:
            return
        if self.engine is None:
            nb = (counts_row.numel() - 1) // (C * C) - 1 if C else None
            was = self.model.training
            self.model.eval()
            try:
                for i, (x, y) in enumerate(feeder.epoch()):
                    nv = min(B, rows - i * B)
                    logits = self._forward(x, False).float()
                    if nb is None:
                        C = logits.shape[1]
                        nb = (counts_row.numel() - 1) // (C * C) - 1
                    if int(y[:nv].min()) < 0 or int(y[:nv].max()) >= C:
                        raise ValueError(f"score: labels must be in 0..{C - 1}")
                    counts_row.add_(score_counts_torch(logits[:nv], y[:nv], nb).to(counts_row.device))
            finally:
                self.model.train(was)
            return
        nbins = (counts_row.numel() - 1) // (C * C) - 1
        graphs = self.use_graph
        if graphs and (not self._score_graphs or self._score_bufs[0][0].numel() != counts_row.numel() - 1):
            self._capture_score(nbins)
        if not graphs and (self._score_bufs is None or self._score_bufs[0][0].numel() != counts_row.numel() - 1):
            self._alloc_score_bufs(nbins)
        (counts, loss, err), nv, _ = self._score_bufs
        counts.zero_(); loss.zero_(); err.zero_()
        if graphs:
            self._run_epoch(feeder, False, None, score=True)
        else:
            for i, (x, y) in enumerate(feeder.epoch()):
                self.engine.preprocess(x, 0, False, False)
                nv[0].fill_(min(B, rows - i * B))
                self._score_step(0, y)
        if int(err.item()):
            raise ValueError(f"score: labels must be in 0..{C - 1}")
        counts_row[:-1].add_(counts.to(counts_row.device, torch.float64))
        counts_row[-1:].add_(loss.to(counts_row.device))

    # ------------------------------------------------------------------ public API
    def prepare(self) -> None:
        """Capture the CUDA graphs now rather than at the first step (a rank with several clients captures once,
        before any client's state is installed). No-op without graphs or when they exist."""
        if self.use_graph and (not self._graphs if self.engine is not None else self._graph_train is None):
            self._capture()

    def train_step(self, x_u8: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        """One optimisation step on a uint8 NHWC batch. Returns a device tensor [loss, ncorrect]."""
        if self.use_graph:
            if self._graph_train is None:
                self._capture()
            if self.engine is not None:
                self.engine.preprocess(x_u8, 0, True, self.augment)     # straight into X0[0], no staging copy
                self.static_y2[0].copy_(y, non_blocking=True)
            else:
                self.static_x.copy_(x_u8, non_blocking=True)
                self.static_y.copy_(y, non_blocking=True)
            self._graph_train.replay()
            self.replayed_launches += self.graph_launches[0]
        else:
            self._train_eager(x_u8, y)
        return self.out_train

    def head_step(self, x_u8: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        """One head-only step (personal layers only, conv base frozen). Graph-replayed on the tcgen05 engine; eager
        on the autograd backends. Returns a device tensor [loss, ncorrect]."""
        if self.use_graph and self.engine is not None:
            if ("head", 0) not in self._graphs:
                self._capture_head()
            self.engine.preprocess(x_u8, 0, True, self.augment)
            self.static_y2[0].copy_(y, non_blocking=True)
            self._graphs[("head", 0)].replay()
            self.replayed_launches += self.head_launches
            return self.out_train2[0]
        self._head_eager(x_u8, y)
        return self.out_train

    def eval_step(self, x_u8: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        if self.use_graph:
            if self._graph_eval is None:
                self._capture()
            if self.engine is not None:
                self.engine.preprocess(x_u8, 0, False, False)
                self.static_y2[0].copy_(y, non_blocking=True)
            else:
                self.static_x.copy_(x_u8, non_blocking=True)
                self.static_y.copy_(y, non_blocking=True)
            self._graph_eval.replay()
            self.replayed_launches += self.graph_launches[1]
        else:
            self._eval_eager(x_u8, y)
        return self.out_eval

    def _run_epoch(self, feeder, train: bool, stats: Optional[torch.Tensor], nxt=None, head: bool = False,
                   score: bool = False) -> None:
        """One pass over ``feeder``; per-step [loss, ncorrect] land in ``stats`` (pinned host rows).

        tcgen05 engine + CUDA graphs: software pipeline over batches — batch i+1 is fetched (H2D or
        on-device gather) and pre-processed into the other X0 slot on ``prep_stream`` while the captured
        graph of step i runs on the main stream; events hand the slots back and forth. ``nxt`` =
        (feeder, train) of the pass that follows: its first batch is staged under this pass's last
        step, so consecutive passes (train -> validation -> next epoch) have no pipeline-fill bubble. ``head``: a
        training pass of head-only steps (pre-processed and staged as a train pass). ``score``: a pass of the captured
        score graphs into ``_score_bufs`` (``stats`` unused): each slot's valid row count is set as it is staged, so
        the rows the feeder wraps into the last batch are not counted, and nothing is read back."""
        if self.engine is None or not self.use_graph:
            for i, (x, y) in enumerate(feeder.epoch()):
                out = self.head_step(x, y) if head else self.train_step(x, y) if train else self.eval_step(x, y)
                stats[i].copy_(out, non_blocking=True)       # D2H of the step's loss/accuracy
            return
        if not self._graphs and not score:
            self._capture()
        if head and ("head", 0) not in self._graphs:
            self._capture_head()
        main, prep, sst = torch.cuda.current_stream(self.device), self.prep_stream, self.stats_stream
        n = feeder.steps
        outs = self.out_train2 if train else self.out_eval2
        rows, staged = len(feeder.indices) if score else 0, [0]

        def stage(it, slot: int, tr: bool) -> None:
            with torch.cuda.stream(prep):
                prep.wait_event(self._slot_free[slot])        # the graph that last read this slot is done
                x, y = next(it)                               # feeder work (gather / wait for H2D) on prep
                self.engine.preprocess(x, slot, tr, self.augment and tr)
                self.static_y2[slot].copy_(y, non_blocking=True)
                if score:
                    self._score_bufs[1][slot].fill_(min(feeder.bs, rows - staged[0] * feeder.bs))
                    staged[0] += 1
                self._slot_ready[slot].record(prep)

        pre, self._pre = self._pre, None
        if pre is not None and pre[0] is feeder and pre[1] == train:
            it, s0 = pre[2], pre[3]                           # batch 0 was staged by the previous pass
        else:
            if pre is not None:
                pre[2].close()
            prep.wait_stream(main)
            for ev in self._slot_free + self._stats_done:
                ev.record(main)
            it, s0 = iter(feeder.epoch()), 0
            stage(it, 0, train)
        for i in range(n):
            slot = (s0 + i) & 1
            if i + 1 < n:
                stage(it, slot ^ 1, train)
            elif nxt is not None and nxt[0] is not None and nxt[0].steps > 0:
                nit = iter(nxt[0].epoch())
                stage(nit, slot ^ 1, nxt[1])
                self._pre = (nxt[0], nxt[1], nit, slot ^ 1)
            main.wait_event(self._slot_ready[slot])
            if score:
                self._score_graphs[slot].replay()
                self._slot_free[slot].record(main)
                continue
            main.wait_event(self._stats_done[slot])           # result buffer of this slot has been read back
            self._graphs[("head" if head else train, slot)].replay()
            self._slot_free[slot].record(main)
            with torch.cuda.stream(sst):                      # D2H of the step's loss/accuracy, off the main stream
                sst.wait_event(self._slot_free[slot])
                stats[i].copy_(outs[slot], non_blocking=True)
                self._stats_done[slot].record(sst)
        self.replayed_launches += n * (self.score_launches if score else self.head_launches if head
                                       else self.graph_launches[0 if train else 1])
        with torch.cuda.stream(prep):
            for _ in it:                                      # let the feeder finish its bookkeeping
                pass
        main.wait_stream(sst)

    def _drop_prefetch(self) -> None:
        pre, self._pre = getattr(self, "_pre", None), None
        if pre is not None:
            pre[2].close()
            torch.cuda.current_stream(self.device).wait_stream(self.prep_stream)

    def fit(self, train: BatchFeeder, val: Optional[BatchFeeder], epochs: int,
            early_stopping: Optional[int] = 5, restore_best: bool = True,
            reduce_lr_patience: Optional[int] = 2, reduce_lr_factor: float = 0.3, min_lr: float = 1e-6,
            checkpoint_path: Optional[str] = None,
            on_epoch: Optional[Callable[[int, EpochStats], None]] = None, head_only: bool = False) -> List[EpochStats]:
        """The reference's ``model.fit(train_ds, validation_data=val_ds, callbacks=[checkpoint,
        early, lr_red], epochs=epoch)`` (FLPyfhelin.py:193). With ``fedprox_mu > 0`` the model at entry is the
        proximal anchor of every update; the reported losses stay the data loss. ``head_only``: FedRep's head phase
        (DESIGN.md §10) -- only the personal layers train, with the same Adam state and step counter, and no
        checkpoint, ReduceLROnPlateau or EarlyStopping callback runs."""
        if self.anchor is not None:
            self.anchor.copy_(self.pack.trainable())
        hist: List[EpochStats] = []
        best_loss, best_acc, wait_es, wait_lr = float("inf"), -1.0, 0, 0
        best_weights = None
        B = self.cfg.batch_size
        lr_scale_host = float(self.lr_scale.item())
        nval = val.steps if val is not None else 0
        ts_all, vs_all = self._stat_buffers(train.steps, nval)    # pinned once (cudaHostAlloc is slow)
        for ep in range(epochs):
            self.model.train()
            ts = ts_all[: train.steps]
            has_val = val is not None and val.steps > 0
            again = (train, True) if ep + 1 < epochs else None
            self._run_epoch(train, True, ts, nxt=(val, False) if has_val else again, head=head_only)
            vs = None
            if has_val:
                self.model.eval()
                vs = vs_all[:nval]
                self._run_epoch(val, False, vs, nxt=again)
            if self.cuda:
                torch.cuda.current_stream(self.device).synchronize()
            loss = float(ts[:, 0].mean())
            acc = float(ts[:, 1].sum()) / (train.steps * B)
            vloss = float(vs[:, 0].mean()) if vs is not None else float("nan")
            vacc = float(vs[:, 1].sum()) / (val.steps * B) if vs is not None else float("nan")
            st = EpochStats(loss, acc, vloss, vacc, lr_scale_host)
            hist.append(st)
            if on_epoch:
                on_epoch(ep, st)
            if head_only:
                continue
            # ModelCheckpoint(monitor='accuracy', save_best_only=True)
            if checkpoint_path and acc > best_acc:
                torch.save({"flat": self.pack.flat.detach().cpu(), "epoch": ep, "accuracy": acc}, checkpoint_path)
            best_acc = max(best_acc, acc)
            # ReduceLROnPlateau(monitor='loss') and EarlyStopping(monitor='loss')
            if loss < best_loss:
                best_loss, wait_es, wait_lr = loss, 0, 0
                if early_stopping is not None and restore_best:
                    best_weights = self.pack.flat.clone()
            else:
                wait_es += 1
                wait_lr += 1
                if reduce_lr_patience is not None and wait_lr >= reduce_lr_patience:
                    cur = lr_scale_host * self.cfg.lr
                    new = max(cur * reduce_lr_factor, min_lr)
                    lr_scale_host = new / self.cfg.lr
                    self.lr_scale.fill_(lr_scale_host)
                    wait_lr = 0
                if early_stopping is not None and wait_es >= early_stopping:
                    if restore_best and best_weights is not None:
                        self.pack.flat.copy_(best_weights)
                        if self.engine is not None:
                            self.engine.after_restore()
                    break
        if self.engine is not None:
            self._drop_prefetch()
        return hist

    def _stat_buffers(self, ntrain: int, nval: int):
        cur = getattr(self, "_stats", None)
        if cur is None or cur[0].shape[0] < ntrain or cur[1].shape[0] < max(nval, 1):
            mk = (lambda n: torch.zeros(n, 2, dtype=torch.float32).pin_memory()) if self.cuda else \
                (lambda n: torch.zeros(n, 2, dtype=torch.float32))
            self._stats = (mk(max(ntrain, 1)), mk(max(nval, 1)))
        return self._stats

    def reset_optimizer(self) -> None:
        self.m.zero_(); self.v.zero_(); self.step_t.zero_(); self.lr_scale.fill_(1.0)
        self.pack.grad.zero_()

    def state_dict(self) -> Dict[str, torch.Tensor]:
        sd = {"m": self.m.cpu(), "v": self.v.cpu(), "step": self.step_t.cpu(), "lr_scale": self.lr_scale.cpu()}
        if self.engine is not None:
            sd["prep_count"] = torch.tensor(self.engine.prep_count, dtype=torch.int64)   # augmentation stream position
        return sd

    def load_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        self.m.copy_(sd["m"]); self.v.copy_(sd["v"]); self.step_t.copy_(sd["step"]); self.lr_scale.copy_(sd["lr_scale"])
        if self.engine is not None and "prep_count" in sd:
            self.engine.prep_count = int(sd["prep_count"])

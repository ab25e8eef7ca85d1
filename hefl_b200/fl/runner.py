"""Federated round loop of encrypted FedAvg: M >= 1 clients per rank (``clients_per_rank``, one process per GPU,
DESIGN.md §9); a one-client rank is the M = 1 case of the same round.

One round = what the reference's notebook cell 3 does once (N:233-272):
``train_clients`` (FLPyfhelin.py:179-198) -> ``export_encrypted_clients_weights`` (:242) ->
``aggregate_encrypted_weights`` (:366) -> ``decrypt_import_weights`` (:263), but

* clients are concurrent ranks, not iterations of a loop, and start every round from the same
  global model (true FedAvg; ``compat_sequential_clients`` reproduces quirk Q1 in the
  single-process simulation),
* there is an outer round loop (the reference runs exactly one, Q2),
* the pickle-file "network" and the server loop are replaced by the ciphertext all-reduce,
* averaging is a sum in ciphertext space with 1/K folded into the decode scale; with
  ``fedavg_weighting="samples"`` each client also folds K·n_k/N into its encode scale, so the
  decrypted result is McMahan et al.'s sample-weighted FedAvg.

Roles: every rank holds the public context; the secret key is generated (OS entropy) and kept by
the key-holder rank alone (default rank 0), which owns no chunk of the fused all-reduce, decrypts
the aggregate and broadcasts the averaged plaintext model.
"""
from __future__ import annotations

import contextlib
import hashlib
import json
import math
import os
import secrets
from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from ..config import FLConfig
from ..he.context import CKKSContext, CtBatch
from ..models import ParamPack, create_model
from ..models.cnn import MedCNN, SmallCNN
from ..parallel import LoopbackTransport, make_transport
from ..utils import DeviceTimer, JsonlLogger, StageTimes
from .data import BatchFeeder, SyntheticImageDataset, dirichlet_partition, shard_range, split_train_val
from .explain import _ig_torch, check_gradcam, check_ig, gradcam_torch
from .fedeval import check_fedeval_options, count_len, metrics_from_confusion, metrics_from_counts
from .server_opt import ServerOptimizer, check_server_options, reference_step
from .trainer import LocalTrainer

FEDAVG_WEIGHTINGS = ("uniform", "samples")


def check_client_options(cfg: FLConfig) -> None:
    """Reject out-of-range client placement / sampling settings (they arrive from flags and environment variables)."""
    if not (isinstance(cfg.clients_per_rank, int) and cfg.clients_per_rank >= 1):
        raise ValueError(f"clients_per_rank must be an integer >= 1, got {cfg.clients_per_rank!r}")
    if not 0 < cfg.client_fraction <= 1:
        raise ValueError(f"client_fraction must be in (0, 1], got {cfg.client_fraction}")


def select_clients(cfg: FLConfig, num_clients: int, rnd: int) -> List[int]:
    """The ids that train in round ``rnd``: all of them, or max(1, round(C*K)) drawn without replacement from a
    generator seeded by (seed, round), so every rank computes the same set without communicating."""
    if cfg.client_fraction >= 1:
        return list(range(num_clients))
    count = max(1, round(cfg.client_fraction * num_clients))
    g = torch.Generator().manual_seed((cfg.seed * 1_000_003 + rnd) & 0x7FFFFFFFFFFFFFFF)
    return sorted(torch.randperm(num_clients, generator=g)[:count].tolist())


def check_noniid_options(cfg: FLConfig) -> None:
    """Reject out-of-range non-IID settings (they arrive from flags and environment variables)."""
    if not cfg.dirichlet_alpha >= 0:
        raise ValueError(f"dirichlet_alpha must be >= 0 (0 = IID shards), got {cfg.dirichlet_alpha}")
    if not cfg.fedprox_mu >= 0:
        raise ValueError(f"fedprox_mu must be >= 0 (0 = plain local Adam), got {cfg.fedprox_mu}")
    if cfg.fedavg_weighting not in FEDAVG_WEIGHTINGS:
        raise ValueError(f"fedavg_weighting must be one of {FEDAVG_WEIGHTINGS}, got {cfg.fedavg_weighting!r}")


# the sequential CNNs, whose Dense layers are the tail of the parameter vector (DESIGN.md §10), and how many they have
PERSONAL_MODELS = {"medcnn": len(MedCNN.dense_units) + 1, "cnn2": len(SmallCNN.dense_units) + 1}


def check_personal_options(cfg: FLConfig) -> None:
    """Reject personalisation settings the round cannot honour (they arrive from flags and environment variables)."""
    p, e = cfg.personal_layers, cfg.personal_head_epochs
    if not (isinstance(p, int) and p >= 0):
        raise ValueError(f"personal_layers must be an integer >= 0 (0 = one global model), got {p!r}")
    if not (isinstance(e, int) and e >= 0):
        raise ValueError(f"personal_head_epochs must be an integer >= 0, got {e!r}")
    if e > 0 and p == 0:
        raise ValueError("personal_head_epochs > 0 trains personal layers: it needs personal_layers > 0")
    if p == 0:
        return
    if cfg.model not in PERSONAL_MODELS:
        raise ValueError(f"personal_layers needs one of the sequential CNNs {tuple(PERSONAL_MODELS)}, got model "
                         f"{cfg.model!r} (a ResNet's fc sits between its trainable parameters and BatchNorm statistics)")
    if p > PERSONAL_MODELS[cfg.model]:
        raise ValueError(f"personal_layers must be at most {PERSONAL_MODELS[cfg.model]}, the Dense layers of "
                         f"{cfg.model}, got {p}")
    if cfg.compat_sequential_clients:
        raise ValueError("personal_layers does not combine with compat_sequential_clients")


class FederatedRunner:
    def __init__(self, cfg: FLConfig, rank: int = 0, world: int = 1, group=None,
                 device: Optional[torch.device] = None, samples_per_client: Optional[int] = None, dataset=None,
                 test_dataset=None):
        check_noniid_options(cfg)
        check_fedeval_options(cfg)
        check_server_options(cfg)
        check_client_options(cfg)
        check_personal_options(cfg)
        self.cfg = cfg
        self.rank, self.world, self.group = rank, world, group
        self.device = device or torch.device(cfg.device if torch.cuda.is_available() or cfg.device == "cpu" else "cpu")
        torch.manual_seed(cfg.seed)                     # the reference seeds nothing (Q12)
        self.model = create_model(cfg.model, cfg.in_channels, cfg.num_classes, cfg.image_size).to(self.device)
        self.pack = ParamPack(self.model)
        # personalisation (DESIGN.md §10): flat[:n_shared] is federated, the trailing Dense layers stay with each client;
        # every client starts from head0, the personal layers of the seeded initial model
        self.n_shared = self.pack.dense_tail_start(cfg.personal_layers) if cfg.personal_layers else self.pack.numel
        self.n_personal = self.pack.numel - self.n_shared
        self.head0 = self.pack.flat[self.n_shared:].clone() if self.n_personal else None
        self.trainer = LocalTrainer(self.model, self.pack, cfg, self.device)
        hp = cfg.he_params()
        self.ctx = CKKSContext(hp["n"], prime_bits=hp["prime_bits"], scale_bits=hp["scale_bits"],
                               device=self.device, sec=cfg.sec)
        # Trust model (the reference's roles: the aggregator works with get_pk only, FLPyfhelin.py:370; get_sk is
        # opened in decrypt alone, :284). The key holder generates the pair from OS entropy, keeps sk, and every
        # other rank only ever receives pk. It owns no chunk of the fused all-reduce, so it never loads a peer's
        # un-aggregated ciphertext; it decrypts the aggregate and broadcasts the averaged plaintext model.
        self.key_holder = int(cfg.key_holder) if world > 1 else -1
        if self.key_holder >= world:
            raise ValueError(f"key_holder {self.key_holder} is not a rank of this {world}-client federation")
        self.has_sk = world == 1 or self.key_holder < 0 or rank == self.key_holder
        self._setup_keys()
        self.n_ct = self.ctx.num_ct(self.n_shared, cfg.packing)
        self.ct_numel = self.n_ct * 2 * self.ctx.L * self.ctx.n
        kind = cfg.transport
        if self.device.type == "cpu" and kind == "fused":
            kind = "gloo" if world > 1 else "loopback"
        self.transport = make_transport(kind, self.ctx, self.ct_numel, world=world, group=group,
                                        **({"algo": cfg.allreduce_algo, "timeout_s": cfg.timeout_s,
                                            "no_owner": self.key_holder} if kind == "fused" else {}))
        self._pair_seeds = self._agree_pair_seeds() if (cfg.pairwise_masks and world > 1) else None
        # clients: rank r hosts ids r*M .. r*M+M-1 of a federation of K = world*M; everything a client draws is keyed
        # by its id, so a client trains the same wherever it is placed (DESIGN.md §9)
        M = int(cfg.clients_per_rank)
        self.clients_per_rank, self.num_clients = M, world * M
        self.client_ids = list(range(rank * M, rank * M + M))
        datasets = list(dataset) if isinstance(dataset, (list, tuple)) else [dataset] if dataset is not None else None
        if datasets is not None and len(datasets) != M:
            raise ValueError(f"dataset: {len(datasets)} datasets for {M} clients per rank (one per client, in id order)")
        # data: IID contiguous shard of a synthetic set (FLPyfhelin.py:75-78), 90/10 split (:85)
        # or, with ``dataset`` (e.g. ImageFolderDataset of this client's shard), real images: 10 % validate
        pool = parts = None
        if datasets is None and cfg.dirichlet_alpha > 0:
            # label-skew shard: this client's Dirichlet part of one pooled set of K x per samples (the pool and the
            # partition are the same on every rank); 10 % of the part validates
            per = samples_per_client or (cfg.steps_per_epoch * cfg.batch_size + cfg.val_steps * cfg.batch_size)
            pool = SyntheticImageDataset(self.num_clients * per, cfg.image_size, cfg.in_channels, cfg.num_classes,
                                         seed=cfg.seed, pin=False)
            parts = dirichlet_partition(pool.labels, self.num_clients, cfg.dirichlet_alpha, cfg.seed, cfg.batch_size)
        self.clients: List[Dict] = []
        for i, cid in enumerate(self.client_ids):
            if datasets is not None:
                ds = datasets[i]
                per = len(ds)
                nval = int(per * 0.1)
            elif pool is not None:
                ds = pool.subset(parts[cid])
                per = len(ds)
                nval = int(per * 0.1)
            else:
                per = samples_per_client or (cfg.steps_per_epoch * cfg.batch_size + cfg.val_steps * cfg.batch_size)
                ds = SyntheticImageDataset(per, cfg.image_size, cfg.in_channels, cfg.num_classes, seed=cfg.seed + 17 * cid)
                nval = cfg.val_steps * cfg.batch_size
            counts = torch.bincount(ds.labels[nval:per].long(),
                                    minlength=int(getattr(ds, "classes", cfg.num_classes))).tolist()
            self.clients.append({"id": cid, "dataset": ds, "nval": nval, "per": per, "n_train": per - nval,
                                 "label_counts": counts})
        del pool
        # federated evaluation (DESIGN.md §13): one test set per client, in id order, else its 10 % validation split
        tests = list(test_dataset) if isinstance(test_dataset, (list, tuple)) else \
            [test_dataset] if test_dataset is not None else None
        if tests is not None and len(tests) != M:
            raise ValueError(f"test_dataset: {len(tests)} datasets for {M} clients per rank (one per client, in id order)")
        for c, t in zip(self.clients, tests or [None] * M):
            c["test"] = (t, range(len(t))) if t is not None else (c["dataset"], range(c["nval"]))
        self._fed_feeds: Dict[int, BatchFeeder] = {}
        if cfg.fed_eval_every or tests is not None:
            self._check_fedeval(tests)
        c0 = self.clients[0]
        self.dataset, self.n_train, self.label_counts = c0["dataset"], c0["n_train"], c0["label_counts"]   # n_k
        per, nval = c0["per"], c0["nval"]
        self.train_feed = BatchFeeder(self.dataset, range(nval, per), cfg.batch_size, self.device,
                                      shuffle=True, seed=cfg.seed + c0["id"])
        vc = next((c for c in self.clients if c["nval"]), None)
        self.val_feed = BatchFeeder(vc["dataset"], range(0, vc["nval"]), cfg.batch_size, self.device,
                                    shuffle=True, seed=cfg.seed + vc["id"]) if vc is not None else None
        if M > 1:
            # per-client state that persists across rounds, swapped into the trainer around each client's fit: Adam
            # m / v, step and LR scale in [M, n] device tensors (the captured graphs keep the trainer's buffers),
            # the engine's augmentation position, the feeders' shuffle generators and the torch RNG state. A
            # one-client rank keeps its client's state where it lives: in the trainer, the feeders and the RNG.
            n = self.pack.n_trainable
            self._c_m = torch.empty(M, n, dtype=torch.float32, device=self.device)
            self._c_v = torch.empty(M, n, dtype=torch.float32, device=self.device)
            self._c_step = torch.empty(M, 1, dtype=torch.int64, device=self.device)
            self._c_lr = torch.empty(M, 1, dtype=torch.float32, device=self.device)
            self._c_head = self.head0.repeat(M, 1) if self.n_personal else None
            self._load_clients_state(None)              # every client starts fresh
        self._selected: List[int] = list(range(self.num_clients))
        self._plain_sum: Optional[torch.Tensor] = None
        self._clear_pending()
        self.round = 0
        self.participating = True        # set False to sit a round out (needs cfg.allow_dropouts on every rank); with
                                         # several clients per rank also a list of M flags, one per client
        self._active = None              # K: the round's contributing clients, once the ranks agreed on it
        self._n_total = None             # N = sum of n_k over the round's contributors (sample-weighted FedAvg)
        self.timer = DeviceTimer(self.device)
        self.log = JsonlLogger(cfg.log_jsonl, rank)
        self.global_flat = self.pack.flat.clone()       # x_t: the global model of the round, snapshot by run_round
        # server optimizer (DESIGN.md §8): the state lives with whoever decrypts -- the key holder, or every rank
        # when every rank holds sk (each then applies the same deterministic step)
        self.server_opt = (ServerOptimizer.from_config(cfg, self.pack.n_trainable - self.n_personal, self.device)
                           if cfg.server_opt != "fedavg" and self.has_sk else None)
        self._avg_out = None                  # debug_precision with a server step: the decoded average of the round
        self.history: List[Dict] = []

    # ------------------------------------------------------------------ keys and randomness
    def _setup_keys(self) -> None:
        cfg = self.cfg
        if cfg.deterministic_crypto:
            # bit-reproducible runs (tests, bench.py): everything from the PUBLIC cfg.seed -- never in a deployment
            sk, self.pk = self.ctx.keygen(seed=cfg.seed)
            self.sk = sk if self.has_sk else None
            return
        gen_rank = self.key_holder if self.key_holder >= 0 else 0
        if self.world == 1 or self.rank == gen_rank:
            sk, pk = self.ctx.keygen(seed=secrets.randbits(63))
        else:
            sk = torch.empty(self.ctx.L, self.ctx.n, dtype=torch.int64, device=self.device)
            pk = torch.empty(2, self.ctx.L, self.ctx.n, dtype=torch.int64, device=self.device)
        if self.world > 1:
            dist.broadcast(pk, src=gen_rank, group=self.group)
            if self.key_holder < 0:          # "every client can decrypt" mode: sk is handed out explicitly
                dist.broadcast(sk, src=gen_rank, group=self.group)
        self.pk = pk
        self.sk = sk if self.has_sk else None

    def _encrypt_seed(self, client: Optional[int] = None) -> int:
        """Fresh randomness for every encryption call. Re-running a round (resume, retry) must never reuse
        (u, e0, e1) on different weights, and a seed derived from public values lets anybody strip the mask.
        ``client``: the id whose update is encrypted (the rank's id when it hosts one client)."""
        if self.cfg.deterministic_crypto:
            cid = self.rank if client is None else client
            return (self.cfg.seed * 1_000_003 + self.round * 1009 + cid) & 0x7FFFFFFFFFFFFFFF
        return secrets.randbits(63)

    def _agree_pair_seeds(self):
        """One 63-bit seed per peer. X25519 key agreement over the process group: only the two ends of a
        pair can derive their seed. Returns (seeds, signs) with sign +1 towards higher ranks, -1 towards lower."""
        peers = [j for j in range(self.world) if j != self.rank]
        if self.cfg.deterministic_crypto:
            def ps(i, j):
                h = hashlib.sha256(f"hefl-pair-{self.cfg.seed}-{min(i, j)}-{max(i, j)}".encode()).digest()
                return int.from_bytes(h[:8], "little") >> 1
            seeds = [ps(self.rank, j) for j in peers]
        else:
            from cryptography.hazmat.primitives import serialization
            from cryptography.hazmat.primitives.asymmetric.x25519 import X25519PrivateKey, X25519PublicKey

            priv = X25519PrivateKey.generate()
            pub = priv.public_key().public_bytes(serialization.Encoding.Raw, serialization.PublicFormat.Raw)
            mine = torch.tensor(list(pub), dtype=torch.uint8, device=self.device)
            allp = [torch.empty_like(mine) for _ in range(self.world)]
            dist.all_gather(allp, mine, group=self.group)
            seeds = []
            for j in peers:
                shared = priv.exchange(X25519PublicKey.from_public_bytes(bytes(allp[j].cpu().tolist())))
                seeds.append(int.from_bytes(hashlib.sha256(b"hefl-pair" + shared).digest()[:8], "little") >> 1)
        signs = [1 if j > self.rank else -1 for j in peers]
        return seeds, signs

    def _mask(self, data: torch.Tensor, chunk: int = 0) -> None:
        if self._pair_seeds is None:
            return
        seeds, signs = self._pair_seeds
        self.ctx.ops.pairwise_mask_(data, seeds, signs, (self.round * 4096 + chunk) & 0xFFFFFFFF, self.ctx.L,
                                    self.ctx.logn, self.ctx.consts_cpu)

    # ------------------------------------------------------------------ stages
    def local_train(self, early_stopping: Optional[int] = None, order: Optional[List[int]] = None):
        """Train this rank's clients selected for the round, one after another from the current global model
        (``order``: their local slots, default ascending). Every update but the last is encrypt-accumulated into the
        rank's ciphertext buffer; the last stays installed in ``pack.flat`` for ``encrypt_update`` /
        ``fedavg_pipelined`` to add. Returns a dict local slot -> epoch history."""
        self._selected = select_clients(self.cfg, self.num_clients, self.round)
        chosen = set(self._selected)
        local = [i for i, cid in enumerate(self.client_ids) if cid in chosen]
        order = local if order is None else [i for i in order if i in local]
        swap = self.clients_per_rank > 1
        if swap:
            self.global_flat.copy_(self.pack.flat)
            if self._c_rng is None:
                # every client starts from the RNG state a one-client rank holds when its first step runs: after capture
                self.trainer.prepare()
                self._c_rng = [self._rng_state()] * self.clients_per_rank
        self._clear_pending()
        self._enc_buf = self.transport.buffer(self.ct_numel)
        weighted = self.cfg.fedavg_weighting == "samples"
        self._plain_sum = (torch.zeros(self.n_shared, dtype=torch.float64, device=self.device)
                           if self.cfg.debug_precision else None)
        hists: Dict[int, list] = {}
        for j, i in enumerate(order):
            with self.timer.stage("train"):
                if j:
                    self.pack.load_flat(self.global_flat)
                    if self.trainer.engine is not None:
                        self.trainer.engine.after_restore()
                val = self._swap_in(i) if swap else self.val_feed
                head = (self.trainer.fit(self.train_feed, val, self.cfg.personal_head_epochs, head_only=True)
                        if self.cfg.personal_head_epochs else [])
                hists[i] = head + self.trainer.fit(self.train_feed, val, self.cfg.local_epochs,
                                                   early_stopping=early_stopping)
                if swap:
                    self._swap_out(i)
            if self._plain_sum is not None and self._client_takes_part(i):
                self._plain_sum.add_(self.shared().double(), alpha=self.clients[i]["n_train"] if weighted else 1)
            if j + 1 < len(order):
                with self.timer.stage("encrypt"):
                    self._accumulate(i, self._enc_buf)
        self._last_client = order[-1] if order else None
        return hists

    # ------------------------------------------------------------------ per-client state
    def _rng_state(self):
        return (torch.get_rng_state(), torch.cuda.get_rng_state(self.device) if self.device.type == "cuda" else None)

    def _set_rng_state(self, st) -> None:
        torch.set_rng_state(st[0])
        if st[1] is not None:
            torch.cuda.set_rng_state(st[1], self.device)

    def _swap_in(self, i: int) -> Optional[BatchFeeder]:
        """Install client slot ``i``'s state in the trainer and point the feeders at its shard; returns its
        validation feeder (None when it has no validation samples)."""
        tr, c = self.trainer, self.clients[i]
        tr.m.copy_(self._c_m[i]); tr.v.copy_(self._c_v[i]); tr.step_t.copy_(self._c_step[i]); tr.lr_scale.copy_(self._c_lr[i])
        if tr.engine is not None:
            tr.engine.prep_count = self._c_prep[i]
        if self.n_personal:
            self.pack.flat[self.n_shared:].copy_(self._c_head[i])        # over the global base
        self._set_rng_state(self._c_rng[i])
        self.train_feed.retarget(c["dataset"], range(c["nval"], c["per"]), self._c_gen[i][0])
        if not c["nval"]:
            return None
        self.val_feed.retarget(c["dataset"], range(0, c["nval"]), self._c_gen[i][1])
        return self.val_feed

    def _swap_out(self, i: int) -> None:
        tr = self.trainer
        self._c_m[i].copy_(tr.m); self._c_v[i].copy_(tr.v); self._c_step[i].copy_(tr.step_t); self._c_lr[i].copy_(tr.lr_scale)
        if tr.engine is not None:
            self._c_prep[i] = tr.engine.prep_count
        if self.n_personal:
            self._c_head[i].copy_(self.pack.flat[self.n_shared:])
        self._c_rng[i] = self._rng_state()

    def shared(self) -> torch.Tensor:
        """The federated part of the installed model: all of it, or the base before the personal layers."""
        return self.pack.flat[: self.n_shared]

    def _install_shared(self, vec: torch.Tensor) -> None:
        """Install the new global model (the federated part only: personal layers stay as they are)."""
        self.shared().copy_(vec.to(self.pack.flat.device, torch.float32).reshape(-1)[: self.n_shared])

    @contextlib.contextmanager
    def _client_head(self, client: Optional[int]):
        """Install client slot ``client``'s personal layers for the block and restore the installed ones on exit (None
        or a one-client rank, whose client's layers are the installed ones, swaps nothing)."""
        if client is not None and not 0 <= client < self.clients_per_rank:
            raise ValueError(f"client slot {client} is not one of this rank's {self.clients_per_rank}")
        if client is None or not self.n_personal or self.clients_per_rank == 1:
            yield
            return
        head = self.pack.flat[self.n_shared:]
        saved = head.clone()
        head.copy_(self._c_head[client])
        try:
            yield
        finally:
            head.copy_(saved)

    def _client_takes_part(self, i: int) -> bool:
        p = self.participating
        return bool(p[i] if isinstance(p, (list, tuple)) else p) or not self.cfg.allow_dropouts

    def _accumulate(self, i: int, buf: torch.Tensor) -> None:
        """Encrypt client slot ``i``'s trained model (in ``pack.flat``) with its own seed and FedAvg weight and add
        it into ``buf`` mod q; the first ciphertext of the round overwrites the buffer."""
        self._agree_on_participants()
        if not self._client_takes_part(i):
            return
        self.ctx.encrypt(self.shared(), self.pk, seed=self._encrypt_seed(self.client_ids[i]), packing=self.cfg.packing,
                         out=buf, weight=self.fedavg_weight(i), accumulate=self._enc_count > 0)
        self._enc_count += 1

    def _contributors(self) -> float:
        """K of this round: the number of selected clients that take part (participation mask, SURVEY.md §5.3). A
        rank none of whose clients takes part still joins the collective with an encryption of zeros, so the fused
        kernel and its barriers are unchanged."""
        if self._active is not None:
            return float(self._active)
        return float(self.transport.contributors())

    def _agree_on_participants(self) -> None:
        """K and N of the round, once, before its first encryption: each rank counts its selected clients that take
        part and sums their n_k, and one all-reduce of [count, n_k sum] (float64) over the ranks gives K and the
        total N for sample-weighted FedAvg. Without dropouts or sample weighting no collective runs (every rank knows
        the selection, so K is its size), nor in an in-process loopback federation of several ranks."""
        if self._agreed:
            return
        self._agreed = True
        weighted = self.cfg.fedavg_weighting == "samples"
        chosen = set(self._selected)
        mine = [i for i, cid in enumerate(self.client_ids) if cid in chosen and self._client_takes_part(i)]
        t = [float(len(mine)), float(sum(self.clients[i]["n_train"] for i in mine))]
        reduce = (self.cfg.allow_dropouts or weighted) and self.world > 1 \
            and not isinstance(self.transport, LoopbackTransport)
        if reduce:
            tt = torch.tensor(t, dtype=torch.float64, device=self.device)
            dist.all_reduce(tt, op=dist.ReduceOp.SUM, group=self.group)
            t = tt.tolist()
        if reduce or self.world == 1:
            self._active = int(round(t[0]))
            self._n_total = t[1] if weighted else None
        else:
            self._active, self._n_total = len(self._selected), None

    def _my_samples(self, i: int) -> int:
        """n_k: client slot ``i``'s training samples, 0 when it sits the round out."""
        return self.clients[i]["n_train"] if self._client_takes_part(i) else 0

    def fedavg_weight(self, i: int = 0) -> float:
        """w_k = K·n_k / N of client slot ``i``, folded into the encode scale (1.0 for uniform FedAvg). Σ w_k = K, so
        the aggregate has the magnitude bound of uniform FedAvg; equal shards give exactly 1.0."""
        n = self._my_samples(i)
        if not self._n_total or n == 0:
            return 1.0
        return self._contributors() * n / self._n_total

    def _clear_pending(self) -> None:
        """Start the rank's next ciphertext. A one-client rank's installed model is always its client's update, so it
        stays pending (a caller may load weights and encrypt without ``local_train``); with several clients
        ``local_train`` names the slot whose model is installed."""
        self._enc_buf, self._enc_count, self._agreed = None, 0, False
        self._last_client = 0 if self.clients_per_rank == 1 else None

    def _rank_update(self):
        """Agree on K and N if this round has not yet, and return what completes the rank's ciphertext: (buffer,
        values, weight, seed, accumulate). The values are the installed model of the last trained client, zeros
        under the rank's own seed when none of its clients takes part, or None when the buffer already holds every
        contribution."""
        self._agree_on_participants()
        buf = self._enc_buf if self._enc_buf is not None else self.transport.buffer(self.ct_numel)
        last, acc = self._last_client, self._enc_count > 0
        self._clear_pending()
        if last is not None and self._client_takes_part(last):
            return buf, self.shared(), self.fedavg_weight(last), self._encrypt_seed(self.client_ids[last]), acc
        if acc:
            return buf, None, 1.0, 0, True
        return buf, torch.zeros_like(self.shared()), 1.0, self._encrypt_seed(self.num_clients + self.rank), False

    def _encrypt_chunk(self, update, c0: int, c1: int, ci: int = 0) -> CtBatch:
        """Ciphertexts ``c0 .. c1 - 1`` of the rank's update (``update``: what ``_rank_update`` returned), written
        into the matching view of its buffer and masked with chunk index ``ci``. Each ciphertext draws its
        randomness at its own index (``ct_offset``), so before the mask the words do not depend on the chunking."""
        buf, flat, weight, seed, acc = update
        ctx, vpc = self.ctx, self.ctx.values_per_ct(self.cfg.packing)
        nv = min(self.n_shared, c1 * vpc) - c0 * vpc
        view = buf[c0 * 2 * ctx.L * ctx.n: c1 * 2 * ctx.L * ctx.n]
        if flat is not None:
            ct = ctx.encrypt(flat[c0 * vpc: c0 * vpc + nv], self.pk, seed=seed, packing=self.cfg.packing, out=view,
                             ct_offset=c0, weight=weight, accumulate=acc)
        else:                                # every client of the rank is already in the buffer
            ct = CtBatch(view.view(c1 - c0, 2, ctx.L, ctx.n), ctx.scale, nv, self.cfg.packing)
        self._mask(ct.data, chunk=ci)
        return ct

    def _decode(self, agg: CtBatch, k: float, offset: int = 0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The aggregate of ``k`` clients decoded into global values ``offset .. offset + agg.nvals - 1`` of ``out``: the
        fused server step or the plain average (nothing on a rank without sk). Returns ``out``, or without it a new
        vector of the shared part: for the plain average the decrypt's own result, installed without a copy."""
        if self.server_opt is not None:
            # x_{t+1} = step(x_t, average): decoded and stepped in one launch, broadcast where the average was
            out = torch.empty_like(self.shared()) if out is None else out
            self.server_opt.step(self.ctx, agg, self.sk, k, self.global_flat[: self.n_shared], out, offset=offset,
                                 avg_out=self._avg_out)
        elif self.has_sk:
            avg = self.ctx.decrypt(agg, self.sk, divide_by=k)
            if out is None:
                return avg
            out[offset: offset + avg.numel()].copy_(avg)
        return torch.empty_like(self.shared()) if out is None else out

    def _publish(self, avg: torch.Tensor) -> None:
        """Broadcast the new global model (and ``_avg_out`` when set) from the key holder, install it as the shared
        part on every rank and refresh the engine's weight layouts from it."""
        if self.key_holder >= 0:
            avg = avg.to(self.pack.flat.dtype).contiguous()
            dist.broadcast(avg, src=self.key_holder, group=self.group)
            if self._avg_out is not None:
                dist.broadcast(self._avg_out, src=self.key_holder, group=self.group)
        self._install_shared(avg)
        if self.trainer.engine is not None:
            self.trainer.engine.after_restore()

    def encrypt_update(self) -> CtBatch:
        """The rank's ciphertext of the round: the last trained client added into the buffer its co-located clients
        were accumulated into (an encryption of zeros when none of them takes part), masked once."""
        update = self._rank_update()
        with self.timer.stage("encrypt"):
            return self._encrypt_chunk(update, 0, self.n_ct)

    def aggregate(self, ct: CtBatch) -> CtBatch:
        with self.timer.stage("aggregate"):
            data = self.transport.allreduce(ct.data)
            return CtBatch(data, ct.scale, ct.nvals, ct.packing)

    def decrypt_apply(self, agg: CtBatch) -> None:
        with self.timer.stage("decrypt"):
            k = self._contributors()
            if k == 0:                                       # nobody took part: keep the current global model
                return
            self._publish(self._decode(agg, k))

    # ------------------------------------------------------------------ chunked, overlapped FedAvg
    def fedavg_pipelined(self, chunk_cts: int = 256) -> None:
        """encode+encrypt of chunk i+1, the all-reduce of chunk i and decrypt+decode of chunk i-1 run concurrently on
        three CUDA streams (SURVEY.md §5.7: the scaling axis of this workload is ciphertext volume; ResNet-18 is 1.5 GB
        of ciphertext per client); on the CPU the chunks run in order. Result is identical to the unchunked path:
        chunks are whole ciphertexts and every chunk uses its own seed offset."""
        ctx, dev, n_ct = self.ctx, self.device, self.n_ct
        cuda = dev.type == "cuda"
        vpc = ctx.values_per_ct(self.cfg.packing)
        # the rank's other clients are already in the buffer; the last one is encrypted chunk by chunk into it
        update = self._rank_update()
        k = self._contributors()
        if k == 0:
            return
        out = torch.empty_like(self.shared())
        if self.server_opt is not None:
            self.server_opt.ensure_state()               # on the current stream, before the three streams fork
        s_enc = s_comm = s_dec = cur = None              # torch.cuda.stream(None) leaves the current stream in place
        if cuda:
            # the three streams live as long as the runner: the caching allocator keeps one pool per stream, so
            # fresh streams every round meant fresh cudaMallocs (and cudaFree stalls) every round
            if getattr(self, "_pipe_streams", None) is None:
                self._pipe_streams = tuple(torch.cuda.Stream(dev) for _ in range(3))
            s_enc, s_comm, s_dec = self._pipe_streams
            cur = torch.cuda.current_stream(dev)
            for st in (s_enc, s_comm, s_dec):
                st.wait_stream(cur)
        # The three stages only overlap if they fit on the chip together: encrypt / decrypt are persistent
        # one-CTA-per-SM kernels and the all-reduce is a copy engine that saturates NVLink from a few SMs, so the
        # SMs are partitioned for the duration of the pipeline (encrypt gets what the other two leave).
        split = None
        if self.world > 1 and cuda and self.transport.name == "fused":
            ar, dec = 24, 28 if self.has_sk else 0
            enc = torch.cuda.get_device_properties(dev).multi_processor_count - ar - dec
            if min(enc, ar) >= 2 * ctx.L:
                split = (enc, dec, ar)
                ctx.ops.set_he_cta_limits(0, enc, dec)
                saved_blocks, self.transport.blocks = self.transport.blocks, ar
        timeline = [] if cuda and os.environ.get("HEFL_TIMELINE") else None

        def mark(stream):
            if not cuda:
                return None
            e = torch.cuda.Event(enable_timing=timeline is not None)
            e.record(stream)
            return e

        with self.timer.stage("fedavg_pipelined"):
            t_origin = mark(cur) if timeline is not None else None
            for ci, c0 in enumerate(range(0, n_ct, chunk_cts)):
                rec = {"chunk": ci}
                with torch.cuda.stream(s_enc):
                    if timeline is not None:
                        rec["enc0"] = mark(s_enc)
                    ct = self._encrypt_chunk(update, c0, min(n_ct, c0 + chunk_cts), ci)
                    rec["enc1"] = mark(s_enc)
                with torch.cuda.stream(s_comm):
                    if cuda:
                        s_comm.wait_event(rec["enc1"])
                    if timeline is not None:
                        rec["ar0"] = mark(s_comm)
                    data = self.transport.allreduce(ct.data)
                    rec["ar1"] = mark(s_comm)
                with torch.cuda.stream(s_dec):
                    if cuda:
                        s_dec.wait_event(rec["ar1"])
                    if timeline is not None:
                        rec["dec0"] = mark(s_dec)
                    self._decode(CtBatch(data, ct.scale, ct.nvals, ct.packing), k, offset=c0 * vpc, out=out)
                    if timeline is not None:
                        rec["dec1"] = mark(s_dec)
                if timeline is not None:
                    timeline.append(rec)
            if cuda:
                for st in (s_dec, s_comm, s_enc):
                    cur.wait_stream(st)
            if split is not None:
                ctx.ops.set_he_cta_limits(0, 0, 0)
                self.transport.blocks = saved_blocks
            if timeline is not None:
                torch.cuda.synchronize(dev)
                rows = [{"chunk": r["chunk"], **{k: round(t_origin.elapsed_time(r[k]), 4) for k in r if k != "chunk"}}
                        for r in timeline]
                if self.rank == 0:
                    with open(os.environ["HEFL_TIMELINE"], "w") as f:
                        json.dump({"world": self.world, "n_ct": n_ct, "chunk_cts": chunk_cts, "sm_split_enc_dec_ar": split,
                                   "unit": "ms since the start of the FedAvg stage", "chunks": rows}, f, indent=1)
            self._publish(out)

    def guard_finite(self) -> None:
        """NaN/Inf guard on decoded weights (failure detection, SURVEY.md §5.3)."""
        if not bool(torch.isfinite(self.pack.flat).all()):
            raise FloatingPointError(f"round {self.round}: decrypted weights are not finite")

    # ------------------------------------------------------------------ round
    def run_round(self, check: bool = False, pipelined: Optional[bool] = None) -> Dict:
        self.global_flat.copy_(self.pack.flat)       # x_t of the server step
        hists = self.local_train()
        # plaintext FedAvg oracle (SURVEY.md §5.5 "CKKS precision: max abs error vs plaintext FedAvg"): the ranks'
        # sums of their clients' (n_k-weighted) updates as local_train trained them, over the agreed K or N. An
        # in-process loopback federation of several ranks has no process group to sum them over.
        oracle = self.cfg.debug_precision and (self.world == 1 or not isinstance(self.transport, LoopbackTransport))
        # with a server step the error is the decoded average's, not the stepped model's: the decode also writes it here
        self._avg_out = torch.empty_like(self.shared()) if oracle and self.cfg.server_opt != "fedavg" else None
        if pipelined is None:
            pipelined = self.device.type == "cuda" and self.n_ct > 512 and self.transport.name in ("fused", "nccl", "gloo")
        if pipelined:
            self.fedavg_pipelined()
        else:
            self.decrypt_apply(self.aggregate(self.encrypt_update()))
        fed = None
        if self.cfg.fed_eval_every and (self.round + 1) % self.cfg.fed_eval_every == 0:
            with self.timer.stage("fed_eval"):
                fed = self.evaluate_federated()
        if self.cfg.debug_poison:
            self.poison_buffers()
        times = self.timer.resolve()
        if hasattr(self.transport, "check_status"):
            self.transport.check_status()
        if check:
            self.guard_finite()
        hist = hists.get(0)
        rec = {"round": self.round, "rank": self.rank, "stage_ms": times,
               "loss": hist[-1].loss if hist else None, "accuracy": hist[-1].accuracy if hist else None,
               "transport": self.transport.name, "n_ct": self.n_ct, "ct_bytes": self.ct_numel * 8,
               "n_train": self.n_train, "fedavg_weight": self.fedavg_weight(), "label_counts": self.label_counts,
               "server_opt": self.cfg.server_opt}
        if self.n_personal:                          # the personal model on the client's own held-out 10 %
            rec["val_accuracy"] = hist[-1].val_accuracy if hist else None
        if self.clients_per_rank > 1 or self.cfg.client_fraction < 1:
            rec.update(self._client_records(hists))
        if fed is not None:
            rec["fed_eval"] = fed
        if oracle:
            if self.world > 1:
                dist.all_reduce(self._plain_sum, op=dist.ReduceOp.SUM, group=self.group)
            kk = self._n_total if self._n_total is not None else self._contributors()
            if kk > 0:
                avg = self._avg_out if self._avg_out is not None else self.shared()
                err = float((avg.double() - self._plain_sum / kk).abs().max())
                rec["ckks_max_abs_err"] = err
                rec["ckks_precision_bits"] = float(-math.log2(err)) if err > 0 else float("inf")
        self.history.append(rec)
        self.round += 1
        return rec

    def _client_records(self, hists: Dict[int, list]) -> Dict:
        """Round-record fields of a rank with several clients or client sampling: loss / accuracy as the sample-weighted
        mean over its trained clients, n_train / fedavg_weight / label_counts summed over those that took part, the
        round's selection, and per client."""
        clients, n_sum, w_sum = [], 0, 0.0
        counts = [0] * len(self.label_counts)
        for i in sorted(hists):
            c, h = self.clients[i], hists[i]
            w = self.fedavg_weight(i) if self._client_takes_part(i) else 0.0
            clients.append({"id": c["id"], "n_train": c["n_train"], "fedavg_weight": w,
                            "loss": h[-1].loss if h else None, "accuracy": h[-1].accuracy if h else None,
                            "label_counts": c["label_counts"]})
            if self.n_personal:
                clients[-1]["val_accuracy"] = h[-1].val_accuracy if h else None
            if self._client_takes_part(i):
                n_sum, w_sum = n_sum + c["n_train"], w_sum + w
                counts = [a + b for a, b in zip(counts, c["label_counts"])]
        scored = [(c["n_train"], c) for c in clients if c["loss"] is not None]
        tot = sum(n for n, _ in scored)
        personal = {"val_accuracy": sum(n * c["val_accuracy"] for n, c in scored) / tot if tot else None} \
            if self.n_personal else {}
        return {**personal,"loss": sum(n * c["loss"] for n, c in scored) / tot if tot else None,
                "accuracy": sum(n * c["accuracy"] for n, c in scored) / tot if tot else None,
                "n_train": n_sum, "fedavg_weight": w_sum, "label_counts": counts,
                "selected": list(self._selected), "clients": clients}

    POISON = 0x7FF8DEADBEEF7FF8          # > every q_l: a stale word can never pass for a residue

    def poison_buffers(self) -> None:
        """Debug mode (``debug_poison`` / HEFL_DEBUG_POISON=1, SURVEY.md §5.2): after the round's result is
        installed, every buffer that carried ciphertext words is overwritten, so a later round that reads
        something it did not write this round (stale tile, missed barrier) decodes to garbage and trips
        ``guard_finite`` / the plaintext cross-check instead of silently reusing last round's data."""
        buf = self.transport.buffer(self.ct_numel)
        buf.fill_(self.POISON)
        out = getattr(self.transport, "out", None)
        if isinstance(out, torch.Tensor):
            out.fill_(self.POISON)
        self.poisoned = getattr(self, "poisoned", 0) + 1

    def run(self, rounds: Optional[int] = None) -> List[Dict]:
        out = []
        for _ in range(rounds or self.cfg.rounds):
            rec = self.run_round(check=True)
            rec["stage_ms_max"] = StageTimes.max_over_ranks(rec["stage_ms"], self.device, self.group)
            self.log.write(rec)
            out.append(rec)
        return out

    # ------------------------------------------------------------------ evaluation (notebook N:262-270)
    @torch.no_grad()
    def evaluate(self, dataset, batch_size: Optional[int] = None, client: Optional[int] = None) -> Dict[str, float]:
        """Weighted precision / recall / F1 and accuracy of the current global model on ``dataset`` — the four
        numbers the reference's notebook reports after aggregation (sklearn ``average='weighted'``, N:267-270).
        Runs the plain PyTorch forward of the model (any backend / device); not a hot path. ``client``: a local slot
        whose personal layers are installed for the evaluation (the installed ones are restored afterwards); None
        scores the installed model."""
        with self._client_head(client):
            bs = batch_size or self.cfg.batch_size
            self.model.eval()
            preds = []
            for i in range(0, len(dataset), bs):
                x = dataset.images[i:i + bs].to(self.device, non_blocking=True)
                x = x.permute(0, 3, 1, 2).float() * (1.0 / 255.0)
                preds.append(self.model(x).float().argmax(1).cpu())
            self.model.train()
        return classification_metrics(dataset.labels.cpu(), torch.cat(preds), int(getattr(dataset, "classes", self.cfg.num_classes)))

    def explain(self, images_u8: torch.Tensor, stage: int = 4, target=None, client: Optional[int] = None,
                batch_size: Optional[int] = None):
        """Grad-CAM of the installed model (DESIGN.md §11): ``(probs [N, C], cams [N, S, S])``, both fp32 on the CPU,
        for uint8 NHWC scans ``images_u8`` [N, S, S, in_channels]. ``cams`` are the maps of the class score at conv
        stage ``stage`` (1..n), upsampled to S x S and scaled to [0, 1]. ``target``: None (each scan's predicted
        class), an int, or N class indices (-1 = predicted). ``client``: as in ``evaluate``. Runs on the hand-written
        engine in input slot 0 when the trainer has one (in batches of its fixed batch size, the last one padded;
        ``batch_size`` is not used there), else ``gradcam_torch`` in batches of ``batch_size``. Not to be called
        while ``fit`` runs; the weights, optimiser state, augmentation position and RNG are left as they were."""
        with self._client_head(client):
            N = int(images_u8.shape[0])
            targets = check_gradcam(self.model, stage, target, N)
            self._check_images(images_u8)
            cfg = self.cfg
            S, C = cfg.image_size, self.model.num_classes
            probs = torch.empty(N, C, dtype=torch.float32)
            cams = torch.empty(N, S, S, dtype=torch.float32)
            eng = self.trainer.engine
            if eng is None:
                bs = batch_size or cfg.batch_size
                for i in range(0, N, bs):
                    p, c = gradcam_torch(self.model, images_u8[i:i + bs], stage, targets[i:i + bs])
                    probs[i:i + bs], cams[i:i + bs] = p.float().cpu(), c.float().cpu()
                return probs, cams
            B, dev = eng.B, self.device
            x = torch.zeros(B, S, S, cfg.in_channels, dtype=torch.uint8, device=dev)
            tgt = torch.full((B,), -1, dtype=torch.int64, device=dev)
            logits = torch.zeros(B, C, dtype=torch.float32, device=dev)
            cam = torch.zeros(B, S, S, dtype=torch.float32, device=dev)
            for i in range(0, N, B):
                nv = min(B, N - i)
                if nv < B:                                   # padding rows: explained, never written back
                    x.zero_()
                    tgt.fill_(-1)
                x[:nv].copy_(images_u8[i:i + nv])
                tgt[:nv].copy_(targets[i:i + nv])
                eng.preprocess(x, 0, False, False)
                eng.gradcam_staged(0, stage, tgt, logits, cam, nv)
                probs[i:i + nv] = torch.softmax(logits[:nv].cpu(), dim=1)
                cams[i:i + nv] = cam[:nv].cpu()
            return probs, cams

    # ------------------------------------------------------------------ federated evaluation (DESIGN.md §13)
    def _check_fedeval(self, tests=None) -> None:
        first = self.clients[0]["dataset"]
        check_fedeval_options(self.cfg, self.model.num_classes, self.n_ct * self.ctx.values_per_ct(self.cfg.packing),
                              tests if tests is not None else [c["test"][0] for c in self.clients],
                              getattr(first, "class_indices", None))

    def _eval_seed(self, cid: int) -> int:
        """Encryption randomness of client ``cid``'s count vector: never the seed of its model update."""
        if self.cfg.deterministic_crypto:
            h = hashlib.sha256(f"hefl-fedeval-{self.cfg.seed}-{self.round}-{cid}".encode()).digest()
            return int.from_bytes(h[:8], "little") >> 1
        return secrets.randbits(63)

    def _fed_feed(self, i: int) -> Optional[BatchFeeder]:
        ds, idx = self.clients[i]["test"]
        if len(idx) == 0:
            return None
        if i not in self._fed_feeds:
            self._fed_feeds[i] = BatchFeeder(ds, idx, self.cfg.batch_size, self.device, shuffle=False)
        return self._fed_feeds[i]

    @torch.no_grad()
    def evaluate_federated(self) -> Dict:
        """Federated evaluation of the deployed models (DESIGN.md §13); a collective that every rank must call. Every
        local client, selected this round or not, scores the global model with its own personal layers on its test
        set (``test_dataset``, else its 10 % validation split). Each client's count vector is encrypted with its own
        seed and accumulated into a prefix of the rank's ciphertext buffer (weight 1: counts are sums), masked at
        stream index round*4096 + 4095, all-reduced, decrypted by the key holder (or every rank holding sk) and
        broadcast as float64. Returns ``metrics_from_counts`` of the sum, and under ``"local"`` this rank's clients'
        plaintext metrics, which never leave the rank. Raises FloatingPointError if a decoded count is negative or
        more than 0.25 from an integer. The global model, the server optimizer and the training state are untouched."""
        self._check_fedeval()
        cfg, ctx, dev = self.cfg, self.ctx, self.device
        C, nb = self.model.num_classes, cfg.fed_eval_bins
        V = count_len(C, nb)
        rows = torch.zeros(self.clients_per_rank, V, dtype=torch.float64, device=dev)
        for i in range(self.clients_per_rank):
            feed = self._fed_feed(i)
            if feed is not None:
                with self._client_head(i):
                    self.trainer.score(feed, rows[i])
        n1 = ctx.num_ct(V, cfg.packing)
        view = self.transport.buffer(self.ct_numel)[: n1 * 2 * ctx.L * ctx.n]
        for i in range(self.clients_per_rank):        # an empty client adds an encryption of zeros
            ct = ctx.encrypt(rows[i].float(), self.pk, seed=self._eval_seed(self.client_ids[i]), packing=cfg.packing,
                             out=view, accumulate=i > 0)
        self._mask(ct.data, chunk=4095)
        data = self.transport.allreduce(ct.data)
        vec = torch.empty(V, dtype=torch.float64, device=dev)
        if self.has_sk:
            vec.copy_(ctx.decrypt(CtBatch(data, ct.scale, V, cfg.packing), self.sk, divide_by=1.0).double())
        if self.key_holder >= 0:
            dist.broadcast(vec, src=self.key_holder, group=self.group)
        vec = vec.cpu()
        counts = vec[:-1].round()
        if bool(((vec[:-1] - counts).abs() > 0.25).any()) or bool((counts < 0).any()):
            raise FloatingPointError(f"round {self.round}: decoded evaluation counts are not non-negative integers "
                                     f"(largest distance {float((vec[:-1] - counts).abs().max()):.3g})")
        out = metrics_from_counts(torch.cat([counts, vec[-1:]]), C, nb)
        out["local"] = [{"id": cid, **metrics_from_counts(rows[i].cpu(), C, nb)} for i, cid in enumerate(self.client_ids)]
        return out

    def _check_images(self, images_u8: torch.Tensor) -> None:
        S, ch = self.cfg.image_size, self.cfg.in_channels
        if tuple(images_u8.shape[1:]) != (S, S, ch) or images_u8.dtype != torch.uint8:
            raise ValueError(f"images must be uint8 [N, {S}, {S}, {ch}], got {tuple(images_u8.shape)} "
                             f"{images_u8.dtype}")

    def attribute(self, images_u8: torch.Tensor, steps: int = 32, target=None, client: Optional[int] = None,
                  batch_size: Optional[int] = None):
        """Integrated Gradients of the installed model (DESIGN.md §12): ``(probs [N, C], attr [N, S, S], gap [N])``,
        all fp32 on the CPU, for uint8 NHWC scans ``images_u8`` [N, S, S, in_channels]. ``attr`` is the pixel-level
        attribution of the class score against the black image, summed over the input channels, with ``steps``
        (1..1024) midpoint-rule path points; ``gap`` is its completeness error, sum(attr) - (score - black score).
        ``target``: None (each scan's predicted class), an int, or N class indices (-1 = predicted). ``client`` and
        ``batch_size``: as in ``explain``; the engine uses input slots 0 and 1. Not to be called while ``fit`` runs;
        the weights, optimiser state, augmentation position and RNG are left as they were."""
        return self._attribute(images_u8, steps, target, client, batch_size)[:3]

    def _attribute(self, images_u8, steps, target, client, batch_size=None):
        """``attribute``'s results followed by the resolved targets, the scores and the black image's scores (int64
        and fp32 [N], CPU)."""
        with self._client_head(client):
            N = int(images_u8.shape[0])
            targets = check_ig(self.model, steps, target, N)
            self._check_images(images_u8)
            cfg = self.cfg
            S, C = cfg.image_size, self.model.num_classes
            probs = torch.empty(N, C, dtype=torch.float32)
            attr = torch.empty(N, S, S, dtype=torch.float32)
            tres = torch.empty(N, dtype=torch.int64)
            score = torch.empty(N, dtype=torch.float32)
            base = torch.empty(N, dtype=torch.float32)
            eng = self.trainer.engine
            if eng is None:
                bs = batch_size or cfg.batch_size
                for i in range(0, N, bs):
                    r = _ig_torch(self.model, images_u8[i:i + bs], steps, targets[i:i + bs])
                    for dst, v in zip((probs, attr, score, base, tres), r):
                        dst[i:i + bs] = v.detach().to("cpu", dst.dtype)
            else:
                B, dev = eng.B, self.device
                x = torch.zeros(B, S, S, cfg.in_channels, dtype=torch.uint8, device=dev)
                tgt = torch.full((B,), -1, dtype=torch.int64, device=dev)
                logits = torch.zeros(B, C, dtype=torch.float32, device=dev)
                blog = torch.zeros(B, C, dtype=torch.float32, device=dev)
                att = torch.zeros(B, S, S, dtype=torch.float32, device=dev)
                for i in range(0, N, B):
                    nv = min(B, N - i)
                    if nv < B:                                   # padding rows: attributed, never written back
                        x.zero_()
                        tgt.fill_(-1)
                    x[:nv].copy_(images_u8[i:i + nv])
                    tgt[:nv].copy_(targets[i:i + nv])
                    eng.preprocess(x, 1, False, False)
                    t = eng.ig_staged(steps, tgt, logits, blog, att, nv)[:nv, None]
                    probs[i:i + nv] = torch.softmax(logits[:nv].cpu(), dim=1)
                    attr[i:i + nv] = att[:nv].cpu()
                    tres[i:i + nv] = t[:, 0].cpu()
                    score[i:i + nv] = logits[:nv].gather(1, t)[:, 0].cpu()
                    base[i:i + nv] = blog[:nv].gather(1, t)[:, 0].cpu()
            gap = (attr.double().sum((1, 2)) - (score.double() - base.double())).float()
            return probs, attr, gap, tres, score, base

    # ------------------------------------------------------------------ checkpoint / resume
    def save_checkpoint(self, path: str) -> None:
        """Round index + global model (rank 0 -> ``path``) and, PER RANK, optimiser moments, LR state, RNG, the
        feeders' shuffle generators and, with several clients per rank, every client's state (``path.rank{r}``) so
        that a resumed multi-round run equals an uninterrupted one (SURVEY.md §5.4)."""
        if self.rank == 0:
            flat = self.pack.flat.detach().cpu()
            if self.n_personal:                      # the global file holds no client's personal layers
                flat = torch.cat([flat[: self.n_shared], self.head0.cpu()])
            torch.save({"round": self.round, "flat": flat, "config": self.cfg.to_json()}, path)
        torch.save({"round": self.round, "opt": self.trainer.state_dict(), "rng": torch.get_rng_state(),
                    "cuda_rng": torch.cuda.get_rng_state(self.device) if self.device.type == "cuda" else None,
                    "feeds": [f.gen.get_state() if f is not None else None for f in (self.train_feed, self.val_feed)],
                    "server": self.server_opt.state_dict() if self.server_opt is not None else None,
                    "clients": self._clients_state() if self.clients_per_rank > 1 else None,
                    "heads": {"ids": torch.tensor(self.client_ids), "head": self._heads().cpu()} if self.n_personal else None},
                   f"{path}.rank{self.rank}")

    def _heads(self) -> torch.Tensor:
        """[M, n_personal]: every client's personal layers (a one-client rank's are the installed ones)."""
        return self._c_head if self.clients_per_rank > 1 else self.pack.flat[self.n_shared:].unsqueeze(0)

    def _load_heads(self, st: Optional[Dict]) -> None:
        """The clients' personal layers from a rank file, or head0 for every client when it holds none of them."""
        if not self.n_personal:
            return
        mine = st is not None and st["ids"].tolist() == self.client_ids
        heads = st["head"].to(self.device) if mine else self.head0.expand(self.clients_per_rank, -1)
        self._heads().copy_(heads)

    def _clients_state(self) -> Dict:
        """Every client's persistent state (several clients per rank): optimiser, augmentation position, shuffle
        generators and RNG."""
        rng = self._c_rng
        return {"ids": torch.tensor(self.client_ids), "m": self._c_m.cpu(), "v": self._c_v.cpu(),
                "step": self._c_step.cpu(), "lr_scale": self._c_lr.cpu(), "prep_count": torch.tensor(self._c_prep),
                "gen": [[g.get_state() for g in pair] for pair in self._c_gen],
                "rng": [r[0] for r in rng] if rng is not None else None,
                "cuda_rng": [r[1] for r in rng] if rng is not None and rng[0][1] is not None else None}

    def _load_clients_state(self, st: Optional[Dict]) -> None:
        M = self.clients_per_rank
        if st is None or st["ids"].tolist() != self.client_ids:          # no state of these clients: start fresh
            self._c_m.zero_(); self._c_v.zero_(); self._c_step.zero_(); self._c_lr.fill_(1.0)
            self._c_prep = [0] * M
            self._c_gen = [(torch.Generator().manual_seed(self.cfg.seed + cid),
                            torch.Generator().manual_seed(self.cfg.seed + cid)) for cid in self.client_ids]
            self._c_rng = None
            return
        self._c_m.copy_(st["m"]); self._c_v.copy_(st["v"]); self._c_step.copy_(st["step"]); self._c_lr.copy_(st["lr_scale"])
        self._c_prep = [int(x) for x in st["prep_count"]]
        for pair, states in zip(self._c_gen, st["gen"]):
            for g, gs in zip(pair, states):
                g.set_state(gs)
        if st["rng"] is None:
            self._c_rng = None
        else:
            cuda = st["cuda_rng"] if self.device.type == "cuda" else None
            self._c_rng = [(st["rng"][i], cuda[i] if cuda is not None else None) for i in range(M)]
            self.trainer.prepare()         # the states were taken after capture: capture now, not inside a fit

    def load_checkpoint(self, path: str) -> None:
        ck = torch.load(path, map_location="cpu", weights_only=True)      # tensors and plain containers only
        self.round = int(ck["round"])
        self.pack.load_flat(ck["flat"])
        mine = f"{path}.rank{self.rank}"
        if os.path.exists(mine):
            st = torch.load(mine, map_location="cpu", weights_only=True)
            self.trainer.load_state_dict(st["opt"])
            if int(st["opt"]["step"]) > 0:
                self.trainer.prepare()     # the RNG state was taken after capture: capture now, not inside a fit
            torch.set_rng_state(st["rng"])
            if st.get("cuda_rng") is not None and self.device.type == "cuda":
                torch.cuda.set_rng_state(st["cuda_rng"], self.device)
            for f, gs in zip((self.train_feed, self.val_feed), st.get("feeds") or ()):
                if f is not None and gs is not None:
                    f.gen.set_state(gs)
            if self.clients_per_rank > 1:
                self._load_clients_state(st.get("clients"))
            self._load_heads(st.get("heads"))
            if self.server_opt is not None:          # the server state sits in the key holder's own file
                if st.get("server") is not None:
                    self.server_opt.load_state_dict(st["server"])
                else:
                    self.server_opt.reset()
        else:                                       # no state of this rank (e.g. a different world size): start it fresh
            self.trainer.reset_optimizer()
            if self.clients_per_rank > 1:
                self._load_clients_state(None)
            self._load_heads(None)
            if self.server_opt is not None:
                self.server_opt.reset()
        if self.trainer.engine is not None:
            self.trainer.engine.after_restore()


def classification_metrics(y_true: torch.Tensor, y_pred: torch.Tensor, num_classes: int) -> Dict[str, float]:
    """precision / recall / f1 (support-weighted, zero where undefined — sklearn's ``average='weighted',
    zero_division=0``) and accuracy."""
    y_true, y_pred = y_true.long().flatten(), y_pred.long().flatten()
    n = max(1, y_true.numel())
    num_classes = max(num_classes, int(max(y_true.max(), y_pred.max())) + 1) if y_true.numel() else num_classes
    conf = torch.bincount(y_true * num_classes + y_pred, minlength=num_classes * num_classes)
    return metrics_from_confusion(conf.view(num_classes, num_classes).tolist(), n)


def simulate_clients(cfg: FLConfig, device: Optional[torch.device] = None, rounds: int = 1,
                     drop_client: Optional[int] = None) -> Dict:
    """Single-process simulation of ``cfg.clients`` clients through the loopback transport — the
    reference's own structure (clients = loop iterations, FLPyfhelin.py:184) and our fake
    backend for tests. Returns the encrypted-FedAvg result and the plaintext FedAvg oracle. With
    ``dirichlet_alpha > 0`` the clients hold Dirichlet label-skew parts of the pool; with
    ``fedavg_weighting="samples"`` client k is weighted by n_k / N in both. With a ``server_opt`` other than
    fedavg the fused decode steps the global model along the average: ``global`` is the new model and
    ``global_oracle`` the float64 step (``server_opt.reference_step``) of the plaintext average from the same x_t;
    ``encrypted_avg`` / ``plain_avg`` / ``max_abs_err`` keep describing the average."""
    check_noniid_options(cfg)
    check_server_options(cfg)
    if cfg.personal_layers or cfg.personal_head_epochs:
        raise ValueError("simulate_clients averages one global model: personal_layers / personal_head_epochs need "
                         "FederatedRunner")
    device = device or torch.device("cpu")
    torch.manual_seed(cfg.seed)
    hp = cfg.he_params()
    ctx = CKKSContext(hp["n"], prime_bits=hp["prime_bits"], scale_bits=hp["scale_bits"], device=device,
                      sec=cfg.sec)
    sk, pk = ctx.keygen(seed=cfg.seed)
    model = create_model(cfg.model, cfg.in_channels, cfg.num_classes, cfg.image_size).to(device)
    pack = ParamPack(model)
    trainer = LocalTrainer(model, pack, cfg, device, backend="cudnn", use_graph=False)
    K = cfg.clients
    total = K * (cfg.steps_per_epoch + cfg.val_steps) * cfg.batch_size
    ds = SyntheticImageDataset(total, cfg.image_size, cfg.in_channels, cfg.num_classes, seed=cfg.seed, pin=False)
    if cfg.dirichlet_alpha > 0:
        splits = []
        for part in dirichlet_partition(ds.labels, K, cfg.dirichlet_alpha, cfg.seed, cfg.batch_size):
            nval = int(len(part) * 0.1)
            splits.append((part[nval:].tolist(), part[:nval].tolist()))
    else:
        splits = [split_train_val(*shard_range(total, i, K)) for i in range(K)]
    kept_ids = [i for i in range(K) if not (drop_client is not None and i == drop_client)]
    n_k = [len(splits[i][0]) for i in range(K)]
    n_total = sum(n_k[i] for i in kept_ids)
    weights = [len(kept_ids) * n_k[i] / n_total if cfg.fedavg_weighting == "samples" else 1.0 for i in range(K)]
    lb = LoopbackTransport(ctx, K)
    global_flat = pack.flat.clone()
    sopt = ServerOptimizer.from_config(cfg, pack.n_trainable, device) if cfg.server_opt != "fedavg" else None
    if sopt is not None:
        ref_m = torch.zeros(pack.n_trainable, dtype=torch.float64, device=device)
        ref_v = torch.full((pack.n_trainable,), sopt.hp["tau"] ** 2, dtype=torch.float64, device=device)
    result = {}
    for rnd in range(rounds):
        lb.reset()
        plain = []
        for i in range(K):
            if not cfg.compat_sequential_clients:
                pack.load_flat(global_flat)          # true FedAvg: same starting point
                trainer.reset_optimizer()
            tr, va = splits[i]
            tf = BatchFeeder(ds, tr, cfg.batch_size, device, seed=cfg.seed + i)
            vf = BatchFeeder(ds, va, cfg.batch_size, device, seed=cfg.seed + i) if len(va) else None
            trainer.fit(tf, vf, cfg.local_epochs)
            plain.append(pack.flat.clone())
            ct = ctx.encrypt(pack.flat, pk, seed=cfg.seed * 7919 + rnd * 131 + i, packing=cfg.packing,
                             weight=weights[i])
            if drop_client is not None and i == drop_client:
                lb.drop(i)
            else:
                lb.contribute(i, ct.data)
        agg = CtBatch(lb.reduce(), ctx.scale, pack.numel, cfg.packing)
        k = lb.contributors()
        if sopt is None:
            avg = ctx.decrypt(agg, sk, divide_by=float(k))
        else:
            avg = torch.empty_like(global_flat)
            new = torch.empty_like(global_flat)
            sopt.step(ctx, agg, sk, float(k), global_flat, new, avg_out=avg)
        if cfg.fedavg_weighting == "samples":
            oracle = (sum(n_k[i] * plain[i].double() for i in kept_ids) / n_total).float()
        else:
            oracle = torch.stack([plain[i] for i in kept_ids]).mean(0)
        step_info = {}
        if sopt is not None:
            # the oracle of the step: float64, on the plaintext average, from the same x_t
            g_oracle = reference_step(cfg.server_opt, sopt.hp, global_flat, oracle, ref_m, ref_v, pack.n_trainable)
            step_info = {"global": new, "global_oracle": g_oracle}
            global_flat = new.clone()
        else:
            global_flat = avg.clone()
        pack.load_flat(global_flat)
        result = {"encrypted_avg": avg, "plain_avg": oracle, "contributors": k, "n_train": n_k,
                  "fedavg_weights": weights, "max_abs_err": float((avg - oracle).abs().max()), **step_info}
    result["model"] = model
    result["pack"] = pack
    result["ctx"] = ctx
    return result

"""Data pipeline (SURVEY.md L0; FLPyfhelin.py:38-114).

* ``prep_df`` scans ``folder/<label>/<file>`` exactly like the reference (:38-55).
* ``SyntheticImageDataset`` stands in for the medical image folders (no dataset offline):
  uint8 NHWC images in pinned host memory with a label-dependent pattern so that training
  has signal.
* ``shard_range`` is the reference's IID contiguous shard (:75-78, remainder dropped, Q9);
  ``split_train_val`` is Keras' ``validation_split=0.1`` (:85 — the first 10 % validate);
  ``dirichlet_partition`` gives non-IID label-skew shards of unequal size instead.
* ``BatchFeeder`` streams batches host->device from pinned memory on a copy stream
  (double-buffered), which is what the end-to-end benchmark times.
"""
from __future__ import annotations

import os
from typing import Iterator, List, Optional, Tuple

import numpy as np
import torch


def prep_df(folder: str, shuffle: bool = True, seed: Optional[int] = None):
    """DataFrame ['Path','Label'] of absolute paths, optionally shuffled (FLPyfhelin.py:38-55)."""
    import pandas as pd

    rows = []
    for sub in os.scandir(folder):
        if sub.is_dir():
            for name in sorted(os.listdir(sub.path)):
                rows.append([os.path.join(os.path.abspath(sub.path), name), sub.name])
    df = pd.DataFrame(rows, columns=["Path", "Label"])
    if shuffle:
        df = df.sample(frac=1, random_state=seed).reset_index(drop=True)
    return df


def shard_range(total: int, index: int, num_client: int) -> Tuple[int, int]:
    ratio = int(total / num_client)
    start = index * ratio
    return start, start + ratio


def split_train_val(start: int, end: int, val_frac: float = 0.1) -> Tuple[range, range]:
    n = end - start
    nval = int(n * val_frac)
    return range(start + nval, end), range(start, start + nval)


def dirichlet_partition(labels, num_clients: int, alpha: float, seed: int, min_train: int = 1,
                        val_frac: float = 0.1, max_draws: int = 100) -> List[torch.Tensor]:
    """Label-skew shards: for every class, its indices are permuted and split among the clients at the cut
    points of proportions drawn from Dirichlet(alpha, ..., alpha). Small alpha gives each client a few dominant
    classes and unequal sizes; large alpha approaches the pool's class mix. Every client must keep at least
    ``min_train`` training samples after the ``val_frac`` validation split; otherwise the whole partition is
    drawn again with ``seed + attempt``. The result depends only on (labels, num_clients, alpha, seed), so every
    rank computes the same partition without communication. Returns one sorted int64 index tensor per client."""
    if alpha <= 0:
        raise ValueError(f"dirichlet_alpha must be > 0 for a label-skew partition, got {alpha}")
    labels = np.asarray(labels.cpu() if isinstance(labels, torch.Tensor) else labels).reshape(-1)
    sizes: List[int] = []
    for attempt in range(max_draws):
        rng = np.random.default_rng(seed + attempt)
        parts: List[List[np.ndarray]] = [[] for _ in range(num_clients)]
        for c in np.unique(labels):
            idx = rng.permutation(np.flatnonzero(labels == c))
            cuts = (np.cumsum(rng.dirichlet([alpha] * num_clients))[:-1] * len(idx)).astype(np.int64)
            for k, piece in enumerate(np.split(idx, cuts)):
                parts[k].append(piece)
        out = [np.sort(np.concatenate(p)) for p in parts]
        sizes = [len(o) for o in out]
        if all(n - int(n * val_frac) >= min_train for n in sizes):
            return [torch.from_numpy(o.astype(np.int64)) for o in out]
    raise ValueError(f"dirichlet_partition: no draw of {max_draws} gave every one of {num_clients} clients "
                     f"{min_train} training samples (alpha={alpha}, {len(labels)} samples; last client sizes "
                     f"{sizes}); raise alpha or the pool size, or lower the client count")


class SyntheticImageDataset:
    """``n`` uint8 images [n, H, W, C] (pinned when CUDA is present) and int64 labels."""

    def __init__(self, n: int, image_size: int = 256, channels: int = 3, classes: int = 2,
                 seed: int = 0, pin: Optional[bool] = None):
        g = torch.Generator().manual_seed(seed)
        self.labels = torch.randint(0, classes, (n,), generator=g)
        base = torch.randint(0, 160, (n, image_size, image_size, channels), generator=g, dtype=torch.uint8)
        # class signal: a bright square whose position depends on the label
        q = max(2, image_size // 4)
        for c in range(classes):
            idx = (self.labels == c).nonzero().flatten()
            if idx.numel() == 0:
                continue
            r0 = (c * q) % max(1, image_size - q)
            base[idx, r0:r0 + q, r0:r0 + q, :] += 90
        self.images = base
        pin = torch.cuda.is_available() if pin is None else pin
        if pin:
            self.images = self.images.pin_memory()
            self.labels = self.labels.pin_memory()
        self.n = n
        self.classes = classes

    def subset(self, idx: torch.Tensor, pin: Optional[bool] = None) -> "SyntheticImageDataset":
        """A dataset of rows ``idx`` of this one (a client's shard of a pooled set)."""
        out = object.__new__(SyntheticImageDataset)
        out.images, out.labels = self.images[idx], self.labels[idx]
        if torch.cuda.is_available() if pin is None else pin:
            out.images, out.labels = out.images.pin_memory(), out.labels.pin_memory()
        out.n, out.classes = len(idx), self.classes
        return out

    def __len__(self) -> int:
        return self.n


class ImageFolderDataset:
    """The reference's image folders (``folder/<label>/<file>``, FLPyfhelin.py:38-55) for the product path:
    this client's IID contiguous shard (:75-78) is decoded once (PIL, bilinear resize to the model's input
    size, :104; a thread pool decodes in parallel) into pinned uint8 NHWC memory, from where ``BatchFeeder``
    streams it to the GPU. Same attributes as ``SyntheticImageDataset``. Class indices come from the sorted
    label names of the WHOLE folder, so every client agrees on them. ``dirichlet_alpha > 0`` replaces the
    contiguous shard by client ``index``'s part of a ``dirichlet_partition`` of the whole shuffled folder's labels
    (each part keeps at least ``min_train`` training images); only that part is decoded."""

    def __init__(self, folder: str, image_size: int = 256, channels: int = 3, index: int = 0, num_clients: int = 1,
                 shuffle_seed: Optional[int] = 0, workers: int = 8, pin: Optional[bool] = None,
                 stream: bool = False, dirichlet_alpha: float = 0.0, min_train: int = 1):
        from concurrent.futures import ThreadPoolExecutor

        df = prep_df(folder, shuffle=shuffle_seed is not None, seed=shuffle_seed)
        if len(df) == 0:
            raise FileNotFoundError(f"no images under {folder}/<label>/")
        names = sorted(set(df["Label"]))
        self.class_indices = {l: i for i, l in enumerate(names)}
        if dirichlet_alpha > 0:
            all_labels = np.array([self.class_indices[l] for l in df["Label"]], dtype=np.int64)
            part = dirichlet_partition(all_labels, num_clients, dirichlet_alpha, shuffle_seed or 0, min_train)[index]
            rows = df.iloc[part.numpy()]
        else:
            lo, hi = shard_range(len(df), index, num_clients)
            rows = df.iloc[lo:hi]
        self.filenames = list(rows["Path"])
        n = len(self.filenames)
        self.image_size, self.channels = image_size, channels
        labels = torch.tensor([self.class_indices[l] for l in rows["Label"]], dtype=torch.int64)
        pin = torch.cuda.is_available() if pin is None else pin
        self.n = n
        self.classes = len(names)
        self.stream = bool(stream)
        if self.stream:
            # flow_from_dataframe semantics (FLPyfhelin.py:88-112): nothing is decoded up front, every batch is
            # decoded when it is asked for (``load_batch``), so the shard need not fit in host memory
            self._pool = ThreadPoolExecutor(max_workers=max(1, workers))
            self.images = None
            self.image_shape = (image_size, image_size, channels)
            self.labels = labels.pin_memory() if pin else labels
            return
        imgs = torch.zeros(n, image_size, image_size, channels, dtype=torch.uint8)

        def load(i: int) -> None:
            imgs[i] = torch.from_numpy(np.ascontiguousarray(_decode(self.filenames[i], image_size, channels)))

        with ThreadPoolExecutor(max_workers=max(1, workers)) as ex:
            list(ex.map(load, range(n)))
        self.images = imgs.pin_memory() if pin else imgs
        self.image_shape = tuple(imgs.shape[1:])
        self.labels = labels.pin_memory() if pin else labels

    def load_batch(self, sel: torch.Tensor, out: torch.Tensor) -> None:
        """Decode the images ``sel`` (indices into this shard) into ``out`` [len(sel), H, W, C] uint8 (pinned
        staging memory of the feeder) on the thread pool."""
        idx = [int(i) for i in sel]

        def load(k: int) -> None:
            out[k] = torch.from_numpy(np.ascontiguousarray(_decode(self.filenames[idx[k]], self.image_size, self.channels)))

        if getattr(self, "_pool", None) is not None:
            list(self._pool.map(load, range(len(idx))))
        else:
            for k in range(len(idx)):
                load(k)

    def __len__(self) -> int:
        return self.n


def _decode(path: str, size: int, channels: int) -> np.ndarray:
    """uint8 [size, size, channels] from an image file (or a .npy array), bilinear resize."""
    if path.endswith(".npy"):
        arr = np.load(path)
        if arr.ndim == 2:
            arr = arr[:, :, None]
        if arr.shape[0] != size or arr.shape[1] != size:
            t = torch.from_numpy(arr).permute(2, 0, 1)[None].float()
            t = torch.nn.functional.interpolate(t, size=(size, size), mode="bilinear", align_corners=False)
            arr = t[0].permute(1, 2, 0).round().clamp(0, 255).to(torch.uint8).numpy()
    else:
        from PIL import Image

        img = Image.open(path).convert("RGB" if channels == 3 else "L").resize((size, size), Image.BILINEAR)
        arr = np.asarray(img)
        if arr.ndim == 2:
            arr = arr[:, :, None]
    if arr.shape[2] != channels:
        arr = arr[:, :, :1].repeat(channels, axis=2) if arr.shape[2] == 1 else arr[:, :, :channels]
    return arr.astype(np.uint8)


class BatchFeeder:
    """Fixed-size batches over an index range. On CUDA every step's images go host->device
    straight from the pinned dataset (one async copy per row, issued by the native
    ``gather_h2d_`` op on a copy stream) while the previous batch computes."""

    def __init__(self, ds: SyntheticImageDataset, indices: range, batch_size: int, device: torch.device,
                 shuffle: bool = True, seed: int = 0, drop_last: bool = False):
        from .. import _ext

        self.ops = _ext.ops()
        self.ds = ds
        self.indices = torch.tensor(list(indices), dtype=torch.int64)
        self.bs = batch_size
        self.device = device
        self.shuffle = shuffle
        self.gen = torch.Generator().manual_seed(seed)
        self.cuda = device.type == "cuda"
        self.copy_stream = torch.cuda.Stream(device) if self.cuda else None
        n = len(self.indices)
        self.steps = n // batch_size if drop_last else (n + batch_size - 1) // batch_size
        self.streaming = getattr(ds, "images", None) is None      # decode-per-batch dataset (ImageFolderDataset(stream=True))
        img_shape = tuple(ds.image_shape) if self.streaming else tuple(ds.images.shape[1:])
        shp = (batch_size, *img_shape)
        self._stage_x = ([torch.empty(shp, dtype=torch.uint8).pin_memory() if self.cuda else torch.empty(shp, dtype=torch.uint8)
                          for _ in range(2)] if self.streaming else None)
        self._pending = [False, False]      # slot has an H2D copy in flight that still reads its pinned staging
        self._stage_y = [torch.empty(batch_size, dtype=torch.int64).pin_memory() if self.cuda
                         else torch.empty(batch_size, dtype=torch.int64) for _ in range(2)]
        self._dev_x = [torch.empty(shp, dtype=torch.uint8, device=device) for _ in range(2)]
        self._dev_y = [torch.empty(batch_size, dtype=torch.int64, device=device) for _ in range(2)]
        self._ready = [torch.cuda.Event() if self.cuda else None for _ in range(2)]
        self._consumed = [torch.cuda.Event() if self.cuda else None for _ in range(2)]
        self.bytes_per_step = int(np.prod(shp)) + batch_size * 8
        self.drop_last = drop_last

    def retarget(self, ds, indices, gen: torch.Generator) -> None:
        """Serve another client of the rank: its dataset, index set and shuffle generator, through the same
        pinned staging buffers, device slots and copy stream (pinned memory is slow to allocate and finite)."""
        shape = tuple(ds.image_shape) if getattr(ds, "images", None) is None else tuple(ds.images.shape[1:])
        if shape != tuple(self._dev_x[0].shape[1:]) or (getattr(ds, "images", None) is None) != self.streaming:
            raise ValueError(f"retarget: every client of a rank needs images of one shape, got {shape}")
        self.ds = ds
        self.indices = torch.tensor(list(indices), dtype=torch.int64)
        n = len(self.indices)
        self.steps = n // self.bs if self.drop_last else (n + self.bs - 1) // self.bs
        self.gen = gen

    def _order(self) -> torch.Tensor:
        if self.shuffle:
            return self.indices[torch.randperm(len(self.indices), generator=self.gen)]
        return self.indices

    def _issue(self, order: torch.Tensor, step: int, slot: int) -> None:
        n = len(order)
        sel = order[(torch.arange(self.bs) + step * self.bs) % n]  # wrap the last partial batch
        if not self.cuda:
            if self.streaming:
                self.ds.load_batch(sel, self._stage_x[slot])
                self._dev_x[slot].copy_(self._stage_x[slot])
            else:
                self._dev_x[slot].copy_(self.ds.images[sel])
            self._dev_y[slot].copy_(self.ds.labels[sel])
            return
        if self._pending[slot]:
            # the previous copy out of this slot's pinned staging (possibly issued by the PREVIOUS epoch) must
            # have completed before the host rewrites it
            self._ready[slot].synchronize()
            self._pending[slot] = False
        torch.index_select(self.ds.labels, 0, sel, out=self._stage_y[slot])
        if self.streaming:
            self.ds.load_batch(sel, self._stage_x[slot])     # host decode of batch i+1 overlaps the GPU on batch i
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(self._consumed[slot])
            if self.streaming:
                self._dev_x[slot].copy_(self._stage_x[slot], non_blocking=True)
            else:
                self.ops.gather_h2d_(self._dev_x[slot], self.ds.images, sel)
            self._dev_y[slot].copy_(self._stage_y[slot], non_blocking=True)
            self._ready[slot].record(self.copy_stream)
        self._pending[slot] = True

    def epoch(self) -> Iterator[Tuple[torch.Tensor, torch.Tensor]]:
        """Yields device tensors (uint8 NHWC images, int64 labels); batch i+1 copies while i computes."""
        order = self._order()
        if self.cuda:
            cur = torch.cuda.current_stream(self.device)
            for ev in self._consumed:
                ev.record(cur)
        self._issue(order, 0, 0)
        for step in range(self.steps):
            slot = step & 1
            if step + 1 < self.steps:
                self._issue(order, step + 1, 1 - slot)
            if self.cuda:
                torch.cuda.current_stream(self.device).wait_event(self._ready[slot])
            yield self._dev_x[slot], self._dev_y[slot]
            if self.cuda:
                self._consumed[slot].record(torch.cuda.current_stream(self.device))


def augment_batch(x: torch.Tensor, gen: Optional[torch.Generator], shear: float = 0.2, zoom: float = 0.2,
                  hflip: bool = True) -> torch.Tensor:
    """Keras ImageDataGenerator(shear_range, zoom_range, horizontal_flip) on the device
    (FLPyfhelin.py:80-86). ``x`` is float [B,C,H,W]; one random affine per sample."""
    import math

    B = x.shape[0]
    dev = x.device
    r = torch.rand(B, 4, generator=gen, device=dev)
    sh = (r[:, 0] * 2 - 1) * shear * (math.pi / 180.0)   # Keras shear_range is in degrees
    zx = 1.0 + (r[:, 1] * 2 - 1) * zoom
    zy = 1.0 + (r[:, 2] * 2 - 1) * zoom
    flip = torch.where(r[:, 3] < 0.5, -1.0, 1.0) if hflip else torch.ones(B, device=dev)
    theta = torch.zeros(B, 2, 3, device=dev, dtype=x.dtype)
    theta[:, 0, 0] = (zx * flip).to(x.dtype)
    theta[:, 0, 1] = (-torch.sin(sh) * zx).to(x.dtype)
    theta[:, 1, 1] = (torch.cos(sh) * zy).to(x.dtype)
    grid = torch.nn.functional.affine_grid(theta, list(x.shape), align_corners=False)
    return torch.nn.functional.grid_sample(x, grid, mode="bilinear", padding_mode="border", align_corners=False)


class ResidentFeeder:
    """Device-resident variant of ``BatchFeeder`` (the whole shard lives in HBM; batches are
    gathered on the device). Used for the device-only timing pass of bench.py; the shard
    (>= 126 MB for the reference shape) is larger than L2, so no batch is served from cache."""

    def __init__(self, ds: SyntheticImageDataset, indices: range, batch_size: int, device: torch.device,
                 shuffle: bool = True, seed: int = 0):
        idx = torch.tensor(list(indices), dtype=torch.int64)
        self.images = ds.images[idx].to(device)
        self.labels = ds.labels[idx].to(device)
        self.bs = batch_size
        self.device = device
        self.shuffle = shuffle
        self.gen = torch.Generator(device=device).manual_seed(seed) if device.type == "cuda" else torch.Generator().manual_seed(seed)
        n = len(idx)
        self.n = n
        self.steps = (n + batch_size - 1) // batch_size
        self.bytes_per_step = 0

    def epoch(self):
        n = self.n
        order = torch.randperm(n, generator=self.gen, device=self.device) if self.shuffle else torch.arange(n, device=self.device)
        ar = torch.arange(self.bs, device=self.device)
        for step in range(self.steps):
            sel = order[(ar + step * self.bs) % n]
            yield self.images[sel], self.labels[sel]

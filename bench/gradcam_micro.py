"""Grad-CAM (DESIGN.md §11): what the gradcam kernel, the engine's explain step and the PyTorch path cost.

1. The gradcam kernel alone at each stage's shape of the medical CNN (batch 32, 256 x 256): the HBM bytes it must
   move (G and X[s] read once, the S x S fp32 maps written once) computed from the shapes, its median time over 20
   launches with L2 flushed before each, and the rate reached.
2. MedCNNEngine.gradcam_staged on a full batch at stages 2, 4 and 6, with its native launch count.
3. The same batch through gradcam_torch (fp32, cuDNN) on the same card, alternated with 2.

Weights are the engine's own after a few training steps on the synthetic set.

    python bench/gradcam_micro.py [--in-channels 3|1] [--out result.json]
    python bench/gradcam_micro.py --bytes-only          # the shape and byte table, no GPU needed

Prints one JSON object with the card's name, power limit and max SM clock beside the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

B, S = 32, 256
CONV = (32, 32, 32, 64, 64, 128)
LAUNCHES = 20


def stage_shapes():
    """(stage, Hp, C) of the medical CNN at S x S."""
    rows, h = [], S
    for s, c in enumerate(CONV, 1):
        h = (h - 2) // 2
        rows.append((s, h, c))
    return rows


def kernel_bytes(Hp, C):
    """HBM bytes the gradcam kernel must move: G and X[s] (bf16) read once, the fp32 maps written once."""
    read = 2 * B * Hp * Hp * C * 2
    write = B * S * S * 4
    return read, write


def median_ms(fn, flush):
    import torch

    ts = []
    for _ in range(LAUNCHES):
        flush()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--in-channels", type=int, default=3, choices=(1, 3))
    ap.add_argument("--train-steps", type=int, default=3)
    ap.add_argument("--bytes-only", action="store_true", help="print the shape and byte table and exit")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    table = []
    for s, Hp, C in stage_shapes():
        rd, wr = kernel_bytes(Hp, C)
        table.append({"stage": s, "Hp": Hp, "C": C, "read_bytes": rd, "write_bytes": wr})
    if args.bytes_only:
        print(json.dumps({"batch": B, "image": S, "gradcam_kernel": table}))
        return
    import copy

    import torch

    from hefl_b200 import _ext
    from hefl_b200.config import FLConfig
    from hefl_b200.fl.data import SyntheticImageDataset
    from hefl_b200.fl.explain import gradcam_torch
    from hefl_b200.fl.trainer import LocalTrainer
    from hefl_b200.models import ParamPack, create_model
    from multiclient_micro import card

    if not torch.cuda.is_available():
        raise SystemExit("gradcam_micro.py needs a CUDA device")
    ops, dev, ch = _ext.ops(), torch.device("cuda"), args.in_channels
    torch.manual_seed(0)
    model = create_model("medcnn", ch, 2, S).to(dev)
    pack = ParamPack(model)
    tr = LocalTrainer(model, pack, FLConfig(model="medcnn", in_channels=ch), dev)
    ds = SyntheticImageDataset(B * (args.train_steps + 1), S, ch, 2, seed=1, pin=False)
    for i in range(args.train_steps):
        tr.train_step(ds.images[i * B:(i + 1) * B].to(dev), ds.labels[i * B:(i + 1) * B].to(dev))
    torch.cuda.synchronize()
    eng = tr.engine
    x = ds.images[-B:].to(dev).contiguous()
    scrub = torch.ones(64 << 20, dtype=torch.float32, device=dev)       # 256 MB > the 50 MB L2

    def flush():                        # a read, so that no dirty line of the flush is written back under the kernel
        scrub.sum()

    # 1. the kernel alone, on the engine's own X[s] and a gradient-shaped bf16 G
    eng.preprocess(x, 0, False, False)
    eng.forward_convs(0, False)
    cam = torch.empty(B, S, S, dtype=torch.float32, device=dev)
    g = torch.Generator(device="cuda").manual_seed(2)
    for row in table:
        s, Hp, C = row["stage"], row["Hp"], row["C"]
        G = (torch.randn(B * Hp * Hp, C, device=dev, generator=g) * 1e-3).to(torch.bfloat16)
        ms = median_ms(lambda: ops.gradcam(eng.X[s], G, cam, B, Hp, C, S, B), flush)
        row.update(ms=ms, tb_per_s=(row["read_bytes"] + row["write_bytes"]) / (ms * 1e-3) / 1e12)
    # 2 / 3. the explain step on the engine against gradcam_torch in fp32 on cuDNN, alternated
    torch.backends.cudnn.benchmark = True
    ref = copy.deepcopy(model).float()
    tgt = torch.full((B,), -1, dtype=torch.int64, device=dev)
    logits = torch.empty(B, 2, dtype=torch.float32, device=dev)
    steps = []
    for s in (2, 4, 6):
        def engine():
            eng.preprocess(x, 0, False, False)
            eng.gradcam_staged(0, s, tgt, logits, cam, B)

        def torch_path():
            gradcam_torch(ref, x, s)

        engine(); torch_path()
        torch.cuda.synchronize()
        n0 = int(ops.launch_count())
        engine()
        torch.cuda.synchronize()
        launches = int(ops.launch_count()) - n0
        e_ms, t_ms = [], []
        for _ in range(3):
            e_ms.append(median_ms(engine, flush))
            t_ms.append(median_ms(torch_path, flush))
        steps.append({"stage": s, "engine_ms": statistics.median(e_ms), "engine_native_launches": launches,
                      "gradcam_torch_fp32_ms": statistics.median(t_ms)})
    res = {"card": card(), "batch": B, "image": S, "in_channels": ch, "gradcam_kernel": table, "explain_step": steps}
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

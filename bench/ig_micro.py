"""Integrated Gradients (DESIGN.md §12): what the input_grad0 kernel, one path point and ``attribute`` cost.

1. The input_grad0 kernel alone at batch 32, 256 x 256, RGB and grayscale: the HBM bytes it must move (the pooled
   gradient and the codes read once, the fp32 accumulator read and written once) computed from the shapes, its median
   time over 20 launches with L2 flushed before each, and the share of the 3.35 TB/s data-sheet bandwidth reached.
2. One path point of MedCNNEngine.ig_staged (scale, forward with codes, seeded head, dgrad chain, input_grad0) as the
   difference of ig_staged at m = 9 and m = 1 over 8, with the native launches per path point.
3. FederatedRunner.attribute for 32 scans at m = 32 against integrated_gradients_torch (fp32, cuDNN) on the same
   card, alternated.

Weights are the engine's own after a few training steps on the synthetic set.

    python bench/ig_micro.py [--out result.json]
    python bench/ig_micro.py --bytes-only          # the byte table, no GPU needed

Prints one JSON object with the card's name, power limit and max SM clock, read in the same run, beside the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

B, S, CO = 32, 256, 32
LAUNCHES = 20
HBM_TBS = 3.35            # H100 SXM data sheet


def kernel_bytes(ci):
    """HBM bytes input_grad0 must move: g (bf16) and codes (u8) of layer 1's pooled output read once, the fp32
    [B, S, S, ci] accumulator read and written once."""
    Hp = (S - 2) // 2
    g = B * Hp * Hp * CO * 2
    codes = B * Hp * Hp * CO
    acc = B * S * S * ci * 4
    return {"in_channels": ci, "g_bytes": g, "code_bytes": codes, "acc_bytes_rw": 2 * acc, "bytes": g + codes + 2 * acc}


def median_ms(fn, flush, n=LAUNCHES):
    import torch

    ts = []
    for _ in range(n):
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
    ap.add_argument("--train-steps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=32, help="path points of the attribute comparison")
    ap.add_argument("--bytes-only", action="store_true", help="print the byte table and exit")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    table = [kernel_bytes(ci) for ci in (3, 1)]
    if args.bytes_only:
        print(json.dumps({"batch": B, "image": S, "input_grad0": table}))
        return
    import copy

    import torch

    from hefl_b200 import _ext
    from hefl_b200.config import FLConfig
    from hefl_b200.fl import FederatedRunner
    from hefl_b200.fl.data import SyntheticImageDataset
    from hefl_b200.fl.explain import integrated_gradients_torch
    from multiclient_micro import card

    if not torch.cuda.is_available():
        raise SystemExit("ig_micro.py needs a CUDA device")
    ops, dev = _ext.ops(), torch.device("cuda")
    scrub = torch.ones(64 << 20, dtype=torch.float32, device=dev)       # 256 MB > the 50 MB L2

    def flush():                        # a read, so that no dirty line of the flush is written back under the kernel
        scrub.sum()

    # 1. the kernel alone on gradient-shaped inputs
    g = torch.Generator(device="cuda").manual_seed(2)
    Hp = (S - 2) // 2
    grad = (torch.randn(B * Hp * Hp, CO, device=dev, generator=g) * 1e-3).to(torch.bfloat16)
    code = torch.randint(0, 8, (B * Hp * Hp, CO), device=dev, generator=g, dtype=torch.uint8)
    for row in table:
        ci = row["in_channels"]
        w = (torch.randn(CO * ci * 9, device=dev, generator=g) * 0.1).to(torch.bfloat16)
        acc = torch.zeros(B, S, S, ci, device=dev)
        ms = median_ms(lambda: ops.input_grad0(grad, code, w, acc, B, S, ci, B), flush)
        row.update(us=ms * 1e3, tb_per_s=row["bytes"] / (ms * 1e-3) / 1e12)
        row["share_of_hbm"] = row["tb_per_s"] / HBM_TBS

    # 2 / 3. on the engine of a trained runner
    torch.manual_seed(0)
    run = FederatedRunner(FLConfig(model="medcnn", local_epochs=1, steps_per_epoch=2, val_steps=1), device=dev)
    ds = SyntheticImageDataset(B * (args.train_steps + 1), S, 3, 2, seed=1, pin=False)
    for i in range(args.train_steps):
        run.trainer.train_step(ds.images[i * B:(i + 1) * B].to(dev), ds.labels[i * B:(i + 1) * B].to(dev))
    torch.cuda.synchronize()
    eng = run.trainer.engine
    x = ds.images[-B:]
    xd = x.to(dev)
    tgt = torch.full((B,), -1, dtype=torch.int64, device=dev)
    logits, base = (torch.empty(B, 2, device=dev) for _ in range(2))
    attr = torch.empty(B, S, S, device=dev)

    def ig(m):
        eng.preprocess(xd, 1, False, False)
        eng.ig_staged(m, tgt, logits, base, attr, B)

    ig(1); ig(9)
    torch.cuda.synchronize()
    n0 = int(ops.launch_count())
    ig(1)
    torch.cuda.synchronize()
    n1 = int(ops.launch_count())
    ig(9)
    torch.cuda.synchronize()
    per_point_launches = (int(ops.launch_count()) - n1 - (n1 - n0)) // 8
    t1, t9 = [], []
    for _ in range(3):
        t1.append(median_ms(lambda: ig(1), flush, 10))
        t9.append(median_ms(lambda: ig(9), flush, 10))
    point = {"ms": (statistics.median(t9) - statistics.median(t1)) / 8, "native_launches": per_point_launches,
             "ig_staged_m1_ms": statistics.median(t1), "ig_staged_m9_ms": statistics.median(t9)}

    torch.backends.cudnn.benchmark = True
    ref = copy.deepcopy(run.model).float()
    m = args.steps

    def engine():
        run.attribute(x, steps=m)

    def torch_path():
        integrated_gradients_torch(ref, x, m)

    engine(); torch_path()
    torch.cuda.synchronize()
    e_ms, t_ms = [], []
    for _ in range(3):
        e_ms.append(median_ms(engine, flush, 3))
        t_ms.append(median_ms(torch_path, flush, 3))
    res = {"card": card(), "batch": B, "image": S, "input_grad0": table, "path_point": point,
           "attribute": {"scans": B, "steps": m, "engine_ms": statistics.median(e_ms),
                         "integrated_gradients_torch_fp32_ms": statistics.median(t_ms)}}
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

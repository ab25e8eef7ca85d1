"""Personalised federated learning (DESIGN.md §10): what a head-only step and a smaller ciphertext cost.

1. LocalTrainer.train_step against the head-only step, both graph-replayed, of the medical CNN on the tcgen05 engine
   (batch 32, 256 x 256) for personal_layers = 1, 2, 3.
2. head_forward_backward at every backward depth (0 eval, 1 full, 2 / 3 / 4 head-only) on the medical CNN's head.
3. The encrypt and decrypt stages of the round at 109 ciphertexts (the whole model) and at the ciphertext counts of
   the shared base (109, 105, 73 for personal_layers 1, 2, 3; n = 4096, L = 3, slot packing).

    python bench/personal_micro.py [--out result.json] [--iters 50]

Prints one JSON object with the card's name and power limit beside the numbers. Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from multiclient_micro import card, timed  # noqa: E402


def steps(iters):
    import torch

    from hefl_b200.config import FLConfig
    from hefl_b200.fl.trainer import LocalTrainer
    from hefl_b200.models import ParamPack, create_model

    dev = torch.device("cuda")
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randint(0, 256, (32, 256, 256, 3), device="cuda", generator=g, dtype=torch.int64).to(torch.uint8)
    y = torch.randint(0, 2, (32,), device="cuda", generator=g)
    rows = []
    for p in (1, 2, 3):
        torch.manual_seed(0)
        model = create_model("medcnn", 3, 2, 256).to(dev)
        pack = ParamPack(model)
        tr = LocalTrainer(model, pack, FLConfig(model="medcnn", personal_layers=p, personal_head_epochs=1), dev)
        rows.append({"personal_layers": p, "train_step_ms": timed(lambda: tr.train_step(x, y), iters),
                     "head_step_ms": timed(lambda: tr.head_step(x, y), iters),
                     "launches_per_step": {"train": tr.graph_launches[0], "head": tr.head_launches}})
    return rows, tr


def depths(tr, iters):
    import torch

    eng, pack = tr.engine, tr.pack
    y = torch.zeros(eng.B, dtype=torch.int64, device="cuda")
    out = torch.zeros(2, device="cuda")
    feat = eng.X[eng.n]
    return {str(d): timed(lambda: tr.ops.head_forward_backward(feat, pack.flat, pack.grad, eng.head_offs, y, eng.dfeat,
                                                                 eng.h1_buf, eng.dh1_buf, out, eng.B, eng.F, eng.H1,
                                                                 eng.H2, eng.C, d), iters)
            for d in range(5)}


def he_stages(iters):
    import torch

    from hefl_b200.he.context import CKKSContext
    from hefl_b200.models import ParamPack, create_model

    pack = ParamPack(create_model("medcnn", 3, 2, 256))
    ctx = CKKSContext(4096, prime_bits=(36, 36, 37), scale_bits=40, device="cuda")
    sk, pk = ctx.keygen(seed=1)
    rows = []
    for p in (0, 1, 2, 3):
        n = pack.dense_tail_start(p) if p else pack.numel
        vals = torch.randn(n, device="cuda") * 0.05
        ct = ctx.encrypt(vals, pk, seed=2)
        rows.append({"personal_layers": p, "values": n, "ciphertexts": ctx.num_ct(n),
                     "encrypt_ms": timed(lambda: ctx.encrypt(vals, pk, seed=2), iters),
                     "decrypt_ms": timed(lambda: ctx.decrypt(ct, sk, divide_by=8.0), iters)})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("personal_micro.py needs a CUDA device")
    step_rows, tr = steps(args.iters)
    res = {"card": card(), "steps_batch32_256px": step_rows, "head_forward_backward_ms_by_depth": depths(tr, args.iters),
           "he_stages": he_stages(args.iters)}
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

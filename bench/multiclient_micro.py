"""Several federated clients per GPU: what the rank's ciphertext sum costs, and what a round costs per client.

1. encrypt-accumulate (ct = ct + Enc(m) mod q in the encryption's store) against encrypt into a fresh buffer
   followed by local_sum_modq, at the medical CNN's shape (n = 4096, L = 3, C = 109) and ResNet-18's (n = 8192,
   L = 4, C = 2857), with the ciphertext bytes each moves beyond the encryption itself.
2. One-GPU round time of the medical CNN (tcgen05 engine, batch 32, 256 x 256, CUDA graphs) with M = 1, 2, 4, 8
   clients, and the per-client switch (global-model load + weight relayout + optimiser/RNG state copies) timed
   apart from training.

    python bench/multiclient_micro.py [--out result.json] [--local-epochs 1] [--iters 20]

Prints one JSON object with the card's name and power limit beside the numbers. Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    import torch

    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [v.strip() for v in q.split(",")]
    except Exception as e:                   # the numbers stay usable; the missing field says why
        info["power_limit"] = f"unknown ({type(e).__name__})"
    return info


def timed(fn, iters):
    import torch

    fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def accumulate_vs_sum(iters):
    import torch

    from hefl_b200.he.context import CKKSContext

    rows = []
    for n, bits, C in ((4096, (36, 36, 37), 109), (8192, (54, 54, 54, 55), 2857)):
        ctx = CKKSContext(n, prime_bits=bits, scale_bits=40, device="cuda")
        _, pk = ctx.keygen(seed=1)
        ops, L = ctx.ops, ctx.L
        msg = torch.randint(-2**30, 2**30, (C, n), dtype=torch.int64, device="cuda")
        acc = ops.encrypt(msg, pk, C, L, ctx.logn, ctx.tables, ctx.consts, None, 3, 0)
        tmp, out = torch.empty_like(acc), torch.empty_like(acc)
        words = acc.numel()

        def fused():
            ops.encrypt_out(msg, pk, C, L, ctx.logn, ctx.tables, ctx.consts, None, 5, 0, acc, True)

        def separate():
            ops.encrypt_out(msg, pk, C, L, ctx.logn, ctx.tables, ctx.consts, None, 5, 0, tmp)
            ops.local_sum_modq([acc, tmp], out, L, ctx.logn, ctx.consts)

        def plain():
            ops.encrypt_out(msg, pk, C, L, ctx.logn, ctx.tables, ctx.consts, None, 5, 0, tmp)

        t_plain, t_fused, t_sep = [], [], []
        for _ in range(3):                    # alternate the arms: the host is shared
            t_plain.append(timed(plain, iters))
            t_fused.append(timed(fused, iters))
            t_sep.append(timed(separate, iters))
        rows.append({"n": n, "L": L, "C": C, "ct_bytes": words * 8,
                     "encrypt_ms": min(t_plain), "encrypt_accumulate_ms": min(t_fused),
                     "encrypt_then_local_sum_ms": min(t_sep),
                     # beyond the encryption's own store: one read of the accumulator, against a read of the
                     # fresh ciphertext and of the accumulator and a store of the sum (plus a fresh buffer)
                     "extra_bytes_accumulate": words * 8, "extra_bytes_separate": 3 * words * 8,
                     "extra_buffer_bytes_separate": words * 8})
        del acc, tmp, out, msg
        torch.cuda.empty_cache()
    return rows


def rounds(local_epochs, counts):
    import torch

    from hefl_b200.config import FLConfig
    from hefl_b200.fl import FederatedRunner

    rows = []
    for M in counts:
        cfg = FLConfig(model="medcnn", local_epochs=local_epochs, nn_backend="tcgen05", device="cuda",
                       transport="fused", deterministic_crypto=True, clients_per_rank=M)
        run = FederatedRunner(cfg, device=torch.device("cuda"))
        run.run_round(check=True)                            # capture, algorithm warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rec = run.run_round(check=True)
        torch.cuda.synchronize()
        row = {"clients_per_rank": M, "round_ms": (time.perf_counter() - t0) * 1e3,
               "stage_ms": rec["stage_ms"], "loss": rec["loss"]}
        if M > 1:
            def switch():
                for i in range(M):
                    run.pack.load_flat(run.global_flat)
                    run.trainer.engine.after_restore()
                    run._swap_in(i)
                    run._swap_out(i)
            row["switch_ms_per_client"] = timed(switch, 5) / M
        rows.append(row)
        del run
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--local-epochs", type=int, default=1)
    ap.add_argument("--clients", default="1,2,4,8")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        print(json.dumps({"error": "multiclient_micro.py needs a CUDA device"}))
        return 1
    res = {"card": card(), "encrypt_accumulate": accumulate_vs_sum(args.iters),
           "medcnn_round": {"local_epochs": args.local_epochs,
                            "rows": rounds(args.local_epochs, [int(v) for v in args.clients.split(",")])}}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())

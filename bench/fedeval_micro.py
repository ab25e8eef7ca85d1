"""Federated evaluation (DESIGN.md §13): what scoring and the count ciphertext cost.

1. head_logits (the 8-CTA cluster head, forward only) and score_stats alone at batch 32, C = 2, 100 bins: median of
   20 launches with L2 flushed before each.
2. A 1,024-scan pass of LocalTrainer.score (graph-replayed, pipelined, 256 x 256 RGB) against FederatedRunner.evaluate's
   PyTorch forward on the same scans, alternated three times.
3. Encrypt + all-reduce + decrypt of one rank's count ciphertext (V = 405 values, one ciphertext at n4096_l3) on the
   fused transport of a one-rank federation.

    python bench/fedeval_micro.py [--out result.json]

Prints one JSON object with the card's name, power limit and max SM clock, read in the same run, beside the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

B, C, NBINS, SCANS = 32, 2, 100, 1024


def median_ms(fn, flush, n=20):
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
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    from hefl_b200 import _ext
    from hefl_b200.config import FLConfig
    from hefl_b200.fl import FederatedRunner
    from hefl_b200.fl.data import BatchFeeder, SyntheticImageDataset
    from hefl_b200.fl.fedeval import count_len
    from multiclient_micro import card

    if not torch.cuda.is_available():
        raise SystemExit("fedeval_micro.py needs a CUDA device")
    ops, dev = _ext.ops(), torch.device("cuda")
    scrub = torch.ones(64 << 20, dtype=torch.float32, device=dev)       # 256 MB > the 50 MB L2

    def flush():
        scrub.sum()

    cfg = FLConfig(model="medcnn", local_epochs=1, steps_per_epoch=2, val_steps=1, deterministic_crypto=True)
    run = FederatedRunner(cfg, device=dev)
    eng, tr = run.trainer.engine, run.trainer

    # 1. the two kernels on the engine's own buffers
    g = torch.Generator(device="cuda").manual_seed(3)
    feat = torch.rand(B, eng.F, device=dev, generator=g).to(torch.bfloat16)
    logits = torch.zeros(B, C, device=dev)
    labels = torch.randint(0, C, (B,), device=dev, generator=g)
    nv = torch.tensor([B], dtype=torch.int32, device=dev)
    counts = torch.zeros(C * C * (NBINS + 1), dtype=torch.int32, device=dev)
    loss = torch.zeros(1, dtype=torch.float64, device=dev)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    probs = torch.zeros(B, C, device=dev)
    head = lambda: ops.head_logits(feat, run.pack.flat, eng.head_offs, eng.h1_buf, eng.dh1_buf, logits, B, eng.F,  # noqa: E731
                                   eng.H1, eng.H2, C)
    stats = lambda: ops.score_stats(logits, labels, nv, probs, counts, loss, err, NBINS)  # noqa: E731
    for _ in range(3):
        head(), stats()
    kernels = {"head_logits_us": 1e3 * median_ms(head, flush), "score_stats_us": 1e3 * median_ms(stats, flush)}

    # 2. a 1,024-scan scoring pass against evaluate's PyTorch forward
    ds = SyntheticImageDataset(SCANS, cfg.image_size, 3, C, seed=7, pin=True)
    feed = BatchFeeder(ds, range(SCANS), B, dev, shuffle=False)
    row = torch.zeros(count_len(C, NBINS), dtype=torch.float64, device=dev)
    tr.score(feed, row)                                  # captures the score graphs
    run.evaluate(ds)
    torch.cuda.synchronize()
    s_ms, e_ms = [], []
    for _ in range(3):
        t0 = time.perf_counter()
        tr.score(feed, row)
        torch.cuda.synchronize()
        s_ms.append(1e3 * (time.perf_counter() - t0))
        t0 = time.perf_counter()
        run.evaluate(ds)
        torch.cuda.synchronize()
        e_ms.append(1e3 * (time.perf_counter() - t0))
    scoring = {"scans": SCANS, "score_pass_ms": statistics.median(s_ms), "evaluate_torch_ms": statistics.median(e_ms),
               "score_us_per_scan": 1e3 * statistics.median(s_ms) / SCANS, "score_launches_per_batch": tr.score_launches}

    # 3. the count ciphertext: encrypt into the symmetric buffer, all-reduce, decrypt
    ctx, V = run.ctx, count_len(C, NBINS)
    vec = row.float()
    view = run.transport.buffer(run.ct_numel)[: 2 * ctx.L * ctx.n]

    def he_round():
        ct = ctx.encrypt(vec, run.pk, seed=1, packing=cfg.packing, out=view)
        data = run.transport.allreduce(ct.data)
        from hefl_b200.he.context import CtBatch

        ctx.decrypt(CtBatch(data, ct.scale, V, cfg.packing), run.sk, divide_by=1.0)

    for _ in range(3):
        he_round()
    cipher = {"values": V, "ciphertexts": ctx.num_ct(V, cfg.packing), "bytes": 2 * ctx.L * ctx.n * 8,
              "encrypt_allreduce_decrypt_us": 1e3 * median_ms(he_round, flush)}
    res = {"card": card(), "batch": B, "image": cfg.image_size, "classes": C, "bins": NBINS, "kernels": kernels,
           "scoring": scoring, "count_ciphertext": cipher}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

"""Ciphertext all-reduce bandwidth sweep (BASELINE.json configs[3]): ring degree 2^12..2^15 x
1..8 RNS limbs, fused NVLink kernel (two_shot / one_shot / multimem) vs NCCL all-reduce + mod-q
kernel. Device-timed (CUDA events, warm-up, max over ranks). Launch with torchrun.

Reports, per (n, L, algo): time, algorithm bandwidth S/t, bus bandwidth 2(P-1)/P * S/t and the
fraction of the nominal 450 GB/s per-direction NVLink 4 bandwidth of an H100 SXM.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hefl_b200.he.context import CKKSContext  # noqa: E402
from hefl_b200.parallel import CollectiveTransport, FusedTransport  # noqa: E402

NVLINK_GBS = 450.0                 # H100 SXM, NVLink 4, per direction (data sheet: 900 GB/s bidirectional)


def timed(fn, iters, warmup, device):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    t = torch.tensor([s.elapsed_time(e) / iters], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cts", type=int, default=64)
    ap.add_argument("--logn", default="12,13,14,15")
    ap.add_argument("--limbs", default="1,2,3,4,5,6,7,8")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default="gpurun_out/allreduce_sweep.json")
    args = ap.parse_args()
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    device = torch.device("cuda", torch.cuda.current_device())
    dist.init_process_group("nccl", device_id=device)
    results = []
    max_numel = args.cts * 2 * 8 * (1 << 15)
    for logn in [int(v) for v in args.logn.split(",")]:
        n = 1 << logn
        for L in [int(v) for v in args.limbs.split(",")]:
            ctx = CKKSContext(n, prime_bits=(54,) * L, scale_bits=40, device=device, enforce_security=False)
            numel = args.cts * 2 * L * n
            nbytes = numel * 8
            gen = torch.Generator(device=device).manual_seed(rank)
            src = torch.stack([torch.randint(0, q, (args.cts, 2, n), generator=gen, device=device, dtype=torch.int64)
                               for q in ctx.primes], dim=2).contiguous()
            ft = FusedTransport(ctx, numel, timeout_s=20.0)
            coll = CollectiveTransport(ctx, numel)
            algos = ["two_shot", "one_shot"] + (["multimem"] if ft.sym.mc_ptr else [])
            row = {"logn": logn, "L": L, "cts": args.cts, "mbytes": nbytes / 1e6, "world": world}
            # NCCL + mod baseline (in place on a private buffer; refilled each iteration outside timing is
            # unnecessary: sums stay < 2^64 for the few timed iterations because every call reduces mod q)
            buf = coll.buffer(numel).view_as(src)
            buf.copy_(src)
            t = timed(lambda: coll.allreduce(buf), args.iters, 3, device)
            row["nccl_ms"] = t
            for algo in algos:
                if algo == "one_shot" and nbytes > 64e6:
                    continue
                ft.algo = algo
                x = ft.buffer(numel).view_as(src)
                x.copy_(src)
                t = timed(lambda: ft.allreduce(x), args.iters, 3, device)
                ft.check_status()
                row[algo + "_ms"] = t
            best = min(v for k, v in row.items() if k.endswith("_ms") and not k.startswith("nccl"))
            row["best_fused_ms"] = best
            row["speedup_vs_nccl"] = row["nccl_ms"] / best
            row["busbw_gbs"] = 2 * (world - 1) / world * nbytes / best / 1e6
            row["frac_nvlink_nominal"] = row["busbw_gbs"] / NVLINK_GBS
            row["best_algo"] = min((v, k[:-3]) for k, v in row.items() if k.endswith("_ms") and not k.startswith(("nccl", "best")))[1]
            results.append(row)
            if rank == 0:
                print(json.dumps(row), flush=True)
            del ft, coll, src, buf, x
            torch.cuda.empty_cache()
    if rank == 0:
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
        json.dump({"world": world, "nvlink_gbs_nominal": NVLINK_GBS,
                   "rows": results}, open(args.out, "w"), indent=1)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

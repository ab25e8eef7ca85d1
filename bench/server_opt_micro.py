#!/usr/bin/env python
"""Cost of the server-optimizer step fused into the CKKS decode on one GPU (CUDA events, L2 flushed).

For each size, from the same decrypted residues:
  * ``decode``: the plain decode (``ckks_decode_residues``, fp32 average out);
  * ``fused <opt>``: ``ckks_decode_server_step_`` (decode + step in one launch) for each optimizer;
  * ``unfused <opt>``: the plain decode followed by the same step written as torch ops.
Every launch (or launch sequence) is timed on its own, after a write of 256 MB that evicts the L2, and each
variant is repeated ``--reps`` times in rotation with the others. Sizes: the medical CNN (222,722 values,
n4096_l3), ResNet-18 (n8192_l4) and ResNet-50 (n16384_l4). The card's name, power limit and max SM clock are
printed with the numbers.

  python bench/server_opt_micro.py [--iters 20] [--reps 3] [--out bench_out/server_opt_micro.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

OPTS = {"fedavgm": 1, "fedadagrad": 2, "fedyogi": 3, "fedadam": 4}


def card():
    import torch

    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:  # noqa: BLE001
        info["power_limit"] = f"unavailable ({e})"
    return info


def torch_step(name, x, a, m, v, nt, lr=0.1, b1=0.9, b2=0.99, tau=1e-3):
    """The step of DESIGN.md §8 as eager torch ops on the fp32 average (the unfused comparison)."""
    import torch

    out = a.clone()
    d = a[:nt] - x[:nt]
    if name == "fedavgm":
        m.mul_(b1).add_(d)
        torch.add(x[:nt], m, alpha=lr, out=out[:nt])
        return out
    m.mul_(b1).add_(d, alpha=1 - b1)
    if name == "fedadagrad":
        v.addcmul_(d, d)
    elif name == "fedyogi":
        d2 = d * d
        v.sub_((1 - b2) * d2 * torch.sign(v - d2))
    else:
        v.mul_(b2).addcmul_(d, d, value=1 - b2)
    out[:nt] = x[:nt] + lr * m / (v.sqrt() + tau)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="medcnn,resnet18,resnet50")
    ap.add_argument("--out", default=os.path.join(ROOT, "bench_out", "server_opt_micro.json"))
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("server_opt_micro.py needs a CUDA device")
    from hefl_b200.config import HE_PRESETS
    from hefl_b200.he.context import CKKSContext
    from hefl_b200.models import ParamPack, create_model

    dev = torch.device("cuda")
    flush = torch.empty(64 << 20, dtype=torch.float32, device=dev)      # 256 MB > the 50 MB L2

    def timeit(fn):
        """median us of one call, each call after an L2 flush, timed alone"""
        ts = []
        for i in range(args.iters + 3):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            if i >= 3:
                ts.append(a.elapsed_time(b) * 1000.0)
        return statistics.median(ts)

    res = {"device": card(), "iters": args.iters, "reps": args.reps, "sizes": {}}
    print(json.dumps(res["device"]), flush=True)
    specs = {"medcnn": ("n4096_l3", None), "resnet18": ("n8192_l4", ("resnet18", 3, 1000, 224)),
             "resnet50": ("n16384_l4", ("resnet50", 3, 1000, 224))}
    for label in args.sizes.split(","):
        preset, model = specs[label]
        if model is None:
            numel = nt = 222722
        else:
            pack = ParamPack(create_model(*model))
            numel, nt = pack.numel, pack.n_trainable
            del pack
        hp = HE_PRESETS[preset]
        ctx = CKKSContext(hp["n"], prime_bits=hp["prime_bits"], scale_bits=hp["scale_bits"], device=dev)
        sk, pk = ctx.keygen(seed=1)
        gen = torch.Generator(device="cuda").manual_seed(2)
        x = torch.randn(numel, device=dev, generator=gen) * 0.05
        ct = ctx.encrypt(x + torch.randn(numel, device=dev, generator=gen) * 0.01, pk, seed=3)
        res_ = ctx.decrypt_residues(ct, sk)
        del ct
        torch.cuda.empty_cache()
        inv = 1.0 / ctx.scale
        out = torch.empty_like(x)
        m = torch.zeros(nt, device=dev)
        v = torch.full((nt,), 1e-6, device=dev)
        variants = {"decode": lambda: ctx.ops.ckks_decode_residues(res_, ctx.consts_cpu, ctx.q0_inv_q1, ctx.logn, inv,
                                                                    ctx.rot, ctx.ksi, numel)}
        for name, code in OPTS.items():
            variants[f"fused {name}"] = (lambda code=code: ctx.ops.ckks_decode_server_step_(
                res_, ctx.consts_cpu, ctx.q0_inv_q1, ctx.logn, inv, ctx.rot, ctx.ksi, numel, 0, nt, x, out, m, v,
                code, 0.1, 0.9, 0.99, 1e-3, None))
            variants[f"unfused {name}"] = (lambda name=name: torch_step(
                name, x, ctx.ops.ckks_decode_residues(res_, ctx.consts_cpu, ctx.q0_inv_q1, ctx.logn, inv, ctx.rot,
                                                      ctx.ksi, numel), m, v, nt))
        times = {k: [] for k in variants}
        for _ in range(args.reps):
            for k, fn in variants.items():
                times[k].append(timeit(fn))
        row = {"preset": preset, "values": numel, "n_trainable": nt, "ciphertexts": ctx.num_ct(numel),
               "median_us": {k: round(statistics.median(t), 2) for k, t in times.items()},
               "reps_us": {k: [round(t, 2) for t in ts] for k, ts in times.items()}}
        res["sizes"][label] = row
        base = row["median_us"]["decode"]
        print(f"{label} ({preset}, {numel} values, {row['ciphertexts']} ciphertexts): decode {base:.1f} us", flush=True)
        for name in OPTS:
            f, u = row["median_us"][f"fused {name}"], row["median_us"][f"unfused {name}"]
            print(f"  {name:11s} fused {f:9.1f} us (x{f / base:.3f} of decode)   decode + torch step {u:9.1f} us",
                  flush=True)
        del res_, x, out, m, v, ctx
        torch.cuda.empty_cache()

    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()

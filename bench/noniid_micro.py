#!/usr/bin/env python
"""Cost of the FedProx term in the Adam kernels on one GPU (CUDA events).

Pairs, each timed alternately 5 times (the two arms share the clock and the neighbours' load):
  * ``adam_step_`` without / with the anchor, at the medical CNN's 222,722 parameters and at ResNet-18's count;
  * one ``train_step`` (CUDA graph) of the medical-CNN engine at mu = 0 / mu = 0.01.
The proximal term adds one fp32 read of the anchor per parameter (0.9 MB per medical-CNN step).

  python bench/noniid_micro.py [--iters 200] [--out bench_out/noniid_micro.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "bench_out", "noniid_micro.json"))
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("noniid_micro.py needs a CUDA device")
    from hefl_b200 import _ext
    from hefl_b200.config import FLConfig
    from hefl_b200.fl.trainer import LocalTrainer
    from hefl_b200.models import ParamPack, create_model

    ops = _ext.ops()
    dev = torch.device("cuda")

    def timeit(fn):
        for _ in range(10):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b) * 1000.0 / args.iters       # us per call

    def pair(name, off, on):
        t0, t1 = [], []
        for _ in range(args.reps):
            t0.append(timeit(off))
            t1.append(timeit(on))
        m0, m1 = statistics.median(t0), statistics.median(t1)
        res[name] = {"plain_us": [round(t, 3) for t in t0], "prox_us": [round(t, 3) for t in t1],
                     "plain_median_us": round(m0, 3), "prox_median_us": round(m1, 3),
                     "prox_over_plain": round(m1 / m0, 4)}
        print(f"{name:34s} plain {m0:9.2f} us   prox {m1:9.2f} us   x{m1 / m0:.3f}", flush=True)

    res = {"device": card(), "iters": args.iters, "reps": args.reps}
    print(json.dumps(res["device"]))
    n18 = ParamPack(create_model("resnet18", 3, 2, 256)).n_trainable
    for label, n in (("medcnn", 222722), ("resnet18", n18)):
        p = torch.randn(n, device=dev)
        g, m, v = torch.zeros_like(p), torch.zeros_like(p), torch.zeros_like(p)
        anchor = p.clone()
        sh = torch.zeros(n, dtype=torch.bfloat16, device=dev)
        st = torch.ones(1, dtype=torch.int64, device=dev)
        pair(f"adam_step_ {label} (n={n})",
             lambda: ops.adam_step_(p, g, m, v, sh, st, None, 1e-3, 1e-4, 0.9, 0.999, 1e-7),
             lambda: ops.adam_step_(p, g, m, v, sh, st, None, 1e-3, 1e-4, 0.9, 0.999, 1e-7, anchor, 0.01))

    def trainer(mu):
        torch.manual_seed(0)
        cfg = FLConfig(model="medcnn", batch_size=32, nn_backend="tcgen05", fedprox_mu=mu)
        model = create_model("medcnn").to(dev)
        pack = ParamPack(model)
        return LocalTrainer(model, pack, cfg, dev, backend="tcgen05", use_graph=True, augment=True), pack

    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randint(0, 256, (32, 256, 256, 3), dtype=torch.uint8, device=dev, generator=g)
    y = torch.randint(0, 2, (32,), device=dev, generator=g)
    tr0, _ = trainer(0.0)
    tr1, pk1 = trainer(0.01)
    tr1.anchor.copy_(pk1.trainable())
    pair("train_step(graph) medcnn mu 0 / 0.01", lambda: tr0.train_step(x, y), lambda: tr1.train_step(x, y))

    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()

"""Per-kernel timing of the medical CNN's tap-GEMM launches of layers 2-6 as the training step makes them
(B = 32 at 256x256): the pooled forward (with arg-max codes) and the dgrad. CUDA events, warm-up, L2 flushed
before every launch. Each time is set against the HBM bytes the kernel must move at 3.35 TB/s:
forward = input read + pooled values and codes written; dgrad = dY read + gX written.

--debug-masks also times every kernel with parts of its work skipped (1 = TMA data, 2 = MMAs, 4 = epilogue);
that needs a build with HEFL_NVCC_EXTRA=-DHEFL_CONV_DEBUG. Writes bench_out/tap_gemm_micro.json (or --out)."""
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from hefl_b200 import _ext
from hefl_b200.config import FLConfig
from hefl_b200.models import ParamPack, create_model
from hefl_b200.ops.conv_engine import MedCNNEngine

HBM = 3.35e12
ops = _ext.ops()
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")


def timeit(fn, iters=20, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record(); torch.cuda.synchronize()
        ts.append(s.elapsed_time(e) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--debug-masks", action="store_true")
    ap.add_argument("--out", default="bench_out/tap_gemm_micro.json")
    args = ap.parse_args()
    B = 32
    dev = torch.device("cuda")
    model = create_model("medcnn").to(dev)
    pack = ParamPack(model)
    eng = MedCNNEngine(model, pack, FLConfig(model="medcnn", batch_size=B), dev)
    x = torch.randint(0, 256, (B, 256, 256, 3), dtype=torch.uint8, device="cuda")
    # one real step leaves X, codes and every dY[l] / gX[l] filled with the step's own data
    eng.train_step(x, torch.randint(0, 2, (B,), device="cuda"), torch.zeros(2, device="cuda"), augment=True)

    res = {"device": torch.cuda.get_device_name(), "kernels": {}}
    masks = [(0, "full")] + ([(4, "no epilogue"), (2, "no MMA"), (1, "no TMA"), (6, "no MMA+epilogue")]
                             if args.debug_masks else [])

    def run(name, fn, mb, extra):
        row = dict(extra)
        for mask, tag in masks:
            ops.conv_set_debug(mask)
            row[f"{tag} us"] = round(timeit(fn), 2)
        ops.conv_set_debug(0)
        t = row["full us"]
        row["MB"] = round(mb / 1e6, 2)
        row["TB/s"] = round(mb / (t * 1e-6) / 1e12, 3)
        row["bound us"] = round(mb / HBM * 1e6, 2)
        res["kernels"][name] = row
        print(f"{name:6s} " + "  ".join(f"{k}={v}" for k, v in row.items()), flush=True)

    for l in range(1, eng.n):
        h, ck, co = eng.H[l], eng.CK[l], eng.Co[l]
        hp = (h - 2) // 2
        P = B * h * h
        mb = P * ck * 2 + B * hp * hp * co * 3
        run(f"fwd{l}", lambda l=l, h=h: ops.conv_fwd_pool(eng.X[l], eng._wf(l), eng.bias[l], eng.X[l + 1],
                                                            eng.amax[l], B, h, h, eng.CK[l], eng.Co[l], False, 3),
            mb, {"H": h, "CK": ck, "CO": co})
    for l in range(eng.n - 1, 0, -1):
        h = eng.H[l]
        P = B * h * h
        mb = P * eng.Co[l] * 2 + P * eng.Ci[l] * 2
        run(f"dgrad{l}", lambda l=l, h=h: ops.conv_dgrad(eng.dY[l], eng._wd(l), eng.gX[l], B, h, h, eng.Co[l],
                                                           eng.Ci[l]),
            mb, {"H": h, "CK": eng.Co[l], "CO": eng.Ci[l]})
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()

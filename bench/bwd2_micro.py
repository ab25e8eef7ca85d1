"""Layer 2's backward of the medical CNN at the training step's shape (B = 32, 256x256, the 127 map, CK = Co = 32) on
the step's own data: the fused conv_dgrad_wgrad (data and weight gradient from one pass over dY, then the partial
reduce) against the standalone pair the step used before (conv_dgrad on one stream, conv_wgrad with its reduce on a
second, as train_step_staged issues them) and against each of the two alone. CUDA events, L2 flushed before every
launch, median of 20 launches; the arms are alternated --rounds times in one process. Bytes are what the work must
move through HBM: dgrad = dY read + gX written, wgrad = X and dY read, fused = X and dY read + gX written.

--debug-masks also times the fused kernel with parts of its work skipped (1 = TMA data, 2 = MMAs, 4 = gX store,
8 = weight gradient); that needs a build with HEFL_NVCC_EXTRA=-DHEFL_CONV_DEBUG. Writes bench_out/bwd2_micro.json
(or --out)."""
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
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--debug-masks", action="store_true")
    ap.add_argument("--out", default="bench_out/bwd2_micro.json")
    args = ap.parse_args()
    B = 32
    dev = torch.device("cuda")
    model = create_model("medcnn").to(dev)
    pack = ParamPack(model)
    eng = MedCNNEngine(model, pack, FLConfig(model="medcnn", batch_size=B), dev)
    x = torch.randint(0, 256, (B, 256, 256, 3), dtype=torch.uint8, device="cuda")
    # one real step leaves X[1], dY[1] and the layer's weights filled with the step's own data
    eng.train_step(x, torch.randint(0, 2, (B,), device="cuda"), torch.zeros(2, device="cuda"), augment=True)
    l = 1
    h, ck, co = eng.H[l], eng.CK[l], eng.Co[l]
    assert eng.dgrad_wgrad[l] and ck == co == 32
    X, dY, Wd, gX, dW = eng.X[l], eng.dY[l], eng._wd(l), eng.gX[l], eng._dw(l)
    side = torch.cuda.Stream(dev)

    def dgrad():
        ops.conv_dgrad(dY, Wd, gX, B, h, h, co, ck)

    def wgrad():
        ops.conv_wgrad(X, dY, dW, B, h, h, ck, co)

    def pair():
        main = torch.cuda.current_stream()
        side.wait_stream(main)
        with torch.cuda.stream(side):
            wgrad()
        dgrad()
        main.wait_stream(side)

    def fused():
        ops.conv_dgrad_wgrad(X, dY, Wd, gX, dW, B, h, h, ck, co)

    P = B * h * h
    act = P * 32 * 2
    macs = 9 * P * 32 * 32                      # per GEMM, valid-or-not pixels alike
    arms = {"pair (dgrad + wgrad on two streams)": (pair, 3 * act, 2 * macs),
            "fused (dgrad_wgrad + reduce)": (fused, 3 * act, 2 * macs),
            "dgrad alone": (dgrad, 2 * act, macs),
            "wgrad + reduce alone": (wgrad, 2 * act, macs)}
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, (fn, _, _) in arms.items():
            times[k].append(timeit(fn))
    res = {"device": torch.cuda.get_device_name(), "B": B, "H": h, "rounds": args.rounds, "arms": {}}
    for k, (_, nbytes, nmac) in arms.items():
        ts = sorted(times[k])
        t = ts[len(ts) // 2]
        row = {"us": [round(v, 2) for v in times[k]], "median us": round(t, 2), "MB": round(nbytes / 1e6, 1),
               "GMAC": round(nmac / 1e9, 2), "TB/s": round(nbytes / (t * 1e-6) / 1e12, 3),
               "bound us": round(nbytes / HBM * 1e6, 2)}
        res["arms"][k] = row
        print(f"{k:38s} " + "  ".join(f"{a}={v}" for a, v in row.items()), flush=True)
    if args.debug_masks:
        res["fused masks"] = {}
        for mask, tag in [(0, "full"), (1, "no TMA data"), (2, "no MMA"), (4, "no gX store"), (8, "no wgrad part"),
                          (6, "no MMA + gX store")]:
            ops.conv_set_debug(mask)
            res["fused masks"][tag] = round(timeit(fused), 2)
        ops.conv_set_debug(0)
        print("fused, parts skipped (us): " + "  ".join(f"{k}={v}" for k, v in res["fused masks"].items()), flush=True)
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()

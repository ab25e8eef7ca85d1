"""Per-kernel timing of the medical CNN's six pooled forward kernels, as the training step launches them
(layer 1 on the compact RGB input, B = 32 at 256x256), with and without arg-max codes (training / evaluation).
CUDA events, warm-up, L2 flushed before every launch. Each time is set against the HBM bytes the kernel must
move (input read, pooled values and codes written) at 3.35 TB/s.

--debug-masks also times every kernel with parts of its work skipped (1 = TMA data, 2 = MMAs, 4 = epilogue);
that needs a build with HEFL_NVCC_EXTRA=-DHEFL_CONV_DEBUG. Writes bench_out/fwd_pool_micro.json (or --out)."""
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
    ap.add_argument("--out", default="bench_out/fwd_pool_micro.json")
    args = ap.parse_args()
    B = 32
    dev = torch.device("cuda")
    model = create_model("medcnn").to(dev)
    pack = ParamPack(model)
    eng = MedCNNEngine(model, pack, FLConfig(model="medcnn", batch_size=B), dev)
    x = torch.randint(0, 256, (B, 256, 256, 3), dtype=torch.uint8, device="cuda")
    eng.train_step(x, torch.randint(0, 2, (B,), device="cuda"), torch.zeros(2, device="cuda"), augment=True)
    eng.preprocess(x, 0, train=False, augment=False)
    assert eng.compact0 and eng.fwd_pair >= 1, "the default RGB engine runs layer 1 on the compact pair-row kernel"

    def launch(l, train):
        h, am = eng.H[l], eng.amax[l] if train else None
        if l == 0:
            ops.conv_fwd_pool_pair(eng.x0(0), eng._wf0c(), eng.bias[0], eng.X[1], am, B, h, h, eng.CK[0], eng.Co[0],
                                   True, 3, True)
        else:
            ops.conv_fwd_pool(eng.X[l], eng._wf(l), eng.bias[l], eng.X[l + 1], am, B, h, h, eng.CK[l], eng.Co[l],
                              False, 3)

    res = {"device": torch.cuda.get_device_name(), "kernels": {}}
    masks = [(0, "full")] + ([(4, "no epilogue"), (2, "no MMA"), (1, "no TMA"), (6, "no MMA+epilogue")]
                             if args.debug_masks else [])
    for l in range(eng.n):
        h = eng.H[l]
        hp = (h - 2) // 2
        in_bytes = B * h * h * (8 if l == 0 else eng.CK[l] * 2)
        out_bytes = B * hp * hp * eng.Co[l] * 2
        code_bytes = B * hp * hp * eng.Co[l]
        row = {"H": h, "CK": eng.CK[l], "CO": eng.Co[l]}
        for train in (True, False):
            mb = in_bytes + out_bytes + (code_bytes if train else 0)
            tag = "train" if train else "eval"
            for mask, name in masks:
                ops.conv_set_debug(mask)
                t = timeit(lambda: launch(l, train))
                row[f"{tag} {name} us"] = round(t, 2)
            ops.conv_set_debug(0)
            t = row[f"{tag} full us"]
            row[f"{tag} MB"] = round(mb / 1e6, 2)
            row[f"{tag} TB/s"] = round(mb / (t * 1e-6) / 1e12, 3)
            row[f"{tag} bound us"] = round(mb / HBM * 1e6, 2)
        res["kernels"][f"fwd{l}"] = row
        print(f"fwd{l} H={h:3d} " + "  ".join(f"{k}={v}" for k, v in row.items() if k not in ("H",)))
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()

"""Layer 1 of the medical CNN on its two RGB input layouts: s-packed [P, 16] (32 bytes per pixel) vs compact [P, 4]
(R, G, B, 0; 8 bytes per pixel). Times preprocess_u8, the pair-row forward (fwd0) and the masked-GEMM weight
gradient (wgrad0) on the same seeded batch (32 x 256 x 256), the two layouts alternated run by run, CUDA events,
L2 flushed before every launch. Records the card, its power limit and max SM clock with the numbers."""
import argparse, json, os, statistics, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from hefl_b200 import _ext


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        vals = [v.strip() for v in r.stdout.splitlines()[0].split(",")]
        return dict(zip(q.split(","), vals))
    except Exception as e:           # the numbers still stand; say where the card data went
        return {"name": torch.cuda.get_device_name(), "query_error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7, help="alternated runs per layout")
    ap.add_argument("--iters", type=int, default=20, help="timed launches per run (median taken)")
    ap.add_argument("--out", default=os.path.join("bench_out", "layer1_micro.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("layer1_micro needs a CUDA device")
    ops = _ext.ops()
    B, H, Co = 32, 256, 32
    Hp, P = (H - 2) // 2, B * H * H
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randint(0, 256, (B, H, H, 3), dtype=torch.uint8, device="cuda", generator=g)
    w = (torch.randn(Co, 3, 3, 3, device="cuda", generator=g) * 0.3).to(torch.bfloat16)
    bias = torch.randn(Co, device="cuda", generator=g) * 0.1
    Ws = torch.zeros(3, Co, 16, dtype=torch.bfloat16, device="cuda")
    Ws[:, :, :9] = w.permute(2, 0, 3, 1).reshape(3, Co, 9)
    Wc = torch.zeros(3, 2, Co, 4, 4, dtype=torch.bfloat16, device="cuda")
    for dx in range(2):
        Wc[:, dx, :, dx:dx + 3, :3] = w.permute(2, 0, 3, 1)
    Xs = torch.zeros(P + 8, 16, dtype=torch.bfloat16, device="cuda")
    Xc = torch.zeros(P, 4, dtype=torch.bfloat16, device="cuda")
    seed = 99
    out = {k: torch.zeros(B * Hp * Hp, Co, dtype=torch.bfloat16, device="cuda") for k in ("s", "c")}
    am = {k: torch.zeros(B * Hp * Hp, Co, dtype=torch.uint8, device="cuda") for k in ("s", "c")}
    gp = (torch.randn(B * Hp * Hp, Co, device="cuda", generator=g)).to(torch.bfloat16)
    dW = torch.zeros(145 * 32, dtype=torch.float32, device="cuda")
    ops.preprocess_u8(x, None, Xs[:P], seed, None, True)
    ops.preprocess_u8(x, None, Xc, seed, None, True, True)
    kern = {
        "spacked": {
            "preprocess": lambda: ops.preprocess_u8(x, None, Xs[:P], seed, None, True),
            "fwd0": lambda: ops.conv_fwd_pool_pair(Xs, Ws.view(-1), bias, out["s"], am["s"], B, H, H, 16, Co, True),
            "wgrad0": lambda: ops.wgrad0_gather(Xs, gp, am["s"], dW, B, H, H, True),
        },
        "compact": {
            "preprocess": lambda: ops.preprocess_u8(x, None, Xc, seed, None, True, True),
            "fwd0": lambda: ops.conv_fwd_pool_pair(Xc, Wc.view(-1), bias, out["c"], am["c"], B, H, H, 16, Co, True, 3, True),
            "wgrad0": lambda: ops.wgrad0_gather(Xc, gp, am["c"], dW, B, H, H, True, 3, True),
        },
    }
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def run(fn):
        ts = []
        for _ in range(args.iters):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fn(); b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b) * 1e3)
        return statistics.median(ts)

    for lay in kern.values():          # warm-up: modules loaded, tensor maps and attributes set
        for fn in lay.values():
            for _ in range(3):
                fn()
    torch.cuda.synchronize()
    same = bool(torch.equal(out["s"], out["c"]) and torch.equal(am["s"], am["c"]))
    samples = {lay: {k: [] for k in kern[lay]} for lay in kern}
    for _ in range(args.runs):
        for k in ("preprocess", "fwd0", "wgrad0"):
            for lay in kern:
                samples[lay][k].append(run(kern[lay][k]))
    # X0 bytes each kernel moves: written once by preprocess, read by fwd0 and by wgrad0
    x0_mb = {"spacked": P * 32 / 1e6, "compact": P * 8 / 1e6}
    res = {"card": card(), "shape": {"B": B, "H": H, "W": H, "Co": Co}, "runs": args.runs, "iters": args.iters,
           "x0_MB": x0_mb, "fwd0_outputs_bit_identical": same, "us": {}}
    for lay in kern:
        res["us"][lay] = {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                          for k, v in samples[lay].items()}
    for k in ("preprocess", "fwd0", "wgrad0"):
        s, c = res["us"]["spacked"][k], res["us"]["compact"][k]
        print(f"{k:11s} spacked {s['median']:7.1f} us [{s['min']:.1f}, {s['max']:.1f}]   "
              f"compact {c['median']:7.1f} us [{c['min']:.1f}, {c['max']:.1f}]")
    print(json.dumps({"card": res["card"], "fwd0_outputs_bit_identical": same}))
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()

"""Per-kernel timing of one medical-CNN training step on the tcgen05 engine (CUDA events,
warm-up, L2 flushed between iterations). Writes gpurun_out/nn_micro.json."""
# --in-channels 1 times the grayscale arm (rs-packed layer 1) and writes its report to --out, by default
# bench_out/nn_micro_c1.json; --out also moves the RGB report.
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, torch.nn.functional as F
from hefl_b200 import _ext
from hefl_b200.config import FLConfig
from hefl_b200.models import ParamPack, create_model
from hefl_b200.ops.conv_engine import MedCNNEngine

ops = _ext.ops()
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")


def timeit(fn, iters=10, warmup=3):
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
    ap.add_argument("--in-channels", type=int, choices=(1, 3), default=3)
    ap.add_argument("--out", default=None, help="JSON report path")
    args = ap.parse_args()
    C = args.in_channels
    B = 32
    cfg = FLConfig(model="medcnn", batch_size=B, in_channels=C)
    dev = torch.device("cuda")
    model = create_model("medcnn", in_channels=C).to(dev)
    pack = ParamPack(model)
    eng = MedCNNEngine(model, pack, cfg, dev)
    x = torch.randint(0, 256, (B, 256, 256, C), dtype=torch.uint8, device="cuda")
    y = torch.randint(0, 2, (B,), device="cuda")
    out = torch.zeros(2, device="cuda")
    eng.train_step(x, y, out, augment=True)
    res = {}
    th = eng._make_theta()
    res["make_theta(torch)"] = timeit(lambda: eng._make_theta())
    res["preprocess"] = timeit(lambda: ops.preprocess_u8(x, None, eng.X[0], 99, None, eng.spack0))
    for l in range(eng.n):
        h = eng.H[l]
        res[f"fwd{l}"] = timeit(lambda l=l, h=h: ops.conv_fwd_pool(eng.X[l], eng._wf(l), eng.bias[l], eng.X[l + 1], eng.amax[l], B, h, h, eng.CK[l], eng.Co[l], eng.spack0 and l == 0, C))
        if l == 0 and eng.fwd_pair:
            res["fwd0(tap-GEMM, not used)"] = res["fwd0"]
            res["fwd0"] = timeit(lambda: ops.conv_fwd_pool_pair(eng._x0_bufs[0], eng._wf(0), eng.bias[0], eng.X[1], eng.amax[0], B, h, h, eng.CK[0], eng.Co[0], eng.spack0, C))
    g = torch.randn(B, 512, device="cuda").to(torch.bfloat16).view_as(eng.X[eng.n]).contiguous()
    for l in range(eng.n - 1, -1, -1):
        h = eng.H[l]
        gin = g if l == eng.n - 1 else eng.gX[l + 1]
        if l == 0:
            res["wgrad0(gather from pooled grad)"] = timeit(lambda: ops.wgrad0_gather(eng._x0_bufs[0], gin, eng.amax[0], eng._dw(0), B, h, h))
            res["wgrad0(masked GEMMs, mma.sync)"] = timeit(lambda: ops.wgrad0_gather(eng._x0_bufs[0], gin, eng.amax[0], eng._dw(0), B, h, h, eng.spack0, C))
            eng.dY[0] = torch.zeros(eng.P[0], eng.Co[0], dtype=torch.bfloat16, device="cuda")
        res[f"unpool{l}"] = timeit(lambda l=l, h=h, gin=gin: ops.unpool_relu(gin, eng.amax[l], eng.X[l + 1], eng.dY[l], B, h, h, eng.Co[l]))
        res[f"wgrad{l}(tcgen05)"] = timeit(lambda l=l, h=h: ops.conv_wgrad(eng.X[l], eng.dY[l], eng._dw(l), B, h, h, eng.CK[l], eng.Co[l]))
        if l > 0:
            res[f"dgrad{l}"] = timeit(lambda l=l, h=h: ops.conv_dgrad(eng.dY[l], eng._wd(l), eng.gX[l], B, h, h, eng.Co[l], eng.Ci[l]))
    res["finalize"] = timeit(lambda: ops.conv_grad_finalize(eng.dW32, eng.table, pack.grad))
    res["relayout"] = timeit(lambda: eng.after_update())

    def head():
        feat = eng.X[eng.n].view(B, -1).float().requires_grad_(True)
        logits = eng._head(feat)
        loss = F.cross_entropy(logits, y)
        loss.backward()
        return feat.grad.to(torch.bfloat16)
    res["head(torch fwd+bwd)"] = timeit(head)
    head_call = lambda: ops.head_forward_backward(eng.X[eng.n], pack.flat, pack.grad, eng.head_offs, y, eng.dfeat, eng.h1_buf, eng.dh1_buf, out, B, eng.F, eng.H1, eng.H2, eng.C, True)
    res["head(cluster kernel)"] = timeit(head_call)
    m = torch.zeros_like(pack.grad); v = torch.zeros_like(pack.grad); st = torch.ones(1, dtype=torch.int64, device="cuda")
    res["adam"] = timeit(lambda: ops.adam_step_(pack.trainable(), pack.grad, m, v, eng.shadow, st, None, 1e-3, 1e-4, 0.9, 0.999, 1e-7))
    from hefl_b200.fl.trainer import LocalTrainer
    tr = LocalTrainer(model, pack, cfg, dev, backend="tcgen05", use_graph=False)
    eng = tr.engine
    def full_step():
        tr.train_step(x, y)
    res["train_step(eager)"] = timeit(full_step, iters=5)
    # whole step as a CUDA graph
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        full_step()
    torch.cuda.synchronize()
    gph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gph):
        full_step()
    res["train_step(graph)"] = timeit(lambda: gph.replay(), iters=10)
    skip = ("train_step", "head(torch", "make_theta", "unpool0", "wgrad0(tcgen05)")
    tot = sum(v for k, v in res.items() if not k.startswith(skip))
    for k, v in res.items():
        print(f"{k:24s} {v:9.1f} us")
    print(f"{'sum of parts':24s} {tot:9.1f} us")
    out = args.out or (None if C == 3 else os.path.join("bench_out", f"nn_micro_c{C}.json"))
    if out is not None:
        os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
        json.dump(res, open(out, "w"), indent=1)
        return
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump(res, open("gpurun_out/nn_micro.json", "w"), indent=1)


if __name__ == "__main__":
    main()

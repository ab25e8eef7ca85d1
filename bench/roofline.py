"""profiles/roofline.md: per-kernel achieved fraction of the measured roofline (MEASURED_PEAKS.json) for one
training step of the medical CNN at batch 32, from the stand-alone kernel times in profiles/nn_micro.json
(CUDA events, L2 flushed) and analytic byte / FLOP counts of each kernel (minimum traffic: every operand
read once, every result written once)."""
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
HBM = float(peaks.get("hbm_gbs", peaks.get("hbm_copy_gbs", 3350.0)))           # GB/s (H100 SXM data sheet)
TF = float(peaks.get("bf16_tflops", peaks.get("cublas_bf16_tflops", 989.0)))     # TFLOP/s (H100 SXM data sheet, dense)
t = json.load(open(os.path.join(ROOT, "profiles", "nn_micro.json")))

B = 32
H = [256, 127, 62, 30, 14, 6, 2]          # input side of layer l (H[6] = feature map)
Ci = [3, 32, 32, 32, 64, 64]
CK = [16, 32, 32, 32, 64, 64]
Co = [32, 32, 32, 64, 64, 128]
rows = []


def add(name, key, bytes_, flops):
    if key not in t:
        return
    us = t[key]
    gbs = bytes_ / us / 1e3
    tf = flops / us / 1e6
    rows.append((name, us, bytes_ / 1e6, gbs, gbs / HBM, flops / 1e9, tf, tf / TF))


add("preprocess (uint8 -> bf16 [P,16], affine)", "preprocess", B * 256 * 256 * (3 + 32), 0)
for l in range(6):
    P_in = B * H[l] * H[l]
    Ho = H[l] - 2
    P_pool = B * H[l + 1] * H[l + 1]
    fl = 2.0 * B * Ho * Ho * 9 * Ci[l] * Co[l]
    add(f"conv{l + 1} fwd + bias + ReLU + pool", f"fwd{l}", P_in * CK[l] * 2 + P_pool * Co[l] * 3, fl)
add("dense head fwd + loss + bwd (cluster)", "head(cluster kernel)", (512 * 128 + 128 * 64 + 128) * 4 * 2 + B * 512 * 4, 2.0 * 3 * B * (512 * 128 + 128 * 64 + 128))
for l in range(5, 0, -1):
    P_in = B * H[l] * H[l]
    P_pool = B * H[l + 1] * H[l + 1]
    Ho = H[l] - 2
    fl = 2.0 * B * Ho * Ho * 9 * Ci[l] * Co[l]
    add(f"conv{l + 1} un-pool (+ReLU mask)", f"unpool{l}", P_pool * Co[l] * 5 + P_in * Co[l] * 2, 0)
    add(f"conv{l + 1} wgrad (tcgen05, MN-major)", f"wgrad{l}(tcgen05)", P_in * (CK[l] + Co[l]) * 2, fl)
    add(f"conv{l + 1} dgrad (tcgen05)", f"dgrad{l}", P_in * (Co[l] + Ci[l]) * 2, fl)
P_pool = B * H[1] * H[1]
add("conv1 wgrad (masked GEMMs from the pooled gradient, mma.sync)", "wgrad0(masked GEMMs, mma.sync)",
    B * 256 * 256 * 32 + P_pool * 32 * 3, 2.0 * P_pool * 32 * 27)
add("conv1 wgrad (round-1 kernel: FP32-pipe gather, fallback)", "wgrad0(gather from pooled grad)",
    B * 256 * 256 * 32 + P_pool * 32 * 3, 2.0 * P_pool * 32 * 27)
add("Adam (222,722 parameters, bf16 shadow)", "adam", 222722 * (4 * 7 + 2), 0)

out = ["# Roofline table — one training step of the medical CNN, batch 32, one H100\n",
       f"Denominators (MEASURED_PEAKS.json): HBM copy {HBM:.0f} GB/s, cuBLAS bf16 {TF:.0f} TFLOP/s. Times are the",
       "stand-alone kernel times of `profiles/nn_micro.json` (CUDA events, warm-up, L2 flushed between iterations);",
       "bytes and FLOPs are the analytic minimum for the kernel (operands read once, results written once;",
       "FLOPs of the real, un-padded problem). In the step graph kernels overlap (two streams + PDL), so the",
       "step takes ≈290 µs, less than the sum of this column.\n",
       "| kernel | µs | MB | GB/s | of HBM | GFLOP | TFLOP/s | of bf16 peak |", "|---|---|---|---|---|---|---|---|"]
for r in rows:
    out.append(f"| {r[0]} | {r[1]:.1f} | {r[2]:.1f} | {r[3]:.0f} | {r[4]:.2f} | {r[5]:.2f} | {r[6]:.1f} | {r[7]:.3f} |")
out.append("")
out.append("Reading: every kernel of this model is far from the bf16 tensor peak by construction (3–128 channels, "
           "arithmetic intensity 10–150 FLOP/B at best) and the large ones sit at 0.2–0.5 of the HBM roofline; what "
           "separates them from it is per-tile latency and instruction issue in the epilogues (DESIGN.md §4, "
           "`profiles/ncu_summary.md`), not bandwidth or tensor throughput.")
open(os.path.join(ROOT, "profiles", "roofline.md"), "w").write("\n".join(out) + "\n")
print("\n".join(out))

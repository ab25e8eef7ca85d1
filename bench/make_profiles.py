"""Turn the scratch artefacts in gpurun_out/ into the tracked summaries under profiles/."""
import csv
import glob
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "profiles")
GO = os.path.join(ROOT, "gpurun_out")
PEAKS = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {"hbm_gbs": 6650.0, "bf16_tflops": 1590.0}

KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed", "sm__inst_executed.sum.per_cycle_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size",
        "launch__block_size", "launch__shared_mem_per_block_dynamic", "sm__cycles_elapsed.max",
        "l1tex__m_xbar2l1tex_read_bytes_mem_global_op_tma_ld.sum"]


def ncu_raw_all(path):
    """Every kernel of a report: list of ({metric: (value, unit)}, kernel name)."""
    r = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True)
    rows = list(csv.reader(r.stdout.splitlines()))
    if len(rows) < 3:
        return []
    hdr, units = rows[0], rows[1]
    out = []
    for vals in rows[2:]:
        d = {h: (v, u) for h, u, v in zip(hdr, units, vals)}
        out.append((d, d.get("Kernel Name", ("", ""))[0]))
    return out


def launches(path):
    with open(path) as f:
        lines = [l for l in f if not l.startswith("==")]
    out = []
    for r in csv.DictReader(lines):
        t = float(r["Metric Value"].replace(",", ""))
        u = r["Metric Unit"]
        t = t / 1000 if u == "ns" else (t * 1000 if u == "ms" else t)
        out.append((re.sub(r"\(.*", "", r["Kernel Name"]).replace("void ", ""), r["Grid Size"], t))
    return out


def main():
    os.makedirs(OUT, exist_ok=True)
    md = ["# ncu captures (`--set full --clock-control none --import-source on`, one GPU)\n",
          f"Roofline denominators (MEASURED_PEAKS.json): HBM copy {PEAKS.get('hbm_gbs')} GB/s, cuBLAS bf16 "
          f"{PEAKS.get('bf16_tflops')} TFLOP/s burst.\n"]
    reports = []
    for rep in sorted(glob.glob(os.path.join(GO, "*.ncu-rep"))):
        seen = set()
        for d, name in ncu_raw_all(rep):
            key = re.sub(r"\(.*", "", name)
            if key in seen:                     # one entry per distinct kernel of a report
                continue
            seen.add(key)
            reports.append((rep, d, name))
    for rep, d, name in reports:
        md.append(f"\n## {os.path.basename(rep)} — `{name[:130]}`\n")
        md.append("| metric | value | unit |\n|---|---|---|")
        for k in KEYS:
            if k in d:
                md.append(f"| {k} | {d[k][0]} | {d[k][1]} |")
        try:
            t_us = float(d["gpu__time_duration.sum"][0])
            t_us = t_us if d["gpu__time_duration.sum"][1] == "us" else t_us / 1000 if d["gpu__time_duration.sum"][1] == "ns" else t_us * 1000
            rd = float(d["dram__bytes_read.sum"][0]); wr = float(d["dram__bytes_write.sum"][0])
            scale = {"Mbyte": 1e6, "Gbyte": 1e9, "Kbyte": 1e3, "byte": 1}
            tot = rd * scale.get(d["dram__bytes_read.sum"][1], 1) + wr * scale.get(d["dram__bytes_write.sum"][1], 1)
            gbs = tot / t_us / 1e3
            md.append(f"\nDRAM traffic {tot / 1e6:.1f} MB in {t_us:.1f} us = {gbs:.0f} GB/s = "
                      f"{gbs / PEAKS.get('hbm_gbs', 6650):.2f} of measured HBM copy bandwidth.")
        except Exception as e:  # noqa: BLE001
            md.append(f"\n(derived numbers unavailable: {e})")
    open(os.path.join(OUT, "ncu_summary.md"), "w").write("\n".join(md) + "\n")

    for lf in sorted(glob.glob(os.path.join(GO, "launches*.csv"))):
        rows = launches(lf)
        name = os.path.basename(lf).replace(".csv", "")
        with open(os.path.join(OUT, name + ".md"), "w") as f:
            f.write(f"# Kernel launch list ({name}; `ncu --metrics gpu__time_duration.sum`, serialized, cold caches: compare shares)\n\n")
            f.write("| # | kernel | grid | us |\n|---|---|---|---|\n")
            for i, (k, g, t) in enumerate(rows):
                f.write(f"| {i} | `{k[:90]}` | {g} | {t:.1f} |\n")
            f.write(f"\nTotal {sum(t for *_, t in rows):.1f} us over {len(rows)} launches.\n")
    for jf in ["nn_micro.json", "he_micro_v1.json", "he_micro_v2.json", "tcconv_micro.json", "allreduce_sweep_2gpu.json", "allreduce_sweep_8gpu.json",
               "allreduce_sweep_4gpu.json", "mp2.json"]:
        p = os.path.join(GO, jf)
        if os.path.exists(p):
            json.dump(json.load(open(p)), open(os.path.join(OUT, jf), "w"), indent=1)
    print("profiles written:", sorted(os.listdir(OUT)))


if __name__ == "__main__":
    main()

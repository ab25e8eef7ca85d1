"""In-tree build of the native library ``hefl_b200/_native.so``.

* ``.cu`` files are compiled by nvcc for sm_90a only (``-gencode arch=compute_90a,
  code=sm_90a -lineinfo``) and do **not** include PyTorch headers (seconds per file);
* ``*_bindings.cpp`` files are compiled by g++ against the PyTorch headers and register
  ``torch.ops.hefl.*``;
* objects are cached by a content hash of (source, headers, flags), so the GPU box, which
  receives the built ``.so`` with the snapshot, never rebuilds.

Run ``python -m hefl_b200._build`` (or ``__graft_entry__.build()``) to build.
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "csrc"
OUT_DIR = Path(__file__).resolve().parent
OBJ_DIR = OUT_DIR / "_obj"
LIB_PATH = OUT_DIR / "_native.so"

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CXX = os.environ.get("HEFL_CXX", "/usr/bin/g++")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
] + os.environ.get("HEFL_NVCC_EXTRA", "").split()      # e.g. HEFL_NVCC_EXTRA="-DHEFL_CONV_DEBUG" (experiments)

CUDA_SOURCES = [
    "he/cuda/he_kernels.cu",
    "he/cuda/he_kernels2.cu",
    "he/cuda/he_eval2.cu",
    "comm/allreduce_modq.cu",
    "nn/conv_tcgen05.cu",
    "nn/gemm_tcgen05.cu",
    "nn/nn_kernels.cu",
    "nn/resnet_kernels.cu",
    "nn/wgrad_gather.cu",
    "nn/wgrad0_mma.cu",
    "nn/head_cluster.cu",
    "nn/gradcam.cu",
    "nn/input_grad.cu",
    "nn/score.cu",
]
HOST_SOURCES = [
    "he/host_math.cpp",
]
BINDING_SOURCES = [
    "he/he_bindings.cpp",
    "comm/comm_bindings.cpp",
    "nn/nn_bindings.cpp",
]


def _headers_digest(subdirs) -> str:
    """Digest of the headers a source directory can see: its own, csrc/he (shared arithmetic) and csrc/common
    (Hopper plumbing)."""
    h = hashlib.sha256()
    for sub in sorted(set(subdirs) | {"he", "common"}):
        for p in sorted((CSRC / sub).rglob("*")):
            if p.suffix in (".h", ".cuh", ".hpp"):
                h.update(p.read_bytes())
    return h.hexdigest()


def _torch_flags():
    import torch
    from torch.utils import cpp_extension as ce

    inc = [f"-I{p}" for p in ce.include_paths()]
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    lib_dir = Path(torch.__file__).parent / "lib"
    return inc, abi, lib_dir


def _compile_one(src: Path, obj: Path, cmd: list[str], digest: str, log: list[str]) -> None:
    stamp = obj.with_suffix(obj.suffix + ".stamp")
    if obj.exists() and stamp.exists() and stamp.read_text() == digest:
        return
    t0 = time.time()
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"compile failed: {' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
    (obj.with_suffix(obj.suffix + ".log")).write_text(r.stdout + r.stderr)
    stamp.write_text(digest)
    log.append(f"  built {src.relative_to(ROOT)} in {time.time() - t0:.1f}s")


def build(verbose: bool = True, force: bool = False) -> Path:
    """Compile every source (if stale) and link ``_native.so``. Returns its path."""
    OBJ_DIR.mkdir(exist_ok=True)
    inc, abi, torch_lib = _torch_flags()
    hdr_cache = {}

    def hdr_for(src: Path) -> str:
        sub = src.relative_to(CSRC).parts[0]
        if sub not in hdr_cache:
            hdr_cache[sub] = _headers_digest([sub])
        return hdr_cache[sub]

    cuda_inc = "/usr/local/cuda/include"
    jobs = []
    objs = []
    log: list[str] = []

    def digest_for(src: Path, flags: list[str]) -> str:
        h = hashlib.sha256()
        h.update(src.read_bytes())
        h.update(hdr_for(src).encode())
        # include paths differ between the CPU box and the GPU box; they do not change the object
        h.update(" ".join(f for f in flags if not f.startswith("-I")).encode())
        return h.hexdigest()

    for rel in CUDA_SOURCES:
        src = CSRC / rel
        if not src.exists():
            continue
        obj = OBJ_DIR / (rel.replace("/", "_") + ".o")
        cmd = [NVCC, *NVCC_FLAGS, f"-I{CSRC}", "-c", str(src), "-o", str(obj)]
        jobs.append((src, obj, cmd, digest_for(src, NVCC_FLAGS)))
        objs.append(obj)
    host_flags = ["-O3", "-std=c++17", "-fPIC", "-fopenmp", f"-I{CSRC}", f"-I{cuda_inc}"]
    for rel in HOST_SOURCES:
        src = CSRC / rel
        obj = OBJ_DIR / (rel.replace("/", "_") + ".o")
        cmd = [CXX, *host_flags, "-c", str(src), "-o", str(obj)]
        jobs.append((src, obj, cmd, digest_for(src, host_flags)))
        objs.append(obj)
    bind_flags = ["-O2", "-std=c++17", "-fPIC", "-fopenmp", f"-D_GLIBCXX_USE_CXX11_ABI={abi}",
                  "-DTORCH_EXTENSION_NAME=_native", f"-I{CSRC}", f"-I{cuda_inc}", *inc,
                  "-Wno-deprecated-declarations"]
    for rel in BINDING_SOURCES:
        src = CSRC / rel
        if not src.exists():
            continue
        obj = OBJ_DIR / (rel.replace("/", "_") + ".o")
        cmd = [CXX, *bind_flags, "-c", str(src), "-o", str(obj)]
        jobs.append((src, obj, cmd, digest_for(src, bind_flags)))
        objs.append(obj)

    if force:
        for _, obj, _, _ in jobs:
            st = obj.with_suffix(obj.suffix + ".stamp")
            if st.exists():
                st.unlink()

    with cf.ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 2)) as ex:
        futs = [ex.submit(_compile_one, *j, log) for j in jobs]
        for f in futs:
            f.result()

    link_digest = hashlib.sha256(
        "".join(o.with_suffix(o.suffix + ".stamp").read_text() for o in objs).encode()).hexdigest()
    link_stamp = OUT_DIR / "_native.so.stamp"
    if not (LIB_PATH.exists() and link_stamp.exists() and link_stamp.read_text() == link_digest):
        cmd = [CXX, "-shared", "-o", str(LIB_PATH), *map(str, objs),
               f"-L{torch_lib}", "-lc10", "-ltorch_cpu", "-ltorch", "-lc10_cuda", "-ltorch_cuda",
               "-L/usr/local/cuda/lib64", "-lcudart", "-fopenmp",
               f"-Wl,-rpath,{torch_lib}", "-Wl,--no-as-needed"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed: {' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
        link_stamp.write_text(link_digest)
        log.append(f"  linked {LIB_PATH.relative_to(ROOT)}")
    if verbose:
        for line in log:
            print(line, file=sys.stderr)
        if not log:
            print("  native library up to date", file=sys.stderr)
    return LIB_PATH


if __name__ == "__main__":
    build(verbose=True, force="--force" in sys.argv)

"""Which CUDA kernels a piece of work launched, as torch.profiler reports them (shared by the GPU test modules)."""
import re
import time
import warnings

import torch


def kernels_run(fn, attempts=5):
    """Runs fn() under torch.profiler and returns (its result, the names of the CUDA kernels it launched).

    Now and then the profiler hands back a trace with no device activity at all although fn launched native
    kernels (the launch counter moved). Such a trace says nothing about which kernel ran, so fn, which must be
    repeatable, runs again under a fresh profiler, up to `attempts` times. Empty traces can come several in a row and
    then stop, so each retry waits a little longer before it starts. A trace with any kernel in it is final."""
    from torch.profiler import ProfilerActivity, profile

    from hefl_b200 import _ext

    ops = _ext.ops()
    for attempt in range(attempts):
        if attempt:
            time.sleep(0.25 * attempt)
        torch.cuda.synchronize()
        launches = int(ops.launch_count())
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        if names or int(ops.launch_count()) == launches:
            break
        warnings.warn("torch.profiler returned no device activity for launched kernels; running again")
    return out, names


def ran(names, kernel):
    """True if a launched kernel's demangled name contains `kernel` (e.g. "ntt2_kernel<12, true, 3u>") as a whole
    identifier."""
    pat = re.compile(r"(?<![\w])" + re.escape(kernel))
    return any(pat.search(n) for n in names)

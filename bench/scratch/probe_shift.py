import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch
from hefl_b200 import _ext
ops = _ext.ops()
for CK in (64, 32, 16):
    A = torch.randn(144, CK, device="cuda").to(torch.bfloat16)
    Bm = torch.randn(32, CK, device="cuda").to(torch.bfloat16)
    res = []
    for s in range(0, 10):
        out = ops.umma_shift_probe(A, Bm, CK, s)
        torch.cuda.synchronize()
        ref = A[s:s + 128].float() @ Bm.float().t()
        res.append(float((out - ref).abs().max()) < 1e-2)
    print("CK", CK, "ok per shift 0..9:", "".join("1" if r else "0" for r in res))

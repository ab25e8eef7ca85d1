"""hefl_b200 — H100-native encrypted federated learning engine.

Packed-CKKS FedAvg with hand-written sm_90a kernels (NTT/INTT, CKKS codec, fused
encrypt/decrypt, fused ciphertext all-reduce over NVLink peer memory, tensor-core implicit-GEMM
convolution), plus a compatibility surface that keeps the reference's ``FLPyfhelin`` function
names, Pyfhel 2.3.1-style key generation and pickle file layout
(the reference's FLPyfhelin.py).

Sub-packages: ``he`` (scheme), ``ops`` (kernel wrappers), ``models`` (CNNs), ``parallel``
(symmetric memory + collectives), ``fl`` (round loop), ``compat`` (Pyfhel / FLPyfhelin
shims), ``utils``.
"""
__version__ = "0.1.0"

from .config import FLConfig  # noqa: E402,F401

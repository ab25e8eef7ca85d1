"""``from Pyfhel import Pyfhel, PyPtxt, PyCtxt`` (FLPyfhelin.py:27, notebook N:21) resolved by the
hefl_b200 shim: Pyfhel 2.3.1 call signatures, H100-native kernels underneath."""
from hefl_b200.compat.pyfhel_shim import PyCtxt, Pyfhel, PyPtxt  # noqa: F401

__version__ = "2.3.1+hefl_b200"

"""``from FLPyfhelin import *`` keeps working (notebook N:21): thin re-export of
hefl_b200.compat.FLPyfhelin, the H100-native counterpart of /root/reference/FLPyfhelin.py."""
from hefl_b200.compat.FLPyfhelin import *  # noqa: F401,F403
from hefl_b200.compat import FLPyfhelin as _impl

configure = _impl.configure


def __getattr__(name):          # live view of the module globals (BS, image_size, ...)
    return getattr(_impl, name)

"""fhe_rs_b200 -- H100-native (sm_90a) engine for the BFV ciphertext-arithmetic hot path of
tlepoint/fhe.rs, behind the C ABI of include/fhe_b200.h.

`fhe_rs_b200.bfv` mirrors the reference's fhe::bfv interface for that path.  The CUDA
extension (libfhe_b200.so) is mandatory: there is no CPU fallback."""
from . import _capi  # noqa: F401
from .bfv import *  # noqa: F401,F403
from . import mbfv  # noqa: F401,E402  (fhe::mbfv, multiparty BFV)

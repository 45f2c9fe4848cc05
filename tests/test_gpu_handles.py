"""GPU tests of the device memory the handles of the C ABI own: freeing a batch, key, encoder, secret key,
multiplicator or relinearization-key generator gives back what it took, and a creation that fails part-way keeps
nothing.  Run with `-m gpu`."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DEGREE, T, SIZES = 1 << 14, 786433, [62] * 4
REPS = 4   # handles of each type per cycle


@pytest.fixture(scope="module")
def F():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


def test_handles_give_back_their_memory(oracle, F):
    """five cycles of creating and freeing every handle type keep no device memory.  Each cycle also makes
    multiplicators whose creation fails after it uploaded the NTT tables of a prime of its own: the extended basis is a
    new prime with a valid root followed by a prime of the parameter set with a wrong one ("psi differs").  At 2^14 x 4
    moduli the handles of any one type take 2 MB or more per cycle, so a type that kept its memory would show far above
    the 4 MB the comparison allows for the driver's own bookkeeping."""
    import torch
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    gpar = F.BfvParameters(DEGREE, T, moduli_sizes=SIZES, device=0)
    moduli, L = gpar.moduli(), len(SIZES)
    rng = np.random.default_rng(11)
    seed = (C.c_uint8 * 32)(*range(32))
    coeffs = np.ascontiguousarray(rng.integers(-1, 2, DEGREE, dtype=np.int64))
    key_words = np.zeros(L * L * DEGREE, np.uint64)
    crp = F.mbfv.CommonRandomPoly._generate(gpar, L, 0, bytes(seed))
    one = (C.c_uint8 * 1)(1)

    # a 50-bit NTT-friendly prime the parameter set does not have, with the root a host-only set of its own gives it
    new_q = oracle.generate_prime(50, 2 * DEGREE, 1 << 50)
    assert new_q is not None and new_q not in moduli
    own = F.BfvParameters(DEGREE, T, moduli=[new_q], device=-1)
    new_psi, q0_psi = C.c_uint64(), C.c_uint64()
    assert lib.fhe_b200_params_psi(own._h, new_q, C.byref(new_psi)) == _capi.OK
    assert lib.fhe_b200_params_psi(gpar._h, moduli[0], C.byref(q0_psi)) == _capi.OK

    def multiplicator(basis, psi):
        b = np.ascontiguousarray(np.array(basis, dtype=np.uint64))
        ps = None if psi is None else np.ascontiguousarray(np.array(psi, dtype=np.uint64))
        h = C.c_void_p()
        rc = lib.fhe_b200_multiplicator_create(gpar._h, 0, one, 1, one, 1, one, 1, one, 1, b.ctypes.data, len(b),
                                               None if ps is None else ps.ctypes.data, one, 1, one, 1, C.byref(h))
        return rc, h

    def cycle():
        for _ in range(REPS):
            h = C.c_void_p()
            assert lib.fhe_b200_batch_alloc(gpar._h, 1, 2, 0, _capi.NTT, C.byref(h)) == _capi.OK
            assert lib.fhe_b200_batch_free(h) == _capi.OK
            h = C.c_void_p()
            assert lib.fhe_b200_ksk_upload(gpar._h, 0, 0, key_words.ctypes.data, key_words.ctypes.data, L,
                                           C.byref(h)) == _capi.OK
            assert lib.fhe_b200_ksk_free(h) == _capi.OK
            h = C.c_void_p()
            assert lib.fhe_b200_encoder_create(gpar._h, None, C.byref(h)) == _capi.OK
            assert lib.fhe_b200_encoder_free(h) == _capi.OK
            sk = C.c_void_p()
            assert lib.fhe_b200_secret_key_create(gpar._h, coeffs.ctypes.data, C.byref(sk)) == _capi.OK
            h = C.c_void_p()
            assert lib.fhe_b200_rkg_create(sk, crp._h, 10, seed, C.byref(h), None) == _capi.OK
            assert lib.fhe_b200_rkg_free(h) == _capi.OK
            assert lib.fhe_b200_secret_key_free(sk) == _capi.OK
            rc, h = multiplicator(moduli + [new_q], None)
            assert rc == _capi.OK
            assert lib.fhe_b200_multiplicator_free(h) == _capi.OK
            rc, h = multiplicator([new_q, moduli[0]], [new_psi.value, (q0_psi.value + 1) % moduli[0]])
            assert rc == _capi.INVALID_ARGUMENT and b"psi differs" in lib.fhe_b200_last_error()
            assert h.value is None
        assert lib.fhe_b200_sync(None) == _capi.OK
    cycle()                                   # the parameter set's tables and scratch pool are built on first use
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(5):
        cycle()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 4 << 20

"""The three key-switch code paths must produce the same words: the default (the digit transforms' rows pass fused
with the inner product), FHE_B200_KSMAC=tma (rows pass, then the TMA inner-product kernel) and FHE_B200_KSMAC=classic
(per-thread inner product), plus the default with one-ciphertext chunks and the TMA inner product at digit ring
depths 3 and 4 (FHE_B200_KS_STAGES; the depth-3 run also takes the ring-depth-2 cols pass, FHE_B200_TMA_COLS=2, which
the mixed-size case enters with reduction on load).  Each path runs this file as a script in a
subprocess (the switch is read once per process) and the outputs are compared word for word.  The oracle checks of
test_gpu_parity.py pin the default path to the reference; this test pins the alternatives to it.

Shapes: set C (N = 2^15, 14 x 62-bit) mul+relin, rotation and a stand-alone key switch; set C with a level-0 key
serving level-1 ciphertexts (13 digits against 14 key limbs); N = 2^14 with four limbs; N = 2^13 with moduli of mixed
sizes (Barrett limbs, digits reduced as the transform reads them)."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PATHS = {"fused": {}, "tma": {"FHE_B200_KSMAC": "tma"}, "classic": {"FHE_B200_KSMAC": "classic"},
         "fused_chunk1": {"FHE_B200_CHUNK": "1"},
         "tma_stages3": {"FHE_B200_KSMAC": "tma", "FHE_B200_KS_STAGES": "3", "FHE_B200_TMA_COLS": "2"},
         "tma_stages4": {"FHE_B200_KSMAC": "tma", "FHE_B200_KS_STAGES": "4"}}


def _rows(rng, moduli, prefix, degree):
    a = np.zeros(tuple(prefix) + (len(moduli), degree), np.uint64)
    for i, q in enumerate(moduli):
        a[..., i, :] = rng.integers(0, q, size=tuple(prefix) + (degree,), dtype=np.uint64)
    return a


def compute(out_path):
    sys.path.insert(0, ROOT)
    import fhe_rs_b200 as F
    res = {}
    cases = [("c", 1 << 15, 786433, [62] * 14, 0, 2, True), ("c_lv1", 1 << 15, 786433, [62] * 14, 1, 2, False),
             ("n14", 1 << 14, 786433, [62] * 4, 0, 2, True), ("mixed", 1 << 13, 65537, [62, 40, 30], 0, 5, True)]
    for name, degree, t, sizes, ct_level, count, ks in cases:
        rng = np.random.default_rng(len(res) + 31)
        par = F.BfvParameters(degree, t, moduli_sizes=sizes, device=0)
        key_mod = par.moduli()
        ct_mod = key_mod[:len(key_mod) - ct_level]   # level l drops the last l moduli
        n_dig = len(ct_mod)
        kc, gc = _rows(rng, key_mod, (2, n_dig), degree), _rows(rng, key_mod, (2, n_dig), degree)
        rk = F.RelinearizationKey.from_arrays(par, kc[0], kc[1], ciphertext_level=ct_level, key_level=0)
        gk = F.GaloisKey.from_arrays(par, 3, gc[0], gc[1], ciphertext_level=ct_level, key_level=0)
        A = F.Ciphertext.from_host(par, _rows(rng, ct_mod, (count, 2), degree), level=ct_level)
        B = F.Ciphertext.from_host(par, _rows(rng, ct_mod, (count, 2), degree), level=ct_level)
        res[name + "_mul_relin"] = F.Multiplicator.default(rk).multiply(A, B).to_host()
        res[name + "_galois"] = gk.relinearize(A).to_host()
        if ks:
            k = F.KeySwitchingKey.from_arrays(par, kc[0], kc[1], ciphertext_level=0, key_level=0)
            X = F.Ciphertext.from_host(par, _rows(rng, key_mod, (count, 1), degree), repr=F.POWER_BASIS)
            res[name + "_key_switch"] = k.key_switch(X, 0).to_host()
    np.savez(out_path, **res)


def test_key_switch_paths_agree(tmp_path):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    got = {}
    for name, env in PATHS.items():
        out = os.path.join(str(tmp_path), name + ".npz")
        r = subprocess.run([sys.executable, os.path.abspath(__file__), out], cwd=ROOT, env=dict(os.environ, **env),
                           capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        got[name] = np.load(out)
    keys = sorted(got["fused"].files)
    assert len(keys) == 11
    for name in PATHS:
        assert sorted(got[name].files) == keys
        for k in keys:
            assert got[name][k].dtype == np.uint64
            assert (got[name][k] == got["fused"][k]).all(), "%s: %s differs from the fused path" % (name, k)


if __name__ == "__main__":
    compute(sys.argv[1])

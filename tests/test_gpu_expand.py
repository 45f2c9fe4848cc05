"""Oblivious expansion on the device (fhe_b200_expand, EvaluationKey::expands of evaluation_key.rs:192-256): bit-exact
against the CPU oracle per query, with keys at the ciphertext level and leveled ones, at the MulPIR and Set C shapes, in
a MulPIR server response, across chunks, and through the C++ mirror.  Run with `-m gpu`."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MULPIR_T = (1 << 20) + (1 << 19) + (1 << 17) + (1 << 16) + (1 << 14) + 1   # examples/mulpir.rs:36


@pytest.fixture(scope="module")
def F():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


def _setup(oracle, F, degree, t, sizes, levels, ct_level, key_level, seed):
    """parameters, secret key, and the expansion keys of `levels` levels (oracle dict and device EvaluationKey)"""
    opar = oracle.BfvParameters(degree, t, moduli_sizes=sizes)
    gpar = F.BfvParameters(degree, t, moduli=opar.moduli, device=0)
    rng = np.random.default_rng(seed)
    sk = oracle.SecretKey(opar, rng)
    ogk, ek = {}, F.EvaluationKey(gpar)
    for l in range(levels):
        e = (degree >> l) + 1
        ogk[e] = oracle.GaloisKey(sk, e, rng, ct_level, key_level)
        ek.add_galois_key(F.GaloisKey.from_arrays(gpar, e, *ogk[e].ksk.arrays(), ciphertext_level=ct_level,
                                                  key_level=key_level))
    return opar, gpar, rng, sk, ogk, ek


@pytest.mark.parametrize("degree", [16, 64])
@pytest.mark.parametrize("ct_level,key_level", [(0, 0), (1, 0)])
def test_expands_matches_oracle(oracle, F, degree, ct_level, key_level):
    """sizes 1, 2, 3, 5, 8, 13 and N; Q = 1 and 3 queries in one call; output i of query q is entry i*Q + q"""
    t = 1153
    logn = degree.bit_length() - 1
    opar, gpar, rng, sk, ogk, ek = _setup(oracle, F, degree, t, [62] * 3, logn, ct_level, key_level, degree + ct_level)
    octs = [sk.encrypt(rng.integers(0, t, degree), ct_level, rng) for _ in range(3)]
    X = F.Ciphertext.from_host(gpar, np.stack([c.to_array() for c in octs]), level=ct_level)
    X1 = F.Ciphertext.from_host(gpar, octs[0].to_array()[None], level=ct_level)
    for size in (1, 2, 3, 5, 8, 13, degree):
        exp = [[c.to_array() for c in oracle.expands(opar, ogk, o, size)] for o in octs]
        got = ek.expands_batch(X, size).to_host()
        assert got.shape[0] == 3 * size
        for i in range(size):
            for q in range(3):
                assert (got[i * 3 + q] == exp[q][i]).all(), (size, i, q)
        one = ek.expands(X1, size)
        assert len(one) == size
        for i in range(size):
            assert (one[i].to_host()[0] == exp[0][i]).all(), (size, i)


def test_mulpir_shape_expansion_decrypts(oracle, F):
    """examples/mulpir.rs: N = 8192, moduli 50/55/55, its t, keys of EvaluationKeyBuilder::new_leveled(&sk, 1, 0), the
    query at level 1 expanded to dim1 + dim2 = 115: bit-exact, and output k decrypts to 1 at the two chosen indices and
    to 0 elsewhere"""
    size, level = 115, 7
    opar, gpar, rng, sk, ogk, ek = _setup(oracle, F, 8192, MULPIR_T, [50, 55, 55], level, 1, 0, 8192)
    inv = pow(1 << level, -1, MULPIR_T)
    chosen = (17, 58 + 40)
    pt = np.zeros(size, np.int64)
    pt[list(chosen)] = inv
    query = sk.encrypt(pt, 1, rng)
    got = ek.expands_batch(F.Ciphertext.from_host(gpar, query.to_array()[None], level=1), size).to_host()
    exp = oracle.expands(opar, ogk, query, size)
    for k in range(size):
        assert (got[k] == exp[k].to_array()).all(), k
        dec = sk.decrypt(oracle.Ciphertext.from_array(opar, got[k], 1))
        assert int(dec[0]) == (1 if k in chosen else 0) and not dec[1:].any(), k


def test_set_c_expansion(oracle, F):
    """Set C (N = 2^15, 14 x 62-bit): size 4 against the oracle; size 1024 -- two chunks at the last level -- equal to
    the per-level composition of fhe_b200_galois, sub, mul_plain and add the parent build ran"""
    degree, t = 1 << 15, 65537
    opar, gpar, rng, sk, ogk, ek = _setup(oracle, F, degree, t, [62] * 14, 2, 0, 0, 15)
    query = sk.encrypt(rng.integers(0, t, 4), 0, rng)
    X = F.Ciphertext.from_host(gpar, query.to_array()[None])
    got = ek.expands_batch(X, 4).to_host()
    for k, c in enumerate(oracle.expands(opar, ogk, query, 4)):
        assert (got[k] == c.to_array()).all(), k
    # size 1024: keys of the other eight levels are random words (both routes use the same ones)
    moduli = gpar.moduli()
    for l in range(2, 10):
        kw = np.zeros((2, 14, 14, degree), np.uint64)
        for j, q in enumerate(moduli):
            kw[:, :, j] = rng.integers(0, q, size=(2, 14, degree), dtype=np.uint64)
        ek.add_galois_key(F.GaloisKey.from_arrays(gpar, (degree >> l) + 1, kw[0], kw[1]))
        del kw
    size = 1024
    fast = ek.expands_batch(X, size)
    lo = X.clone()
    for l in range(10):
        step = 1 << l
        sub = ek.gk[(degree >> l) + 1].relinearize(lo)
        hi = lo.clone()
        hi -= sub
        hi.mul_plain(oracle.expansion_monomial(opar, l).c)
        lo += sub
        nxt = F.Ciphertext(gpar, 2 * step)
        for src, first in ((lo, 0), (hi, step)):
            F.bfv.check(F._capi.lib().fhe_b200_batch_copy_range(nxt._h, first, src._h, 0, 1, step, 0))
        lo = nxt
        del sub, hi
    buf_a = np.empty((64, 2, 14, degree), np.uint64)
    buf_b = np.empty_like(buf_a)
    for first in range(0, size, 64):
        fast.to_host(buf_a, first)
        lo.to_host(buf_b, first)
        assert (buf_a == buf_b).all(), first


def test_mulpir_server_response(oracle, F):
    """the server side of examples/mulpir.rs:160-182 at N = 8192 on a 5 x 4 database of level-1 plaintexts: expand,
    take the first dim1 outputs, dot_product_scalar with every database column, ct x ct with the second-dimension
    selectors, sum, relinearize, switch to the last level -- bit-exact against the oracle's same sequence, and the
    response decrypts to the selected row"""
    dim1, dim2 = 5, 4
    size, level = dim1 + dim2, 4
    opar, gpar, rng, sk, ogk, ek = _setup(oracle, F, 8192, MULPIR_T, [50, 55, 55], level, 1, 0, 77)
    ork = oracle.RelinearizationKey(sk, rng, 1, 1)
    grk = F.RelinearizationKey.from_arrays(gpar, *ork.ksk.arrays(), ciphertext_level=1, key_level=1)
    ctx1 = opar.context_at_level(1)
    db = rng.integers(0, MULPIR_T, size=(dim1 * dim2, 8192)).astype(np.uint64)
    pts = [oracle.Poly.from_u64(ctx1, db[k], oracle.NTT) for k in range(dim1 * dim2)]
    row, col = 3, 2
    inv = pow(1 << level, -1, MULPIR_T)
    qv = np.zeros(size, np.int64)
    qv[row], qv[dim1 + col] = inv, inv
    query = sk.encrypt(qv, 1, rng)
    # oracle
    oexp = oracle.expands(opar, ogk, query, size)
    oout = None
    for i in range(dim2):
        d = oracle.dot_product_scalar(oexp[:dim1], [pts[k * dim2 + i] for k in range(dim1)])
        prod = d.mul(oexp[dim1 + i])
        oout = prod if oout is None else oout.add(prod)
    oout = ork.relinearizes(oout).switch_to_level(2)
    # device
    expanded = ek.expands_batch(F.Ciphertext.from_host(gpar, query.to_array()[None], level=1), size)
    query_vec, selectors = expanded.take(0, dim1), expanded.take(dim1, dim2)
    columns = np.stack([pts[k * dim2 + i].c for i in range(dim2) for k in range(dim1)])   # [column i][k]
    dots = F.dot_product_scalar(query_vec, F.Ciphertext.from_host(gpar, columns[:, None], level=1), n_terms=dim1)
    prods = dots * selectors
    out = prods.take(0, 1)
    for i in range(1, dim2):
        out += prods.take(i, 1)
    resp = grk.relinearizes(out).switch_to_level(2).to_host()[0]
    assert (resp == oout.to_array()).all()
    dec = sk.decrypt(oracle.Ciphertext.from_array(opar, resp, 2))
    assert (dec == db[row * dim2 + col]).all()


def test_expansion_launches_per_level(F):
    """one batched Galois call and one butterfly per level: expanding to 64 (six levels) launches at most six times
    what expanding to 2 (one level) launches"""
    from fhe_rs_b200 import _capi
    degree = 64
    par = F.BfvParameters(degree, 1153, moduli_sizes=[62] * 3, device=0)
    rng = np.random.default_rng(5)
    moduli = par.moduli()

    def rnd(*shape):
        a = np.zeros(shape + (3, degree), np.uint64)
        for j, q in enumerate(moduli):
            a[..., j, :] = rng.integers(0, q, size=shape + (degree,), dtype=np.uint64)
        return a
    ek = F.EvaluationKey(par)
    for l in range(6):
        k = rnd(2, 3)
        ek.add_galois_key(F.GaloisKey.from_arrays(par, (degree >> l) + 1, k[0], k[1]))
    X = F.Ciphertext.from_host(par, rnd(1, 2))
    counts = {}
    for size in (2, 64, 2, 64):   # the first pass builds the tables
        c0 = _capi.lib().fhe_b200_launch_count()
        ek.expands_batch(X, size).sync()
        counts[size] = _capi.lib().fhe_b200_launch_count() - c0
    assert 0 < counts[64] <= 6 * counts[2], counts


def test_expand_errors(F):
    """the error codes of fhe_b200_expand and fhe_b200_batch_copy_range"""
    import ctypes as C
    from fhe_rs_b200 import _capi
    L = _capi.lib()
    degree = 16
    par = F.BfvParameters(degree, 1153, moduli_sizes=[62] * 3, device=0)
    other = F.BfvParameters(degree, 1153, moduli_sizes=[62] * 3, device=0)
    rng = np.random.default_rng(9)
    moduli = par.moduli()

    def rnd(count, parts, limbs=3):
        a = np.zeros((count, parts, limbs, degree), np.uint64)
        for j in range(limbs):
            a[:, :, j] = rng.integers(0, moduli[j], size=(count, parts, degree), dtype=np.uint64)
        return a
    k = rnd(2, 3)
    keys = [F.KeySwitchingKey(par, k[0], k[1]), F.KeySwitchingKey(par, k[0], k[1])]   # level 0
    k1 = rnd(2, 3)
    key_l1 = F.KeySwitchingKey(par, k1[0, :2], k1[1, :2], ciphertext_level=1, ksk_level=0)
    key_other = F.KeySwitchingKey(other, k[0], k[1])
    X = F.Ciphertext.from_host(par, rnd(2, 2))

    def call(ct, size, ks, out, n=None):
        arr = (C.c_void_p * max(1, len(ks)))(*[x._h.value if x is not None else None for x in ks])
        return L.fhe_b200_expand(ct._h, size, C.cast(arr, C.POINTER(C.c_void_p)), len(ks) if n is None else n,
                                 out._h, None)

    out4 = F.Ciphertext(par, 8)
    assert call(X, 4, keys, out4) == _capi.OK
    assert call(X, 0, keys, out4) == _capi.INVALID_ARGUMENT                          # InvalidExpansionSize
    assert call(X, degree + 1, keys, F.Ciphertext(par, 2 * (degree + 1))) == _capi.INVALID_ARGUMENT
    assert call(X, 4, keys, out4, n=1) == _capi.INVALID_ARGUMENT                     # Missing GaloisKey
    assert call(X, 4, [keys[0], None], out4) == _capi.INVALID_ARGUMENT
    assert call(X, 4, [keys[0], key_l1], out4) == _capi.INVALID_LEVEL                # key for another level
    assert call(X, 4, [keys[0], key_other], out4) == _capi.CONTEXT_MISMATCH          # key of other parameters
    X3 = F.Ciphertext.from_host(par, rnd(2, 3))
    assert call(X3, 4, keys, F.Ciphertext(par, 8, 3)) == _capi.BAD_POLY_COUNT
    Xp = F.Ciphertext.from_host(par, rnd(2, 2), repr=F.POWER_BASIS)
    assert call(Xp, 4, keys, out4) == _capi.INVALID_REPRESENTATION
    assert call(X, 4, keys, F.Ciphertext(par, 6)) == _capi.INVALID_ARGUMENT          # wrong out shape
    assert call(X, 4, keys, F.Ciphertext(par, 8, level=1)) == _capi.INVALID_ARGUMENT
    X8 = F.Ciphertext.from_host(par, rnd(8, 2))
    assert call(X8, 1, [], X8) == _capi.INVALID_ARGUMENT                             # out aliases ct
    assert call(X, 1, [], F.Ciphertext(par, 2)) == _capi.OK                          # size 1: a copy
    # copy_range
    dst = F.Ciphertext(par, 3)
    assert L.fhe_b200_batch_copy_range(dst._h, 0, X8._h, 1, 3, 3, None) == _capi.OK
    assert (dst.to_host() == X8.to_host()[1::3]).all()
    assert L.fhe_b200_batch_copy_range(dst._h, 0, X8._h, 2, 3, 3, None) == _capi.INVALID_ARGUMENT   # 2 + 6 = 8
    assert L.fhe_b200_batch_copy_range(dst._h, 1, X8._h, 0, 1, 3, None) == _capi.INVALID_ARGUMENT
    assert L.fhe_b200_batch_copy_range(dst._h, 0, X8._h, 0, 0, 1, None) == _capi.INVALID_ARGUMENT
    assert L.fhe_b200_batch_copy_range(X8._h, 0, X8._h, 1, 1, 1, None) == _capi.INVALID_ARGUMENT
    assert L.fhe_b200_batch_copy_range(F.Ciphertext(par, 1, 3)._h, 0, X8._h, 0, 1, 1, None) == _capi.BAD_POLY_COUNT
    assert L.fhe_b200_batch_copy_range(dst._h, 0, Xp._h, 0, 1, 1, None) == _capi.INVALID_REPRESENTATION
    assert L.fhe_b200_batch_copy_range(F.Ciphertext(par, 1, level=1)._h, 0, X8._h, 0, 1, 1, None) == _capi.INVALID_LEVEL


@pytest.mark.parametrize("env", [{"FHE_B200_CHUNK": "2", "FHE_B200_STREAMS": "1"}, {"FHE_B200_CHUNK": "2"},
                                 {"FHE_B200_CHUNK": "2", "FHE_B200_STREAMS": "4"}])
def test_expand_across_chunks(F, env):
    """a Q = 7 expansion whose levels span several chunks (dealt over 1, 2 and 4 side streams, one chunk straddling the
    partial last level's spill boundary) equals seven Q = 1 expansions (tests/expand_chunk_probe.py)"""
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "expand_chunk_probe.py")], cwd=ROOT,
                         env=dict(os.environ, **env), capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "expand chunk probe ok" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]


def test_cpp_mirror_expands_and_inner_sum(oracle, F, tmp_path):
    """EvaluationKey::{expands, expands_batch, computes_inner_sum} and Ciphertext::take of include/fhe_b200.hpp equal
    the Python mirror"""
    degree, t, size, count = 64, 1153, 13, 2
    exps = sorted({(degree >> l) + 1 for l in range(4)} | {pow(3, 1 << k, 2 * degree) for k in range(5)}
                  | {2 * degree - 1})
    opar = oracle.BfvParameters(degree, t, moduli_sizes=[62] * 3)
    gpar = F.BfvParameters(degree, t, moduli=opar.moduli, device=0)
    rng = np.random.default_rng(31)
    sk = oracle.SecretKey(opar, rng)
    ek = F.EvaluationKey(gpar)
    lines = ["%d %d 3 %d %d %d" % (degree, t, size, count, len(exps)), " ".join(map(str, opar.moduli)),
             " ".join(map(str, exps))]
    for k, e in enumerate(exps):
        c0, c1 = oracle.GaloisKey(sk, e, rng).ksk.arrays()
        c0.tofile(str(tmp_path / ("gk%d_c0.bin" % k)))
        c1.tofile(str(tmp_path / ("gk%d_c1.bin" % k)))
        ek.add_galois_key(F.GaloisKey.from_arrays(gpar, e, c0, c1))
    (tmp_path / "args.txt").write_text("\n".join(lines) + "\n")
    words = np.stack([sk.encrypt(rng.integers(0, t, degree), 0, rng).to_array() for _ in range(count)])
    words.tofile(str(tmp_path / "ct.bin"))
    X = F.Ciphertext.from_host(gpar, words)
    exe = str(tmp_path / "expand_test")
    lib_dir = os.path.join(ROOT, "fhe_rs_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "expand_test.cpp"), "-o", exe,
                           "-L", lib_dir, "-lfhe_b200", "-Wl,-rpath," + lib_dir])
    out = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
    batch = ek.expands_batch(X, size).to_host()
    listed = np.concatenate([b.to_host() for b in ek.expands(X, size)])
    assert (np.fromfile(str(tmp_path / "out_batch.bin"), np.uint64) == batch.ravel()).all()
    assert (np.fromfile(str(tmp_path / "out_list.bin"), np.uint64) == listed.ravel()).all()
    assert (np.fromfile(str(tmp_path / "out_inner.bin"), np.uint64) == ek.computes_inner_sum(X).to_host().ravel()).all()

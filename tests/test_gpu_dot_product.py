"""Ciphertext dot products (fhe_b200_dot_product, _keyed) and batch sums (fhe_b200_batch_sum), and their Python / C++
mirrors.

Every output is compared word for word with the reference's sequence built from existing device calls, each pinned to
the oracle elsewhere: the batched product (fhe_b200_mul), the sum of the products (a host sum modulo each limb, or a
chain of fhe_b200_add), fhe_b200_relinearize and fhe_b200_switch_down; the MulPIR response and the voting tally are
also checked against the tests that compute them with host loops.  The chunking and kernel switches are rerun in
subprocesses (tests/dot_product_chunk_probe.py).  Run with `-m gpu`."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
TESTS = os.path.join(ROOT, "tests")
if TESTS not in sys.path:
    sys.path.insert(0, TESTS)

from dot_product_chunk_probe import DotSetup, host_sum, rand_rows, word_checks   # noqa: E402
from edge_inputs import BOUNDARY_PRIMES   # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def F():
    from conftest import has_gpu
    if not has_gpu():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


# ---- batch sums

@pytest.mark.parametrize("parts", [1, 2, 3, 4])
def test_batch_sum_parts_and_representations(F, parts):
    """1 to 4 parts, NTT and power basis, from zero and accumulating, at run lengths 1, 2, 5, 64, 65 and 1000, on
    words at q - 1 (a 64-bit accumulator would overflow after four terms)"""
    from fhe_rs_b200 import _capi
    degree = 16
    par = F.BfvParameters(degree, 1153, moduli_sizes=[62, 62, 62], device=0)
    moduli = [int(q) for q in par.moduli()]
    rng = np.random.default_rng(parts)
    for n_terms, groups in ((1, 3), (2, 4), (5, 3), (64, 2), (65, 3), (1000, 1)):
        w = rand_rows(rng, moduli, (groups * n_terms, parts), degree)
        w[: n_terms] = np.array(moduli, np.uint64)[:, None] - 1   # group 0: every word at q - 1
        for repr_ in (_capi.NTT, _capi.POWER_BASIS):
            X = F.Ciphertext.from_host(par, w, 0, repr_)
            got = X.sum(n_terms)
            assert got.representation == repr_
            exp = host_sum(w, moduli, n_terms)
            assert (got.to_host() == exp).all(), (n_terms, repr_)
            base = rand_rows(rng, moduli, (groups, parts), degree)
            out = F.Ciphertext.from_host(par, base, 0, repr_)
            X.sum(n_terms, out=out)
            both = host_sum(np.concatenate([base[:, None], exp[:, None]], axis=1).reshape((-1,) + base.shape[1:]),
                            moduli, 2)
            assert (out.to_host() == both).all(), (n_terms, repr_)


def test_batch_sum_long_runs_at_the_boundary_primes(F):
    """runs of 1000 and 4096 words at q - 1 and random words modulo the boundary primes: the Barrett reduction of
    non-Solinas limbs and the thinnest Solinas margin take 128-bit sums far above 2^64"""
    degree = 16
    moduli = [BOUNDARY_PRIMES["solinas_max_c"], BOUNDARY_PRIMES["non_solinas_min"], BOUNDARY_PRIMES["above_2_61"]]
    par = F.BfvParameters(degree, 65537, moduli=moduli, device=0)
    rng = np.random.default_rng(21)
    for n_terms, groups in ((1000, 2), (4096, 1)):
        w = rand_rows(rng, moduli, (groups * n_terms, 2), degree)
        w[:n_terms] = np.array(moduli, np.uint64)[:, None] - 1
        X = F.Ciphertext.from_host(par, w)
        assert (X.sum(n_terms).to_host() == host_sum(w, moduli, n_terms)).all(), n_terms


def test_batch_sum_equals_add_chain(F):
    """one batch_sum equals the chain of fhe_b200_add calls it replaces, and the whole batch sums by default"""
    par = F.BfvParameters(1 << 13, 786433, moduli_sizes=[62, 40, 30], device=0)
    moduli = [int(q) for q in par.moduli()]
    rng = np.random.default_rng(3)
    X = F.Ciphertext.from_host(par, rand_rows(rng, moduli, (12, 2), 1 << 13))
    for n_terms in (1, 4, 12):
        got = X.sum(n_terms).to_host()
        for g in range(12 // n_terms):
            acc = X.take(g * n_terms, 1)
            for i in range(1, n_terms):
                acc += X.take(g * n_terms + i, 1)
            assert (got[g] == acc.to_host()[0]).all(), (n_terms, g)
    assert (X.sum().to_host() == X.sum(12).to_host()).all()


def test_batch_sum_multiplication_basis(F):
    """batches over the multiplication basis sum limb by limb like any other"""
    degree = 64
    par = F.BfvParameters(degree, 1153, moduli_sizes=[62, 62], device=0)
    basis = [int(q) for q in par.mul_basis(0)]
    rng = np.random.default_rng(9)
    w = rand_rows(rng, basis, (6, 3), degree)
    X = F.Ciphertext.from_host(par, w, 0, mul_basis=True)
    assert (X.sum(3).to_host() == host_sum(w, basis, 3)).all()
    out = F.Ciphertext(par, 2, 3, 0, mul_basis=True)
    out.upload(np.zeros((2, 3, len(basis), degree), np.uint64))
    X.sum(3, out=out)
    assert (out.to_host() == host_sum(w, basis, 3)).all()


# ---- dot products

def _shapes():
    return {
        "n16": (16, 1153, [62] * 3, None),
        "n64": (64, 1153, [62] * 3, None),
        "mixed": (1 << 13, 65537, [62, 30, 50], None),
        "boundary": (1 << 13, 65537, None, [BOUNDARY_PRIMES["solinas_max_c"], BOUNDARY_PRIMES["non_solinas_min"],
                                            BOUNDARY_PRIMES["above_2_61"]]),
    }


@pytest.mark.parametrize("name", list(_shapes()))
def test_dot_product_every_level_key_and_switch(F, name):
    """at every operand level: no key (3 parts), a key at the ciphertext level, a leveled key (one level up) and, at the
    single-modulus level, a base-2^b key; switched to every level at or below the operands'"""
    degree, t, sizes, moduli = _shapes()[name]
    n_mod = len(moduli or sizes)
    for level in range(n_mod):
        for key_level in sorted({level, max(0, level - 1)}):
            S = DotSetup(F, degree, t, sizes, level, key_level, 3, 4, 10 * level + key_level, moduli=moduli)
            for out_level in range(level, n_mod):
                S.check(out_level)
                if key_level == level:
                    S.check(out_level, with_key=False)


def test_dot_product_set_c(F):
    """set C (N = 2^15, 14 x 62 bits) at level 0 with a level-0 key, and at level 1 with a level-0 key, switched two
    levels down"""
    S = DotSetup(F, 1 << 15, 786433, [62] * 14, 0, 0, 2, 3, 1)
    S.check()
    S.check(with_key=False)
    S = DotSetup(F, 1 << 15, 786433, [62] * 14, 1, 0, 2, 2, 2)
    S.check(3)


@pytest.mark.parametrize("shared", ["a", "b"])
def test_dot_product_shared_operand_and_one_term(F, shared):
    """either operand shared by every group, at group counts that repeat it within one chunk, and n_terms = 1"""
    for groups, n_terms in ((5, 3), (1, 7), (9, 1)):
        S = DotSetup(F, 64, 1153, [62] * 3, 0, 0, groups, n_terms, groups, shared=shared)
        S.check()
        S.check(2, with_key=False)


def test_dot_product_against_the_oracle(oracle, F):
    """N = 64: the oracle's loop of mul, add, relinearizes and switch_to_level with a real key"""
    degree, t = 64, 1153
    opar = oracle.BfvParameters(degree, t, moduli_sizes=[62] * 3)
    gpar = F.BfvParameters(degree, t, moduli=opar.moduli, device=0)
    rng = np.random.default_rng(11)
    sk = oracle.SecretKey(opar, rng)
    ork = oracle.RelinearizationKey(sk, rng, 0, 0)
    grk = F.RelinearizationKey.from_arrays(gpar, *ork.ksk.arrays())
    n_terms = 5
    xs = [sk.encrypt(rng.integers(0, t, degree).astype(np.int64), 0, rng) for _ in range(2 * n_terms)]
    oout = None
    for i in range(n_terms):
        p = xs[i].mul(xs[n_terms + i])
        oout = p if oout is None else oout.add(p)
    oout = ork.relinearizes(oout).switch_to_level(1)
    A = F.Ciphertext.from_host(gpar, np.stack([c.to_array() for c in xs[:n_terms]]))
    B = F.Ciphertext.from_host(gpar, np.stack([c.to_array() for c in xs[n_terms:]]))
    got = F.dot_product(A, B, n_terms, grk, level=1).to_host()[0]
    assert (got == oout.to_array()).all()


def test_chunk_word_checks(F):
    """the chunk-cutting cases of the probe, in this process (default chunking)"""
    word_checks(F)


# ---- keyed

def test_keyed_groups_equal_single_key_calls(F):
    """group g of the keyed call equals the single-key call with rks[index[g]]; more than 64 keys in one call"""
    degree = 64
    for n_keys, groups in ((3, 7), (70, 70)):
        S = DotSetup(F, degree, 1153, [62] * 3, 0, 0, groups, 2, n_keys)
        rng = np.random.default_rng(n_keys)
        rks = []
        for _ in range(n_keys):
            c = rand_rows(rng, S.moduli, (2, 3), degree)
            rks.append(F.RelinearizationKey.from_arrays(S.par, c[0], c[1]))
        index = [(g * 5 + 1) % n_keys for g in range(groups)]
        got = F.dot_product_keyed(S.A, S.B, 2, rks, index, level=1).to_host()
        for k in sorted(set(index)):
            exp = S.got(1, rks[k])
            for g in range(groups):
                if index[g] == k:
                    assert (got[g] == exp[g]).all(), (n_keys, g)


def test_clients_dot_products_decrypt_under_their_own_keys(F):
    """eight clients with device-generated keys: each group's relinearized dot product decrypts to the dot product of
    the plaintext vectors under its own secret key, and not under a neighbour's"""
    degree, t, n, n_terms = 64, 1153, 8, 4
    par = F.BfvParameters(degree, t, moduli_sizes=[62, 62, 62], device=0)
    sks = F.SecretKey.random_vec(par, n, seed=bytes(range(32)))
    rks = [F.RelinearizationKey.new(sk, seed=bytes([c + 1]) * 32) for c, sk in enumerate(sks)]
    rng = np.random.default_rng(5)
    enc = F.Encoding.simd()
    xv = rng.integers(0, t, (n, n_terms, degree)).astype(np.uint64)
    yv = rng.integers(0, t, (n, n_terms, degree)).astype(np.uint64)
    A = np.concatenate([sks[c].try_encrypt(F.PlaintextVec.try_encode(xv[c].reshape(-1), enc, par),
                                           seed=bytes([c + 41]) * 32).to_host() for c in range(n)])
    B = np.concatenate([sks[c].try_encrypt(F.PlaintextVec.try_encode(yv[c].reshape(-1), enc, par),
                                           seed=bytes([c + 81]) * 32).to_host() for c in range(n)])
    out = F.dot_product_keyed(F.Ciphertext.from_host(par, A), F.Ciphertext.from_host(par, B), n_terms, rks,
                              list(range(n)))
    for c in range(n):
        want = (xv[c].astype(object) * yv[c].astype(object)).sum(axis=0) % t
        dec = sks[c].try_decrypt(out.take(c, 1)).try_decode(enc)
        assert (dec.astype(object) == want).all(), c
        wrong = sks[(c + 1) % n].try_decrypt(out.take(c, 1)).try_decode(enc)
        assert not (wrong.astype(object) == want).all(), c


# ---- reference workloads

def test_mulpir_response_in_one_call(oracle, F):
    """the server response of test_gpu_expand.py::test_mulpir_server_response (examples/mulpir.rs:160-183) with its
    second dimension as one dot_product call: the same words as that test's loop of take / += / relinearizes /
    switch_to_level, and the oracle's"""
    from test_gpu_expand import MULPIR_T, _setup
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
    expanded = ek.expands_batch(F.Ciphertext.from_host(gpar, query.to_array()[None], level=1), size)
    query_vec, selectors = expanded.take(0, dim1), expanded.take(dim1, dim2)
    columns = np.stack([pts[k * dim2 + i].c for i in range(dim2) for k in range(dim1)])
    dots = F.dot_product_scalar(query_vec, F.Ciphertext.from_host(gpar, columns[:, None], level=1), n_terms=dim1)
    prods = dots * selectors
    loop = prods.take(0, 1)
    for i in range(1, dim2):
        loop += prods.take(i, 1)
    loop = grk.relinearizes(loop).switch_to_level(2).to_host()[0]
    resp = F.dot_product(dots, selectors, dim2, grk, level=2).to_host()[0]
    assert (resp == loop).all()
    oexp = oracle.expands(opar, ogk, query, size)
    oout = None
    for i in range(dim2):
        d = oracle.dot_product_scalar(oexp[:dim1], [pts[k * dim2 + i] for k in range(dim1)])
        p = d.mul(oexp[dim1 + i])
        oout = p if oout is None else oout.add(p)
    assert (resp == ork.relinearizes(oout).switch_to_level(2).to_array()).all()
    dec = sk.decrypt(oracle.Ciphertext.from_array(opar, resp, 2))
    assert (dec == db[row * dim2 + col]).all()


def test_voting_tally_in_one_call(oracle, F):
    """examples/voting.rs:142-147: 1000 ballots under a collective key summed by one batch_sum give _sum_tree's words,
    and the collective decryption is the number of yes votes"""
    from test_gpu_mbfv import _sum_tree, keys
    degree, t, moduli = 4096, 4096, [0xffffee001, 0xffffc4001, 0x1ffffe0001]
    gpar = F.BfvParameters(degree, t, moduli=moduli, device=0)
    opar = oracle.BfvParameters(degree, t, moduli=moduli)
    rng = np.random.default_rng(1000)
    _, gsks = keys(oracle, F, opar, gpar, rng, 10)
    crp = F.mbfv.CommonRandomPoly.new(gpar)
    pk = F.mbfv.aggregate([F.mbfv.PublicKeyShare(g, crp) for g in gsks])
    votes = rng.integers(0, 2, size=1000, dtype=np.uint64)
    values = np.zeros(1000 * degree, np.uint64)
    values[::degree] = votes
    ballots = pk.try_encrypt(F.PlaintextVec.try_encode(values, F.Encoding.poly(), gpar))
    tally = ballots.sum()
    assert (tally.to_host() == _sum_tree(ballots).to_host()).all()
    pt = F.mbfv.aggregate([F.mbfv.DecryptionShare(g, tally) for g in gsks])
    got = pt.try_decode(F.Encoding.poly())
    assert int(got[0]) == int(votes.sum()) and not got[1:].any()


# ---- launches, errors, memory

def test_fewer_launches_and_transforms_than_the_loop(F):
    """a dot product of n terms launches fewer kernels than mul + (n - 1) adds + relinearize, and a batch sum one.
    Forward NTT rows (fhe_b200_ntt_row_count): with a key the dot product transforms the 2 parts of its group where the
    batched mul transforms the 3 parts of every term, 3Ln - 2L rows fewer; without a key 3 parts per group, 3L(n - 1)
    fewer.  Inverse rows: the relinearization's backward transform of c2 (L rows) is skipped.  Everything else (the
    product's own transforms, the key switch's digits) is the same in both routes."""
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    n = 16
    S = DotSetup(F, 1 << 13, 786433, [62, 62], 0, 0, 1, n, 4)
    L = len(S.moduli)

    def counts(fn):
        before = (lib.fhe_b200_launch_count(), lib.fhe_b200_ntt_row_count(0), lib.fhe_b200_ntt_row_count(1))
        fn()
        after = (lib.fhe_b200_launch_count(), lib.fhe_b200_ntt_row_count(0), lib.fhe_b200_ntt_row_count(1))
        return [a - b for a, b in zip(after, before)]

    def loop(relin):
        prods = S.A * S.B
        acc = prods.take(0, 1)
        for i in range(1, n):
            acc += prods.take(i, 1)
        return S.rk.relinearizes(acc) if relin else acc

    S.got(0)   # warm the scratch pool and tables
    dot, ref = counts(lambda: S.got(0)), counts(lambda: loop(True))
    assert ref[0] - dot[0] >= n - 1, (dot, ref)
    assert ref[1] - dot[1] == 3 * L * n - 2 * L, (dot, ref)
    assert ref[2] - dot[2] == L, (dot, ref)
    dot3, ref3 = counts(lambda: S.got(0, None)), counts(lambda: loop(False))
    assert ref3[1] - dot3[1] == 3 * L * (n - 1), (dot3, ref3)
    assert ref3[2] == dot3[2], (dot3, ref3)
    prods = S.A * S.B
    assert counts(lambda: prods.sum()) == [1, 0, 0]


def test_refusals_write_nothing_and_keep_no_memory(F):
    """every error of the new calls; the output words and device memory are unchanged by each refusal"""
    import ctypes as C
    import torch
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    degree = 1 << 13
    S = DotSetup(F, degree, 786433, [62, 62], 0, 0, 2, 3, 1)
    other = DotSetup(F, degree, 786433, [62, 62], 0, 0, 2, 3, 2)
    l1 = DotSetup(F, degree, 786433, [62, 62], 1, 1, 2, 3, 3, par=S.par)
    par = S.par
    out2, out3, out3_l1 = F.Ciphertext(par, 2, 2), F.Ciphertext(par, 2, 3), F.Ciphertext(par, 2, 3, 1)
    sum_out, sum_out3 = F.Ciphertext(par, 2, 2), F.Ciphertext(par, 2, 3)
    out_mb = F.Ciphertext(par, 2, 2, 0, mul_basis=True)
    sum_pb = F.Ciphertext(par, 2, 2, 0, _capi.POWER_BASIS)
    P = S.A.clone().into_power_basis()
    three = F.Ciphertext(par, 6, 3)
    sentinels = [(b, b.to_host()) for b in (out2, out3, out3_l1, sum_out, sum_pb, S.A, S.B)]
    bad, dot, dk, bs = _capi.INVALID_ARGUMENT, lib.fhe_b200_dot_product, lib.fhe_b200_dot_product_keyed, \
        lib.fhe_b200_batch_sum
    rk = S.rk.ksk._h

    def arr(hs):
        a = (C.c_void_p * max(1, len(hs)))(*[getattr(h, "value", h) for h in hs])
        return C.cast(a, C.POINTER(C.c_void_p))

    def u(v):
        return (C.c_uint32 * max(1, len(v)))(*v)
    cases = [
        ("sum null", lambda: bs(None, 3, 0, sum_out._h, None), bad),
        ("sum aliased", lambda: bs(S.A._h, 3, 0, S.A._h, None), bad),
        ("sum no terms", lambda: bs(S.A._h, 0, 0, sum_out._h, None), bad),
        ("sum counts", lambda: bs(S.A._h, 2, 0, sum_out._h, None), bad),
        ("sum parts", lambda: bs(S.A._h, 3, 0, sum_out3._h, None), _capi.BAD_POLY_COUNT),
        ("sum level", lambda: bs(l1.A._h, 3, 0, sum_out._h, None), _capi.INVALID_LEVEL),
        ("sum parameters", lambda: bs(other.A._h, 3, 0, sum_out._h, None), _capi.CONTEXT_MISMATCH),
        ("sum mul basis", lambda: bs(S.A._h, 3, 0, out_mb._h, None), _capi.CONTEXT_MISMATCH),
        ("sum accumulate repr", lambda: bs(S.A._h, 3, 1, sum_pb._h, None), _capi.INVALID_REPRESENTATION),
        ("dot null", lambda: dot(None, S.B._h, 3, rk, out2._h, None), bad),
        ("dot aliased", lambda: dot(S.A._h, S.B._h, 3, None, S.A._h, None), bad),
        ("dot no terms", lambda: dot(S.A._h, S.B._h, 0, rk, out2._h, None), bad),
        ("dot counts", lambda: dot(S.A._h, S.B._h, 2, rk, out2._h, None), bad),
        ("dot out parts", lambda: dot(S.A._h, S.B._h, 3, rk, out3._h, None), _capi.BAD_POLY_COUNT),
        ("dot out parts no key", lambda: dot(S.A._h, S.B._h, 3, None, out2._h, None), _capi.BAD_POLY_COUNT),
        ("dot operand parts", lambda: dot(three._h, S.B._h, 3, rk, out2._h, None), _capi.BAD_POLY_COUNT),
        ("dot levels differ", lambda: dot(S.A._h, l1.B._h, 3, None, out3._h, None), _capi.INVALID_LEVEL),
        ("dot out below", lambda: dot(l1.A._h, l1.B._h, 3, None, out3._h, None), _capi.INVALID_LEVEL),
        ("dot representation", lambda: dot(P._h, S.B._h, 3, rk, out2._h, None), _capi.INVALID_REPRESENTATION),
        ("dot parameters", lambda: dot(S.A._h, other.B._h, 3, rk, out2._h, None), _capi.CONTEXT_MISMATCH),
        ("dot key parameters", lambda: dot(S.A._h, S.B._h, 3, other.rk.ksk._h, out2._h, None),
         _capi.CONTEXT_MISMATCH),
        ("dot key level", lambda: dot(S.A._h, S.B._h, 3, l1.rk.ksk._h, out2._h, None), _capi.INVALID_LEVEL),
        ("keyed null list", lambda: dk(S.A._h, S.B._h, 3, None, 1, u([0, 0]), out2._h, None), bad),
        ("keyed no keys", lambda: dk(S.A._h, S.B._h, 3, arr([rk]), 0, u([0, 0]), out2._h, None), bad),
        ("keyed null index", lambda: dk(S.A._h, S.B._h, 3, arr([rk]), 1, None, out2._h, None), bad),
        ("keyed null key", lambda: dk(S.A._h, S.B._h, 3, arr([rk, None]), 2, u([0, 0]), out2._h, None), bad),
        ("keyed index beyond", lambda: dk(S.A._h, S.B._h, 3, arr([rk]), 1, u([0, 1]), out2._h, None), bad),
        ("keyed key level", lambda: dk(S.A._h, S.B._h, 3, arr([rk, l1.rk.ksk._h]), 2, u([0, 1]), out2._h, None),
         _capi.INVALID_LEVEL),
    ]
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for what, call, code in cases:
        got = call()
        assert got == code, (what, got, lib.fhe_b200_last_error())
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 4 << 20
    for b, words in sentinels:
        assert (b.to_host() == words).all()


def test_cpp_mirror(F, tmp_path):
    """the C++ mirror's batch_sum, dot_product and dot_product_keyed give the Python mirror's words"""
    S = DotSetup(F, 64, 1153, [62] * 3, 0, 0, 3, 4, 12, shared="b")
    rng = np.random.default_rng(13)
    c = rand_rows(rng, S.moduli, (2, 3), 64)
    rk2 = F.RelinearizationKey.from_arrays(S.par, c[0], c[1])
    index = [1, 0, 1]
    lines = ["%d %d %d %d %d" % (64, 1153, len(S.moduli), 3, 4), " ".join(map(str, S.moduli)),
             " ".join(map(str, index))]
    (tmp_path / "args.txt").write_text("\n".join(lines) + "\n")
    S.A.to_host().tofile(str(tmp_path / "a.bin"))
    S.B.to_host().tofile(str(tmp_path / "b.bin"))
    for k, rk in enumerate((S.rk, rk2)):
        c0, c1 = rk.ksk.arrays()
        c0.tofile(str(tmp_path / ("k%d_c0.bin" % k)))
        c1.tofile(str(tmp_path / ("k%d_c1.bin" % k)))
    exe = str(tmp_path / "dot_product_test")
    lib_dir = os.path.join(ROOT, "fhe_rs_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "dot_product_test.cpp"), "-o", exe,
                           "-L", lib_dir, "-lfhe_b200", "-Wl,-rpath," + lib_dir])
    out = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
    want = {"sum": S.A.sum(4).to_host(), "dot": F.dot_product(S.A, S.B, 4, S.rk, 1).to_host(),
            "dot3": F.dot_product(S.A, S.B, 4).to_host(),
            "keyed": F.dot_product_keyed(S.A, S.B, 4, [S.rk, rk2], index).to_host()}
    for name, w in want.items():
        assert (np.fromfile(str(tmp_path / ("out_%s.bin" % name)), np.uint64) == w.ravel()).all(), name


SWITCHES = {"tma": {"FHE_B200_KSMAC": "tma"}, "classic": {"FHE_B200_KSMAC": "classic"},
            "scaler": {"FHE_B200_SCALER": "classic"}, "ntt_fast": {"FHE_B200_NTT": "fast"},
            "ntt_tma": {"FHE_B200_NTT": "tma"}, "no_fusion": {"FHE_B200_NO_TENSOR_FUSION": "1"},
            "chunk1": {"FHE_B200_CHUNK": "1"}, "chunk2": {"FHE_B200_CHUNK": "2"}, "chunk4": {"FHE_B200_CHUNK": "4"},
            "streams1": {"FHE_B200_STREAMS": "1"}, "streams2": {"FHE_B200_STREAMS": "2"},
            "streams4": {"FHE_B200_STREAMS": "4"}}


def test_switch_reruns():
    """the probe's word checks under each kernel and chunking switch, one process per switch, side by side"""
    procs, fails = {}, {}
    try:
        for name, env in SWITCHES.items():
            e = dict(os.environ, **env)
            procs[name] = subprocess.Popen([sys.executable, os.path.join(TESTS, "dot_product_chunk_probe.py")],
                                           cwd=ROOT, env=e, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        for name, p in procs.items():
            out, _ = p.communicate(timeout=1800)
            if p.returncode != 0 or "WORD CHECKS OK" not in out:
                fails[name] = out[-3000:]
    finally:   # a timeout or a failed start leaves no process behind
        for p in procs.values():
            if p.poll() is None:
                p.kill()
                p.wait()
    assert not fails, fails

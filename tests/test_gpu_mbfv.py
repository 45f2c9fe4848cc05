"""GPU tests of multiparty BFV on the device (fhe::mbfv): for the same seeds every share and aggregate equals
tests/mbfv_reference.py's restatement on the oracle word for word; the reference's protocol tests and its `voting`
example run with device objects only; the aggregation sum against numpy, the from_shares lift in the band
q_0 / 2 < t < q_0, the error codes, chunking and the NTT switches.  Run with `-m gpu`."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import edge_inputs as E
import encrypt_reference as R
import mbfv_reference as M

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VAR = 10


@pytest.fixture(scope="module")
def F():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


# name -> (degree, t or None for a 40-bit prime, moduli sizes or an edge_inputs.CLIENT_SHAPES name)
SHAPES = {
    "n16": (16, 1153, [62, 62, 62]),
    "setA": (1 << 12, 1032193, [62, 62]),
    "mixed": (1 << 13, None, [62, 30, 50]),
    "q0_barrett": (1 << 13, 786433, "q0_barrett"),
    "q0_above_2_61": (1 << 13, 786433, "q0_above_2_61"),
    "q0_solinas_max_c": (1 << 13, 786433, "q0_solinas_max_c"),
    "q1_barrett": (1 << 13, 786433, "q1_barrett"),
    "setC": (1 << 15, 786433, [62] * 14),
    "n2_16": (1 << 16, 786433, [62] * 3),
}
BIG = {"setC", "n2_16"}


def params(oracle, F, name):
    degree, t, spec = SHAPES[name]
    if t is None:
        t = oracle.generate_prime(40, 2 * degree, 1 << 40)
    moduli = E.client_moduli(spec) if isinstance(spec, str) else oracle.BfvParameters.generate_moduli(spec, degree)
    return oracle.BfvParameters(degree, t, moduli=moduli), F.BfvParameters(degree, t, moduli=moduli, device=0)


def seed_of(rng):
    return rng.integers(0, 256, size=32, dtype=np.uint8).tobytes()


def keys(oracle, F, opar, gpar, rng, n):
    osks = [oracle.SecretKey(opar, rng) for _ in range(n)]
    return osks, [F.SecretKey(gpar, o.coeffs) for o in osks]


def upload(F, gpar, cts, level):
    return F.Ciphertext.from_host(gpar, np.stack([c.to_array() for c in cts]), level)


@pytest.mark.parametrize("name", list(SHAPES))
def test_mbfv_parity(oracle, F, name):
    """CRPs, public key shares and their aggregate, decryption / secret-key-switch / public-key-switch shares and their
    aggregates at every level (one ciphertext per level at the large shapes) equal the restatement word for word"""
    opar, gpar = params(oracle, F, name)
    rng = np.random.default_rng(opar.degree + len(opar.moduli))
    big = name in BIG
    P, last, n = 3, len(opar.moduli) - 1, opar.degree
    osks, gsks = keys(oracle, F, opar, gpar, rng, P)
    # CommonRandomPoly::new_vec and new_leveled
    seed = seed_of(rng)
    crps = F.mbfv.CommonRandomPoly.new_vec(gpar, seed)
    ocrps = M.crp(opar, seed, len(opar.moduli))
    for g, o in zip(crps, ocrps):
        assert (g.batch.to_host()[0, 0] == o.c).all()
    seed = seed_of(rng)
    assert (F.mbfv.CommonRandomPoly.new_leveled(gpar, last, seed).batch.to_host()[0, 0] == M.crp(opar, seed, 1, last)[0].c).all()
    # PublicKeyShare and PublicKey::from_shares
    ss = [seed_of(rng) for _ in range(P)]
    gsh = [F.mbfv.PublicKeyShare(g, crps[0], s) for g, s in zip(gsks, ss)]
    osh = [M.pk_share(o, [ocrps[0]], s, VAR)[0] for o, s in zip(osks, ss)]
    for g, o in zip(gsh, osh):
        assert (g.p0_share.to_host()[0, 0] == o.c).all()
    gpk = F.mbfv.aggregate(gsh)
    opk = M.pk_aggregate(opar, osh, ocrps[0])
    assert (gpk.c.to_host()[0] == opk.to_array()).all()
    outs_o, outs_g = osks[1:] + osks[:1], gsks[1:] + gsks[:1]
    levels = range(last + 1)
    count = 1 if big else 2
    for level in levels:
        values = rng.integers(0, opar.plaintext, size=count * n, dtype=np.uint64)
        ms = [R.to_poly(opar, values[k * n:(k + 1) * n], level) for k in range(count)]
        octs = R.encrypt_pk(opar, opk, seed_of(rng), count, level, VAR, ms)
        ct = upload(F, gpar, octs, level)
        # DecryptionShare and Plaintext::from_shares
        ss = [seed_of(rng) for _ in range(P)]
        gd = [F.mbfv.DecryptionShare(g, ct, s) for g, s in zip(gsks, ss)]
        od = [M.sks_share(o, None, octs, s, VAR) for o, s in zip(osks, ss)]
        for g, o in zip(gd, od):
            got = g.h_share.to_host()
            assert all((got[k, 0] == o[k].c).all() for k in range(count)), level
        pts = F.mbfv.Aggregate.from_shares(F.PlaintextVec, gd)
        if count == 1:
            assert type(F.mbfv.Aggregate.from_shares(F.Plaintext, gd)) is F.Plaintext
        got = pts.batch.to_host()
        for k in range(count):
            exp, w = M.from_shares(octs[k], [o[k] for o in od])
            assert (got[k, 0] == exp.c).all() and (w == values[k * n:(k + 1) * n]).all(), (level, k)
        assert (pts.try_decode(F.Encoding.poly_at_level(level)) == values).all()
        # SecretKeySwitchShare to the rotated keys and Ciphertext::from_shares
        ss = [seed_of(rng) for _ in range(P)]
        gs = [F.mbfv.SecretKeySwitchShare(g, go, ct, s) for g, go, s in zip(gsks, outs_g, ss)]
        os_ = [M.sks_share(o, oo, octs, s, VAR) for o, oo, s in zip(osks, outs_o, ss)]
        for g, o in zip(gs, os_):
            got = g.h_share.to_host()
            assert all((got[k, 0] == o[k].c).all() for k in range(count)), level
        got = F.mbfv.aggregate(gs).to_host()
        for k in range(count):
            assert (got[k] == M.sks_aggregate(octs[k], [o[k] for o in os_]).to_array()).all(), (level, k)
        # PublicKeySwitchShare to the aggregated key and Ciphertext::from_shares
        ss = [seed_of(rng) for _ in range(P)]
        gp = [F.mbfv.PublicKeySwitchShare(g, gpk, ct, s) for g, s in zip(gsks, ss)]
        op = [M.pks_share(o, opk, octs, s, VAR) for o, s in zip(osks, ss)]
        for g, o in zip(gp, op):
            got = g.h_share.to_host()
            assert all((got[k] == o[k].to_array()).all() for k in range(count)), level
        got = F.mbfv.Aggregate.from_shares(F.Ciphertext, gp).to_host()
        for k in range(count):
            assert (got[k] == M.pks_aggregate(octs[k], [o[k] for o in op]).to_array()).all(), (level, k)


def summed_key(F, gpar, osks):
    return F.SecretKey(gpar, np.sum([o.coeffs for o in osks], axis=0).astype(np.int64))


@pytest.mark.parametrize("n_parties", [5, 11])
def test_protocols_with_device_objects(oracle, F, n_parties):
    """the reference's protocol tests with device objects only, at every level: the aggregated public key encrypts for
    SecretKey(sum s_i); collective decryption; secret and public key switches followed by decryption"""
    opar, gpar = params(oracle, F, "setA" if n_parties == 5 else "n16")
    rng = np.random.default_rng(40 + n_parties)
    n, last = opar.degree, len(opar.moduli) - 1
    osks, gsks = keys(oracle, F, opar, gpar, rng, n_parties)
    crp = F.mbfv.CommonRandomPoly.new(gpar)
    pk = F.mbfv.aggregate([F.mbfv.PublicKeyShare(g, crp) for g in gsks])
    ssum = summed_key(F, gpar, osks)
    _, outs = keys(oracle, F, opar, gpar, rng, n_parties)
    out_sk = F.SecretKey(gpar, oracle.SecretKey(opar, rng).coeffs)
    out_pk = F.PublicKey.new(out_sk)
    for level in range(last + 1):
        enc = F.Encoding.poly_at_level(level)
        values = rng.integers(0, opar.plaintext, size=3 * n, dtype=np.uint64)
        ct = pk.try_encrypt(F.PlaintextVec.try_encode(values, enc, gpar))
        assert (ssum.try_decrypt(ct).try_decode(enc) == values).all()                      # protocol_creates_valid_pk
        pts = F.mbfv.aggregate([F.mbfv.DecryptionShare(g, ct) for g in gsks])              # encrypt_decrypt
        assert (pts.try_decode(enc) == values).all()
        ct2 = F.mbfv.aggregate([F.mbfv.SecretKeySwitchShare(g, o, ct) for g, o in zip(gsks, outs)])
        assert (F.mbfv.aggregate([F.mbfv.DecryptionShare(o, ct2) for o in outs]).try_decode(enc) == values).all()
        ct3 = F.mbfv.aggregate([F.mbfv.PublicKeySwitchShare(g, out_pk, ct) for g in gsks])
        assert (out_sk.try_decrypt(ct3).try_decode(enc) == values).all()
        # collective_keys_enable_homomorphic_addition
        ct4 = ct + ct
        exp = (values * 2) % opar.plaintext
        assert (F.mbfv.aggregate([F.mbfv.DecryptionShare(g, ct4) for g in gsks]).try_decode(enc) == exp).all()


def _sum_tree(batch):
    """the sum of the ciphertexts of a batch, by halving"""
    while batch.count > 1:
        h = batch.count // 2
        a = batch.take(0, h)
        a += batch.take(h, h)
        batch = a if batch.count % 2 == 0 else _concat(a, batch.take(2 * h, 1))
    return batch


def _concat(a, b):
    import fhe_rs_b200 as F
    words = np.concatenate([a.to_host(), b.to_host()])
    return F.Ciphertext.from_host(a.par, words, a.level)


def test_voting_example(oracle, F):
    """examples/voting.rs: N = 4096, t = 4096, three moduli, 10 parties, 1000 votes encrypted under the collective key
    and summed; the collective decryption of the tally is the number of yes votes"""
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
    tally = _sum_tree(ballots)
    pt = F.mbfv.aggregate([F.mbfv.DecryptionShare(g, tally) for g in gsks])
    got = pt.try_decode(F.Encoding.poly())
    assert int(got[0]) == int(votes.sum()) and not got[1:].any()


def band(oracle, F):
    q0 = oracle.generate_prime(30, 32, 1 << 30)
    moduli = [q0] + oracle.BfvParameters.generate_moduli([62], 16)
    return (oracle.BfvParameters(16, q0 - 2, moduli=moduli), F.BfvParameters(16, q0 - 2, moduli=moduli, device=0))


def test_from_shares_against_try_decrypt_in_the_band(oracle, F):
    """q_0 / 2 < t < q_0 with two plaintext-context moduli: the device's from_shares gives the values and the
    restatement's words, the device's try_decrypt the oracle's ((v + t) mod q_0) mod t, and the two differ"""
    opar, gpar = band(oracle, F)
    t, q0 = opar.plaintext, opar.moduli[0]
    rng = np.random.default_rng(77)
    osks, gsks = keys(oracle, F, opar, gpar, rng, 2)
    values = np.array([0, 1, 2, 3, t - 1, t - 2, t // 2, t // 2 + 1, 5, t // 2 - 1, 9, 10, 11, 12, 13, 14],
                      dtype=np.uint64)
    enc = F.Encoding.poly()
    ct = F.mbfv.aggregate([F.mbfv.PublicKeyShare(g, F.mbfv.CommonRandomPoly.new(gpar)) for g in gsks[:1]]) \
        .try_encrypt(F.PlaintextVec.try_encode(values, enc, gpar))
    one = F.SecretKey(gpar, osks[0].coeffs)
    seed = seed_of(rng)
    d = F.mbfv.DecryptionShare(one, ct, seed)
    pts = F.mbfv.aggregate([d])
    assert (pts.try_decode(enc) == values).all()
    oct_ = oracle.Ciphertext.from_array(opar, ct.to_host()[0], 0)
    exp, _ = M.from_shares(oct_, M.sks_share(osks[0], None, [oct_], seed, VAR))
    assert (pts.batch.to_host()[0, 0] == exp.c).all()
    direct = one.try_decrypt(ct).try_decode(enc)
    assert (direct == osks[0].decrypt(oct_)).all()
    centred = [v if v <= t // 2 else v - t for v in values.tolist()]
    assert (direct != values).sum() == sum(1 for v in centred if v >= q0 - t) > 0


@pytest.mark.parametrize("n,first_max", [(1, False), (1, True), (2, False), (64, False), (65, True)])
def test_shares_sum_against_numpy(oracle, F, n, first_max):
    """fhe_b200_shares_sum at set C against a numpy sum modulo each q: random shares and shares holding q - 1 in every
    word (every other share, starting with share 0 when first_max); 65 shares take two launches.  The output may be
    any of the shares, also one past the first launch's 64"""
    from fhe_rs_b200 import _capi
    opar, gpar = params(oracle, F, "setC")
    rng = np.random.default_rng(n)
    q = np.array(opar.moduli, dtype=np.uint64)[:, None]
    words = []
    for i in range(n):
        w = (q - np.uint64(1)) * np.ones((14, opar.degree), np.uint64) if (i % 2) != first_max else \
            rng.integers(0, 1 << 62, size=(14, opar.degree), dtype=np.uint64) % q
        words.append(w)
    shares = [F.Ciphertext.from_host(gpar, w[None, None]) for w in words]
    out = F.Ciphertext(gpar, 1, 1, 0)
    hs = (C.c_void_p * n)(*[s._h for s in shares])
    _capi.check(_capi.lib().fhe_b200_shares_sum(hs, n, out._h, None))
    acc = np.zeros((14, opar.degree), np.uint64)
    for w in words:
        acc = (acc + w) % q
    assert (out.to_host()[0, 0] == acc).all()
    # out may be one of the shares: the last one (past the first launch when n = 65), then the first
    for k in (n - 1, 0):
        _capi.check(_capi.lib().fhe_b200_shares_sum(hs, n, shares[k]._h, None))
        assert (shares[k].to_host()[0, 0] == acc).all(), k
        shares[k].upload(words[k][None, None])


def test_errors_and_memory(oracle, F):
    import torch
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    opar, gpar = params(oracle, F, "n16")
    rng = np.random.default_rng(5)
    osks, gsks = keys(oracle, F, opar, gpar, rng, 2)
    other = F.BfvParameters(16, 1153, moduli=opar.moduli, device=0)
    osk_other = F.SecretKey(other, osks[0].coeffs)
    seed = bytes(32)
    sk = gsks[0]._h
    crp0 = F.mbfv.CommonRandomPoly.new(gpar, seed).batch
    crp1 = F.mbfv.CommonRandomPoly.new_leveled(gpar, 1, seed).batch
    ct = F.mbfv.aggregate([F.mbfv.PublicKeyShare(gsks[0], F.mbfv.CommonRandomPoly(crp0))]).try_encrypt(count=2)
    ct3 = F.Ciphertext(gpar, 2, 3, 0)
    one = F.Ciphertext(gpar, 2, 1, 0)
    two = F.Ciphertext(gpar, 2, 2, 0)
    pk = F.mbfv.aggregate([F.mbfv.PublicKeyShare(gsks[0], F.mbfv.CommonRandomPoly(crp0))]).c
    pk1 = F.Ciphertext(gpar, 1, 2, 1)
    hs = lambda *b: (C.c_void_p * len(b))(*[x._h for x in b])  # noqa: E731
    out1 = F.Ciphertext(gpar, 1, 1, 0)
    cases = [
        (_capi.INVALID_ARGUMENT, lambda: lib.fhe_b200_pk_share(sk, crp0._h, 0, seed, out1._h, None)),   # variance
        (_capi.INVALID_ARGUMENT, lambda: lib.fhe_b200_pk_share(sk, crp0._h, 33, seed, out1._h, None)),
        (_capi.INVALID_LEVEL, lambda: lib.fhe_b200_pk_share(sk, crp1._h, VAR, seed, out1._h, None)),
        (_capi.CONTEXT_MISMATCH, lambda: lib.fhe_b200_pk_share(osk_other._h, crp0._h, VAR, seed, out1._h, None)),
        (_capi.INVALID_ARGUMENT, lambda: lib.fhe_b200_pk_share(sk, crp0._h, VAR, seed, one._h, None)),
        (_capi.INVALID_ARGUMENT, lambda: lib.fhe_b200_pk_aggregate(hs(), 0, crp0._h, pk._h, None)),          # NoShares
        (_capi.INVALID_LEVEL, lambda: lib.fhe_b200_pk_aggregate(hs(out1), 1, crp1._h, pk._h, None)),
        (_capi.INVALID_ARGUMENT, lambda: lib.fhe_b200_pk_aggregate(hs(out1, one), 2, crp0._h, pk._h, None)),  # shape
        (_capi.INVALID_ARGUMENT, lambda: lib.fhe_b200_shares_sum(hs(), 0, one._h, None)),
        (_capi.INVALID_ARGUMENT, lambda: lib.fhe_b200_shares_sum(hs(one, two), 2, one._h, None)),
        (_capi.BAD_POLY_COUNT, lambda: lib.fhe_b200_sks_share(sk, None, ct3._h, VAR, seed, one._h, None)),
        (_capi.CONTEXT_MISMATCH, lambda: lib.fhe_b200_sks_share(sk, osk_other._h, ct._h, VAR, seed, one._h, None)),
        (_capi.INVALID_ARGUMENT, lambda: lib.fhe_b200_sks_share(sk, None, ct._h, VAR, seed, two._h, None)),
        (_capi.INVALID_ARGUMENT, lambda: lib.fhe_b200_sks_aggregate(ct._h, hs(), 0, two._h, None)),
        (_capi.BAD_POLY_COUNT, lambda: lib.fhe_b200_sks_aggregate(ct3._h, hs(one), 1, two._h, None)),
        (_capi.INVALID_ARGUMENT, lambda: lib.fhe_b200_sks_aggregate(ct._h, hs(two), 1, two._h, None)),
        (_capi.INVALID_LEVEL, lambda: lib.fhe_b200_pks_share(sk, pk1._h, ct._h, VAR, seed, two._h, None)),
        (_capi.BAD_POLY_COUNT, lambda: lib.fhe_b200_pks_share(sk, pk._h, ct3._h, VAR, seed, two._h, None)),
        (_capi.CONTEXT_MISMATCH, lambda: lib.fhe_b200_pks_share(osk_other._h, pk._h, ct._h, VAR, seed, two._h, None)),
        (_capi.INVALID_ARGUMENT, lambda: lib.fhe_b200_pks_aggregate(ct._h, hs(one), 1, two._h, None)),
        (_capi.INVALID_ARGUMENT, lambda: lib.fhe_b200_decryption_aggregate(gpar.encoder(), ct._h, hs(), 0, one._h, None)),
        (_capi.CONTEXT_MISMATCH, lambda: lib.fhe_b200_decryption_aggregate(other.encoder(), ct._h, hs(one), 1, one._h, None)),
        (_capi.INVALID_ARGUMENT, lambda: lib.fhe_b200_decryption_aggregate(gpar.encoder(), ct._h, hs(one), 1, two._h, None)),
        (_capi.INVALID_ARGUMENT, lambda: lib.fhe_b200_crp_generate(gpar._h, seed, two._h, None)),
    ]
    for code, call in cases:
        assert call() == code, (code, lib.fhe_b200_last_error())
    pb = F.Ciphertext(gpar, 2, 1, 0, F.POWER_BASIS)
    assert lib.fhe_b200_decryption_aggregate(gpar.encoder(), ct._h, hs(pb), 1, one._h, None) == _capi.INVALID_REPRESENTATION
    # t >= q_0: UNSUPPORTED
    big_t = F.BfvParameters(16, opar.moduli[0] + 2, moduli=opar.moduli, device=0)
    b_ct, b_one = F.Ciphertext(big_t, 1, 2, 0), F.Ciphertext(big_t, 1, 1, 0)
    assert lib.fhe_b200_decryption_aggregate(big_t.encoder(), b_ct._h, hs(b_one), 1, b_one._h, None) == _capi.UNSUPPORTED
    with pytest.raises(F.FheError):
        F.mbfv.Aggregate.from_shares(F.PublicKey, [F.mbfv.DecryptionShare(gsks[0], ct)])
    # refused calls and dropped shares keep no device memory (set A: every share batch holds 64 KB x parts x count)
    a_opar, a_gpar = params(oracle, F, "setA")
    a_osks, a_gsks = keys(oracle, F, a_opar, a_gpar, rng, 2)
    a_ct = a_gsks[0].try_encrypt(count=64)

    def cycle():
        d = [F.mbfv.DecryptionShare(g, a_ct) for g in a_gsks]
        F.mbfv.aggregate(d)
        F.mbfv.aggregate([F.mbfv.PublicKeySwitchShare(g, F.PublicKey.new(a_gsks[0]), a_ct) for g in a_gsks])
        for v in (0, 33):
            assert lib.fhe_b200_sks_share(a_gsks[0]._h, None, a_ct._h, v, seed, d[0].h_share._h, None) == _capi.INVALID_ARGUMENT
        torch.cuda.synchronize()
    cycle()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(5):
        cycle()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 8 << 20


@pytest.mark.parametrize("name", ["n16", "setC"])
def test_rkg_parity(oracle, F, name):
    """RelinKeyGenerator on 3 and 14 limbs: round-1 shares, their aggregate, round-2 shares and the aggregated key's
    words equal the restatement; the key is an ordinary relinearization key"""
    opar, gpar = params(oracle, F, name)
    rng = np.random.default_rng(3 * opar.degree + 1)
    P, L = 3, len(opar.moduli)
    osks, gsks = keys(oracle, F, opar, gpar, rng, P)
    seed = seed_of(rng)
    crps = F.mbfv.CommonRandomPoly.new_vec(gpar, seed)
    ocrps = M.crp(opar, seed, L)
    su, s1, s2 = ([seed_of(rng) for _ in range(P)] for _ in range(3))
    gens = [F.mbfv.RelinKeyGenerator(g, crps, x) for g, x in zip(gsks, su)]
    us = [M.rkg_u(opar, x, VAR) for x in su]
    g1 = [g.round_1(x) for g, x in zip(gens, s1)]
    o1 = [M.rkg_round1(o, ocrps, u, x, VAR) for o, u, x in zip(osks, us, s1)]
    for g, o in zip(g1, o1):
        assert (g.h0.to_host()[:, 0] == np.stack([p.c for p in o[0]])).all()
        assert (g.h1.to_host()[:, 0] == np.stack([p.c for p in o[1]])).all()
    gr1 = F.mbfv.aggregate(g1)
    or1 = M.rkg_r1_aggregate(o1)
    assert gr1.round == "R1Aggregated"
    assert (gr1.h0.to_host()[:, 0] == np.stack([p.c for p in or1[0]])).all()
    assert (gr1.h1.to_host()[:, 0] == np.stack([p.c for p in or1[1]])).all()
    g2 = [g.round_2(gr1, x) for g, x in zip(gens, s2)]
    o2 = [M.rkg_round2(o, u, or1[0], or1[1], x, VAR) for o, u, x in zip(osks, us, s2)]
    for g, o in zip(g2, o2):
        assert (g.h0.to_host()[:, 0] == np.stack([p.c for p in o[0]])).all()
        assert (g.h1.to_host()[:, 0] == np.stack([p.c for p in o[1]])).all()
    rk = F.mbfv.Aggregate.from_shares(F.RelinearizationKey, g2)
    c0, c1 = M.rkg_aggregate(o2, or1[1])
    got0, got1 = rk.ksk.arrays()
    assert (got0 == c0).all() and (got1 == c1).all()
    # the device relinearizes with it as the oracle does with the same words
    ork = oracle.RelinearizationKey.from_ksk(oracle.KeySwitchingKey.from_arrays(opar, c0, c1))
    ct3 = np.stack([rng.integers(0, 1 << 62, size=(3, L, opar.degree), dtype=np.uint64)
                    % np.array(opar.moduli, dtype=np.uint64)[None, :, None]])
    exp = ork.relinearizes(oracle.Ciphertext.from_array(opar, ct3[0], 0))
    assert (rk.relinearizes(F.Ciphertext.from_host(gpar, ct3)).to_host()[0] == exp.to_array()).all()


@pytest.mark.parametrize("name", ["setA", "n16"])
def test_collective_relin_key_multiplies(oracle, F, name):
    """relin_key_gen.rs relinearization_works with device objects only: the collective key feeds mul_relin with mod
    switching (Multiplicator::default + enable_mod_switching) and the product decrypts collectively to the slot-wise
    product"""
    opar, gpar = params(oracle, F, name)
    rng = np.random.default_rng(91)
    n, t = opar.degree, opar.plaintext
    _, gsks = keys(oracle, F, opar, gpar, rng, 5)
    pk = F.mbfv.aggregate([F.mbfv.PublicKeyShare(g, F.mbfv.CommonRandomPoly.new(gpar, b"k" * 32)) for g in gsks])
    crps = F.mbfv.CommonRandomPoly.new_vec(gpar)
    gens = [F.mbfv.RelinKeyGenerator(g, crps) for g in gsks]
    r1 = F.mbfv.aggregate([g.round_1() for g in gens])
    rk = F.mbfv.aggregate([g.round_2(r1) for g in gens])
    v1, v2 = (rng.integers(0, t, size=4 * n, dtype=np.uint64) for _ in range(2))
    enc = F.Encoding.simd()
    a, b = (pk.try_encrypt(F.PlaintextVec.try_encode(v, enc, gpar)) for v in (v1, v2))
    m = F.Multiplicator.default(rk)
    m.enable_mod_switching()
    ct = m.multiply(a, b)
    assert ct.level == 1 and len(ct) == 2
    got = F.mbfv.aggregate([F.mbfv.DecryptionShare(g, ct) for g in gsks]).try_decode(F.Encoding.simd_at_level(1))
    assert (got == (v1 * v2) % np.uint64(t)).all()


def test_rkg_errors_and_memory(oracle, F):
    """the generator's refusals, and no device memory kept after rkg_free (set A: u, the shares and the key)"""
    import torch
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    seed = bytes(32)
    one_par = F.BfvParameters(16, 1153, moduli=oracle.BfvParameters.generate_moduli([62], 16), device=0)
    one_sk = F.SecretKey(one_par, np.zeros(16, np.int64))
    one_crp = F.mbfv.CommonRandomPoly._generate(one_par, 1, 0, seed)
    h = C.c_void_p()
    assert lib.fhe_b200_rkg_create(one_sk._h, one_crp._h, VAR, seed, C.byref(h), None) == _capi.UNSUPPORTED
    opar, gpar = params(oracle, F, "setA")
    rng = np.random.default_rng(8)
    _, gsks = keys(oracle, F, opar, gpar, rng, 2)
    short = F.mbfv.CommonRandomPoly._generate(gpar, 1, 0, seed)
    leveled = F.mbfv.CommonRandomPoly._generate(gpar, 2, 1, seed)
    assert lib.fhe_b200_rkg_create(gsks[0]._h, short._h, VAR, seed, C.byref(h), None) == _capi.INVALID_ARGUMENT
    assert b"InvalidCommonRandomPolynomialCount" in lib.fhe_b200_last_error()
    assert lib.fhe_b200_rkg_create(gsks[0]._h, leveled._h, VAR, seed, C.byref(h), None) == _capi.INVALID_LEVEL
    with pytest.raises(F.FheError):
        F.mbfv.RelinKeyGenerator(gsks[0], [F.mbfv.CommonRandomPoly(short)])
    crps = F.mbfv.CommonRandomPoly.new_vec(gpar)
    gen = F.mbfv.RelinKeyGenerator(gsks[0], crps)
    with pytest.raises(F.FheError):
        gen.round_2(gen.round_1())                       # round 2 takes the round-1 aggregate
    wrong = F.Ciphertext(gpar, 3, 1, 0)
    assert lib.fhe_b200_rkg_round1(gen._h, seed, wrong._h, wrong._h, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_rkg_aggregate(None, None, 0, gen.round_1().h1._h, C.byref(h), None) == _capi.INVALID_ARGUMENT
    del gen

    def cycle():
        gens = [F.mbfv.RelinKeyGenerator(g, crps) for g in gsks]
        r1 = F.mbfv.aggregate([g.round_1() for g in gens])
        F.mbfv.aggregate([g.round_2(r1) for g in gens])
        torch.cuda.synchronize()
    cycle()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(5):
        cycle()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 4 << 20


@pytest.mark.parametrize("streams", ["1", "2", "4"])
def test_mbfv_chunking(streams):
    """every call over several chunks on 1, 2 and 4 streams gives the words of the whole call"""
    env = dict(os.environ, FHE_B200_CHUNK="3", FHE_B200_STREAMS=streams)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "mbfv_chunk_probe.py")], env=env,
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "mbfv chunk probe ok" in out.stdout, out.stdout + out.stderr


@pytest.mark.parametrize("env", [{"FHE_B200_NTT": "fast"}, {"FHE_B200_GENERIC_NTT": "1"}],
                         ids=lambda e: ",".join("%s=%s" % kv for kv in e.items()))
def test_alternate_code_paths(F, env):
    """the same words under the other NTT implementations"""
    out = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "tests/test_gpu_mbfv.py",
                          "-k", "test_mbfv_parity and (n16 or setA or mixed or q0_barrett) or test_voting_example or "
                          "test_rkg_parity and n16",
                          "-p", "no:cacheprovider"],
                         cwd=ROOT, env=dict(os.environ, **env), capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stdout[-4000:] + out.stderr[-4000:]


def test_cpp_mbfv(tmp_path, oracle, F):
    """tests/cpp/mbfv_test.cpp: every mbfv object made through the mbfv namespace of include/fhe_b200.hpp has the
    words the Python mirror makes from the same seeds"""
    from fhe_rs_b200 import wire
    opar, gpar = params(oracle, F, "setA")
    rng = np.random.default_rng(12)
    n, count = opar.degree, 3
    osks, gsks = keys(oracle, F, opar, gpar, rng, 2)
    seeds = [seed_of(rng) for _ in range(15)]
    ct = gsks[0].try_encrypt(count=count)
    for k, o in enumerate(osks):
        (tmp_path / ("sk%d.bin" % k)).write_bytes(wire.encode_secret_key([int(c) for c in o.coeffs]))
    (tmp_path / "seeds.bin").write_bytes(b"".join(seeds))
    np.array(opar.moduli, np.uint64).tofile(str(tmp_path / "moduli.bin"))
    ct.to_host().tofile(str(tmp_path / "ct.bin"))
    exe = str(tmp_path / "mbfv_test")
    lib_dir = os.path.join(ROOT, "fhe_rs_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "mbfv_test.cpp"), "-o", exe,
                           "-L", lib_dir, "-lfhe_b200", "-Wl,-rpath," + lib_dir])
    out = subprocess.run([exe, str(n), str(opar.plaintext), str(count), str(tmp_path)], capture_output=True, text=True,
                         timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
    got = lambda name: np.fromfile(str(tmp_path / name), np.uint64)  # noqa: E731
    s = iter(seeds)
    crps = F.mbfv.CommonRandomPoly.new_vec(gpar, next(s))
    assert (got("crp.bin") == np.concatenate([c.batch.to_host().ravel() for c in crps])).all()
    pk = F.mbfv.aggregate([F.mbfv.PublicKeyShare(g, crps[0], next(s)) for g in gsks])
    assert (got("pk.bin") == pk.c.to_host().ravel()).all()
    dec = F.mbfv.aggregate([F.mbfv.DecryptionShare(g, ct, next(s)) for g in gsks])
    assert (got("dec.bin") == dec.batch.to_host().ravel()).all()
    sks = F.mbfv.aggregate([F.mbfv.SecretKeySwitchShare(gsks[0], gsks[1], ct, next(s)),
                            F.mbfv.SecretKeySwitchShare(gsks[1], gsks[0], ct, next(s))])
    assert (got("sks.bin") == sks.to_host().ravel()).all()
    pks = F.mbfv.aggregate([F.mbfv.PublicKeySwitchShare(g, pk, ct, next(s)) for g in gsks])
    assert (got("pks.bin") == pks.to_host().ravel()).all()
    gens = [F.mbfv.RelinKeyGenerator(g, crps, next(s)) for g in gsks]
    r1 = F.mbfv.aggregate([g.round_1(next(s)) for g in gens])
    assert (got("r1.bin") == np.concatenate([r1.h0.to_host().ravel(), r1.h1.to_host().ravel()])).all()
    c0, c1 = F.mbfv.aggregate([g.round_2(r1, next(s)) for g in gens]).ksk.arrays()
    assert (got("rk.bin") == np.concatenate([c0.ravel(), c1.ravel()])).all()

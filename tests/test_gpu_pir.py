"""SealPIR on the device (fhe_b200_transcode, fhe_b200_fold, the EvaluationKey message), bit-exact against the oracle's
restatement in tests/pir_reference.py:

  * the transcoder at every (in, out) width pair in 1..64 x 1..64 on rows of random lengths (0 and 1 included) with
    strides, truncation and padding; byte input and output from pageable, pinned and CUDA memory; 2^16 rows of 62-bit
    words to 20 bits;
  * the fold against fhe_b200_encode of the oracle's transcoded values: 1, 2 and 3 parts, 1 and 3 limbs, NTT and
    power-basis input, output at levels 0 and 1, E a multiple of N and not; its refusals and the memory they leave;
  * the SealPIR example (sealpir.rs:158-273) with its parameters: the server's responses equal the oracle's word for
    word and the device client recovers the element; at the example's default size, device only;
  * the EvaluationKey message of a device-generated key: expansions and rotations with the decoded key are identical;
  * chunking, through tests/pir_chunk_probe.py in a subprocess."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import encode_reference as ER
import pir_reference as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def F():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


@pytest.fixture(scope="module")
def par(F):
    return F.BfvParameters(64, 1153, moduli_sizes=[62] * 3, device=0)


def _random_rows(rng, n_rows, max_len):
    lens = [0, 1] + list(rng.integers(0, max_len + 1, size=n_rows - 2))
    rows = [rng.integers(0, 1 << 64, size=n, dtype=np.uint64) for n in lens]
    return lens, rows


# ------------------------------------------------------------------------------------------ transcoder
def test_transcoder_every_width_pair(F, par):
    """1..64 x 1..64: five rows (lengths 0, 1 and random) in a strided 2-D array; out_len truncates some rows and pads
    others"""
    rng = np.random.default_rng(5)
    for in_bits in range(1, 65):
        lens, rows = _random_rows(rng, 5, 40)
        stride = max(lens) + 3
        a = np.zeros((5, stride), np.uint64)
        for r, row in enumerate(rows):
            a[r, :len(row)] = row
        for out_bits in range(1, 65):
            full = -(-max(lens) * in_bits // out_bits)
            out_len = max(1, full - 2 + (out_bits % 5))
            src = a[:, :max(lens)]
            want = R.rows_reference([a[r, :max(lens)] for r in range(5)], in_bits, out_bits, out_len)
            wide = np.full((5, out_len + 4), 7, np.uint64)
            got = F.transcode_bidirectional(par, src, in_bits, out_bits, out_len=out_len, out=wide[:, 2:2 + out_len])
            assert (got == want).all(), (in_bits, out_bits)
            assert (wide[:, :2] == 7).all() and (wide[:, 2 + out_len:] == 7).all()
        # per-row lengths: one call per row, the row's own length
        for out_bits in (1, 8, 20, 63, 64):
            for row in rows:
                got = F.transcode_bidirectional(par, row, in_bits, out_bits)
                assert list(got) == R.transcode_bidirectional(row, in_bits, out_bits)


def test_transcoder_bytes_every_memory(F, par, oracle):
    import torch
    rng = np.random.default_rng(6)
    for nbits in (1, 7, 8, 20, 36, 62, 64):
        words = rng.integers(0, 1 << 64, size=(3, 50), dtype=np.uint64) & np.uint64((1 << nbits) - 1)
        want = np.array([list(oracle.transcode_to_bytes(w, nbits)) for w in words], np.uint8)
        by = np.array([list(bytes(rng.integers(0, 256, 77, dtype=np.uint8))) for _ in range(3)], np.uint8)
        want_from = np.array([oracle.transcode_from_bytes(bytes(b), nbits) for b in by], np.uint64)
        for kind in ("pageable", "pinned", "cuda"):
            def put(x):
                if kind == "pageable":
                    return x
                t = torch.from_numpy(x)
                return t.pin_memory() if kind == "pinned" else t.cuda()
            out = put(np.zeros(want.shape, np.uint8))
            F.transcode_to_bytes(par, put(words), nbits, out=out)
            assert (np.asarray(out.cpu() if kind != "pageable" else out) == want).all(), (nbits, kind)
            out2 = put(np.zeros(want_from.shape, np.uint64))
            F.transcode_from_bytes(par, put(by), nbits, out=out2)
            assert (np.asarray(out2.cpu() if kind != "pageable" else out2) == want_from).all(), (nbits, kind)
            # host in, device out and the reverse
            got = F.transcode_from_bytes(par, by, nbits) if kind == "pageable" else \
                F.transcode_from_bytes(par, put(by), nbits)
            assert (got == want_from).all()


def test_transcoder_large(F):
    """2^16 rows of 62-bit words (N = 2^16 parameters) to 20 bits, from and to CUDA memory"""
    import torch
    par = F.BfvParameters(1 << 16, 65537, moduli_sizes=[62], device=0)
    rng = np.random.default_rng(7)
    a = rng.integers(0, 1 << 62, size=(1 << 16, 33), dtype=np.uint64)
    out = torch.zeros((1 << 16, 103), dtype=torch.uint64, device="cuda")
    F.transcode_bidirectional(par, torch.from_numpy(a).cuda(), 62, 20, out=out)
    got = out.cpu().numpy()
    for r in (0, 1, 12345, (1 << 16) - 1):
        assert list(got[r]) == R.transcode_bidirectional(a[r], 62, 20), r
    # every row, vectorised: the first value of each is the low 20 bits of its first word
    assert (got[:, 0] == (a[:, 0] & np.uint64((1 << 20) - 1))).all()


def test_transcoder_refusals_with_device(F, par):
    import torch
    _capi = F._capi
    x = torch.zeros(64, dtype=torch.uint64, device="cuda")
    p = x.data_ptr()
    lib = _capi.lib()
    free0 = torch.cuda.mem_get_info()[0]
    assert lib.fhe_b200_transcode(par._h, p, 8, 8, 8, 62, p + 32, 8, 8, 8, 20, 1, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_transcode(par._h, p, 8, 8, 8, 0, p + 256, 8, 8, 8, 20, 1, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_transcode(par._h, p, 8, 8, 8, 62, p + 256, 8, 8, 8, 20, 0, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_transcode(par._h, p, 8, 0, 0, 62, p + 256, 8, 8, 8, 20, 1, None) == _capi.OK
    F._capi.check(lib.fhe_b200_sync(None))
    assert not x[32:40].cpu().numpy().any()                      # the empty stream pads with zeros
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 4 << 20


# ------------------------------------------------------------------------------------------ fold
def _fold_case(F, oracle, degree, n_moduli, parts, ct_level, repr, in_bits, out_bits, out_level, count, seed):
    opar = oracle.BfvParameters(degree, 1153, moduli_sizes=[62] * n_moduli)
    gpar = F.BfvParameters(degree, 1153, moduli=opar.moduli, device=0)
    L = n_moduli - ct_level
    rng = np.random.default_rng(seed)
    words = rng.integers(0, 1 << 64, size=(count, parts, L, degree), dtype=np.uint64)
    ct = F.Ciphertext.from_host(gpar, words, level=ct_level, repr=repr)
    pv = ct.fold(in_bits, out_bits, out_level)
    got = pv.batch.to_host()[:, 0]
    E = -(-L * degree * in_bits // out_bits)
    P = -(-parts * E // degree)
    assert got.shape[0] == P * count and pv.level == out_level
    for j in range(count):
        vals = R.fold_values(words[j], in_bits, out_bits)
        assert len(vals) == parts * E
        want = F.PlaintextVec.try_encode(vals, F.Encoding.poly_at_level(out_level), gpar).poly_ntt()
        assert want.shape[0] == P
        assert (want == ER.try_encode(opar, vals, False, out_level)).all()
        for i in range(P):
            assert (got[i * count + j] == want[i]).all(), (i, j)


@pytest.mark.parametrize("parts", [1, 2, 3])
@pytest.mark.parametrize("ct_level", [0, 2])                    # 3 limbs, 1 limb
@pytest.mark.parametrize("repr_", ["ntt", "power"])
def test_fold_matches_encode(oracle, F, parts, ct_level, repr_):
    repr = F.NTT if repr_ == "ntt" else F.POWER_BASIS
    for in_bits, out_bits, out_level in ((36, 20, 1), (40, 20, 0), (62, 62, 1), (64, 7, 0), (1, 64, 1)):
        _fold_case(F, oracle, 64, 3, parts, ct_level, repr, in_bits, out_bits, out_level, 3,
                   parts * 100 + ct_level * 10 + in_bits)


def test_fold_refusals(F, par):
    import torch
    _capi = F._capi
    lib = _capi.lib()
    other = F.BfvParameters(64, 1153, moduli_sizes=[62] * 3, device=0)
    ct = F.Ciphertext(par, 2, 2, 0)
    E = -(-3 * 64 * 36 // 20)
    P = -(-2 * E // 64)
    good = F.Ciphertext(par, P * 2, 1, 1)
    cases = [
        (ct, 36, 20, F.Ciphertext(other, P * 2, 1, 1), _capi.CONTEXT_MISMATCH),
        (ct, 36, 20, F.Ciphertext(par, P * 2, 1, 0, mul_basis=True), _capi.CONTEXT_MISMATCH),
        (F.Ciphertext(par, 2, 2, 0, mul_basis=True), 36, 20, good, _capi.CONTEXT_MISMATCH),
        (ct, 36, 20, F.Ciphertext(par, P * 2, 2, 1), _capi.BAD_POLY_COUNT),
        (ct, 36, 20, F.Ciphertext(par, P * 2 + 1, 1, 1), _capi.INVALID_ARGUMENT),
        (ct, 0, 20, good, _capi.INVALID_ARGUMENT),
        (ct, 36, 65, good, _capi.INVALID_ARGUMENT),
        (ct, 65, 20, good, _capi.INVALID_ARGUMENT),
    ]
    free1 = torch.cuda.mem_get_info()[0]
    for a, ib, ob, out, code in cases:
        assert lib.fhe_b200_fold(a._h, ib, ob, out._h, None) == code, (ib, ob, code)
    one = F.Ciphertext(par, 1, 1, 0)
    assert lib.fhe_b200_fold(one._h, 64, 64, one._h, None) == _capi.INVALID_ARGUMENT    # out aliasing ct
    assert lib.fhe_b200_fold(None, 36, 20, good._h, None) == _capi.INVALID_ARGUMENT
    assert torch.cuda.mem_get_info()[0] >= free1 - (4 << 20)


# ------------------------------------------------------------------------------------------ SealPIR
def _sealpir_device(F, gpar, ek, query_ct, db_t, dim1, dim2):
    """the server on the device: expand, first dimension, switch, fold, second dimension, switch"""
    X = ek.expands_batch(query_ct, dim1 + dim2)
    first = F.dot_product_scalar(X.take(0, dim1), db_t, n_terms=dim1).switch_to_level(gpar.max_level())
    in_bits, out_bits = int(gpar.moduli()[0]).bit_length(), gpar.plaintext().bit_length() - 1
    pts = first.fold(in_bits, out_bits, 1)
    return F.dot_product_scalar(X.take(dim1, dim2), pts, n_terms=dim2).switch_to_level(gpar.max_level())


def _encode_database(F, gpar, database_t, dim1, dim2, epp):
    """encode_database (util.rs:95-145) on the device, the plaintexts transposed for the first dimension: entry
    i * dim1 + k holds row k * dim2 + i.  database_t: CUDA uint8 tensor [n][elements_size]"""
    import torch
    n, es = database_t.shape
    N, nbits = gpar.degree(), gpar.plaintext().bit_length() - 1
    flat = torch.zeros((dim1, dim2, epp * es), dtype=torch.uint8, device="cuda")
    flat.view(-1)[: n * es] = database_t.reshape(-1)
    vals = torch.empty((dim2, dim1, N), dtype=torch.uint64, device="cuda")
    for k in range(dim1):     # rows k * dim2 + i, i < dim2, land at i * dim1 + k: an output row stride of dim1 * N
        F.transcode_from_bytes(gpar, flat[k], nbits, out_len=N, out=vals[:, k, :])
    return F.PlaintextVec.try_encode(vals.view(-1), F.Encoding.poly_at_level(1), gpar)


def _client_device(F, gpar, dsk, responses, index, es, epp):
    """sealpir.rs:222-273 on the device"""
    import torch
    N, nbits = gpar.degree(), gpar.plaintext().bit_length() - 1
    in_bits = int(gpar.moduli()[0]).bit_length()
    lvl = gpar.max_level()
    dec = torch.empty(responses.count * N, dtype=torch.uint64, device="cuda")
    dsk.try_decrypt(responses).try_decode(F.Encoding.poly_at_level(lvl), out=dec)
    E = -(-N * in_bits // nbits)
    ct = F.Ciphertext(gpar, 1, 2, lvl, F.NTT)
    dptr, nw = C.c_void_p(), C.c_size_t()
    F._capi.check(F._capi.lib().fhe_b200_batch_device_ptr(ct._h, C.byref(dptr), C.byref(nw)))
    # unfold the two polynomials straight into the ciphertext's storage: rows of E values -> N words of in_bits
    F._capi.check(F._capi.lib().fhe_b200_transcode(gpar._h, dec.data_ptr(), 8, E, E, nbits, dptr,
                                                   8, N, N, in_bits, 2, None))
    vals = torch.empty(N, dtype=torch.uint64, device="cuda")
    dsk.try_decrypt(ct).try_decode(F.Encoding.poly_at_level(lvl), out=vals)
    plaintext = F.transcode_to_bytes(gpar, vals, nbits)
    off = index % epp
    return bytes(plaintext[off * es:(off + 1) * es])


def test_sealpir_parity_with_oracle(oracle, F):
    import torch
    N, t = R.SEALPIR_DEGREE, R.SEALPIR_T
    opar = oracle.BfvParameters(N, t, moduli_sizes=R.SEALPIR_SIZES)
    gpar = F.BfvParameters(N, t, moduli=opar.moduli, device=0)
    rng = np.random.default_rng(11)
    n_el, es = 4096, 64
    database = rng.integers(0, 256, size=(n_el, es), dtype=np.uint8)
    epp, rows, dim1, dim2 = R.layout(N, t, n_el, es)
    assert (dim1, dim2) == (6, 5)
    # database: the device encoding equals the oracle's
    vals = R.database_values(database, N, t)
    odb = ER.try_encode(opar, vals.reshape(-1), False, 1)
    ddb = _encode_database(F, gpar, torch.from_numpy(database).cuda(), dim1, dim2, epp)
    got_db = ddb.poly_ntt()
    for i in range(dim2):
        for k in range(dim1):
            assert (got_db[i * dim1 + k] == odb[k * dim2 + i]).all(), (i, k)
    # keys: EvaluationKeyBuilder::new_leveled(&sk, 1, 0).enable_expansion(level)
    sk = oracle.SecretKey(opar, rng)
    level = (dim1 + dim2 - 1).bit_length()
    ogk = {(N >> l) + 1: oracle.GaloisKey(sk, (N >> l) + 1, rng, 1, 0) for l in range(level)}
    ek = F.EvaluationKey(gpar, 1, 0)
    for e, g in ogk.items():
        ek.add_galois_key(F.GaloisKey.from_arrays(gpar, e, *g.ksk.arrays(), ciphertext_level=1, key_level=0))
    ek = F.EvaluationKey.from_bytes(gpar, ek.to_bytes())       # the server starts from the message
    dsk = F.SecretKey(gpar, sk.coeffs)
    for index in (0, 4095, int(rng.integers(0, n_el))):
        q = sk.encrypt(R.query_values(dim1, dim2, index, epp, t), 1, rng)
        qct = F.Ciphertext.from_bytes(gpar, [F.Ciphertext.from_host(gpar, q.to_array()[None], level=1).to_bytes()[0]])
        resp = _sealpir_device(F, gpar, ek, qct, ddb, dim1, dim2)
        want = R.server_response(opar, ogk, odb, q, dim1, dim2)
        got = resp.to_host()
        assert got.shape[0] == len(want) == 4
        for i, w in enumerate(want):
            assert (got[i] == w.to_array()).all(), (index, i)
        answer = _client_device(F, gpar, dsk, resp, index, es, epp)
        assert answer == database[index].tobytes(), index

        def odecrypt(words, lv):
            return sk.decrypt(oracle.Ciphertext.from_array(opar, np.asarray(words, np.uint64), lv))
        assert R.client_answer(opar, odecrypt, [w.to_array() for w in want], index, es) == database[index].tobytes()


def test_sealpir_default_size_device_only(F):
    """the example's defaults: 65 536 elements of 1 024 bytes, dim1 = dim2 = 81; keys generated on the device and sent
    as an EvaluationKey message, the query as a Ciphertext message, the responses as messages"""
    import torch
    N, t = R.SEALPIR_DEGREE, R.SEALPIR_T
    gpar = F.BfvParameters(N, t, moduli_sizes=R.SEALPIR_SIZES, device=0)
    n_el, es = 65536, 1024
    epp, rows, dim1, dim2 = R.layout(N, t, n_el, es)
    assert (dim1, dim2) == (81, 81)
    g = torch.Generator(device="cuda").manual_seed(3)
    database = torch.randint(0, 256, (n_el, es), dtype=torch.uint8, device="cuda", generator=g)
    ddb = _encode_database(F, gpar, database, dim1, dim2, epp)
    rng = np.random.default_rng(12)
    dsk = F.SecretKey(gpar, rng.integers(-1, 2, size=N))
    level = (dim1 + dim2 - 1).bit_length()
    ek_msg = F.EvaluationKeyBuilder.new_leveled(dsk, 1, 0).enable_expansion(level).build(seed=bytes(32)).to_bytes()
    ek = F.EvaluationKey.from_bytes(gpar, ek_msg)
    assert (ek.ciphertext_level, ek.evaluation_key_level) == (1, 0)
    partial = (rows - 1) * epp + int(rng.integers(0, n_el - (rows - 1) * epp))
    for index in (0, n_el - 1, partial, int(rng.integers(0, n_el))):
        pts = F.PlaintextVec.try_encode(R.query_values(dim1, dim2, index, epp, t), F.Encoding.poly_at_level(1), gpar)
        query_msg = dsk.try_encrypt(pts, seed=bytes([index % 256]) * 32).to_bytes()
        resp = _sealpir_device(F, gpar, ek, F.Ciphertext.from_bytes(gpar, query_msg), ddb, dim1, dim2)
        resp = F.Ciphertext.from_bytes(gpar, resp.to_bytes())
        answer = _client_device(F, gpar, dsk, resp, index, es, epp)
        assert answer == database[index].cpu().numpy().tobytes(), index


# ------------------------------------------------------------------------------------------ EvaluationKey message
def test_evaluation_key_message_device(F):
    par = F.BfvParameters(64, 1153, moduli_sizes=[62] * 3, device=0)
    rng = np.random.default_rng(13)
    sk = F.SecretKey(par, rng.integers(-1, 2, size=64))
    for ct_level, key_level in ((0, 0), (1, 0), (1, 1)):
        ek = F.EvaluationKeyBuilder.new_leveled(sk, ct_level, key_level).enable_expansion(6).enable_inner_sum() \
            .enable_column_rotation(3).build(seed=bytes(range(32)))
        data = ek.to_bytes()
        back = F.EvaluationKey.from_bytes(par, data)
        assert back.to_bytes() == data and sorted(back.gk) == sorted(ek.gk)
        assert (back.ciphertext_level, back.evaluation_key_level) == (ct_level, key_level)
        x = sk.try_encrypt(F.PlaintextVec.try_encode(rng.integers(0, 1153, 64), F.Encoding.poly_at_level(ct_level), par),
                           seed=bytes(32))
        for a, b in zip(ek.expands(x, 37), back.expands(x, 37)):
            assert (a.to_host() == b.to_host()).all()
        assert (ek.rotates_rows(x).to_host() == back.rotates_rows(x).to_host()).all()
        assert (ek.rotates_columns_by(x, 3).to_host() == back.rotates_columns_by(x, 3).to_host()).all()
        assert (ek.computes_inner_sum(x).to_host() == back.computes_inner_sum(x).to_host()).all()


def test_evaluation_key_message_refusals(F):
    import torch
    par = F.BfvParameters(64, 1153, moduli_sizes=[62] * 3, device=0)
    rng = np.random.default_rng(14)
    sk = F.SecretKey(par, rng.integers(-1, 2, size=64))
    ek = F.EvaluationKeyBuilder.new_leveled(sk, 1, 0).enable_row_rotation().build(seed=bytes(32))
    msgs = [g.to_bytes() for g in ek.gk.values()]
    free0 = torch.cuda.mem_get_info()[0]
    for levels in ((0, 0), (1, 1), (2, 0)):
        with pytest.raises(F.WireError) as e:
            F.EvaluationKey.from_bytes(par, F.wire.encode_evaluation_key(msgs, *levels))
        assert e.value.variant == "InvalidLevel" and e.value.code == F._capi.INVALID_LEVEL
    # a compact key without its expanded c1
    k0, k1 = ek.gk[127].ksk.arrays()
    import fhe_rs_b200.wire as W
    blobs = F.Ciphertext.from_host(par, np.ascontiguousarray(k0[:, None]), 0, F.NTT).to_packed()
    c0 = [W.encode_rq(W.REP_NTTSHOUP, 64, memoryview(blobs[i, 0])) for i in range(k0.shape[0])]
    seeded = W.encode_galois_key(W.encode_ksk(c0, [], bytes(32), 1, 0, 0), 127)
    with pytest.raises(F.WireError) as e:
        F.EvaluationKey.from_bytes(par, F.wire.encode_evaluation_key([seeded], 1, 0))
    assert e.value.variant == "SeedExpansion" and e.value.code == F._capi.UNSUPPORTED
    got = F.EvaluationKey.from_bytes(par, F.wire.encode_evaluation_key([seeded], 1, 0), seeded_c1={127: k1})
    assert all((a == b).all() for a, b in zip(got.gk[127].ksk.arrays(), (k0, k1)))
    del got, blobs
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 8 << 20


# ------------------------------------------------------------------------------------------ chunking
@pytest.mark.parametrize("env", [{"FHE_B200_CHUNK": "2", "FHE_B200_STREAMS": "1"},
                                 {"FHE_B200_CHUNK": "2", "FHE_B200_STREAMS": "2"},
                                 {"FHE_B200_CHUNK": "3", "FHE_B200_STREAMS": "4"}])
def test_pir_across_chunks(F, env):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "pir_chunk_probe.py")], cwd=ROOT,
                         env=dict(os.environ, **env), capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "pir chunk probe ok" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]


# ------------------------------------------------------------------------------------------ layouts and the C++ mirror
def test_transcoder_input_layouts(F, par):
    """strided, broadcast and overlapping input rows (numpy and CUDA) give the values of their contiguous copies; an
    output that cannot be written in place is refused and left untouched"""
    import torch
    base = np.arange(1, 41, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    overlapping = np.lib.stride_tricks.as_strided(base, shape=(4, 10), strides=(8, 8))
    for a in (base[::2], np.broadcast_to(base[:10], (4, 10)), overlapping, base.reshape(4, 10)[::-1],
              base.reshape(4, 10)[:, ::2]):
        want = R.rows_reference(list(np.atleast_2d(np.array(a))), 62, 20, 40)
        got = F.transcode_bidirectional(par, a, 62, 20, out_len=40)
        assert (np.atleast_2d(got) == want).all()
    t = torch.from_numpy(np.ascontiguousarray(base)).cuda()
    for a in (t[:10].expand(4, 10), t[::2], t.view(4, 10)[:, ::2], t.as_strided((4, 10), (1, 1))):
        want = R.rows_reference(list(np.atleast_2d(a.cpu().numpy())), 62, 20, 40)
        got = F.transcode_bidirectional(par, a, 62, 20, out_len=40)
        assert (np.atleast_2d(got) == want).all()
    buf = np.full(80, 5, np.uint64)
    cbuf = torch.full((80,), 5, dtype=torch.int64, device="cuda").view(torch.uint64)
    for out in (buf[::2], buf.reshape(8, 10)[:4, ::2], cbuf[::2]):
        with pytest.raises(F.FheError) as e:
            F.transcode_bidirectional(par, base[:40], 62, 20, out_len=len(out), out=out)
        assert e.value.code == F._capi.INVALID_ARGUMENT
    assert (buf == 5).all() and (cbuf.view(torch.int64).cpu().numpy() == 5).all()


def test_cpp_mirror_equals_python(oracle, F, tmp_path):
    """include/fhe_b200.hpp / fhe_b200_wire.hpp: Ciphertext::fold, the three transcoders and EvaluationKey to_bytes /
    evaluation_key_from_bytes give the Python mirror's words and bytes"""
    import struct
    from test_pir_cpu import pir_driver
    run = pir_driver(tmp_path)
    gpar = F.BfvParameters(64, 1153, moduli_sizes=[62] * 3, device=0)
    rng = np.random.default_rng(21)
    count, parts, level, in_bits, out_bits, out_level = 3, 2, 1, 36, 20, 1
    words = rng.integers(0, 1 << 64, size=(count, parts, 2, 64), dtype=np.uint64)
    rows = rng.integers(0, 1 << 64, size=(3, 25), dtype=np.uint64)
    sk = F.SecretKey(gpar, rng.integers(-1, 2, size=64))
    ek = F.EvaluationKeyBuilder.new_leveled(sk, 1, 0).enable_expansion(3).enable_row_rotation().build(seed=bytes(32))
    msg = ek.to_bytes()
    hdr = struct.pack("<11I", count, parts, level, F.NTT, in_bits, out_bits, out_level, 3, 25, 13, 7)
    res = dict(run("device", 64, 1153, gpar.moduli(), 0,
                   [("h", hdr), ("c", words.tobytes()), ("r", rows.tobytes()), ("m", msg)]))
    want_fold = F.Ciphertext.from_host(gpar, words, level=level).fold(in_bits, out_bits, out_level).poly_ntt()
    assert (np.frombuffer(res["f"], np.uint64) == want_fold.reshape(-1)).all()
    assert (np.frombuffer(res["t"], np.uint64) == F.transcode_bidirectional(gpar, rows, 13, 7).reshape(-1)).all()
    b = F.transcode_to_bytes(gpar, rows[0], 13)
    assert res["b"] == b.tobytes()
    assert (np.frombuffer(res["y"], np.uint64) == F.transcode_from_bytes(gpar, b, 13)).all()
    assert res["k"] == msg == F.EvaluationKey.from_bytes(gpar, msg).to_bytes()
    bad = F.wire.encode_evaluation_key([g.to_bytes() for g in ek.gk.values()], 0, 0)
    res = dict(run("device", 64, 1153, gpar.moduli(), 0,
                   [("h", hdr), ("c", words.tobytes()), ("r", rows.tobytes()), ("m", bad)]))
    assert res["w"] == b"InvalidLevel"

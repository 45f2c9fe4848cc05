"""CPU checks behind tests/test_gpu_pir.py (SealPIR on the device):

  * the oracle's transcode_bidirectional (tests/pir_reference.py) bit by bit against a bit-stream statement at every
    (in, out) width in 1..64 x 1..64 for row lengths 0..100, the reference's own properties (fhe-util/src/lib.rs:322-371)
    extended to widths 63 and 64, and the masking of words wider than in_bits;
  * the EvaluationKey message (bfv.proto:34-38): the host codec's bytes equal the google.protobuf runtime's for the same
    key order, shuffled and repeated keys decode as the reference's HashMap does, and the reference's proto_conversion
    and serialize cases (keys/evaluation_key.rs:887-972) on the oracle;
  * the refusals of fhe_b200_transcode and fhe_b200_fold that need no device."""
import ctypes as C

import numpy as np
import pytest

import pir_reference as R


@pytest.fixture(scope="module")
def F():
    from fhe_rs_b200 import build
    build.build()
    import fhe_rs_b200
    return fhe_rs_b200


# ------------------------------------------------------------------------------------------ oracle transcoder
def test_oracle_transcoder_matches_bit_stream():
    rng = np.random.default_rng(1)
    for in_bits in range(1, 65):
        rows = [rng.integers(0, 1 << 63, size=n, dtype=np.uint64) * 2 + rng.integers(0, 2, size=n, dtype=np.uint64)
                for n in range(0, 101, 7)]
        rows += [rng.integers(0, 2, size=1, dtype=np.uint64)]
        for out_bits in range(1, 65):
            for row in rows:
                assert R.transcode_bidirectional(row, in_bits, out_bits) == R.bitstream(row, in_bits, out_bits), \
                    (in_bits, out_bits, len(row))


@pytest.mark.parametrize("n", list(range(0, 101)))
def test_oracle_transcoder_every_length(n):
    rng = np.random.default_rng(n)
    row = rng.integers(0, 1 << 64, size=n, dtype=np.uint64)
    for in_bits, out_bits in ((1, 64), (64, 1), (7, 13), (13, 7), (62, 20), (20, 62), (64, 64), (63, 8), (8, 63)):
        assert R.transcode_bidirectional(row, in_bits, out_bits) == R.bitstream(row, in_bits, out_bits)


def test_oracle_transcoder_reference_properties(oracle):
    """lib.rs:322-371: equal to transcode_to_bytes at 8 output bits, round trips both ways, the empty round trip"""
    rng = np.random.default_rng(2)
    for nbits in list(range(1, 65)):
        a = rng.integers(0, 1 << 64, size=37, dtype=np.uint64) & np.uint64((1 << nbits) - 1)
        b = R.transcode_bidirectional(a, nbits, 8)
        assert bytes(b) == oracle.transcode_to_bytes(a, nbits)
        back = R.transcode_bidirectional(b, 8, nbits)
        assert back[:len(a)] == [int(x) for x in a] and not any(back[len(a):])
        assert R.transcode_bidirectional(a, nbits, nbits) == [int(x) for x in a]
        by = bytes(rng.integers(0, 256, size=41, dtype=np.uint8))
        assert R.transcode_bidirectional(list(by), 8, nbits) == oracle.transcode_from_bytes(by, nbits)
        assert bytes(R.transcode_bidirectional(R.transcode_bidirectional(list(by), 8, nbits), nbits, 8))[:41] == by
    for i in range(1, 65):
        for o in range(1, 65):
            assert R.transcode_bidirectional([], i, o) == []


def test_oracle_transcoder_masks_wide_words():
    row = [(1 << 64) - 1, 0x123456789ABCDEF0, 1 << 63]
    for in_bits in range(1, 64):
        masked = [v & ((1 << in_bits) - 1) for v in row]
        for out_bits in (1, 8, 20, 64):
            assert R.transcode_bidirectional(row, in_bits, out_bits) == R.transcode_bidirectional(masked, in_bits,
                                                                                                  out_bits)


# ------------------------------------------------------------------------------------------ EvaluationKey message
def _keys(oracle, par, exps, seed, ct_level=0, key_level=0):
    rng = np.random.default_rng(seed)
    sk = oracle.SecretKey(par, rng)
    return {e: oracle.GaloisKey(sk, e, rng, ct_level, key_level) for e in exps}


def _cases(degree):
    logn = degree.bit_length() - 1
    return [R.builder_exponents(degree), R.builder_exponents(degree, row_rotation=True),
            R.builder_exponents(degree, inner_sum=True), R.builder_exponents(degree, expansion=logn),
            R.builder_exponents(degree, inner_sum=True, expansion=logn)]


@pytest.mark.parametrize("n_moduli", [1, 6, 5])
def test_reference_proto_conversion_and_serialize(oracle, n_moduli):
    """evaluation_key.rs:887-972 on default_arc(n_moduli, 16): every builder case round trips through the message"""
    par = oracle.BfvParameters(16, 1153, moduli_sizes=[62] * n_moduli)
    for k, exps in enumerate(_cases(16)):
        gks = _keys(oracle, par, exps, 10 * n_moduli + k)
        data = R.evaluation_key_to_bytes(gks, 0, 0)
        got, ct_level, ek_level = R.evaluation_key_from_bytes(par, data)
        assert (ct_level, ek_level) == (0, 0) and sorted(got) == exps
        for e in exps:
            for a, b in zip(got[e].ksk.arrays(), gks[e].ksk.arrays()):
                assert (a == b).all()


def test_host_codec_bytes_equal_runtime(oracle, F):
    """wire.encode_evaluation_key of the GaloisKey messages equals the runtime's bytes, for levels 0 and nonzero and
    for any key order; decode_evaluation_key returns the messages in wire order"""
    import fhe_wire as W
    par = oracle.BfvParameters(16, 1153, moduli_sizes=[62] * 3)
    exps = R.builder_exponents(16, inner_sum=True, expansion=2)
    for levels in ((0, 0), (1, 0), (1, 1), (2, 1)):
        gks = _keys(oracle, par, exps, sum(levels), *levels)
        for order in (exps, exps[::-1], [exps[2], exps[0]] + exps[1:2] + exps[3:]):
            want = R.evaluation_key_to_bytes(gks, levels[0], levels[1], order)
            msgs = [W.galois_key_to_bytes(gks[e]) for e in order]
            assert F.wire.encode_evaluation_key(msgs, *levels) == want
            got_msgs, a, b = F.wire.decode_evaluation_key(want)
            assert (a, b) == levels and [bytes(m) for m in got_msgs] == msgs
    assert F.wire.encode_evaluation_key([], 0, 0) == b""
    assert F.wire.decode_evaluation_key(b"") == ([], 0, 0)


def test_shuffled_and_repeated_keys(oracle):
    """runtime bytes with the keys shuffled and one exponent twice: the later key wins, as HashMap::insert"""
    par = oracle.BfvParameters(16, 1153, moduli_sizes=[62] * 2)
    exps = R.builder_exponents(16, row_rotation=True, expansion=3)
    a, b = _keys(oracle, par, exps, 1), _keys(oracle, par, exps, 2)
    m = R.EvaluationKeyProto()
    import fhe_wire as W
    for gk in (a[exps[2]], a[exps[0]], b[exps[2]], a[exps[1]], a[exps[3]]):
        m.gk.add().ParseFromString(W.galois_key_to_bytes(gk))
    got, _, _ = R.evaluation_key_from_bytes(par, m.SerializeToString())
    assert sorted(got) == exps
    assert (got[exps[2]].ksk.arrays()[0] == b[exps[2]].ksk.arrays()[0]).all()
    assert (got[exps[0]].ksk.arrays()[0] == a[exps[0]].ksk.arrays()[0]).all()


def test_oracle_level_refusals(oracle):
    par = oracle.BfvParameters(16, 1153, moduli_sizes=[62] * 3)
    gks = _keys(oracle, par, [17, 9], 3, 1, 0)
    for levels in ((0, 0), (1, 1), (2, 0)):
        with pytest.raises(R.EvaluationKeyError, match="InvalidLevel"):
            R.evaluation_key_from_bytes(par, R.evaluation_key_to_bytes(gks, *levels))
    with pytest.raises(R.EvaluationKeyError, match="InvalidLevel"):
        R.evaluation_key_from_bytes(par, R.evaluation_key_to_bytes({}, 3, 0))
    assert R.evaluation_key_from_bytes(par, R.evaluation_key_to_bytes({}, 2, 0))[1:] == (2, 0)


def test_empty_message_level_refusal_host_only(F):
    """the Python codec: an empty message beyond the maximum level is InvalidLevel, at the maximum it decodes (no key
    needs the device)"""
    par = F.BfvParameters(16, 1153, moduli_sizes=[62] * 3, device=-1)
    ek = F.EvaluationKey.from_bytes(par, F.wire.encode_evaluation_key([], 2, 1))
    assert (ek.ciphertext_level, ek.evaluation_key_level, ek.gk) == (2, 1, {})
    assert F.EvaluationKey.from_bytes(par, ek.to_bytes()).ciphertext_level == 2
    with pytest.raises(F.WireError) as e:
        F.EvaluationKey.from_bytes(par, F.wire.encode_evaluation_key([], 3, 0))
    assert e.value.variant == "InvalidLevel" and e.value.code == F._capi.INVALID_LEVEL
    assert F.EvaluationKey(par).ciphertext_level == 0 and F.EvaluationKey(par).evaluation_key_level == 0


# ------------------------------------------------------------------------------------------ refusals without a device
def test_symbols_declared(F):
    lib = F._capi.lib()
    for name in ("fhe_b200_transcode", "fhe_b200_fold"):
        assert hasattr(lib, name) and name in F._capi.SYMBOLS


def test_transcode_refusals_host_only(F):
    _capi = F._capi
    lib = _capi.lib()
    par = F.BfvParameters(16, 1153, moduli_sizes=[62] * 2, device=-1)
    src = np.arange(64, dtype=np.uint64)
    dst = np.zeros(64, np.uint64)
    s, d = src.ctypes.data, dst.ctypes.data

    def call(p=par._h, i=s, ie=8, il=4, ist=4, ib=62, o=d, oe=8, ol=4, ost=4, ob=20, rows=2):
        return lib.fhe_b200_transcode(p, i, ie, il, ist, ib, o, oe, ol, ost, ob, rows, None)

    assert call() == _capi.NO_DEVICE
    assert call(il=0, i=None) == _capi.NO_DEVICE           # an empty input row is valid
    bad = [dict(p=None), dict(ib=0), dict(ib=65), dict(ob=0), dict(ob=65), dict(ie=4), dict(oe=2),
           dict(ie=1, ib=7), dict(oe=1, ob=20), dict(rows=0), dict(ist=3), dict(ost=3), dict(i=None),
           dict(o=None), dict(o=s + 16), dict(i=d + 8), dict(o=s, ol=1, ost=1, rows=1, il=1, ist=1)]
    for kw in bad:
        assert call(**kw) == _capi.INVALID_ARGUMENT, kw
    # adjacent ranges do not overlap
    assert call(o=s + 8 * 8, rows=2) == _capi.NO_DEVICE
    with pytest.raises(F.FheError) as e:
        F.transcode_bidirectional(par, src, 62, 20)
    assert e.value.code == _capi.NO_DEVICE


def test_fold_refusals_host_only(F):
    _capi = F._capi
    lib = _capi.lib()
    assert lib.fhe_b200_fold(None, 36, 20, None, None) == _capi.INVALID_ARGUMENT
    par = F.BfvParameters(16, 1153, moduli_sizes=[62] * 2, device=-1)
    h = C.c_void_p()
    assert lib.fhe_b200_batch_alloc(par._h, 1, 2, 0, _capi.NTT, C.byref(h)) == _capi.NO_DEVICE


def test_row_layouts(F):
    """inputs whose rows are not contiguous at a stride of at least their length (strided, broadcast, overlapping,
    reversed) are copied before the device reads them; such outputs are refused instead of written to a copy"""
    import torch
    from fhe_rs_b200.bfv import _rows
    base = np.arange(40, dtype=np.uint64)
    overlapping = np.lib.stride_tricks.as_strided(base, shape=(4, 10), strides=(8, 8))
    for a in (base[::2], np.broadcast_to(base[:10], (4, 10)), overlapping, base.reshape(4, 10)[::-1],
              base.reshape(4, 10)[:, ::2], torch.from_numpy(base[:10]).expand(4, 10), torch.from_numpy(base)[::2]):
        ptr, rows, n, stride, keep, _ = _rows(a, 8, "")
        assert stride >= n
        flat = np.asarray(keep).reshape(-1) if not hasattr(keep, "is_cuda") else keep.reshape(-1).numpy()
        want = np.asarray(a).reshape(rows, n)
        got = np.lib.stride_tricks.as_strided(flat, shape=(rows, n), strides=(stride * 8, 8))
        assert (got == want).all()
        with pytest.raises(F.FheError) as e:
            _rows(a, 8, "", output=True)
        assert e.value.code == F._capi.INVALID_ARGUMENT
    # rows of a wider buffer are written in place, at its stride
    wide = np.zeros((3, 12), np.uint64)
    ptr, rows, n, stride, keep, _ = _rows(wide[:, 1:9], 8, "", output=True)
    assert (ptr, rows, n, stride) == (wide.ctypes.data + 8, 3, 8, 12) and keep.base is not None
    ro = np.zeros(8, np.uint64)
    ro.flags.writeable = False
    with pytest.raises(F.FheError):
        _rows(ro, 8, "", output=True)
    with pytest.raises(F.FheError):
        _rows([0, 1, 2], 8, "", output=True)


def pir_driver(tmp_dir):
    """builds tests/cpp/pir_test.cpp; returns run(mode, degree, t, moduli, device, records) -> [(tag, bytes)]"""
    import os
    import struct
    import subprocess
    from fhe_rs_b200 import build
    build.build()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(str(tmp_dir), "pir_test")
    lib_dir = os.path.join(root, "fhe_rs_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(root, "include"),
                           os.path.join(root, "tests", "cpp", "pir_test.cpp"), "-o", exe,
                           "-L", lib_dir, "-lfhe_b200", "-Wl,-rpath," + lib_dir])

    def run(mode, degree, t, moduli, device, records):
        mpath, ipath, opath = (os.path.join(str(tmp_dir), n) for n in ("moduli.bin", "in.bin", "out.bin"))
        np.array(moduli, np.uint64).tofile(mpath)
        with open(ipath, "wb") as f:
            f.write(b"".join(tag.encode() + struct.pack("<I", len(m)) + m for tag, m in records))
        subprocess.check_call([exe, mode, str(degree), str(t), str(device), mpath, ipath, opath], timeout=600)
        out, pos, res = open(opath, "rb").read(), 0, []
        while pos < len(out):
            (n,) = struct.unpack_from("<I", out, pos + 1)
            res.append((chr(out[pos]), out[pos + 5:pos + 5 + n]))
            pos += 5 + n
        return res
    return run


def test_cpp_codec_bytes_equal_runtime(oracle, F, tmp_path):
    """include/fhe_b200_wire.hpp: encode_evaluation_key equals the runtime's bytes for any key order, its decoder gives
    the messages back in wire order, and a message without keys beyond the maximum level is InvalidLevel"""
    import struct
    import fhe_wire as W
    run = pir_driver(tmp_path)
    par = oracle.BfvParameters(16, 1153, moduli_sizes=[62] * 3)
    exps = R.builder_exponents(16, inner_sum=True, expansion=2)
    for levels, order_kind in (((0, 0), 0), ((1, 0), 1), ((2, 1), 2), ((3, 0), 0)):
        gks = _keys(oracle, par, exps, sum(levels), *[min(x, 2) for x in levels])
        order = (exps, exps[::-1], exps[1:] + exps[:1])[order_kind]
        msgs = [W.galois_key_to_bytes(gks[e]) for e in order]
        res = run("codec", 16, 1153, par.moduli, -1, [("h", struct.pack("<II", *levels))] + [("g", m) for m in msgs])
        assert res[0] == ("k", R.evaluation_key_to_bytes(gks, levels[0], levels[1], order))
        assert [r[1] for r in res[1:-1]] == msgs and all(r[0] == "g" for r in res[1:-1])
        if levels[0] > 2:
            assert res[-1] == ("w", b"InvalidLevel")
        else:
            assert res[-1] == ("l", struct.pack("<II", *levels))

"""CPU checks behind tests/test_gpu_widths.py, the modulus-width tests.

  * the single-modulus decomposition (key_switching_key.rs:92-97) at every q_0 width from 10 to 62: log_base, the
    digit count (3 at odd widths), the reference test's noise bound (:595-627) and the gadget's closed form;
  * the bit transcoder (fhe-util/src/lib.rs:71-146) at every width from 1 to 62 against a bit-by-bit restatement,
    and the oracle's reading of fields in [q, 2^nbits) (rq/convert.rs:148-159: kept as they are in the power basis,
    transformed in the NTT one);
  * both host codecs of key messages (fhe_rs_b200.bfv and include/fhe_b200_wire.hpp through tests/cpp/ksk_wire_test.cpp)
    on host-only parameters: 3-digit messages pass every message check (only the device upload is left, which fails
    with NO_DEVICE), and wrong digit counts are refused with WrongPolynomialCount, as oracle/fhe_wire.py does."""
import os
import struct
import subprocess

import numpy as np
import pytest

import edge_inputs as E
import keygen_reference as K

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIDTHS = list(range(10, 63))


@pytest.fixture(scope="module")
def F():
    from fhe_rs_b200 import build
    build.build()
    import fhe_rs_b200
    return fhe_rs_b200


@pytest.fixture(scope="module")
def ow(oracle):
    import fhe_wire
    return fhe_wire


def ksk_codec(tmp_dir):
    """builds tests/cpp/ksk_wire_test.cpp; returns run(degree, t, moduli, device, messages) -> [(tag, bytes)]"""
    from fhe_rs_b200 import build
    build.build()                               # the header links against the C ABI library (no-op when it is current)
    exe = os.path.join(str(tmp_dir), "ksk_wire_test")
    lib_dir = os.path.join(ROOT, "fhe_rs_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "ksk_wire_test.cpp"), "-o", exe,
                           "-L", lib_dir, "-lfhe_b200", "-Wl,-rpath," + lib_dir])

    def run(degree, t, moduli, device, messages):
        mpath, ipath, opath = (os.path.join(str(tmp_dir), n) for n in ("moduli.bin", "in.bin", "out.bin"))
        np.array(moduli, np.uint64).tofile(mpath)
        with open(ipath, "wb") as f:
            f.write(b"".join(struct.pack("<I", len(m)) + m for m in messages))
        subprocess.check_call([exe, str(degree), str(t), str(device), mpath, ipath, opath], timeout=600)
        out, pos, res = open(opath, "rb").read(), 0, []
        while pos < len(out):
            (n,) = struct.unpack_from("<I", out, pos + 1)
            res.append((chr(out[pos]), out[pos + 5:pos + 5 + n]))
            pos += 5 + n
        assert len(res) == len(messages)
        return res
    return run


def log_base_of(q: int):
    """key_switching_key.rs:92-97 in plain integers: log_modulus = ilog2(next_power_of_two(q)), base log_modulus / 2,
    ceil(log_modulus / log_base) digits"""
    p = 1
    while p < q:
        p <<= 1
    log_modulus = p.bit_length() - 1
    log_base = log_modulus // 2
    return log_base, -(-log_modulus // log_base)


# ------------------------------------------------------------------------------------------------- decomposition

@pytest.mark.parametrize("bits", WIDTHS)
def test_decomposition_at_every_width(oracle, bits):
    """A key at the single-modulus last level of [q_0, 62, 62] for every q_0 width: log_base = bits / 2 (rounded
    down) and 3 digits at odd widths, 2 at even ones; the digits of the oracle's decomposition recompose every
    input; c0 + c1 s - input p stays within bits(q) / 2 + 10 bits (the reference test's bound); the restated gadget
    is 2^(i log_base), which the device reduces as (1 << i log_base) mod q_0."""
    degree = 16
    moduli = E.decomposition_moduli(bits, degree)
    q = moduli[0]
    assert q.bit_length() == bits
    par = oracle.BfvParameters(degree, 97, moduli=moduli)
    last = len(moduli) - 1
    ctx = par.context_at_level(last)
    log_base, n_dig = log_base_of(q)
    assert (log_base, n_dig) == (bits // 2, 3 if bits % 2 else 2)
    assert oracle._ksk_log_base(ctx) == (log_base, n_dig)
    g = K.gadget(par, last, last)
    assert g == [1 << (i * log_base) for i in range(n_dig)]
    assert [(1 << (i * log_base)) % q for i in range(n_dig)] == [pow(2, i * log_base, q) for i in range(n_dig)]
    rng = np.random.default_rng(bits)
    for trial in range(4):
        sk = oracle.SecretKey(par, rng)
        p = oracle.Poly.from_i64(ctx, oracle.sample_vec_cbd(degree, 10, rng))
        ksk = oracle.KeySwitchingKey(sk, p, last, last, rng)
        assert ksk.log_base == log_base and len(ksk.c0) == len(ksk.c1) == n_dig
        inp = oracle.Poly.random(ctx, oracle.POWER_BASIS, rng)
        if trial == 0:
            inp.c[0] = q - 1
        x = [int(v) for v in inp.c[0]]
        mask = (1 << log_base) - 1
        assert all(sum(((v >> (i * log_base)) & mask) * g[i] for i in range(n_dig)) == v for v in x)
        c0, c1 = ksk.key_switch(inp)
        c2 = c0.copy().iadd(c1.copy().imul(sk.s_ntt(ctx))).into_power_basis()
        c3 = inp.copy().into_ntt().imul(p.copy().into_ntt()).into_power_basis()
        for a, b in zip(c2.c[0], c3.c[0]):
            d = (int(a) - int(b)) % q
            assert min(d.bit_length(), (q - d).bit_length()) <= q.bit_length() // 2 + 10, (bits, trial)


# ---------------------------------------------------------------------------------------------------- bit packer

def pack_bits(values, nbits):
    """transcode_to_bytes bit by bit: bit b of value k is bit k nbits + b of the stream, LSB first"""
    bits = [(int(v) >> b) & 1 for v in values for b in range(nbits)]
    bits += [0] * (-len(bits) % 8)
    return bytes(sum(bits[i + b] << b for b in range(8)) for i in range(0, len(bits), 8))


def unpack_bits(data, nbits):
    """transcode_from_bytes bit by bit: full nbits fields, then whatever bits are left as one more value"""
    bits = [(byte >> b) & 1 for byte in data for b in range(8)]
    out = [sum(bits[i + b] << b for b in range(nbits)) for i in range(0, len(bits) - nbits + 1, nbits)]
    rest = bits[len(out) * nbits:]
    if rest:
        out.append(sum(x << b for b, x in enumerate(rest)))
    return out


def pack_words(words, moduli):
    """Rq coefficients of power-basis words [..., L, N] (whole rows of N = 8k fields), vectorized: [..., bytes]; the
    restatement of transcode_to_bytes per limb used where the oracle's byte loop is too slow (N = 2^16)"""
    rows = []
    for i, q in enumerate(moduli):
        nb = (int(q) - 1).bit_length()
        w = words[..., i, :]
        bits = ((w[..., None] >> np.arange(nb, dtype=np.uint64)) & np.uint64(1)).astype(np.uint8)
        rows.append(np.packbits(bits.reshape(w.shape[:-1] + (-1,)), axis=-1, bitorder="little"))
    return np.concatenate(rows, axis=-1)


@pytest.mark.parametrize("degree,sizes", [(8, [62, 17, 40, 10, 33, 55]), (64, [61, 13, 24, 48]), (16, [1, 2, 7, 9])])
def test_vectorized_packer(oracle, degree, sizes):
    """pack_words equals the oracle's transcode_to_bytes per limb, on fields below and above q"""
    rng = np.random.default_rng(degree)
    moduli = [(1 << (s - 1)) + 1 if s > 1 else 2 for s in sizes]
    x = np.stack([np.stack([rng.integers(0, 1 << s, size=degree, dtype=np.uint64) for s in sizes]) for _ in range(3)])
    x[0] = np.array([(1 << s) - 1 for s in sizes], np.uint64)[:, None]
    got = pack_words(x, moduli)
    for c in range(3):
        assert got[c].tobytes() == b"".join(oracle.transcode_to_bytes(x[c, i], s) for i, s in enumerate(sizes))


@pytest.mark.parametrize("nbits", range(1, 63))
def test_transcode_every_width(oracle, nbits):
    """transcode_to_bytes / transcode_from_bytes at every field width from 1 to 62 against the bit-by-bit
    restatement: rows of 0, q - 1, 2^nbits - 1, alternating 0 / 2^nbits - 1 and random values, for 8 and 16 values
    (whole bytes) and 13 (a partial last byte)"""
    rng = np.random.default_rng(nbits)
    top = (1 << nbits) - 1
    q = (1 << (nbits - 1)) + 1 if nbits > 1 else 2       # bitlen(q - 1) = nbits
    for size in (8, 13, 16):
        rows = {"zero": [0] * size, "q-1": [q - 1] * size, "top": [top] * size,
                "alternating": [top * (k % 2) for k in range(size)],
                "random": [int(v) for v in rng.integers(0, top, size=size, dtype=np.uint64, endpoint=True)]}
        for name, row in rows.items():
            b = oracle.transcode_to_bytes(row, nbits)
            assert b == pack_bits(row, nbits), (nbits, size, name)
            assert len(b) == -(-size * nbits // 8)
            back = oracle.transcode_from_bytes(b, nbits)
            assert back == unpack_bits(b, nbits), (nbits, size, name)
            assert back[:size] == row
        # wider values are masked to their low nbits bits
        wide = [int(v) for v in rng.integers(0, 1 << 63, size=size, dtype=np.uint64)]
        assert oracle.transcode_to_bytes(wide, nbits) == pack_bits([v & top for v in wide], nbits)


@pytest.mark.parametrize("degree,moduli", [(16, [65537]), (16, "62"), (16, "31"), (8, "mixed")],
                         ids=["65537", "62", "31", "mixed_n8"])
def test_oracle_reads_fields_at_or_above_q(oracle, degree, moduli):
    """poly_from_rq_coefficients of blobs whose fields lie in [q, 2^nbits): the power basis keeps them as they are
    (rq/convert.rs:148-159), the NTT representation is the transform of the reduced words (the forward transform
    takes inputs below 4p).  tests/test_gpu_widths.py holds the device to these words."""
    if moduli == "mixed":
        moduli = oracle.BfvParameters.generate_moduli([62, 17, 40, 10, 33], degree)
    elif isinstance(moduli, str):
        moduli = [E.prime_of_width(int(moduli), degree)]
    ctx = oracle.Context(moduli, degree)
    rng = np.random.default_rng(degree + len(moduli))
    per_limb = [E.pack_rows(q, degree, rng) for q in moduli]
    for name in per_limb[0]:
        rows = np.stack([r[name] for r in per_limb])
        blob = b"".join(oracle.transcode_to_bytes(rows[i], (q - 1).bit_length()) for i, q in enumerate(moduli))
        pb = oracle.poly_from_rq_coefficients(ctx, blob, oracle.POWER_BASIS)
        assert (pb.c == rows).all(), name
        reduced = np.stack([rows[i] % np.uint64(q) for i, q in enumerate(moduli)])
        ntt = oracle.poly_from_rq_coefficients(ctx, blob, oracle.NTT)
        assert (ntt.c == oracle.Poly(ctx, oracle.POWER_BASIS, reduced.copy()).into_ntt().c).all(), name
        if name.startswith("field"):
            assert (rows >= np.array(moduli, np.uint64)[:, None]).all()
    assert (65537 - 1).bit_length() == 17


# ---------------------------------------------------------------------------------------------------- key codecs

def key_messages(oracle, ow, bits, rng):
    """(parameter set, message of a last-level key, messages with one c0 / c1 polynomial too many or too few)"""
    moduli = E.decomposition_moduli(bits, 16)
    par = oracle.BfvParameters(16, 97, moduli=moduli)
    last = len(moduli) - 1
    sk = oracle.SecretKey(par, rng)
    ksk = oracle.KeySwitchingKey(sk, oracle.Poly.random(par.context_at_level(last), oracle.POWER_BASIS, rng), last,
                                 last, rng)
    good = ow.ksk_to_bytes(ksk)
    bad = []
    for field, change in (("c0", -1), ("c0", 1), ("c1", -1), ("c1", 1)):
        m = ow.KeySwitchingKeyProto()
        m.ParseFromString(good)
        rep = getattr(m, field)
        if change < 0:
            del rep[-1]
        else:
            rep.append(rep[0])
        bad.append((field, m.SerializeToString()))
    return par, ksk, good, bad


@pytest.mark.parametrize("bits", [11, 17, 31, 45, 61, 62, 30, 10])
def test_key_codecs_digit_counts(oracle, ow, F, tmp_path, bits):
    """the oracle's codec, the Python mirror's and the C++ host's on the key message of a last-level key: the right
    count (3 digits at odd widths) passes every check; one polynomial more or less in c0 or c1 is WrongPolynomialCount;
    and so is a 3-digit message read with a set whose q_0 has an even width (2 digits), and vice versa"""
    from fhe_rs_b200 import _capi
    rng = np.random.default_rng(bits)
    par, ksk, good, bad = key_messages(oracle, ow, bits, rng)
    assert len(ksk.c0) == (3 if bits % 2 else 2)
    back = ow.ksk_from_bytes(par, good)
    assert back.log_base == ksk.log_base and all((a.c == b.c).all() for a, b in zip(back.c0 + back.c1, ksk.c0 + ksk.c1))
    gpar = F.BfvParameters(16, 97, moduli=par.moduli, device=-1)
    with pytest.raises(F.FheError) as e:              # past every message check: the upload needs the device
        F.KeySwitchingKey.from_bytes(gpar, good)
    assert e.value.code == _capi.NO_DEVICE and not isinstance(e.value, F.WireError)
    for field, msg in bad:
        with pytest.raises(ow.WireError, match="WrongPolynomialCount:KeySwitchingKey" + field.upper()):
            ow.ksk_from_bytes(par, msg)
        with pytest.raises(F.WireError) as e:
            F.KeySwitchingKey.from_bytes(gpar, msg)
        assert e.value.variant == "WrongPolynomialCount" and e.value.code == _capi.BAD_POLY_COUNT
        assert "KeySwitchingKey" + field.upper() in str(e.value)
    run = ksk_codec(tmp_path)
    res = run(16, 97, par.moduli, -1, [good] + [m for _, m in bad])
    assert res[0] == ("e", str(_capi.NO_DEVICE).encode())
    assert all(r == ("w", b"WrongPolynomialCount") for r in res[1:])
    # the same bytes under a q_0 one bit wider (narrower at 62): the count is ceil(width / the message's log_base)
    # (:406-411), checked before anything else is read: 10 -> 11 and 30 -> 31 bits take a 2-digit message to a set
    # that wants 3 (at the odd widths and 62 -> 61 the count still fits)
    other = bits + 1 if bits < 62 else 61
    if -(-other // ksk.log_base) != len(ksk.c0):
        opar = oracle.BfvParameters(16, 97, moduli=E.decomposition_moduli(other, 16))
        gopar = F.BfvParameters(16, 97, moduli=opar.moduli, device=-1)
        with pytest.raises(ow.WireError, match="WrongPolynomialCount:KeySwitchingKeyC0"):
            ow.ksk_from_bytes(opar, good)
        with pytest.raises(F.WireError) as e:
            F.KeySwitchingKey.from_bytes(gopar, good)
        assert e.value.variant == "WrongPolynomialCount"
        assert run(16, 97, opar.moduli, -1, [good]) == [("w", b"WrongPolynomialCount")]
    else:
        assert bits % 2 == 1 or bits == 62


# ---------------------------------------------------------------------------------------------- parameter sets

def test_width_sets(oracle, F):
    """the sets of tests/test_gpu_widths.py: the N = 64 sets cover every width from 10 to 62, with q_0 narrow in two
    and wide in two, t below every q_0; the host tables of each build; the lazy-bound bases sit on either side of
    the reduce-on-load decision"""
    covered = []
    for name, (degree, t, sizes) in E.WIDTH_SETS.items():
        moduli = oracle.BfvParameters.generate_moduli(sizes, degree)
        assert [q.bit_length() for q in moduli] == sizes and t < moduli[0], name
        gpar = F.BfvParameters(degree, t, moduli=moduli, device=-1)
        assert gpar.moduli() == moduli
        if degree == 64:
            covered += sizes
    assert sorted(covered) == WIDTHS
    assert sorted(E.WIDTH_SETS[n][2][0] for n in E.WIDTH_SETS if n.startswith("n64")) == [10, 11, 60, 61]
    for degree in (1 << 13,):
        b = E.lazy_bound_bases(degree)
        qi, qj = max(b["unreduced"]), b["unreduced"][1]
        assert qj > 1 << 60 and qi - 1 < 4 * qj and 4 * qj - qi < 1 << 21       # unreduced, within a hair of 4 q_j
        qi, qj = max(b["reduced"]), b["reduced"][1]
        assert qj < 1 << 60 and qi - 1 >= 4 * qj                                # must be reduced
        qi, qj = max(b["reduced_8x"]), b["reduced_8x"][1]
        assert 4 * qj < qi < 8 * qj and 8 * qj - qi < 1 << 53
        for moduli in b.values():
            assert all(q % (2 * degree) == 1 and oracle.is_prime(q) for q in moduli)
            F.BfvParameters(degree, 786433, moduli=moduli, device=-1)
    # 65537 = 2^16 + 1: a 17-bit field, accepted by the library's modulus check
    F.BfvParameters(16, 97, moduli=[E.prime_of_width(62, 16), 65537], device=-1)

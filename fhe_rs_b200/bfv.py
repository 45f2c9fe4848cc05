"""Host-side mirror of the reference's `fhe::bfv` interface for the accelerated path
(BfvParameters, Ciphertext, Multiplicator, RelinearizationKey, GaloisKey / EvaluationKey),
implemented purely on top of the C ABI in include/fhe_b200.h.

Same names, argument meaning and error behaviour as the reference items cited in each
docstring (paths relative to /root/reference/crates).  Differences forced by the device:
a `Ciphertext` here is a *batch* of ciphertexts of one level resident in HBM (the reference's
operators act on one ciphertext; per-ciphertext FFI would be launch/PCIe bound, SURVEY 8b),
and keys are either generated on the device from a SecretKey and a seeded ChaCha20 stream or constructed from
their NTT-domain words (as after deserialization, key_switching_key.rs:418-482).
No CPU fallback exists: every operation is a CUDA launch behind the C ABI."""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _capi, wire
from ._capi import NTT, POWER_BASIS, FheError, check
from .wire import WireError

__all__ = ["BfvParameters", "BfvParametersBuilder", "Ciphertext", "KeySwitchingKey", "RelinearizationKey", "RGSWCiphertext",
           "GaloisKey", "EvaluationKey", "Multiplicator", "ScalingFactor", "dot_product_scalar", "FheError", "WireError", "NTT", "POWER_BASIS",
           "Encoding", "Plaintext", "PlaintextVec", "SecretKey", "PublicKey", "EvaluationKeyBuilder",
           "transcode_bidirectional", "transcode_to_bytes", "transcode_from_bytes", "key_switch_keyed",
           "relinearizes_keyed", "multiply_keyed", "galois_keyed", "rotates_columns_by_keyed", "rotates_rows_keyed",
           "expands_keyed", "expands_batch_keyed", "external_products_keyed", "galois_many", "galois_many_hoisted",
           "linear_transform", "linear_transform_steps", "encode_diagonals",
           "computes_inner_sum_keyed", "dot_product", "dot_product_keyed"]


def _release(free_name: str, handle) -> None:
    """Call a C-ABI destructor from __del__; at interpreter shutdown the module globals may already be gone, in which
    case the process is about to release everything anyway."""
    try:
        getattr(_capi.lib(), free_name)(handle)
    except Exception:  # noqa: BLE001
        pass


def _ptr(a: np.ndarray) -> int:
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data


class BfvParameters:
    """fhe::bfv::BfvParameters (bfv/parameters.rs:88-114), built by
    BfvParametersBuilder::build (:560-738).  `device=-1` builds the host tables only."""

    def __init__(self, degree: int, plaintext_modulus: int, moduli: Optional[Sequence[int]] = None,
                 moduli_sizes: Optional[Sequence[int]] = None, psi: Optional[Sequence[int]] = None,
                 device: int = 0, plaintext_psi: Optional[int] = None, variance: int = 10):
        """plaintext_psi: the 2N-th root of unity for the plaintext modulus (the reference's
        NttOperator::new(t).omegas[N/2], for SIMD words interchangeable with a Rust process); None selects the
        default rule of fhe_b200_params_create.  variance: BfvParameters::variance, the parameter of the centred
        binomial errors of encryption, 1..32 (parameters.rs:384-388, :449-454)."""
        L = _capi.lib()
        if not 1 <= int(variance) <= 32:
            raise FheError(_capi.INVALID_ARGUMENT, "InvalidVariance: %d is outside 1..32" % variance)
        self.variance = int(variance)
        self._enc = None
        self._plaintext_psi = plaintext_psi
        if (moduli is None) == (moduli_sizes is None):
            # parameters.rs:455-466
            raise FheError(_capi.INVALID_ARGUMENT, "exactly one of moduli / moduli_sizes must be given")
        pt = int(plaintext_modulus)
        if pt <= 0:
            raise FheError(_capi.INVALID_ARGUMENT, "plaintext modulus must be positive")
        pt_bytes = pt.to_bytes(max(1, (pt.bit_length() + 7) // 8), "little")
        buf = (C.c_uint8 * len(pt_bytes)).from_buffer_copy(pt_bytes)
        h = C.c_void_p()
        if moduli is not None:
            m = np.ascontiguousarray(np.array([int(x) for x in moduli], dtype=np.uint64))
            ps = None
            if psi is not None:
                ps = np.ascontiguousarray(np.array([int(x) for x in psi], dtype=np.uint64))
                if len(ps) != 2 * len(m) + 1:
                    raise FheError(_capi.INVALID_ARGUMENT, "psi needs one root per modulus and extension prime")
            check(L.fhe_b200_params_create(device, degree, _ptr(m), len(m), C.addressof(buf), len(pt_bytes),
                                           _ptr(ps) if ps is not None else None, C.byref(h)))
        else:
            if psi is not None:
                raise FheError(_capi.INVALID_ARGUMENT, "psi requires explicit moduli")
            s = np.ascontiguousarray(np.array(list(moduli_sizes), dtype=np.uint32))
            check(L.fhe_b200_params_create_from_sizes(device, degree, s.ctypes.data, len(s), C.addressof(buf),
                                                      len(pt_bytes), C.byref(h)))
        self._h = h
        self.device = device
        self._plaintext = pt
        self._degree = L.fhe_b200_params_degree(h)
        n = L.fhe_b200_params_n_moduli(h)
        out = np.zeros(n, np.uint64)
        check(L.fhe_b200_params_moduli(h, _ptr(out)))
        self._moduli = [int(x) for x in out]

    def __del__(self):
        e, self._enc = getattr(self, "_enc", None), None
        if e:
            _release("fhe_b200_encoder_free", e)
        h, self._h = getattr(self, "_h", None), None
        if h:
            _release("fhe_b200_params_destroy", h)

    def encoder(self):
        """the fhe_b200_encoder handle (ntt_operator + matrix_reps_index_map, parameters.rs:71-75, :713-726),
        created on first use"""
        if self._enc is None:
            h = C.c_void_p()
            psi = C.c_uint64(int(self._plaintext_psi)) if self._plaintext_psi is not None else None
            check(_capi.lib().fhe_b200_encoder_create(self._h, C.byref(psi) if psi is not None else None, C.byref(h)))
            self._enc = h
        return self._enc

    def encoder_tables(self, level: int = 0) -> Dict[str, object]:
        """Host precompute inspection: SIMD index map, NTT tables of t (None when t has no NTT operator), and the
        level's q_mod_t and delta residues."""
        L, n = _capi.lib(), self._degree
        imap, om, zi = np.zeros(n, np.uint32), np.zeros(n, np.uint64), np.zeros(n, np.uint64)
        qmt, delta = C.c_uint64(), np.zeros(len(self._moduli) - level, np.uint64)
        code = L.fhe_b200_debug_encoder_tables(self.encoder(), level, None, _ptr(om), _ptr(zi), None, None)
        if code not in (_capi.OK, _capi.NTT_UNAVAILABLE):
            check(code)
        check(L.fhe_b200_debug_encoder_tables(self.encoder(), level, _ptr(imap), None, None, C.byref(qmt), _ptr(delta)))
        has_ntt = code == _capi.OK
        return dict(index_map=imap, omegas=om if has_ntt else None, zetas_inv=zi if has_ntt else None,
                    q_mod_t=qmt.value, delta=delta)

    def degree(self) -> int:  # parameters.rs:130
        return self._degree

    def to_bytes(self) -> bytes:
        """BfvParameters::to_bytes (parameters.rs:741-759): the Parameters message (bfv.proto:40-48)"""
        return wire.encode_parameters(self._degree, self._moduli, self._plaintext, self.variance)

    @staticmethod
    def from_bytes(data: bytes, device: int = 0) -> "BfvParameters":
        """BfvParameters::try_deserialize (parameters.rs:762-789): built with the message's explicit moduli and variance,
        so every builder error keeps its code (a variance of 0, the proto3 default, is InvalidVariance)."""
        degree, moduli, plaintext, variance = wire.decode_parameters(data)
        return BfvParameters(degree, plaintext, moduli=moduli, device=device, variance=variance)

    def moduli(self):  # parameters.rs:136
        return list(self._moduli)

    def plaintext(self) -> int:
        return self._plaintext

    def max_level(self) -> int:  # parameters.rs:173
        return len(self._moduli) - 1

    def mul_basis(self, level: int = 0):
        """level moduli followed by the extension primes (parameters.rs:660-700)."""
        L = _capi.lib()
        n = C.c_uint32()
        check(L.fhe_b200_params_mul_basis(self._h, level, None, C.byref(n)))
        out = np.zeros(n.value, np.uint64)
        check(L.fhe_b200_params_mul_basis(self._h, level, _ptr(out), C.byref(n)))
        return [int(x) for x in out]

    def psi(self, q: int) -> int:
        r = C.c_uint64()
        check(_capi.lib().fhe_b200_params_psi(self._h, q, C.byref(r)))
        return r.value

    def scaler_tables(self, level: int, which: int) -> Dict[str, object]:
        """Host precompute inspection: RnsScaler tables (rns/scaler.rs:52-73)."""
        L = _capi.lib()
        nf, nt, sh = C.c_uint32(), C.c_uint32(), C.c_uint32()
        check(L.fhe_b200_debug_scaler_tables(self._h, level, which, C.byref(nf), C.byref(nt), C.byref(sh),
                                             *([None] * 8)))
        f, t = nf.value, nt.value
        gamma, omega, tg = np.zeros(t, np.uint64), np.zeros((t, f), np.uint64), np.zeros(3, np.uint64)
        tol, toh, tos = np.zeros(f, np.uint64), np.zeros(f, np.uint64), np.zeros(f, np.uint8)
        tgl, tgh = np.zeros(f, np.uint64), np.zeros(f, np.uint64)
        check(L.fhe_b200_debug_scaler_tables(self._h, level, which, C.byref(nf), C.byref(nt), C.byref(sh),
                                             _ptr(gamma), _ptr(omega), _ptr(tg), _ptr(tol), _ptr(toh), _ptr(tos),
                                             _ptr(tgl), _ptr(tgh)))
        return dict(n_from=f, n_to=t, shift=sh.value, gamma=gamma, omega=omega, theta_gamma=tg,
                    theta_omega_lo=tol, theta_omega_hi=toh, theta_omega_sign=tos,
                    theta_garner_lo=tgl, theta_garner_hi=tgh)

    def ntt_tables(self, q: int) -> Dict[str, object]:
        n = self._degree
        om, oms, zi, zis = (np.zeros(n, np.uint64) for _ in range(4))
        ninv = C.c_uint64()
        check(_capi.lib().fhe_b200_debug_ntt_tables(self._h, q, _ptr(om), _ptr(oms), _ptr(zi), _ptr(zis),
                                                    C.byref(ninv)))
        return dict(omegas=om, omegas_shoup=oms, zetas_inv=zi, zetas_inv_shoup=zis, size_inv=ninv.value)


class BfvParametersBuilder:
    """fhe::bfv::BfvParametersBuilder (bfv/parameters.rs:319-388)."""

    def __init__(self):
        self._degree = 0
        self._plaintext = 0
        self._moduli = None
        self._sizes = None
        self._psi = None
        self._variance = 10

    def set_degree(self, degree: int):
        self._degree = degree
        return self

    def set_plaintext_modulus(self, t: int):
        self._plaintext = t
        return self

    def set_moduli(self, moduli: Sequence[int]):
        self._moduli = list(moduli)
        return self

    def set_moduli_sizes(self, sizes: Sequence[int]):
        self._sizes = list(sizes)
        return self

    def set_ntt_roots(self, psi: Sequence[int]):
        """2N-th roots per [moduli..., extension primes...] (the reference's own, for interchange)."""
        self._psi = list(psi)
        return self

    def set_variance(self, variance: int):
        """the error variance, 1..32 (checked by build, parameters.rs:384-388)"""
        self._variance = variance
        return self

    def build(self, device: int = 0) -> BfvParameters:
        return BfvParameters(self._degree, self._plaintext, self._moduli, self._sizes, self._psi, device,
                             variance=self._variance)

    build_arc = build


class Ciphertext:
    """A device-resident batch of fhe::bfv::Ciphertext (bfv/ciphertext.rs:18-32): `count`
    ciphertexts of `parts` polynomials at `level`, words [count][parts][limbs][N]."""

    def __init__(self, par: BfvParameters, count: int, parts: int = 2, level: int = 0, repr: int = NTT,
                 stream: int = 0, mul_basis: bool = False):
        h = C.c_void_p()
        f = _capi.lib().fhe_b200_batch_alloc_mul_basis if mul_basis else _capi.lib().fhe_b200_batch_alloc
        check(f(par._h, count, parts, level, repr, C.byref(h)))
        self._h, self.par, self.stream, self.mul_basis = h, par, stream, mul_basis

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            _release("fhe_b200_batch_free", h)

    # -- shape
    def _info(self):
        c, p, lv, lm, r = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_int()
        check(_capi.lib().fhe_b200_batch_info(self._h, C.byref(c), C.byref(p), C.byref(lv), C.byref(lm), C.byref(r)))
        return c.value, p.value, lv.value, lm.value, r.value

    @property
    def count(self):
        return self._info()[0]

    def __len__(self):  # Ciphertext::len -> number of polynomials (ciphertext.rs:118)
        return self._info()[1]

    @property
    def level(self):
        return self._info()[2]

    @property
    def limbs(self):
        return self._info()[3]

    @property
    def representation(self):
        return self._info()[4]

    def shape(self):
        c, p, _, lm, _ = self._info()
        return (c, p, lm, self.par.degree())

    # -- transfer
    @staticmethod
    def from_host(par: BfvParameters, words: np.ndarray, level: int = 0, repr: int = NTT, stream: int = 0,
                  mul_basis: bool = False) -> "Ciphertext":
        """words: u64 [count][parts][limbs][N] as Vec<u64>::from(&Poly) (rq/convert.rs:474-503)."""
        words = np.ascontiguousarray(words, dtype=np.uint64)
        if words.ndim != 4 or words.shape[3] != par.degree():
            raise FheError(_capi.INVALID_ARGUMENT, "expected [count][parts][limbs][N] words")
        ct = Ciphertext(par, words.shape[0], words.shape[1], level, repr, stream, mul_basis)
        if ct.limbs != words.shape[2]:
            raise FheError(_capi.CONTEXT_MISMATCH, "limb count does not match the level")
        check(_capi.lib().fhe_b200_batch_upload(ct._h, 0, words.shape[0], _ptr(words), stream))
        check(_capi.lib().fhe_b200_sync(stream))
        return ct

    def _check_words(self, words: np.ndarray, first: int):
        """[n][parts][limbs][N] contiguous u64 with first + n <= count -- anything else would overrun a buffer"""
        shape = self.shape()
        if words.dtype != np.uint64 or not words.flags["C_CONTIGUOUS"]:
            raise FheError(_capi.INVALID_ARGUMENT, "expected a C-contiguous uint64 array")
        if words.ndim != 4 or tuple(words.shape[1:]) != tuple(shape[1:]):
            raise FheError(_capi.INVALID_ARGUMENT, "expected [n][%d][%d][%d] words" % tuple(shape[1:]))
        if first < 0 or first + words.shape[0] > shape[0]:
            raise FheError(_capi.INVALID_ARGUMENT, "range exceeds batch")

    def upload(self, words: np.ndarray, first: int = 0):
        words = np.ascontiguousarray(words, dtype=np.uint64)
        self._check_words(words, first)
        check(_capi.lib().fhe_b200_batch_upload(self._h, first, words.shape[0], _ptr(words), self.stream))
        check(_capi.lib().fhe_b200_sync(self.stream))   # `words` may be a temporary: do not return before it is read

    def to_host(self, out: Optional[np.ndarray] = None, first: int = 0) -> np.ndarray:
        """ciphertexts [first, first + len(out)) (all of them from `first` on when out is None)"""
        if out is None:
            shape = self.shape()
            out = np.empty((shape[0] - first,) + tuple(shape[1:]), np.uint64)
        self._check_words(out, first)
        check(_capi.lib().fhe_b200_batch_download(self._h, first, out.shape[0], _ptr(out), self.stream))
        return out

    # -- wire format (rq/convert.rs:17-131): Rq.coefficients blobs, one per polynomial
    def packed_bytes_per_poly(self) -> int:
        n = C.c_size_t()
        check(_capi.lib().fhe_b200_batch_packed_bytes(self._h, C.byref(n)))   # per batch: a mul-basis batch has L + E limbs
        return n.value

    def to_packed(self) -> np.ndarray:
        """[count][parts][packed_bytes] uint8: what `Rq::from(&poly).coefficients` holds for every polynomial"""
        c, p, _, _, _ = self._info()
        out = np.empty((c, p, self.packed_bytes_per_poly()), np.uint8)
        check(_capi.lib().fhe_b200_batch_pack(self._h, 0, c, _ptr(out), self.stream))
        return out

    @staticmethod
    def from_packed(par: "BfvParameters", blobs: np.ndarray, level: int = 0, repr: int = NTT,
                    stream: int = 0) -> "Ciphertext":
        """inverse of to_packed: `Poly::<R>::try_convert_from(&Rq, ctx, ..)` for every polynomial"""
        blobs = np.ascontiguousarray(blobs, dtype=np.uint8)
        ct = Ciphertext(par, blobs.shape[0], blobs.shape[1], level, repr, stream)
        if blobs.shape[2] != ct.packed_bytes_per_poly():
            raise FheError(_capi.INVALID_ARGUMENT, "InvalidCoefficientCount: blob size does not match the context")
        check(_capi.lib().fhe_b200_batch_unpack(ct._h, 0, blobs.shape[0], _ptr(blobs), stream))
        check(_capi.lib().fhe_b200_sync(stream))
        return ct

    # -- protobuf messages (bfv/ciphertext.rs:230-317; fhe_traits::Serialize / DeserializeParametrized)
    def to_bytes(self) -> list:
        """`ct.to_bytes()` for every ciphertext of the batch: one encoded fhers.bfv.Ciphertext each, every part an
        fhers.rq.Rq with representation NTT (the unseeded branch of ciphertext.rs:240-252).  The coefficient packing
        runs on the device; only the few bytes of framing are host work."""
        c, p, lv, _, r = self._info()
        if r != NTT:
            raise FheError(_capi.INVALID_REPRESENTATION, "Ciphertext polynomials are Poly<Ntt> (ciphertext.rs:18-32)")
        blobs = self.to_packed()
        self.sync()
        deg = self.par.degree()
        return [wire.encode_ciphertext([wire.encode_rq(wire.REP_NTT, deg, memoryview(blobs[i, j])) for j in range(p)],
                                       b"", lv) for i in range(c)]

    @staticmethod
    def from_bytes(par: "BfvParameters", messages: Sequence[bytes], seeded_halves: Optional[np.ndarray] = None,
                   stream: int = 0) -> "Ciphertext":
        """`Ciphertext::from_bytes(bytes, &par)` (ciphertext.rs:259-317) for a batch of messages of one level and part
        count.  A message that carries a seed instead of its last polynomial needs `seeded_halves[i]`: the NTT words
        [limbs][N] of `Poly::random_from_seed(ctx, seed)`, expanded by the Rust host (include/fhe_b200.h explains why
        the device does not)."""
        if len(messages) == 0:
            raise FheError(_capi.INVALID_ARGUMENT, "no messages")
        dec = [wire.decode_ciphertext(m) for m in messages]
        level = dec[0][2]
        if level > par.max_level():
            raise WireError("InvalidLevel", _capi.INVALID_LEVEL, "level %d, max %d" % (level, par.max_level()))
        n_rq = len(dec[0][0])
        seeded = bool(dec[0][1])
        for c, seed, lv in dec:
            if lv != level or len(c) != n_rq or bool(seed) != seeded:
                raise FheError(_capi.INVALID_ARGUMENT, "a batch holds ciphertexts of one level, part count and kind")
            if seed and len(seed) != 32:
                raise WireError("InvalidSeedSize", detail="%d bytes, expected 32" % len(seed))
        body = Ciphertext(par, len(dec), n_rq, level, NTT, stream)
        _unpack_rq(body, [c for c, _, _ in dec], wire.REP_NTT)
        if not seeded:
            return body
        if seeded_halves is None:
            raise WireError("SeedExpansion", _capi.UNSUPPORTED,
                            "the message carries a seed: pass the host-expanded last polynomial (ciphertext.rs:287-300)")
        halves = np.ascontiguousarray(seeded_halves, dtype=np.uint64)
        if halves.shape != (len(dec), body.limbs, par.degree()):
            raise FheError(_capi.INVALID_ARGUMENT, "expected seeded_halves as [count][limbs][N]")
        words = np.concatenate([body.to_host(), halves[:, None]], axis=1)
        return Ciphertext.from_host(par, words, level, NTT, stream)

    def device_ptr(self) -> int:
        p, n = C.c_void_p(), C.c_size_t()
        check(_capi.lib().fhe_b200_batch_device_ptr(self._h, C.byref(p), C.byref(n)))
        return p.value

    def sync(self):
        check(_capi.lib().fhe_b200_sync(self.stream))

    def _like(self, parts: Optional[int] = None, level: Optional[int] = None) -> "Ciphertext":
        c, p, lv, _, r = self._info()
        return Ciphertext(self.par, c, parts or p, lv if level is None else level, r, self.stream)

    def clone(self) -> "Ciphertext":
        out = self._like()
        check(_capi.lib().fhe_b200_batch_copy(out._h, self._h, self.stream))
        return out

    def take(self, first: int, n: int, stride: int = 1) -> "Ciphertext":
        """a new batch of the n ciphertexts first, first + stride, ..., first + (n-1)*stride (fhe_b200_batch_copy_range)"""
        c, p, lv, _, r = self._info()
        out = Ciphertext(self.par, n, p, lv, r, self.stream)
        check(_capi.lib().fhe_b200_batch_copy_range(out._h, 0, self._h, first, stride, n, self.stream))
        return out

    # -- representation (Poly::into_ntt / into_power_basis, rq/mod.rs:535, :590)
    def into_ntt(self) -> "Ciphertext":
        check(_capi.lib().fhe_b200_ntt_forward(self._h, self.stream))
        return self

    def into_power_basis(self) -> "Ciphertext":
        check(_capi.lib().fhe_b200_ntt_backward(self._h, self.stream))
        return self

    # -- operators (bfv/ops/mod.rs:15-358)
    def __iadd__(self, rhs: "Ciphertext"):
        check(_capi.lib().fhe_b200_add(self._h, rhs._h, self.stream))
        return self

    def __isub__(self, rhs: "Ciphertext"):
        check(_capi.lib().fhe_b200_sub(self._h, rhs._h, self.stream))
        return self

    def __add__(self, rhs: "Ciphertext") -> "Ciphertext":
        out = self.clone()
        out += rhs
        return out

    def __sub__(self, rhs: "Ciphertext") -> "Ciphertext":
        out = self.clone()
        out -= rhs
        return out

    def __neg__(self) -> "Ciphertext":
        out = self.clone()
        check(_capi.lib().fhe_b200_neg(out._h, out.stream))
        return out

    def sum(self, n_terms: Optional[int] = None, out: Optional["Ciphertext"] = None) -> "Ciphertext":
        """Ciphertext += folded over runs (bfv/ops/mod.rs:54-69): entry g of the result is the sum of entries
        g*n_terms .. g*n_terms + n_terms - 1.  n_terms None sums the whole batch into one ciphertext.  The result
        has this batch's parts, level, representation and basis (the multiplication basis included).  With `out`, the
        sums are added to out's entries and out is returned.  One device call (fhe_b200_batch_sum)."""
        count = self.count
        n = count if n_terms is None else int(n_terms)
        if n <= 0 or count % n:
            raise FheError(_capi.INVALID_ARGUMENT, "a batch of %d entries does not split into runs of %s" % (count, n_terms))
        if out is None:
            c, p, lv, _, r = self._info()
            res = Ciphertext(self.par, c // n, p, lv, r, self.stream, self.mul_basis)
        else:
            res = out
        check(_capi.lib().fhe_b200_batch_sum(self._h, n, 0 if out is None else 1, res._h, self.stream))
        return res

    def __mul__(self, rhs: "Ciphertext") -> "Ciphertext":
        """&Ciphertext * &Ciphertext, no relinearization (ops/mod.rs:259-358): n x m parts -> n + m - 1 parts."""
        out = self._like(parts=len(self) + len(rhs) - 1)
        check(_capi.lib().fhe_b200_mul(self._h, rhs._h, out._h, self.stream))
        return out

    def mul_plain(self, poly_ntt) -> "Ciphertext":
        """Ciphertext *= &Plaintext (ops/mod.rs:229-238), in place.  poly_ntt: a device `Plaintext` / `PlaintextVec`
        (1 or count entries), or the plaintext's `poly_ntt` words, [limbs][N] (shared by the batch) or
        [count][limbs][N] (one plaintext per ciphertext)."""
        if isinstance(poly_ntt, PlaintextVec):
            check(_capi.lib().fhe_b200_mul_plain_batch(self._h, poly_ntt.batch._h, self.stream))
            return self
        w = np.ascontiguousarray(poly_ntt, dtype=np.uint64)
        n = 1 if w.ndim == 2 else w.shape[0]
        check(_capi.lib().fhe_b200_mul_plain(self._h, _ptr(w), n, self.stream))
        return self

    def switch_down(self) -> "Ciphertext":
        """Ciphertext::switch_down (ciphertext.rs:148-161), in place."""
        check(_capi.lib().fhe_b200_switch_down(self._h, self.stream))
        return self

    def add_plain(self, poly, subtract: bool = False) -> "Ciphertext":
        """Ciphertext += &Plaintext / -= &Plaintext (ops/mod.rs:88-97, :188-197), in place: `poly` is a device
        `Plaintext` / `PlaintextVec` (to_poly() is derived on the device), or the plaintext's `to_poly()` words
        (delta-scaled, NTT), [limbs][N] shared by the batch or [count][limbs][N]."""
        if isinstance(poly, PlaintextVec):
            check(_capi.lib().fhe_b200_add_plain_batch(self._h, poly.batch._h, 1 if subtract else 0, self.stream))
            return self
        w = np.ascontiguousarray(poly, dtype=np.uint64)
        n = 1 if w.ndim == 2 else w.shape[0]
        check(_capi.lib().fhe_b200_add_plain(self._h, _ptr(w), n, 1 if subtract else 0, self.stream))
        return self

    def sub_plain(self, poly: np.ndarray) -> "Ciphertext":
        return self.add_plain(poly, subtract=True)

    def max_switchable_level(self) -> int:  # ciphertext.rs:187-189
        return self.par.max_level()

    def switch_to_level(self, target_level: int) -> "Ciphertext":
        """Ciphertext::switch_to_level (ciphertext.rs:164-184): only moves down; InvalidLevel otherwise."""
        if target_level < self.level or target_level > self.max_switchable_level():
            raise FheError(_capi.INVALID_LEVEL, "InvalidLevel: level %d, min %d, max %d"
                           % (target_level, self.level, self.max_switchable_level()))
        while self.level < target_level:
            self.switch_down()
        return self

    def substitute(self, exponent: int) -> "Ciphertext":
        """Poly::substitute on every polynomial, in either representation (rq/mod.rs:360-408)."""
        out = self._like()
        check(_capi.lib().fhe_b200_substitute(self._h, exponent, out._h, self.stream))
        return out

    def fold(self, in_bits: int, out_bits: int, level: int) -> "PlaintextVec":
        """The reply fold of the SealPIR server (examples/sealpir.rs:176-200) of every ciphertext: the stored words of
        each part transcoded from in_bits to out_bits, concatenated over the parts and encoded as
        PlaintextVec::try_encode(values, Encoding::poly_at_level(level)) (fhe_b200_fold).  Plaintext i of ciphertext
        j is entry i * count + j of the result, the operand dot_product_scalar(selectors, pts, n_terms=count) takes."""
        n = self.par.degree()
        per_ct = 1
        if 1 <= in_bits <= 64 and 1 <= out_bits <= 64:     # (otherwise fhe_b200_fold refuses the widths)
            e = -(-self.limbs * n * in_bits // out_bits)
            per_ct = -(-len(self) * e // n)
        out = Ciphertext(self.par, per_ct * self.count, 1, level, NTT, self.stream)
        check(_capi.lib().fhe_b200_fold(self._h, in_bits, out_bits, out._h, self.stream))
        return PlaintextVec(out, Encoding.poly_at_level(level))

    def scale(self, which: int) -> "Ciphertext":
        """Poly::scale with the level's extender (0) / down scaler (1) (rq/mod.rs:669, rq/scaler.rs:55)."""
        c, p, lv, _, r = self._info()
        out = Ciphertext(self.par, c, p, lv, r, self.stream, mul_basis=(which == 0))
        check(_capi.lib().fhe_b200_scale(self._h, which, out._h, self.stream))
        return out


class Encoding:
    """fhe::bfv::Encoding (bfv/encoding.rs): Poly or Simd, at a level."""

    def __init__(self, kind: int, level: int = 0):
        self.kind, self.level = kind, level

    @staticmethod
    def poly() -> "Encoding":
        return Encoding(_capi.ENCODING_POLY)

    @staticmethod
    def simd() -> "Encoding":
        return Encoding(_capi.ENCODING_SIMD)

    @staticmethod
    def poly_at_level(level: int) -> "Encoding":
        return Encoding(_capi.ENCODING_POLY, level)

    @staticmethod
    def simd_at_level(level: int) -> "Encoding":
        return Encoding(_capi.ENCODING_SIMD, level)

    def __eq__(self, o):
        return isinstance(o, Encoding) and (self.kind, self.level) == (o.kind, o.level)

    def __repr__(self):
        return "Encoding(%s, level=%d)" % ("simd" if self.kind == _capi.ENCODING_SIMD else "poly", self.level)


def _values_source(values):
    """(pointer, count, is_signed, keep-alive) of the values to encode.  numpy arrays (and sequences) live in
    pageable host memory; a torch tensor may be pinned host or CUDA memory.  The signedness is the dtype's: signed
    64-bit words are reduced into [0, t) first (the reference's &[i64] encoders), unsigned ones are not."""
    if hasattr(values, "data_ptr") and hasattr(values, "is_cuda"):   # torch.Tensor
        import torch
        if values.dtype not in (torch.int64, torch.uint64) or not values.is_contiguous():
            raise FheError(_capi.INVALID_ARGUMENT, "expected a contiguous int64 or uint64 tensor")
        return values.data_ptr(), values.numel(), values.dtype == torch.int64, values
    a = np.asarray(values)
    if a.size == 0:
        a = np.zeros(0, np.uint64)
    if a.dtype.kind not in "iu" or a.ndim != 1:
        raise FheError(_capi.INVALID_ARGUMENT, "expected a 1-D array of 64-bit integers")
    a = np.ascontiguousarray(a, dtype=np.int64 if a.dtype.kind == "i" else np.uint64)
    return a.ctypes.data, a.size, a.dtype.kind == "i", a


class PlaintextVec:
    """fhe::bfv::PlaintextVec (bfv/plaintext_vec.rs:20-103): `count` plaintexts of one encoding, their poly_ntt
    resident on the device as a 1-part batch (`batch`, [count][1][limbs][N])."""

    def __init__(self, batch: Ciphertext, encoding: Encoding):
        self.batch, self.encoding, self.par = batch, encoding, batch.par

    @classmethod
    def try_encode(cls, values, encoding: Encoding, par: BfvParameters, stream: int = 0):
        """PlaintextVec::try_encode (plaintext_vec.rs:37-103) on the device: values[k*N, (k+1)*N) become plaintext k.
        `values`: a 1-D int64 / uint64 numpy array or sequence, or a contiguous torch tensor (pinned host or CUDA)."""
        ptr, n, signed, keep = _values_source(values)
        cls._check_count(n, par)
        count = max(1, -(-n // par.degree()))
        batch = Ciphertext(par, count, 1, encoding.level, NTT, stream)
        check(_capi.lib().fhe_b200_encode(par.encoder(), encoding.kind, 1 if signed else 0, ptr if n else None, n,
                                          batch._h, stream))
        check(_capi.lib().fhe_b200_sync(stream))   # `values` may be a temporary: it has been read when this returns
        del keep
        return cls(batch, encoding)

    @staticmethod
    def _check_count(n: int, par: BfvParameters):
        """a PlaintextVec takes any number of values (Plaintext overrides this)"""

    def __len__(self):
        return self.batch.count

    @property
    def level(self) -> int:
        return self.batch.level

    def poly_ntt(self) -> np.ndarray:
        """the poly_ntt words of every plaintext, [count][limbs][N]"""
        return self.batch.to_host()[:, 0]

    def resolve_encoding(self, encoding: Optional[Encoding] = None) -> Encoding:
        """Plaintext::resolve_encoding (plaintext.rs:137-153)"""
        if self.encoding is None and encoding is None:
            raise FheError(_capi.INVALID_ARGUMENT, "PlaintextError::MissingEncoding")
        if self.encoding is not None and encoding is not None and self.encoding != encoding:
            raise FheError(_capi.INVALID_ARGUMENT, "EncodingError::Mismatch: found %r, expected %r"
                           % (encoding, self.encoding))
        return self.encoding if self.encoding is not None else encoding

    def try_decode(self, encoding: Optional[Encoding] = None, signed: bool = False, out=None):
        """Vec<u64>::try_decode / Vec<i64>::try_decode (signed=True) (plaintext.rs:374-459) of every plaintext on the
        device: values [count * N], plaintext k at [k*N, (k+1)*N).  `out` (optional): a contiguous numpy array or
        torch tensor (host, pinned or CUDA) of count * N 64-bit words that receives them; otherwise a new numpy array
        of uint64 (int64 when signed) is returned."""
        enc = self.resolve_encoding(encoding)
        n = self.batch.count * self.par.degree()
        if out is None:
            out = np.empty(n, np.int64 if signed else np.uint64)
        if hasattr(out, "data_ptr") and hasattr(out, "is_cuda"):   # torch.Tensor
            if out.element_size() != 8 or not out.is_contiguous() or out.numel() != n:
                raise FheError(_capi.INVALID_ARGUMENT, "expected a contiguous 64-bit tensor of %d words" % n)
            ptr = out.data_ptr()
        else:
            if out.dtype.itemsize != 8 or out.dtype.kind not in "iu" or not out.flags["C_CONTIGUOUS"] or out.size != n:
                raise FheError(_capi.INVALID_ARGUMENT, "expected a contiguous 64-bit array of %d words" % n)
            ptr = out.ctypes.data
        st = self.batch.stream
        check(_capi.lib().fhe_b200_decode(self.par.encoder(), enc.kind, 1 if signed else 0, self.batch._h, ptr, n, st))
        check(_capi.lib().fhe_b200_sync(st))
        return out


class SecretKey:
    """fhe::bfv::SecretKey (keys/secret_key.rs:25-53) on the device, from its N signed coefficients or drawn on the
    device (SecretKey.random / random_vec).  Encryption, decryption and noise measurement run on the device; the device
    copy of s is erased when the key is released.  Encryption and key generation (RelinearizationKey.new, GaloisKey.new,
    EvaluationKeyBuilder, try_encrypt_rgsw) draw their randomness from the seeded ChaCha20 stream of
    include/fhe_b200.h."""

    def __init__(self, par: BfvParameters, coeffs):
        c = np.array(coeffs, dtype=np.int64)   # our own copy, kept for to_bytes (the reference keeps SecretKey.coeffs)
        if c.ndim != 1 or c.size != par.degree():
            raise FheError(_capi.INVALID_ARGUMENT, "a secret key has N = %d coefficients" % par.degree())
        self._coeffs = c
        h = C.c_void_p()
        check(_capi.lib().fhe_b200_secret_key_create(par._h, _ptr(c), C.byref(h)))
        self._h, self.par = h, par

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            _release("fhe_b200_secret_key_free", h)
        c = getattr(self, "_coeffs", None)
        if c is not None:
            c[:] = 0

    @staticmethod
    def random(par: BfvParameters, seed: Optional[bytes] = None) -> "SecretKey":
        """SecretKey::random (secret_key.rs:42-45): s = sample_vec_cbd(N, par.variance) drawn on the device from the
        seeded stream (role 18, key 0).  seed: 32 bytes; None draws os.urandom(32) (a seed must never be reused)."""
        return SecretKey.random_vec(par, 1, seed)[0]

    @staticmethod
    def random_vec(par: BfvParameters, n: int, seed: Optional[bytes] = None) -> "List[SecretKey]":
        """n independent SecretKey::random keys in one device call (key k is stream word 13 = k), e.g. one per party of
        multiparty BFV.  The coefficients stay on the device; to_bytes downloads them."""
        hs = (C.c_void_p * max(1, int(n)))()
        check(_capi.lib().fhe_b200_secret_keys_random(par._h, int(n), par.variance, _seed(seed),
                                                      C.cast(hs, C.POINTER(C.c_void_p)), 0))
        out = []
        for h in hs[:n]:
            sk = SecretKey.__new__(SecretKey)
            sk._coeffs, sk._h, sk.par = None, C.c_void_p(h), par
            out.append(sk)
        return out

    def to_bytes(self) -> bytes:   # secret_key.rs:142-148
        if self._coeffs is not None:
            return wire.encode_secret_key(self._coeffs.tolist())
        c = self._download_coeffs()
        try:
            return wire.encode_secret_key(c.tolist())
        finally:
            c[:] = 0

    def _download_coeffs(self) -> np.ndarray:
        """the key's N signed coefficients from the device (fhe_b200_secret_key_coeffs); the caller erases them"""
        c = np.zeros(self.par.degree(), np.int64)
        check(_capi.lib().fhe_b200_secret_key_coeffs(self._h, _ptr(c), 0))
        return c

    @staticmethod
    def from_bytes(par: BfvParameters, data: bytes) -> "SecretKey":   # secret_key.rs:151-175
        return SecretKey(par, wire.decode_secret_key(data, par.degree()))

    def try_encrypt(self, pts: Optional[PlaintextVec] = None, seed: Optional[bytes] = None, count: int = 1,
                    level: int = 0) -> Ciphertext:
        """SecretKey::try_encrypt (secret_key.rs:100-136, :181-193) of every plaintext of `pts` on the device: a batch
        of one fresh ciphertext per plaintext, at the plaintexts' level.  pts None encrypts `count` zeros at `level`.
        seed: the 32 bytes that key the stream; None draws os.urandom(32) (a seed must never be reused)."""
        return _encrypt(_capi.lib().fhe_b200_encrypt_sk, self._h, self.par, pts, seed, count, level)

    def try_encrypt_rgsw(self, pts: PlaintextVec, seed: Optional[bytes] = None) -> "List[RGSWCiphertext]":
        """SecretKey::try_encrypt into an RGSWCiphertext (rgsw_ciphertext.rs:94-120) of every plaintext of `pts`, at
        the plaintexts' level, in one device call.  seed as for try_encrypt."""
        b = pts.batch
        hs = (C.c_void_p * (2 * b.count))()
        check(_capi.lib().fhe_b200_rgsw_encrypt(self._h, b._h, self.par.variance, _seed(seed),
                                                C.cast(hs, C.POINTER(C.c_void_p)), b.stream))
        k = [KeySwitchingKey._adopt(self.par, h, b.level, b.level, b.stream) for h in hs]
        return [RGSWCiphertext(k[2 * p], k[2 * p + 1]) for p in range(b.count)]

    def try_decrypt(self, ct: Ciphertext) -> PlaintextVec:
        """SecretKey::try_decrypt (secret_key.rs:198-260) of every ciphertext of the batch: plaintexts with no
        encoding (decode them with try_decode(encoding))."""
        out = Ciphertext(self.par, ct.count, 1, ct.level, NTT, ct.stream)
        check(_capi.lib().fhe_b200_decrypt(self._h, ct._h, out._h, ct.stream))
        return PlaintextVec(out, None)

    def measure_noise(self, ct: Ciphertext) -> np.ndarray:
        """SecretKey::measure_noise (secret_key.rs:55-98) of every ciphertext: uint32 [count]"""
        out = np.zeros(ct.count, np.uint32)
        check(_capi.lib().fhe_b200_measure_noise(self._h, ct._h, _ptr(out), ct.stream))
        check(_capi.lib().fhe_b200_sync(ct.stream))
        return out


def _seed(seed: Optional[bytes]) -> bytes:
    """the 32 bytes that key the device's ChaCha20 stream; None draws os.urandom(32)"""
    seed = os.urandom(32) if seed is None else bytes(seed)
    if len(seed) != 32:
        raise FheError(_capi.INVALID_ARGUMENT, "a seed is 32 bytes, got %d" % len(seed))
    return seed


def _encrypt(fn, key, par: BfvParameters, pts: Optional[PlaintextVec], seed: Optional[bytes], count: int,
             level: int) -> Ciphertext:
    seed = _seed(seed)
    b = pts.batch if pts is not None else None
    out = Ciphertext(par, b.count if b else count, 2, b.level if b else level, NTT, b.stream if b else 0)
    check(fn(key, b._h if b else None, par.variance, seed, out._h, out.stream))
    return out


class PublicKey:
    """fhe::bfv::PublicKey (keys/public_key.rs:17-22): its c, one 2-part ciphertext at level 0, on the device."""

    def __init__(self, par: BfvParameters, c: Ciphertext):
        if c.count != 1 or len(c) != 2:
            raise FheError(_capi.INVALID_ARGUMENT, "a public key is one 2-part ciphertext")
        if c.level != 0:
            raise FheError(_capi.INVALID_LEVEL, "InvalidPublicKeyLevel: %d, expected 0" % c.level)
        self.par, self.c = par, c

    @staticmethod
    def new(sk: SecretKey, seed: Optional[bytes] = None) -> "PublicKey":
        """PublicKey::new (public_key.rs:26-38): a secret-key encryption of zero at level 0"""
        return PublicKey(sk.par, sk.try_encrypt(None, seed))

    def try_encrypt(self, pts: Optional[PlaintextVec] = None, seed: Optional[bytes] = None, count: int = 1,
                    level: int = 0) -> Ciphertext:
        """PublicKey::try_encrypt (public_key.rs:45-92) of every plaintext of `pts`, as SecretKey.try_encrypt"""
        return _encrypt(_capi.lib().fhe_b200_encrypt_pk, self.c._h, self.par, pts, seed, count, level)

    def to_bytes(self) -> bytes:   # public_key.rs:95-107: both parts (a device-encrypted key carries no seed)
        return wire.encode_public_key(self.c.to_bytes()[0])

    @staticmethod
    def from_bytes(par: BfvParameters, data: bytes, seeded_c1: Optional[np.ndarray] = None) -> "PublicKey":
        """PublicKey::from_bytes (public_key.rs:109-149).  The reference writes a compact message (c0 and the seed
        of c1); decoding one needs `seeded_c1`, the [limbs][N] NTT words of c1 expanded by the Rust host, as
        Ciphertext.from_bytes does.  A key at a level other than 0 is InvalidPublicKeyLevel."""
        msg = wire.decode_public_key(data)
        _, seed, level = wire.decode_ciphertext(msg)
        if level != 0:
            raise WireError("InvalidPublicKeyLevel", _capi.INVALID_LEVEL, "level %d, expected 0" % level)
        if seed and seeded_c1 is None:
            raise WireError("SeedExpansion", _capi.UNSUPPORTED, "the message carries a seed: pass the host-expanded c1")
        halves = None if seeded_c1 is None else np.asarray(seeded_c1, dtype=np.uint64)[None]
        return PublicKey(par, Ciphertext.from_bytes(par, [msg], halves))


class Plaintext(PlaintextVec):
    """fhe::bfv::Plaintext (bfv/plaintext.rs:20-27): one plaintext, at most N values (TooManyValues otherwise,
    plaintext.rs:311-345)."""

    @staticmethod
    def _check_count(n: int, par: BfvParameters):
        if n > par.degree():
            raise FheError(_capi.INVALID_ARGUMENT, "TooManyValues: %d, maximum %d" % (n, par.degree()))


def _unpack_rq(batch: "Ciphertext", rq_messages, want_rep: int) -> None:
    """`Poly::<R>::from_bytes(bytes, ctx)` (rq/serialize.rs:23-31 -> rq/convert.rs:46-161) for every polynomial of
    `batch`: rq_messages[i][j] is the encoded Rq of part j of ciphertext i.  Framing and checks here, unpacking (and
    the forward NTT of an NTT batch) on the device."""
    par, nbytes = batch.par, batch.packed_bytes_per_poly()
    count, parts = batch.count, len(batch)
    limbs, deg = batch.limbs, par.degree()
    blobs = np.zeros((count, parts, nbytes), np.uint8)
    for i, polys in enumerate(rq_messages):
        for j, msg in enumerate(polys):
            rep, degree, coeffs = wire.decode_rq(msg)
            if degree * nbytes != len(coeffs) * deg:          # sum_i serialization_length(degree) (convert.rs:76-88)
                raise WireError("InvalidCoefficientCount", detail="%d bytes for degree %d" % (len(coeffs), degree))
            if rep != want_rep:
                raise WireError("RepresentationMismatch", _capi.INVALID_REPRESENTATION,
                                "found %d, expected %d" % (rep, want_rep))
            if degree != deg and (limbs != 1 or degree > deg):
                # TryConvertFrom<Vec<u64>> for Poly<PowerBasis> (convert.rs:148-192): q.len() * degree words, or -- one
                # modulus only -- a shorter low-order polynomial, zero-extended (the zero bytes already in `blobs`)
                raise WireError("InvalidCoefficientCount", detail="degree %d in a context of degree %d" % (degree, deg))
            blobs[i, j, :len(coeffs)] = np.frombuffer(coeffs, np.uint8)
    check(_capi.lib().fhe_b200_batch_unpack(batch._h, 0, count, _ptr(blobs), batch.stream))
    check(_capi.lib().fhe_b200_sync(batch.stream))


class KeySwitchingKey:
    """fhe::bfv::KeySwitchingKey (keys/key_switching_key.rs:22-45) from its NTT-domain words:
    c0, c1 = [n_digits][ksk_limbs][N] (the `coefficients` of the Poly<NttShoup> elements)."""

    def __init__(self, par: BfvParameters, c0: np.ndarray, c1: np.ndarray, ciphertext_level: int = 0,
                 ksk_level: int = 0):
        c0 = np.ascontiguousarray(c0, dtype=np.uint64)
        c1 = np.ascontiguousarray(c1, dtype=np.uint64)
        if c0.shape != c1.shape or c0.ndim != 3 or c0.shape[2] != par.degree():
            raise FheError(_capi.INVALID_ARGUMENT, "expected c0, c1 as [digits][limbs][N]")
        if c0.shape[1] != len(par.moduli()) - ksk_level:
            raise FheError(_capi.CONTEXT_MISMATCH, "key limb count does not match ksk_level")
        h = C.c_void_p()
        check(_capi.lib().fhe_b200_ksk_upload(par._h, ciphertext_level, ksk_level, _ptr(c0), _ptr(c1),
                                              c0.shape[0], C.byref(h)))
        self._set(par, h, ciphertext_level, ksk_level, 0)

    def _set(self, par: BfvParameters, h, ciphertext_level: int, ksk_level: int, stream: int):
        self._h, self.par, self._stream = h, par, stream
        self.ciphertext_level, self.ksk_level = ciphertext_level, ksk_level
        # key_switching_key.rs:92-126: a key level with one modulus decomposes in base 2^(log_modulus / 2), otherwise
        # there is one digit per ciphertext limb
        log_modulus = (int(par.moduli()[0]) - 1).bit_length()
        single = len(par.moduli()) - ksk_level == 1
        self.log_base = log_modulus // 2 if single else 0
        self.n_digits = -(-log_modulus // self.log_base) if single else len(par.moduli()) - ciphertext_level

    @staticmethod
    def _adopt(par: BfvParameters, h, ciphertext_level: int, ksk_level: int, stream: int = 0) -> "KeySwitchingKey":
        """a key handle the library generated on `stream`"""
        k = KeySwitchingKey.__new__(KeySwitchingKey)
        k._set(par, C.c_void_p(h), ciphertext_level, ksk_level, stream)
        return k

    def arrays(self):
        """the key's NTT-domain words read back from the device: (c0, c1), each [n_digits][ksk_limbs][N]"""
        shape = (self.n_digits, len(self.par.moduli()) - self.ksk_level, self.par.degree())
        c0, c1 = np.empty(shape, np.uint64), np.empty(shape, np.uint64)
        check(_capi.lib().fhe_b200_ksk_download(self._h, _ptr(c0), _ptr(c1), self._stream))
        return c0, c1

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            _release("fhe_b200_ksk_free", h)

    # -- protobuf message (keys/key_switching_key.rs:365-482)
    def to_bytes(self) -> bytes:
        """KeySwitchingKeyProto::from(&ksk).encode_to_vec(), unseeded branch: every c0_i and c1_i as an Rq with
        representation NTTSHOUP (its coefficients are the power-basis words, packed on the device)."""
        c0, c1 = self.arrays()
        par, nd = self.par, c0.shape[0]
        tmp = Ciphertext.from_host(par, np.ascontiguousarray(np.stack([c0, c1], axis=1)), self.ksk_level, NTT)
        blobs = tmp.to_packed()
        tmp.sync()
        deg = par.degree()
        enc = [[wire.encode_rq(wire.REP_NTTSHOUP, deg, memoryview(blobs[i, j])) for i in range(nd)] for j in range(2)]
        return wire.encode_ksk(enc[0], enc[1], b"", self.ciphertext_level, self.ksk_level, self.log_base)

    @staticmethod
    def from_bytes(par: "BfvParameters", data: bytes, seeded_c1: Optional[np.ndarray] = None) -> "KeySwitchingKey":
        """KeySwitchingKey::try_convert_from(&KeySwitchingKeyProto, par) (key_switching_key.rs:388-482).  A key whose
        c1 row travels as a seed needs `seeded_c1`: [digits][limbs][N] NTT words of generate_c1 (:130-146), expanded by
        the Rust host."""
        k = wire.decode_ksk(data)
        ct_level, ksk_level, log_base = k["ciphertext_level"], k["ksk_level"], k["log_base"]
        for lv in (ksk_level, ct_level):
            if lv > par.max_level():
                raise WireError("InvalidLevel", _capi.INVALID_LEVEL, "level %d, max %d" % (lv, par.max_level()))
        if log_base != 0:
            if ksk_level != par.max_level() or ct_level != par.max_level():
                raise WireError("InvalidKeySwitchingDecompositionLevels", _capi.INVALID_LEVEL)
            # as coded (:406-408): the first modulus of the parameter set sizes the decomposition
            log_modulus = (int(par.moduli()[0]) - 1).bit_length()
            c0_size = -(-log_modulus // log_base)
        else:
            c0_size = len(par.moduli()) - ct_level
        if len(k["c0"]) != c0_size:
            raise WireError("WrongPolynomialCount", _capi.BAD_POLY_COUNT,
                            "KeySwitchingKeyC0: expected %d, found %d" % (c0_size, len(k["c0"])))
        seed = k["seed"]
        if not seed:
            if len(k["c1"]) != c0_size:
                raise WireError("WrongPolynomialCount", _capi.BAD_POLY_COUNT,
                                "KeySwitchingKeyC1: expected %d, found %d" % (c0_size, len(k["c1"])))
            tmp = Ciphertext(par, c0_size, 2, ksk_level, NTT)
            _unpack_rq(tmp, list(zip(k["c0"], k["c1"])), wire.REP_NTTSHOUP)
            words = tmp.to_host()
            tmp.sync()
            c0, c1 = np.ascontiguousarray(words[:, 0]), np.ascontiguousarray(words[:, 1])
        else:
            if len(seed) != 32:
                raise WireError("InvalidKeySwitchingSeedLength", detail="%d bytes, expected 32" % len(seed))
            if seeded_c1 is None:
                raise WireError("SeedExpansion", _capi.UNSUPPORTED,
                                "the key carries a seed: pass the host-expanded c1 row (key_switching_key.rs:130-146)")
            tmp = Ciphertext(par, c0_size, 1, ksk_level, NTT)
            _unpack_rq(tmp, [(m,) for m in k["c0"]], wire.REP_NTTSHOUP)
            c0 = np.ascontiguousarray(tmp.to_host()[:, 0])
            tmp.sync()
            c1 = np.ascontiguousarray(seeded_c1, dtype=np.uint64)
            if c1.shape != c0.shape:
                raise FheError(_capi.INVALID_ARGUMENT, "expected seeded_c1 as [digits][limbs][N]")
        key = KeySwitchingKey(par, c0, c1, ct_level, ksk_level)
        if key.log_base != log_base:
            # the reference would compute with whatever base the message names; the device derives the base from the
            # key level (fhe_b200_ksk_upload), so a message that disagrees is refused rather than reinterpreted
            raise WireError("InvalidKeySwitchingDecompositionLevels", _capi.UNSUPPORTED,
                            "log_base %d does not match the key level (expected %d)" % (log_base, key.log_base))
        return key

    @staticmethod
    def from_arrays(par: BfvParameters, c0, c1, ciphertext_level: int = 0, key_level: int = 0) -> "KeySwitchingKey":
        return KeySwitchingKey(par, c0, c1, ciphertext_level, key_level)

    def key_switch(self, p: Ciphertext, part: int = 0) -> Ciphertext:
        """KeySwitchingKey::key_switch (key_switching_key.rs:241-270, :323-362) on polynomial `part` of a
        POWER_BASIS batch; returns the (c0, c1) pair as a 2-part NTT batch at the key level."""
        out = Ciphertext(self.par, p.count, 2, self.ksk_level, NTT, p.stream)
        check(_capi.lib().fhe_b200_key_switch(p._h, part, self._h, out._h, p.stream))
        return out


class RGSWCiphertext:
    """fhe::bfv::RGSWCiphertext (bfv/rgsw_ciphertext.rs:20-24): two key-switching keys (for m and m*s)."""

    def __init__(self, ksk0: KeySwitchingKey, ksk1: KeySwitchingKey):
        if ksk0.ksk_level != ksk0.ciphertext_level or ksk1.ksk_level != ksk1.ciphertext_level \
                or ksk0.ciphertext_level != ksk1.ciphertext_level:
            raise FheError(_capi.INVALID_LEVEL, "RGSW key-switching keys must share one level")  # rgsw_ciphertext.rs:58-70
        self.ksk0, self.ksk1 = ksk0, ksk1

    @staticmethod
    def from_arrays(par: BfvParameters, k0c0, k0c1, k1c0, k1c1, level: int = 0) -> "RGSWCiphertext":
        return RGSWCiphertext(KeySwitchingKey(par, k0c0, k0c1, level, level), KeySwitchingKey(par, k1c0, k1c1, level, level))

    def to_bytes(self) -> bytes:  # rgsw_ciphertext.rs:30-37
        return wire.encode_rgsw(self.ksk0.to_bytes(), self.ksk1.to_bytes())

    @staticmethod
    def from_bytes(par: BfvParameters, data: bytes) -> "RGSWCiphertext":  # rgsw_ciphertext.rs:39-71
        m0, m1 = wire.decode_rgsw(data)
        k0, k1 = KeySwitchingKey.from_bytes(par, m0), KeySwitchingKey.from_bytes(par, m1)
        if k0.ksk_level != k0.ciphertext_level or k0.ciphertext_level != k1.ciphertext_level \
                or k1.ciphertext_level != k1.ksk_level:
            raise WireError("InconsistentKeySwitchingLevels", _capi.INVALID_LEVEL)
        return RGSWCiphertext(k0, k1)

    def external_product(self, ct: Ciphertext) -> Ciphertext:
        """&Ciphertext * &RGSWCiphertext (rgsw_ciphertext.rs:122-155): key-switch both parts, add."""
        if ct.level != self.ksk0.ciphertext_level:
            raise FheError(_capi.INVALID_LEVEL, "Ciphertext and RGSWCiphertext must have the same level")
        if len(ct) != 2:
            raise FheError(_capi.BAD_POLY_COUNT, "Ciphertext must have two parts")
        pb = ct.clone().into_power_basis()
        out = self.ksk0.key_switch(pb, part=0)
        out += self.ksk1.key_switch(pb, part=1)
        return out


class RelinearizationKey:
    """fhe::bfv::RelinearizationKey (keys/relinearization_key.rs:23-26)."""

    def __init__(self, ksk: KeySwitchingKey):
        self.ksk = ksk

    @staticmethod
    def new(sk: SecretKey, seed: Optional[bytes] = None) -> "RelinearizationKey":
        """RelinearizationKey::new (relinearization_key.rs:28-31), generated on the device"""
        return RelinearizationKey.new_leveled(sk, 0, 0, seed)

    @staticmethod
    def new_leveled(sk: SecretKey, ciphertext_level: int, key_level: int,
                    seed: Optional[bytes] = None) -> "RelinearizationKey":
        """RelinearizationKey::new_leveled (relinearization_key.rs:33-65), generated on the device from the seeded
        stream (seed as for SecretKey.try_encrypt)"""
        h = C.c_void_p()
        check(_capi.lib().fhe_b200_relin_key_generate(sk._h, ciphertext_level, key_level, sk.par.variance, _seed(seed),
                                                      C.byref(h), 0))
        return RelinearizationKey(KeySwitchingKey._adopt(sk.par, h.value, ciphertext_level, key_level))

    @staticmethod
    def from_arrays(par: BfvParameters, c0, c1, ciphertext_level: int = 0, key_level: int = 0):
        return RelinearizationKey(KeySwitchingKey(par, c0, c1, ciphertext_level, key_level))

    def to_bytes(self) -> bytes:  # relinearization_key.rs:113-119, :137-141
        return wire.encode_relinearization_key(self.ksk.to_bytes())

    @staticmethod
    def from_bytes(par: BfvParameters, data: bytes) -> "RelinearizationKey":  # relinearization_key.rs:121-135
        return RelinearizationKey(KeySwitchingKey.from_bytes(par, wire.decode_relinearization_key(data)))

    def relinearizes(self, ct: Ciphertext) -> Ciphertext:
        """RelinearizationKey::relinearizes (relinearization_key.rs:70-103): (c0,c1,c2) -> (c0,c1).
        (The reference mutates `ct`; a device batch changes shape, so the result is returned.)"""
        out = ct._like(parts=2)
        check(_capi.lib().fhe_b200_relinearize(ct._h, self.ksk._h, out._h, ct.stream))
        return out


class GaloisKey:
    """fhe::bfv::GaloisKey (keys/galois_key.rs:18-22)."""

    def __init__(self, exponent: int, ksk: KeySwitchingKey):
        self.exponent, self.ksk = exponent, ksk

    @staticmethod
    def new(sk: SecretKey, exponent: int, ciphertext_level: int = 0, key_level: int = 0,
            seed: Optional[bytes] = None) -> "GaloisKey":
        """GaloisKey::new (galois_key.rs:26-60), generated on the device (seed as for SecretKey.try_encrypt)"""
        return _galois_keys(sk, [exponent], ciphertext_level, key_level, seed)[0]

    @staticmethod
    def from_arrays(par: BfvParameters, exponent: int, c0, c1, ciphertext_level: int = 0, key_level: int = 0):
        return GaloisKey(exponent, KeySwitchingKey(par, c0, c1, ciphertext_level, key_level))

    def to_bytes(self) -> bytes:  # galois_key.rs:146-153
        return wire.encode_galois_key(self.ksk.to_bytes(), self.exponent)

    @staticmethod
    def from_bytes(par: BfvParameters, data: bytes, seeded_c1: Optional[np.ndarray] = None) -> "GaloisKey":
        """galois_key.rs:155-173; `seeded_c1` as for KeySwitchingKey.from_bytes"""
        msg, exponent = wire.decode_galois_key(data)
        ksk = KeySwitchingKey.from_bytes(par, msg, seeded_c1)
        exponent %= 2 * par.degree()            # SubstitutionExponent::new (rq/mod.rs:99-106)
        if exponent & 1 == 0:
            raise WireError("InvalidSubstitutionExponent", _capi.INVALID_EXPONENT, str(exponent))
        return GaloisKey(exponent, ksk)

    def relinearize(self, ct: Ciphertext) -> Ciphertext:
        """GaloisKey::relinearize (galois_key.rs:63-86)."""
        out = ct._like()
        check(_capi.lib().fhe_b200_galois(ct._h, self.exponent, self.ksk._h, out._h, ct.stream))
        return out


def _galois_keys(sk: SecretKey, exponents: Sequence[int], ciphertext_level: int, key_level: int,
                 seed: Optional[bytes]) -> "List[GaloisKey]":
    """one device call for every exponent: key k of the call (stream word 13) is exponents[k]"""
    two_n = 2 * sk.par.degree()
    exps = [int(e) % two_n for e in exponents]      # SubstitutionExponent::new (rq/mod.rs:99-106)
    arr = (C.c_uint32 * max(1, len(exps)))(*exps)
    hs = (C.c_void_p * max(1, len(exps)))()
    check(_capi.lib().fhe_b200_galois_keys_generate(sk._h, arr, len(exps), ciphertext_level, key_level,
                                                    sk.par.variance, _seed(seed), C.cast(hs, C.POINTER(C.c_void_p)),
                                                    0))
    return [GaloisKey(e, KeySwitchingKey._adopt(sk.par, hs[k], ciphertext_level, key_level))
            for k, e in enumerate(exps)]


class EvaluationKey:
    """fhe::bfv::EvaluationKey (keys/evaluation_key.rs:21-310): a map Galois exponent -> GaloisKey, and the levels
    of the ciphertexts it takes and of its keys (both 0 unless an EvaluationKeyBuilder or a message sets them)."""

    def __init__(self, par: BfvParameters, ciphertext_level: int = 0, evaluation_key_level: int = 0):
        self.par = par
        self.gk: Dict[int, GaloisKey] = {}
        self.ciphertext_level, self.evaluation_key_level = ciphertext_level, evaluation_key_level

    def to_bytes(self) -> bytes:
        """EvaluationKey::to_bytes (evaluation_key.rs:293-297, :494-505), the Galois keys in ascending exponent order"""
        return wire.encode_evaluation_key([self.gk[e].to_bytes() for e in sorted(self.gk)], self.ciphertext_level,
                                          self.evaluation_key_level)

    @staticmethod
    def from_bytes(par: BfvParameters, data: bytes,
                   seeded_c1: Optional[Dict[int, np.ndarray]] = None) -> "EvaluationKey":
        """EvaluationKey::from_bytes (evaluation_key.rs:299-310, :507-550): every key through GaloisKey.from_bytes, a
        key at other levels than the message's or a ciphertext level beyond the parameters' -> InvalidLevel, and a
        repeated exponent keeps the later key.  `seeded_c1`: exponent -> the host-expanded c1 of a compact key."""
        msgs, ct_level, ek_level = wire.decode_evaluation_key(data)
        ek = EvaluationKey(par, ct_level, ek_level)
        for m in msgs:
            exponent = wire.decode_galois_key(m)[1] % (2 * par.degree())
            gk = GaloisKey.from_bytes(par, m, (seeded_c1 or {}).get(exponent))
            for got, want in ((gk.ksk.ciphertext_level, ct_level), (gk.ksk.ksk_level, ek_level)):
                if got != want:
                    raise WireError("InvalidLevel", _capi.INVALID_LEVEL, "level %d, expected %d" % (got, want))
            ek.add_galois_key(gk)
        if ct_level > par.max_level():
            raise WireError("InvalidLevel", _capi.INVALID_LEVEL, "level %d, max %d" % (ct_level, par.max_level()))
        return ek

    def add_galois_key(self, gk: GaloisKey):
        self.gk[gk.exponent % (2 * self.par.degree())] = gk

    def supports_row_rotation(self) -> bool:
        return (2 * self.par.degree() - 1) in self.gk

    def supports_column_rotation_by(self, i: int) -> bool:
        return pow(3, i, 2 * self.par.degree()) in self.gk

    def supports_inner_sum(self) -> bool:  # evaluation_key.rs:40-53
        n = self.par.degree()
        i, ok = 1, self.supports_row_rotation()
        while i < n // 2:
            ok = ok and self.supports_column_rotation_by(i)
            i *= 2
        return ok

    def computes_inner_sum(self, ct: Ciphertext) -> Ciphertext:
        """EvaluationKey::computes_inner_sum (evaluation_key.rs:56-100)."""
        return computes_inner_sum_keyed(ct, [self], [0] * ct.count)

    def inner_sum_keys(self) -> "List[GaloisKey]":
        """the keys of the inner sum's steps: column rotations by 1, 2, 4, ..., N/4, then the row rotation"""
        if not self.supports_inner_sum():
            raise FheError(_capi.INVALID_ARGUMENT, "EvaluationKeyError: inner sum not supported by this key")
        n = self.par.degree()
        return [self.gk[pow(3, 1 << l, 2 * n)] for l in range(n.bit_length() - 2)] + [self.gk[2 * n - 1]]

    def supports_expansion(self, level: int) -> bool:  # evaluation_key.rs:175-189
        n = self.par.degree()
        return level == 0 or (level <= n.bit_length() - 1 and all(((n >> l) + 1) in self.gk for l in range(level)))

    def expands_batch(self, ct: Ciphertext, size: int) -> Ciphertext:
        """EvaluationKey::expands (evaluation_key.rs:192-256) of every ciphertext of `ct` (Q queries) as one batch of
        size * Q: entry i*Q + q is output i of query q (fhe_b200_expand)."""
        n = self.par.degree()
        level = max(0, (size - 1).bit_length())
        keys = (C.c_void_p * max(1, level))()
        for l in range(level):
            gk = self.gk.get((n >> l) + 1) if l < n.bit_length() - 1 else None
            keys[l] = gk.ksk._h.value if gk is not None else None
        # (an out-of-range size allocates a placeholder: fhe_b200_expand rejects the size before it looks at `out`)
        out = Ciphertext(self.par, size * ct.count if 0 < size <= n else 1, 2, ct.level, NTT, ct.stream)
        check(_capi.lib().fhe_b200_expand(ct._h, size, C.cast(keys, C.POINTER(C.c_void_p)), level, out._h, ct.stream))
        return out

    def expands(self, ct: Ciphertext, size: int, monomials: Optional[Sequence[np.ndarray]] = None):
        """EvaluationKey::expands (evaluation_key.rs:192-256), oblivious expansion of eprint 2019/1483: a list of `size`
        batches of ct.count ciphertexts, output i of every query.  `monomials` is accepted for older callers and
        ignored: the monomials -x^(N - 2^l) (:465-474) are fixed by the parameters and built by the library."""
        if size == 0 or size > self.par.degree():
            raise FheError(_capi.INVALID_ARGUMENT, "EvaluationKeyError: invalid expansion size")
        whole = self.expands_batch(ct, size)
        q = ct.count
        return [whole.take(i * q, q) for i in range(size)]

    def rotates_rows(self, ct: Ciphertext) -> Ciphertext:  # evaluation_key.rs:110-126
        e = 2 * self.par.degree() - 1
        if e not in self.gk:
            raise FheError(_capi.INVALID_ARGUMENT, "EvaluationKeyError: row rotation not supported by this key")
        return self.gk[e].relinearize(ct)

    def rotates_columns_by(self, ct: Ciphertext, i: int) -> Ciphertext:  # evaluation_key.rs:145-170
        e = pow(3, i, 2 * self.par.degree())  # :278-286
        if e not in self.gk:
            raise FheError(_capi.INVALID_ARGUMENT, "EvaluationKeyError: column rotation not supported by this key")
        return self.gk[e].relinearize(ct)

    def rotates_columns_by_many(self, ct: Ciphertext, steps: Sequence[int]) -> Ciphertext:
        """rotates_columns_by(ct_q, steps[i]) for every step and every ciphertext of ct (Q = ct.count) in one device call
        (fhe_b200_galois_many): entry i*Q + q of the result is ciphertext q rotated by steps[i]"""
        return galois_many(ct, *self._many_args(ct, steps))

    def rotates_columns_by_many_hoisted(self, ct: Ciphertext, steps: Sequence[int]) -> Ciphertext:
        """rotates_columns_by_many, word for word, with each ciphertext's rotations computed from one digit
        decomposition of it when it has two or more (fhe_b200_galois_many_hoisted)"""
        return galois_many_hoisted(ct, *self._many_args(ct, steps))[0]

    def linear_transform(self, ct: Ciphertext, diags: "PlaintextVec", baby: int,
                         n_diags: Optional[int] = None) -> Ciphertext:
        """sum_k diag_k (.) rotates_columns_by(ct, k) of every ciphertext by baby-step/giant-step diagonals in one
        device call (fhe_b200_linear_transform); `diags` from encode_diagonals"""
        n = _n_diags(ct, diags, n_diags)
        two_n = 2 * self.par.degree()
        gks = []
        for i in linear_transform_steps(n, baby):
            e = pow(3, i, two_n)
            if e not in self.gk:
                raise FheError(_capi.INVALID_ARGUMENT,
                               "EvaluationKeyError: column rotation by %d not supported by this key" % i)
            gks.append(self.gk[e])
        return linear_transform(ct, diags, baby, gks, n)[0]

    def _many_args(self, ct: Ciphertext, steps: Sequence[int]):
        two_n = 2 * self.par.degree()
        exps = [pow(3, int(i), two_n) for i in steps]
        for i, e in zip(steps, exps):
            if e not in self.gk:
                raise FheError(_capi.INVALID_ARGUMENT,
                               "EvaluationKeyError: column rotation by %d not supported by this key" % i)
        keys = sorted(set(exps))
        gks = [self.gk[e] for e in keys]
        q = ct.count
        index = [keys.index(e) for e in exps for _ in range(q)]
        return gks, index, [j for _ in exps for j in range(q)]


class EvaluationKeyBuilder:
    """fhe::bfv::EvaluationKeyBuilder (keys/evaluation_key.rs:318-491): the Galois keys of an EvaluationKey, generated
    on the device in one call."""

    def __init__(self, sk: SecretKey, ciphertext_level: int = 0, evaluation_key_level: int = 0):
        self.sk = sk
        self.ciphertext_level, self.evaluation_key_level = ciphertext_level, evaluation_key_level
        self.inner_sum = self.row_rotation = False
        self.expansion_level = 0
        self.column_rotation = set()

    @staticmethod
    def new(sk: SecretKey) -> "EvaluationKeyBuilder":
        return EvaluationKeyBuilder(sk)

    @staticmethod
    def new_leveled(sk: SecretKey, ciphertext_level: int, evaluation_key_level: int) -> "EvaluationKeyBuilder":
        """evaluation_key.rs:353-383"""
        if ciphertext_level > sk.par.max_level():
            raise FheError(_capi.INVALID_LEVEL, "InvalidLevel: %d, max %d" % (ciphertext_level, sk.par.max_level()))
        if evaluation_key_level > ciphertext_level:
            raise FheError(_capi.INVALID_LEVEL, "InvalidLevel: %d, max %d" % (evaluation_key_level, ciphertext_level))
        return EvaluationKeyBuilder(sk, ciphertext_level, evaluation_key_level)

    def enable_expansion(self, level: int) -> "EvaluationKeyBuilder":
        """evaluation_key.rs:386-398"""
        max_level = self.sk.par.degree().bit_length() - 1
        if level > max_level:
            raise FheError(_capi.INVALID_LEVEL, "InvalidLevel: %d, max %d" % (level, max_level))
        self.expansion_level = level
        return self

    def enable_inner_sum(self) -> "EvaluationKeyBuilder":
        self.inner_sum = True
        return self

    def enable_row_rotation(self) -> "EvaluationKeyBuilder":
        self.row_rotation = True
        return self

    def enable_column_rotation(self, i: int) -> "EvaluationKeyBuilder":
        """evaluation_key.rs:414-426: steps 1 .. N/2 - 1"""
        n = self.sk.par.degree()
        if not 1 <= i < n // 2:
            raise FheError(_capi.INVALID_ARGUMENT,
                           "EvaluationKeyError::InvalidRotationStep: %d, expected 1..%d" % (i, n // 2 - 1))
        self.column_rotation.add(pow(3, i, 2 * n))
        return self

    def exponents(self) -> List[int]:
        """the Galois exponents build() generates keys for (evaluation_key.rs:439-463), ascending"""
        n = self.sk.par.degree()
        idx = set(self.column_rotation)
        if self.row_rotation or self.inner_sum:
            idx.add(2 * n - 1)
        if self.inner_sum:
            i = 1
            while i < n // 2:
                idx.add(pow(3, i, 2 * n))
                i *= 2
        for l in range(self.expansion_level):
            idx.add((n >> l) + 1)
        return sorted(idx)

    def build(self, seed: Optional[bytes] = None) -> EvaluationKey:
        """EvaluationKeyBuilder::build (evaluation_key.rs:429-491): every Galois key in one device call, the exponents
        ascending, so a seed fixes the key of each exponent"""
        ek = EvaluationKey(self.sk.par, self.ciphertext_level, self.evaluation_key_level)
        exps = self.exponents()
        if exps:
            for gk in _galois_keys(self.sk, exps, self.ciphertext_level, self.evaluation_key_level, seed):
                ek.add_galois_key(gk)
        return ek


def dot_product_scalar(cts: "Ciphertext", pts, n_terms: Optional[int] = None) -> "Ciphertext":
    """fhe::bfv::dot_product_scalar (bfv/ops/dot_product.rs:55-184): sum_i cts[i] * pts[i].

    `cts` is a batch of ciphertexts, `pts` a batch of NTT plaintext polynomials (a one-part `Ciphertext` batch, or
    u64 words [count][limbs][N] = Plaintext::poly_ntt).  With `n_terms` smaller than the batch, the call computes
    count / n_terms independent dot products at once; an operand holding exactly n_terms entries is shared by all of
    them (the expanded PIR query of examples/mulpir.rs:153-181).  A device `PlaintextVec` is used in place."""
    if isinstance(pts, PlaintextVec):
        pts = pts.batch
    if not isinstance(pts, Ciphertext):
        w = np.ascontiguousarray(pts, dtype=np.uint64)
        if w.ndim != 3:
            raise FheError(_capi.INVALID_ARGUMENT, "expected [count][limbs][N] plaintext words")
        if w.shape[0] == 0:
            raise FheError(_capi.INVALID_ARGUMENT, "DotProductError::EmptyInput")
        pts = Ciphertext.from_host(cts.par, w[:, None], cts.level, NTT, cts.stream)
    n = n_terms if n_terms is not None else max(cts.count, pts.count)
    if n <= 0:
        raise FheError(_capi.INVALID_ARGUMENT, "DotProductError::EmptyInput")
    groups = max(cts.count, pts.count) // n
    out = Ciphertext(cts.par, max(groups, 1), len(cts), cts.level, NTT, cts.stream)
    check(_capi.lib().fhe_b200_dot_product_scalar(cts._h, pts._h, n, out._h, cts.stream))
    return out


def _rows(a, elem: int, what: str, output: bool = False):
    """(pointer, rows, length, row stride in elements, keep-alive, is_2d) of a 1-D or 2-D array of `elem`-byte integers:
    a numpy array (or, as input, a sequence or bytes) in pageable memory, or a torch tensor (pinned host or CUDA).  The
    library reads and writes rows of contiguous elements at a row stride of at least the row length.  An input laid out
    otherwise (a strided view, broadcast or overlapping rows) is copied first; an output laid out otherwise is refused,
    because the values would land in a copy the caller never sees."""
    def bad(why):
        return FheError(_capi.INVALID_ARGUMENT, "%s: expected a 1-D or 2-D array of %d-byte integers%s" % (why, elem, what))

    def in_place(ndim, shape, strides):   # strides in elements
        if ndim == 1:
            return shape[0] <= 1 or strides[0] == 1
        return shape[0] * shape[1] == 0 or ((shape[1] <= 1 or strides[1] == 1) and (shape[0] <= 1 or strides[0] >= shape[1]))

    if hasattr(a, "data_ptr") and hasattr(a, "is_cuda"):   # torch.Tensor
        if a.element_size() != elem or a.is_floating_point() or a.is_complex() or a.dim() not in (1, 2):
            raise bad("wrong element type or rank")
        if not in_place(a.dim(), tuple(a.shape), tuple(a.stride())):
            if output:
                raise bad("the output's rows are not contiguous at a stride of at least their length")
            a = a.contiguous()
        rows, n = (1, a.shape[0]) if a.dim() == 1 else tuple(a.shape)
        stride = a.stride(0) if a.dim() == 2 and rows > 1 else n
        return a.data_ptr(), rows, n, stride, a, a.dim() == 2
    if output and not isinstance(a, np.ndarray):
        raise bad("the output must be a numpy array or a torch tensor")
    if isinstance(a, (bytes, bytearray, memoryview)):
        a = np.frombuffer(a, np.uint8)
    a = np.asarray(a)
    if a.size == 0 and a.dtype.kind not in "iu" and not output:
        a = a.astype(np.uint8 if elem == 1 else np.uint64)
    if a.dtype.kind not in "iu" or a.dtype.itemsize != elem or a.ndim not in (1, 2):
        raise bad("wrong element type or rank")
    strides = tuple(x // elem if x % elem == 0 else -1 for x in a.strides)
    if not in_place(a.ndim, a.shape, strides):
        if output:
            raise bad("the output's rows are not contiguous at a stride of at least their length")
        a = np.ascontiguousarray(a)
        strides = tuple(x // elem for x in a.strides)
    if output and not a.flags.writeable:
        raise bad("the output is read-only")
    rows, n = (1, a.shape[0]) if a.ndim == 1 else a.shape
    stride = strides[0] if a.ndim == 2 and rows > 1 else n
    return a.ctypes.data, rows, n, stride, a, a.ndim == 2


def _transcode(par: BfvParameters, a, in_elem: int, in_bits: int, out_elem: int, out_bits: int,
               out_len: Optional[int], out, stream: int):
    ptr, rows, n, stride, keep, two_d = _rows(a, in_elem, " (input)")
    if out_len is None:
        out_len = -(-n * in_bits // out_bits) if 1 <= in_bits <= 64 and 1 <= out_bits <= 64 else 0
    if out is None:
        out = np.empty((rows, out_len) if two_d else out_len, np.uint64 if out_elem == 8 else np.uint8)
    optr, orows, olen, ostride, okeep, _ = _rows(out, out_elem, " (output)", output=True)
    if orows != rows or olen != out_len:
        raise FheError(_capi.INVALID_ARGUMENT, "output must hold %d rows of %d values" % (rows, out_len))
    check(_capi.lib().fhe_b200_transcode(par._h, ptr if n else None, in_elem, n, stride, in_bits,
                                         optr if out_len else None, out_elem, out_len, ostride, out_bits, rows, stream))
    check(_capi.lib().fhe_b200_sync(stream))
    del keep, okeep
    return out


def transcode_bidirectional(par: BfvParameters, a, input_nbits: int, output_nbits: int, out_len: Optional[int] = None,
                            out=None, stream: int = 0):
    """fhe_util::transcode_bidirectional (fhe-util/src/lib.rs:148-187) of every row of `a` (u64 words, 1-D or 2-D
    with contiguous rows) on the device of `par` (fhe_b200_transcode).  Each row gives its first `out_len` values
    (default: all ceil(len * input_nbits / output_nbits) of them), zero-padded past the stream.  `out`: an array or
    tensor (host, pinned or CUDA) of that shape receiving them; otherwise a new uint64 numpy array is returned."""
    return _transcode(par, a, 8, input_nbits, 8, output_nbits, out_len, out, stream)


def transcode_to_bytes(par: BfvParameters, a, nbits: int, out_len: Optional[int] = None, out=None, stream: int = 0):
    """fhe_util::transcode_to_bytes (lib.rs:68-108) of every row of `a`: uint8 output, as transcode_bidirectional"""
    return _transcode(par, a, 8, nbits, 1, 8, out_len, out, stream)


def transcode_from_bytes(par: BfvParameters, b, nbits: int, out_len: Optional[int] = None, out=None, stream: int = 0):
    """fhe_util::transcode_from_bytes (lib.rs:110-146) of every row of `b` (bytes, uint8): uint64 output, as
    transcode_bidirectional"""
    return _transcode(par, b, 1, 8, 8, nbits, out_len, out, stream)


class ScalingFactor:
    """fhe_math::rns::ScalingFactor (rns/scaler.rs:20-58): numerator / denominator."""

    def __init__(self, numerator: int, denominator: int):
        if denominator == 0:
            raise FheError(_capi.INVALID_ARGUMENT, "The denominator of a scaling factor should be non-zero")
        self.numerator, self.denominator = int(numerator), int(denominator)

    @staticmethod
    def one() -> "ScalingFactor":
        return ScalingFactor(1, 1)

    @property
    def is_one(self) -> bool:
        return self.numerator == self.denominator


def _le(x: int):
    b = int(x).to_bytes(max(1, (int(x).bit_length() + 7) // 8), "little")
    return (C.c_uint8 * len(b)).from_buffer_copy(b), len(b)


class Multiplicator:
    """fhe::bfv::Multiplicator (bfv/ops/mul.rs:22-33).  `default(rk)` is the default strategy (mul.rs:101-138: extend
    by factor 1, scale by t/Q, relinearize) on the fused path; `new` / `new_leveled` (mul.rs:37-75) build a custom
    strategy from scaling factors and an extended basis."""

    def __init__(self, rk: Optional[RelinearizationKey] = None, par: Optional[BfvParameters] = None, level: int = 0):
        self.rk = rk
        self.par = rk.ksk.par if rk is not None else par
        self.level = rk.ksk.ciphertext_level if rk is not None else level
        self.mod_switch = False
        self._h = None   # custom-strategy handle

    @staticmethod
    def default(rk: RelinearizationKey) -> "Multiplicator":
        return Multiplicator(rk)

    @staticmethod
    def new(lhs: ScalingFactor, rhs: ScalingFactor, extended_basis, post: ScalingFactor,
            par: BfvParameters, psi=None) -> "Multiplicator":
        return Multiplicator.new_leveled(lhs, rhs, extended_basis, post, 0, par, psi)

    @staticmethod
    def new_leveled(lhs: ScalingFactor, rhs: ScalingFactor, extended_basis, post: ScalingFactor, level: int,
                    par: BfvParameters, psi=None) -> "Multiplicator":
        m = Multiplicator(None, par, level)
        basis = np.ascontiguousarray(np.array([int(q) for q in extended_basis], dtype=np.uint64))
        ps = None
        if psi is not None:
            ps = np.ascontiguousarray(np.array([int(psi[int(q)]) for q in basis], dtype=np.uint64))
        args = []
        for f in (lhs, rhs):
            for v in (f.numerator, f.denominator):
                args += list(_le(v))
        pn, pd = _le(post.numerator), _le(post.denominator)
        h = C.c_void_p()
        check(_capi.lib().fhe_b200_multiplicator_create(
            par._h, level, *args, basis.ctypes.data, len(basis), ps.ctypes.data if ps is not None else None,
            pn[0], pn[1], pd[0], pd[1], C.byref(h)))
        m._h = h
        m.extended_basis = [int(q) for q in basis]
        return m

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            _release("fhe_b200_multiplicator_free", h)

    def enable_relinearization(self, rk: RelinearizationKey):  # mul.rs:141-151
        if rk.ksk.par is not self.par or rk.ksk.ciphertext_level != self.level:
            raise FheError(_capi.CONTEXT_MISMATCH, "ParameterMismatch")
        self.rk = rk
        return self

    def enable_mod_switching(self):  # mul.rs:155-162
        if self.level >= self.par.max_level():
            raise FheError(_capi.NO_MORE_CONTEXT, "NoMoreContext")
        self.mod_switch = True
        return self

    def multiply(self, lhs: Ciphertext, rhs: Ciphertext) -> Ciphertext:
        """Multiplicator::multiply (mul.rs:165-243)."""
        if lhs.level != self.level or rhs.level != self.level:
            raise FheError(_capi.INVALID_LEVEL, "InvalidLevel")  # mul.rs:168-181
        ms = 1 if self.mod_switch else 0
        if self._h is None:
            out = lhs._like(parts=2, level=self.level + ms)
            check(_capi.lib().fhe_b200_mul_relin(lhs._h, rhs._h, self.rk.ksk._h, ms, out._h, lhs.stream))
            return out
        out = lhs._like(parts=2 if self.rk is not None else 3, level=self.level + ms)
        check(_capi.lib().fhe_b200_multiplicator_multiply(
            self._h, lhs._h, rhs._h, self.rk.ksk._h if self.rk is not None else None, ms, out._h, lhs.stream))
        return out


# ---- per-ciphertext keys: one batch, one key per ciphertext (a server answering many clients).  `index[j]` names the
# key of ciphertext j (for expands_keyed: of query j); output j is what the single-key method gives on ciphertext j
# with that key.  One device call each (the fhe_b200_*_keyed entry points of include/fhe_b200.h).

def _keyed_args(ksks: Sequence["KeySwitchingKey"], index, count: int):
    idx = np.ascontiguousarray(np.asarray(index, dtype=np.int64).reshape(-1))
    if idx.size != count:
        raise FheError(_capi.INVALID_ARGUMENT, "expected one key index per ciphertext (%d), got %d" % (count, idx.size))
    if idx.size and (idx.min() < 0 or idx.max() > 0xFFFFFFFF):
        raise FheError(_capi.INVALID_ARGUMENT, "key index out of range")
    hs = (C.c_void_p * max(1, len(ksks)))(*[k._h.value for k in ksks])
    ix = (C.c_uint32 * max(1, idx.size))(*[int(v) for v in idx])
    return C.cast(hs, C.POINTER(C.c_void_p)), len(ksks), ix


def key_switch_keyed(p: Ciphertext, part: int, ksks: Sequence["KeySwitchingKey"], index) -> Ciphertext:
    """KeySwitchingKey.key_switch of ciphertext j of `p` with ksks[index[j]]"""
    args = _keyed_args(ksks, index, p.count)
    out = Ciphertext(p.par, p.count, 2, ksks[0].ksk_level if ksks else p.level, NTT, p.stream)
    check(_capi.lib().fhe_b200_key_switch_keyed(p._h, part, *args, out._h, p.stream))
    return out


def relinearizes_keyed(ct: Ciphertext, rks: Sequence["RelinearizationKey"], index) -> Ciphertext:
    """RelinearizationKey.relinearizes of ciphertext j with rks[index[j]]"""
    args = _keyed_args([rk.ksk for rk in rks], index, ct.count)
    out = ct._like(parts=2)
    check(_capi.lib().fhe_b200_relinearize_keyed(ct._h, *args, out._h, ct.stream))
    return out


def multiply_keyed(lhs: Ciphertext, rhs: Ciphertext, rks: Sequence["RelinearizationKey"], index,
                   mod_switch: bool = False) -> Ciphertext:
    """Multiplicator.default(rks[index[j]]).multiply of the pair j (with enable_mod_switching when mod_switch)"""
    ms = 1 if mod_switch else 0
    args = _keyed_args([rk.ksk for rk in rks], index, lhs.count)
    out = lhs._like(parts=2, level=lhs.level + ms)
    check(_capi.lib().fhe_b200_mul_relin_keyed(lhs._h, rhs._h, *args, ms, out._h, lhs.stream))
    return out


def galois_keyed(ct: Ciphertext, gks: Sequence["GaloisKey"], index) -> Ciphertext:
    """GaloisKey.relinearize of ciphertext j with gks[index[j]]; every key must be for the same exponent"""
    if gks and any(g.exponent != gks[0].exponent for g in gks):
        raise FheError(_capi.INVALID_ARGUMENT, "the Galois keys of one call must share their exponent")
    args = _keyed_args([g.ksk for g in gks], index, ct.count)
    out = ct._like()
    check(_capi.lib().fhe_b200_galois_keyed(ct._h, gks[0].exponent if gks else 1, *args, out._h, ct.stream))
    return out


def galois_many(ct: Ciphertext, gks: Sequence["GaloisKey"], index, source=None) -> Ciphertext:
    """GaloisKey.relinearize of ciphertext source[j] (j when source is None) with gks[index[j]], each key with its own
    exponent: one device call for many rotations of one ciphertext or of many (fhe_b200_galois_many)"""
    return _galois_many(ct, gks, index, source, False)[0]


def galois_many_hoisted(ct: Ciphertext, gks: Sequence["GaloisKey"], index, source=None) -> Tuple[Ciphertext, int]:
    """galois_many, word for word, with the rotations of each source ciphertext that has two or more outputs computed
    from one digit decomposition of its c1 (fhe_b200_galois_many_hoisted).  Returns the result and how many outputs
    were hoisted.  Synchronises the stream once when any source has two or more outputs."""
    return _galois_many(ct, gks, index, source, True)


def _galois_many(ct, gks, index, source, hoisted):
    count = ct.count
    if source is not None:
        src = np.ascontiguousarray(np.asarray(source, dtype=np.int64).reshape(-1))
        if src.size and (src.min() < 0 or src.max() > 0xFFFFFFFF):
            raise FheError(_capi.INVALID_ARGUMENT, "source index out of range")
        count = src.size
        sp = (C.c_uint32 * max(1, src.size))(*[int(v) for v in src])
    else:
        sp = None
    keys, n, ix = _keyed_args([g.ksk for g in gks], index, count)
    exps = (C.c_uint32 * max(1, len(gks)))(*[int(g.exponent) & 0xFFFFFFFF for g in gks])
    out = Ciphertext(ct.par, max(count, 1), 2, ct.level, NTT, ct.stream)
    if not hoisted:
        check(_capi.lib().fhe_b200_galois_many(ct._h, sp, keys, exps, n, ix, out._h, ct.stream))
        return out, 0
    n_hoisted = C.c_uint32(0)
    check(_capi.lib().fhe_b200_galois_many_hoisted(ct._h, sp, keys, exps, n, ix, out._h, C.byref(n_hoisted),
                                                   ct.stream))
    return out, n_hoisted.value


def linear_transform_steps(n_diags: int, baby: int) -> List[int]:
    """the column rotation steps a linear transform of n_diags diagonals with baby step `baby` needs keys for (to
    enable in EvaluationKeyBuilder): the baby steps 1 .. baby - 1, then the giant steps baby, 2 baby, .."""
    if not 1 <= baby <= n_diags:
        raise FheError(_capi.INVALID_ARGUMENT, "the baby step must be 1 .. n_diags, got %d" % baby)
    return list(range(1, baby)) + list(range(baby, n_diags, baby))


def _n_diags(ct: Ciphertext, diags: "PlaintextVec", n_diags: Optional[int]) -> int:
    if n_diags is not None:
        return int(n_diags)
    if getattr(diags, "n_diags", None) is not None:
        return diags.n_diags
    return len(diags)


def linear_transform(ct: Ciphertext, diags: "PlaintextVec", baby: int, gks: Sequence["GaloisKey"],
                     n_diags: Optional[int] = None) -> Tuple[Ciphertext, int]:
    """out[c] = sum_g rot_{g baby}(sum_i diags[g baby + i] (.) rot_i(ct[c])) (rot_0 the identity) for every ciphertext
    of ct, word for word the composition of rotates_columns_by, mul_plain and + (fhe_b200_linear_transform).  `diags`:
    a PlaintextVec (or 1-part NTT batch) of n_diags diagonals shared by every ciphertext, or n_diags per ciphertext;
    n_diags defaults to the count encode_diagonals recorded, else len(diags).  gks: Galois keys holding at least the
    steps of linear_transform_steps.  Returns the result and how many (ciphertext, baby step) rotations were computed
    unhoisted.  Synchronises the stream once when it hoists."""
    batch = diags.batch if isinstance(diags, PlaintextVec) else diags
    n = _n_diags(ct, diags, n_diags)
    keys = (C.c_void_p * max(1, len(gks)))(*[g.ksk._h.value for g in gks])
    exps = (C.c_uint32 * max(1, len(gks)))(*[int(g.exponent) & 0xFFFFFFFF for g in gks])
    out = Ciphertext(ct.par, max(ct.count, 1), 2, ct.level, NTT, ct.stream)
    n_fallback = C.c_uint32(0)
    check(_capi.lib().fhe_b200_linear_transform(ct._h, batch._h, n, baby, C.cast(keys, C.POINTER(C.c_void_p)), exps,
                                                len(gks), out._h, C.byref(n_fallback), ct.stream))
    return out, n_fallback.value


def diagonals(matrices, half: int, n_diags: int, baby: int) -> np.ndarray:
    """the slot values encode_diagonals encodes, [count][n_diags][2 * half] uint64 (see there)"""
    m = np.asarray(matrices)
    if m.dtype.kind not in "iu":
        raise FheError(_capi.INVALID_ARGUMENT, "expected integer matrices")
    if m.ndim == 2:
        m = np.stack([m, m])
    if m.ndim == 3:
        m = m[None]
    if m.ndim != 4 or m.shape[1:] != (2, half, half):
        raise FheError(_capi.INVALID_ARGUMENT, "expected (N/2) x (N/2) matrices: one, a pair (one per slot row), or "
                       "a stack of pairs [count][2][N/2][N/2]")
    if not 1 <= n_diags <= half or not 1 <= baby <= n_diags:
        raise FheError(_capi.INVALID_ARGUMENT, "n_diags must be 1 .. N/2 and the baby step 1 .. n_diags")
    r = np.arange(half)
    k = np.arange(half)
    # d[c][q][k][r] = M_cq[r][(r + k) mod half]
    d = m[:, :, r[None, :], (r[None, :] + k[:, None]) % half]
    if np.any(d[:, :, n_diags:] != 0):
        raise FheError(_capi.INVALID_ARGUMENT, "a diagonal beyond the first n_diags = %d is not zero" % n_diags)
    d = d[:, :, :n_diags]
    for j in range(baby, n_diags):   # rotated right by the giant step g * baby of diagonal j
        d[:, :, j] = np.roll(d[:, :, j], (j // baby) * baby, axis=-1)
    return np.ascontiguousarray(d.transpose(0, 2, 1, 3).reshape(m.shape[0], n_diags, 2 * half))


def encode_diagonals(par: BfvParameters, matrices, baby: int, level: int = 0,
                     n_diags: Optional[int] = None) -> "PlaintextVec":
    """The diagonals of a slot-wise linear map for linear_transform, SIMD-encoded on the device.  `matrices`: one
    (N/2) x (N/2) integer matrix for both slot rows, a pair [2][N/2][N/2] (one per row), or a stack of pairs
    [count][2][N/2][N/2] (one map per ciphertext); entries are taken mod t.  Diagonal k is M[r][(r + k) mod N/2] in
    slot r of each row, rotated right by its giant step g * baby (k = g * baby + i) on the host; the result holds
    diagonals 0 .. n_diags - 1 (default N/2) of each map in that order.  A non-zero diagonal from n_diags on is
    refused."""
    half = par.degree() // 2
    n = half if n_diags is None else int(n_diags)
    t = par.plaintext()
    m = np.asarray(matrices)
    if m.dtype.kind in "iu":
        m = np.mod(m.astype(np.int64) if m.dtype.kind == "i" else m, t).astype(np.uint64)
    d = diagonals(m, half, n, baby)
    pv = PlaintextVec.try_encode(d.reshape(-1), Encoding.simd_at_level(level), par)
    pv.n_diags = n
    return pv


def computes_inner_sum_keyed(ct: Ciphertext, eks: Sequence["EvaluationKey"], index) -> Ciphertext:
    """EvaluationKey.computes_inner_sum of ciphertext j with eks[index[j]] (evaluation_key.rs:56-100), one device call
    (fhe_b200_inner_sum_keyed; fhe_b200_inner_sum for a single key)"""
    sets = [ek.inner_sum_keys() for ek in eks]
    _, _, ix = _keyed_args([], index, ct.count)
    n_gks = ct.par.degree().bit_length() - 1
    arr = (C.c_void_p * max(1, n_gks * len(sets)))(*[g.ksk._h.value for gs in sets for g in gs])
    keys = C.cast(arr, C.POINTER(C.c_void_p))
    out = ct._like()
    if len(sets) == 1:
        check(_capi.lib().fhe_b200_inner_sum(ct._h, keys, n_gks, out._h, ct.stream))
    else:
        check(_capi.lib().fhe_b200_inner_sum_keyed(ct._h, keys, n_gks, len(sets), ix, out._h, ct.stream))
    return out


def _galois_of(eks: Sequence["EvaluationKey"], exponent: int, what: str) -> "List[GaloisKey]":
    for ek in eks:
        if exponent % (2 * ek.par.degree()) not in ek.gk:
            raise FheError(_capi.INVALID_ARGUMENT, "EvaluationKeyError: %s not supported by this key" % what)
    return [ek.gk[exponent % (2 * ek.par.degree())] for ek in eks]


def rotates_columns_by_keyed(ct: Ciphertext, eks: Sequence["EvaluationKey"], index, i: int) -> Ciphertext:
    """EvaluationKey.rotates_columns_by(ct_j, i) with eks[index[j]] (evaluation_key.rs:145-170)"""
    return galois_keyed(ct, _galois_of(eks, pow(3, i, 2 * ct.par.degree()), "column rotation"), index)


def rotates_rows_keyed(ct: Ciphertext, eks: Sequence["EvaluationKey"], index) -> Ciphertext:
    """EvaluationKey.rotates_rows(ct_j) with eks[index[j]] (evaluation_key.rs:110-126)"""
    return galois_keyed(ct, _galois_of(eks, 2 * ct.par.degree() - 1, "row rotation"), index)


def expands_keyed(ct: Ciphertext, eks: Sequence["EvaluationKey"], index, size: int) -> "List[Ciphertext]":
    """EvaluationKey.expands of query q of `ct` with eks[index[q]]: a list of `size` batches, batch i holding output i
    of every query (as EvaluationKey.expands)"""
    whole = expands_batch_keyed(ct, eks, index, size)
    q = ct.count
    return [whole.take(i * q, q) for i in range(size)]


def expands_batch_keyed(ct: Ciphertext, eks: Sequence["EvaluationKey"], index, size: int) -> Ciphertext:
    """expands_keyed as one batch of size * Q: entry i*Q + q is output i of query q (as EvaluationKey.expands_batch)"""
    n = ct.par.degree()
    if size == 0 or size > n:
        raise FheError(_capi.INVALID_ARGUMENT, "EvaluationKeyError: invalid expansion size")
    level = max(0, (size - 1).bit_length())
    hs = []
    for ek in eks:
        for l in range(level):
            gk = ek.gk.get((n >> l) + 1)
            hs.append(gk.ksk._h.value if gk is not None else None)
    keys, _, ix = _keyed_args([], index, ct.count)
    arr = (C.c_void_p * max(1, len(hs)))(*hs)
    out = Ciphertext(ct.par, size * ct.count, 2, ct.level, NTT, ct.stream)
    check(_capi.lib().fhe_b200_expand_keyed(ct._h, size, C.cast(arr, C.POINTER(C.c_void_p)), level, len(eks), ix,
                                            out._h, ct.stream))
    return out


def external_products_keyed(cts: Ciphertext, rgsws: Sequence["RGSWCiphertext"], index) -> Ciphertext:
    """&cts[j] * &rgsws[index[j]] (rgsw_ciphertext.rs:122-155): two keyed key switches and an add, as
    RGSWCiphertext.external_product composes them"""
    if any(r.ksk0.ciphertext_level != cts.level for r in rgsws):
        raise FheError(_capi.INVALID_LEVEL, "Ciphertext and RGSWCiphertext must have the same level")
    if len(cts) != 2:
        raise FheError(_capi.BAD_POLY_COUNT, "Ciphertext must have two parts")
    pb = cts.clone().into_power_basis()
    out = key_switch_keyed(pb, 0, [r.ksk0 for r in rgsws], index)
    out += key_switch_keyed(pb, 1, [r.ksk1 for r in rgsws], index)
    return out


# ---- dot products of ciphertext vectors (examples/mulpir.rs:176-183): sum_i a[i] * b[i] with one relinearization
# and one switch_to_level per group, in one device call.

def _dot_groups(a: Ciphertext, b: Ciphertext, n_terms: int) -> int:
    n = int(n_terms)
    count = max(a.count, b.count)
    if n <= 0 or count % n:
        raise FheError(_capi.INVALID_ARGUMENT, "DotProductError::OperandCountMismatch: %d entries, n_terms %s"
                       % (count, n_terms))
    return count // n


def dot_product(a: Ciphertext, b: Ciphertext, n_terms: int, rk: Optional[RelinearizationKey] = None,
                level: Optional[int] = None) -> Ciphertext:
    """out[g] = sum_{i < n_terms} a[g*n_terms + i] * b[g*n_terms + i], relinearized with `rk` (3 parts without one)
    and switched to `level` (default: the operands' level).  Either operand may hold n_terms entries only, shared by
    every group.  Words equal the reference's loop of mul, +=, relinearizes and switch_to_level (fhe_b200_dot_product)."""
    groups = _dot_groups(a, b, n_terms)
    out = Ciphertext(a.par, groups, 2 if rk is not None else 3, a.level if level is None else level, NTT, a.stream)
    check(_capi.lib().fhe_b200_dot_product(a._h, b._h, int(n_terms), rk.ksk._h if rk is not None else None, out._h,
                                           a.stream))
    return out


def dot_product_keyed(a: Ciphertext, b: Ciphertext, n_terms: int, rks: Sequence[RelinearizationKey], index,
                      level: Optional[int] = None) -> Ciphertext:
    """dot_product with group g relinearized by rks[index[g]]: one key index per group, not per term
    (fhe_b200_dot_product_keyed)"""
    groups = _dot_groups(a, b, n_terms)
    args = _keyed_args([rk.ksk for rk in rks], index, groups)
    out = Ciphertext(a.par, groups, 2, a.level if level is None else level, NTT, a.stream)
    check(_capi.lib().fhe_b200_dot_product_keyed(a._h, b._h, int(n_terms), *args, out._h, a.stream))
    return out

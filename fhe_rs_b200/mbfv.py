"""Host-side mirror of the reference's `fhe::mbfv` (multiparty BFV, crates/fhe/src/mbfv, eprint 2020/304) on the C ABI
of include/fhe_b200.h.

WARNING: experimental, incomplete and not audited, as the reference's module.  The errors of every share are the
ordinary BfvParameters::variance errors, not smudging noise (the reference's own TODO), so a decryption share may leak
information about the secret key share.  No noise flooding is added.

Every share holds device batches and covers a whole batch: a SecretKeySwitchShare, DecryptionShare or
PublicKeySwitchShare of a `Ciphertext` batch is one share per ciphertext, made in one call.  The randomness comes from
the seeded ChaCha20 stream of include/fhe_b200.h (seed None draws os.urandom(32))."""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence

from . import _capi
from ._capi import NTT, FheError, check
from .bfv import (BfvParameters, Ciphertext, KeySwitchingKey, Plaintext, PlaintextVec, PublicKey, RelinearizationKey,
                  SecretKey, _release, _seed)

__all__ = ["CommonRandomPoly", "PublicKeyShare", "SecretKeySwitchShare", "DecryptionShare", "PublicKeySwitchShare",
           "RelinKeyGenerator", "RelinKeyShare", "Aggregate", "aggregate"]


class CommonRandomPoly:
    """mbfv::CommonRandomPoly (crp.rs:8-44): a uniform NTT polynomial every party shares.  `batch` is a 1-part batch
    with one CRP per entry (one entry for a single CRP)."""

    def __init__(self, batch: Ciphertext):
        self.batch, self.par = batch, batch.par

    @staticmethod
    def new(par: BfvParameters, seed: Optional[bytes] = None) -> "CommonRandomPoly":   # crp.rs:17-19
        return CommonRandomPoly.new_leveled(par, 0, seed)

    @staticmethod
    def new_vec(par: BfvParameters, seed: Optional[bytes] = None) -> "List[CommonRandomPoly]":   # crp.rs:25-32
        """one CRP per ciphertext modulus, drawn in one call (entry k of the call is CRP k)"""
        b = CommonRandomPoly._generate(par, len(par.moduli()), 0, seed)
        return [CommonRandomPoly(b.take(k, 1)) for k in range(b.count)]

    @staticmethod
    def new_leveled(par: BfvParameters, level: int, seed: Optional[bytes] = None) -> "CommonRandomPoly":   # :35-43
        return CommonRandomPoly(CommonRandomPoly._generate(par, 1, level, seed))

    @staticmethod
    def _generate(par: BfvParameters, count: int, level: int, seed: Optional[bytes]) -> Ciphertext:
        seed = _seed(seed)
        b = Ciphertext(par, count, 1, level, NTT)
        check(_capi.lib().fhe_b200_crp_generate(par._h, seed, b._h, b.stream))
        return b

    def level(self) -> int:
        return self.batch.level


def _handles(batches: Sequence[Ciphertext]):
    """the batch handles as a `const fhe_b200_batch* const*` table"""
    return (C.c_void_p * len(batches))(*[b._h for b in batches])


class PublicKeyShare:
    """mbfv::PublicKeyShare (public_key_gen.rs:11-58): p0 = -crp s + e at level 0, one per entry of the CRP batch."""

    def __init__(self, sk_share: SecretKey, crp: CommonRandomPoly, seed: Optional[bytes] = None):
        seed = _seed(seed)
        self.par, self.crp = sk_share.par, crp
        self.p0_share = Ciphertext(self.par, crp.batch.count, 1, 0, NTT)
        check(_capi.lib().fhe_b200_pk_share(sk_share._h, crp.batch._h, self.par.variance, seed, self.p0_share._h,
                                            self.p0_share.stream))


class SecretKeySwitchShare:
    """mbfv::SecretKeySwitchShare (secret_key_switch.rs:14-96): h = (s_in - s_out) c1 + e for every ciphertext of the
    2-part batch `ct`."""

    def __init__(self, sk_input_share: SecretKey, sk_output_share: Optional[SecretKey], ct: Ciphertext,
                 seed: Optional[bytes] = None):
        seed = _seed(seed)
        self.par, self.ct = sk_input_share.par, ct
        self.h_share = Ciphertext(self.par, ct.count, 1, ct.level, NTT, ct.stream)
        out_h = sk_output_share._h if sk_output_share is not None else None
        check(_capi.lib().fhe_b200_sks_share(sk_input_share._h, out_h, ct._h, self.par.variance, seed,
                                             self.h_share._h, ct.stream))


class DecryptionShare(SecretKeySwitchShare):
    """mbfv::DecryptionShare (secret_key_switch.rs:117-143): the secret key switch to the zero key."""

    def __init__(self, sk_input_share: SecretKey, ct: Ciphertext, seed: Optional[bytes] = None):
        super().__init__(sk_input_share, None, ct, seed)


class PublicKeySwitchShare:
    """mbfv::PublicKeySwitchShare (public_key_switch.rs:13-93): (h0, h1) = (u pk0 + s c1 + e0, u pk1 + e1) for every
    ciphertext of `ct`, with the public key switched down to ct's level.  `h_share` is a 2-part batch."""

    def __init__(self, sk_share: SecretKey, public_key: PublicKey, ct: Ciphertext, seed: Optional[bytes] = None):
        seed = _seed(seed)
        self.par, self.ct = sk_share.par, ct
        self.h_share = Ciphertext(self.par, ct.count, 2, ct.level, NTT, ct.stream)
        check(_capi.lib().fhe_b200_pks_share(sk_share._h, public_key.c._h, ct._h, self.par.variance, seed,
                                             self.h_share._h, ct.stream))


class RelinKeyShare:
    """mbfv::RelinKeyShare<R> (relin_key_gen.rs:14-34): h0, h1 as 1-part level-0 batches of one polynomial per
    level-0 modulus; `round` is "R1", "R1Aggregated" or "R2"; a round-2 share keeps the round-1 aggregate it was made
    from (`last_round`), which RelinearizationKey's aggregation needs."""

    def __init__(self, par: BfvParameters, h0: Ciphertext, h1: Ciphertext, round: str,
                 last_round: "Optional[RelinKeyShare]" = None):
        self.par, self.h0, self.h1, self.round, self.last_round = par, h0, h1, round, last_round


class RelinKeyGenerator:
    """mbfv::RelinKeyGenerator (relin_key_gen.rs:36-96): u lives on the device and is erased when the generator is
    released.  crp: the CRPs of CommonRandomPoly.new_vec, one per level-0 modulus."""

    def __init__(self, sk_share: SecretKey, crp: "Sequence[CommonRandomPoly]", seed: Optional[bytes] = None):
        seed = _seed(seed)
        self.par, self._sk = sk_share.par, sk_share
        L = len(self.par.moduli())
        if len(crp) != L:
            raise FheError(_capi.INVALID_ARGUMENT, "MultipartyError::InvalidCommonRandomPolynomialCount: %d, expected %d"
                           % (len(crp), L))
        self._crp = Ciphertext(self.par, L, 1, 0, NTT)   # the CRPs side by side, kept as long as the generator
        for i, c in enumerate(crp):
            check(_capi.lib().fhe_b200_batch_copy_range(self._crp._h, i, c.batch._h, 0, 1, 1, self._crp.stream))
        h = C.c_void_p()
        check(_capi.lib().fhe_b200_rkg_create(sk_share._h, self._crp._h, self.par.variance, seed, C.byref(h),
                                              self._crp.stream))
        self._h = h

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            _release("fhe_b200_rkg_free", h)

    def _pair(self):
        L = len(self.par.moduli())
        return Ciphertext(self.par, L, 1, 0, NTT), Ciphertext(self.par, L, 1, 0, NTT)

    def round_1(self, seed: Optional[bytes] = None) -> RelinKeyShare:   # relin_key_gen.rs:98-104
        h0, h1 = self._pair()
        check(_capi.lib().fhe_b200_rkg_round1(self._h, _seed(seed), h0._h, h1._h, h0.stream))
        return RelinKeyShare(self.par, h0, h1, "R1")

    def round_2(self, r1: RelinKeyShare, seed: Optional[bytes] = None) -> RelinKeyShare:   # relin_key_gen.rs:106-110
        if r1.round != "R1Aggregated":
            raise FheError(_capi.INVALID_ARGUMENT, "round 2 takes the aggregate of the round-1 shares")
        h0, h1 = self._pair()
        check(_capi.lib().fhe_b200_rkg_round2(self._h, r1.h0._h, r1.h1._h, _seed(seed), h0._h, h1._h, h0.stream))
        return RelinKeyShare(self.par, h0, h1, "R2", r1)


def _r1_aggregate(shares) -> RelinKeyShare:   # relin_key_gen.rs:200-222
    if any(not isinstance(s, RelinKeyShare) or s.round != "R1" for s in shares):
        raise FheError(_capi.INVALID_ARGUMENT, "RelinKeyShare<R1Aggregated> aggregates round-1 shares")
    first = shares[0]
    h0, h1 = first.h0._like(), first.h1._like()
    for out, part in ((h0, "h0"), (h1, "h1")):
        check(_capi.lib().fhe_b200_shares_sum(_handles([getattr(s, part) for s in shares]), len(shares), out._h,
                                              out.stream))
    return RelinKeyShare(first.par, h0, h1, "R1Aggregated")


def _relin_key(shares) -> RelinearizationKey:   # relin_key_gen.rs:299-350
    if any(not isinstance(s, RelinKeyShare) or s.round != "R2" for s in shares):
        raise FheError(_capi.INVALID_ARGUMENT, "RelinearizationKey aggregates round-2 shares")
    first = shares[0]
    h = C.c_void_p()
    check(_capi.lib().fhe_b200_rkg_aggregate(_handles([s.h0 for s in shares]), _handles([s.h1 for s in shares]),
                                             len(shares), first.last_round.h1._h, C.byref(h), first.h0.stream))
    return RelinearizationKey(KeySwitchingKey._adopt(first.par, h.value, 0, 0, first.h0.stream))


def _shares(shares) -> list:
    shares = list(shares)
    if not shares:
        raise FheError(_capi.INVALID_ARGUMENT, "MultipartyError::NoShares")
    return shares


class Aggregate:
    """mbfv::Aggregate (aggregate.rs): `Aggregate.from_shares(T, shares)` is the reference's `T::from_shares(shares)`
    for T = PublicKey (PublicKeyShare), Ciphertext (SecretKeySwitchShare or PublicKeySwitchShare), PlaintextVec /
    Plaintext (DecryptionShare; one plaintext per ciphertext, encoding None; Plaintext for one ciphertext),
    RelinKeyShare (round-1 RelinKeyShares into RelinKeyShare<R1Aggregated>) and RelinearizationKey (round-2 ones).  The first share supplies the CRP or the
    ciphertext, as in the reference."""

    @staticmethod
    def from_shares(target, shares):
        shares = _shares(shares)
        first = shares[0]
        if target is PublicKey and isinstance(first, PublicKeyShare):
            return _public_key(shares)
        if target is Ciphertext and isinstance(first, SecretKeySwitchShare) and not isinstance(first, DecryptionShare):
            return _switched(shares, "fhe_b200_sks_aggregate")
        if target is Ciphertext and isinstance(first, PublicKeySwitchShare):
            return _switched(shares, "fhe_b200_pks_aggregate")
        if isinstance(target, type) and issubclass(target, PlaintextVec) and isinstance(first, DecryptionShare):
            pts = _plaintexts(shares)
            if target is Plaintext:
                if len(pts) != 1:
                    raise FheError(_capi.INVALID_ARGUMENT, "a Plaintext is the decryption of one ciphertext")
                return Plaintext(pts.batch, None)
            return pts
        if target is RelinKeyShare and isinstance(first, RelinKeyShare):
            return _r1_aggregate(shares)
        if target is RelinearizationKey and isinstance(first, RelinKeyShare):
            return _relin_key(shares)
        raise FheError(_capi.INVALID_ARGUMENT, "no Aggregate of %s from %s" % (getattr(target, "__name__", target),
                                                                             type(first).__name__))


def aggregate(shares):
    """AggregateIter::aggregate (aggregate.rs): the type the shares aggregate into"""
    shares = _shares(shares)
    first = shares[0]
    if isinstance(first, PublicKeyShare):
        return _public_key(shares)
    if isinstance(first, DecryptionShare):
        return _plaintexts(shares)
    if isinstance(first, SecretKeySwitchShare):
        return _switched(shares, "fhe_b200_sks_aggregate")
    if isinstance(first, PublicKeySwitchShare):
        return _switched(shares, "fhe_b200_pks_aggregate")
    if isinstance(first, RelinKeyShare):
        return _r1_aggregate(shares) if first.round == "R1" else _relin_key(shares)
    raise FheError(_capi.INVALID_ARGUMENT, "not a share: %s" % type(first).__name__)


def _same_kind(shares, kind) -> None:
    for s in shares:
        if type(s) is not kind:
            raise FheError(_capi.INVALID_ARGUMENT, "cannot aggregate a %s with a %s" % (kind.__name__, type(s).__name__))


def _public_key(shares) -> PublicKey:   # public_key_gen.rs:60-77
    _same_kind(shares, PublicKeyShare)
    crp = shares[0].crp.batch
    if crp.count != 1:
        raise FheError(_capi.INVALID_ARGUMENT, "a public key is made from one CRP")
    pk = Ciphertext(shares[0].par, 1, 2, 0, NTT, crp.stream)
    check(_capi.lib().fhe_b200_pk_aggregate(_handles([s.p0_share for s in shares]), len(shares), crp._h, pk._h,
                                            pk.stream))
    return PublicKey(shares[0].par, pk)


def _switched(shares, fn: str) -> Ciphertext:   # secret_key_switch.rs:98-115, public_key_switch.rs:95-112
    _same_kind(shares, type(shares[0]))
    ct = shares[0].ct
    out = Ciphertext(ct.par, ct.count, 2, ct.level, NTT, ct.stream)
    check(getattr(_capi.lib(), fn)(ct._h, _handles([s.h_share for s in shares]), len(shares), out._h, out.stream))
    return out


def _plaintexts(shares) -> PlaintextVec:   # secret_key_switch.rs:145-186
    _same_kind(shares, DecryptionShare)
    ct = shares[0].ct
    out = Ciphertext(ct.par, ct.count, 1, ct.level, NTT, ct.stream)
    check(_capi.lib().fhe_b200_decryption_aggregate(ct.par.encoder(), ct._h, _handles([s.h_share for s in shares]),
                                                    len(shares), out._h, out.stream))
    return PlaintextVec(out, None)

"""Run by tests/test_gpu_mbfv.py::test_mbfv_chunking in a subprocess with a small FHE_B200_CHUNK and 1, 2 or 4
FHE_B200_STREAMS: CRPs, every share and every aggregate, the relinearization key protocol included, over batches that
span several chunks must give the words the stream and the restatement define for the whole call."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import encrypt_reference as R  # noqa: E402
import fhe_oracle as orc  # noqa: E402
import fhe_rs_b200 as F  # noqa: E402
import mbfv_reference as M  # noqa: E402

degree, t, count, level = 1 << 12, 1032193, 11, 1
opar = orc.BfvParameters(degree, t, moduli_sizes=[62] * 4)
par = F.BfvParameters(degree, t, moduli=opar.moduli, device=0)
rng = np.random.default_rng(int(os.environ.get("FHE_B200_CHUNK", "0")) + 700)
seed = lambda: rng.integers(0, 256, 32, dtype=np.uint8).tobytes()  # noqa: E731
osks = [orc.SecretKey(opar, rng) for _ in range(2)]
sks = [F.SecretKey(par, o.coeffs) for o in osks]

s = seed()
crps = F.mbfv.CommonRandomPoly._generate(par, count, level, s).to_host()[:, 0]
assert all((crps[k] == o.c).all() for k, o in enumerate(M.crp(opar, s, count, level)))
s = seed()
crp0 = F.mbfv.CommonRandomPoly._generate(par, count, 0, s)
ocrp0 = M.crp(opar, s, count, 0)
s = seed()
pks = F.mbfv.PublicKeyShare(sks[0], F.mbfv.CommonRandomPoly(crp0), s).p0_share.to_host()[:, 0]
assert all((pks[k] == o.c).all() for k, o in enumerate(M.pk_share(osks[0], ocrp0, s, 10)))

opk = M.pk_aggregate(opar, [M.pk_share(o, ocrp0[:1], seed(), 10)[0] for o in osks], ocrp0[0])
gpk = F.PublicKey(par, F.Ciphertext.from_host(par, opk.to_array()[None]))
values = rng.integers(0, t, size=count * degree, dtype=np.uint64)
octs = R.encrypt_pk(opar, opk, seed(), count, level, 10,
                    [R.to_poly(opar, values[k * degree:(k + 1) * degree], level) for k in range(count)])
ct = F.Ciphertext.from_host(par, np.stack([c.to_array() for c in octs]), level)

ss = [seed() for _ in sks]
gd = [F.mbfv.DecryptionShare(g, ct, x) for g, x in zip(sks, ss)]
od = [M.sks_share(o, None, octs, x, 10) for o, x in zip(osks, ss)]
for g, o in zip(gd, od):
    got = g.h_share.to_host()
    assert all((got[k, 0] == o[k].c).all() for k in range(count))
pts = F.mbfv.aggregate(gd).batch.to_host()
for k in range(count):
    assert (pts[k, 0] == M.from_shares(octs[k], [o[k] for o in od])[0].c).all(), k

ss = [seed() for _ in sks]
gs = F.mbfv.aggregate([F.mbfv.SecretKeySwitchShare(g, sks[1], ct, x) for g, x in zip(sks, ss)]).to_host()
os_ = [M.sks_share(o, osks[1], octs, x, 10) for o, x in zip(osks, ss)]
assert all((gs[k] == M.sks_aggregate(octs[k], [o[k] for o in os_]).to_array()).all() for k in range(count))

ss = [seed() for _ in sks]
gp = F.mbfv.aggregate([F.mbfv.PublicKeySwitchShare(g, gpk, ct, x) for g, x in zip(sks, ss)]).to_host()
op = [M.pks_share(o, opk, octs, x, 10) for o, x in zip(osks, ss)]
assert all((gp[k] == M.pks_aggregate(octs[k], [o[k] for o in op]).to_array()).all() for k in range(count))
# RelinKeyGenerator: rounds over the 4 CRPs / digits and the key's aggregate, in chunks of one digit
s = seed()
crps = F.mbfv.CommonRandomPoly.new_vec(par, s)
ocrps = M.crp(opar, s, 4)
su, s1, s2 = ([seed() for _ in sks] for _ in range(3))
gens = [F.mbfv.RelinKeyGenerator(g, crps, x) for g, x in zip(sks, su)]
us = [M.rkg_u(opar, x, 10) for x in su]
g1 = [g.round_1(x) for g, x in zip(gens, s1)]
o1 = [M.rkg_round1(o, ocrps, u, x, 10) for o, u, x in zip(osks, us, s1)]
for g, o in zip(g1, o1):
    assert (g.h0.to_host()[:, 0] == np.stack([p.c for p in o[0]])).all()
    assert (g.h1.to_host()[:, 0] == np.stack([p.c for p in o[1]])).all()
r1, or1 = F.mbfv.aggregate(g1), M.rkg_r1_aggregate(o1)
g2 = [g.round_2(r1, x) for g, x in zip(gens, s2)]
o2 = [M.rkg_round2(o, u, or1[0], or1[1], x, 10) for o, u, x in zip(osks, us, s2)]
c0, c1 = F.mbfv.aggregate(g2).ksk.arrays()
e0, e1 = M.rkg_aggregate(o2, or1[1])
assert (c0 == e0).all() and (c1 == e1).all()
print("mbfv chunk probe ok, chunk", os.environ.get("FHE_B200_CHUNK"), "streams", os.environ.get("FHE_B200_STREAMS"))

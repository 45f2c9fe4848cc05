"""The persistent TMA-fed kernels share a flat list of work items over a grid sized from the device: CTA b of a grid of
g takes items [items*b/g, items*(b+1)/g) (the TMA scaler: items b, b+g, ...), items are (limb, tile, ciphertext) with
the ciphertext innermost, and twiddles / key tiles are staged once per run of items that share them.  A staging or
ring-phase bug at one CTA boundary corrupts one tile of one ciphertext in the middle of a batch, so these tests check
every word of every output ciphertext at batch counts chosen to cut runs, chunks and streams.

The model tests (`-k model`) check on the CPU that the chosen counts reach each work-split regime of each kernel for
the SM counts of the H100 PCIe (114) and SXM (132), and on the device at hand."""
import json
import os
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import work_split_cases as W  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE = os.path.join(ROOT, "tests", "work_split_probe.py")


# ------------------------------------------------------------------------------------------------ model of the split
def cta_ranges(items, grid):
    """(lo, hi) of every CTA: the integer formula of the persistent kernels"""
    return [(items * b // grid, items * (b + 1) // grid) for b in range(grid)]


def grid_of(items, sm, per_sm):
    return min(items, sm * per_sm)


# CTAs per SM.  Fixed by __launch_bounds__ in ntt.cu (cols: ring depth 3, FHE_B200_TMA_COLS=2 ring depth 2, keyed by
# log2(N) - 6; rows: pair kernel, one-tile kernel; tensor rows), or an occupancy query (every value it could return).
COLS_MINB = {7: 4, 8: 2, 9: 1}
COLS_MINB_D2 = {7: 6, 8: 3, 9: 1}
ROWS_PAIR_MINB, ROWS_ONE_MINB, TENSOR_MINB = 3, 4, 2
OCCUPANCY = tuple(range(1, 9))
KERNELS = ("cols", "cols_d2", "rows_pair", "rows_one", "tensor_rows", "ks_rows_mac", "ksmac_tma", "scale_tma")


def chunks(count, chunk=256, streams=2):
    """ciphertexts per chunk of capi.cu::ChunkRunner"""
    if streams >= 2 and count > chunk and chunk >= streams:
        chunk = -(-chunk // streams)
    return [min(chunk, count - c0) for c0 in range(0, count, chunk)]


class Launch:
    """one launch of a persistent kernel: its items, the length of the runs that share staged constants, the
    ciphertexts of its chunk and the CTAs per SM it may get"""

    def __init__(self, kernel, items, run, cts, per_sm):
        self.kernel, self.items, self.run, self.cts, self.per_sm = kernel, items, run, cts, per_sm

    def unit(self):
        return self.items // self.cts   # items per ciphertext


def ntt_launches(logn, lpp, n_polys, tma_forced=False, d2=False, limb_inner=False, cts=None):
    """a two-pass TMA transform of n_polys polynomials of lpp limbs (ntt.cu::launch_ntt_tma), if it takes the TMA path"""
    if not (tma_forced or n_polys >= 8):
        return []
    cts = cts or n_polys
    tpr = (1 << (logn - 6)) // 16
    cols_k = "cols_d2" if d2 else "cols"
    minb = (COLS_MINB_D2 if d2 else COLS_MINB)[logn - 6]
    # cols: twiddles per limb; with the digit broadcast the limb is innermost (a new limb every item)
    out = [Launch(cols_k, lpp * 4 * n_polys, 1 if limb_inner else 4 * n_polys, cts, (minb,))]
    if limb_inner:
        return out   # its rows pass is the fused key switch
    if n_polys % 2 == 0:
        out.append(Launch("rows_pair", lpp * tpr * n_polys // 2, n_polys // 2, cts, (ROWS_PAIR_MINB,)))
    else:
        out.append(Launch("rows_one", lpp * tpr * n_polys, n_polys, cts, (ROWS_ONE_MINB,)))
    return out


def key_switch_launches(logn, n_dig, lk, c, cfg):
    n = 1 << logn
    tma = cfg.get("ntt") == "tma"
    if not (lk > 1 and (tma or c * n_dig >= 8)):
        return []   # not digit-adjacent: the per-thread inner product
    out = ntt_launches(logn, lk, c * n_dig, True, cfg.get("d2"), limb_inner=True, cts=c)
    if cfg.get("ksmac") == "tma":
        # the unfused rows pass of the digit transforms (digit-adjacent: pairs only for an even digit count)
        np_, tpr = c * n_dig, (n >> 6) // 16
        if np_ % 2 == 0 and n_dig % 2 == 0:
            out.append(Launch("rows_pair", lk * tpr * np_ // 2, np_ // 2, c, (ROWS_PAIR_MINB,)))
        else:
            out.append(Launch("rows_one", lk * tpr * np_, np_, c, (ROWS_ONE_MINB,)))
        out.append(Launch("ksmac_tma", lk * (n // 128) * c, c, c, OCCUPANCY))
    else:
        out.append(Launch("ks_rows_mac", lk * (n // 128) * c, c, c, OCCUPANCY))
    return out


def launches(name, count, cfg):
    """the persistent-kernel launches of the shape's operations on a count-`count` batch under switch set `cfg`"""
    s = W.SHAPES[name]
    logn, L = s["logn"], len(s["sizes"])
    n = 1 << logn
    K = 2 * L + 1          # the multiplication basis: L + L + 1 limbs of the default strategy
    solinas = all(b == 62 for b in s["sizes"])
    tma, d2 = cfg.get("ntt") == "tma", cfg.get("d2", False)
    ops = W.ops_for(name, count)
    out = []
    for c in chunks(count, cfg.get("chunk", 256), cfg.get("streams", 2)):
        for p in (1, 2, 3):
            if "fwd%d" % p in ops or "bwd%d" % p in ops:
                out += ntt_launches(logn, L, p * c, tma, d2, cts=c)
        for level, mul, rot in ((0, "mul", "rot3"), (1, "l1_mul", "l1_rot")):
            Ll = L - level
            if mul in ops:
                out += ntt_launches(logn, Ll, 2 * c, tma, d2, cts=c)                       # operands to power basis
                out += [Launch("scale_tma", 2 * c * (n // 128), n // 128, c, OCCUPANCY)]    # extension (62-bit primes)
                out += ntt_launches(logn, K - Ll, 2 * c, tma, d2, cts=c)                   # extension limbs forward
                if tma or 3 * c >= 8:
                    out.append(Launch("tensor_rows", K * ((n >> 6) // 16) * c, c, c, (TENSOR_MINB,)))
                out += ntt_launches(logn, K, 3 * c, True, d2, cts=c)[:1] if (tma or 3 * c >= 8) else []
                if solinas:
                    out.append(Launch("scale_tma", 3 * c * (n // 128), n // 128, c, OCCUPANCY))
                out += ntt_launches(logn, Ll, 2 * c, tma, d2, cts=c)
                out += key_switch_launches(logn, Ll, L, c, cfg)
            if rot in ops:
                out += ntt_launches(logn, Ll, c, tma, d2, cts=c)
                out += key_switch_launches(logn, Ll, L, c, cfg)
        if "ks" in ops:
            out += ntt_launches(logn, L, c, tma, d2, cts=c)
            out += key_switch_launches(logn, L, L, c, cfg)
        if "decrypt" in ops and solinas:
            out.append(Launch("scale_tma", c * (n // 128), n // 128, c, OCCUPANCY))   # one output row: polys == cts
    return out


# the switch sets the module runs (test_sweep_under_switch), as the model sees them: part 2's N = 2^13 shapes again,
# and under FHE_B200_NTT=tma also N = 2^14 and N = 2^15 at 1 and 3 ciphertexts, where only the forced TMA path puts
# fewer items than SMs into the cols pass
N13 = {"n13_2x62": None, "n13_62_40_30": None}
SWEEP_ENVS = [
    ({"FHE_B200_TMA_COLS": "2", "FHE_B200_NTT": "tma"}, N13),
    ({"FHE_B200_KS_STAGES": "3"}, N13),
    ({"FHE_B200_KS_STAGES": "4", "FHE_B200_KSMAC": "tma", "FHE_B200_NTT": "tma"}, N13),
    ({"FHE_B200_SCALE_UNROLL": "4"}, N13),
    ({"FHE_B200_NTT": "tma"}, dict(N13, n14_8x62=None, n15_14x62=[1, 3])),
    ({"FHE_B200_STREAMS": "1"}, N13),
    ({"FHE_B200_CHUNK": "5", "FHE_B200_STREAMS": "3"}, N13),
    ({"FHE_B200_CHUNK": "13", "FHE_B200_STREAMS": "4"}, N13),
]


def cfg_of(env):
    return {"ntt": env.get("FHE_B200_NTT"), "d2": env.get("FHE_B200_TMA_COLS") == "2", "ksmac": env.get("FHE_B200_KSMAC"),
            "chunk": int(env.get("FHE_B200_CHUNK", 256)), "streams": int(env.get("FHE_B200_STREAMS", 2))}


def sweep_counts(shapes):
    return {name: counts or W.SHAPES[name]["counts"] for name, counts in shapes.items()}


def all_launches():
    out = [x for name in W.SHAPES for c in W.SHAPES[name]["counts"] for x in launches(name, c, cfg_of({}))]
    for env, shapes in SWEEP_ENVS:
        out += [x for name, counts in sweep_counts(shapes).items() for c in counts for x in launches(name, c, cfg_of(env))]
    return out


def regimes(launch, sm, per_sm):
    """the regimes one launch reaches on `sm` SMs at `per_sm` CTAs per SM"""
    cap = sm * per_sm
    items, run = launch.items, launch.run
    got = set()
    if items < cap or launch.unit() >= cap:   # (a) cannot happen when one ciphertext already fills the grid
        got.add("a")
    if items < cap:
        got.add("a")
    if cap < items <= cap + launch.unit():   # the first count whose items exceed one CTA each
        got.add("b")
    if launch.kernel == "scale_tma":   # grid-stride: CTA b takes b, b + g, ...
        g = grid_of(items, sm, per_sm)
        starts = [(b, b + g * ((items - 1 - b) // g)) for b in range(g)]
        rng = [(lo, hi + 1) for lo, hi in starts]
    else:
        rng = cta_ranges(items, grid_of(items, sm, per_sm))
    if any(lo % run for lo, hi in rng if hi > lo) and any(hi % run for lo, hi in rng if hi > lo):
        got.add("c")
    if launch.cts == 1:
        got.add("d")
    return got


def missing_regimes(sm, launches_=None):
    """[(kernel, CTAs per SM, regime)] that no launch of the module reaches on `sm` SMs"""
    ls = all_launches() if launches_ is None else launches_
    miss = []
    for k in KERNELS:
        mine = [x for x in ls if x.kernel == k]
        opts = sorted(set(p for x in mine for p in x.per_sm)) or [None]
        for m in opts:
            have = set()
            for x in mine:
                if m in x.per_sm:
                    have |= regimes(x, sm, m)
            for r in "abcd":
                if r not in have:
                    miss.append((k, m, r))
    return miss


def test_model_cta_ranges():
    """the ranges tile [0, items) exactly, every CTA has one when items >= grid, and they match the kernels' u32
    arithmetic ((u64)items * b / grid)"""
    for items, grid in ((1, 1), (5, 7), (133, 132), (528, 528), (529, 528), (16 * 67, 264), (1 << 20, 456)):
        g = min(items, grid)
        r = cta_ranges(items, g)
        assert r[0][0] == 0 and r[-1][1] == items
        assert all(r[k][1] == r[k + 1][0] for k in range(g - 1))
        assert all(hi > lo for lo, hi in r)
        assert max(hi - lo for lo, hi in r) - min(hi - lo for lo, hi in r) <= 1
    assert chunks(259) == [128, 128, 3] and chunks(256) == [256] and chunks(12, 5, 3) == [2] * 6
    assert chunks(67, 13, 4) == [4] * 16 + [3] and chunks(7, 5, 3) == [2, 2, 2, 1]


@pytest.mark.parametrize("sm", [114, 132])
def test_model_regimes(sm, monkeypatch):
    """for the H100 PCIe (114 SMs) and SXM (132 SMs): for every persistent kernel and every CTAs-per-SM value it may
    get, the module's counts reach (a) items < grid capacity, (b) the first count above it, (c) a CTA range that starts
    and one that ends inside a run, and (d) runs of one ciphertext"""
    assert missing_regimes(sm) == []
    # the model notices a count that stops reaching a regime: without 14 ciphertexts at N = 2^13 no launch of the
    # 6-CTA-per-SM cols kernel (FHE_B200_TMA_COLS=2) is the first above one wave on 132 SMs
    monkeypatch.setitem(W.SHAPES["n13_2x62"], "counts", [c for c in W.SHAPES["n13_2x62"]["counts"] if c != 14])
    assert (("cols_d2", 6, "b") in missing_regimes(sm)) == (sm == 132)


@pytest.mark.gpu
def test_model_regimes_on_this_device(F):
    import torch
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    assert missing_regimes(sm) == [], sm


# ------------------------------------------------------------------------------------------------ parity on the device
@pytest.fixture(scope="module")
def F():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


_EXPECTED = {}


def expected(name):
    """the oracle's digests of every output ciphertext of the shape, computed once per module"""
    if name not in _EXPECTED:
        _EXPECTED[name] = W.oracle_expected(name, max(1, min(16, os.cpu_count() or 1)))
    return _EXPECTED[name]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(W.SHAPES))
def test_every_word_against_oracle(F, name):
    """default switches: every word of every output ciphertext of every operation at every count of the shape"""
    got = W.device_digests(F, name)
    exp = expected(name)
    assert set(got) == set(exp)
    bad = W.compare(got, exp)
    assert bad == [], bad[:20]


def _probe(args, env, timeout=850):
    out = subprocess.run([sys.executable, PROBE] + args, cwd=ROOT, env=dict(os.environ, **env), capture_output=True,
                         text=True, timeout=timeout)
    assert out.returncode == 0 and "work split probe ok" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("env,shapes", SWEEP_ENVS, ids=[",".join("%s=%s" % (k[9:], v) for k, v in e.items())
                                                        for e, _ in SWEEP_ENVS])
def test_sweep_under_switch(F, env, shapes, tmp_path):
    """the sweep again under each switch that changes a kernel's ring depth, residency or the chunking"""
    path = str(tmp_path / "sweep.json")
    _probe(["sweep", path, json.dumps(sweep_counts(shapes))], env)
    with open(path) as f:
        got = json.load(f)
    for name, counts in sweep_counts(shapes).items():
        exp = {k: v for k, v in expected(name).items() if int(k.split("@")[1]) in counts}
        bad = W.compare(got[name], exp)
        assert bad == [], (name, bad[:20])


NO_PERSISTENT = {"FHE_B200_NTT": "fast", "FHE_B200_KSMAC": "classic", "FHE_B200_SCALER": "classic",
                 "FHE_B200_NO_TENSOR_FUSION": "1"}


@pytest.mark.gpu
def test_benchmarked_batch_against_no_persistent_path(F, tmp_path):
    """520 set-C pairs (4 x 128 + 8), every product and rotation: the default path equals the path with no persistent
    kernel at all (one CTA per tile, one thread per word), which is itself pinned to the oracle at 0, 259 and 519"""
    _probe(["bench", str(tmp_path / "default.json")], {})
    _probe(["bench", str(tmp_path / "plain.json"), "--oracle"], NO_PERSISTENT)
    with open(tmp_path / "default.json") as f:
        a = json.load(f)
    with open(tmp_path / "plain.json") as f:
        b = json.load(f)
    assert b["oracle_checked"] == [0, 259, 519]
    for op in ("mul", "rot3"):
        assert len(a[op]) == len(b[op]) == 520
        diff = [i for i in range(520) if a[op][i] != b[op][i]]
        assert diff == [], (op, diff[:20])


@pytest.mark.gpu
def test_host_threads_share_parameters(F):
    """include/fhe_b200.h: a parameter set may be shared by host threads.  Four threads on their own streams, with
    different counts and levels, build the parameter set's lazy tables concurrently; their results equal the same calls
    made one thread at a time."""
    out = _probe(["threads"], {"FHE_B200_CHUNK": "4"})
    assert "threads probe ok" in out.stdout

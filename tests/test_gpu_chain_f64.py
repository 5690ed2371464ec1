"""The filter kernels behind stage 1 (k_dfir_reg, k_poly_reg, k_fir_reg, k_firr_reg and their tiled fall-backs) against
float64 references, sample by sample, from output 0 of the stream.

Part A (CPU): plain numpy float64 restatements of FIR / DecimatingFIR (fir.h:62-83, decimating_fir.h:45-68) and of the
polyphase resampler (polyphase_resampler.h:69-99; bank as in polyphase_bank.h), pinned to the oracle's fp32 blocks with the
per-sample bound below.  Part B (GPU): every register-window build through a stand-alone block (same scheduler, same dispatch
as the front end), with asymmetric random taps and a chunk schedule that hits tile edges, both decimation parities, stale
samples past a short chunk and graph replay.  Part C (GPU): RAW VFOs in the front end against the exact-phase oracle, with a
complex-gain gate and an edge-against-interior gate that an RMS over the whole stream cannot give.

Per-sample bound (fp32 accumulation, any summation order, split sums included): for every output and real component
    |y - y64| <= (T_eff + 2) 2^-24 sum_k |h_k| (|Re x| + |Im x|)
with T_eff the taps of that output (taps per phase for the resampler); a cascade adds the stage bounds and carries the incoming
bound through sum_k |h_k|.  No tolerance here is fitted to a run.
"""
import numpy as np
import pytest
from scipy.signal import oaconvolve

from util import noise_iq, rel_rms

U = 2.0 ** -24                      # unit round-off of fp32
REF_FLOOR = 2.0 ** -40              # float64 FFT convolution error, relative to sum|h| max|x|: far below any fp32 rounding
MAX_CHUNK = 1000000                 # a stand-alone block's chunk limit (STREAM_BUFFER_SIZE)

# ---------------------------------------------------------------------------------------------- routing (mirrors engine.cpp)
DFR_R = {(4, 27): 8, (2, 69): 4, (2, 12): 8, (8, 54): 4, (8, 44): 4, (8, 36): 4}   # outputs per thread (dfir_reg.cuh:107-112)
DFR_MAXT = 72                                                                     # kernels.cuh: DfrParams.taps
POLY_REG = {(16, 25), (5, 6), (2, 3), (4, 5), (2, 5)}                             # tails_reg.cuh:138-140
TS_TILE = 256                                                                     # k_fir_reg / k_firr_reg outputs per CTA
PR_PER = 32                                                                       # k_poly_reg periods per CTA
PLAN_RATIO = {(2, 69): 2, (2, 12): 4, (4, 27): 8, (8, 54): 16, (8, 44): 32, (8, 36): 64}   # plan whose stage 0 is (D, T)


def routes_dfir_reg(D, T):
    """engine.cpp:1273-1277 (dfr_ok) with dfir_reg.cuh:100-102"""
    return D > 1 and T <= DFR_MAXT and (D, T) in DFR_R


def routes_fir_reg(D, T):
    """engine.cpp:1454: decimation 1, at most 2000 taps (the chunk offset of a decimation-1 filter is always 0)"""
    return D == 1 and T <= 2000


def routes_firr_reg(T):
    """engine.cpp:1504"""
    return T <= 2000


def routes_poly_reg(L, M, tpp):
    """engine.cpp:1472"""
    return (L, M) in POLY_REG and tpp <= 512


# ---------------------------------------------------------------------------------------------- float64 references
def _corr(x, h):
    """z[o] = sum_k h[k] x[o + k] for o = 0 .. len(x) - len(h)  (float64)"""
    if x.size < h.size:
        return np.zeros(0, x.dtype)
    if h.size <= 64 or x.size <= 4 * h.size:
        return np.convolve(x, h[::-1], "valid")
    return oaconvolve(x, h[::-1], "valid")


def _hist(v, k):
    return np.concatenate([np.zeros(k, v.dtype), v])


def _abs_parts(x):
    return np.abs(x.real) + (np.abs(x.imag) if np.iscomplexobj(x) else 0.0)


def fir_f64(x, e, h, D=1):
    """FIR / DecimatingFIR from zero history: y[m] = sum_k h[k] xh[m D + k], xh = [T-1 zeros | x].
    x: float64 input, e: per-sample bound of x's error (None = exact fp32 input).  Returns (y, bound of y)."""
    h = np.asarray(h, np.float64)
    T = h.size
    y = _corr(_hist(x, T - 1), h)[::D]
    a = _abs_parts(x) + (2.0 * e if e is not None else 0.0)
    ah = np.abs(h)
    b = (T + 2) * U * _corr(_hist(a, T - 1), ah)[::D]
    if e is not None:
        b = b + _corr(_hist(e, T - 1), ah)[::D]
    return y, b + REF_FLOOR * ah.sum() * (float(a.max()) if a.size else 0.0)


def poly_bank(taps, L):
    """buildPolyphaseBank: bank[(L-1) - i % L][i // L] = taps[i], zero-padded to ceil(T / L) taps per phase"""
    taps = np.asarray(taps, np.float64)
    tpp = -(-taps.size // L)
    bank = np.zeros((L, tpp))
    i = np.arange(taps.size)
    bank[(L - 1) - i % L, i // L] = taps
    return bank


def poly_out_index(n, L, M):
    """outputs m of an n-sample stream: off = m M // L (< n), bank row ph = m M % L"""
    m = np.arange((n * L + M - 1) // M, dtype=np.int64)
    return (m * M) // L, (m * M) % L


def poly_f64(x, e, taps, L, M):
    """PolyphaseResampler from zero history: y[m] = sum_j bank[ph][j] xh[off + j], xh = [tpp-1 zeros | x]"""
    bank = poly_bank(taps, L)
    tpp = bank.shape[1]
    off, ph = poly_out_index(x.size, L, M)
    xh = _hist(x, tpp - 1)
    a = _abs_parts(x) + (2.0 * e if e is not None else 0.0)
    ah = _hist(a, tpp - 1)
    eh = _hist(e, tpp - 1) if e is not None else None
    y = np.zeros(off.size, x.dtype)
    b = np.zeros(off.size)
    for p in range(L):
        sel = ph == p
        if not sel.any():
            continue
        o = off[sel]
        y[sel] = _corr(xh, bank[p])[o]
        b[sel] = (tpp + 2) * U * _corr(ah, np.abs(bank[p]))[o]
        if eh is not None:
            b[sel] += _corr(eh, np.abs(bank[p]))[o]
    return y, b + REF_FLOOR * np.abs(bank).sum(axis=1).max() * (float(a.max()) if a.size else 0.0)


# ---------------------------------------------------------------------------------------------- chunk bookkeeping
def fir_counts(sched, D):
    """per-chunk outputs and the chunk's offset into [history | data] (DecimatingFIR::process's `offset`)"""
    off, outs, offs = 0, [], []
    for n in sched:
        no = (n - off + D - 1) // D if off < n else 0
        offs.append(off)
        outs.append(no)
        off = off + no * D - n
    return outs, offs


def poly_counts(sched, L, M):
    off, ph, outs = 0, 0, []
    for n in sched:
        avail = (n - off) * L - ph
        no = (avail + M - 1) // M if avail > 0 else 0
        tend = ph + no * M
        off, ph = off + tend // L - n, tend % L
        outs.append(no)
    return outs


def cascade_counts(sched, stages):
    """stages: ("fir", D) / ("poly", L, M); returns the last stage's outputs per chunk"""
    cur = list(sched)
    for s in stages:
        cur = fir_counts(cur, s[1])[0] if s[0] == "fir" else poly_counts(cur, s[1], s[2])
    return cur


def schedule(tile_in, T, total=200000, seed=0, repeat=None):
    """0- and 1-sample chunks, one shorter than T-1, one CTA tile and one sample either side, a long chunk followed by short
    ones (stale samples of the long one lie past the end of the short ones), >= 3 repeats of one size (the recorded launch
    list is replayed as a graph), odd sizes (both parities of a decimation offset) filling up to `total`."""
    rng = np.random.default_rng(seed)
    rep = repeat or tile_in
    s = [0, 1, max(0, (T - 2) // 2), 3, tile_in, tile_in + 1, tile_in - 1, 0, 1]
    s += [min(MAX_CHUNK, max(60000, 8 * tile_in)), 7, 2, 13, 1]
    s += [rep] * 6
    while sum(s) + 12000 + tile_in + 1 < total:
        s.append(int(rng.integers(500, 12000)) | 1)
    s.append(tile_in + 1)
    while sum(s) < total:
        s.append(min(total - sum(s), MAX_CHUNK))
    return [int(v) for v in s]


def predec_schedule(tile, T, seed):
    """behind a large predecimator a resampler tile is longer than a chunk: the same kinds of chunk, capped at the chunk
    limit, repeats of a whole resampler period, 6 M samples (~300 outputs at 1 kS/s from 20.48 MS/s)"""
    return schedule(MAX_CHUNK - 1, T, 6000000, seed, repeat=tile // 8)


# ---------------------------------------------------------------------------------------------- cases of part B
def _cases():
    c = []
    for (D, T) in DFR_R:
        c.append(("dfir_D%d_T%d_random" % (D, T), "firc", dict(D=D, T=T, taps="random")))
        c.append(("dfir_D%d_T%d_plan" % (D, T), "firc", dict(D=D, T=T, taps="plan")))
    for r in (4, 32, 64, 512, 4096):
        c.append(("decim_%d" % r, "decim", dict(ratio=r)))
    for T in (1, 2, 7, 8, 9, 63, 64, 65, 255, 1000, 2000):
        c.append(("fir_cr_T%d" % T, "firc", dict(D=1, T=T, taps="random")))
        c.append(("fir_rr_T%d" % T, "firr", dict(T=T)))
    for rates in ((300e3, 250e3), (48e3, 32e3), (250e3, 200e3), (250e3, 160e3), (20.48e6, 1e3)):
        c.append(("resamp_%g_%g" % rates, "resamp", dict(rates=rates)))
    # tiled fall-backs: the same checks, routed away from the register kernels
    c.append(("fallback_dfir_D3_T50", "firc", dict(D=3, T=50, taps="random")))
    c.append(("fallback_fir_cr_T2001", "firc", dict(D=1, T=2001, taps="random")))
    c.append(("fallback_fir_rr_T2001", "firr", dict(T=2001)))
    c.append(("fallback_resamp_48000_44100", "resamp", dict(rates=(48e3, 44.1e3))))
    return c


CASES = _cases()
CASE_IDS = [c[0] for c in CASES]


def _random_taps(T, seed):
    return np.random.default_rng(1000 + seed).uniform(-1.0, 1.0, T).astype(np.float32)


class Spec:
    """what one case runs: its stages (for the reference and the counts), its taps, input kind, chunk schedule"""

    def __init__(self, oracle, name, kind, p):
        from sdrplusplus_b200 import frontend
        self.name, self.kind, self.p = name, kind, p
        self.complex = kind != "firr"
        seed = CASE_IDS.index(name)
        self.total = 200000
        if kind == "firc":
            D, T = p["D"], p["T"]
            h = oracle.decim_taps(PLAN_RATIO[(D, T)], 0) if p["taps"] == "plan" else _random_taps(T, seed)
            assert h.size == T
            self.stages = [("fir", D, h)]
            tile = TS_TILE if D == 1 else 128 * DFR_R.get((D, T), 4) * D
        elif kind == "firr":
            self.stages = [("fir", 1, _random_taps(p["T"], seed))]
            tile = TS_TILE
        elif kind == "decim":
            plan = oracle.decim_plan(p["ratio"])
            self.stages = [("fir", D, oracle.decim_taps(p["ratio"], k)) for k, (D, T) in enumerate(plan)]
            D0, T0 = plan[0]
            tile = 128 * DFR_R.get((D0, T0), 4) * D0
            self.total = max(200000, 2048 * p["ratio"])      # >= 2048 outputs
        else:
            rp = frontend.resamp_plan(*p["rates"])
            self.stages = []
            if rp["predec_ratio"] > 1:
                self.stages = [("fir", D, oracle.decim_taps(rp["predec_ratio"], k)) for k, (D, T) in enumerate(rp["stages"])]
            L, M = rp["interp"], rp["decim"]
            taps = oracle.resamp_taps(*p["rates"])
            assert taps.size == rp["ntaps"] and poly_bank(taps, L).shape[1] == rp["taps_per_phase"]
            self.stages.append(("poly", L, M, taps))
            self.plan = rp
            tile = PR_PER * M * rp["predec_ratio"]
        self.T = max(len(s[-1]) for s in self.stages)
        self.tile = tile
        self.sched = predec_schedule(tile, self.T, seed) if tile > MAX_CHUNK else schedule(tile, self.T, self.total, seed)
        self.total = sum(self.sched)
        self.single = len(self.stages) == 1

    def counts(self):
        return cascade_counts(self.sched, [s[:2] if s[0] == "fir" else s[:3] for s in self.stages])

    def reference(self, x):
        y, e = x.astype(np.complex128 if self.complex else np.float64), None
        for s in self.stages:
            y, e = fir_f64(y, e, s[2], s[1]) if s[0] == "fir" else poly_f64(y, e, s[3], s[1], s[2])
        return y, e

    def signal(self):
        seed = 77 + CASE_IDS.index(self.name)
        if self.complex:
            return noise_iq(self.total, seed, 1.0)
        return np.random.default_rng(seed).uniform(-1.0, 1.0, self.total).astype(np.float32)

    def gpu_block(self, sb):
        s0 = self.stages[0]
        if self.kind == "firc":
            return sb.Block.fir_cr(s0[2], s0[1])
        if self.kind == "firr":
            return sb.Block.fir_rr(s0[2])
        if self.kind == "decim":
            return sb.Block.decim(self.p["ratio"])
        return sb.Block.resamp(*self.p["rates"])

    def oracle_block(self, oracle):
        s0 = self.stages[0]
        if self.kind == "firc":
            return oracle.fir_cr(s0[2]) if s0[1] == 1 else oracle.decfir_cr(s0[2], s0[1])
        if self.kind == "firr":
            return oracle.fir_rr(s0[2])
        if self.kind == "decim":
            return oracle.decim(self.p["ratio"])
        return oracle.resamp(*self.p["rates"])


def _feed(block, x, sched, cplx):
    """one process() call per chunk; returns the per-chunk outputs"""
    xf = x.view(np.float32) if cplx else x
    w = 2 if cplx else 1
    outs, pos = [], 0
    for n in sched:
        y = block.process(xf[w * pos: w * (pos + n)])
        outs.append(y.view(np.complex64) if cplx else y)
        pos += n
    assert pos == x.size
    return outs


def _ratio(y, y64, b):
    y = np.asarray(y)
    if np.iscomplexobj(y64):
        err = np.maximum(np.abs(y.real - y64.real), np.abs(y.imag - y64.imag))
    else:
        err = np.abs(y - y64)
    return err / b


# ---------------------------------------------------------------------------------------------- part A (CPU)
REF_CHECKS = [("decfir", D, T) for (D, T) in DFR_R] + [("decfir", 3, 50), ("fir_cr", 1, 1), ("fir_cr", 1, 2000),
                                                       ("fir_cr", 1, 63), ("fir_rr", 1, 65), ("fir_rr", 1, 2000)]


@pytest.mark.parametrize("kind,D,T", REF_CHECKS)
def test_fir_reference_matches_oracle(oracle, kind, D, T):
    """the float64 FIR reference's index convention and output count are those of the reference's fp32 blocks"""
    h = np.random.default_rng(T * 7 + D).uniform(-1.0, 1.0, T).astype(np.float32)
    cplx = kind != "fir_rr"
    n = 200000
    x = noise_iq(n, T + D, 1.0) if cplx else np.random.default_rng(T).uniform(-1, 1, n).astype(np.float32)
    tile = TS_TILE if D == 1 else 128 * DFR_R.get((D, T), 4) * D
    sched = schedule(tile, T, n, T)
    blk = oracle.fir_rr(h) if kind == "fir_rr" else (oracle.decfir_cr(h, D) if kind == "decfir" else oracle.fir_cr(h))
    outs = _feed(blk, x, sched, cplx)
    assert [o.size for o in outs] == fir_counts(sched, D)[0]
    y64, b = fir_f64(x.astype(np.complex128 if cplx else np.float64), None, h, D)
    y = np.concatenate(outs)
    assert y.size == y64.size == len(range(0, n, D))
    r = float(np.max(_ratio(y, y64, b)))
    assert r <= 1.0, r


@pytest.mark.parametrize("rates", [(300e3, 250e3), (48e3, 32e3), (250e3, 200e3), (250e3, 160e3), (48e3, 44.1e3), (20.48e6, 1e3)])
def test_resampler_reference_matches_oracle(oracle, rates):
    """the float64 polyphase reference (bank layout, phase / offset recurrence, output count) against the oracle's fp32
    RationalResampler, the predecimator cascade included"""
    q = oracle.resamp_plan(*rates)
    L, M = q["interp"], q["decim"]
    taps = oracle.resamp_taps(*rates)
    stages = []
    if q["predec_ratio"] > 1:
        stages = [("fir", D, oracle.decim_taps(q["predec_ratio"], k)) for k, (D, T) in enumerate(oracle.decim_plan(q["predec_ratio"]))]
    stages.append(("poly", L, M, taps))
    tile = PR_PER * M * q["predec_ratio"]
    sched = predec_schedule(tile, q["taps_per_phase"], L) if tile > MAX_CHUNK else schedule(tile, q["taps_per_phase"], 200000, L)
    n = sum(sched)
    x = noise_iq(n, L + M, 1.0)
    outs = _feed(oracle.resamp(*rates), x, sched, True)
    assert [o.size for o in outs] == cascade_counts(sched, [s[:2] if s[0] == "fir" else s[:3] for s in stages])
    y64, e = x.astype(np.complex128), None
    for s in stages:
        y64, e = fir_f64(y64, e, s[2], s[1]) if s[0] == "fir" else poly_f64(y64, e, s[3], s[1], s[2])
    y = np.concatenate(outs)
    assert y.size == y64.size
    r = float(np.max(_ratio(y, y64, e)))
    assert r <= 1.0, r


def test_impulse_answer_of_the_references():
    """the index formulas the GPU impulse checks use agree with the references (an asymmetric table shows a reversal)"""
    h = np.arange(1, 12, dtype=np.float32)
    x = np.zeros(100)
    x[40] = 1.0
    for D in (1, 2, 3):
        y, _ = fir_f64(x, None, h, D)
        want = np.zeros(len(range(0, 100, D)))
        for m in range(want.size):
            k = h.size - 1 + 40 - m * D
            if 0 <= k < h.size:
                want[m] = h[k]
        assert np.array_equal(y.round(9), want)
    bank = poly_bank(h, 3)
    y, _ = poly_f64(x, None, h, 3, 5)
    off, ph = poly_out_index(100, 3, 5)
    tpp = bank.shape[1]
    want = np.array([bank[p, 40 + tpp - 1 - o] if 0 <= 40 + tpp - 1 - o < tpp else 0.0 for o, p in zip(off, ph)])
    assert np.array_equal(y.round(9), want)


@pytest.mark.parametrize("name", CASE_IDS)
def test_case_routes_where_intended(oracle, name):
    """each part-B case reaches the kernel build it is named after (same predicates as the scheduler), and its chunk
    schedule has what it needs: a CTA tile and one sample either side, empty and 1-sample chunks, repeats, and both
    parities of a decimation offset for k_dfir_reg"""
    kind, p = dict((c[0], c[1:]) for c in CASES)[name]
    sp = Spec(oracle, name, kind, p)
    fallback = name.startswith("fallback")
    for s in sp.stages:
        if s[0] == "fir" and kind == "firr":
            assert routes_firr_reg(s[2].size) != fallback
        elif s[0] == "fir" and s[1] == 1:
            assert routes_fir_reg(1, s[2].size) != fallback
        elif s[0] == "fir":
            D, T = s[1], s[2].size
            if kind == "firc":
                assert routes_dfir_reg(D, T) != fallback
        else:
            assert routes_poly_reg(s[1], s[2], poly_bank(s[3], s[1]).shape[1]) != fallback
    if kind == "decim":
        D0, T0 = sp.stages[0][1], sp.stages[0][2].size
        assert all(routes_dfir_reg(s[1], s[2].size) for s in sp.stages[1:])
        assert routes_dfir_reg(D0, T0) == (p["ratio"] not in (512, 4096))
    sched = sp.sched
    assert 0 in sched and 1 in sched
    t = min(sp.tile, MAX_CHUNK - 1)
    assert {t - 1, t, t + 1} <= set(sched)
    assert max(sched.count(v) for v in set(sched) if v > 1) >= 3
    if sp.T > 2:
        assert min(v for v in sched if v > 0) < sp.T - 1
    if kind == "firc" and sp.stages[0][1] > 1:
        D = sp.stages[0][1]
        outs, offs = fir_counts(sched, D)
        # k_dfir_reg: sh = (offset + first output of the tile * D) & 1 (dfir_reg.cuh:34-35), = offset & 1 for even D
        assert {o & 1 for o, n in zip(offs, outs) if n > 0} == {0, 1}


def test_cascade_cases_cover_every_dfir_build(oracle):
    """Block.decim(4 / 32 / 64 / 512 / 4096) runs every k_dfir_reg build at least once behind another stage"""
    seen = set()
    for r in (4, 32, 64, 512, 4096):
        seen |= {st for st in oracle.decim_plan(r)[1:] if routes_dfir_reg(*st)} | {oracle.decim_plan(r)[0]}
    assert set(DFR_R) <= seen


# ---------------------------------------------------------------------------------------------- part B (GPU)
@pytest.fixture(scope="module")
def sb():
    import sdrplusplus_b200 as m
    from sdrplusplus_b200 import lib
    L = lib.load()
    assert L.b200_device_count() > 0
    assert L.b200_init(0) == 0
    return m


def _impulse_positions(sp, n):
    """impulses at every residue mod D, at chunk starts (and one sample either side) and at CTA tile edges inside chunks,
    far enough apart that no output sees two of them"""
    s0 = sp.stages[0]
    if s0[0] == "fir":
        D, T = s0[1], s0[2].size
        sep = T + D + 1
    else:
        L, M = s0[1], s0[2]
        D, T = M, poly_bank(s0[3], L).shape[1]
        sep = T + M // L + 2
    starts = np.cumsum([0] + sp.sched[:-1])
    cand = []
    for st, ln in zip(starts, sp.sched):
        cand += [st - 1, st, st + 1]
        for k in range(1, 4):
            cand += [st + k * sp.tile - 1, st + k * sp.tile]
    step = max(sep, 257)
    cand += [i * (step + D) + i % D for i in range(1, n // (step + D))]     # every residue mod D along the stream
    keep, last = [], -sep
    for c in sorted(set(int(v) for v in cand if 0 <= v < n)):
        if c - last >= sep:
            keep.append(c)
            last = c
    keep = np.array(keep)
    if s0[0] == "fir" and D > 1:
        assert set(keep % D) == set(range(D))
    return keep


def _impulse_expected(sp, pos, vals, nout):
    s0 = sp.stages[0]
    y = np.zeros(nout, np.complex128 if sp.complex else np.float64)
    if s0[0] == "fir":
        D, h = s0[1], s0[2].astype(np.float64)
        T = h.size
        for p, v in zip(pos, vals):
            m = np.arange(-(-p // D), min(nout - 1, (p + T - 1) // D) + 1)
            y[m] = h[T - 1 + p - m * D] * v
    else:
        L, M = s0[1], s0[2]
        bank = poly_bank(s0[3], L)
        tpp = bank.shape[1]
        off, ph = poly_out_index(sum(sp.sched), L, M)
        for p, v in zip(pos, vals):
            m = np.arange(-(-p * L // M), min(nout, -(-(p + tpp) * L // M)))
            m = m[(off[m] >= p) & (off[m] <= p + tpp - 1)]
            y[m] = bank[ph[m], p + tpp - 1 - off[m]] * v
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_IDS)
def test_chain_kernel_vs_float64(sb, oracle, report, name):
    kind, p = dict((c[0], c[1:]) for c in CASES)[name]
    sp = Spec(oracle, name, kind, p)
    x = sp.signal()
    counts = sp.counts()
    blk = sp.gpu_block(sb)
    outs = _feed(blk, x, sp.sched, sp.complex)
    # 1. output count, chunk by chunk
    assert [o.size for o in outs] == counts
    # 2. every sample within the fp32 bound, from output 0
    y64, b = sp.reference(x)
    y = np.concatenate(outs)
    assert y.size == y64.size
    r = _ratio(y, y64, b)
    worst = float(np.max(r)) if r.size else 0.0
    report["chain_f64_" + name] = {"max_err_over_bound": worst, "worst_output": int(np.argmax(r)) if r.size else -1,
                                   "outputs": int(y.size), "rel_rms": rel_rms(y, y64)}
    assert worst <= 1.0, (worst, int(np.argmax(r)), y.size)
    # 4. reset() + the same input gives the bits of a fresh block
    blk.reset()
    again = np.concatenate(_feed(blk, x, sp.sched, sp.complex))
    assert np.array_equal(again.view(np.uint32), y.view(np.uint32))
    blk.close()
    # 3. unit impulses return the taps exactly, at the predicted outputs, and 0 elsewhere (one stage only)
    if sp.single:
        n = x.size
        pos = _impulse_positions(sp, n)
        vals = np.where(np.arange(pos.size) % 2 == 0, 1.0, 1j) if sp.complex else np.where(np.arange(pos.size) % 2 == 0, 1.0, -2.0)
        imp = np.zeros(n, np.complex64 if sp.complex else np.float32)
        imp[pos] = vals
        blk = sp.gpu_block(sb)
        yi = np.concatenate(_feed(blk, imp, sp.sched, sp.complex))
        blk.close()
        want = _impulse_expected(sp, pos, vals, yi.size)
        bad = np.flatnonzero(yi != want)
        assert bad.size == 0, (bad[:8], yi[bad[:8]], want[bad[:8]])


# ---------------------------------------------------------------------------------------------- part C (GPU): RAW VFOs in situ
FS_C = 2.4e6
C_RATES = [250e3] * 3 + [125e3] * 3 + [50e3] * 5 + [24e3] * 5 + [15e3] * 5 + [12.5e3] * 5   # 26 VFOs
SCHED_C = [0, 1, 7, 100003] + [240000] * 6 + [131071, 5, 0, 160001, 3, 120000, 239999]
FS_G = 100e6
OFFS_G = [5e6, -5e6, 15e6, -15e6, 25e6, -25e6, 35e6, -35e6]
SCHED_G = [0, 1, 300001] + [1 << 20] * 3 + [7, 499999, 777777]
EDGE = 64
C_OPTIONS = [{}, {"tails": 1}, {"tails": 0}, {"ft_regall": 0}, {"ft_prereg": 0}]


def test_in_situ_plans_reach_every_register_build(oracle):
    """the 2.4 MS/s VFO set puts k_dfir_reg (2,69) (2,12) (4,27), k_poly_reg 5/6 2/3 16/25 4/5 and k_fir_reg behind
    stage 1, more than 16 VFOs of one stage kind at one level (two launch batches), and its repeated chunk is a whole
    period of every plan (identical launch parameters: graph replay)"""
    from sdrplusplus_b200 import frontend
    dfr, poly = set(), set()
    deep = 0
    for r in C_RATES:
        p = frontend.resamp_plan(FS_C, r)
        behind = p["stages"][1:]
        assert all(routes_dfir_reg(*st) for st in behind)
        dfr |= set(behind)
        assert routes_poly_reg(p["interp"], p["decim"], p["taps_per_phase"])
        poly.add((p["interp"], p["decim"]))
        bw = 0.8 * r
        assert routes_fir_reg(1, oracle.lowpass(bw / 2, 0.1 * bw / 2, r).size)
        deep += len(p["stages"]) == 3
        assert 240000 % (p["predec_ratio"] * p["decim"]) == 0
    assert dfr == {(2, 69), (2, 12), (4, 27)}
    assert poly == {(5, 6), (2, 3), (16, 25), (4, 5)}
    assert deep > 16
    g = frontend.resamp_plan(FS_G, 250e3)
    assert all(routes_dfir_reg(*st) for st in g["stages"][1:]) and set(g["stages"][1:]) == {(4, 27), (2, 69)}


def _c_offsets():
    return [-1.1e6 + k * (2.2e6 / len(C_RATES)) + 1234.5 for k in range(len(C_RATES))]


@pytest.fixture(scope="module")
def c_input():
    n = sum(SCHED_C)
    x = noise_iq(n, 4242, 0.5)
    return x


def _oracle_raw(oracle, x, fs, sched, cfgs):
    """exact-phase oracle RxVFO per VFO, chunk by chunk"""
    oracle.set_rotator_mode(1)
    try:
        res = []
        xf = x.view(np.float32)
        for (off, rate, bw) in cfgs:
            v = oracle.rxvfo(fs, rate, bw, off)
            parts, pos = [], 0
            for n in sched:
                parts.append(v.process(xf[2 * pos: 2 * (pos + n)]).view(np.complex64))
                pos += n
            res.append(parts)
        return res
    finally:
        oracle.set_rotator_mode(0)


@pytest.fixture(scope="module")
def c_oracle(oracle, c_input):
    cfgs = [(o, r, 0.8 * r) for o, r in zip(_c_offsets(), C_RATES)]
    return cfgs, _oracle_raw(oracle, c_input, FS_C, SCHED_C, cfgs)


def _gate_vfo(parts_gpu, parts_ref):
    """count, rel_rms, fitted complex gain and edge-against-interior for one VFO"""
    assert [p.size for p in parts_gpu] == [p.size for p in parts_ref]
    y = np.concatenate(parts_gpu).astype(np.complex128)
    yo = np.concatenate(parts_ref).astype(np.complex128)
    e_rms = rel_rms(y, yo)
    g = np.vdot(yo, y) / np.vdot(yo, yo)
    e = np.abs(y - yo) / np.sqrt(np.mean(np.abs(yo) ** 2))
    edge = np.zeros(y.size, bool)
    for b in np.cumsum([0] + [p.size for p in parts_ref[:-1]]):
        edge[max(0, b - EDGE): b + EDGE] = True
    assert edge.any() and (~edge).sum() >= 1000
    p999 = float(np.percentile(e[~edge], 99.9))
    ratio = float(e[edge].max() / p999) if p999 > 0 else (0.0 if e[edge].max() == 0 else np.inf)
    return {"rel_rms": e_rms, "gain_re": float(g.real), "gain_im": float(g.imag), "abs_g_minus_1": float(abs(g - 1)),
            "edge_over_p999": ratio, "outputs": int(y.size)}


def _check(res):
    assert res["rel_rms"] < 1e-5, res
    assert res["abs_g_minus_1"] < 2e-6, res
    assert res["edge_over_p999"] <= 4.0, res


@pytest.mark.gpu
@pytest.mark.parametrize("opts", C_OPTIONS, ids=lambda o: "_".join("%s%d" % kv for kv in sorted(o.items())) or "default")
def test_raw_vfos_in_front_end_vs_exact_phase_oracle(sb, c_input, c_oracle, report, opts):
    cfgs, ref = c_oracle
    fe = sb.FrontEnd(FS_C, max(SCHED_C))
    for k, v in opts.items():
        fe.set_option(k, v)
    ids = [fe.add_vfo(sb.VfoConfig.raw(o, r, bw)) for (o, r, bw) in cfgs]
    got = {vid: [] for vid in ids}
    pos = 0
    for n in SCHED_C:
        outs, _ = fe.process(c_input[pos:pos + n])
        for vid in ids:
            got[vid].append(outs[vid])
        pos += n
    hits = fe.stat("graph_hits")
    fe.close()
    res = [_gate_vfo(got[vid], ref[k]) for k, vid in enumerate(ids)]
    tag = "_".join("%s%d" % kv for kv in sorted(opts.items())) or "default"
    report["chain_f64_in_situ_2p4msps_" + tag] = {"per_vfo": res, "graph_hits": int(hits),
                                                  "max_abs_g_minus_1": max(r["abs_g_minus_1"] for r in res),
                                                  "max_edge_over_p999": max(r["edge_over_p999"] for r in res),
                                                  "max_rel_rms": max(r["rel_rms"] for r in res)}
    for r, c in zip(res, cfgs):
        _check(dict(r, vfo=c))
    if not opts:
        assert hits > 0


@pytest.mark.gpu
def test_raw_vfos_behind_tma_stage1_100msps(sb, oracle, report):
    """8 VFOs on the 5 MHz grid at 100 MS/s: (4,27) and (2,69) in registers behind the TMA filter-bank stage 1, then 16/25"""
    n = sum(SCHED_G)
    x = noise_iq(n, 4243, 0.5)
    cfgs = [(o, 250e3, 200e3) for o in OFFS_G]
    ref = _oracle_raw(oracle, x, FS_G, SCHED_G, cfgs)
    fe = sb.FrontEnd(FS_G, max(SCHED_G))
    ids = [fe.add_vfo(sb.VfoConfig.raw(o, r, bw)) for (o, r, bw) in cfgs]
    got = {vid: [] for vid in ids}
    pos = 0
    for c in SCHED_G:
        outs, _ = fe.process(x[pos:pos + c])
        for vid in ids:
            got[vid].append(outs[vid])
        pos += c
    fe.close()
    res = [_gate_vfo(got[vid], ref[k]) for k, vid in enumerate(ids)]
    report["chain_f64_in_situ_100msps"] = {"per_vfo": res, "max_abs_g_minus_1": max(r["abs_g_minus_1"] for r in res),
                                           "max_edge_over_p999": max(r["edge_over_p999"] for r in res)}
    for r, c in zip(res, cfgs):
        _check(dict(r, vfo=c))

"""float64 references of the FIR stages, the polyphase resampler and stage 1, their chunk bookkeeping, and the per-VFO gate
shared by the sample-by-sample kernel tests (test_gpu_chain_f64.py, test_gpu_stage1_f64.py, test_gpu_fm_audio_f64.py)."""
import math

import numpy as np
from scipy.signal import oaconvolve

from util import rel_rms

U = 2.0 ** -24                      # unit round-off of fp32
REF_FLOOR = 2.0 ** -40              # float64 FFT convolution error, relative to sum|h| max|x|: far below any fp32 rounding
EDGE = 64                           # outputs either side of a chunk boundary that count as "edge" in _gate_vfo
MAX_CHUNK = 1000000                 # a stand-alone block's chunk limit (STREAM_BUFFER_SIZE)
TWO64 = 1 << 64
_KTWOPI = np.longdouble("6.283185307179586476925286766559")

# ---------------------------------------------------------------------------------------------- routing (mirrors the library)
DFR_R = {(4, 27): 8, (2, 69): 4, (2, 12): 8, (8, 54): 4, (8, 44): 4, (8, 36): 4}   # outputs per thread (dfir_reg.cuh:107-112)
DFR_MAXT = 72                                                                     # kernels.cuh: DfrParams.taps
POLY_REG = {(16, 25), (5, 6), (2, 3), (4, 5), (2, 5)}                             # tails_reg.cuh:138-140
TS_TILE = 256                                                                     # k_fir_reg / k_firr_reg outputs per CTA
PFB_CASES = {(5, 5), (6, 5), (4, 5), (3, 7), (2, 7)}  # kernels.cu: PFB_CASE (log2 D, QC)


def routes_dfir_reg(D, T):
    """engine.cpp:1273-1277 (dfr_ok) with dfir_reg.cuh:100-102"""
    return D > 1 and T <= DFR_MAXT and (D, T) in DFR_R


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


# ---------------------------------------------------------------------------------------------- polyphase resampler
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


# ---------------------------------------------------------------------------------------------- stage 1 (test_gpu_stage1_f64.py's docstring derives its bound)
def w_u64(offset_hz, fs):
    """XdStage::set_offset_rad(hz_to_rads(-offset, fs)): angle of the fp32-rounded phasor, in turns * 2^64"""
    rad = 2.0 * math.pi * (-offset_hz / fs)
    dre, dim = np.float32(math.cos(rad)), np.float32(math.sin(rad))
    turns = np.arctan2(np.longdouble(dim), np.longdouble(dre)) / _KTWOPI
    scaled = turns * np.longdouble(18446744073709551616.0)
    lim = np.longdouble(9223372036854775807.0)
    scaled = min(max(scaled, -lim), lim)
    return int(np.round(scaled)) % TWO64


def _signed(r):
    r %= TWO64
    return r - TWO64 if r >= (1 << 63) else r


def pfb_detect(ws, T):
    """Scheduler::run: smallest P <= 10 with e^{j w P} within 8e-6 rad over the window of the same sign +-1 for every job,
    mapped to the kernel's PS = 8 / 10 instantiation.  Returns (PS, sigma), (0, 1) when no filter-bank form applies."""
    for P in range(1, 11):
        tol = (8e-6 / 6.283185307179586) * P / T * 18446744073709551616.0
        sg, ok = 0, True
        for w in ws:
            r = (w * P) % TWO64
            d0, d1 = float(_signed(r)), float(_signed(r - (1 << 63)))
            sv = 1 if abs(d0) <= tol else (-1 if abs(d1) <= tol else 0)
            if sv == 0 or (sg != 0 and sv != sg):
                ok = False
                break
            sg = sv
        if not ok:
            continue
        for PS in (8, 10):
            if PS % P == 0:
                return PS, (-1 if (sg < 0 and (PS // P) & 1) else 1)
    return 0, 1


def pfb_eps(w, PS, sigma):
    """signed distance (rad) of w PS from 0 (sigma = +1) or 1/2 turn (sigma = -1), from the exact u64 w"""
    r = (w * PS) % TWO64
    return _signed(r if sigma > 0 else r - (1 << 63)) * (2.0 * math.pi / TWO64)


def plan_of(oracle, ratio):
    if ratio == 1:
        return [(1, np.ones(1, np.float32))]
    return [(D, np.asarray(oracle.decim_taps(ratio, k), np.float32)) for k, (D, T) in enumerate(oracle.decim_plan(ratio))]


def rotate_f64(x, sched, offs, fs):
    """the exact-phase translator: x (complex128, integer chunks already scaled) rotated by the u64 phase of each sample,
    offs[c] the VFO offset chunk c was translated with"""
    n = x.size
    ph = np.empty(n, np.uint64)
    phase, pos = 0, 0
    for c, off in zip(sched, offs):
        w = w_u64(off, fs)
        ph[pos:pos + c] = np.uint64(phase) + np.uint64(w) * np.arange(c, dtype=np.uint64)
        phase = (phase + w * c) % TWO64
        pos += c
    ang = (ph >> np.uint64(11)).astype(np.float64) * (2.0 * math.pi / 2.0 ** 53)
    return x * np.exp(1j * ang)


def drift_weights(T, PS):
    """|floor(k / PS) - floor(T / (2 PS))|: how far tap k's drift is from the centred correction"""
    k = np.arange(T)
    return np.abs(k // PS - T // (2 * PS)).astype(np.float64)


def stage1_f64(x, sched, offs, h, D, fs, eps=0.0, PS=0):
    """exact-phase translator + DecimatingFIR from zero history (the specification form), with the per-component bound of
    the module docstring; eps / PS: the largest filter-bank drift a chunk may carry (0: complex-tap builds only)"""
    T = h.size
    z = rotate_f64(x, sched, offs, fs)
    hh = np.asarray(h, np.float64)
    y = _corr(_hist(z, T - 1), hh)[::D]
    ax = _hist(np.abs(x), T - 1)
    A = math.sqrt(2.0) * _corr(ax, np.abs(hh))[::D]
    b = (4 * T + 4 * PS + 40) * U * A + REF_FLOOR * np.abs(hh).sum() * 2.0 * float(np.abs(x).max(initial=0.0))
    if PS:
        b = b + math.sqrt(2.0) * abs(eps) * _corr(ax, np.abs(hh) * drift_weights(T, PS))[::D]
    return y, b

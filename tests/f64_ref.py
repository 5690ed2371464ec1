"""float64 references of the FIR stages, the polyphase resampler and stage 1, the FM discriminator, the audio chain, the
stereo branch of BroadcastFM and PowerSquelch, their chunk bookkeeping, and the per-VFO gate shared by the sample-by-sample
kernel tests (test_gpu_chain_f64.py, test_gpu_stage1_f64.py, test_gpu_fm_audio_f64.py, test_gpu_stereo_squelch_f64.py).

Stereo branch (stereo_f64; kernels k_st_pilot, k_st_pll, k_st_mix, then the 15 kHz low-pass over l + j r).  Input: the
discriminator output q64 with its per-sample bound e_q (quad_f64's carried bound).  Per term:
  * pilot: p = sum_k h_k m[i + k] over [T-1 zeros | m], h = the library's taps::bandPass<complex_t>(18750, 19250, 3000, fs,
    odd) (b200_taps_bandpass, bit-identical to the oracle's), re and im each T sequential fmaf: fir_f64 on h.real / h.imag;
  * angle: the fp32 p lies within b_p = hypot(b_re, b_im) of p64, so its angle is within asin(b_p / |p64|) (pi when that
    reaches 1), plus 3 ulp of atan2f; where that disk reaches the negative real axis atan2f may return the angle 2 pi away,
    which the err wrap turns into 2 pi - 2P: added there;
  * PLL: the recurrence of pll.h with the library's fp32 constants taken as exact numbers (alpha, beta of
    PhaseControlLoop<float>::criticallyDamped in float steps for bandwidth 25000 / fs, P = FL_M_PI_REF, step 2P, f0, fmin, fmax
    = fl32(hz_to_rads(19000 / 18750 / 19250, fs))), from (theta, f) = (0, f0), vco = e^{j theta} before the update.  The phase
    detector is exactly linear (err = angle - theta, wrapped), so between two trajectories (dtheta, df) follows
        df'     = c (df + beta (da - dtheta)) + e_f
        dtheta' = dtheta + df' + alpha (da - dtheta) + e_theta
    where c = 1 while the float64 frequency is inside [fmin, fmax] and c = 0 while it is clamped (both trajectories then hold
    the same fp32 limit).  The clamp is active in every pull-in: the very first pilot angle is already further from theta = 0
    than (fmax - f0) / beta.  A step whose raw float64 frequency lies within its own bound of a limit would make c unknown:
    the reference counts such steps ("ambiguous clamps"); the tests assert there are none.  Per-step inputs: da = the angle
    term above plus u (|a| + |theta|) (the err subtraction) and u P where err may be wrapped; e_f = u (|beta err| + |f'|);
    e_theta = u (|alpha err| + |f' + alpha err| + |theta'|) plus u P where theta may be wrapped (either side).  While the
    clamp is ever active the perturbation is carried exactly as generators (one column per input, pruned below 2^-60); after the last clamped step the
    system is time-invariant, A = [[1 - alpha - beta, 1], [-beta, 1]], and the bound is the convolution of the inputs with the
    |impulse responses| of A (computed until they fall below 2^-60).  The difference equations are exact, not a
    linearisation: the roundings are taken on the float64 values, and the same roundings of the perturbed values differ by
    at most u times the perturbation, which the factor 1 + 2^-10 covers.  Where ||a - theta| - P| lies within the
    perturbation the two trajectories may wrap err 2P apart ("ambiguous err wraps"): such a step takes an input of 2P.
    After the first ambiguous wrap or clamp the vco angle bound is pi (always true, so "vacuous"): the stand-alone
    blocks never get there; inside the front end stage 1's a-priori bound makes the pilot angle bound wide enough that they
    do, early in the pull-in.  The gain and edge gates leave out the pull-in (up to the last clamped step plus the length
    of A's impulse response) and the outputs that ill-conditioned discriminator samples reach;
  * vco: the angle bound, plus |2P - 2 pi| where theta lies within its bound of +-P (one trajectory wrapped, the other not),
    capped at pi; sincosf adds 2 ulp per component;
  * mix: md = q[i - delay] (0 before the stream start), delay = (T - 1) / 2 + 1; lmr = 2 Re(md conj(vco)^2), l = md + lmr,
    r = md - lmr in k_st_mix's statement order: |lmr - lmr64| <= 2 (e_md (1 + 4 eps) + |md| (2 dv + 4 eps) + 3.1 u (|md| +
    e_md) (1 + 4 eps)) with eps = 2^-22 the sincosf error, and l, r add e_md + e_lmr + u |l|;
  * low-pass (lowPass on): fir_f64 with the 15 kHz / 4 kHz taps on l + j r.

PowerSquelch (squelch_f64; kernels k_sq_sum, k_sq_gate).  The decision is 10 log10(mean |y|) >= (float)level per chunk, the
mean in float64.  launch_squelch sizes nparts = clamp(ceil(max_n / 4096), 1, 256) from the batch's longest chunk, so each
thread sums m = ceil(n / (nparts 256)) terms; the reference takes nparts from the chunk itself, the larger m.  Relative bound of the fp32 mean, over the sum S of |y|: the input bound
sqrt(2) sum e_y (absolute), |x| (two products, a sum, a square root: 3u), the thread's run (m u), the 5-level shuffle tree (5u),
the 8 warp sums (8u), (float)tot (u), (float)n (u when n > 2^24), the division (u).  In dB: 10 / ln 10 times the relative
bound, plus 2 ulp of log10f (times 10) and the rounding of the product.  A chunk is ambiguous where its float64 margin is
within that bound; a closed chunk is exact zeros."""
import math

import numpy as np
from scipy.signal import lfilter, oaconvolve

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


# ---------------------------------------------------------------------------------------------- discriminator and audio chain
# (test_gpu_fm_audio_f64.py's docstring derives their bounds)
P32 = float(np.float32(3.1415926535))          # FL_M_PI_REF (kernels.cu, oracle/sdrpp_oracle.c FL_M_PI)
TWO_P = 2.0 * P32                              # 2.0f * FL_M_PI_REF, exact
ATAN2_ULP = 3


def ulp32(v):
    """fp32 ulp of a value of magnitude up to v (a hair above v, so a result that rounds up to the next binade is covered)"""
    v = np.maximum(np.asarray(v, np.float64) * (1.0 + 2.0 ** -20), 2.0 ** -126)
    return np.exp2(np.floor(np.log2(v)) - 23.0)


def inv_dev_of(dev, sr):
    """QuadStage::configure / quad_init: (float)(1.0 / hz_to_rads(dev, sr))"""
    return float(np.float32(1.0 / (2.0 * math.pi * (dev / sr))))


def quad_f64(z, b, inv_dev, angles32=False):
    """discriminator reference and bound (module docstring).  z: IQ (float64 or exact fp32), b: per-component bound of the
    input (None = exact).  angles32: take the angles as fp32 atan2f values (the bit-level known answers of the reference).
    Returns (q64, bound, ambiguous mask, q64 of the other wrap branch, bound to carry into the next stage)."""
    z = np.asarray(z)
    if angles32:
        th = np.arctan2(z.imag.astype(np.float32), z.real.astype(np.float32)).astype(np.float64)
    else:
        z = z.astype(np.complex128)
        th = np.arctan2(z.imag, z.real)
    prev = np.concatenate([[0.0], th[:-1]])
    raw = th - prev
    d = raw.copy()
    d[raw > P32] -= TWO_P
    d[raw <= -P32] += TWO_P
    q = d * inv_dev
    if b is None:
        cond = np.zeros(th.size)
    else:
        r = math.sqrt(2.0) * np.asarray(b, np.float64) / np.maximum(np.abs(z), 1e-300)
        cond = np.where(r < 1.0, np.arcsin(np.minimum(r, 1.0)), np.pi)
    A = cond + ATAN2_ULP * ulp32(np.abs(th) + cond)
    flip = (cond > 0) & (np.pi - np.abs(th) <= A)
    Ap = np.concatenate([[0.0], A[:-1]])
    flipp = np.concatenate([[False], flip[:-1]])
    E = A + Ap + U * (np.abs(th) + np.abs(prev) + A + Ap)
    E = E + (flip.astype(np.float64) + flipp) * 2.0 * (P32 - np.pi)
    E = E + np.where(np.abs(raw) + E >= P32, U * P32, 0.0)
    cap = 2.0 * P32 * inv_dev * (1.0 + 2.0 * U)
    bq = np.minimum(inv_dev * (E + U * (np.abs(d) + E)), cap)
    amb = np.abs(np.abs(d) - P32) <= E
    alt = (d - np.sign(d) * TWO_P) * inv_dev
    return q, bq, amb, alt, np.where(amb, cap, bq)


def quad_ratio(q, q64, bq, amb, alt):
    q = np.asarray(q, np.float64)
    err = np.abs(q - q64)
    err = np.where(amb, np.minimum(err, np.abs(q - alt)), err)
    return err / bq


def deemph_coefs(tau, sr):
    dt = np.float32(1.0 / sr)
    a = np.float32(float(dt) / (tau + float(dt)))
    return float(a), float(np.float32(np.float32(1.0) - a))


def deemph_f64(x, e, a, b, y0=0.0, e0=0.0):
    """y = a x + b y[-1] per component from state y0 (complex l + j r), with the recursion bound of the module docstring"""
    x = np.asarray(x, np.complex128)
    e = np.zeros(x.size) if e is None else np.asarray(e, np.float64)
    y = lfilter([a], [1.0, -b], x, zi=np.array([b * y0], np.complex128))[0]
    ax = np.maximum(np.abs(x.real), np.abs(x.imag))
    yp = np.concatenate([[y0], y[:-1]])
    ayp = np.maximum(np.abs(yp.real), np.abs(yp.imag))
    f = a * (1 + 3 * U) * e + 3 * U * (a * ax + b * ayp)
    beta = b * (1 + 3 * U)
    eb = lfilter([1.0], [1.0, -beta], f, zi=np.array([beta * e0]))[0]
    return y, eb + REF_FLOOR * float(np.abs(y).max(initial=0.0))


def volume_f64(x, e, volume, muted):
    g = 0.0 if muted else float(np.float32(np.float32(volume) ** np.float32(2)))
    ax = np.maximum(np.abs(x.real), np.abs(x.imag))
    return x * g, (e * g + U * g * (ax + e)) if g else np.zeros(x.size)


def _ratio_c(y, y64, b):
    """per-component error over the bound (an exact answer with a zero bound, a muted output, counts as 0)"""
    y = np.asarray(y).astype(np.complex128)
    err = np.maximum(np.abs(y.real - y64.real), np.abs(y.imag - y64.imag))
    return np.where(b > 0, err / np.where(b > 0, b, 1.0), np.where(err == 0, 0.0, np.inf))


def _chunk_index(counts):
    """chunk of every output, from per-chunk output counts"""
    return np.repeat(np.arange(len(counts)), counts)


# ---------------------------------------------------------------------------------------------- the radio's VFO, in float64
def audio_lp_taps(oracle, cfg):
    from sdrplusplus_b200 import lib as L
    osr = cfg.out_samplerate
    if not cfg.low_pass:
        return None
    if cfg.demod == L.DEMOD_NFM:
        return oracle.lowpass(cfg.bandwidth / 2.0, cfg.bandwidth / 2.0 * 0.1, osr)       # fm.h:123
    return oracle.lowpass(15000.0, 4000.0, osr)                                           # broadcast_fm.h:45


def quad_dev(cfg):
    from sdrplusplus_b200 import lib as L
    return cfg.bandwidth / 2.0 if cfg.demod == L.DEMOD_NFM else cfg.deviation


def chan_taps(oracle, bw, osr):
    return np.ones(1, np.float32) if bw == osr else oracle.lowpass(bw / 2.0, bw / 2.0 * 0.1, osr)


def vfo_audio_f64(oracle, x, sched, fs, cfgs, info=None):
    """one FM VFO of the front end in float64; cfgs[c] is the configuration chunk c ran with.  Returns (l + j r, bound,
    ambiguous wraps, reach): reach is the part of the bound that comes from ill-conditioned discriminator samples (ambiguous
    wraps and samples at the cap) or the stereo PLL's pull-in, carried through the same stages with |taps|.  A RAW VFO
    returns its IF samples (complex) and a zero reach.  info (a dict) receives the squelch decisions ("squelch") and the stereo branch's counts ("stereo")."""
    from sdrplusplus_b200 import frontend, lib as L
    info = {} if info is None else info
    c0 = cfgs[0]
    osr = c0.out_samplerate
    rp = frontend.resamp_plan(fs, osr)
    pr = rp["predec_ratio"]
    plan = [(D, oracle.decim_taps(pr, k)) for k, (D, T) in enumerate(rp["stages"])]
    D0, h0 = plan[0]
    PS, eps = 0, 0.0
    for o in sorted(set(c.offset for c in cfgs)):
        w = w_u64(o, fs)
        ps, sg = pfb_detect([w], h0.size)
        if ps:
            PS, eps = max(PS, ps), max(eps, abs(pfb_eps(w, ps, sg)))
    y, b = stage1_f64(x, sched, [c.offset for c in cfgs], h0, D0, fs, eps, PS)
    stages = [("fir", D0)]
    for D, h in plan[1:]:
        y, b = fir_f64(y, b, h, D)
        stages.append(("fir", D))
    if rp["ntaps"]:
        y, b = poly_f64(y, b, oracle.resamp_taps(fs, osr), rp["interp"], rp["decim"])
        stages.append(("poly", rp["interp"], rp["decim"]))
    # channel filter, swapped at chunk boundaries; every change passes through the identity, so each stretch of one low-pass
    # starts from cleared history
    ci = _chunk_index(cascade_counts(sched, stages))
    bws = np.array([c.bandwidth for c in cfgs])[ci]
    yc, bc = np.empty_like(y), np.empty_like(b)
    starts = [0] + [i for i in range(1, y.size) if bws[i] != bws[i - 1]] + [y.size]
    for s0, s1 in zip(starts[:-1], starts[1:]):
        if s0 > 0:
            assert bws[s0] == osr or bws[s0 - 1] == osr, "a low-pass -> low-pass change is not modelled here"
        yc[s0:s1], bc[s0:s1] = fir_f64(y[s0:s1], b[s0:s1], chan_taps(oracle, float(bws[s0]), osr), 1)
    if c0.squelch_on:
        # radio IF chain: PowerSquelch between the channel filter and the demodulator, one decision per chunk
        cnt = cascade_counts(sched, stages)
        dec, mar, bd, am = squelch_f64(yc, bc, cnt, [c.squelch_level for c in cfgs])
        info["squelch"] = {"open": dec, "margin_db": mar, "bound_db": bd, "ambiguous": am, "counts": cnt}
        closed = ~dec[_chunk_index(cnt)]
        yc, bc = yc.copy(), bc.copy()
        yc[closed], bc[closed] = 0.0, 0.0
    if c0.demod == L.DEMOD_RAW:
        return yc, bc, 0, np.zeros(yc.size)
    inv = inv_dev_of(quad_dev(c0), osr)
    q, bq, amb, alt, carry = quad_f64(yc, bc, inv)
    t = np.where(amb | (bq >= 2.0 * P32 * inv), carry, 0.0)
    if c0.demod == L.DEMOD_WFM_STEREO:
        y, b, st = stereo_f64(q, carry, osr, c0.low_pass, t)
        t = st.pop("reach")
        info["stereo"] = st
    else:
        h = audio_lp_taps(oracle, c0)
        if h is not None:
            a, ea = fir_f64(q, carry, h, 1)
            t = fir_f64(t, None, np.abs(h), 1)[0]
        else:
            a, ea = q, carry
        y, b = a + 1j * a, ea
    if c0.af_samplerate > 0:
        afs = c0.af_samplerate
        ap = frontend.resamp_plan(osr, afs)
        for k, (D, T) in enumerate(ap["stages"]):
            h = oracle.decim_taps(ap["predec_ratio"], k)
            y, b = fir_f64(y, b, h, D)
            t = fir_f64(t, None, np.abs(h), D)[0]
            stages.append(("fir", D))
        if ap["ntaps"]:
            h = oracle.resamp_taps(osr, afs)
            y, b = poly_f64(y, b, h, ap["interp"], ap["decim"])
            t = poly_f64(t, None, np.abs(h), ap["interp"], ap["decim"])[0]
            stages.append(("poly", ap["interp"], ap["decim"]))
        ci = _chunk_index(cascade_counts(sched, stages))
        hp_on = np.array([c.af_high_pass for c in cfgs], bool)[ci]
        if hp_on.any():
            # a high-pass switched off is skipped and keeps its delay line: it filters the samples of its "on" stretches
            hp = oracle.highpass(300.0, 100.0, afs)
            yh, bh = fir_f64(y[hp_on], b[hp_on], hp, 1)
            y, b, t = y.copy(), b.copy(), t.copy()
            y[hp_on], b[hp_on], t[hp_on] = yh, bh, fir_f64(t[hp_on], None, np.abs(hp), 1)[0]
        taus = np.array([c.af_deemph_tau for c in cfgs])[ci]
        if (taus > 0).any():
            assert (taus > 0).all(), "de-emphasis switched off is not modelled here"
            yo, bo, to = np.empty_like(y), np.empty_like(b), np.empty_like(t)
            y0, e0, t0 = 0.0, 0.0, 0.0
            cut = [0] + [i for i in range(1, y.size) if taus[i] != taus[i - 1]] + [y.size]
            for s0, s1 in zip(cut[:-1], cut[1:]):
                aa, bb = deemph_coefs(float(taus[s0]), afs)
                yo[s0:s1], bo[s0:s1] = deemph_f64(y[s0:s1], b[s0:s1], aa, bb, y0, e0)
                to[s0:s1] = lfilter([aa], [1.0, -bb], t[s0:s1], zi=np.array([bb * t0]))[0]
                if s1 > s0:
                    y0, e0, t0 = yo[s1 - 1], bo[s1 - 1], to[s1 - 1]
            y, b, t = yo, bo, to
    if any(c.af_volume_on for c in cfgs):
        ci = _chunk_index(cascade_counts(sched, stages))
        yv, bv = np.empty_like(y), np.empty_like(b)
        for k, c in enumerate(cfgs):
            sel = ci == k
            if c.af_volume_on:
                yv[sel], bv[sel] = volume_f64(y[sel], b[sel], c.af_volume, c.af_muted)
                t = t.copy()
                t[sel] *= 0.0 if c.af_muted else float(np.float32(np.float32(c.af_volume) ** np.float32(2)))
            else:
                yv[sel], bv[sel] = y[sel], b[sel]
        y, b = yv, bv
    return y, b, int(amb.sum()), t


def vfo_counts(oracle, fs, cfg, sched):
    from sdrplusplus_b200 import frontend
    rp = frontend.resamp_plan(fs, cfg.out_samplerate)
    st = [("fir", D) for D, T in rp["stages"]] + ([("poly", rp["interp"], rp["decim"])] if rp["ntaps"] else [])
    if cfg.af_samplerate > 0:
        ap = frontend.resamp_plan(cfg.out_samplerate, cfg.af_samplerate)
        st += [("fir", D) for D, T in ap["stages"]] + ([("poly", ap["interp"], ap["decim"])] if ap["ntaps"] else [])
    return cascade_counts(sched, st)

def _gate_clean(y, yo, clean, counts, restarts=()):
    """f64_ref._gate_vfo's fitted gain and edge-against-interior ratio over the outputs in `clean`; the stream's first EDGE
    outputs (the start transient, where the partly filled windows give the discriminator small |z|), and the first EDGE
    outputs of each chunk in `restarts` (a filter restarted from cleared history), count as neither edge nor interior"""
    edge = np.zeros(y.size, bool)
    for bnd in np.cumsum(counts[:-1]):
        edge[max(0, bnd - EDGE): bnd + EDGE] = True
    clean = clean.copy()
    clean[:EDGE] = False
    for k in restarts:
        at = int(sum(counts[:k]))
        clean[at: at + EDGE] = False
    assert (edge & clean).any() and (~edge & clean).sum() >= 1000
    yc, oc = y[clean], yo[clean]
    g = float(np.dot(oc, yc) / np.dot(oc, oc))
    e = np.abs(y - yo) / math.sqrt(float(np.mean(oc ** 2)))
    p999 = float(np.percentile(e[~edge & clean], 99.9))
    emax = float(e[edge & clean].max())
    ratio = emax / p999 if p999 > 0 else (0.0 if emax == 0 else np.inf)
    return {"rel_rms": float(np.linalg.norm(yc - oc) / np.linalg.norm(oc)), "gain": g, "abs_g_minus_1": abs(g - 1.0),
            "edge_over_p999": ratio, "outputs": int(y.size), "gated_outputs": int(clean.sum())}


# ---------------------------------------------------------------------------------------------- stereo branch and squelch
ST_PHASE_LIMIT = 1e-3               # a step whose phase bound exceeds this is counted as ill-conditioned
ST_SLACK = 1.0 + 2.0 ** -10         # second-order terms of the linearisation
SINCOS_EPS = 2.0 ** -22             # 2 ulp of sincosf on a component of magnitude <= 1
SQ_TILE, SQ_MAXPARTS = 256 * 16, 256


def pll_constants(fs):
    """StereoStage::configure / the oracle's pll_init + wfm_stereo_create: PhaseControlLoop<float>::criticallyDamped with its
    float locals for bandwidth 25000 / fs, and the float-narrowed 19000 / 18750 / 19250 Hz"""
    f32 = np.float32
    bw = f32(25000.0 / fs)
    damp = f32(math.sqrt(2.0) / 2.0)
    den = f32((1.0 + 2.0 * float(damp) * float(bw)) + float(bw * bw))          # bw * bw is a float product
    alpha = (f32(4) * damp * bw) / den
    beta = (f32(4) * bw * bw) / den

    def rads(hz):
        return float(f32(2.0 * math.pi * (hz / fs)))
    return {"alpha": float(alpha), "beta": float(beta), "f0": rads(19000.0), "fmin": rads(18750.0), "fmax": rads(19250.0)}


def stereo_taps(fs):
    from sdrplusplus_b200 import frontend
    return frontend.taps_bandpass(18750.0, 19250.0, 3000.0, fs, True)


def stereo_delay(T):
    return (T - 1) // 2 + 1


def _lti_responses(alpha, beta):
    """theta and f rows of A^k v for the three input kinds (angle, f rounding, theta rounding), k = 0.. until < 2^-60"""
    A = np.array([[1.0 - alpha - beta, 1.0], [-beta, 1.0]])
    V = np.array([[alpha + beta, 1.0, 1.0], [beta, 1.0, 0.0]])
    out = []
    while np.abs(V).max() >= 2.0 ** -60:
        out.append(V.copy())
        V = A @ V
    return np.array(out)                                   # (K, 2, 3)


def _pll_f64(a, c):
    """the PLL recurrence in float64: per step theta (for vco), err (wrapped), raw err, f (after the clamp), raw f, raw theta"""
    n = a.size
    P, two_p = P32, TWO_P
    al, be, fmin, fmax = c["alpha"], c["beta"], c["fmin"], c["fmax"]
    th, f = 0.0, c["f0"]
    o = np.empty((6, n))
    thl, errl, rawl, fl, frl, trl = ([0.0] * n for _ in range(6))
    al_ = a.tolist()
    for i in range(n):
        thl[i] = th
        raw = al_[i] - th
        err = raw - two_p if raw > P else (raw + two_p if raw <= -P else raw)
        fr = f + be * err
        f = fmax if fr > fmax else (fmin if fr < fmin else fr)
        tr = th + (f + al * err)
        th = tr
        while th > P:
            th -= two_p
        while th < -P:
            th += two_p
        errl[i], rawl[i], fl[i], frl[i], trl[i] = err, raw, f, fr, tr
    for k, v in enumerate((thl, errl, rawl, fl, frl, trl)):
        o[k] = v
    return o


def stereo_f64(q, e_q, fs, lowpass, reach=None):
    """BroadcastFM's stereo branch behind the discriminator (module docstring).  q: float64 discriminator output of the stream,
    e_q its bound, reach: the part of e_q from ill-conditioned discriminator samples (None: none).  Returns (l + j r, bound,
    info): info holds the reach of the output, the counts of ambiguous err wraps, ambiguous clamps and ill steps, the last
    clamped step, and the float64 frequency's smallest distance to a limit over its bound."""
    q = np.asarray(q, np.float64)
    n = q.size
    e_q = np.zeros(n) if e_q is None else np.asarray(e_q, np.float64)
    h = stereo_taps(fs).astype(np.complex128)
    T = h.size
    dl = stereo_delay(T)
    c = pll_constants(fs)
    al, be = c["alpha"], c["beta"]
    pr, br = fir_f64(q, e_q, h.real, 1)
    pi_, bi = fir_f64(q, e_q, h.imag, 1)
    p = pr + 1j * pi_
    bp = np.hypot(br, bi)
    ap = np.abs(p)
    a = np.angle(p)
    ratio = bp / np.maximum(ap, 1e-300)
    cond = np.where(ratio < 1.0, np.arcsin(np.minimum(ratio, 1.0)), np.pi)
    da = cond + ATAN2_ULP * ulp32(np.abs(a) + cond)
    da = da + np.where((cond > 0) & (np.pi - np.abs(a) <= da), 2.0 * np.pi - TWO_P, 0.0)
    th, err, raw, f, fr, tr = _pll_f64(a, c)
    da = da + U * (np.abs(a) + np.abs(th) + da) + np.where(np.abs(raw) > P32 - 0.01, U * P32, 0.0)
    dfr = U * (np.abs(be * err) + np.abs(f)) * (1 + 2.0 ** -20)
    dth = U * (np.abs(al * err) + np.abs(f + al * err) + np.abs(tr)) * (1 + 2.0 ** -20) + np.where(np.abs(tr) > P32 - 0.01, U * P32, 0.0)
    clamped = (fr > c["fmax"]) | (fr < c["fmin"])
    last = int(np.flatnonzero(clamped)[-1]) + 1 if clamped.any() else 0
    Bth = np.zeros(n)                                      # bound of theta as used at step i (before its update)
    Bf = np.zeros(n)                                       # bound of f after step i
    Bfr = np.zeros(n)                                      # bound of the raw f of step i
    amb_wrap = np.zeros(n, bool)
    amb_clamp = np.zeros(n, bool)
    # generators while the clamp is ever active: column = input, rows (theta, f)
    G = np.zeros((2, 0))
    mag = np.zeros(0)
    for i in range(last):
        Bth[i] = ST_SLACK * float(np.abs(G[0]) @ mag)
        pert = da[i] + Bth[i]
        if abs(abs(raw[i]) - P32) <= pert:
            amb_wrap[i] = True
        # raw f = f + beta (a - theta): generators, then the new angle input
        rf = G[1] - be * G[0]
        Bfr[i] = ST_SLACK * (float(np.abs(rf) @ mag) + be * da[i])
        if (abs(fr[i] - c["fmax"]) <= Bfr[i]) or (abs(fr[i] - c["fmin"]) <= Bfr[i]):
            amb_clamp[i] = True
        cc = 0.0 if clamped[i] else 1.0
        f_new = cc * rf
        th_new = G[0] + f_new - al * G[0]
        G = np.concatenate([np.vstack([th_new, f_new]),
                            np.array([[cc * be + al, 1.0, 1.0], [cc * be, 1.0, 0.0]])], axis=1)
        mag = np.concatenate([mag, [da[i] + (TWO_P if amb_wrap[i] else 0.0), dfr[i], dth[i]]])
        Bf[i] = ST_SLACK * float(np.abs(G[1]) @ mag)
        keep = np.abs(G).max(axis=0) >= 2.0 ** -60
        G, mag = G[:, keep], mag[keep]
    R = _lti_responses(al, be)
    A = np.array([[1.0 - al - be, 1.0], [-be, 1.0]])
    if last < n:
        # what the clamped stretch left in the state (G: the state after step last - 1), carried by A^k
        S = G
        for k in range(n - last):
            Bth[last + k] += ST_SLACK * float(np.abs(S[0]) @ mag)
            S = A @ S
            Bf[last + k] += ST_SLACK * float(np.abs(S[1]) @ mag)
            if S.size == 0 or np.abs(S).max() < 2.0 ** -60:
                break
        # inputs from `last` on, through the time-invariant system: the input of step j reaches the state after step j + k
        # through R[k]; theta as used at step i is the state after step i - 1
        ins = np.stack([da, dfr, dth])
        ins[:, :last] = 0.0
        idx = np.arange(last, n)
        Bth0 = Bth.copy()
        for _ in range(4):
            ins_a = ins[0] + np.where(amb_wrap, TWO_P, 0.0)
            ins_a[:last] = 0.0
            th_b, f_b = np.zeros(n), np.zeros(n)
            for j, v in enumerate((ins_a, ins[1], ins[2])):
                th_b += np.convolve(v, np.abs(R[:, 0, j]))[:n]
                f_b += np.convolve(v, np.abs(R[:, 1, j]))[:n]
            Bth = Bth0 + ST_SLACK * np.concatenate([[0.0], th_b[:-1]])
            new_amb = amb_wrap.copy()
            new_amb[idx] |= np.abs(np.abs(raw[idx]) - P32) <= da[idx] + Bth[idx]
            if (new_amb == amb_wrap).all():
                break
            amb_wrap = new_amb
        Bf = Bf + ST_SLACK * f_b
        Bf_prev = np.concatenate([[0.0], Bf[:-1]])
        Bfr[idx] = Bf_prev[idx] + be * (da[idx] + Bth[idx])
        amb_clamp[idx] |= (np.abs(fr[idx] - c["fmax"]) <= Bfr[idx]) | (np.abs(fr[idx] - c["fmin"]) <= Bfr[idx])
    # after the first ambiguous err wrap or clamp the two trajectories may part: from the next step on the vco angle bound is
    # pi, which holds whatever the loop does ("vacuous")
    amb_any = amb_wrap | amb_clamp
    vac_from = int(np.flatnonzero(amb_any)[0]) + 1 if amb_any.any() else n
    ill = (Bth > ST_PHASE_LIMIT) | amb_wrap
    near = (np.abs(th - P32) <= Bth) | (np.abs(th + P32) <= Bth)
    dv = np.minimum(np.pi, Bth + np.where(near, abs(TWO_P - 2.0 * np.pi), 0.0))
    dv[vac_from:] = np.pi
    settled = min(n, last + R.shape[0])
    # mix
    md = np.concatenate([np.zeros(dl), q])[:n]
    e_md = np.concatenate([np.zeros(dl), e_q])[:n]
    lmr = 2.0 * md * np.cos(2.0 * th)
    eps = SINCOS_EPS
    amd = np.abs(md)
    e_lmr = 2.0 * (e_md * (1 + 4 * eps) + amd * (2 * dv + 4 * eps) + 3.1 * U * (amd + e_md) * (1 + 4 * eps))
    l64, r64 = md + lmr, md - lmr
    e_l = e_md + e_lmr + U * (np.abs(l64) + e_md + e_lmr)
    e_r = e_md + e_lmr + U * (np.abs(r64) + e_md + e_lmr)
    y = l64 + 1j * r64
    b = np.maximum(e_l, e_r)
    # reach: outputs of the pull-in (up to the last clamped step plus the length of A's impulse response) and outputs whose
    # bound carries an ill-conditioned discriminator sample (in the pilot window or as md): left out of the gain and edge gates
    dirty = np.zeros(n, bool)
    dirty[:settled] = True
    if reach is not None:
        rp = fir_f64(np.asarray(reach, np.float64), None, np.abs(h), 1)[0]
        dirty |= (rp > 0) | (np.concatenate([np.zeros(dl), reach])[:n] > 0)
    t = np.where(dirty, b, 0.0)
    if lowpass:
        from sdrplusplus_b200 import frontend
        hl = frontend.taps_lowpass(15000.0, 4000.0, fs)
        y, b = fir_f64(y, b, hl, 1)
        t = fir_f64(t, None, np.abs(hl), 1)[0]
    dist = np.minimum(f - c["fmin"], c["fmax"] - f)
    free = ~clamped
    free[:last] = False
    info = {"reach": t, "ambiguous_wraps": int(amb_wrap.sum()), "ambiguous_clamps": int(amb_clamp.sum()),
            "ill_steps": int(ill.sum()), "clamped_steps": int(clamped.sum()), "last_clamped": last - 1,
            "settled_from": settled, "vacuous_from": vac_from,
            "clamp_margin_over_bound": float(np.min(dist[free] / np.maximum(Bf[free], 1e-300))) if free.any() else np.inf,
            "max_phase_bound": float(Bth[~ill].max(initial=0.0)), "delay": dl, "taps": T, "theta": th, "vco_bound": dv}
    return y, b, info


def squelch_nparts(max_n):
    """launch_squelch: CTAs per job from the batch's longest chunk"""
    return min(SQ_MAXPARTS, max(1, (int(max_n) + SQ_TILE - 1) // SQ_TILE))


def squelch_f64(y, e_y, counts, level):
    """PowerSquelch per chunk (module docstring).  y: float64 IQ of the stream, e_y its per-component bound (None = exact),
    counts: samples per chunk, level: dB (scalar or per chunk).  Each thread's run is taken with nparts from the chunk's own
    length: a batch's longer job only raises nparts, which shortens the runs, so this is the larger bound.  Returns (open (float64 decision), margin dB, bound dB, ambiguous)."""
    y = np.asarray(y, np.complex128)
    e_y = np.zeros(y.size) if e_y is None else np.asarray(e_y, np.float64)
    counts = [int(c) for c in counts]
    lev = np.broadcast_to(np.asarray(level, np.float64), (len(counts),))
    dec, mar, bnd, amb = [], [], [], []
    pos = 0
    for c, n in enumerate(counts):
        a = np.abs(y[pos:pos + n])
        S = float(a.sum())
        E = math.sqrt(2.0) * float(e_y[pos:pos + n].sum())
        pos += n
        if n == 0:
            dec.append(False), mar.append(-np.inf), bnd.append(0.0), amb.append(False)
            continue
        m = -(-n // (squelch_nparts(n) * 256))
        rel = (3 + m + 5 + 8 + 1 + 1 + (1 if n > (1 << 24) else 0)) * U
        mean = S / n
        lv = float(np.float32(lev[c]))
        with np.errstate(divide="ignore"):
            db = 10.0 * math.log10(mean) if mean > 0 else -np.inf
        if mean > 0:
            r = rel * (1 + 2 * rel) + E / S + REF_FLOOR
            L = abs(math.log10(mean))
            bd = 10.0 / math.log(10.0) * (r / max(1e-300, 1.0 - r)) + 10.0 * 2.0 * float(ulp32(L)) + float(ulp32(10.0 * L + 20.0 * float(ulp32(L))))
        else:
            bd = np.inf if E > 0 else 0.0
        dec.append(bool(db >= lv))
        mar.append(db - lv)
        bnd.append(bd)
        amb.append(bool(abs(db - lv) <= bd) if np.isfinite(db) else bool(E > 0))
    return np.array(dec), np.array(mar), np.array(bnd), np.array(amb)

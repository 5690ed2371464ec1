"""The spectrum branch (k_fft_single, k_fft_p1 / k_fft_p2, k_fftr_p1 / k_fftr_p2 and the dB epilogue) against a float64
reference, bin by bin, on every line from line 0.

Reference.  A line's frame is nz samples of the stream taken as exact values (cf32 as is, integer samples times the fp32
ingest scale of their chunk, in float64), times the plan's fp32 window including its (-1)^n sign (frontend.window, which
test_abi.py pins to the oracle bit for bit), zero-padded to N and transformed by np.fft.fft in float64: X_k, from the
windowed samples y_n.

A-priori per-bin bound.  With L = log2 N and u = 2^-24:
    |X^_k - X_k| <= B_k = (eta (L + 1) + c0) u sum_n |y_n|,   eta = 8,  c0 = 1 (+1 for a scale that is not a power of two)
  * One radix-2 level: an output node is fl(a + b) or fl(fl(a - b) * w^).  The add or subtract rounds each component once:
    u |a +- b|.  The twiddle w^ differs from w by at most u (the fp32 `tw` and `tw_fine` tables, rounded from double; the
    FR_COS / FR_SIN constants, printed to 10 digits, 1.01 u), and the complex product rounds by at most 3 u |p| (cmulf with
    or without fma, fr_mul_w's fmaf form, and the RSQRT2 forms: one add and one multiply per component).  That is 5 u.  The
    radix-8 passes of fft_dif_smem rotate by W8^i (mul_w8_1 / mul_w8_3: 3 u) before the table twiddle of the same level,
    8 u in all.  eta = 8 covers every level of every build.
  * One more level for the four-step twiddle between the passes: coarse * fine (u each, 3 u for their product) times the
    data (3 u) is 8 u in k_fftr_p1; sincospif in k_fft_p1 (1 ulp per component on an exact argument, 2 u) times the data,
    5 u.  The single-pass build has no such level; the bound keeps the term.
  * An error made at a node reaches each output through unit-modulus twiddles, and at every level the nodes that feed one
    output partition the inputs, so a level adds at most eta u sum |y| to any bin.
  * c0: the window product x * w rounds once (u |y|); an integer sample times a scale that is not a power of two rounds once
    more.
  * Second-order terms (intermediate values grown by (1 + eta u)^L) are covered by a factor 1 + 2 (eta (L + 1) + c0) u.
Nothing here is fitted to a run.

The dB step.  power_db computes m2 = (x^2 + y^2) nf (2 u relative; nf = 1 / N^2 is exact), log2f (1 ulp: 2 u |l|) and
l * 3.0103f (the product and the rounded constant, u each).  So a line value is within delta = (9 + 5 |dB|) u dB of
10 log10(|X^ / N|^2), and the gate per bin is the interval
    20 log10(max(|X| - B, 0) / N) - delta  <=  line[k]  <=  20 log10((|X| + B) / N) + delta,
the magnitudes bounded by the reverse triangle inequality.  Below -370 dB the fp32 power may be subnormal or zero: the
lower end drops to -460 dB (under log2 of the smallest subnormal), the upper end takes the absolute rounding of subnormal
products (2^-148 on the power), and the clamp value -127 * 3.0103f of a power that underflowed to zero is admitted.

Gates, on every line: every bin inside its interval; norm-wise ||  |X^| - |X|  ||_2 <= (eta (L + 1) + c0) u sqrt(N) ||y||_2
(Higham's bound for the same network: each level is sqrt(2) times a unitary map, so the local errors of a level, at most
eta u times its output, reach the output at most eta u sqrt(N) ||y||_2 in norm) plus the dB rounding; the gain
sum |X^|^2 / sum |X|^2 within the square of that bound of 1.  Known answers where the bound is tight: an all-zero frame gives
the clamp value bit for bit, an impulse a flat line, an impulse pair the cosine pattern (which carries the relative sign of
two window values), and a rectangular-window tone on an exact bin its peak on that bin.  b200_fft_raw gets the same bound on
the complex value.
"""
import math

import numpy as np
import pytest

from f64_ref import U
from util import fm_carrier, noise_iq

ETA = 8.0
CF32, CS16, CS8 = 0, 1, 2
MAX_GRID_Y = 65535                                   # kernels.cu: FFT_MAX_GRID_Y
CLAMP_DB = np.float32(-127.0) * np.float32(3.01029995663981209120)
SUBNORMAL_DB = -460.0                                # below 10 log10(2^-149)
SUBNORMAL_EDGE = -370.0


# ---------------------------------------------------------------------------------------------- mirrors of the host code
def fft_plan(N):
    """FftCore::create: (logN, logN1, logN2); single pass up to 8192 points"""
    L = N.bit_length() - 1
    if N <= 8192:
        return L, L, 0
    return L, (L + 1) // 2, L - (L + 1) // 2


def reg_pair(logn):
    """(RA, RB) of a register pass of length 2^logn (launch_fft_fmt's FR_P1 / FR_P2, FftCore::create's window_p)"""
    return {8: (16, 16), 9: (16, 32), 10: (32, 32)}[logn]


def uses_reg(N):
    """fft_plan_uses_reg"""
    _, l1, l2 = fft_plan(N)
    return l2 > 0 and 8 <= l1 <= 10 and 8 <= l2 <= 10


def fft_build(N, fft=1, cta=8, raw=False, tables=True):
    """launch_fft_fmt's kernel selection: "single", "smem" (k_fft_p1 / k_fft_p2) or
    "reg<RA>x<RB>/<RA>x<RB>_c<cta>_<tab|gl>" (k_fftr_p1 / k_fftr_p2 with their template arguments)"""
    _, l1, l2 = fft_plan(N)
    if l2 == 0:
        return "single"
    if fft >= 1 and not raw and uses_reg(N):
        (a1, b1), (a2, b2) = reg_pair(l1), reg_pair(l2)
        return "reg%dx%d/%dx%d_c%d_%s" % (a1, b1, a2, b2, 4 if cta == 4 else 8, "tab" if tables else "gl")
    return "smem"


def fft_launches(N, nb):
    """launches of one launch_fft_frames call over nb frames"""
    return 0 if nb <= 0 else -(-nb // MAX_GRID_Y) * (1 if fft_plan(N)[2] == 0 else 2)


def fe_fft_launches(N, nz, interval, fft_v, chunks, fstart=0, pos=0, frame_fmt=CF32, frame_scale=0.0):
    """fe_fft_chunk: the spectrum branch's launches per chunk (conversions and transforms; copies are not launches).
    chunks: [(count, fmt, ingest scale as fp32, 0 for cf32)].  Returns (launches per chunk, framing state)."""
    out = []
    for count, fmt, isc in chunks:
        end, n = pos + count, 0
        pending = fstart < pos
        same = frame_fmt == fmt and (fmt == CF32 or frame_scale == isc)
        if pending and (not fft_v or not same) and frame_fmt != CF32:
            n += 1
            frame_fmt, frame_scale = CF32, 0.0
        if pending and (not fft_v or not same):
            if min(fstart + nz, end) > pos:
                n += 1
            if fstart + nz <= end:
                n += fft_launches(N, 1)
                fstart += interval
        if fstart + nz <= end:
            nb = (end - fstart - nz) // interval + 1
            n += fft_launches(N, nb)
            fstart += interval * nb
        if pos <= fstart < end:
            if fft_v:
                frame_fmt, frame_scale = fmt, isc
            else:
                n += 1
                frame_fmt, frame_scale = CF32, 0.0
        out.append(n)
        pos = end
    return out, (fstart, pos, frame_fmt, frame_scale)


# ---------------------------------------------------------------------------------------------- float64 reference and gates
def bound_coef(N, c0):
    L = N.bit_length() - 1
    k = (ETA * (L + 1) + c0) * U
    return k * (1.0 + 2.0 * k)


def window64(win, nz):
    from sdrplusplus_b200 import frontend
    return frontend.window(win, nz).astype(np.float64)


def _db_slack(d):
    return (9.0 + 5.0 * np.abs(d)) * U


def db_interval(A, B, N):
    """per-bin interval of a dB line value, |X| = A, bound B"""
    with np.errstate(divide="ignore"):
        lo = 20.0 * np.log10(np.maximum(A - B, 0.0) / N)
    # + 2^-148: the squares and the product with nf round to subnormals with an absolute error of 2^-150 each
    hi = 10.0 * np.log10((A + B) ** 2 / (float(N) * N) + 2.0 ** -148)
    lo = lo - _db_slack(np.maximum(lo, SUBNORMAL_DB))
    hi = hi + _db_slack(hi)
    lo = np.where(lo < SUBNORMAL_EDGE, SUBNORMAL_DB, lo)
    return lo, hi


def db_inside(line, lo, hi):
    """line within [lo, hi], or the clamp value of a power that may have underflowed to zero"""
    return ((line >= lo) & (line <= hi)) | ((lo <= SUBNORMAL_DB) & (line == np.float64(CLAMP_DB)))


class Stats:
    """worst figures over the lines of one case"""

    def __init__(self):
        self.frac, self.norm, self.gain, self.lines = 0.0, 0.0, 0.0, 0

    def add(self, frac, norm, gain):
        self.frac, self.norm, self.gain = max(self.frac, frac), max(self.norm, norm), max(self.gain, gain)
        self.lines += 1

    def row(self):
        return {"bound_used": self.frac, "norm_ratio": self.norm, "gain_minus_1": self.gain, "lines": self.lines}


def _check_line(line, X, S, N, c0, st, what):
    """one dB line against X (complex128, N bins); S = sum |y|"""
    coef = bound_coef(N, c0)
    B = coef * S
    A = np.abs(X)
    lo, hi = db_interval(A, B, N)
    line = np.asarray(line, np.float64)
    bad = np.flatnonzero(~db_inside(line, lo, hi))
    assert bad.size == 0, "%s: %d bins outside their interval, first k=%d: %r not in [%r, %r] (|X|/N %r)" % (
        what, bad.size, bad[0], line[bad[0]], lo[bad[0]], hi[bad[0]], A[bad[0]] / N)
    Ah = N * 10.0 ** (line / 20.0)
    slack = _db_slack(np.maximum(np.abs(lo), np.abs(hi))) * (math.log(10.0) / 20.0) * 1.01
    live = (lo > SUBNORMAL_DB) & (hi > SUBNORMAL_EDGE)          # the used fraction over normal fp32 powers
    frac = float(np.max(np.abs(Ah - A)[live] / (B + slack * (A + B))[live], initial=0.0))
    nX = float(np.linalg.norm(A))
    tol_n = coef * nX + float(np.linalg.norm(slack * (A + B)))
    err_n = float(np.linalg.norm(Ah - A))
    assert err_n <= tol_n, "%s: norm-wise %r > %r" % (what, err_n, tol_n)
    g = float(np.sum(Ah ** 2) / np.sum(A ** 2)) if nX > 0 else 1.0
    e = tol_n / nX if nX > 0 else 0.0
    assert abs(g - 1.0) <= (1.0 + e) ** 2 - 1.0, "%s: gain %r" % (what, g)
    st.add(frac, err_n / tol_n if tol_n > 0 else 0.0, abs(g - 1.0))


def _check_raw(raw, X, S, N, c0, st, what):
    coef = bound_coef(N, c0)
    B = coef * S
    d = np.abs(np.asarray(raw, np.complex128) - X)
    bad = np.flatnonzero(d > B)
    assert bad.size == 0, "%s: %d bins beyond the bound, first k=%d: %r > %r" % (what, bad.size, bad[0], d[bad[0]], B)
    nX = float(np.linalg.norm(X))
    err_n = float(np.linalg.norm(d))
    assert err_n <= coef * nX, "%s: norm-wise %r > %r" % (what, err_n, coef * nX)
    g = float(np.sum(np.abs(raw.astype(np.complex128)) ** 2) / np.sum(np.abs(X) ** 2)) if nX > 0 else 1.0
    assert abs(g - 1.0) <= (1.0 + coef) ** 2 - 1.0, "%s: gain %r" % (what, g)
    st.add(float(d.max() / B) if B > 0 else 0.0, err_n / (coef * nX) if nX > 0 else 0.0, abs(g - 1.0))


def check_lines(lines, Y, N, c0, st, what, raw=False):
    """lines (F, N) against the float64 transforms of the windowed frames Y (F, nz), every bin"""
    F = Y.shape[0]
    assert lines.shape == (F, N), (what, lines.shape, (F, N))
    step = max(1, (1 << 22) // N)
    for f0 in range(0, F, step):
        X = np.fft.fft(Y[f0:f0 + step], n=N, axis=1)
        S = np.abs(Y[f0:f0 + step]).sum(axis=1)
        for i in range(X.shape[0]):
            chk = _check_raw if raw else _check_line
            chk(lines[f0 + i], X[i], S[i], N, c0, st, "%s line %d" % (what, f0 + i))


def check_flat(lines, amp, N, c0, st, what):
    """one impulse of windowed value magnitude amp[f] per frame: every bin of line f within the interval of |X_k| = amp[f]"""
    amp = np.asarray(amp, np.float64)
    B = bound_coef(N, c0) * amp
    lo, hi = db_interval(amp, B, N)
    mn, mx = lines.min(axis=1).astype(np.float64), lines.max(axis=1).astype(np.float64)
    bad = np.flatnonzero(~(db_inside(mn, lo, hi) & db_inside(mx, lo, hi)))
    assert bad.size == 0, "%s: frame %d: [%r, %r] not in [%r, %r]" % (what, bad[0], mn[bad[0]], mx[bad[0]], lo[bad[0]], hi[bad[0]])
    lin = N * 10.0 ** (np.stack([mn, mx], 1) / 20.0)
    live = (lo > SUBNORMAL_DB) & (hi > SUBNORMAL_EDGE)
    if live.any():
        st.add(float(np.max(np.abs(lin - amp[:, None])[live] / B[live, None])), 0.0, 0.0)


# ---------------------------------------------------------------------------------------------- inputs
def stream_f64(parts):
    """[(samples, fmt, scale)] -> the stream's exact values (complex128)"""
    out = []
    for x, fmt, sc in parts:
        if fmt == CF32:
            out.append(np.asarray(x, np.complex64).astype(np.complex128))
        else:
            v = np.asarray(x).reshape(-1, 2).astype(np.float64) * float(np.float32(sc))
            out.append(v[:, 0] + 1j * v[:, 1])
    return np.concatenate(out) if out else np.empty(0, np.complex128)


def frames_of(x, fstart, nz, interval, count):
    idx = fstart + np.arange(count, dtype=np.int64)[:, None] * interval + np.arange(nz, dtype=np.int64)[None, :]
    return x[idx]


def gen_chunk(rng, n, fmt, amp=0.3):
    if fmt == CF32:
        return (rng.uniform(-amp, amp, 2 * n).astype(np.float32)).view(np.complex64)
    if fmt == CS16:
        return rng.integers(-20000, 20000, (n, 2), dtype=np.int16)
    return rng.integers(-120, 120, (n, 2), dtype=np.int8)


def ragged(total, lo, hi, seed):
    rng = np.random.default_rng(seed)
    s = []
    while sum(s) < total:
        s.append(int(rng.integers(lo, hi)))
    return s


def impulse_positions(N, nz, cta):
    """the frame's first and last samples, N - 1, and for the register builds every a and every t of pass 1's
    n = (a RB + t) N2 + n2 at the first and last column of a CTA (columns 0, cta - 1, cta, 2 cta - 1, N2 - 1)"""
    L, l1, l2 = fft_plan(N)
    p = {0, nz - 1, N - 1}
    if uses_reg(N):
        RA, RB = reg_pair(l1)
        N2 = 1 << l2
        cols = [0, cta - 1, cta, 2 * cta - 1, N2 - 1]
        for i in range(max(RA, RB)):
            a, t = i % RA, (7 * i + 3) % RB
            p.add((a * RB + t) * N2 + cols[i % len(cols)])
    elif l2:
        N1, N2 = 1 << l1, 1 << l2
        p |= {N2 - 1, N2, (N1 - 1) * N2, N // 2 + 1}
    return sorted(q for q in p if q < nz)


def tone_bins(N, cta, seed):
    """bins k = r0 + rl + N1 k2 with every residue rl of a pass-2 CTA (and, single pass, spread over the line)"""
    rng = np.random.default_rng(seed)
    L, l1, l2 = fft_plan(N)
    N1 = 1 << l1
    if l2 == 0:
        return sorted({1, N - 1, N // 2} | {int(v) for v in rng.integers(0, N, 5)})
    R = 4 if cta == 4 else 8
    return [int(R * rng.integers(0, N1 // R) + rl + N1 * rng.integers(0, N >> l1)) for rl in range(R)]


# ---------------------------------------------------------------------------------------------- CPU part
@pytest.mark.parametrize("N", [8, 16, 64, 512, 4096, 8192, 16384, 1 << 16, 1 << 17, 1 << 18, 1 << 19, 1 << 20])
def test_reference_and_bound_hold_for_the_oracle(oracle, N):
    """the oracle's fp32 spectrum (its own radix-4 Stockham FFT and VOLK's dB form) sits inside the bound, raw and dB, for
    each window and a padded frame"""
    st = Stats()
    for win, nz in [(0, N), (1, N - 1), (2, max(1, int(0.6 * N)) | 1)]:
        x = noise_iq(nz, N + win, 1.0)
        y = x.astype(np.complex128) * window64(win, nz)
        w32 = np.asarray(oracle.window_buf(win, nz), np.float64)
        assert np.array_equal(w32, window64(win, nz))
        check_lines(oracle.fft_raw(N, nz, win, x)[None, :], y[None, :], N, 1, st, "oracle raw %d" % N, raw=True)
        check_lines(oracle.fft_frame(N, nz, win, x)[None, :], y[None, :], N, 1, st, "oracle dB %d" % N)
    assert st.frac <= 1.0


def test_gates_see_frame_and_window_faults(oracle):
    """what the peak-relative gate lets through fails here: a frame one sample late, the weakest bins 1 dB high, a window
    value of the wrong sign"""
    N, nz = 1 << 16, 1 << 16
    x = noise_iq(nz + 1, 3, 1.0)
    w = window64(2, nz)
    y = x[:nz].astype(np.complex128) * w
    good = oracle.fft_frame(N, nz, 2, x[:nz])
    check_lines(good[None, :], y[None, :], N, 1, Stats(), "good")
    faults = {"shift": oracle.fft_frame(N, nz, 2, x[1:]),
              "weak_1dB": np.where(good < np.median(good), good + np.float32(1.0), good).astype(np.float32)}
    xs = x[:nz].copy()
    xs[nz // 2] *= -1                            # one sample's window sign flipped
    faults["sign"] = oracle.fft_frame(N, nz, 2, xs)
    for name, line in faults.items():
        with pytest.raises(AssertionError):
            check_lines(line[None, :], y[None, :], N, 1, Stats(), name)


def _sa(N, nz, win, build):
    return dict(N=N, nz=nz, win=win, build=build)


def _standalone_cases():
    """b200_fft_frame / b200_fft_raw: the handle writes the complex output on every call (fft_run), so both take
    k_fft_single or k_fft_p1 / k_fft_p2 (one frame: C = R = 4), whatever "fft" and "fft_cta" are.  The handle counts no
    launches, so these cases check none; the front-end cases do."""
    cases = []
    for i, L in enumerate(range(3, 23)):
        N = 1 << L
        for j, nz in enumerate([N, N - 1, max(3, int(0.6 * N)) | 1]):
            cases.append(dict(name="sa_%d_nz%d" % (N, nz), N=N, nz=nz, win=(i + j) % 3, fft=1, cta=8, build=fft_build(N, raw=True)))
    return cases


SA_CASES = _standalone_cases()
SA_NAMED = {"sa_1048576_nz1048576": "smem", "sa_65536_nz65536": "smem", "sa_2097152_nz2097152": "smem",
            "sa_4194304_nz4194304": "smem", "sa_8192_nz8192": "single", "sa_8_nz8": "single", "sa_16384_nz16384": "smem"}


def _fe(name, N, fmt, v, cta, fs, rate, win, total, lo, hi, build, scales=None, fft=1, first=0, **kw):
    """first: a first chunk of that many samples, then ragged chunks of lo .. hi samples up to `total`"""
    return dict(name=name, N=N, fmt=fmt, v=v, cta=cta, fs=fs, rate=rate, win=win, total=total, lo=lo, hi=hi, build=build,
                scales=scales, fft=fft, first=first, **kw)


def smem_geometry(N, nb, sms=132):
    """launch_fft_fmt's columns / rows per CTA (C, R) of k_fft_p1 / k_fft_p2 for a batch of nb frames (132 SMs: H100 SXM)"""
    _, l1, l2 = fft_plan(N)
    N1, N2 = 1 << l1, 1 << l2
    C = 16
    while C > 4 and (N2 // C) * nb < 2 * sms:
        C >>= 1
    while N1 * C * 8 > 196608 and C > 1:
        C >>= 1
    R = 16
    while R > 4 and (N1 // R) * nb < 2 * sms:
        R >>= 1
    while R * (N2 + 1) * 8 > 196608 and R > 1:
        R >>= 1
    return min(C, N2), min(R, N1)


FE_CASES = [
    # 2^16: (16, 16) / (16, 16)
    _fe("r16_cf32_v1_c8_span6", 1 << 16, CF32, 1, 8, 2.4e6, 20.0, 2, 1_300_000, 9000, 15000, "reg16x16/16x16_c8_tab"),
    _fe("r16_cs16_v0_c4_nz_lt_N", 1 << 16, CS16, 0, 4, 1e6, 20.0, 0, 600_000, 20000, 70000, "reg16x16/16x16_c4_gl"),
    _fe("r16_cs8_v1_c4_batched", 1 << 16, CS8, 1, 4, 65536 * 20.0, 20.0, 1, 2_000_000, 300000, 700000, "reg16x16/16x16_c4_tab"),
    _fe("r16_cs16_v1_c8_scales", 1 << 16, CS16, 1, 8, 2.4e6, 20.0, 0, 1_000_000, 20000, 50000, "reg16x16/16x16_c8_tab",
        scales=[3.1e-5, 3.1e-5, 3.1e-5, 2.7e-5, 1.0 / 32768, 1.0 / 32768, 4.1e-5]),
    # 2^17: (16, 32) / (16, 16)
    _fe("r17_cf32_v1_c4_skip0", 1 << 17, CF32, 1, 4, 131072 * 20.0, 20.0, 2, 1_500_000, 50000, 300000, "reg16x32/16x16_c4_tab"),
    _fe("r17_cs16_v1_c8_scale", 1 << 17, CS16, 1, 8, 4e6, 20.0, 0, 1_400_000, 60000, 250000, "reg16x32/16x16_c8_tab",
        scales=[3.1e-5]),
    _fe("r17_cs8_v0_c8", 1 << 17, CS8, 0, 8, 2.4e6, 20.0, 1, 900_000, 30000, 200000, "reg16x32/16x16_c8_gl"),
    # 2^18: (16, 32) / (16, 32)
    _fe("r18_cs16_v0_c8", 1 << 18, CS16, 0, 8, 262144 * 20.0, 20.0, 1, 1_800_000, 70000, 500000, "reg16x32/16x32_c8_gl"),
    # 2^19: (32, 32) / (16, 32)
    _fe("r19_cf32_v0_c4", 1 << 19, CF32, 0, 4, 524288 * 20.0, 20.0, 2, 3_000_000, 200000, 900000, "reg32x32/16x32_c4_gl"),
    _fe("r19_cs16_v1_c4_scales", 1 << 19, CS16, 1, 4, 12e6, 20.0, 0, 3_200_000, 150000, 400000, "reg32x32/16x32_c4_tab",
        scales=[2.9e-5, 2.9e-5, 3.3e-5, 3.3e-5, 3.3e-5]),
    _fe("r19_cs8_v1_c8", 1 << 19, CS8, 1, 8, 10e6, 20.0, 1, 2_000_000, 100000, 700000, "reg32x32/16x32_c8_tab"),
    # 2^20: (32, 32) / (32, 32)
    _fe("r20_cf32_v1_c8_nz_lt_N", 1 << 20, CF32, 1, 8, 2.4e6, 20.0, 2, 1_000_000, 90000, 400000, "reg32x32/32x32_c8_tab"),
    _fe("r20_cs16_v0_c4", 1 << 20, CS16, 0, 4, 30e6, 20.0, 1, 5_000_000, 400000, 1200000, "reg32x32/32x32_c4_gl"),
    _fe("r20_cs8_v1_c4_span3", 1 << 20, CS8, 1, 4, 100e6, 20.0, 0, 12_000_000, 450000, 550000, "reg32x32/32x32_c4_tab"),
    # the register builds with tables off that the cases above do not reach
    _fe("r16_cf32_v0_c8", 1 << 16, CF32, 0, 8, 65536 * 20.0, 20.0, 1, 600_000, 30000, 150000, "reg16x16/16x16_c8_gl"),
    _fe("r17_cs16_v0_c4", 1 << 17, CS16, 0, 4, 3e6, 20.0, 2, 1_000_000, 50000, 250000, "reg16x32/16x16_c4_gl",
        scales=[3.7e-5]),
    _fe("r18_cs8_v0_c4", 1 << 18, CS8, 0, 4, 262144 * 20.0, 20.0, 0, 1_400_000, 100000, 500000, "reg16x32/16x32_c4_gl"),
    _fe("r19_cs8_v0_c8", 1 << 19, CS8, 0, 8, 524288 * 20.0, 20.0, 2, 2_800_000, 200000, 900000, "reg32x32/16x32_c8_gl"),
    _fe("r20_cf32_v0_c8", 1 << 20, CF32, 0, 8, 1048576 * 20.0, 20.0, 1, 5_300_000, 350000, 2000000, "reg32x32/32x32_c8_gl"),
    # "fft" 0: the shared-memory two-pass dB path (k_fft_p1 / k_fft_p2), skip 0.  The first chunk completes enough frames
    # for C = R = 16 columns / rows per CTA; the ragged chunks behind it give small batches (C, R down to 4) and a
    # straddling frame in every chunk.
    _fe("s16_cf32_v1", 1 << 16, CF32, 1, 8, 65536 * 20.0, 20.0, 2, 26 << 16, 1 << 15, 3 << 16, "smem", fft=0,
        first=(20 << 16) + 12345),
    _fe("s17_cs16_v0_scale", 1 << 17, CS16, 0, 8, 131072 * 20.0, 20.0, 1, 25 << 17, 1 << 16, 3 << 17, "smem", fft=0,
        first=(20 << 17) + 777, scales=[3.1e-5]),
    _fe("s18_cs8_v1", 1 << 18, CS8, 1, 8, 262144 * 20.0, 20.0, 0, 15 << 18, 1 << 17, 3 << 18, "smem", fft=0,
        first=(10 << 18) + 4321),
    _fe("s19_cs16_v1", 1 << 19, CS16, 1, 8, 524288 * 20.0, 20.0, 2, 14 << 19, 1 << 18, 3 << 19, "smem", fft=0,
        first=(10 << 19) + 99),
    _fe("s20_cf32_v0", 1 << 20, CF32, 0, 8, 1048576 * 20.0, 20.0, 2, 10 << 20, 1 << 19, 3 << 20, "smem", fft=0,
        first=(6 << 20) + 5),
    _fe("s20_cs8_v1", 1 << 20, CS8, 1, 8, 1048576 * 20.0, 20.0, 1, 9 << 20, 1 << 19, 3 << 20, "smem", fft=0,
        first=(6 << 20) + 3),
    # framing restarts: an empty chunk, then set_fft mid-stream while a frame is staged
    _fe("r16_empty_chunk_set_fft", 1 << 16, CF32, 1, 8, 2.4e6, 20.0, 2, 1_000_000, 30000, 60000, "reg16x16/16x16_c8_tab",
        empty_at=4, refft_at=12, refft=(1 << 17, 15.0, 0)),
    # behind the decimator and the DC blocker: the stream is the front end's CF32 IQ tap
    _fe("r16_decim4_dc_cs16", 1 << 16, CS16, 1, 8, 10e6, 20.0, 2, 2_400_000, 100000, 300000, "reg16x16/16x16_c8_tab",
        decim=4, dc=True),
]
FE_IDS = [c["name"] for c in FE_CASES]
KA_CASES = [(1 << L, cta) for L in range(16, 21) for cta in (8, 4)]


def test_cases_reach_the_builds_they_are_named_after():
    for c in SA_CASES:
        assert c["build"] == fft_build(c["N"], raw=True), c
        if c["name"] in SA_NAMED:
            assert c["build"] == SA_NAMED[c["name"]], c
    # every window on at least one size of each stand-alone build
    for b in ("single", "smem"):
        assert {c["win"] for c in SA_CASES if c["build"] == b} == {0, 1, 2}, b
    for c in FE_CASES:
        assert c["build"] == fft_build(c["N"], c["fft"], c["cta"], tables=c["v"] != 0), c
    # every register build, (size, fft_cta, tables), through the front end: on noise, or (2^18 with tables) on the
    # known-answer streams.  A covering set: the input formats are spread over each size, not crossed with every
    # (fft_cta, tables) pair.
    reached = {(c["N"], c["cta"], c["v"] != 0) for c in FE_CASES if c["build"].startswith("reg")}
    reached |= {(N, cta, True) for N, cta in KA_CASES}
    assert reached == {(1 << L, cta, t) for L in range(16, 21) for cta in (4, 8) for t in (False, True)}, sorted(reached)
    # the shared-memory dB path at every size 2^16 .. 2^20, cf32 and integer input, fft_v 0 and 1, its widest CTAs reached
    sm = [c for c in FE_CASES if c["build"] == "smem"]
    assert {c["N"] for c in sm} == {1 << L for L in range(16, 21)}
    assert {c["fmt"] for c in sm} == {CF32, CS16, CS8} and {c["v"] for c in sm} == {0, 1}
    for c in sm:
        assert smem_geometry(c["N"], c["first"] // c["N"]) == (16, 16), c["name"]
        assert smem_geometry(c["N"], 1) == (4, 4), c["name"]
    # every register build, (RA, RB) pairs by CTA width, reached by the known-answer streams
    assert {fft_build(N, 1, cta) for N, cta in KA_CASES} == {
        "reg16x16/16x16_c8_tab", "reg16x16/16x16_c4_tab", "reg16x32/16x16_c8_tab", "reg16x32/16x16_c4_tab",
        "reg16x32/16x32_c8_tab", "reg16x32/16x32_c4_tab", "reg32x32/16x32_c8_tab", "reg32x32/16x32_c4_tab",
        "reg32x32/32x32_c8_tab", "reg32x32/32x32_c4_tab"}
    assert fft_build(1 << 18, 1, 8, tables=False) in {c["build"] for c in FE_CASES}
    # every (RA, RB) pair in both passes, cf32 / cs16 / cs8, fft_v 0 / 1 and fft_cta 4 / 8 on each front-end size
    for N in (1 << 16, 1 << 17, 1 << 19, 1 << 20):
        cs = [c for c in FE_CASES if c["N"] == N]
        assert {c["fmt"] for c in cs} == {CF32, CS16, CS8} and {c["v"] for c in cs} == {0, 1} and {c["cta"] for c in cs} == {4, 8}
    # the two over-65,535-frame cases reach the single-pass and the shared-memory two-pass builds
    assert fft_build(16) == "single" and fft_build(16384) == "smem"
    assert fe_fft_launches(16, 16, 16, 1, [((1 << 20) + 5, CF32, 0.0), (1 << 20, CF32, 0.0)])[0] == [2, 2]
    assert fe_fft_launches(16384, 16, 16, 1, [(1 << 20, CF32, 0.0)])[0] == [4]


def test_launch_mirror_counts_conversions():
    """fft_v 0 converts a staged part and transforms the straddling frame on its own; fft_v 1 does neither for one format,
    and converts when the ingest scale changes while a frame is staged"""
    N, nz, iv = 1 << 16, 1 << 16, 1 << 16
    ch = [(40000, CS16, np.float32(1 / 32768))] * 4
    assert fe_fft_launches(N, nz, iv, 1, ch)[0] == [0, 2, 0, 2]
    assert fe_fft_launches(N, nz, iv, 0, ch)[0] == [1, 4, 1, 4]
    ch2 = ch[:1] + [(40000, CS16, np.float32(3.1e-5))] + ch[2:]
    # chunk 1 converts the staged part and its own, then stages the next frame at its scale; chunk 2 (the default scale
    # again) converts that part and its own; chunk 3 extends the cf32 frame by a conversion and transforms it alone
    assert fe_fft_launches(N, nz, iv, 1, ch2)[0] == [0, 4, 2, 3]


# ---------------------------------------------------------------------------------------------- GPU part
@pytest.fixture(scope="module")
def sb():
    import sdrplusplus_b200 as m
    from sdrplusplus_b200 import lib
    L = lib.load()
    assert L.b200_device_count() > 0
    assert L.b200_init(0) == 0
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("case", SA_CASES, ids=[c["name"] for c in SA_CASES])
def test_standalone_fft_vs_float64(sb, report, case):
    N, nz, win = case["N"], case["nz"], case["win"]
    w = window64(win, nz)
    st, st_raw = Stats(), Stats()
    x = noise_iq(nz, N + nz, 1.0)
    h = sb.SpectrumHandler(N, nz, win)
    try:
        y = x.astype(np.complex128) * w
        check_lines(h.frame(x)[None, :], y[None, :], N, 1, st, case["name"])
        check_lines(h.raw(x)[None, :], y[None, :], N, 1, st_raw, case["name"] + " raw", raw=True)
        if (nz == N and N <= 1 << 20) or N < 64:
            _known_answers(sb, h, N, nz, win, w, case["cta"], st, case["name"])
    finally:
        h.close()
    report["spectrum_f64_" + case["name"]] = dict(st.row(), build=case["build"], raw=st_raw.row())


def _known_answers(sb, h, N, nz, win, w, cta, st, name):
    # all zeros: the clamp value, bit for bit; raw exactly zero
    z = np.zeros(nz, np.complex64)
    assert np.array_equal(h.frame(z).view(np.uint32), np.full(N, CLAMP_DB, np.float32).view(np.uint32)), name
    assert not np.any(h.raw(z)), name
    rng = np.random.default_rng(N + cta)
    # impulses: a flat line at 20 log10 |x w| / N, every bin; raw: the exact phase ramp at a few positions
    pos = impulse_positions(N, nz, cta)
    for j, n0 in enumerate(pos):
        x = np.zeros(nz, np.complex64)
        x[n0] = np.complex64(complex(rng.uniform(0.5, 2.0), rng.uniform(-2.0, 2.0)))
        yv = complex(x[n0]) * w[n0]
        if abs(yv) == 0.0:
            continue
        check_flat(h.frame(x)[None, :], [abs(yv)], N, 1, st, "%s impulse at %d" % (name, n0))
        if j < 4:
            X = yv * np.exp(-2j * np.pi * ((np.arange(N, dtype=np.int64) * n0) % N) / N)
            _check_raw(h.raw(x), X, abs(yv), N, 1, Stats(), "%s raw impulse at %d" % (name, n0))
    # impulse pairs: the cosine pattern, which carries the relative sign of the two window values
    for n0, n1 in [(0, 1), (1, nz - 1), (nz // 3, nz // 3 + 2), (pos[len(pos) // 2], nz - 2)]:
        if n0 == n1 or max(n0, n1) >= nz:
            continue
        x = np.zeros(nz, np.complex64)
        x[n0], x[n1] = 1.0, np.complex64(0.75 - 0.5j)
        y = x.astype(np.complex128) * w
        check_lines(h.frame(x)[None, :], y[None, :], N, 1, st, "%s pair %d,%d" % (name, n0, n1))
    # rectangular-window tones on exact bins: the peak on the predicted bin (DC sits at N/2: the (-1)^n twist)
    if nz != N:
        return
    ht = h if win == 0 else sb.SpectrumHandler(N, N, 0)
    try:
        n = np.arange(N, dtype=np.int64)
        w0 = window64(0, N)
        for k in tone_bins(N, cta, N):
            x = (0.5 * np.exp(2j * np.pi * (((k - N // 2) * n) % N) / N)).astype(np.complex64)
            y = x.astype(np.complex128) * w0
            line = ht.frame(x)
            assert int(np.argmax(line)) == k, (name, k, int(np.argmax(line)))
            check_lines(line[None, :], y[None, :], N, 1, st, "%s tone at %d" % (name, k))
    finally:
        if ht is not h:
            ht.close()


def _run_fe(sb, case, chunks, scales, fft=True, taps=False):
    """feeds chunks [(samples, fmt)]; returns (lines per FFT config, launches per chunk, tap stream parts)"""
    from sdrplusplus_b200 import lib
    fe = sb.FrontEnd(case["fs"], max(max(len(c) for c, _ in chunks), 1))
    lines, launches, tap = [[]], [], []
    try:
        fe.set_option("fft_v", case["v"])
        fe.set_option("fft_cta", case["cta"])
        fe.set_option("fft", case.get("fft", 1))
        if case.get("decim"):
            fe.set_decimation(case["decim"])
        if case.get("dc"):
            fe.set_dc_blocking(True)
        tid = fe.bind_iq(lib.IQ_CF32) if taps else None
        if fft:
            fe.set_fft(case["N"], case["rate"], case["win"])
        for k, (x, fmt) in enumerate(chunks):
            if fft and case.get("refft_at") == k:
                fe.set_fft(*case["refft"])
                lines.append([])
            if scales[k] is not None:
                fe.set_ingest_scale(fmt, scales[k])
            l0 = fe.launch_count()
            outs, ln = fe.process(x, fmt)
            launches.append(fe.launch_count() - l0)
            if ln.size:
                lines[-1].append(ln)
            if taps:
                tap.append(outs[tid])
    finally:
        fe.close()
    return [(l[0] if len(l) == 1 else np.concatenate(l)) if l else np.empty((0, 1), np.float32) for l in lines], launches, tap


def _fe_inputs(case):
    seed = FE_IDS.index(case["name"]) if case["name"] in FE_IDS else 99
    first = case.get("first", 0)
    sizes = ([first] if first else []) + ragged(case["total"] - first, case["lo"], case["hi"], seed)
    if case.get("empty_at") is not None:
        sizes.insert(case["empty_at"], 0)
    rng = np.random.default_rng(1000 + seed)
    fmt = case["fmt"]
    chunks = [(gen_chunk(rng, n, fmt), fmt) for n in sizes]
    sc = case["scales"]
    default = {CF32: 0.0, CS16: 1.0 / 32768, CS8: 1.0 / 128}[fmt]
    scales = [None if fmt == CF32 or sc is None else sc[k % len(sc)] for k in range(len(chunks))]
    eff = [default if s is None else s for s in scales]
    return chunks, scales, eff


@pytest.mark.gpu
@pytest.mark.parametrize("case", FE_CASES, ids=FE_IDS)
def test_frontend_lines_vs_float64(sb, report, case):
    """every line of a front end from line 0 against the float64 transform of the samples at fstart + f (nz + skip)"""
    from sdrplusplus_b200 import frontend
    chunks, scales, eff = _fe_inputs(case)
    taps = bool(case.get("decim") or case.get("dc"))
    lines, launches, tap = _run_fe(sb, case, chunks, scales, taps=taps)
    _, base, _ = _run_fe(sb, case, chunks, scales, fft=False)
    if taps:
        x = np.concatenate(tap).astype(np.complex128)
        fs_eff = case["fs"] / case.get("decim", 1)
        c0 = 1
    else:
        x = stream_f64([(c, f, s) for (c, f), s in zip(chunks, eff)])
        fs_eff = case["fs"]
        c0 = 1 if all(f == CF32 or float(np.float32(s)) == 2.0 ** round(math.log2(s)) for (_, f), s in zip(chunks, eff)) else 2
    # framing: each FFT configuration starts at the stream position where it was set
    configs = [(0, case["N"], case["rate"], case["win"])]
    if case.get("refft_at") is not None:
        p = sum(len(c) for c, _ in chunks[:case["refft_at"]])
        configs.append((p, *case["refft"]))
    st = Stats()
    want = []
    for i, (p0, N, rate, win) in enumerate(configs):
        nz, skip = frontend.fft_frame_params(fs_eff, N, rate)
        iv = nz + skip
        p1 = configs[i + 1][0] if i + 1 < len(configs) else x.size
        nl = (p1 - p0 - nz) // iv + 1 if p1 - p0 >= nz else 0
        assert nl >= 2, (case["name"], nl)
        assert lines[i].shape == (nl, N), (case["name"], i, lines[i].shape, nl)
        Y = frames_of(x, p0, nz, iv, nl) * window64(win, nz)[None, :]
        check_lines(lines[i], Y, N, c0, st, "%s config %d" % (case["name"], i))
        want.append((N, nz, iv, p0, p1))
    if not taps and case.get("refft_at") is None:
        N, nz, iv, _, _ = want[0]
        info = [(len(c), f, float(np.float32(s)) if f != CF32 else 0.0) for (c, f), s in zip(chunks, eff)]
        exp, _ = fe_fft_launches(N, nz, iv, case["v"], info)
        assert [a - b for a, b in zip(launches, base)] == exp, (case["name"], launches, base, exp)
    report["spectrum_f64_" + case["name"]] = dict(st.row(), build=case["build"])


def _frames_through_fe(sb, frames, N, cta, win, seed):
    """frames (nz = N, skip 0) fed to a front end in ragged chunks; returns the lines and the spectrum launches"""
    x = np.concatenate(frames)
    sizes = ragged(x.size, N // 2, 3 * N, seed)
    edges = np.cumsum([0] + sizes)
    chunks = [(x[a:b], CF32) for a, b in zip(edges[:-1], edges[1:]) if b > a]
    case = dict(fs=N * 20.0, v=1, cta=cta, N=N, rate=20.0, win=win)
    lines, launches, _ = _run_fe(sb, case, chunks, [None] * len(chunks))
    _, base, _ = _run_fe(sb, case, chunks, [None] * len(chunks), fft=False)
    exp, _ = fe_fft_launches(N, N, N, 1, [(len(c), CF32, 0.0) for c, _ in chunks])
    assert [a - b for a, b in zip(launches, base)] == exp, (launches, base, exp)
    assert lines[0].shape == (len(frames), N)
    return lines[0]


@pytest.mark.gpu
@pytest.mark.parametrize("N,cta", KA_CASES, ids=["ka_%d_c%d" % c for c in KA_CASES])
def test_register_builds_known_answers(sb, report, N, cta):
    """every register build through the front end, one known answer per frame, frames straddling ragged chunks.  Nuttall
    window: an all-zero frame (the clamp value, bit for bit), an impulse at every a and every t of pass 1's
    n = (a RB + t) N2 + n2 at the first and last columns of a CTA (flat lines), impulse pairs (the cosine pattern and the
    relative sign of two window values).  Rectangular window: tones on exact bins at every residue of a pass-2 CTA, the
    peak on the predicted bin and every other bin inside its bound."""
    rng = np.random.default_rng(N + cta)
    w = window64(2, N)
    pos = impulse_positions(N, N, cta)
    frames = [np.zeros(N, np.complex64)]
    for p in pos:
        x = np.zeros(N, np.complex64)
        x[p] = np.complex64(complex(rng.uniform(0.5, 2.0), rng.uniform(-2.0, 2.0)))
        frames.append(x)
    pairs = [(1, 2), (3, N - 2), (N // 3, N // 3 + 2), (pos[len(pos) // 2], N - 1)]
    for n0, n1 in pairs:
        x = np.zeros(N, np.complex64)
        x[n0], x[n1] = 1.0, np.complex64(0.75 - 0.5j)
        frames.append(x)
    lines = _frames_through_fe(sb, frames, N, cta, 2, N + cta)
    assert np.array_equal(lines[0].view(np.uint32), np.full(N, CLAMP_DB, np.float32).view(np.uint32))
    st = Stats()
    amp = [abs(complex(f[p]) * w[p]) for f, p in zip(frames[1:], pos)]
    check_flat(lines[1:1 + len(pos)], amp, N, 1, st, "impulses")
    Y = np.stack(frames[1 + len(pos):]).astype(np.complex128) * w[None, :]
    check_lines(lines[1 + len(pos):], Y, N, 1, st, "pairs")
    # tones, rectangular window (DC sits at N/2: the (-1)^n twist)
    n = np.arange(N, dtype=np.int64)
    bins = tone_bins(N, cta, N + cta)
    tones = [(0.5 * np.exp(2j * np.pi * (((k - N // 2) * n) % N) / N)).astype(np.complex64) for k in bins]
    lines = _frames_through_fe(sb, tones, N, cta, 0, N + cta + 1)
    assert [int(v) for v in np.argmax(lines, axis=1)] == bins
    check_lines(lines, np.stack(tones).astype(np.complex128) * window64(0, N)[None, :], N, 1, st, "tones")
    report["spectrum_f64_ka_%d_c%d" % (N, cta)] = dict(st.row(), build=fft_build(N, 1, cta))


SPLIT_CASES = [(1 << 16, 1, 1, CF32), (1 << 17, 1, 1, CS16), (1 << 20, 1, 0, CS8), (1 << 16, 0, 1, CS16), (1 << 18, 0, 0, CF32),
               (4096, 1, 1, CS16)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,fft,v,fmt", SPLIT_CASES, ids=["split_%d_fft%d_v%d_f%d" % c for c in SPLIT_CASES])
def test_impulses_at_the_split_of_a_straddling_frame(sb, report, N, fft, v, fmt):
    """every frame straddles a chunk edge at a chosen offset s (the first chunk ends s samples into frame 0, each later
    chunk s' samples into the next frame); the frame holds an impulse pair on its last staged sample s - 1 and its first
    sample from the chunk s, so the staged / direct boundary (FrameSrc::lim) and the ingest scale of the staged part are
    pinned on every frame, not only where a ragged schedule happens to put an edge"""
    _, l1, l2 = fft_plan(N)
    N2 = 1 << l2
    splits = sorted(({1, 2, N2 - 1, N2, N2 + 1, N // 2, N - 2, N - 1} | {int(v) for v in np.random.default_rng(N).integers(1, N, 4)})
                    & set(range(1, N)))
    F = len(splits)
    edges = [f * N + sp for f, sp in enumerate(splits)] + [F * N]
    rng = np.random.default_rng(N + 7)
    if fmt == CF32:
        x = np.zeros(F * N, np.complex64)
        for f, sp in enumerate(splits):
            x[f * N + sp - 1] = np.complex64(complex(rng.uniform(0.5, 1.0), rng.uniform(-1.0, 1.0)))
            x[f * N + sp] = np.complex64(complex(rng.uniform(-1.0, -0.5), rng.uniform(-1.0, 1.0)))
    else:
        x = np.zeros((F * N, 2), np.int16 if fmt == CS16 else np.int8)
        hi = 20000 if fmt == CS16 else 120
        for f, sp in enumerate(splits):
            x[f * N + sp - 1] = rng.integers(hi // 2, hi, 2)
            x[f * N + sp] = -rng.integers(hi // 2, hi, 2)
    chunks = [(x[a:b], fmt) for a, b in zip([0] + edges[:-1], edges)]
    scale = 3.1e-5 if fmt == CS16 else None                   # not a power of two: the staged part's own rounding
    case = dict(fs=N * 20.0, v=v, cta=8, N=N, rate=20.0, win=2, fft=fft)
    lines, launches, _ = _run_fe(sb, case, chunks, [scale] * len(chunks))
    _, base, _ = _run_fe(sb, case, chunks, [scale] * len(chunks), fft=False)
    eff = scale if scale is not None else {CF32: 0.0, CS16: 1.0 / 32768, CS8: 1.0 / 128}[fmt]
    info = [(len(c), fmt, float(np.float32(eff)) if fmt != CF32 else 0.0) for c, _ in chunks]
    exp, _ = fe_fft_launches(N, N, N, v, info)
    assert [a - b for a, b in zip(launches, base)] == exp, (launches, base, exp)
    xs = stream_f64([(x, fmt, eff)])
    assert lines[0].shape == (F, N)
    st = Stats()
    check_lines(lines[0], frames_of(xs, 0, N, N, F) * window64(2, N)[None, :], N, 1 if scale is None else 2, st, "split")
    report["spectrum_f64_split_%d_fft%d_v%d_f%d" % (N, fft, v, fmt)] = dict(st.row(), build=fft_build(N, fft, 8, tables=v != 0))


@pytest.mark.gpu
def test_bench_configuration_every_bin(sb, report):
    """100 MS/s, one 16 Mi-sample chunk, 1 Mi points at 20 fps, the input of test_bench_configuration_one_16mi_chunk_vs_oracle:
    every bin of every line, the noise floor included"""
    fs, n = 100e6, 1 << 24
    x = noise_iq(n, 0x5D12, 0.01).copy()
    for o in [5e6, -5e6, 15e6, -15e6, 25e6, -25e6, 35e6, -35e6]:
        for s in range(0, n, 1 << 21):
            x[s:s + (1 << 21)] += fm_carrier(min(1 << 21, n - s), fs, o, start=s)
    fe = sb.FrontEnd(fs, n)
    try:
        fe.set_fft(1 << 20, 20.0, 2)
        _, lines = fe.process(x)
    finally:
        fe.close()
    from sdrplusplus_b200 import frontend
    nz, skip = frontend.fft_frame_params(fs, 1 << 20, 20.0)
    assert lines.shape == (4, 1 << 20)
    Y = frames_of(x, 0, nz, nz + skip, 4).astype(np.complex128) * window64(2, nz)[None, :]
    st = Stats()
    check_lines(lines, Y, 1 << 20, 1, st, "bench")
    report["spectrum_f64_bench_16mi"] = dict(st.row(), build=fft_build(1 << 20))


@pytest.mark.gpu
def test_more_than_65535_frames_single_pass(sb, report):
    """16 points at fs / 16: 65,536 frames complete in each 1 Mi-sample chunk, the second chunk's first one begun in the
    first (a batch launched in two slices, the first keeping the staged part)"""
    fs, N = 1.6e6, 16
    sizes = [(1 << 20) + 5, 1 << 20]
    rng = np.random.default_rng(16)
    chunks = [(gen_chunk(rng, n, CF32), CF32) for n in sizes]
    case = dict(fs=fs, v=1, cta=8, N=N, rate=fs / 16, win=2)
    lines, launches, _ = _run_fe(sb, case, chunks, [None, None])
    _, base, _ = _run_fe(sb, case, chunks, [None, None], fft=False)
    x = stream_f64([(c, f, 0.0) for c, f in chunks])
    nl = (x.size - 16) // 16 + 1
    assert nl > 2 * MAX_GRID_Y and lines[0].shape == (nl, N)
    st = Stats()
    check_lines(lines[0], frames_of(x, 0, 16, 16, nl) * window64(2, 16)[None, :], N, 1, st, "16-point")
    assert [a - b for a, b in zip(launches, base)] == [2, 2], (launches, base)
    report["spectrum_f64_over_65535_single"] = dict(st.row(), build="single")


@pytest.mark.gpu
def test_more_than_65535_frames_two_pass(sb, report):
    """16,384 points (k_fft_p1 / k_fft_p2) over 16-sample frames at fs / 16: 65,536 frames in one 1 Mi-sample chunk.  Each
    frame holds one impulse of its own size, so every bin of every line has a closed-form interval.
    Footprint: the front end's work buffer holds 65,538 frames of 16,384 float2 (8.6 GB of device memory), its line buffer
    4.3 GB, and the lines come back as one 4.3 GB host array: no smaller chunk completes more than 65,535 two-pass frames."""
    fs, N, n = 1.6e6, 16384, 1 << 20
    F = n // 16
    rng = np.random.default_rng(17)
    f = np.arange(F)
    n0 = (f * 5 + 3) % 16
    amp = (1.0 + (f % 7) / 8.0) * 2.0 ** -(f % 5)
    x = np.zeros(n, np.complex64)
    x[f * 16 + n0] = (amp * np.exp(1j * rng.uniform(0, 2 * np.pi, F))).astype(np.complex64)
    case = dict(fs=fs, v=1, cta=8, N=N, rate=fs / 16, win=0)
    lines, launches, _ = _run_fe(sb, case, [(x, CF32)], [None])
    _, base, _ = _run_fe(sb, case, [(x, CF32)], [None], fft=False)
    assert lines[0].shape == (F, N)
    assert launches[0] - base[0] == 4
    yv = np.abs(x[f * 16 + n0].astype(np.complex128))        # rectangular window: |w| = 1
    st = Stats()
    check_flat(lines[0], yv, N, 1, st, "16384-point")
    report["spectrum_f64_over_65535_two_pass"] = dict(st.row(), build="smem")

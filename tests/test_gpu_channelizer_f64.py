"""The 256-channel polyphase filter-bank channelizer (BASELINE config 3: chanpfb.cuh's k_chan_branch + k_chan_fft behind
b200_chan_process) against a float64 reference, output by output, from output 0 of the stream.

Reference.  With M = 256 channels, P taps per branch, T = M P and the library's fp32 prototype h (b200_chan_prototype,
pinned below to the oracle's windowed sinc bit for bit) and the fp32 input x both taken as exact values,
    y_k[m] = sum_t h[t] x[n0 + t] e^{-j 2 pi k (n0 + t) / M},   n0 = (m - P + 1) M,   x[n] = 0 for n < 0.
n0 is a multiple of M, so with t = p M + r the phasor depends on r only, and
    u_r[m] = sum_p h[p M + r] x[(m + p - P + 1) M + r],      y_k[m] = sum_r u_r[m] e^{-j 2 pi k r / M},
which ref_f64 evaluates in float64: the branch sums with a loop over p (vectorised over (m, r)), then np.fft.fft along r.
The CPU half pins that evaluation to the literal direct form (every channel of a few output times, and the history outputs
m < P - 1) to a float64-level tolerance.

A-priori per-output bound.  u = 2^-24, gamma_P = P u / (1 - P u), L = log2 M = 8, eta = 8.
  * Branch sums (k_chan_branch): each component of u_r[m] is P sequential fp32 FMAs from 0 (ffma2 = two fmaf), so the
    computed branch value differs from u_r[m] by at most b_r[m] = gamma_P A_r[m] in modulus, where
    A_r[m] = sum_p |h[p M + r]| (|Re x| + |Im x|) over the window (A_r also bounds |u_r|).
  * Transform (k_chan_fft: fft_dif_smem with M = 256, radix 8, radix 8, radix 4; the fp32 `tw` table rounded from double).
    One radix-2 level is an add or subtract (u per component), the table twiddle (u), the complex product (3 u) and, in the
    radix-8 passes, the W8 rotation before it (mul_w8_1 / mul_w8_3: 3 u): eta = 8 per level, as in
    test_gpu_spectrum_f64.py.  At every level the nodes feeding one output partition the inputs, so a level adds at most
    eta u sum_r |u^_r| to any channel, with |u^_r| <= (1 + gamma_P) A_r.
  * Branch errors reach each output through unit-modulus twiddles: sum_r b_r.
  * So  |y^_k[m] - y_k[m]| <= B[m] = (gamma_P + eta L u (1 + gamma_P)) S[m] (1 + 2 (gamma_P + eta L u)),  S[m] = sum_r A_r[m],
    the last factor covering products of rounding errors (values grown by (1 + eta u)^L).  Nothing is fitted to a run.
  * Norm-wise (Higham) per output time: the transform is sqrt(M) times a unitary map, so
        || y^[m] - y[m] ||_2 <= (sqrt(M) ||b[m]||_2 + eta L u (||y[m]||_2 + sqrt(M) ||b[m]||_2)) (same slack factor).
  * Gain per channel, fitted over the whole stream: g_k = <y_k, y^_k> / <y_k, y_k>, and by Cauchy-Schwarz
    |g_k - 1| <= sqrt(sum_m B[m]^2) / ||y_k||_2.
An fp32 emulation of the kernels' order uses about 0.3 % of B on noise: the per-output bound only catches gross errors.
The sharp checks are the known answers and the bit identities.

Known answers.  One impulse a at stream position s (residue r = s mod M), no other within T samples: an output time m with
t = s - n0(m) in [0, T) has one nonzero branch, u_r = fl(h[t] a) (u relative), and every butterfly of its transform has a
zero partner: the add or subtract is exact, mul_mj is exact, and only the rotations round.  On the value's path: radix-8
stage A (W8 rotation 3 u, table twiddle u, product 3 u), stage B (mul_mj exact, twiddle u + product 3 u), stage C (4 u), twice;
the radix-4 pass is exact.  So
    |y^_k[m] - a h[t] e^{-j 2 pi k r / M}| <= ((1 + u) (1 + 7 u)^2 (1 + 4 u)^4 - 1) |a h[t]|   (31 u to first order),
for every tap t of the prototype, including the ones near 1e-8 that no RMS figure can see, and every other output is 0.

Host bookkeeping mirrored here: hist = (P - 1) M history samples; a call with 0 < count < hist carries the history with
k_carry (one launch more), count >= hist copies it with one device copy; every call with count > 0 launches k_chan_branch
and k_chan_fft; count = 0 does nothing.
"""
import ctypes as C
import math

import numpy as np
import pytest

from f64_ref import U, REF_FLOOR
from util import noise_iq

M = 256
LOGM = 8
ETA = 8.0
CH_MT = 256                                     # chanpfb.cuh: output times per CTA row of k_chan_branch
FS = 500e6
MAX_N4099 = 4099 * M                            # a handle whose max_chunk allows n_out = 4099
MI = 1 << 20
P_SWEEP = [1, 2, 7, 8, 9, 16, 64, 127, 128, 255]
KA_P = [1, 7, 8, 9, 127, 255]
KA_AMP = np.complex64(0.75 - 0.5j)
B200_EINVAL, B200_ECAP = -1, -5


# ---------------------------------------------------------------------------------------------- mirrors of the host code
def hist_of(P):
    return (P - 1) * M


def history_branch(count, P):
    """b200_chan_process: how the history of the next call is kept ("carry": k_carry, "copy": one device copy)"""
    if count == 0:
        return None
    return "copy" if count >= hist_of(P) else "carry"


def launches_of(count, P):
    """launches of one accepted b200_chan_process call"""
    if count == 0:
        return 0
    return 2 + (1 if history_branch(count, P) == "carry" else 0)


def seam_schedule(P, max_chunk=MAX_N4099):
    """chunk counts that cross every seam: one and two output times, the history length and one output time either side,
    one full CTA row (n_out 256) and one output time more, n_out 4095 (n_out % 8 = 7), 1 Mi samples, an empty call, and
    n_out 4099 where max_chunk allows it"""
    h = hist_of(P)
    want = [256, 512, h - 256, h, h + 256, 65536, 65792, MI - 256, MI, 0, 4099 * M]
    return [c for c in want if c == 0 or 0 < c <= max_chunk]


def mem_kinds(n):
    """(in, out) memory kind of call i: every pair of host pageable, pinned (b200_host_alloc) and device"""
    kinds = [(a, b) for a in ("host", "pinned", "device") for b in ("host", "pinned", "device")]
    return [kinds[(5 * i) % len(kinds)] for i in range(n)]


def prototype_f64(P):
    """taps::windowedSinc(T, pi / M, nuttall) in float64 (what the library rounds to fp32)"""
    T = M * P
    t = np.arange(T, dtype=np.float64) - T / 2.0 + 0.5
    om = math.pi / M
    x = t * om
    s = np.where(x == 0.0, 1.0, np.sin(x) / np.where(x == 0.0, 1.0, x))
    n = t - T / 2.0
    c = [0.355768, 0.487396, 0.144232, 0.012604]
    w = c[0] - c[1] * np.cos(2 * np.pi * n / T) + c[2] * np.cos(4 * np.pi * n / T) - c[3] * np.cos(6 * np.pi * n / T)
    return s * w * (om / math.pi)


# ---------------------------------------------------------------------------------------------- float64 reference and gates
def _rows(x, P):
    """[P - 1 zero rows | x] as rows of M samples (complex128)"""
    x = np.asarray(x).astype(np.complex128)
    return np.concatenate([np.zeros((P - 1) * M, np.complex128), x]).reshape(-1, M)


def ref_f64(x, h, P, m0=0, m1=None):
    """y_k[m] for m0 <= m < m1 through the polyphase identity; also A_r[m] (module docstring)"""
    xr = _rows(x, P)
    n_out = xr.shape[0] - (P - 1)
    m1 = n_out if m1 is None else m1
    H = np.asarray(h, np.float64).reshape(P, M)
    aH = np.abs(H)
    ax = np.abs(xr.real) + np.abs(xr.imag)
    u = np.zeros((m1 - m0, M), np.complex128)
    A = np.zeros((m1 - m0, M))
    for p in range(P):
        u += H[p] * xr[m0 + p: m1 + p]
        A += aH[p] * ax[m0 + p: m1 + p]
    return np.fft.fft(u, axis=1), A


def direct_f64(x, h, P, m_list, channels):
    """the literal direct form: sum over all T taps with the phasor of (n0 + t) mod M"""
    T = M * P
    xh = np.concatenate([np.zeros(T - M, np.complex128), np.asarray(x).astype(np.complex128)])
    h = np.asarray(h, np.float64)
    t = np.arange(T)
    E = np.exp(-2j * np.pi * np.outer(np.asarray(channels), np.arange(M)) / M)
    out = np.empty((len(m_list), len(channels)), np.complex128)
    for a, m in enumerate(m_list):
        n0 = (m - P + 1) * M
        seg = xh[(T - M) + n0: (T - M) + n0 + T]
        out[a] = E[:, (n0 + t) % M] @ (h * seg)
    return out


def bound_coefs(P):
    g = P * U / (1.0 - P * U)
    f = ETA * LOGM * U
    slack = 1.0 + 2.0 * (g + f)
    return g, f, slack


class Stats:
    """worst figures over the outputs of one case, and the per-channel sums of the gain gate"""

    def __init__(self, P):
        self.P = P
        self.frac, self.norm, self.outputs = 0.0, 0.0, 0
        self.num = np.zeros(M, np.complex128)
        self.den = np.zeros(M)
        self.b2 = 0.0

    def gain(self):
        """max |g_k - 1| and its gate, asserted"""
        assert self.outputs > 0
        g = self.num / self.den
        lim = math.sqrt(self.b2) / np.sqrt(self.den)
        bad = np.flatnonzero(np.abs(g - 1.0) > lim)
        assert bad.size == 0, "gain of channel %d: |g - 1| = %r > %r" % (bad[0], abs(g[bad[0]] - 1.0), lim[bad[0]])
        return float(np.max(np.abs(g - 1.0)))

    def row(self):
        return {"bound_used": self.frac, "norm_ratio": self.norm, "gain_minus_1": self.gain(), "outputs": self.outputs}


def check_block(y, Y, A, P, st, what, m0=0):
    """y (n, M) from the library against the float64 Y with the per-output bound, the norm-wise gate per output time and the
    sums of the gain gate"""
    g, f, slack = bound_coefs(P)
    S = A.sum(axis=1)
    B = ((g + f * (1.0 + g)) * S) * slack + REF_FLOOR * S
    d = np.abs(np.asarray(y).astype(np.complex128) - Y)
    over = d > B[:, None]
    if over.any():
        i, k = np.argwhere(over)[0]
        raise AssertionError("%s: %d outputs beyond the bound, first m=%d k=%d: |err| %r > %r (|y| %r)" % (
            what, int(over.sum()), m0 + i, k, d[i, k], B[i], abs(Y[i, k])))
    nb = np.sqrt(M) * g * np.linalg.norm(A, axis=1)
    nY = np.linalg.norm(Y, axis=1)
    tol = (nb + f * (nY + nb)) * slack + REF_FLOOR * S * np.sqrt(M)
    en = np.linalg.norm(d, axis=1)
    bad = np.flatnonzero(en > tol)
    assert bad.size == 0, "%s: norm-wise at m=%d: %r > %r" % (what, m0 + bad[0], en[bad[0]], tol[bad[0]])
    live = B > 0
    if live.any():
        st.frac = max(st.frac, float(np.max(d[live] / B[live, None])))
        st.norm = max(st.norm, float(np.max(en[live] / tol[live])))
    st.num += np.sum(np.conj(Y) * np.asarray(y).astype(np.complex128), axis=0)
    st.den += np.sum(np.abs(Y) ** 2, axis=0)
    st.b2 += float(np.sum(B ** 2))
    st.outputs += y.shape[0]


def check_stream(y, x, h, P, st, what, block=2048):
    """every output of the stream, from output 0"""
    n_out = x.size // M
    assert y.shape == (n_out, M), (what, y.shape, n_out)
    for m0 in range(0, n_out, block):
        m1 = min(n_out, m0 + block)
        lo = max(0, m0 - (P - 1))                       # the first input row output m0 reads
        Y, A = ref_f64(x[lo * M: m1 * M], h, P, m0 - lo, m1 - lo)
        check_block(y[m0:m1], Y, A, P, st, what, m0)


def ka_rel():
    return (1 + U) * (1 + 7 * U) ** 2 * (1 + 4 * U) ** 4 - 1.0


def impulse_stream(P, residues, seed):
    """one impulse KA_AMP per residue at s_i = i (T + M) + r_i: any two at least T + 1 samples apart"""
    T = M * P
    S = T + M
    rng = np.random.default_rng(seed)
    r = rng.permutation(np.asarray(residues, np.int64))
    s = np.arange(r.size, dtype=np.int64) * S + r
    n = (r.size + 1) * S
    x = np.zeros(n, np.complex64)
    x[s] = KA_AMP
    return x, s


def impulse_schedule(P, s, n, max_chunk, seed):
    """ragged chunk counts (multiples of M, both history branches) with a chunk starting at the residue-0 impulse and one
    ending at the residue-255 impulse"""
    rng = np.random.default_rng(seed)
    h = hist_of(P)
    menu = [c for c in (256, 512, h - 256, h, h + 256, 65536, 65792, MI - 256) if 0 < c <= max_chunk]
    cuts = {0, n}
    for v in s:
        if v % M == 0:
            cuts.add(int(v))
        if v % M == M - 1:
            cuts.add(int(v) + 1)
    pos = 0
    for c in menu[:3]:                                  # 256, 512 and hist - 256 first: a carried history early on
        pos += c
        cuts.add(min(pos, n))
    while pos < n:
        pos += int(menu[int(rng.integers(0, len(menu)))] if rng.random() < 0.7 else M * int(rng.integers(1, max_chunk // M + 1)))
        cuts.add(min(pos, n))
    cuts = sorted(cuts)
    out = []
    for a, b in zip(cuts[:-1], cuts[1:]):
        while b - a > max_chunk:
            out.append(max_chunk)
            a += max_chunk
        out.append(b - a)
    return out


def check_impulses(y, s, h, P, st, what):
    """every output of an impulse stream: the known answer on each impulse's support, exact zeros elsewhere"""
    n_out = y.shape[0]
    sup = np.zeros(n_out, bool)
    h = np.asarray(h, np.float64)
    rel = ka_rel()
    a = complex(KA_AMP)
    kk = np.arange(M)
    worst = 0.0
    for v in s:
        q, r = int(v) // M, int(v) % M
        rows = np.arange(q, q + P)
        rows = rows[rows < n_out]
        t = r + (P - 1 - (rows - q)) * M
        want = a * h[t][:, None] * np.exp(-2j * np.pi * ((kk * r) % M) / M)[None, :]
        got = y[rows].astype(np.complex128)
        tol = rel * np.abs(want)
        d = np.abs(got - want)
        bad = d > tol
        if bad.any():
            i, k = np.argwhere(bad)[0]
            raise AssertionError("%s: impulse at %d (r=%d), m=%d tap %d channel %d: %r, want %r (|err| %r > %r)" % (
                what, v, r, rows[i], t[i], k, got[i, k], want[i, k], d[i, k], tol[i, k]))
        live = tol > 0
        if live.any():
            worst = max(worst, float(np.max(d[live] / tol[live])))
        sup[rows] = True
    nz = np.flatnonzero(np.any(y[~sup] != 0, axis=1))
    assert nz.size == 0, "%s: output time %d is not zero outside every impulse's support" % (what, np.flatnonzero(~sup)[nz[0]])
    st.frac = max(st.frac, worst)
    st.outputs += n_out


def stream_input(n, seed):
    """uniform [-1, 1) re / im like the bench's C3 leg, plus tones at channel centres + 0.1 of a channel and a DC term"""
    x = noise_iq(n, seed, 1.0).astype(np.complex128)
    t = np.arange(n, dtype=np.float64)
    for k, a in ((5, 0.7), (100, 0.5), (255, 0.3), (128, 0.2)):
        x += a * np.exp(2j * np.pi * (((k + 0.1) * t) % M) / M)
    x += 0.25 - 0.125j
    return x.astype(np.complex64)


# ---------------------------------------------------------------------------------------------- fp32 emulation (CPU half)
def _tw32():
    k = np.arange(M)
    a = -2.0 * np.pi * k / M
    return (np.cos(a).astype(np.float32) + 1j * np.sin(a).astype(np.float32)).astype(np.complex64)


def _bitrev():
    return np.array([int(format(k, "08b")[::-1], 2) for k in range(M)])


def dif32(u):
    """radix-2 DIF in fp32 with the fp32 twiddle table, natural-order output"""
    tw = _tw32()
    a = np.asarray(u, np.complex64).copy()
    n = a.shape[0]
    nb = M
    while nb >= 2:
        hb = nb // 2
        b = a.reshape(n, M // nb, nb)
        top, bot = b[:, :, :hb], b[:, :, hb:]
        w = tw[np.arange(hb) * (M // nb)]
        a = np.concatenate([top + bot, ((top - bot) * w).astype(np.complex64)], axis=2).reshape(n, M).astype(np.complex64)
        nb = hb
    return a[:, _bitrev()]


def emulate(x, h, P, sched, fault=None):
    """the library's order in fp32 over a chunk schedule: history carried between calls, each branch P sequential fp32
    FMAs per component (products exact in float64, one rounding to fp32 per step), then dif32.  fault: "hist_late" (the
    history taken one output time late), "tap" (tap p = 120 of every branch dropped), "row2" (the second CTA row of each
    call one output time early), "mirror" (channels k <-> M - k), "swap" (re and im swapped in branch 37)"""
    H = np.asarray(h, np.float64).reshape(P, M)
    hist = hist_of(P)
    hb = np.zeros(hist, np.complex64)
    out, pos = [], 0
    for c in sched:
        if c == 0:
            continue
        data = np.concatenate([hb, x[pos:pos + c]])
        pos += c
        n_out = c // M
        rows = data.reshape(-1, M)
        re, im = rows.real.astype(np.float64), rows.imag.astype(np.float64)
        start = np.arange(n_out)
        if fault == "row2":
            sel = (start >= CH_MT) & (start < 2 * CH_MT)
            start[sel] -= 1
        ar = np.zeros((n_out, M), np.float32)
        ai = np.zeros((n_out, M), np.float32)
        for p in range(P):
            if fault == "tap" and p == 120:
                continue
            ar = (H[p] * re[start + p] + ar).astype(np.float32)
            ai = (H[p] * im[start + p] + ai).astype(np.float32)
        if fault == "swap":
            ar[:, 37], ai[:, 37] = ai[:, 37].copy(), ar[:, 37].copy()
        y = dif32(ar + 1j * ai)
        if fault == "mirror":
            y = y[:, (-np.arange(M)) % M]
        out.append(y)
        if hist:
            hb = data[data.size - hist - (M if fault == "hist_late" else 0): data.size - (M if fault == "hist_late" else 0)].copy()
    return np.concatenate(out) if out else np.zeros((0, M), np.complex64)


# ---------------------------------------------------------------------------------------------- CPU half
@pytest.mark.parametrize("P", P_SWEEP)
def test_reference_equals_direct_form(oracle, P):
    """ref_f64 == the literal direct form: every history output m < P - 1 on four channels, every channel of three later
    output times"""
    T = M * P
    h = oracle.lowpass(FS / 512.0, 3.8 * FS / T, FS)
    assert h.size == T
    n_out = P + 40
    x = stream_input(n_out * M, 100 + P)
    Y, A = ref_f64(x, h, P)
    scale = A.sum(axis=1)
    ms = list(range(P - 1)) if P > 1 else [0]
    ch = [0, 1, 127, 255]
    D = direct_f64(x, h, P, ms, ch)
    err = np.abs(Y[np.ix_(ms, ch)] - D) / scale[ms, None]
    assert err.max() <= REF_FLOOR, err.max()
    ms2 = [P - 1, P + 7, n_out - 1]
    D2 = direct_f64(x, h, P, ms2, list(range(M)))
    err2 = np.abs(Y[ms2] - D2) / scale[ms2, None]
    assert err2.max() <= REF_FLOOR, err2.max()


EMU_SCHED = [600 * M, 300 * M, 40 * M, 0, 700 * M]            # P = 127: two CTA rows, both history branches, an empty call


def test_schedules_cross_every_seam():
    for P in P_SWEEP:
        s = seam_schedule(P)
        nouts = {c // M for c in s}
        assert {1, 2, 256, 257, 4095, 4096, 4099} <= nouts and 0 in s, (P, s)
        br = {history_branch(c, P) for c in s} - {None}
        assert br == ({"copy"} if P <= 2 else {"copy", "carry"}), (P, br)
        assert max(s) <= MAX_N4099
        assert len(set(mem_kinds(len(s)))) == 9, (P, s)
    assert {history_branch(c, 127) for c in EMU_SCHED} - {None} == {"copy", "carry"}
    assert max(EMU_SCHED) // M > CH_MT
    # the launch mirror
    assert launches_of(0, 127) == 0 and launches_of(256, 127) == 3 and launches_of(hist_of(127), 127) == 2
    assert launches_of(256, 1) == 2 and launches_of(256, 2) == 2 and launches_of(256, 3) == 3
    # the impulse streams: impulses at the first and the last sample of a chunk, both history branches where they exist
    for P in KA_P:
        x, s = impulse_stream(P, range(M), P)
        sched = impulse_schedule(P, s, x.size, MAX_N4099, P)
        assert sum(sched) == x.size and all(0 < c <= MAX_N4099 and c % M == 0 for c in sched)
        starts = np.cumsum([0] + sched[:-1])
        ends = np.cumsum(sched) - 1
        assert set(s.tolist()) & set(starts.tolist()) and set(s.tolist()) & set(ends.tolist()), P
        assert {history_branch(c, P) for c in sched} - {None} == ({"copy"} if P <= 2 else {"copy", "carry"}), P
        assert np.min(np.diff(s)) >= M * P + 1


@pytest.fixture(scope="module")
def emu_case(oracle):
    P = 127
    T = M * P
    h = oracle.lowpass(FS / 512.0, 3.8 * FS / T, FS)
    x = stream_input(sum(EMU_SCHED), 7)
    xi, s = impulse_stream(P, [0, 1, 37, 128, 200, 254, 255], 9)
    return P, h, x, xi, s


def _all_gates(y, yi, case):
    P, h, x, xi, s = case
    st = Stats(P)
    check_stream(y, x, h, P, st, "emulation")
    row = st.row()
    check_impulses(yi, s, h, P, Stats(P), "emulation impulses")
    return row


def test_emulation_inside_the_bound(emu_case):
    """the fp32 emulation of the kernels' order passes every gate: noise, tones and DC through two CTA rows and both
    history branches, and the impulse answers"""
    P, h, x, xi, s = emu_case
    row = _all_gates(emulate(x, h, P, EMU_SCHED), emulate(xi, h, P, [xi.size]), emu_case)
    assert row["bound_used"] < 0.05, row


@pytest.mark.parametrize("fault", ["hist_late", "tap", "row2", "mirror", "swap"])
def test_gates_see_faults(emu_case, fault):
    """history one output time late, one edge tap dropped (p = 120 of 127), the second CTA row shifted, channels
    mirrored, re and im swapped in one branch: each fails the gates.  The dropped taps (near 1e-7) hide under the bound of
    a full window; they fail it on the start-up outputs, where the edge taps alone see data, and every impulse answer."""
    P, h, x, xi, s = emu_case
    isched = [s[3] - s[3] % M, xi.size - (s[3] - s[3] % M)]       # two calls: the impulse stream crosses a history
    with pytest.raises(AssertionError):
        _all_gates(emulate(x, h, P, EMU_SCHED, fault), emulate(xi, h, P, isched, fault), emu_case)


# ---------------------------------------------------------------------------------------------- GPU half
@pytest.fixture(scope="module")
def L():
    from sdrplusplus_b200 import lib
    l = lib.load()
    assert l.b200_device_count() > 0
    assert l.b200_init(0) == 0
    return l


class Chan:
    """one b200_chan handle; process() takes and returns numpy arrays, through the memory kinds asked for"""

    def __init__(self, L, P, max_chunk):
        self.L, self.P, self.max_chunk = L, P, max_chunk
        self.h = L.b200_chan_create(M, P, max_chunk)
        assert self.h, L.b200_last_error()
        self.pin = []

    def _pinned(self, n):
        for ptr, cap in self.pin:
            if cap >= n and ptr not in self._used:
                self._used.add(ptr)
                return ptr
        ptr = self.L.b200_host_alloc(8 * n)
        assert ptr
        self.pin.append((ptr, n))
        self._used.add(ptr)
        return ptr

    def process(self, x, kind=("host", "host")):
        import torch
        self._used = set()
        n = x.size
        x = np.ascontiguousarray(x, np.complex64)
        ik, ok = kind
        if ik == "host":
            src, imem = x.ctypes.data, 0
        elif ik == "pinned":
            src, imem = self._pinned(max(n, 1)), 0
            C.memmove(src, x.ctypes.data, 8 * n)
        else:
            xt = torch.from_numpy(x.view(np.float32).copy()).cuda()
            src, imem = xt.data_ptr(), 1
        if ok == "host":
            y = np.empty(n, np.complex64)
            dst, omem = y.ctypes.data, 0
        elif ok == "pinned":
            dst, omem = self._pinned(max(n, 1)), 0
        else:
            yt = torch.empty(2 * max(n, 1), dtype=torch.float32, device="cuda")
            dst, omem = yt.data_ptr(), 1
        torch.cuda.synchronize()
        r = self.L.b200_chan_process(self.h, src, n, imem, dst, omem)
        assert r == n // M, (r, self.L.b200_last_error())
        if ok == "pinned":
            y = np.empty(n, np.complex64)
            C.memmove(y.ctypes.data, dst, 8 * n)
        elif ok == "device":
            y = yt[:2 * n].cpu().numpy().view(np.complex64)
        return y.reshape(-1, M)

    def launches(self):
        return self.L.b200_chan_launch_count(self.h)

    def prototype(self):
        T = self.L.b200_chan_prototype(self.h, None, 0)
        h = np.empty(max(T, 1), np.float32)
        assert self.L.b200_chan_prototype(self.h, h.ctypes.data, h.size) == T
        return h[:T]

    def close(self):
        self.L.b200_chan_destroy(self.h)
        for ptr, _ in self.pin:
            self.L.b200_host_free(ptr)
        self.pin = []


def run_schedule(ch, x, sched, kinds=None):
    """feeds x by sched; checks each call's launches against the mirror; returns the outputs (n_out, M)"""
    outs, pos = [], 0
    for i, c in enumerate(sched):
        l0 = ch.launches()
        y = ch.process(x[pos:pos + c], kinds[i] if kinds else ("host", "host"))
        assert ch.launches() - l0 == launches_of(c, ch.P), (c, ch.P, ch.launches() - l0)
        outs.append(y)
        pos += c
    assert pos == x.size
    return np.concatenate(outs)


def _bits_equal(a, b, what):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    va, vb = a.view(np.uint64), b.view(np.uint64)
    bad = np.argwhere(va != vb)
    assert bad.size == 0, "%s: %d outputs differ, first (m, k) = %s" % (what, len(bad), tuple(bad[0]))


def _name(P):
    br = "+".join(sorted({history_branch(c, P) for c in seam_schedule(P)} - {None}))
    no = ",".join(str(c // M) for c in seam_schedule(P) if c // M in (257, 4095, 4099))
    return "P%d-%s-nout%s" % (P, br, no)


@pytest.mark.gpu
@pytest.mark.parametrize("P", P_SWEEP)
def test_prototype_pinned_to_oracle(L, oracle, P):
    """b200_chan_prototype returns T taps, bit-identical to the oracle's windowed sinc, with DC gain 1 where the main lobe
    fits (P >= 7; P = 1 and 2 truncate it: their sum is the float64 formula's)"""
    T = M * P
    ch = Chan(L, P, M)
    try:
        h = ch.prototype()
    finally:
        ch.close()
    assert h.size == T
    ref = oracle.lowpass(FS / 512.0, 3.8 * FS / T, FS)
    assert ref.size == T
    assert np.array_equal(ref.view(np.uint32), h.view(np.uint32))
    s = float(np.sum(h.astype(np.float64)))
    s64 = float(np.sum(prototype_f64(P)))
    assert abs(s - s64) <= T * U * float(np.sum(np.abs(h.astype(np.float64)))), (s, s64)
    if P >= 7:
        assert abs(s - 1.0) < 5e-4, s


@pytest.mark.gpu
@pytest.mark.parametrize("P", P_SWEEP, ids=[_name(P) for P in P_SWEEP])
def test_every_output_across_every_seam(L, report, P):
    """every output from output 0 against the bound, on the seam schedule with every (in, out) memory kind; the bits equal
    one call over the whole stream; launches match the mirror"""
    sched = seam_schedule(P)
    x = stream_input(sum(sched), 1000 + P)
    ch = Chan(L, P, MAX_N4099)
    try:
        h = ch.prototype()
        y = run_schedule(ch, x, sched, mem_kinds(len(sched)))
    finally:
        ch.close()
    one = Chan(L, P, x.size)
    try:
        y1 = run_schedule(one, x, [x.size])
    finally:
        one.close()
    _bits_equal(y, y1, "P=%d schedule vs one call" % P)
    st = Stats(P)
    check_stream(y, x, h, P, st, "P=%d" % P)
    report["channelizer_f64_" + _name(P)] = dict(st.row(), schedule=sched)


@pytest.mark.gpu
def test_c3_bench_shape_256x127_1Mi_device(L, report):
    """the bench's C3 leg: 256 x 127, max_chunk 1 Mi, four 1 Mi-sample chunks, torch device tensors in and out; every output
    against the bound, and the bits of the same stream fed from host memory over the seam schedule"""
    import torch
    P, n = 127, 4 * MI
    x = stream_input(n, 0xC3)
    ch = Chan(L, P, MI)
    try:
        h = ch.prototype()
        xt = torch.from_numpy(x.view(np.float32).copy()).cuda()
        yt = torch.empty(2 * MI, dtype=torch.float32, device="cuda")
        outs = []
        torch.cuda.synchronize()
        for c in range(0, n, MI):
            l0 = ch.launches()
            assert L.b200_chan_process(ch.h, xt.data_ptr() + 8 * c, MI, 1, yt.data_ptr(), 1) == MI // M
            assert ch.launches() - l0 == launches_of(MI, P)
            outs.append(yt.cpu().numpy().view(np.complex64).reshape(-1, M).copy())
        y = np.concatenate(outs)
    finally:
        ch.close()
    sched = seam_schedule(P, MI)
    while sum(sched) < n:
        sched.append(min(MI, n - sum(sched)))
    ch2 = Chan(L, P, MI)
    try:
        y2 = run_schedule(ch2, x, sched)
    finally:
        ch2.close()
    _bits_equal(y, y2, "bench shape: device 1 Mi chunks vs host seam schedule")
    st = Stats(P)
    check_stream(y, x, h, P, st, "c3 bench shape")
    report["channelizer_f64_c3_bench_256x127_1Mi"] = st.row()


@pytest.mark.gpu
@pytest.mark.parametrize("P", KA_P)
def test_impulse_answers_pin_every_tap(L, report, P):
    """one impulse per residue (all 256), T + 1 or more apart, a chunk starting on one and a chunk ending on another: every
    tap of every branch in place within the known-answer bound, every other output exactly 0"""
    x, s = impulse_stream(P, range(M), P)
    sched = impulse_schedule(P, s, x.size, MAX_N4099, P)
    ch = Chan(L, P, MAX_N4099)
    try:
        h = ch.prototype()
        y = run_schedule(ch, x, sched, mem_kinds(len(sched)))
    finally:
        ch.close()
    st = Stats(P)
    check_impulses(y, s, h, P, st, "P=%d impulses" % P)
    report["channelizer_f64_impulses_P%d" % P] = {"ka_used": st.frac, "outputs": st.outputs, "calls": len(sched)}


@pytest.mark.gpu
def test_interleaved_handles_keep_their_own_bits(L):
    """two handles (P = 127 and P = 9) called alternately each give the bits they give alone"""
    cfg = [(127, MAX_N4099, [MI, 256, 512 * M, hist_of(127) - 256, 4099 * M]),
           (9, 65792, [65792, 256, 2048, 0, hist_of(9), 255 * M])]
    xs = [stream_input(sum(s), 50 + P) for P, _, s in cfg]
    alone = []
    for (P, mc, s), x in zip(cfg, xs):
        ch = Chan(L, P, mc)
        try:
            alone.append(run_schedule(ch, x, s))
        finally:
            ch.close()
    chs = [Chan(L, P, mc) for P, mc, _ in cfg]
    try:
        outs, pos = [[], []], [0, 0]
        for i in range(max(len(s) for _, _, s in cfg)):
            for j, (P, mc, s) in enumerate(cfg):
                if i < len(s):
                    outs[j].append(chs[j].process(xs[j][pos[j]:pos[j] + s[i]], mem_kinds(9)[(i + j) % 9]))
                    pos[j] += s[i]
    finally:
        for c in chs:
            c.close()
    for j in range(2):
        _bits_equal(np.concatenate(outs[j]), alone[j], "interleaved handle %d" % j)


@pytest.mark.gpu
def test_rejections_leave_no_trace(L):
    """b200_chan_create refuses bad shapes with a message; b200_chan_process refuses bad counts (B200_ECAP) and null
    arguments (B200_EINVAL) without launching, and the stream after them has the bits of one that never saw them"""
    for args in [(255, 127, 64 * M), (257, 127, 64 * M), (256, 0, 64 * M), (256, 256, 64 * M), (256, 127, 0),
                 (256, 127, 255), (256, 127, 257)]:
        assert L.b200_chan_process(None, None, 0, 0, None, 0) == B200_EINVAL      # leaves "null argument" behind
        assert not L.b200_chan_create(*args), args
        assert b"channelizer" in L.b200_last_error(), (args, L.b200_last_error())
    P, mc = 127, 512 * M
    sched = [256, 300 * M, 512 * M, 256, hist_of(P)]
    x = stream_input(sum(sched), 77)
    ref = Chan(L, P, mc)
    try:
        y_ref = run_schedule(ref, x, sched)
    finally:
        ref.close()
    ch = Chan(L, P, mc)
    junk = np.ones(mc + M, np.complex64)
    out = np.empty(mc + M, np.complex64)
    bad = [(lambda: L.b200_chan_process(ch.h, junk.ctypes.data, 255, 0, out.ctypes.data, 0), B200_ECAP),
           (lambda: L.b200_chan_process(ch.h, junk.ctypes.data, -256, 0, out.ctypes.data, 0), B200_ECAP),
           (lambda: L.b200_chan_process(ch.h, junk.ctypes.data, mc + M, 0, out.ctypes.data, 0), B200_ECAP),
           (lambda: L.b200_chan_process(None, junk.ctypes.data, 256, 0, out.ctypes.data, 0), B200_EINVAL),
           (lambda: L.b200_chan_process(ch.h, None, 256, 0, out.ctypes.data, 0), B200_EINVAL),
           (lambda: L.b200_chan_process(ch.h, junk.ctypes.data, 256, 0, None, 0), B200_EINVAL)]
    try:
        outs, pos = [], 0
        for i, c in enumerate(sched):
            for f, code in bad if i < len(sched) - 1 else []:
                l0 = ch.launches()
                assert f() == code
                assert ch.launches() == l0
            l0 = ch.launches()
            outs.append(ch.process(x[pos:pos + c]))
            assert ch.launches() - l0 == launches_of(c, P)
            pos += c
    finally:
        ch.close()
    _bits_equal(np.concatenate(outs), y_ref, "after rejected calls")

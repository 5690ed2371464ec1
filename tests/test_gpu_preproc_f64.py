"""The front end's pre-processing chain (input PowerDecimator -> full-rate DCBlocker<complex_t> -> Conjugate, preproc.cuh)
against a float64 reference, sample by sample, from output 0 of the stream: the blocker's three-pass parallel scan at every
launch geometry up to the bench's chunk size, every ingest format and scale, every decimator plan family, state changes
between chunks, bit-exact known answers, and stage 1 behind the chain.  The output is read from a CF32 IQ tap, which
test_gpu_iq_tap.py shows to be bit-exact to the stream it reads.

Input.  The blocker's input x is taken as exact values: cf32 samples as they are; integer samples as fl32(fl32(v) * scale)
with the chunk's fp32 ingest scale (one rounding of the product, which the reference and the library share); behind the
decimator, the float64 cascade of the plan's taps (f64_ref.fir_f64 with its per-sample bound e_x).

Recurrence.  r = fl32(50 / fs_eff), the value the library and the reference both use.  In float64 o[i+1] = (1 - r) o[i] +
r x[i], y[i] = x[i] - o[i] (scipy.signal.lfilter), conjugated on output when the conjugate is on.  o starts at 0 at the start
of the stream and after reset(); a chunk with the blocker off passes x unchanged and leaves o as it was.

Bound, per component (the maps o -> (1 - c) o + b have a real slope, so re and im never mix), for every output:
  * the offset k_dcb_apply uses at sample i is the carried offset put through a tree of fp32 steps, compositions and
    applications.  Its depth from any leaf is at most P = 16 + 13 + (2 per + 10) + 13 + 16: up to DCB_RUN steps and 5 + 8
    compositions in k_dcb_reduce, per + 10 + per in k_dcb_scan, 5 + 8 compositions and up to DCB_RUN steps in k_dcb_apply,
    per = ceil(nseg / 1024) and nseg = ceil(n / 4096);
  * every value a node rounds is bounded by X = max |x| of the stream so far: o and every map's b are convex combinations of
    0 and earlier x, and |b| <= c X.  A step (c' = c + r - c r, b' = b + (x - b) r) rounds c' to 3 u c' and b' to
    u (2 r X + 2 r X + c' X); a composition rounds c to 3 u c and b to 3 u c X; an application o' = o - c o + b rounds to
    3 u X; a step of the apply walk (y = x - o, o += y r) to (1 + 4 r) u X <= 3 u X.  A node's error in c moves the result
    by at most that error times X.  So every node adds at most kappa u c_node X with kappa = 8 (c_node = 1 for an
    application or a walk step);
  * every later operation contracts (|1 - c| <= 1), and the nodes of one tree level cover disjoint runs of samples, so an
    error of a node reaches the root multiplied by the product of (1 - c) of the later runs: summed over one level,
    sum_j c_j prod_{l > j} (1 - c_l) = 1 - prod_j (1 - c_j) <= 1.  Each level adds at most kappa u X, and there are P levels.
Hence |o_hat_i - o_i| <= E_k + kappa P u X inside chunk k, where E_{k+1} = (1 - r)^{n_k} E_k + kappa P u X carries the
chunk-end error (E = 0 at the start and after reset(); a chunk with the blocker off leaves it).  On top of that come the
propagated input error e_x + lfilter([0, r], [1, -(1 - r)], e_x), the output subtraction's rounding u |y_hat|, and the float64
recursion's own error 4 2^-53 X / r.  The recursion is evaluated on each case's own chunk schedule: many tiny chunks at a
small r make it loose, and the report shows the used fraction.

Pinning.  On the CPU the reference is pinned to the oracle's fp32 dcblock_c (the reference's sequential loop, whose errors
add along the whole stream: sum_j (1 - r)^{i - j} 3 u X) and decim blocks, and the bound is shown not to be blind to an
offset one sample early.

Gates for each GPU case: every component of every output within its bound, from output 0; for cases with at least 1000
interior outputs, the fitted complex gain against float64 within 1e-6 of 1 (this sees a wrong ingest scale) and the largest
error within 64 outputs of a chunk start or a 4096-sample segment start at most 4x the interior 99.9th percentile.
Nothing here is fitted to a run.
"""
import numpy as np
import pytest
from scipy.signal import lfilter

from f64_ref import U, cascade_counts, fir_f64, pfb_detect, pfb_eps, plan_of, schedule, stage1_f64, w_u64, drift_weights

DCB_RUN, DCB_THREADS = 16, 256                  # preproc.cuh
DCB_SEG = DCB_RUN * DCB_THREADS
SCAN_THREADS = 1024                             # k_dcb_scan's CTA
KAPPA = 8                                       # module docstring: per tree level, in u X
EDGE = 64
CF32, CS16, CS8 = 0, 1, 2
U53 = 2.0 ** -53


# ---------------------------------------------------------------------------------------------- mirrors of the host code
def dcb_geometry(n):
    """launch_preproc / b200_fe_submit: (nseg, per) of a blocker chunk of n samples"""
    nseg = -(-n // DCB_SEG)
    return nseg, -(-nseg // SCAN_THREADS)


def dcb_depth(n):
    return 16 + 13 + (2 * dcb_geometry(n)[1] + 10) + 13 + 16


def preproc_launches(n, dc_on, conj_on):
    """launches the pre-processing block adds for one chunk of n effective samples, without decimation: k_dcb_reduce,
    k_dcb_scan and k_dcb_apply with the blocker on, k_dcb_apply alone for the conjugate, nothing for an empty chunk"""
    if n <= 0 or not (dc_on or conj_on):
        return 0
    return 3 if dc_on else 1


def rate_of(fs_eff):
    return float(np.float32(50.0 / fs_eff))


# ---------------------------------------------------------------------------------------------- float64 reference
class DcbModel:
    """the blocker and the conjugate in float64, chunk by chunk, with the bound of the module docstring"""

    def __init__(self, r):
        self.r = r
        self.reset()
        self.X = 0.0

    def reset(self):
        self.o, self.eo, self.E = 0j, 0.0, 0.0

    def chunk(self, x, ex=None, dc=True, conj=False):
        """x: exact input (complex128), ex: per-sample bound of x's error (None: exact).  Returns (y64, bound)."""
        n = x.size
        ex = np.zeros(n) if ex is None else np.asarray(ex, np.float64)
        if n == 0:
            return np.zeros(0, np.complex128), np.zeros(0)
        ax = np.maximum(np.abs(x.real), np.abs(x.imag))
        self.X = max(self.X, float((ax + ex).max()))
        if not dc:
            y, b = x.copy(), ex.copy()
        else:
            r = self.r
            o, zf = lfilter([0.0, r], [1.0, -(1.0 - r)], x, zi=np.array([self.o], np.complex128))
            eo, zfe = lfilter([0.0, r], [1.0, -(1.0 - r)], ex, zi=np.array([self.eo]))
            self.o, self.eo = complex(zf[0]), float(zfe[0])
            rnd = KAPPA * dcb_depth(n) * U * self.X
            d = self.E + rnd + 4.0 * U53 * self.X / r
            self.E = (1.0 - r) ** n * self.E + rnd
            ao = np.maximum(np.abs(o.real), np.abs(o.imag))
            e = ex + eo + d
            y = x - o
            b = e + U * (ax + ao + e)
        return (np.conj(y) if conj else y), b


def dcb_seq_bound(x, r, sched):
    """the reference's sequential fp32 loop against float64: each step adds (1 + 4 r) u X <= 3 u X to the offset and the
    errors decay with (1 - r); the output adds u |y|"""
    X = float(np.maximum(np.abs(x.real), np.abs(x.imag)).max())
    o = lfilter([0.0, r], [1.0, -(1.0 - r)], x)
    d = lfilter([0.0, 1.0], [1.0, -(1.0 - r)], np.full(x.size, 3.0 * U * X)) + 4.0 * U53 * X / r
    ax = np.maximum(np.abs(x.real), np.abs(x.imag))
    ao = np.maximum(np.abs(o.real), np.abs(o.imag))
    return x - o, d + U * (ax + ao + d)


def ratio_c(y, y64, b):
    """per-sample max-component error over the bound (an exact answer with a zero bound counts as 0)"""
    y = np.asarray(y).astype(np.complex128)
    err = np.maximum(np.abs(y.real - y64.real), np.abs(y.imag - y64.imag))
    return np.where(b > 0, err / np.where(b > 0, b, 1.0), np.where(err == 0, 0.0, np.inf))


def decim_f64(oracle, x, ratio):
    """the PowerDecimator's cascade in float64 from zero history: (y, per-sample bound)"""
    e = None
    for D, h in plan_of(oracle, ratio):
        x, e = fir_f64(x, e, h, D)
    return x, e


def decim_counts(oracle, sched, ratio):
    return cascade_counts(sched, [("fir", D) for D, _ in plan_of(oracle, ratio)])


# ---------------------------------------------------------------------------------------------- inputs
def make_chunk(rng, n, fmt, scale=None, dc=0.25 - 0.125j):
    """(data for FrontEnd.process, exact complex128 value): uniform noise plus a DC the blocker removes"""
    if fmt == CF32:
        c = (rng.uniform(-0.6, 0.6, 2 * n).astype(np.float32).view(np.complex64) + np.complex64(dc)).astype(np.complex64)
        return c, c.astype(np.complex128)
    lim = 32768 if fmt == CS16 else 128
    v = rng.integers(-lim // 2, lim // 2, 2 * n) + np.tile([int(dc.real * lim), int(dc.imag * lim)], n)
    c = np.clip(v, -lim, lim - 1).astype(np.int16 if fmt == CS16 else np.int8)
    sc = np.float32(scale) if scale else np.float32(1.0 / lim)
    f = c.astype(np.float32) * sc
    return c, f.astype(np.float64).view(np.complex128)


# ---------------------------------------------------------------------------------------------- GPU case definitions
GEOM = [0, 1, 15, 16, 17, 4095, 4096, 4097, 4097, 1, 16, 1024 * 4096, 1024 * 4096 + 1, 1024 * 4096 + 1,
        3 * 1024 * 4096 + 5 * 4096 + 7, 17, 3 * 1024 * 4096 + 5 * 4096 + 7, 0, 15]
PROD = [1 << 24, (1 << 25) + 12345, 1, 4097, 777777, 15, 3 * 65536 + 5]


def _fmt_sched(name):
    """(sizes, formats, scales) of the format cases (no decimation, 3200 S/s: r = 1/64)"""
    sizes = [5000, 4097, 12289, 1, 70001, 16, 33333, 8191]
    k = len(sizes)
    if name == "cs16":
        return sizes, [CS16] * k, [None] * k
    if name == "cs8":
        return sizes, [CS8] * k, [None] * k
    if name == "cs16_scale":
        return sizes, [CS16] * k, [3.1e-5] * k
    if name == "cs8_scale":
        return sizes, [CS8] * k, [0.0071] * k
    if name == "cs16_scales":
        return sizes, [CS16] * k, [(None, 2.7e-5, 4.1e-5, 1e-3)[i % 4] for i in range(k)]
    if name == "mixfmt":
        return sizes, [(CF32, CS16, CS8)[i % 3] for i in range(k)], [(None, 2.9e-5, 0.0093)[i % 3] for i in range(k)]
    raise KeyError(name)


FMT_CASES = ["cs16", "cs8", "cs16_scale", "cs8_scale", "cs16_scales", "mixfmt"]
DECIM_RATIOS = [2, 4, 64, 8192]
DECIM_MODES = ["dc", "dc_conj", "off"]


def _decim_sched(ratio):
    total = max(300000, 1100 * ratio)
    s = [1, ratio - 1, 3, ratio, ratio + 1, 0, 7 * ratio + 5, max(1, ratio // 2), 4097]
    big = min(1 << 20, max(60001, 97 * ratio + 3))
    while sum(s) + big < total:
        s.append(big)
        s.append(int(ratio * 3 + 11))
    s.append(max(1, total - sum(s)))
    return s


# ---------------------------------------------------------------------------------------------- CPU part
@pytest.mark.parametrize("r,sched", [(1.0 / 64, [1, 15, 16, 17, 4095, 4097, 20000, 3, 9000]),
                                     (rate_of(2.4e6), schedule(4096, 16, 200000)),
                                     (0.5, [7, 4096, 1, 30000])])
def test_reference_matches_oracle_blocker(oracle, report, r, sched):
    """the float64 recursion against the reference's sequential fp32 loop (the oracle's dcblock_c, chunked the same way),
    every output within the loop's own bound; and the bound is not blind to an offset one sample early"""
    n = sum(sched)
    rng = np.random.default_rng(int(r * 1e6) % 1000)
    x32 = (rng.uniform(-0.6, 0.6, 2 * n).astype(np.float32).view(np.complex64) + np.complex64(0.25 - 0.125j))
    x = x32.astype(np.complex128)
    blk = oracle.dcblock_c(r)
    parts, pos = [], 0
    for c in sched:
        parts.append(blk.process(x32[pos:pos + c].view(np.float32)).view(np.complex64))
        pos += c
    y = np.concatenate(parts)
    y64, b = dcb_seq_bound(x, r, sched)
    m = DcbModel(r)
    ym = np.concatenate([m.chunk(x[p:p + c])[0] for p, c in zip(np.cumsum([0] + sched[:-1]), sched)])
    assert np.allclose(ym, y64, rtol=0, atol=1e-12)
    used = float(ratio_c(y, y64, b).max())
    report["preproc_f64_pin_oracle_r%.3g" % r] = {"used_fraction": used, "outputs": int(n)}
    assert used <= 1.0, used
    # an offset one sample early: o[i] replaced by o[i+1]
    o = x - y64
    early = x - np.concatenate([o[1:], o[-1:]])
    if r >= 1.0 / 64:
        assert float(ratio_c(early, y64, b).max()) > 1.0


def test_blocker_bound_covers_fp32_tree():
    """a float32 emulation of the three passes (run maps, tree composition in the CTA, sequential per-thread scan) on one
    chunk at 1/64 and 1/2 stays within the model's bound: the bound is not tighter than the arithmetic it describes"""
    for r in (1.0 / 64, 0.5, rate_of(100e6)):
        rng = np.random.default_rng(3)
        n = 5 * DCB_SEG + 77
        x32 = (rng.uniform(-0.6, 0.6, 2 * n).astype(np.float32).view(np.complex64) + np.complex64(0.25 - 0.125j))
        y = _emulate_fp32(x32, np.float32(r))
        y64, b = DcbModel(r).chunk(x32.astype(np.complex128))
        assert float(ratio_c(y, y64, b).max()) <= 1.0


def _emulate_fp32(x, r):
    """numpy float32 emulation of k_dcb_reduce / k_dcb_scan / k_dcb_apply for one chunk from zero state (one CTA scan
    thread per segment, a Hillis-Steele tree over the runs of a segment)"""
    f = np.float32
    n = x.size
    nseg = -(-n // DCB_SEG)
    xp = np.zeros(nseg * DCB_SEG, np.complex64)
    xp[:n] = x
    xr = xp.reshape(nseg, DCB_THREADS, DCB_RUN)
    valid = (np.arange(nseg * DCB_SEG) < n).reshape(nseg, DCB_THREADS, DCB_RUN)
    c = np.zeros((nseg, DCB_THREADS), f)
    bre, bim = np.zeros((nseg, DCB_THREADS), f), np.zeros((nseg, DCB_THREADS), f)
    for k in range(DCB_RUN):
        v = valid[:, :, k]
        xk = xr[:, :, k]
        cn = f(c + r) - f(c * r)
        bre = np.where(v, bre + f(f(xk.real - bre) * r), bre).astype(f)
        bim = np.where(v, bim + f(f(xk.imag - bim) * r), bim).astype(f)
        c = np.where(v, cn, c).astype(f)

    def comp(c1, b1r, b1i, c2, b2r, b2i):          # then(first)
        return (f(f(c1 + c2) - f(c1 * c2)), f(f(b1r - f(c2 * b1r)) + b2r), f(f(b1i - f(c2 * b1i)) + b2i))
    ic, ir, ii = c.copy(), bre.copy(), bim.copy()  # inclusive scan over the runs of each segment
    d = 1
    while d < DCB_THREADS:
        pc = np.concatenate([np.zeros((nseg, d), f), ic[:, :-d]], 1)
        pr = np.concatenate([np.zeros((nseg, d), f), ir[:, :-d]], 1)
        pi = np.concatenate([np.zeros((nseg, d), f), ii[:, :-d]], 1)
        ic, ir, ii = comp(pc, pr, pi, ic, ir, ii)
        d *= 2
    seg = np.zeros(nseg, np.complex128)
    o = np.complex64(0)
    for s in range(nseg):                          # segment-start offsets, sequentially
        seg[s] = o
        o = np.complex64(complex(f(f(o.real - f(ic[s, -1] * o.real)) + ir[s, -1]), f(f(o.imag - f(ic[s, -1] * o.imag)) + ii[s, -1])))
    out = np.zeros(nseg * DCB_SEG, np.complex64)
    for s in range(nseg):
        ec = np.concatenate([[f(0)], ic[s, :-1]]).astype(f)
        er = np.concatenate([[f(0)], ir[s, :-1]]).astype(f)
        ei = np.concatenate([[f(0)], ii[s, :-1]]).astype(f)
        ore = f(f(f(seg[s].real) - f(ec * f(seg[s].real))) + er)
        oim = f(f(f(seg[s].imag) - f(ec * f(seg[s].imag))) + ei)
        for k in range(DCB_RUN):
            xk = xr[s, :, k]
            yr, yi = f(xk.real - ore), f(xk.imag - oim)
            out.reshape(nseg, DCB_THREADS, DCB_RUN)[s, :, k] = (yr + 1j * yi).astype(np.complex64)
            ore, oim = f(ore + f(yr * r)), f(oim + f(yi * r))
    return out[:n]


@pytest.mark.parametrize("ratio", [2, 4, 64, 8192])
def test_reference_matches_oracle_decimator(oracle, report, ratio):
    """the float64 cascade of the plan's taps against the oracle's PowerDecimator, chunked the ragged way the GPU cases are,
    cs16 at a scale that is not a power of two: per-chunk counts equal and every output within the cascade's bound"""
    sched = _decim_sched(ratio)[:12] if ratio == 8192 else _decim_sched(ratio)
    n = sum(sched)
    rng = np.random.default_rng(ratio)
    data, x = make_chunk(rng, n, CS16, 3.1e-5)
    blk = oracle.decim(ratio)
    xf = x.astype(np.complex64)
    parts, pos = [], 0
    for c in sched:
        parts.append(blk.process(xf[pos:pos + c].view(np.float32)).view(np.complex64))
        pos += c
    assert [p.size for p in parts] == decim_counts(oracle, sched, ratio)
    y64, b = decim_f64(oracle, x, ratio)
    y = np.concatenate(parts)
    assert y.size == y64.size
    used = float(ratio_c(y, y64, b).max())
    report["preproc_f64_pin_oracle_decim%d" % ratio] = {"used_fraction": used, "outputs": int(y.size)}
    assert used <= 1.0, used


def test_mirror_launch_geometry():
    """launch_preproc's geometry at the named edges, and the launches of the pre-processing block"""
    assert dcb_geometry(1) == (1, 1) and dcb_geometry(4096) == (1, 1) and dcb_geometry(4097) == (2, 1)
    assert dcb_geometry(1024 * 4096) == (1024, 1) and dcb_geometry(1024 * 4096 + 1) == (1025, 2)
    assert dcb_geometry(1 << 24) == (4096, 4)
    assert dcb_geometry((1 << 25) + 12345) == (8196, 9)
    assert dcb_geometry(3 * 1024 * 4096 + 5 * 4096 + 7) == (3078, 4)
    assert [preproc_launches(n, d, c) for n, d, c in [(5, 1, 0), (5, 0, 1), (5, 1, 1), (0, 1, 1), (5, 0, 0)]] == [3, 1, 3, 0, 0]


def _blocker_counts(oracle):
    """every blocker chunk size the GPU cases feed"""
    out = list(GEOM) + list(PROD) + schedule(4096, 16, 400000)
    for name in FMT_CASES:
        out += _fmt_sched(name)[0]
    for ratio in DECIM_RATIOS:
        out += decim_counts(oracle, _decim_sched(ratio), ratio)
    return out


def test_gpu_cases_reach_their_geometry(oracle):
    """the GPU cases reach nseg 1, 1024 and 1025, per 1, 2 and >= 4 with a ragged last scan thread, counts that are not a
    multiple of DCB_RUN, and decimated chunks with no output"""
    counts = [n for n in _blocker_counts(oracle)]
    geo = [dcb_geometry(n) for n in counts if n > 0]
    nsegs, pers = {g[0] for g in geo}, {g[1] for g in geo}
    assert {1, 1024, 1025} <= nsegs
    assert {1, 2} <= pers and max(pers) >= 9
    assert any(p >= 4 and s % p for s, p in geo)
    assert any(n % DCB_RUN for n in counts if n > DCB_SEG)
    assert 0 in counts
    for ratio in DECIM_RATIOS:
        assert 0 in decim_counts(oracle, _decim_sched(ratio), ratio)


# ---------------------------------------------------------------------------------------------- GPU part
@pytest.fixture(scope="module")
def sb():
    import sdrplusplus_b200 as m
    from sdrplusplus_b200 import lib
    L = lib.load()
    assert L.b200_device_count() > 0
    assert L.b200_init(0) == 0
    return m


class Gate:
    """accumulates one case's outputs against the reference: used fraction of the bound, fitted gain, edge ratio"""

    def __init__(self):
        self.worst, self.vv, self.vy, self.n = 0.0, 0j, 0j, 0
        self.err, self.edge, self.pow = [], [], 0.0

    def add(self, y, y64, b, seg_edges=True):
        assert y.size == y64.size, (y.size, y64.size)
        if y.size == 0:
            return
        rr = ratio_c(y, y64, b)
        k = int(np.argmax(rr))
        self.worst = max(self.worst, float(rr[k]))
        assert rr[k] <= 1.0, (self.n + k, float(rr[k]), y[k], y64[k], b[k])
        yc = y.astype(np.complex128)
        self.vv += np.vdot(y64, y64)
        self.vy += np.vdot(y64, yc)
        self.pow += float(np.sum(np.abs(y64) ** 2))
        i = np.arange(y.size)
        ed = i < EDGE
        if seg_edges:
            ed |= (i % DCB_SEG) < EDGE
        ed |= i >= y.size - EDGE           # before the next chunk's start
        self.err.append(np.abs(yc - y64).astype(np.float32))
        self.edge.append(ed)
        self.n += y.size

    def finish(self):
        res = {"max_err_over_bound": self.worst, "outputs": self.n}
        if self.n == 0:
            return res
        err, edge = np.concatenate(self.err), np.concatenate(self.edge)
        if (~edge).sum() >= 1000:
            g = self.vy / self.vv
            res["abs_g_minus_1"] = float(abs(g - 1))
            assert abs(g - 1) <= 1e-6, g
            p999 = float(np.percentile(err[~edge], 99.9))
            em = float(err[edge].max())
            er = em / p999 if p999 > 0 else (0.0 if em == 0 else np.inf)
            res["edge_over_p999"] = er
            assert er <= 4.0, (er, em, p999)
        return res


def _fe(sb, fs, max_chunk, decim=1, dc=True, conj=False):
    fe = sb.FrontEnd(fs, max(1, max_chunk))
    if decim > 1:
        fe.set_decimation(decim)
    fe.set_dc_blocking(dc)
    fe.set_invert_iq(conj)
    tid = fe.bind_iq(sb.lib.IQ_CF32)
    return fe, tid


def _feed(fe, tid, data, fmt, scale):
    if fmt != CF32:
        fe.set_ingest_scale(fmt, scale or 0.0)
    l0 = fe.launch_count()
    outs, _ = fe.process(data, fmt)
    return outs[tid], fe.launch_count() - l0


def _run_stream(sb, fs, sizes, fmts=None, scales=None, dc=True, conj=False, twin=True, seed=0, edits=None, name=""):
    """no decimation: every chunk against the model, and each chunk's launches against a twin without pre-processing"""
    k = len(sizes)
    fmts, scales = fmts or [CF32] * k, scales or [None] * k
    edits = edits or {}
    fe, tid = _fe(sb, fs, max(sizes), 1, dc, conj)
    tw = _fe(sb, fs, max(sizes), 1, False, False) if twin else None
    model, gate = DcbModel(rate_of(fs)), Gate()
    rng = np.random.default_rng(seed)
    state = {"dc": dc, "conj": conj}
    try:
        for c, (n, f, s) in enumerate(zip(sizes, fmts, scales)):
            for key, v in edits.get(c, {}).items():
                state[key] = v
                (fe.set_dc_blocking if key == "dc" else fe.set_invert_iq)(v)
            data, x = make_chunk(rng, n, f, s)
            y, nl = _feed(fe, tid, data, f, s)
            y64, b = model.chunk(x, None, state["dc"], state["conj"])
            gate.add(y, y64, b)
            if not state["dc"]:
                want = np.conj(x.astype(np.complex64)) if state["conj"] else x.astype(np.complex64)
                assert y.tobytes() == want.tobytes(), c
            if tw is not None:
                _, nl0 = _feed(tw[0], tw[1], data, f, s)
                assert nl - nl0 == preproc_launches(n, state["dc"], state["conj"]), (c, n, nl, nl0)
    finally:
        fe.close()
        if tw is not None:
            tw[0].close()
    return gate.finish()


@pytest.mark.gpu
@pytest.mark.parametrize("fs", [3200.0, 100.0])
def test_scan_geometry_at_large_rate(sb, report, fs):
    """r = 1/64 and 1/2: a one-sample error in any offset is far above the bound.  Chunks of 0 .. 4097 samples, the last
    per = 1 chunk (1024 segments), the first per = 2 chunk (1025), an uneven per = 4 chunk, repeats of each"""
    res = _run_stream(sb, fs, GEOM, twin=True, seed=int(fs))
    report["preproc_f64_geometry_fs%d" % fs] = res


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["100M", "2M4"])
def test_production_rates(sb, report, name):
    """100 MS/s with one 16 Mi chunk (the bench's), then 2^25 + 12,345 (per 9), then ragged chunks; 2.4 MS/s on the shared
    chunk schedule, blocker and conjugate on"""
    if name == "100M":
        res = _run_stream(sb, 100e6, PROD, conj=True, twin=False, seed=11)
    else:
        res = _run_stream(sb, 2.4e6, schedule(4096, 16, 400000), conj=True, twin=True, seed=12)
    report["preproc_f64_rate_" + name] = res


@pytest.mark.gpu
@pytest.mark.parametrize("name", FMT_CASES)
def test_formats_into_the_blocker(sb, report, name):
    """cs16 / cs8 straight into k_dcb_reduce / k_dcb_apply (dcb_load with the ingest scale), at the default scale, at a
    scale that is not a power of two, with the scale changing every chunk, and the format changing between chunks"""
    sizes, fmts, scales = _fmt_sched(name)
    report["preproc_f64_fmt_" + name] = _run_stream(sb, 3200.0, sizes, fmts, scales, twin=True, seed=20 + FMT_CASES.index(name))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", DECIM_MODES)
@pytest.mark.parametrize("ratio", DECIM_RATIOS)
def test_decimation_then_blocker(sb, oracle, report, ratio, mode):
    """cs16 at scale 3.1e-5 through k_convert and every plan family of the PowerDecimator, then the blocker (r = 1/64),
    with and without the conjugate, or the decimator alone; ragged chunks, some shorter than the ratio (an empty blocker
    chunk).  Per-chunk output counts are the cascade's"""
    fs = 3200.0 * ratio
    sched = _decim_sched(ratio)
    dc, conj = mode != "off", mode == "dc_conj"
    rng = np.random.default_rng(ratio + len(mode))
    chunks = [make_chunk(rng, n, CS16, 3.1e-5) for n in sched]
    x = np.concatenate([c[1] for c in chunks])
    xd, ed = decim_f64(oracle, x, ratio)
    counts = decim_counts(oracle, sched, ratio)
    fe, tid = _fe(sb, fs, max(sched), ratio, dc, conj)
    model, gate = DcbModel(rate_of(fs / ratio)), Gate()
    got = []
    try:
        pos = 0
        for (data, _), m in zip(chunks, counts):
            y, _ = _feed(fe, tid, data, CS16, 3.1e-5)
            got.append(y.size)
            y64, b = model.chunk(xd[pos:pos + m], ed[pos:pos + m], dc, conj)
            gate.add(y, y64, b)
            pos += m
    finally:
        fe.close()
    assert got == counts
    report["preproc_f64_decim%d_%s" % (ratio, mode)] = gate.finish()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["dc_on_off_on", "conj_on_off", "dc_off_first"])
def test_changes_between_chunks(sb, report, name):
    """the blocker switched off keeps its offset (not decayed) and passes x bit for bit; the conjugate switched off; each
    change followed by a short chunk"""
    sizes = [50001, 30000, 7, 40000, 3, 9000]
    if name == "dc_on_off_on":
        edits = {1: {"dc": False}, 2: {"dc": True}, 4: {"dc": False}, 5: {"dc": True}}
        res = _run_stream(sb, 3200.0, sizes, dc=True, edits=edits, seed=31)
    elif name == "conj_on_off":
        edits = {1: {"conj": False}, 2: {"conj": True}, 3: {"conj": False}}
        res = _run_stream(sb, 3200.0, sizes, dc=True, conj=True, edits=edits, seed=32)
    else:
        edits = {2: {"dc": True}, 3: {"conj": True}}
        res = _run_stream(sb, 3200.0, sizes, dc=False, edits=edits, seed=33)
    report["preproc_f64_change_" + name] = res


@pytest.mark.gpu
def test_reset_mid_stream(sb, oracle):
    """reset() with decimation 4 and the blocker on: from there the outputs equal a fresh front end's, bit for bit (the
    blocker's offset and the decimator's history are both cleared)"""
    fs, ratio = 12800.0, 4
    rng = np.random.default_rng(41)
    a = [make_chunk(rng, n, CS16, 3.1e-5)[0] for n in (30001, 4097, 2)]
    b = [make_chunk(rng, n, CS16, 3.1e-5)[0] for n in (5, 20003, 4097)]
    fe, tid = _fe(sb, fs, 30001, ratio, True, True)
    fresh, tid2 = _fe(sb, fs, 30001, ratio, True, True)
    try:
        for d in a:
            _feed(fe, tid, d, CS16, 3.1e-5)
        fe.reset()
        for d in b:
            y1, _ = _feed(fe, tid, d, CS16, 3.1e-5)
            y2, _ = _feed(fresh, tid2, d, CS16, 3.1e-5)
            assert y1.tobytes() == y2.tobytes()
    finally:
        fe.close()
        fresh.close()


IMPULSE_AT = {  # name: (chunk length, position)
    "run_first": (3 * DCB_SEG + 17, 2 * DCB_RUN), "run_last": (3 * DCB_SEG + 17, 3 * DCB_RUN - 1),
    "thread31_last": (3 * DCB_SEG + 17, 32 * DCB_RUN - 1), "thread32_first": (3 * DCB_SEG + 17, 32 * DCB_RUN),
    "thread127_last": (3 * DCB_SEG + 17, 128 * DCB_RUN - 1), "thread128_first": (3 * DCB_SEG + 17, 128 * DCB_RUN),
    "seg_first": (3 * DCB_SEG + 17, DCB_SEG), "seg_last": (3 * DCB_SEG + 17, 2 * DCB_SEG - 1),
    "chunk_first": (3 * DCB_SEG + 17, 0), "chunk_last": (3 * DCB_SEG + 17, 3 * DCB_SEG + 16),
    "seg1025": (1025 * DCB_SEG + 33, 1024 * DCB_SEG + 100), "seg1025_last": (1025 * DCB_SEG + 33, 1025 * DCB_SEG - 1),
    "big_chunk_last": (1025 * DCB_SEG + 33, 1025 * DCB_SEG + 32),
}


@pytest.mark.gpu
def test_known_answers(sb):
    """bit-exact: zero input gives zeros; with r = 1/64, zero state and zero input elsewhere an impulse x gives y = x on its
    own sample and -r x on the next, and zeros before it, at every boundary of the scan; the conjugate of the output with
    the conjugate off is the output with it on"""
    fe, tid = _fe(sb, 3200.0, 1025 * DCB_SEG + 33, 1, True, False)
    try:
        y, _ = _feed(fe, tid, np.zeros(3 * DCB_SEG + 17, np.complex64), CF32, None)
        assert not y.view(np.uint32).any()
        v = np.complex64(0.75 - 0.5j)
        for name, (n, p) in IMPULSE_AT.items():
            fe.reset()
            z = np.zeros(n, np.complex64)
            z[p] = v
            y, _ = _feed(fe, tid, z, CF32, None)
            assert not y[:p].view(np.uint32).any(), name
            assert y[p] == v, (name, y[p])
            if p + 1 < n:
                assert y[p + 1] == np.complex64(-v / 64), (name, y[p + 1])
                assert np.all(np.abs(y[p + 1:]) <= abs(v) / 64), name
        # the conjugate on the same input
        fe.reset()
        rng = np.random.default_rng(51)
        xs = [make_chunk(rng, n, CF32)[0] for n in (20001, 4097, 3)]
        off = [_feed(fe, tid, d, CF32, None)[0] for d in xs]
    finally:
        fe.close()
    fe, tid = _fe(sb, 3200.0, 20001, 1, True, True)
    try:
        on = [_feed(fe, tid, d, CF32, None)[0] for d in xs]
    finally:
        fe.close()
    for a, b in zip(off, on):
        assert np.conj(a).tobytes() == b.tobytes()


# ---------------------------------------------------------------------------------------------- stage 1 behind the chain
def _s1_gate(oracle, x, sched, offs, fs, ratio, parts, pfb):
    """each RAW VFO (bw == outSR, outSR = fs / ratio) against stage1_f64 and the plan's later stages, with the stage-1
    suite's bound (the filter-bank drift term where the batch is on a grid), gain and edge checks; x taken as exact"""
    plan = plan_of(oracle, ratio)
    D0, h0 = plan[0]
    T = h0.size
    ws = [w_u64(o, fs) for o in offs]
    PS, sg = pfb_detect(ws, T) if pfb else (0, 1)
    worst, gains, edges = 0.0, [], []
    for v, o in enumerate(offs):
        eps = abs(pfb_eps(ws[v], PS, sg)) if PS else 0.0
        y64, b = stage1_f64(x, sched, [o] * len(sched), h0, D0, fs, eps, PS)
        for D, h in plan[1:]:
            y64, b = fir_f64(y64, b, h, D)
        y = np.concatenate(parts[v]).astype(np.complex128)
        assert y.size == y64.size, (y.size, y64.size)
        rr = ratio_c(y, y64, b)
        worst = max(worst, float(rr.max()))
        assert rr.max() <= 1.0, (v, int(np.argmax(rr)), float(rr.max()))
        g = np.vdot(y64, y) / np.vdot(y64, y64)
        resid = eps * float(drift_weights(T, PS).max()) if PS else 0.0
        gains.append(float(abs(g - 1)))
        assert abs(g - 1) <= 1e-6 + resid, (v, g, resid)
        e = np.abs(y - y64)
        edge = np.zeros(y.size, bool)
        for s in np.cumsum([0] + [p.size for p in parts[v][:-1]]):
            edge[max(0, s - EDGE): s + EDGE] = True
        if (~edge).sum() >= 1000:
            er = float(e[edge].max() / np.percentile(e[~edge], 99.9))
            edges.append(er)
            assert er <= 4.0, (v, er)
    return {"max_err_over_bound": worst, "max_abs_g_minus_1": max(gains), "max_edge_over_p999": max(edges) if edges else None}


def _s1_run(sb, fs, ratio, offs, chunks, fmt, scale, decim=1, dc=True, conj=True):
    fe = sb.FrontEnd(fs, max(c.size // (1 if fmt == CF32 else 2) for c in chunks))
    try:
        if decim > 1:
            fe.set_decimation(decim)
        fe.set_dc_blocking(dc)
        fe.set_invert_iq(conj)
        outsr = fs / decim / ratio
        ids = [fe.add_vfo(sb.VfoConfig.raw(o, outsr, outsr)) for o in offs]
        tid = fe.bind_iq(sb.lib.IQ_CF32)
        got, tap, tma, f2 = {v: [] for v in ids}, [], [], []
        for c in chunks:
            if fmt != CF32:
                fe.set_ingest_scale(fmt, scale or 0.0)
            t0, j0 = fe.stat("s1_tma_launches"), fe.stat("s1_f2_jobs")
            outs, _ = fe.process(c, fmt)
            tma.append(fe.stat("s1_tma_launches") - t0)
            f2.append(fe.stat("s1_f2_jobs") - j0)
            tap.append(outs[tid])
            for v in ids:
                got[v].append(outs[v])
    finally:
        fe.close()
    return [got[v] for v in ids], tap, tma, f2


def _bench_run_mirror(oracle, sched):
    """a Run of test_gpu_stage1_f64.py for the bench's 8 RAW VFOs on the cf32 stream behind the blocker"""
    from test_gpu_stage1_f64 import PS10M, Run
    r = Run.__new__(Run)
    r.case = dict(name="preproc_bench", opts={}, retune=None)
    r.ratio = 256
    r.plan = plan_of(oracle, 256)
    r.D, r.T = r.plan[0][0], r.plan[0][1].size
    r.sched = list(sched)
    r.chunk_offs = [list(PS10M)] * len(sched)
    r.offs0 = list(PS10M)
    r.fmts = [CF32] * len(sched)
    r.scales = [None] * len(sched)
    return r


BENCH_S1 = [1 << 24, 1000003]


def test_bench_stage1_mirror(oracle):
    """behind the blocker the bench's cs16 chunks reach stage 1 as cf32: k_xd_tma with the ÷4 epilogue on every VFO; with the
    blocker off the cs16 chunk takes the filter bank and no epilogue"""
    from test_gpu_s1_f2 import f2_chunks
    r = _bench_run_mirror(oracle, BENCH_S1)
    assert r.routes(8) == ["tma", "tma"]
    assert [sum(c) for c in f2_chunks(r)] == [8, 8]
    r.fmts = [CS16] * len(BENCH_S1)
    assert r.routes(8) == ["pfb", "pfb"]


@pytest.mark.gpu
def test_stage1_behind_blocker_bench(sb, oracle, report):
    """the bench's configuration with the pre-processing on: 100 MS/s cs16, one 16 Mi chunk and a ragged one, blocker and
    conjugate on, 8 RAW VFOs on the PS 10 grid behind k_xd_tma with its ÷4 epilogue, against stage1_f64 of the tap's stream;
    with the blocker and conjugate off the same chunks take neither k_xd_tma nor the epilogue"""
    from test_gpu_s1_f2 import f2_chunks
    from test_gpu_stage1_f64 import PS10M
    rng = np.random.default_rng(61)
    chunks = [make_chunk(rng, n, CS16)[0] for n in BENCH_S1]
    parts, tap, tma, f2 = _s1_run(sb, 100e6, 256, PS10M, chunks, CS16, None)
    r = _bench_run_mirror(oracle, BENCH_S1)
    assert tma == [1, 1] and f2 == [sum(c) for c in f2_chunks(r)] == [8, 8], (tma, f2)
    x = np.concatenate(tap).astype(np.complex128)
    res = _s1_gate(oracle, x, BENCH_S1, PS10M, 100e6, 256, parts, True)
    _, _, tma0, f20 = _s1_run(sb, 100e6, 256, PS10M, chunks, CS16, None, dc=False, conj=False)
    assert tma0 == [0, 0] and f20 == [0, 0], (tma0, f20)
    report["preproc_f64_stage1_bench"] = dict(res, tma_launches=tma, f2_jobs=f2)


S1_DECIM = {"pfb": [300e3, -600e3, 900e3], "pipe": [123456.7, -345678.9, 777e3 + 1.5]}


def test_decim_stage1_mirror(oracle):
    """at 2.4 MS/s behind decimation 4, the RAW ratio-8 VFOs on the PS 8 grid take k_xd_pfb and the off-grid ones k_xd_pipe"""
    from test_gpu_stage1_f64 import fir_offsets, s1_route
    D, h = plan_of(oracle, 8)[0]
    sched = decim_counts(oracle, _s1_decim_sched(), 4)
    for build, offs in S1_DECIM.items():
        ws = [w_u64(o, 2.4e6) for o in offs]
        routes = [s1_route(ws, h.size, D, CF32, n, o) for n, o in zip(sched, fir_offsets(sched, D))]
        assert build in routes and set(routes) <= {build, None}, (build, routes)


def _s1_decim_sched():
    return [48000, 7001, 3, 96001, 12288, 1, 48000, 20000]


@pytest.mark.gpu
@pytest.mark.parametrize("build", ["pfb", "pipe"])
def test_stage1_behind_decimation_and_blocker(sb, oracle, report, build):
    """9.6 MS/s cs16 with decimation 4 and the blocker: RAW VFOs at 2.4 MS/s / 8 on k_xd_pfb or k_xd_pipe, against
    stage1_f64 of the tap's stream"""
    rng = np.random.default_rng(71)
    sched = _s1_decim_sched()
    chunks = [make_chunk(rng, n, CS16, 3.1e-5)[0] for n in sched]
    offs = S1_DECIM[build]
    parts, tap, _, _ = _s1_run(sb, 9.6e6, 8, offs, chunks, CS16, 3.1e-5, decim=4, conj=False)
    eff = [t.size for t in tap]
    assert eff == decim_counts(oracle, sched, 4)
    x = np.concatenate(tap).astype(np.complex128)
    report["preproc_f64_stage1_decim4_" + build] = _s1_gate(oracle, x, eff, offs, 2.4e6, 8, parts, build == "pfb")

"""Stage 1 (frequency translator fused with a VFO's first DecimatingFIR: k_xd_tma, k_xd_pfb, k_xd_pipe, k_xd_simple and the
retune edge k_xd_edge) against a float64 reference, sample by sample, from output 0 of the stream.

Reference.  Sample i of the stream is rotated by 2 pi phase(i) / 2^64 with phase(i) = (phase + w n) mod 2^64 in integer
arithmetic, w the u64 increment XdStage::set_offset_rad builds (angle of the fp32-rounded phasor the reference rotates by, at
long-double precision).  A retune starts a new increment at the chunk boundary with the phase continuous, so every sample keeps
the rotation it had when it was translated (FrequencyXlator rotates before the filter's delay line).  Integer chunks are x *
scale with that chunk's scale.  The rotated stream goes through DecimatingFIR from zero history, then through the plan's later
stages (f64_ref.fir_f64, which carries the stage-1 bound).  The CPU part pins this reference to the oracle restatement's
exact-phase RxVFO (bw == outSR: the channel filter is the identity; outSR = fs / ratio: no resampler), retunes included.

A-priori per-sample bound of stage 1, per real component, with A = sqrt(2) sum_k |h_k| |x(i_m + k)|:
    |y - y64| <= (4 T + 4 PS + 40) u A  +  sqrt(2) |eps| sum_k |h_k| |x(i_m + k)| |floor(k / PS) - floor(T / (2 PS))|
(u = 2^-24; PS = 0 and no second term for the complex-tap builds)
  * fp32 taps h_k e^{j w k} (u per component) and accumulation: each component of a complex-tap sum is 2T products and sums,
    <= 2T u sum |h| (|Re x| + |Im x|), <= 4T u sum |h||x| once the output phasor mixes the components; the filter bank's T/PS
    class sums and its PS-term combination with fp32 phasors stay below 4T + 4PS terms of u A;
  * output phasor: sincospif (2 ulp per component, 3 u A) and the phase truncated to its top 32 bits (2 pi 2^-32 rad,
    25 u A); cmulf (3 u A); the integer conversion (float)x * scale (2 u A); the retune edge kernel's per-sample rotation and
    T real fma stay below the same total;
  * filter bank only: the identity residual left by the kernel's centred drift correction.  Both filter-bank kernels sign
    tap k (counted from the window start i_m) by sigma^floor(k / PS) and rotate it by e^{j w (k mod PS)}; the true rotation
    differs by e^{j eps floor(k / PS)}, eps the signed distance (rad) of w PS from 0 (sigma = +1) or 1/2 turn (sigma = -1),
    computed from the exact u64 w, and the output phase adds eps floor(T / (2 PS)).  So the kernel computes exactly
        y_fb[m] = sum_k h_k z(i_m + k) e^{j eps (floor(T / (2 PS)) - floor(k / PS))},   z = x rotated by the exact phase,
    the "filter-bank form", and |e^{j t} - 1| <= |t| gives the second term.
Nothing here is fitted to a run.

Gain.  Per VFO the complex gain g fitted against the filter-bank form (the specification form where a chunk takes a
complex-tap build or the retune edge kernel recomputes an output) is within 1e-6 of 1: at the 8e-6 rad acceptance limit a
dropped or mis-signed drift correction moves it by several times that.  Against the specification form g is within
1e-6 + |eps| max_k |floor(k / PS) - floor(T / (2 PS))|.
"""
import functools
import math

import numpy as np
import pytest

from f64_ref import (PFB_CASES, TWO64, _corr, _hist, _signed, drift_weights, fir_f64, pfb_detect, pfb_eps, plan_of,
                     rotate_f64, stage1_f64, w_u64)
from util import noise_iq

FS = 100e6
RAW_HIST = 1024                                       # engine.h: Scheduler::RAW_HIST
XT_CASES = {(5, 5), (6, 5), (6, 6), (6, 7)}           # kernels.cu: XT_CASE (log2 D, QC)
XT_MAXTAPS = 512                                      # xd_tma.cuh
CF32, CS16, CS8 = 0, 1, 2
PS10M = [5e6, -5e6, 15e6, -15e6, 25e6, -25e6, 35e6, -35e6]     # PS 10, sigma -1 at 100 MS/s
PS10P = [10e6, -20e6, 30e6, -40e6]                              # PS 10, sigma +1
PS8P = [12.5e6, -12.5e6, 37.5e6, -25e6]                         # PS 8, sigma +1
PS8M = [6.25e6, -6.25e6, 18.75e6, -31.25e6]                     # PS 8, sigma -1
OFFGRID = [5e6 + 1234.5, -7.3e6, 21e6 + 77.0]
LIMIT_BASE = 25e6                                               # on this grid point the fp32 phasor steps come closest to the limit


# ---------------------------------------------------------------------------------------------- mirrors of the host code
def s1_route(ws, T, D, fmt, count, offset, variant=8, aligned=True):
    """Scheduler::run's variant choice, then launch_xd_fmt / try_xd_tma / try_xd_pfb / try_xd_pipe, for one chunk of a batch
    whose jobs share T, the chunk offset and the output count (one VFO set through one prototype); `aligned`: the chunk
    pointer is 16-byte aligned.  Returns the build name, None when nothing is launched.  (try_xd_pipe's shared-memory loop,
    which can only decline when not even a 128-output tile fits, is not mirrored.)"""
    n_out = (count - offset + D - 1) // D if offset < count else 0
    if n_out <= 0:
        return None
    QP = (T + D - 1 + D - 1) // D                                   # XdStage::configure
    gpad_len = (D - 1) + (QP + 8) * D
    if gpad_len < (D - 1) + (QP + 8) * D:                           # Scheduler::run: the batch's QP does not fit a job's gpad
        variant = 0
    ps = pfb_detect(ws, T)[0] if variant >= 7 else 0
    logD = D.bit_length() - 1
    pow2 = D >= 2 and (D & (D - 1)) == 0
    if variant >= 7 and ps:
        a0 = offset - (T - 1)
        org = a0 % D
        if variant >= 8 and fmt == CF32 and D in (32, 64) and aligned:
            qc = (T + (org & 1) + D - 1) // D
            sh = org & 1
            for al in (16, 8, 4, 2):
                c = org & (al - 1)
                if (T + c + D - 1) // D == qc:
                    sh = c
                    break
            rows = (count - (org - sh)) // (2 * D) if count - (org - sh) > 0 else 0
            if qc * D <= XT_MAXTAPS and rows >= 8 and (logD, qc) in XT_CASES:
                return "tma"
        if D >= 4 and pow2 and (logD, (T + D - 1) // D) in PFB_CASES:
            return "pfb"
        variant = 6
    if variant >= 1 and pow2:
        # try_xd_pipe: every job shares job 0's alignment (shift 0), so its QP = ceil(T / D) never exceeds the batch's QP
        if (T + D - 1) // D <= QP:
            return "pipe"
    return "simple"


def fir_offsets(sched, D):
    off, offs = 0, []
    for n in sched:
        offs.append(off)
        no = (n - off + D - 1) // D if off < n else 0
        off = off + no * D - n
    return offs


# ---------------------------------------------------------------------------------------------- float64 reference
# (the translator, stage 1 and the filter-bank detection: f64_ref)
def vfo_f64(oracle, x, sched, offs, fs, ratio, eps=0.0, PS=0):
    """RAW VFO with bw == outSR and outSR = fs / ratio: stage 1, then the plan's later DecimatingFIRs (the channel filter is
    the identity tap)"""
    plan = plan_of(oracle, ratio)
    D0, h0 = plan[0]
    y, b = stage1_f64(x, sched, offs, h0, D0, fs, eps, PS)
    for D, h in plan[1:]:
        y, b = fir_f64(y, b, h, D)
    return y, b


def vfo_kernel_form(oracle, x, sched, offs, fs, ratio, chunk_fb):
    """what the kernels compute in exact arithmetic: stage-1 output m takes the filter-bank form (module docstring) when the
    chunk that completes its window (the one holding sample m D) ran a filter-bank build, chunk_fb[c] = (PS, eps), and the
    specification form when chunk_fb[c] is None or its window holds samples of two offsets (the retune edge kernel); then the
    plan's later DecimatingFIRs"""
    plan = plan_of(oracle, ratio)
    D0, h0 = plan[0]
    T = h0.size
    z = _hist(rotate_f64(x, sched, offs, fs), T - 1)
    hh = np.asarray(h0, np.float64)
    y = _corr(z, hh)[::D0]
    last = np.arange(y.size, dtype=np.int64) * D0                     # newest sample of output m's window
    chunk = np.searchsorted(np.cumsum(sched), last, side="right")
    cfg = np.repeat(np.cumsum([0] + [int(offs[c] != offs[c - 1]) for c in range(1, len(sched))]), sched)
    mixed = cfg[np.maximum(last - (T - 1), 0)] != cfg[last]
    for key in {k for k in chunk_fb if k is not None}:
        PS, eps = key
        sel = np.array([chunk_fb[c] == key for c in chunk]) & ~mixed
        if sel.any():
            k = np.arange(T)
            y[sel] = _corr(z, hh * np.exp(1j * eps * (T // (2 * PS) - k // PS)))[::D0][sel]
    for D, h in plan[1:]:
        y = _corr(_hist(y, h.size - 1), np.asarray(h, np.float64))[::D]
    return y


def _ratio(y, y64, b):
    y = np.asarray(y).astype(np.complex128)
    return np.maximum(np.abs(y.real - y64.real), np.abs(y.imag - y64.imag)) / b


def schedule(T, D, total, seed, tile=0):
    """0 and 1 samples, < T-1, D-1 / D / D+1, the TMA minimum (8 super-rows of 2 D) -1 / 0 / +1, one TMA tile +-1, a long
    chunk followed by short ones, repeats, odd sizes (both parities and many residues of the row origin)"""
    rng = np.random.default_rng(seed)
    s = [0, 1, max(1, (T - 2) // 2), D - 1, D, D + 1, 16 * D - 1, 17 * D, 18 * D + 1]
    if tile:
        s += [tile - 1, tile, tile + 1]
    s += [min(1 << 20, max(200000, 40 * D)), 7, 3, 0, 5]
    s += [max(4096, 8 * D)] * 4
    while sum(s) < total - 60000:
        s.append(int(rng.integers(2000, 60000)) | 1)
    s.append(max(1, total - sum(s)))
    return [int(v) for v in s]


# ---------------------------------------------------------------------------------------------- CPU part
RETUNE_KINDS = ["long", "short_with_outputs", "no_output", "two_short", "grid_off_on"]


def retune_schedule(T, D, kind, seed=0):
    """(chunk sizes, per-chunk offset) for one VFO starting at 5 MHz (on the PS 10 grid)"""
    base = [int(np.random.default_rng(seed).integers(20000, 40000)) | 1, 9 * D + 3]
    on, off = 5e6, 5e6 + 1234.5
    if kind == "long":
        s, o = base + [60001, 50000], [on, on, 15e6, 15e6]
    elif kind == "short_with_outputs":
        c = max(D, (T - 1) // 2)
        assert D <= c < T - 1
        s, o = base + [c, 40001, 30000], [on, on, -15e6, -15e6, -15e6]
    elif kind == "no_output":
        s, o = base + [D - 1, 1, 40001], [on, on, 25e6, 25e6, 25e6]
    elif kind == "two_short":
        s, o = base + [D + 1, max(1, (T - 1) // 3), 40001], [on, on, off, -35e6, -35e6]
    else:
        s, o = base + [3 * T + 5, 2, 40001], [on, on, off, on, on]
    return s, o


@pytest.mark.parametrize("ratio", [256, 8192])
@pytest.mark.parametrize("kind", RETUNE_KINDS)
def test_reference_matches_exact_phase_oracle(oracle, ratio, kind):
    """the float64 stage-1 reference (phase continuity across retunes, per-chunk increments, index convention, output
    count) against the oracle restatement's exact-phase RxVFO, every output within the bound"""
    plan = plan_of(oracle, ratio)
    D0, h0 = plan[0]
    T = h0.size
    sched, offs = retune_schedule(T, D0, kind)
    q = oracle.resamp_plan(FS, FS / ratio)
    assert q["predec_ratio"] == ratio and q["interp"] == q["decim"]
    x = noise_iq(sum(sched), ratio + len(kind), 1.0)
    oracle.set_rotator_mode(1)
    try:
        v = oracle.rxvfo(FS, FS / ratio, FS / ratio, offs[0])
        parts, pos = [], 0
        for n, off in zip(sched, offs):
            v.set_offset(off)
            parts.append(v.process(x.view(np.float32)[2 * pos: 2 * (pos + n)]).view(np.complex64))
            pos += n
    finally:
        oracle.set_rotator_mode(0)
    y = np.concatenate(parts)
    y64, b = vfo_f64(oracle, x.astype(np.complex128), sched, offs, FS, ratio)
    assert y.size == y64.size
    r = float(np.max(_ratio(y, y64, b)))
    assert r <= 1.0, r
    # the float64 reference is not blind to the retune: rotating the history with the new increment moves it off
    if kind not in ("long", "grid_off_on"):             # (1234.5 Hz off the grid is too small a step to show here)
        wrong, _ = vfo_f64(oracle, x.astype(np.complex128), sched, [offs[-1]] * len(sched), FS, ratio)
        assert float(np.max(_ratio(wrong, y64, b))) > 1.0


def test_bound_covers_the_filter_bank_residual(oracle):
    """the filter-bank form with the kernel's centred drift correction stays inside the drift term of the bound, for PS 10
    and 8, sigma +-1, the D = 32 and D = 64 plans and a VFO just inside the 8e-6 rad acceptance limit"""
    rng = np.random.default_rng(5)
    cases = [(256, PS10M), (256, PS10P), (256, PS8P), (256, PS8M), (512, PS10M), (2048, PS8P), (4096, PS8M)]
    worst = 0.0
    for ratio, offs in cases:
        D, h = plan_of(oracle, ratio)[0]
        T = h.size
        ws = [w_u64(o, FS) for o in offs]
        PS, sg = pfb_detect(ws, T)
        assert PS in (8, 10)
        edge = limit_offsets(offs[0], T)[0]
        for off in list(offs) + [edge]:
            w = w_u64(off, FS)
            if off == edge:
                assert pfb_detect([w], T) == pfb_detect([w_u64(offs[0], FS)], T)
            eps = pfb_eps(w, PS, sg)
            wr = _signed(w) * (2 * math.pi / TWO64)
            n_out = 64
            x = rng.uniform(-1, 1, (n_out * D + T, 2)).astype(np.float32).astype(np.float64) @ [1, 1j]
            k = np.arange(T)
            win = x[(np.arange(n_out) * D)[:, None] + k[None, :]]
            y_ref = (win * (h * np.exp(1j * wr * k))[None, :]).sum(axis=1)
            sgn = np.where((k // PS) % 2, float(sg), 1.0)
            S = np.stack([(win[:, k % PS == a] * (h[k % PS == a] * sgn[k % PS == a])[None, :]).sum(axis=1) for a in range(PS)], 1)
            y_pfb = np.exp(1j * eps * (T // (2 * PS))) * (S * np.exp(1j * wr * np.arange(PS))[None, :]).sum(axis=1)
            A = math.sqrt(2.0) * (np.abs(win) * np.abs(h)[None, :]).sum(axis=1)
            bnd = math.sqrt(2.0) * abs(eps) * (np.abs(win) * (np.abs(h) * drift_weights(T, PS))[None, :]).sum(axis=1)
            r = float(np.max(np.abs(y_pfb - y_ref) / (bnd + 1e-13 * A)))
            worst = max(worst, r)
    assert worst <= 1.0, worst


@functools.lru_cache(maxsize=None)
def limit_offsets(off, T):
    """(just inside, just outside) the scheduler's 8e-6 rad acceptance limit: stepping away from the grid offset `off` by
    1e-9 rad per sample, the last offset whose fp32-rounded phasor still takes the filter-bank form (worst-case drift) and the
    first that does not"""
    ref = pfb_detect([w_u64(off, FS)], T)
    step = 1e-9 * FS / (2 * math.pi)
    inside = off
    for k in range(1, 2000):
        o = off - k * step
        if pfb_detect([w_u64(o, FS)], T) != ref:
            return inside, o
        inside = o
    raise AssertionError("no acceptance limit found")


def test_grid_families_and_limits_route_as_named(oracle):
    T = plan_of(oracle, 256)[0][1].size
    assert pfb_detect([w_u64(o, FS) for o in PS10M], T) == (10, -1)
    assert pfb_detect([w_u64(o, FS) for o in PS10P], T) == (10, 1)
    assert pfb_detect([w_u64(o, FS) for o in PS8P], T) == (8, 1)
    assert pfb_detect([w_u64(o, FS) for o in PS8M], T) == (8, -1)
    assert pfb_detect([0], T) == (8, 1)
    assert pfb_detect([w_u64(o, FS) for o in OFFGRID], T)[0] == 0
    inside, outside = limit_offsets(LIMIT_BASE, T)
    PS, sg = pfb_detect([w_u64(LIMIT_BASE, FS)], T)
    assert PS and pfb_detect([w_u64(inside, FS)], T) == (PS, sg)
    assert pfb_detect([w_u64(outside, FS)], T)[0] == 0
    # the VFO just inside uses nearly all the drift the scheduler allows: |eps| T / PS close to 8e-6 rad
    assert abs(pfb_eps(w_u64(inside, FS), PS, sg)) * T / PS > 7.5e-6


# ---------------------------------------------------------------------------------------------- GPU cases
def _c(name, ratio, offs, build, fmt="cf32", opts=None, total=1000000, retune=None, scale=None, dup=1):
    return dict(name=name, ratio=ratio, offs=list(offs) * dup, build=build, fmt=fmt, opts=opts or {}, total=total,
                retune=retune, scale=scale)


CASES = [
    # each XT_CASE, PS 10 sigma -1 (config 2 grid)
    _c("tma_r256", 256, PS10M, "tma"),
    _c("tma_r512", 512, PS10M[:4], "tma"),
    _c("tma_r1024", 1024, PS10M[:4], "tma", total=2500000),
    _c("tma_r2048", 2048, PS10M[:4], "tma", total=3000000),
    _c("tma_r4096", 4096, PS10M[:2], "tma", total=4000000),
    # grid families, options, batching
    _c("tma_ps10p", 256, PS10P, "tma"),
    _c("tma_ps8p", 256, PS8P, "tma"),
    _c("tma_ps8m", 256, PS8M, "tma"),
    _c("tma_limit", 256, ["limit"], "tma"),
    _c("tma_stages3_ctas1", 256, PS10M, "tma", opts={"s1_stages": 3, "s1_ctas": 1}),
    _c("tma_20vfos_pair0", 256, PS10M, "tma", opts={"pair": 0}, dup=3, total=600000),
    _c("pfb_s7_cf32", 256, PS10M, "pfb", opts={"s1": 7}),
    _c("pfb_s7_ps8m", 256, PS8M, "pfb", opts={"s1": 7}),
    _c("pfb_limit_s7", 256, ["limit"], "pfb", opts={"s1": 7}),
    _c("pfb_limit_cs16", 256, ["limit"] * 2, "pfb", fmt="cs16"),
    # each PFB_CASE with integer input
    _c("pfb_r8_cs16", 8, PS8P[:2], "pfb", fmt="cs16", total=600000),
    _c("pfb_r16_cs8", 16, PS10M[:2], "pfb", fmt="cs8", total=600000),
    _c("pfb_r128_cs16_scale", 128, PS10M, "pfb", fmt="cs16", scale=[3.1e-5]),
    _c("pfb_r256_cs16_scales", 256, PS10M, "pfb", fmt="cs16", scale=[None, 2.7e-5, 4.1e-5]),
    _c("pfb_r1024_mixfmt", 1024, PS10M[:4], "pfb", fmt="mix", total=2500000, scale=[1.7e-5]),
    # pipe: per-VFO complex taps
    _c("pipe_r2", 2, OFFGRID, "pipe", total=400000),
    _c("pipe_r4_cs16", 4, OFFGRID, "pipe", fmt="cs16", total=400000),
    _c("pipe_r32_pairs", 32, [3.3e6, -3.3e6, 7.1e6, -7.1e6, 1.0e6], "pipe", total=800000),
    _c("pipe_r64_s5", 64, OFFGRID, "pipe", opts={"s1": 5}),
    _c("pipe_r8192", 8192, OFFGRID[:2], "pipe", total=5000000),
    _c("pipe_outside_limit", 256, ["beyond"], "pipe"),
    _c("pipe_s6_grid_mt128", 256, PS10M, "pipe", opts={"s1": 6, "s1_mt": 128}),
    # one thread per output
    _c("simple_s0_r256", 256, PS10M[:4], "simple", opts={"s1": 0}),
    _c("simple_d1", 1, [3.3e6, -12.5e6], "simple", total=200000),
    # retunes (front end)
    _c("retune_r256_short", 256, [5e6], "tma", retune="short_with_outputs"),
    _c("retune_r256_no_output", 256, [5e6], "tma", retune="no_output"),
    _c("retune_r256_two_short", 256, [5e6], "tma", retune="two_short"),
    _c("retune_r256_grid_off_on", 256, [5e6], "tma", retune="grid_off_on"),
    _c("retune_r256_long", 256, [5e6], "tma", retune="long"),
    _c("retune_r8192_short", 8192, [5e6], "pipe", retune="short_with_outputs", total=4000000),
    _c("retune_r8192_two_short", 8192, [5e6], "pipe", retune="two_short", total=4000000),
    _c("retune_r256_cs16_short", 256, [5e6], "pfb", fmt="cs16", retune="short_with_outputs"),
]
CASE_IDS = [c["name"] for c in CASES]


class Run:
    """what one GPU case feeds: chunk sizes, per-chunk format / scale / offsets, the input and its float64 value"""

    def __init__(self, oracle, case):
        self.case = case
        self.ratio = case["ratio"]
        self.plan = plan_of(oracle, self.ratio)
        D, h = self.plan[0]
        self.D, self.T = D, h.size
        seed = CASE_IDS.index(case["name"])
        offs = []
        for o in case["offs"]:
            if o == "limit":
                o = limit_offsets(LIMIT_BASE, self.T)[0]
            elif o == "beyond":
                o = limit_offsets(LIMIT_BASE, self.T)[1]
            offs.append(o)
        self.offs0 = offs
        if case["retune"]:
            s, o = retune_schedule(self.T, D, case["retune"], seed)
            tail = schedule(self.T, D, max(case["total"] - sum(s), 200000), seed)[9:]
            self.sched = s + tail
            self.chunk_offs = [[v] for v in o] + [[o[-1]]] * len(tail)
        else:
            tile = 256 * D if D == 32 else 128 * D
            self.sched = schedule(self.T, D, case["total"], seed, tile)
            self.chunk_offs = [offs] * len(self.sched)
        nc = len(self.sched)
        fmt = case["fmt"]
        if fmt == "mix":
            self.fmts = [(CF32, CS16, CS8)[k % 3] for k in range(nc)]
        else:
            self.fmts = [{"cf32": CF32, "cs16": CS16, "cs8": CS8}[fmt]] * nc
        sc = case["scale"] or [None]
        self.scales = [sc[k % len(sc)] for k in range(nc)]
        rng = np.random.default_rng(900 + seed)
        self.chunks, vals = [], []
        for n, f, s in zip(self.sched, self.fmts, self.scales):
            if f == CF32:
                c = rng.uniform(-1, 1, 2 * n).astype(np.float32)
                v = c.astype(np.float64)
            else:
                lim = 32768 if f == CS16 else 128
                c = rng.integers(-lim, lim, 2 * n).astype(np.int16 if f == CS16 else np.int8)
                scale = np.float32(s) if s else np.float32(1.0 / lim)
                v = c.astype(np.float64) * float(scale)
            self.chunks.append(c)
            vals.append(v)
        v = np.concatenate(vals)
        self.x = v[0::2] + 1j * v[1::2]

    def routes(self, variant, aligned=True):
        """builds reached by the chunks of this case (per chunk), as the scheduler picks them"""
        offsets = fir_offsets(self.sched, self.D)
        out = []
        for n, o, f, co in zip(self.sched, offsets, self.fmts, self.chunk_offs):
            out.append(s1_route([w_u64(v, FS) for v in co], self.T, self.D, f, n, o, variant, aligned))
        return out

    def chunk_fb(self, routes, v):
        """per chunk: (PS, eps of VFO v) when the chunk runs a filter-bank build, else None"""
        out = []
        for rt, co in zip(routes, self.chunk_offs):
            if rt in ("tma", "pfb"):
                PS, sg = pfb_detect([w_u64(o, FS) for o in co], self.T)
                out.append((PS, pfb_eps(w_u64(co[v], FS), PS, sg)))
            else:
                out.append(None)
        return out


def test_gpu_cases_reach_their_build(oracle):
    """every GPU case reaches the build it is named after on some chunk (the scheduler's predicates, mirrored), its chunk
    schedule has a chunk either side of the TMA minimum where TMA applies, and the retune cases have the short chunk after
    the retune that reaches back across the boundary"""
    seen = set()
    for case in CASES:
        r = Run(oracle, case)
        variant = case["opts"].get("s1", 8)
        routes = r.routes(variant)
        assert case["build"] in routes, (case["name"], set(routes))
        if case["build"] == "tma":
            seen.add((r.D.bit_length() - 1, (r.T + r.D - 1) // r.D))
            if not case["retune"]:
                assert set(routes) - {"tma", None}       # the 8-row minimum and short chunks take another build
        if case["build"] == "pfb" and case["fmt"] != "cf32":
            seen.add(("pfb", r.D.bit_length() - 1, (r.T + r.D - 1) // r.D))
        if case["retune"] in ("short_with_outputs", "two_short"):
            k = next(i for i in range(1, len(r.chunk_offs)) if r.chunk_offs[i] != r.chunk_offs[i - 1])
            assert r.sched[k] < r.T - 1
    assert {k for k in seen if k[0] != "pfb"} == XT_CASES
    assert {k[1:] for k in seen if k[0] == "pfb"} == PFB_CASES


# ---------------------------------------------------------------------------------------------- GPU part
@pytest.fixture(scope="module")
def sb():
    import sdrplusplus_b200 as m
    from sdrplusplus_b200 import lib
    L = lib.load()
    assert L.b200_device_count() > 0
    assert L.b200_init(0) == 0
    return m


def _run_front_end(sb, r, chunks=None):
    fe = sb.FrontEnd(FS, max(max(r.sched), 1))
    try:
        for k, v in r.case["opts"].items():
            fe.set_option(k, v)
        outsr = FS / r.ratio
        nv = len(r.chunk_offs[0])
        ids = [fe.add_vfo(sb.VfoConfig.raw(r.chunk_offs[0][v], outsr, outsr)) for v in range(nv)]
        got = {vid: [] for vid in ids}
        t0 = fe.stat("s1_tma_launches")
        prev = r.chunk_offs[0]
        for c, (n, f, s, co) in enumerate(zip(r.sched, r.fmts, r.scales, r.chunk_offs)):
            if co != prev:
                for v, vid in enumerate(ids):
                    fe.set_vfo_offset(vid, co[v])
                prev = co
            if f != CF32:
                fe.set_ingest_scale(f, s or 0.0)
            data = (chunks or r.chunks)[c]
            outs, _ = fe.process(data.view(np.complex64) if f == CF32 else data, f)
            for vid in ids:
                got[vid].append(outs[vid])
        tma = fe.stat("s1_tma_launches") - t0
    finally:
        fe.close()
    return [got[vid] for vid in ids], tma


def _gate_parts(oracle, r, parts, routes):
    """every output of every VFO within the bound, the fitted gain against the kernels' form and the specification form,
    and edge against interior; returns (worst fraction of the bound, |g-1| per VFO, |g_spec-1| per VFO, edge ratios)"""
    worst, gains, gains_spec, edges = 0.0, [], [], []
    for v in range(len(parts)):
        offs = [co[v] for co in r.chunk_offs]
        fb = r.chunk_fb(routes, v)
        keys = [k for k in fb if k is not None]
        PS = max((k[0] for k in keys), default=0)
        eps = max((abs(k[1]) for k in keys), default=0.0)
        y64, b = vfo_f64(oracle, r.x, r.sched, offs, FS, r.ratio, eps, PS)
        y = np.concatenate(parts[v])
        assert y.size == y64.size, (y.size, y64.size)
        ratio = _ratio(y, y64, b)
        k = int(np.argmax(ratio))
        worst = max(worst, float(ratio[k]))
        assert ratio[k] <= 1.0, (v, k, float(ratio[k]), y.size)
        yc = y.astype(np.complex128)
        yk = vfo_kernel_form(oracle, r.x, r.sched, offs, FS, r.ratio, fb)
        g = np.vdot(yk, yc) / np.vdot(yk, yk)
        gains.append(float(abs(g - 1)))
        assert abs(g - 1) <= 1e-6, (v, g)
        gs = np.vdot(y64, yc) / np.vdot(y64, y64)
        gains_spec.append(float(abs(gs - 1)))
        resid = max((abs(k[1]) * float(drift_weights(r.T, k[0]).max()) for k in keys), default=0.0)
        assert abs(gs - 1) <= 1e-6 + resid, (v, gs, resid)
        if y.size >= 4000:
            e = np.abs(yc - y64) / np.sqrt(np.mean(np.abs(y64) ** 2))
            edge = np.zeros(y.size, bool)
            for bnd in np.cumsum([0] + [p.size for p in parts[v][:-1]]):
                edge[max(0, bnd - 64): bnd + 64] = True
            if (~edge).sum() >= 1000:
                er = float(e[edge].max() / np.percentile(e[~edge], 99.9))
                edges.append(er)
                assert er <= 4.0, (v, er)
    return worst, gains, gains_spec, edges


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_IDS)
def test_stage1_vs_float64(sb, oracle, report, name):
    case = CASES[CASE_IDS.index(name)]
    r = Run(oracle, case)
    parts, tma = _run_front_end(sb, r)
    variant = case["opts"].get("s1", 8)
    routes = r.routes(variant)
    nbatch = -(-len(r.offs0) // 16)
    if case["build"] == "tma":
        assert tma == nbatch * routes.count("tma"), (tma, routes.count("tma"))
    worst, gains, gains_spec, edges = _gate_parts(oracle, r, parts, routes)
    report["stage1_f64_" + name] = {"builds": sorted(set(b for b in routes if b)), "tma_launches": int(tma),
                                    "max_err_over_bound": worst, "max_abs_g_minus_1": max(gains),
                                    "max_abs_g_spec_minus_1": max(gains_spec),
                                    "max_edge_over_p999": max(edges) if edges else None, "vfos": len(parts)}


def _impulse_support(plan, pos, n):
    """outputs of the cascade an impulse at input `pos` can reach (interval arithmetic through each DecimatingFIR)"""
    a, b = pos, pos
    for D, h in plan:
        a, b = -(-a // D), (b + h.size - 1) // D
    return a, b


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["pipe_r2", "tma_r256", "pfb_r128_cs16_scale", "retune_r256_two_short"])
def test_stage1_impulse_support(sb, oracle, name):
    """zero input with impulses at every residue mod D, chunk starts +-1, inside the raw history (just before a chunk),
    in the last partial super-row, at the last sample of a TMA chunk that an output's window ends on, and at tile edges:
    every output within the per-sample bound of the float64 answer (an impulse's bound is a small multiple of u times the
    tap it meets, so a missing or extra sample shows), every output outside the predicted support exactly 0; at offset 0 and
    ratio 2 every phasor is 1 and the taps come back bit-exact"""
    case = dict(CASES[CASE_IDS.index(name)])
    if name == "pipe_r2":
        case["offs"] = [0.0]
    r = Run(oracle, case)
    D, T = r.D, r.T
    variant = case["opts"].get("s1", 8)
    prio = []
    if "tma" in r.routes(variant):
        # stretch the first long TMA chunk so that its last output's window ends on its last sample (the ragged end the
        # kernel patches from the chunk), give the difference back to the next chunk, and put an impulse there
        offsets = fir_offsets(r.sched, D)
        c = next(i for i, rt in enumerate(r.routes(variant)) if rt == "tma" and r.sched[i] >= 20 * D and r.sched[i + 1] > 2 * D)
        d = (offsets[c] + 1 - r.sched[c]) % D
        r.sched[c] += d
        r.sched[c + 1] -= d
        assert (r.sched[c] - 1 - offsets[c]) % D == 0 and r.routes(variant)[c] == "tma"
        prio.append(int(sum(r.sched[:c + 1]) - 1))
    n = sum(r.sched)
    starts = np.cumsum([0] + r.sched[:-1])
    sep = T + D + 1
    # one impulse at every residue mod D first, in the middle of the stream, then the others where they keep their distance
    q = -(-sep // D) + 1
    p0 = (n // 2) // D * D
    keep = [p0 + k * q * D + k for k in range(D)]
    for c in prio:
        assert min(abs(c - v) for v in keep) >= sep
        keep.append(c)
    cand = []
    for st, ln in zip(starts, r.sched):
        cand += [st - 1, st, st + 1, st + ln - 2 * D + 1]
        for k in (1, 2):
            cand += [st + k * 128 * D - 1, st + k * 128 * D]
    for c in sorted(set(int(v) for v in cand if 0 <= v < n)):
        if min(abs(c - v) for v in keep) >= sep:
            keep.append(c)
    pos = np.array(sorted(keep))
    assert set(pos % D) == set(range(D)) and pos.max() < n
    vals = np.where(np.arange(pos.size) % 2 == 0, 1.0, 1.0 + 1.0j)
    chunks = []
    x = np.zeros(n, np.complex128)
    p0 = 0
    for c, (ln, f, sc) in enumerate(zip(r.sched, r.fmts, r.scales)):
        sel = (pos >= p0) & (pos < p0 + ln)
        at = pos[sel] - p0
        if f == CF32:
            z = np.zeros(2 * ln, np.float32)
            z[2 * at] = vals[sel].real
            z[2 * at + 1] = vals[sel].imag
            x[pos[sel]] = vals[sel]
        else:
            z = np.zeros(2 * ln, np.int16 if f == CS16 else np.int8)
            z[2 * at] = 100
            x[pos[sel]] = 100.0 * float(np.float32(sc) if sc else np.float32(1.0 / (32768 if f == CS16 else 128)))
        chunks.append(z)
        p0 += ln
    parts, _ = _run_front_end(sb, r, chunks)
    routes = r.routes(variant)
    for v in range(len(parts)):
        y = np.concatenate(parts[v])
        fb = [k for k in r.chunk_fb(routes, v) if k is not None]
        y64, b = vfo_f64(oracle, x, r.sched, [co[v] for co in r.chunk_offs], FS, r.ratio,
                         max((abs(k[1]) for k in fb), default=0.0), max((k[0] for k in fb), default=0))
        assert y.size == y64.size
        rr = _ratio(y, y64, b)
        assert rr.max() <= 1.0, (v, int(np.argmax(rr)), float(rr.max()))
        inside = np.zeros(y.size, bool)
        for p in pos:
            a, b = _impulse_support(r.plan, int(p), n)
            inside[a: b + 1] = True
        bad = np.flatnonzero(~inside & (y != 0))
        assert bad.size == 0, (v, bad[:8], y[bad[:8]])
        if name == "pipe_r2":
            h = r.plan[0][1]
            want = np.zeros(y.size, np.complex64)
            for k, p in enumerate(pos):
                m = np.arange(-(-p // D), min(y.size - 1, (p + T - 1) // D) + 1)
                want[m] = h[T - 1 + p - m * D] * np.complex64(vals[k])
            assert np.array_equal(y, want)


def _block_run(oracle, ratio, kind):
    """a Run for one VFO of the stand-alone RxVFO block: the retune schedule, then long and short chunks, cf32 noise"""
    r = Run.__new__(Run)
    r.case = dict(name="block_%d_%s" % (ratio, kind), opts={})
    r.ratio = ratio
    r.plan = plan_of(oracle, ratio)
    r.D, r.T = r.plan[0][0], r.plan[0][1].size
    sched, offs = retune_schedule(r.T, r.D, kind, 3)
    r.sched = sched + [100001, 9, 200000]
    r.chunk_offs = [[o] for o in offs] + [[offs[-1]]] * 3
    r.offs0 = r.chunk_offs[0]
    r.fmts = [CF32] * len(r.sched)
    r.scales = [None] * len(r.sched)
    r.xf = noise_iq(sum(r.sched), 31 + ratio, 1.0)
    r.x = r.xf.astype(np.complex128)
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("ratio,kind", [(256, "short_with_outputs"), (256, "two_short"), (8192, "no_output")])
def test_block_rxvfo_retune_vs_float64(sb, oracle, report, ratio, kind):
    """the stand-alone RxVFO block: set_offset between chunks, every output against the float64 reference, and its gains"""
    r = _block_run(oracle, ratio, kind)
    blk = sb.Block.rxvfo(FS, FS / ratio, FS / ratio, r.chunk_offs[0][0])
    parts, pos = [], 0
    for n, co in zip(r.sched, r.chunk_offs):
        blk.set_offset(co[0])
        parts.append(blk.process(r.xf.view(np.float32)[2 * pos: 2 * (pos + n)]).view(np.complex64))
        pos += n
    blk.close()
    routes = r.routes(8)
    worst, gains, gains_spec, _ = _gate_parts(oracle, r, [parts], routes)
    report["stage1_f64_block_rxvfo_%d_%s" % (ratio, kind)] = {"builds": sorted(set(b for b in routes if b)),
                                                               "max_err_over_bound": worst, "abs_g_minus_1": gains[0],
                                                               "abs_g_spec_minus_1": gains_spec[0]}


@pytest.mark.gpu
def test_stage1_unaligned_device_chunk(sb, oracle, report):
    """device chunks read in place, 8 bytes off a 16-byte boundary: k_xd_tma declines them (no TMA launch) and the filter
    bank takes every chunk that has outputs; every output against float64, as for the aligned cases"""
    import torch
    from sdrplusplus_b200 import lib as L
    case = dict(CASES[CASE_IDS.index("tma_r256")], offs=PS10M[:4] + ["limit"])
    r = Run(oracle, case)
    routes = r.routes(8, aligned=False)
    assert "tma" not in routes and "pfb" in routes and r.routes(8).count("tma") > 0
    fe = sb.FrontEnd(FS, max(r.sched))
    try:
        outsr = FS / r.ratio
        ids = [fe.add_vfo(sb.VfoConfig.raw(o, outsr, outsr)) for o in r.chunk_offs[0]]
        got = {vid: [] for vid in ids}
        t0 = fe.stat("s1_tma_launches")
        buf = torch.empty(2 * max(r.sched) + 4, dtype=torch.float32, device="cuda")
        for n, c in zip(r.sched, r.chunks):
            dev = buf[2: 2 + 2 * n]
            dev.copy_(torch.from_numpy(c))
            torch.cuda.synchronize()
            ptr = buf.data_ptr() + 8                      # (an empty view reports address 0)
            assert ptr % 16 == 8
            o, bufs, _ = fe._alloc_outputs(n)
            fe.process_ptr(ptr, n, CF32, L.MEM_DEVICE, o)
            for vid in ids:
                got[vid].append(bufs[vid][: 2 * o.vfo_count[vid]].copy().view(np.complex64))
        tma = fe.stat("s1_tma_launches") - t0
    finally:
        fe.close()
    assert tma == 0
    worst, gains, gains_spec, edges = _gate_parts(oracle, r, [got[vid] for vid in ids], routes)
    report["stage1_f64_unaligned_device_chunk"] = {"builds": sorted(set(b for b in routes if b)), "max_err_over_bound": worst,
                                                   "max_abs_g_minus_1": max(gains), "max_abs_g_spec_minus_1": max(gains_spec),
                                                   "max_edge_over_p999": max(edges) if edges else None}

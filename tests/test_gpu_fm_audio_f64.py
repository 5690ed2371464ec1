"""The FM discriminator (k_quad, the fused tail's FT_QUAD phase) and the audio chain behind it (audio low-pass with stereo
duplication, AF resampler, 300 Hz high-pass, de-emphasis, volume) against float64 references, sample by sample, from output 0
of the stream: as stand-alone blocks and inside whole WFM / NFM VFOs of the front end, in every tail build.

Discriminator.  Reference: theta64 = arctan2 (float64) of the float64 IQ, theta[-1] = 0 (Quadrature's initial phase),
d64 = theta64[i] - theta64[i-1] wrapped as math::normalizePhase wraps (normalize_phase.h:6-10): the threshold is the fp32
constant P = FL_M_PI_REF = fl(3.1415926535) (not pi) and the step 2P (exact in fp32); on a wrapped sample 2P differs from
2 pi by 1.7e-7 rad, and that is part of the specification.  q64 = d64 inv_dev with the stage's fp32 inv_dev taken as an
exact coefficient.  Per-sample bound, for input IQ whose components are within b of the reference (b = 0 for an exact
block input), in rad before the scale:
  * conditioning: the fp32 input lies within sqrt(2) b of z, so its angle is within asin(sqrt(2) b / |z|) of theta64
    (pi when that ratio reaches 1), for both samples;
  * atan2f: 3 ulp of the result, both samples (CUDA C++ Programming Guide, "Single-Precision Mathematical Standard Library
    Functions with Maximum ULP Error": atan2f(y,x) 3; glibc's atan2f, which the oracle's CPU blocks call, is listed within it);
  * the subtraction: u (|theta_i| + |theta_i-1| + both terms above), u = 2^-24; the wrap step: u P where a wrap can occur;
  * a perturbed input whose disk reaches the negative real axis can return an angle 2 pi away; the wrap then removes 2P, so
    such a sample adds 2 (P - pi) per operand;
  * the multiply: u inv_dev (|d64| + E).
The sum E inv_dev + u inv_dev (|d64| + E) is capped at 2 P inv_dev (1 + 2u): |q| and |q64| never exceed P inv_dev (1 + u).
Where |d64| lies within E of P either wrap branch is accepted (the other branch is d64 - 2P sign(d64)); such samples are
counted ("ambiguous wraps") and carry the cap into the stages behind.

Audio chain.  Audio low-pass and high-pass: f64_ref.fir_f64 (real data, and l + j r); AF resampler: f64_ref.poly_f64 on l + j r
(stereo_t is two packed floats, the same kernels run it); mono to stereo and the low-pass's stereo duplication: L == R bit for
bit.  De-emphasis y = a x + b y[-1] with a = fl(dt / (tau + dt)), dt = fl(1 / sr), b = fl(1 - a) (deephasis.h:91-94), per
component: two products and a sum, each within u of its result, so
    e[i] = b (1 + 3u) e[i-1] + a (1 + 3u) e_x[i] + 3u (a |x64[i]| + b |y64[i-1]|),
a first-order recursion on non-negative terms (scipy.signal.lfilter).  Volume: one fp32 multiply by g = fl(fl(v)^2).

Whole VFO.  Stage 1 with its bound (f64_ref.stage1_f64; for a VFO on the filter-bank grid with its PS and drift eps), the
plan's later DecimatingFIRs, the resampler, the channel FIR (lowPass(bw/2, 0.1 bw/2, outSR), the identity tap when bw ==
outSR), then the chain above.  Retunes follow stage1_f64; a bandwidth change swaps the channel filter at the chunk boundary,
and after identity -> low-pass the filter starts from cleared history (Chain::add_rxvfo); other changes follow
vfo_settings_oracle.py (a high-pass switched off keeps its delay line; de-emphasis keeps its state across a tau change).
In situ stage 1's a-priori bound dominates; the fitted gain |g - 1| < 2e-6 and the edge-against-interior ratio <= 4
(f64_ref._gate_vfo) carry the fine sensitivity there, the stand-alone blocks carry it for the kernels themselves.
Each front-end option set profiles one chunk and asserts that the kernels behind stage 1 that ran are those the routing
mirror names; every case sets its options, the tail variant ("tails") among them, on its own front end.
No tolerance here is fitted to a run.
"""
import math

import numpy as np
import pytest
from scipy.signal import lfilter

from f64_ref import (P32, PFB_CASES, POLY_REG, TS_TILE, TWO_P, U, _gate_clean, _ratio_c, audio_lp_taps, cascade_counts,
                     chan_taps, deemph_coefs, deemph_f64, fir_f64, inv_dev_of, pfb_detect, poly_f64, quad_f64, quad_ratio,
                     routes_dfir_reg, schedule, vfo_audio_f64, vfo_counts, volume_f64, w_u64)
from util import noise_iq

TAIL_MAX_TAPS = 1024                           # tails.cuh
FT_MAX_L = 64                                  # fused_tail.cuh
FT_MAXST = 8                                   # kernels.cuh
QUAD_TILE = 256                                # k_quad / k_firr_reg outputs per CTA


# ---------------------------------------------------------------------------------------------- routing mirror
def chain_stages(oracle, fs, cfg):
    """the stage list Chain builds for an FM VFO (api.cpp build_vfo_chain): (kind, ...) per stage"""
    from sdrplusplus_b200 import frontend
    osr = cfg.out_samplerate
    rp = frontend.resamp_plan(fs, osr)
    st = [("xd",)] + [("firc", D, T, 2) for D, T in rp["stages"][1:]]
    if rp["ntaps"]:
        st.append(("poly", rp["interp"], rp["decim"], rp["taps_per_phase"]))
    st.append(("firc", 1, chan_taps(oracle, cfg.bandwidth, osr).size, 2))
    st.append(("quad",))
    h = audio_lp_taps(oracle, cfg)
    st.append(("firr", h.size) if h is not None else ("m2s",))
    if cfg.af_samplerate > 0:
        ap = frontend.resamp_plan(osr, cfg.af_samplerate)
        st += [("firc", D, T, 2) for D, T in ap["stages"]]
        if ap["ntaps"]:
            st.append(("poly", ap["interp"], ap["decim"], ap["taps_per_phase"]))
        if cfg.af_high_pass:
            st.append(("firc", 1, oracle.highpass(300.0, 100.0, cfg.af_samplerate).size, 2))
        if cfg.af_deemph_tau > 0:
            st.append(("seq",))
    if cfg.af_volume_on:
        st.append(("scale",))
    return st


def _fusable(s):
    """ft_fusable (engine.cpp)"""
    return s[0] in ("firc", "quad", "firr", "m2s") or (s[0] == "poly" and s[1] <= FT_MAX_L)


def _reg_able(s):
    """Chain::plan_fused's reg_all test of one stage"""
    if s[0] == "firc":
        return (s[1] == 1 and s[2] <= 2000) or (s[1] > 1 and routes_dfir_reg(s[1], s[2]))
    if s[0] == "poly":
        return (s[1], s[2]) in POLY_REG and s[3] <= 512
    if s[0] == "firr":
        return s[1] <= 2000
    return s[0] in ("quad", "m2s")


def fused_range(st, opts):
    """Chain::plan_fused up to its shared-memory plan: (beg, end) of the stages one k_tail_fused launch would run, None
    when the chain is not fused.  Whether the plan fits shared memory is decided at run time: b200_fe_stat("fused_chains")."""
    tails = opts.get("tails", 2)
    pre_reg = opts.get("ft_prereg", 8)
    if tails < 2 or len(st) < 3:
        return None
    beg = 1
    if pre_reg > 0:
        while beg - 1 < pre_reg and beg < len(st) and st[beg][0] == "firc" and st[beg][1] > 1 and routes_dfir_reg(st[beg][1], st[beg][2]):
            beg += 1
    while True:
        end = beg
        while end < len(st) and end - beg < FT_MAXST and _fusable(st[end]):
            end += 1
        if end - beg >= 2 or beg == 1:
            break
        beg -= 1
    if end - beg < 2:
        return None
    if opts.get("ft_regall", 1) and pre_reg > 0 and all(_reg_able(s) for s in st[1:end]):
        return None
    return beg, end


def stage_builds(st, opts, fused):
    """the kernel build each stage behind stage 1 reaches: the scheduler's predicates (engine.cpp Scheduler::run) and
    launch_fir_c / launch_poly / launch_fir_r (kernels.cu) for the stages outside the fused range"""
    tails = opts.get("tails", 2)
    pre_reg = opts.get("ft_prereg", 8)
    out = []
    for i, s in enumerate(st):
        k = s[0]
        if i == 0:
            out.append("stage1")
        elif fused and fused[0] <= i < fused[1]:
            out.append("FT_" + {"firc": "FIRC", "poly": "POLY", "quad": "QUAD", "firr": "FIRR", "m2s": "M2S"}[k])
        elif k == "firc":
            D, T = s[1], s[2]
            if pre_reg > 0 and D > 1 and routes_dfir_reg(D, T):
                out.append("k_dfir_reg")
            elif pre_reg > 0 and D == 1 and T <= 2000:
                out.append("k_fir_reg")          # (the chunk offset of a decimation-1 filter is always 0)
            elif tails >= 1 and D == 1 and T <= TAIL_MAX_TAPS:
                out.append("k_fir_c2")
            elif tails >= 1 and 1 < D <= 64 and T <= TAIL_MAX_TAPS:
                out.append("k_fir_cd")
            else:
                out.append("k_fir_c")
        elif k == "poly":
            L, M, tpp = s[1], s[2], s[3]
            if pre_reg > 0 and tpp <= 512 and (L, M) in POLY_REG:
                out.append("k_poly_reg")
            elif tails >= 1 and (256 * M + L - 1) // L + tpp + 2 <= 8192:
                out.append("k_poly2")
            else:
                out.append("k_poly")
        elif k == "quad":
            out.append("k_quad")
        elif k == "firr":
            if pre_reg > 0 and s[1] <= 2000:
                out.append("k_firr_reg")
            elif tails >= 1 and s[1] <= TAIL_MAX_TAPS:
                out.append("k_fir_r2")
            else:
                out.append("k_fir_r")
        else:
            out.append("k_" + k)
    return out


# ---------------------------------------------------------------------------------------------- CPU: known answers
def test_reference_known_answers():
    """the reference's conventions, bit for bit on fp32 angles: initial phase 0, the wrap threshold P = FL_M_PI_REF with
    the <= -P branch, the step 2P, the scale"""
    for dev, sr in ((75e3, 250e3), (6.25e3, 50e3)):
        inv = inv_dev_of(dev, sr)
        want = np.float32(np.float32(P32) * np.float32(inv))
        half = np.array([1, -1] * 20, np.float32).astype(np.complex64)
        q = quad_f64(half, None, inv, angles32=True)[0].astype(np.float32)
        assert q[0] == 0.0 and q[0].tobytes() == np.float32(0.0).tobytes()
        assert np.array_equal(q[1:].view(np.uint32), np.full(q.size - 1, want).view(np.uint32))
        neg = np.array([1 + 0j, complex(-1.0, -0.0)], np.complex64)
        assert math.copysign(1.0, neg[1].imag) < 0
        q = quad_f64(neg, None, inv, angles32=True)[0].astype(np.float32)
        assert q[1].tobytes() == want.tobytes()
        # a threshold of pi, a '<' on the negative side, or 2 pi as the step would each give another value here
        assert np.float32((P32 - TWO_P) * inv) != want and np.float32(-P32 * inv) != want
        # the float64 reference (exact angles) takes the other branch on (-1, -0) and accepts either
        q64, bq, amb, alt, _ = quad_f64(neg, None, inv)
        assert amb[1] and quad_ratio(np.array([0.0, want]), q64, bq, amb, alt)[1] <= 1.0


# ---------------------------------------------------------------------------------------------- CPU: pins to the oracle
def fm_noise(n, seed):
    """exact fp32 IQ with uniform phase steps in (-pi, pi] (wraps everywhere) and a varying magnitude"""
    rng = np.random.default_rng(seed)
    ph = np.cumsum(rng.uniform(-np.pi, np.pi, n))
    r = rng.uniform(0.05, 1.0, n)
    return (r * np.exp(1j * ph)).astype(np.complex64)


def fm_sweep(n, fs, seed):
    """an FM carrier whose instantaneous frequency swings to +-0.6 fs (past +-fs/2), plus a little noise"""
    t = np.arange(n) / fs
    f = 0.6 * fs * np.sin(2 * np.pi * t * fs / 7919.0 + seed)
    ph = np.cumsum(2 * np.pi * f / fs)
    return (0.7 * np.exp(1j * ph) + noise_iq(n, seed, 0.01)).astype(np.complex64)


def half_turns(n, neg_zero=False):
    x = np.zeros(n, np.complex64)
    x.real[:] = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    if neg_zero:
        x.imag[1::2] = -0.0
    return x


def feed(block, x, sched, in_f, out_f):
    xf = x.view(np.float32) if in_f == 2 else x
    outs, pos = [], 0
    for n in sched:
        y = block.process(xf[in_f * pos: in_f * (pos + n)])
        outs.append(y.reshape(-1, out_f) if out_f == 2 else y)
        pos += n
    return outs


BLOCKS = [("quad_250k", "quad", 75e3, 250e3, None), ("quad_50k", "quad", 6.25e3, 50e3, None),
          ("wfm_lp", "wfm", 75e3, 250e3, True), ("wfm_nolp", "wfm", 75e3, 250e3, False),
          ("nfm_lp", "nfm", 12.5e3, 50e3, True), ("nfm_nolp", "nfm", 12.5e3, 50e3, False)]
BLOCK_IDS = [b[0] for b in BLOCKS]


def block_spec(oracle, name):
    _, kind, p, sr, lp = BLOCKS[BLOCK_IDS.index(name)]
    if kind == "quad":
        inv, h = inv_dev_of(p, sr), None
    elif kind == "wfm":
        inv, h = inv_dev_of(p, sr), (oracle.lowpass(15000.0, 4000.0, sr) if lp else None)
    else:
        inv, h = inv_dev_of(p / 2.0, sr), (oracle.lowpass(p / 2.0, p / 2.0 * 0.1, sr) if lp else None)
    T = h.size if h is not None else 2
    sched = schedule(QUAD_TILE, T, 200000, BLOCK_IDS.index(name))
    return kind, inv, h, sched


def block_reference(x, inv, h):
    q, bq, amb, alt, carry = quad_f64(x, None, inv)
    if h is None:
        return q, bq, amb, alt
    y, b = fir_f64(q, carry, h, 1)
    return y, b, np.zeros(y.size, bool), y


def _block_inputs(name, n):
    seed = 10 + BLOCK_IDS.index(name)
    sr = BLOCKS[BLOCK_IDS.index(name)][3]
    return {"noise": fm_noise(n, seed), "sweep": fm_sweep(n, sr, seed)}


@pytest.mark.parametrize("name", BLOCK_IDS)
def test_block_reference_matches_oracle(oracle, name):
    """the discriminator / audio low-pass reference against the oracle's fp32 blocks (host atan2f) within the same bound, on
    the 0/1-sample and tile-edge schedule: initial phase, scale, wrap constant, tap count, output counts"""
    kind, inv, h, sched = block_spec(oracle, name)
    p = BLOCKS[BLOCK_IDS.index(name)]
    for x in _block_inputs(name, sum(sched)).values():
        blk = {"quad": lambda: oracle.quad(p[2], p[3]), "wfm": lambda: oracle.wfm(p[2], p[3], False, p[4]),
               "nfm": lambda: oracle.nfm(p[3], p[2], p[4])}[kind]()
        outs = feed(blk, x, sched, 2, 1 if kind == "quad" else 2)
        assert [o.shape[0] for o in outs] == list(sched)
        y = np.concatenate(outs)
        if kind != "quad":
            assert np.array_equal(y[:, 0].view(np.uint32), y[:, 1].view(np.uint32))
            y = y[:, 0]
        y64, b, amb, alt = block_reference(x, inv, h)
        r = float(np.max(quad_ratio(y, y64, b, amb, alt)))
        assert r <= 1.0, r


def test_af_blocks_reference_matches_oracle(oracle):
    """AF resampler 250k -> 48k and 50k -> 48k (stereo), the 300 Hz high-pass on (l, r), de-emphasis and the volume"""
    from sdrplusplus_b200 import frontend
    rng = np.random.default_rng(3)
    for (isr, osr) in ((250e3, 48e3), (50e3, 48e3)):
        rp = frontend.resamp_plan(isr, osr)
        assert oracle.resamp_plan(isr, osr)["interp"] == rp["interp"]
        sched = schedule(32 * rp["decim"] * rp["predec_ratio"], rp["taps_per_phase"], 120000, 5)
        x = rng.uniform(-1, 1, (sum(sched), 2)).astype(np.float32)
        outs = feed(oracle.resamp_stereo(isr, osr), x.reshape(-1), sched, 2, 2)
        st = [("fir", D) for D, T in rp["stages"]] + [("poly", rp["interp"], rp["decim"])]
        assert [o.shape[0] for o in outs] == cascade_counts(sched, st)
        y = np.concatenate(outs)
        y64, e = x[:, 0].astype(np.float64) + 1j * x[:, 1], None
        for k, (D, T) in enumerate(rp["stages"]):
            y64, e = fir_f64(y64, e, oracle.decim_taps(rp["predec_ratio"], k), D)
        y64, e = poly_f64(y64, e, oracle.resamp_taps(isr, osr), rp["interp"], rp["decim"])
        assert float(np.max(_ratio_c(y[:, 0] + 1j * y[:, 1], y64, e))) <= 1.0
    hp = oracle.highpass(300.0, 100.0, 48000.0)
    sched = schedule(TS_TILE, hp.size, 60000, 6)
    x = rng.uniform(-1, 1, (sum(sched), 2)).astype(np.float32)
    y = np.concatenate(feed(oracle.fir_cr(hp), x.reshape(-1), sched, 2, 2))
    y64, e = fir_f64(x[:, 0].astype(np.float64) + 1j * x[:, 1], None, hp, 1)
    assert float(np.max(_ratio_c(y[:, 0] + 1j * y[:, 1], y64, e))) <= 1.0
    for tau in (50e-6, 75e-6):
        a, b = deemph_coefs(tau, 48000.0)
        blk = oracle.deemph(tau, 48000.0)
        sched = [0, 1, 7, 3000, 1, 0, 20000]
        y = np.concatenate(feed(blk, x[:sum(sched)].reshape(-1), sched, 2, 2))
        y64, e = deemph_f64(x[:sum(sched), 0].astype(np.float64) + 1j * x[:sum(sched), 1], None, a, b)
        assert float(np.max(_ratio_c(y[:, 0] + 1j * y[:, 1], y64, e))) <= 1.0
        # the GPU kernel's product order (a x + b y), the same value
        yy = np.zeros(2, np.float32)
        for i in range(64):
            yy = (np.float32(a) * x[i] + np.float32(b) * yy).astype(np.float32)
            assert np.array_equal(yy.view(np.uint32), y[i].view(np.uint32))
    v, e = volume_f64(y64, e, 0.7, False)
    assert np.array_equal(v, y64 * float(np.float32(np.float32(0.7) ** np.float32(2))))


def _oracle_vfo_run(oracle, x, fs, sched, cfgs):
    from vfo_settings_oracle import OracleVfo
    oracle.set_rotator_mode(1)
    try:
        v = OracleVfo(oracle, fs, cfgs[0])
        parts, pos = [], 0
        xf = x.view(np.float32)
        for n, c in zip(sched, cfgs):
            v.set(c)
            parts.append(v.process(xf[2 * pos: 2 * (pos + n)]).reshape(-1, 2))
            pos += n
        return parts
    finally:
        oracle.set_rotator_mode(0)


def test_whole_vfo_reference_matches_exact_phase_oracle(oracle):
    """the whole-VFO reference (stage 1 through volume) against the oracle's exact-phase chain: one WFM + AF VFO, one NFM
    VFO and one retune, every output within the bound"""
    from sdrplusplus_b200 import VfoConfig
    fs = 2.4e6
    sched = [0, 1, 7, 50003, 6000, 3, 80001]
    n = sum(sched)
    x = (fm_carrier_at(n, fs, 300e3 + 1234.5, 40e3, 0.4) + fm_carrier_at(n, fs, -400e3, 4e3, 0.4, 1)
         + noise_iq(n, 8, 0.01)).astype(np.complex64)
    wfm = VfoConfig.wfm(300e3 + 1234.5).with_af(48000.0, True, 50e-6).with_volume(0.7)
    nfm = VfoConfig.nfm(-400e3)
    ret = [VfoConfig.wfm(300e3 + 1234.5)] * 4 + [VfoConfig.wfm(-400e3 + 777.0)] * 3
    for cfgs in ([wfm] * len(sched), [nfm] * len(sched), ret):
        ref = _oracle_vfo_run(oracle, x, fs, sched, cfgs)
        y = np.concatenate(ref)
        y64, b, _, _ = vfo_audio_f64(oracle, x.astype(np.complex128), sched, fs, cfgs)
        assert [p.shape[0] for p in ref] == vfo_counts(oracle, fs, cfgs[0], sched)
        assert y.shape[0] == y64.size
        r = float(np.max(_ratio_c(y[:, 0] + 1j * y[:, 1], y64, b)))
        assert r <= 1.0, r


def fm_carrier_at(n, fs, offset, dev, amp, seed=0):
    """an FM carrier with two tones (1 kHz and 3.1 kHz plus a seed-dependent phase)"""
    t = np.arange(n, dtype=np.float64) / fs
    ph = 2 * np.pi * offset * t - (dev * 0.6 / 1000.0) * np.cos(2 * np.pi * 1000.0 * t + seed) \
        - (dev * 0.4 / 3100.0) * np.cos(2 * np.pi * 3100.0 * t + 2 * seed)
    return amp * np.exp(1j * ph)


# ---------------------------------------------------------------------------------------------- the in-situ VFO set
FS_V = 2.4e6
SCHED_V = [0, 1, 7, 100003] + [240000] * 6 + [131071, 5, 0, 160001, 3, 120000, 239999]   # (the repeats: graph replay)
V_OPTIONS = [{}, {"ft_regall": 0}, {"ft_prereg": 0}, {"ft_direct": 0}, {"ft_ob": 64}, {"ft_ob": 301}, {"ft_threads": 128},
             {"ft_threads": 512}, {"tails": 1, "ft_prereg": 0}, {"tails": 0, "ft_prereg": 0}, {"graph": 0}]
V_IDS = ["_".join("%s%d" % kv for kv in sorted(o.items())) or "default" for o in V_OPTIONS]
ON_GRID = 300e3                     # -1/8 turn per sample at 2.4 MS/s: PS 8, the filter bank
PROFILED_CHUNK = 3                  # SCHED_V's first long chunk: outputs on every VFO, not a graph replay


def vfo_set():
    """(config, carrier (offset, deviation, amplitude)) per VFO.  17 WFM VFOs share stage 1's decimation-4 group: the first
    16 fill one launch batch, the 17th (on the filter-bank grid) is alone in the second; the others sit 1234.5 Hz off the
    grid, 120 kHz apart.  The NFM carriers are weak enough not to fade the WFM channels they sit in."""
    from sdrplusplus_b200 import VfoConfig
    v = []
    for k in list(range(11)) + [12, 13, 14, 15]:
        o = -1.02e6 + 120e3 * k + 1234.5
        if k == 14:
            o = -v[3][0].offset                                  # a +- pair (stage 1 shares their sums)
        c = VfoConfig.wfm(o)
        if k in (1, 5):
            c.low_pass = False
        if k == 7:
            c = c.with_af(48000.0, True, 50e-6).with_volume(0.7)
        if k == 9:
            c = c.with_af(48000.0, False, 75e-6)
        v.append((c, (o, 20e3, 0.25)))
    o = 1.05e6 + 1234.5                                          # bandwidth == out rate: identity channel filter, and a
    v.append((VfoConfig.wfm(o, 250e3), (o + 90e3, 45e3, 0.5)))    # carrier swinging past +125 kHz: wraps
    v.append((VfoConfig.wfm(ON_GRID), (ON_GRID, 20e3, 0.25)))
    nfm = [VfoConfig.nfm(-0.96e6), VfoConfig.nfm(-0.48e6), VfoConfig.nfm(0.24e6)]
    nfm[1].low_pass = False
    nfm[2] = nfm[2].with_af(48000.0, True, 0.0)
    v += [(c, (c.offset, 3e3, 0.05)) for c in nfm]
    return v


def test_vfo_set_routes(oracle):
    """the in-situ set: more than 16 FM VFOs at one level (two launch batches), the 17th of stage 1's decimation-4 group
    alone in its batch and on the PS 8 grid (k_xd_pfb), and in every option set the discriminator, audio-FIR, AF-resampler
    and high-pass builds named below are reached"""
    from sdrplusplus_b200 import lib as L
    vs = vfo_set()
    fm = [c for c, _ in vs if c.demod in (L.DEMOD_WFM, L.DEMOD_NFM)]
    assert len(fm) > 16
    from sdrplusplus_b200 import frontend
    d4 = [c for c in fm if frontend.resamp_plan(FS_V, c.out_samplerate)["stages"][0] == (4, 27)]
    assert len(d4) == 17 and d4[16].offset == ON_GRID
    assert pfb_detect([w_u64(ON_GRID, FS_V)], 27) == (8, 1) and pfb_detect([w_u64(c.offset, FS_V) for c in d4[:16]], 27)[0] == 0
    assert (2, (27 + 3) // 4) in PFB_CASES                      # (log2 D, ceil(T / D))
    seen = set()
    for opts in V_OPTIONS:
        fused = 0
        for c in fm:
            st = chain_stages(oracle, FS_V, c)
            fr = fused_range(st, opts)
            fused += fr is not None
            seen |= set(stage_builds(st, opts, fr))
        if opts == {}:
            assert fused == 1                                      # the NFM + AF VFO: its 24/25 AF resampler has no register build
        if opts in ({"ft_regall": 0}, {"ft_prereg": 0}):
            assert fused == len(fm)
    want = {"k_quad", "FT_QUAD", "k_firr_reg", "FT_FIRR", "k_fir_r2", "k_fir_r", "FT_POLY", "k_poly2", "k_poly", "k_poly_reg",
            "k_fir_reg", "FT_FIRC", "k_fir_c", "FT_M2S", "k_m2s", "k_seq", "k_scale", "k_dfir_reg"}
    assert want <= seen, want - seen
    # the WFM + AF VFOs: 250k -> 48k is x4 predecimation, then 96/125 (above the fused tail's 64 classes)
    rp = frontend.resamp_plan(250e3, 48e3)
    assert (rp["predec_ratio"], rp["interp"], rp["decim"]) == (4, 96, 125)
    rp = frontend.resamp_plan(50e3, 48e3)
    assert (rp["predec_ratio"], rp["interp"], rp["decim"]) == (1, 24, 25) and (24, 25) not in POLY_REG


# ---------------------------------------------------------------------------------------------- GPU: stand-alone blocks
@pytest.fixture(scope="module")
def sb():
    import sdrplusplus_b200 as m
    from sdrplusplus_b200 import lib
    L = lib.load()
    assert L.b200_device_count() > 0
    assert L.b200_init(0) == 0
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("name", BLOCK_IDS)
def test_block_vs_float64(sb, oracle, report, name):
    kind, inv, h, sched = block_spec(oracle, name)
    p = BLOCKS[BLOCK_IDS.index(name)]
    mk = {"quad": lambda: sb.Block.quad(p[2], p[3]), "wfm": lambda: sb.Block.wfm(p[2], p[3], False, p[4]),
          "nfm": lambda: sb.Block.nfm(p[3], p[2], p[4])}[kind]
    of = 1 if kind == "quad" else 2
    res = {}
    for sig, x in _block_inputs(name, sum(sched)).items():
        blk = mk()
        outs = feed(blk, x, sched, 2, of)
        assert [o.shape[0] for o in outs] == list(sched)
        y = np.concatenate(outs)
        if of == 2:
            assert np.array_equal(y[:, 0].view(np.uint32), y[:, 1].view(np.uint32))
            y = y[:, 0]
        y64, b, amb, alt = block_reference(x, inv, h)
        r = quad_ratio(y, y64, b, amb, alt)
        k = int(np.argmax(r))
        q_amb = quad_f64(x, None, inv)[2]
        reach = q_amb.astype(np.float64) if h is None else fir_f64(q_amb.astype(np.float64), None, np.abs(h), 1)[0]
        g = _gate_clean(y.astype(np.float64), y64, reach == 0, list(sched))
        res[sig] = dict(g, max_err_over_bound=float(r[k]), worst_output=k, ambiguous_wraps=int(q_amb.sum()),
                        wraps=int(np.sum(np.abs(np.diff(np.angle(x.astype(np.complex128)))) > P32)))
        _check(res[sig], sig)
        blk.reset()
        again = np.concatenate(feed(blk, x, sched, 2, of))
        again = again[:, 0] if of == 2 else again
        assert np.array_equal(again.view(np.uint32), y.view(np.uint32))
        blk.close()
    # the half-turn known answers, bit for bit (the low-pass-on blocks filter them: checked above only)
    if h is None:
        want = np.float32(np.float32(P32) * np.float32(inv))
        for nz in (False, True):
            x = half_turns(sum(sched), nz)
            blk = mk()
            y = np.concatenate(feed(blk, x, sched, 2, of))
            blk.close()
            y = y[:, 0] if of == 2 else y
            assert y[0] == 0.0 and np.all(y[1:].view(np.uint32) == want.view(np.uint32)), (nz, np.flatnonzero(y[1:] != want)[:8])
    report["fm_audio_f64_block_" + name] = res


# ---------------------------------------------------------------------------------------------- GPU: in the front end
@pytest.fixture(scope="module")
def v_input():
    n = sum(SCHED_V)
    x = noise_iq(n, 515, 0.01).astype(np.complex128)
    for k, (c, (o, dev, amp)) in enumerate(vfo_set()):
        x = x + fm_carrier_at(n, FS_V, o, dev, amp, k)
    return x.astype(np.complex64)


@pytest.fixture(scope="module")
def v_reference(oracle, v_input):
    xr = v_input.astype(np.complex128)
    return [vfo_audio_f64(oracle, xr, SCHED_V, FS_V, [c] * len(SCHED_V)) for c, _ in vfo_set()]


def _front_end(sb, fs, max_chunk, opts):
    """a front end with the case's options, set before its VFOs are added"""
    fe = sb.FrontEnd(fs, max_chunk)
    for k, v in opts.items():
        fe.set_option(k, v)
    return fe


TAIL_KERNELS = {"k_quad", "k_firr_reg", "k_fir_r2", "k_fir_r", "k_poly_reg", "k_poly2", "k_poly", "k_fir_reg", "k_fir_c2",
                "k_fir_cd", "k_fir_c", "k_dfir_reg", "k_tail_fused", "k_m2s", "k_seq", "k_scale"}


def _kernel(build):
    return "k_tail_fused" if build.startswith("FT_") else build


def kernels_of(fn):
    """names of the kernels fn() launches (torch.profiler, CUDA activity: every kernel of the process, the library's included)"""
    import re
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = set()
    for e in prof.events():
        m = re.search(r"\bk_[a-z0-9_]+", e.name)
        if m:
            names.add(m.group(0))
    return names


def _audio_gate(parts, y64, b, reach, restarts=()):
    """every output within its bound, L == R (every VFO here is mono), and the gain and edge gates of f64_ref._gate_vfo on
    the left channel over the outputs that ill-conditioned discriminator samples reach with less than one fp32 rounding of
    the output's scale (those carry the discriminator's cap in their bound, which a gain fit cannot resolve)"""
    y = np.concatenate(parts)
    assert y.shape[0] == y64.size, (y.shape, y64.size)
    r = _ratio_c(y[:, 0] + 1j * y[:, 1], y64, b)
    k = int(np.argmax(r)) if r.size else -1
    assert np.array_equal(y[:, 0].view(np.uint32), y[:, 1].view(np.uint32))
    clean = reach <= U * float(np.abs(y64).max(initial=0.0))
    g = _gate_clean(y[:, 0].astype(np.float64), y64.real, clean, [p.shape[0] for p in parts], restarts)
    return dict(g, max_err_over_bound=float(r[k]) if r.size else 0.0, worst_output=k)



def _check(res, name):
    assert res["max_err_over_bound"] <= 1.0, (name, res)
    assert res["abs_g_minus_1"] < 2e-6, (name, res)
    assert res["edge_over_p999"] <= 4.0, (name, res)


@pytest.mark.gpu
@pytest.mark.parametrize("opts", V_OPTIONS, ids=V_IDS)
def test_fm_vfos_in_front_end_vs_float64(sb, oracle, v_input, v_reference, report, opts):
    vs = vfo_set()
    fe = _front_end(sb, FS_V, max(SCHED_V), opts)
    try:
        ids = [fe.add_vfo(c) for c, _ in vs]
        fused = fe.stat("fused_chains")
        got = {vid: [] for vid in ids}
        pos = 0
        ran = None
        for c, n in enumerate(SCHED_V):
            def step():
                outs, _ = fe.process(v_input[pos:pos + n])
                for vid in ids:
                    got[vid].append(outs[vid])
            if c == PROFILED_CHUNK:
                ran = kernels_of(step)
            else:
                step()
            pos += n
        hits = fe.stat("graph_hits")
    finally:
        fe.close()
    res = []
    for k, vid in enumerate(ids):
        c = vs[k][0]
        y64, b, namb, reach = v_reference[k]
        assert [p.shape[0] for p in got[vid]] == vfo_counts(oracle, FS_V, c, SCHED_V)
        st = chain_stages(oracle, FS_V, c)
        fr = fused_range(st, opts)
        r = _audio_gate(got[vid], y64, b, reach)
        r.update(ambiguous_wraps=namb, builds=stage_builds(st, opts, fr), offset=c.offset)
        res.append(r)
    tag = V_IDS[V_OPTIONS.index(opts)]
    want_fused = sum(fused_range(chain_stages(oracle, FS_V, c), opts) is not None for c, _ in vs)
    report["fm_audio_f64_in_situ_2p4msps_" + tag] = {
        "per_vfo": res, "graph_hits": int(hits), "fused_chains": int(fused), "eligible_for_fusion": want_fused,
        "max_err_over_bound": max(r["max_err_over_bound"] for r in res), "max_abs_g_minus_1": max(r["abs_g_minus_1"] for r in res),
        "max_edge_over_p999": max(r["edge_over_p999"] for r in res), "ambiguous_wraps": sum(r["ambiguous_wraps"] for r in res)}
    # the builds that ran in one chunk with outputs on every VFO are those the mirror names: stage 1's filter bank for the
    # VFO alone on the grid, and behind stage 1 exactly the per-VFO builds (a chain the stage list makes eligible for the
    # fused tail may still run per stage when its shared-memory plan, decided at run time, does not fit)
    need, allow = set(), set()
    for c, _ in vs:
        st = chain_stages(oracle, FS_V, c)
        fr = fused_range(st, opts)
        need |= {_kernel(b) for b in stage_builds(st, opts, fr)} & TAIL_KERNELS
        allow |= {_kernel(b) for b in stage_builds(st, opts, None)} & TAIL_KERNELS
    allow |= need
    report["fm_audio_f64_in_situ_2p4msps_" + tag]["kernels_run"] = sorted(ran)
    assert "k_xd_pfb" in ran and "k_xd_pipe" in ran, sorted(ran)
    if fused == want_fused:
        assert ran & TAIL_KERNELS == need, (sorted(ran & TAIL_KERNELS), sorted(need))
    else:
        assert need <= ran & TAIL_KERNELS <= allow, (sorted(ran & TAIL_KERNELS), sorted(need), sorted(allow))
    assert (fused == want_fused) if not opts else (0 < fused <= want_fused or fused == want_fused == 0), (fused, want_fused)
    for r in res:
        _check(r, r["offset"])
    if not opts:
        assert hits > 0


@pytest.mark.gpu
def test_wfm_vfos_behind_tma_stage1_100msps(sb, oracle, report):
    """8 WFM VFOs on the 5 MHz grid at 100 MS/s (the bench's VFO type): k_xd_tma, then the register kernels and k_quad"""
    from sdrplusplus_b200 import VfoConfig
    fs = 100e6
    sched = [0, 1, 300001] + [1 << 20] * 3 + [7, 499999, 777777]
    n = sum(sched)
    offs = [5e6, -5e6, 15e6, -15e6, 25e6, -25e6, 35e6, -35e6]
    x = noise_iq(n, 4244, 0.01).astype(np.complex128)
    for k, o in enumerate(offs):
        x = x + fm_carrier_at(n, fs, o, 40e3, 0.2, k)
    x = x.astype(np.complex64)
    cfgs = [VfoConfig.wfm(o) for o in offs]
    fe = _front_end(sb, fs, max(sched), {})
    try:
        ids = [fe.add_vfo(c) for c in cfgs]
        t0 = fe.stat("s1_tma_launches")
        got = {vid: [] for vid in ids}
        pos = 0
        for m in sched:
            outs, _ = fe.process(x[pos:pos + m])
            for vid in ids:
                got[vid].append(outs[vid])
            pos += m
        tma = fe.stat("s1_tma_launches") - t0
        fused = fe.stat("fused_chains")
    finally:
        fe.close()
    assert tma > 0 and fused == 0
    xr = x.astype(np.complex128)
    res = []
    for c, vid in zip(cfgs, ids):
        y64, b, namb, reach = vfo_audio_f64(oracle, xr, sched, fs, [c] * len(sched))
        r = _audio_gate(got[vid], y64, b, reach)
        r["ambiguous_wraps"] = namb
        res.append(r)
    report["fm_audio_f64_in_situ_100msps"] = {"per_vfo": res, "tma_launches": int(tma),
                                              "max_err_over_bound": max(r["max_err_over_bound"] for r in res),
                                              "max_abs_g_minus_1": max(r["abs_g_minus_1"] for r in res),
                                              "max_edge_over_p999": max(r["edge_over_p999"] for r in res)}
    for r, o in zip(res, offs):
        _check(r, o)


def change_run():
    """(chunk sizes, per-VFO per-chunk configurations): each change at a chunk boundary, followed by a short chunk"""
    from dataclasses import replace
    from sdrplusplus_b200 import VfoConfig
    base = [VfoConfig.wfm(300e3 + 1234.5).with_af(48000.0, False, 50e-6).with_volume(0.7),
            VfoConfig.nfm(-400e3).with_af(48000.0, False, 0.0).with_volume(1.3)]
    sched, cw, cn = [], [], []

    def add(n, w, m):
        sched.append(n)
        cw.append(w)
        cn.append(m)
    w, m = base
    add(120001, w, m)
    w = replace(w, offset=-200e3 + 77.0)                                  # retune
    add(3, w, m)
    add(90001, w, m)
    w = replace(w, bandwidth=250e3)                                       # 150k -> 250k (identity channel filter)
    m = replace(m, af_high_pass=True)                                     # high-pass on (restages the fused tail)
    add(5, w, m)
    add(100001, w, m)
    w = replace(w, bandwidth=120e3, af_deemph_tau=75e-6)                  # 250k -> 120k (cleared history), tau change
    m = replace(m, af_high_pass=False, af_muted=True)                     # high-pass off, mute
    add(1, w, m)
    add(110001, w, m)
    w = replace(w, af_volume=0.3)
    m = replace(m, af_muted=False)
    add(7, w, m)
    add(150000, w, m)
    return sched, [cw, cn]


@pytest.mark.gpu
def test_changes_at_chunk_boundaries(sb, oracle, report):
    fs = FS_V
    sched, cfgs = change_run()
    n = sum(sched)
    x = (fm_carrier_at(n, fs, 300e3 + 1234.5, 30e3, 0.3) + fm_carrier_at(n, fs, -200e3 + 77.0, 30e3, 0.3, 1)
         + fm_carrier_at(n, fs, -400e3, 3e3, 0.3, 2) + noise_iq(n, 99, 0.01)).astype(np.complex64)
    fe = _front_end(sb, fs, max(sched), {})
    try:
        ids = [fe.add_vfo(c[0]) for c in cfgs]
        got = {vid: [] for vid in ids}
        pos = 0
        for k, m in enumerate(sched):
            for vid, c in zip(ids, cfgs):
                if k and c[k] != c[k - 1]:
                    fe.set_vfo_config(vid, c[k])
            outs, _ = fe.process(x[pos:pos + m])
            for vid in ids:
                got[vid].append(outs[vid])
            pos += m
    finally:
        fe.close()
    xr = x.astype(np.complex128)
    res = {}
    for name, vid, c in zip(("wfm_af", "nfm_af"), ids, cfgs):
        y64, b, namb, reach = vfo_audio_f64(oracle, xr, sched, fs, c)
        # identity -> low-pass restarts the channel filter from cleared history: a start transient, like the stream's
        restarts = [k for k in range(1, len(c)) if c[k].bandwidth != c[k - 1].bandwidth and c[k - 1].bandwidth == c[k].out_samplerate]
        res[name] = _audio_gate(got[vid], y64, b, reach, restarts)
        res[name]["ambiguous_wraps"] = namb
    report["fm_audio_f64_changes"] = res
    for name, r in res.items():
        _check(r, name)

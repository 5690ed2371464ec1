"""The stereo branch of BroadcastFM (k_st_pilot, k_st_pll, k_st_mix and the 15 kHz low-pass over l + j r) and PowerSquelch
(k_sq_sum, k_sq_gate) against float64 references, sample by sample and chunk by chunk, from output 0 of the stream: as
stand-alone blocks and inside front-end VFOs.  f64_ref's module docstring derives both bounds (stereo_f64, squelch_f64).

The test programmes put the pilot off the PLL's initial 19 kHz (+37 Hz, -61 Hz, and per-VFO offsets within +-100 Hz in
the front end), so the loop's carried frequency (k_st_pll's state[1]) moves away from its initial value and every chunk
edge has to carry it; L != R, so the difference channel S = (l - r) / 2 is a signal of its own, gated with its own fitted
gain.  The PLL's frequency clamp (+-250 Hz) is active during every pull-in; the reference follows it exactly where the
float64 frequency is clamped or free by more than its bound.  The stand-alone blocks assert that no step is ambiguous (an
err wrap or a clamp within the bound), so their per-sample bound is tight from output 0.  Inside the front end stage 1's
a-priori bound widens the pilot angle bound until the pull-in has ambiguous steps; from the first one the vco angle bound
is pi, which still holds, so every output is checked against it, and the fine sensitivity there comes from the fitted M and
S gains (|g - 1| < 2e-6) and edge-against-interior ratios (<= 4) over the outputs after the pull-in.  Squelch chunks are
scaled to sit 4 bounds above or below the level, so a lost CTA, a lost tail element or a mis-rounded decision flips
a chunk.  No tolerance here is fitted to a run.
"""
import math

import numpy as np
import pytest

from f64_ref import (P32, U, _chunk_index, _gate_clean, _ratio_c, inv_dev_of, quad_f64, schedule, squelch_f64,
                     squelch_nparts, stereo_delay, stereo_f64, stereo_taps, vfo_audio_f64, vfo_counts)
from util import noise_iq

ST_TILE = 256                                   # k_st_pilot / k_st_mix outputs per CTA
SQ_TILE_CAP = 256 * 4096                        # SQ_MAXPARTS CTAs of 4096 samples: k_sq_sum strides beyond


# ---------------------------------------------------------------------------------------------- signals
def mpx(t, pilot_hz, seed):
    """a stereo multiplex with L != R: L+R and L-R tones (seed-dependent), the pilot, L-R on the subcarrier at twice the
    pilot's phase"""
    rng = np.random.default_rng(seed)
    f1, f2, f3 = rng.uniform(300, 4000, 3)
    ph = rng.uniform(0, 2 * np.pi, 4)
    lpr = 0.35 * np.sin(2 * np.pi * f1 * t + ph[0]) + 0.1 * np.sin(2 * np.pi * f2 * t + ph[1])
    lmr = 0.3 * np.sin(2 * np.pi * f3 * t + ph[2])
    wp = 2 * np.pi * pilot_hz * t + ph[3]
    return lpr + 0.1 * np.sin(wp) + lmr * np.sin(2 * wp)


def fm_stereo_iq(n, fs, pilot_hz, seed, offset=0.0, amp=0.5, dev=75e3):
    t = np.arange(n, dtype=np.float64) / fs
    m = mpx(t, pilot_hz, seed)
    ph = 2 * np.pi * offset * t + 2 * np.pi * dev * np.cumsum(m) / fs
    return amp * np.exp(1j * ph)


PROGRAMMES = {"p37": (19037.0, 1), "m61": (18939.0, 2)}


def block_input(fs, name):
    pilot, seed = PROGRAMMES[name]
    n = sum(block_schedule(fs))
    return (fm_stereo_iq(n, fs, pilot, seed) + noise_iq(n, 30 + seed, 0.002)).astype(np.complex64)


def block_schedule(fs, long=True):
    T = stereo_taps(fs).size
    dl, hist = stereo_delay(T), T - 1
    s = schedule(ST_TILE, T, 200000, int(fs) % 97)
    s += [0, 1, dl - 1, dl, dl + 1, 0, hist - 1, hist, hist + 1, 1]
    return s + ([1000000] if long else [3001])


def feed(block, x, sched):
    xf = x.view(np.float32)
    outs, pos = [], 0
    for n in sched:
        outs.append(block.process(xf[2 * pos: 2 * (pos + n)]).reshape(-1, 2))
        pos += n
    return outs


def block_reference(x, fs, lowpass):
    """discriminator (dev 75 kHz) + stereo branch: (l + j r, bound, info, q64, e_q)"""
    inv = inv_dev_of(75e3, fs)
    q, bq, amb, alt, carry = quad_f64(x, None, inv)
    reach = np.where(amb | (bq >= 2.0 * P32 * inv), carry, 0.0)
    y, b, info = stereo_f64(q, carry, fs, lowpass, reach)
    info["discriminator_ambiguous"] = int(amb.sum())
    return y, b, info, q, carry


def ms_gate(y, y64, b, reach, counts, restarts=()):
    """every output within its bound on l and on r; fitted gains and edge ratios of M = (l + r) / 2 and S = (l - r) / 2
    over the outputs the ill-conditioned steps do not reach"""
    y = np.asarray(y, np.float64)
    assert y.shape[0] == y64.size, (y.shape, y64.size)
    r = _ratio_c(y[:, 0] + 1j * y[:, 1], y64, b)
    k = int(np.argmax(r)) if r.size else -1
    clean = reach <= U * float(np.abs(y64).max(initial=0.0))
    gm = _gate_clean((y[:, 0] + y[:, 1]) / 2, (y64.real + y64.imag) / 2, clean, counts, restarts)
    gs = _gate_clean((y[:, 0] - y[:, 1]) / 2, (y64.real - y64.imag) / 2, clean, counts, restarts)
    return {"max_err_over_bound": float(r[k]) if r.size else 0.0, "worst_output": k,
            "M": {kk: gm[kk] for kk in ("abs_g_minus_1", "edge_over_p999", "rel_rms", "gated_outputs")},
            "S": {kk: gs[kk] for kk in ("abs_g_minus_1", "edge_over_p999", "rel_rms", "gated_outputs")}}


def check_ms(res, name):
    assert res["max_err_over_bound"] <= 1.0, (name, res)
    for ch in ("M", "S"):
        assert res[ch]["abs_g_minus_1"] < 2e-6, (name, ch, res)
        assert res[ch]["edge_over_p999"] <= 4.0, (name, ch, res)


# ---------------------------------------------------------------------------------------------- CPU: pins to the oracle
@pytest.mark.parametrize("fs", [250e3, 200e3])
@pytest.mark.parametrize("lowpass", [True, False])
def test_stereo_reference_matches_oracle(oracle, fs, lowpass):
    """the stereo reference against the oracle's fp32 BroadcastFM (glibc atan2f, cosf, sinf), every output from output 0 on
    short and edge chunks: a wrong alpha, beta, f0, fmin, fmax, tap set or delay shows in the pull-in first"""
    from f64_ref import pll_constants
    T = stereo_taps(fs).size
    assert (T, stereo_delay(T)) == ({250e3: 317, 200e3: 253}[fs], {250e3: 159, 200e3: 127}[fs])
    c = pll_constants(fs)
    if fs == 250e3:
        assert abs(c["alpha"] - 0.24565) < 1e-5 and abs(c["beta"] - 0.034740) < 1e-6
    sched = block_schedule(fs, long=False)
    for name in PROGRAMMES:
        x = block_input(fs, name)[:sum(sched)]
        blk = oracle.wfm(75e3, fs, True, lowpass)
        outs = feed(blk, x, sched)
        assert [o.shape[0] for o in outs] == list(sched)
        y = np.concatenate(outs)
        y64, b, info, _, _ = block_reference(x, fs, lowpass)
        assert info["ambiguous_wraps"] == info["ambiguous_clamps"] == 0, info
        assert 0 < info["last_clamped"] < 5000, info
        r = _ratio_c(y[:, 0] + 1j * y[:, 1], y64, b)
        assert float(r.max()) <= 1.0, (name, float(r.max()), int(np.argmax(r)))
        # and the bound is not vacuous: the loop follows the pilot, L - R is there
        assert float(np.abs(y[:, 0] - y[:, 1]).max()) > 0.1


def test_stereo_reference_sees_a_wrong_delay(oracle):
    """the comparison above fails for a reference whose delay is one sample short"""
    import f64_ref
    fs, sched = 250e3, [5000, 3, 20000]
    x = block_input(fs, "p37")[:sum(sched)]
    y = np.concatenate(feed(oracle.wfm(75e3, fs, True, False), x, sched))
    keep = f64_ref.stereo_delay
    try:
        f64_ref.stereo_delay = lambda T: (T - 1) // 2
        y64, b, _, _, _ = block_reference(x, fs, False)
        assert float(_ratio_c(y[:, 0] + 1j * y[:, 1], y64, b).max()) > 1.0
    finally:
        f64_ref.stereo_delay = keep


def squelch_chunks(sizes, level, seed):
    """noise chunks scaled so that each float64 mean of |x| sits at level +- 4 bounds (alternating), rounded to fp32, with
    one chunk carrying a single sample 10^4 times the rest"""
    rng = np.random.default_rng(seed)
    parts = []
    for k, n in enumerate(sizes):
        x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
        if k == 3 and n > 1:
            x[n // 2] *= 1e4
        bd = squelch_f64(x, None, [n], level)[2][0]
        want = level + (4.0 if k % 2 == 0 else -4.0) * bd
        mean = float(np.abs(x.astype(np.complex128)).mean())
        parts.append((x.astype(np.complex128) * (10.0 ** (want / 10.0) / mean)).astype(np.complex64))
    return parts


SQ_SIZES = [1, 2, 255, 256, 4095, 4096, 4097, 65537, 999999, 1000000]
SQ_LEVEL = -23.7


def test_squelch_reference_matches_oracle(oracle, report):
    """decisions against the oracle's sequential fp32 sum on every chunk unambiguous for both; the oracle's own bound is
    (n - 1) u of the sum, so near-threshold chunks where it differs from float64 are the reference's floor, reported"""
    parts = squelch_chunks(SQ_SIZES, SQ_LEVEL, 7)
    x = np.concatenate(parts)
    counts = [p.size for p in parts]
    dec, mar, bd, amb = squelch_f64(x, None, counts, SQ_LEVEL)
    assert not amb.any() and list(dec) == [k % 2 == 0 for k in range(len(counts))], (mar, bd)
    blk = oracle.squelch(SQ_LEVEL)
    floor = []
    for k, p in enumerate(parts):
        y = blk.process(p.view(np.float32)).view(np.complex64)
        is_open = np.array_equal(y.view(np.uint32), p.view(np.uint32))
        assert is_open or not np.any(y.view(np.uint32)), k
        o_bound = 10.0 / math.log(10.0) * (p.size + 4) * U + 1e-6
        if abs(mar[k]) > o_bound:
            assert is_open == dec[k], (k, mar[k], bd[k])
        elif is_open != dec[k]:
            floor.append(k)
    report["squelch_reference_oracle_floor"] = {"chunks_differing_near_threshold": floor, "sizes": counts}
    # wider margins: every decision agrees
    for lv in (-60.0, 10.0):
        d = squelch_f64(x, None, counts, lv)[0]
        blk = oracle.squelch(lv)
        for k, p in enumerate(parts):
            y = blk.process(p.view(np.float32)).view(np.complex64)
            assert np.array_equal(y.view(np.uint32), p.view(np.uint32)) == d[k]


def test_squelch_nparts_mirror():
    assert [squelch_nparts(n) for n in (0, 1, 4096, 4097, 1 << 20, (1 << 20) + 1, 1 << 24)] == [1, 1, 1, 2, 256, 256, 256]


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
@pytest.mark.parametrize("fs", [250e3, 200e3])
@pytest.mark.parametrize("lowpass", [True, False])
def test_stereo_block_vs_float64(sb, report, fs, lowpass):
    sched = block_schedule(fs)
    T = stereo_taps(fs).size
    dl = stereo_delay(T)
    res = {}
    for name in PROGRAMMES:
        x = block_input(fs, name)
        blk = sb.Block.wfm(75e3, fs, stereo=True, lowpass=lowpass)
        outs = feed(blk, x, sched)
        assert [o.shape[0] for o in outs] == list(sched)
        y = np.concatenate(outs)
        y64, b, info, q64, e_q = block_reference(x, fs, lowpass)
        info.pop("theta"), info.pop("vco_bound")
        reach = info.pop("reach")
        assert info["ambiguous_wraps"] == info["ambiguous_clamps"] == 0, info
        r = ms_gate(y, y64, b, reach, list(sched))
        r.update(info)
        # known answers: the delay line starts with zeros; with the low-pass off M is the delayed discriminator output
        assert np.all(y[:dl] == 0.0), np.flatnonzero(y[:dl])[:8]
        if not lowpass:
            md = np.concatenate([np.zeros(dl), q64])[:y.shape[0]]
            e_md = np.concatenate([np.zeros(dl), e_q])[:y.shape[0]]
            yy = y.astype(np.float64)
            m = (yy[:, 0] + yy[:, 1]) / 2
            lim = e_md + U * (np.abs(yy[:, 0]) + np.abs(yy[:, 1])) / 2
            r["M_vs_delayed_discriminator"] = float(np.max(np.abs(m - md) - lim))
            assert np.all(np.abs(m - md) <= lim), np.flatnonzero(np.abs(m - md) > lim)[:8]
        # reset() mid-stream: the bits of a fresh block
        blk.reset()
        k = 24
        again = np.concatenate(feed(blk, x[:sum(sched[:k])], sched[:k]))
        assert np.array_equal(again.view(np.uint32), y[:again.shape[0]].view(np.uint32))
        assert np.all(again[:dl] == 0.0)
        blk.close()
        res[name] = r
        check_ms(r, name)
    report["stereo_f64_block_%dk_lp%d" % (int(fs / 1e3), int(lowpass))] = res


@pytest.mark.gpu
def test_squelch_block_vs_float64(sb, report):
    parts = squelch_chunks(SQ_SIZES, SQ_LEVEL, 11)
    counts = [p.size for p in parts]
    x = np.concatenate(parts)
    dec, mar, bd, amb = squelch_f64(x, None, counts, SQ_LEVEL)
    assert not amb.any()
    blk = sb.Block.squelch(SQ_LEVEL)
    got = []
    for p in parts:
        y = blk.process(p.view(np.float32)).view(np.complex64)
        is_open = np.array_equal(y.view(np.uint32), p.view(np.uint32))
        assert is_open or (y.size == p.size and not np.any(y.view(np.uint32))), p.size
        got.append(is_open)
    blk.close()
    assert got == list(dec), (got, list(dec), list(mar))
    # known answers: unit samples on the axes have mean exactly 1 and log10f(1) = 0: open at 0 dB (>=), closed just above
    ax = np.tile(np.array([1, 1j, -1, -1j], np.complex64), 1025)
    z = np.zeros(4097, np.complex64)
    for lv, want in ((0.0, True), (float(np.nextafter(np.float32(0), np.float32(1))), False)):
        blk = sb.Block.squelch(lv)
        y = blk.process(ax.view(np.float32)).view(np.complex64)
        assert np.array_equal(y.view(np.uint32), ax.view(np.uint32)) == want and (want or not np.any(y.view(np.uint32)))
        y = blk.process(z.view(np.float32)).view(np.complex64)
        assert y.size == z.size and not np.any(y.view(np.uint32))
        blk.close()
    report["squelch_f64_block"] = {"sizes": counts, "margin_over_bound": [float(abs(m) / b) for m, b in zip(mar, bd)],
                                   "ambiguous_chunks": int(amb.sum())}


# ---------------------------------------------------------------------------------------------- GPU: in the front end
FS_V = 2.4e6
# at the stereo stage (2.4 MS/s -> 250 kS/s, 9.6 : 1): 0, 1, < delay and < hist outputs, long chunks, repeats (graph replay)
SCHED_V = [0, 8, 1000, 2900, 100003] + [96000] * 5 + [5, 0, 131071, 1500, 3, 200001]


def stereo_vfo_set():
    """(config, carrier) per VFO: three stereo VFOs (low-pass off; the AF chain; a 200 kS/s IF), two mono WFM, one NFM"""
    from sdrplusplus_b200 import VfoConfig
    from dataclasses import replace
    s1 = VfoConfig.wfm_stereo(-700e3 + 1234.5)
    s1.low_pass = False
    s2 = VfoConfig.wfm_stereo(-250e3 + 777.0).with_af(48000.0, True, 50e-6).with_volume(0.7)
    s3 = replace(VfoConfig.wfm_stereo(300e3 - 432.1), out_samplerate=200e3)
    v = [(s1, ("st", 19037.0, 21)), (s2, ("st", 18939.0, 22)), (s3, ("st", 19071.0, 23)),
         (VfoConfig.wfm(650e3 + 55.5), ("mono", 40e3, 24)), (VfoConfig.wfm(-1.0e6 + 99.0), ("mono", 30e3, 25)),
         (VfoConfig.nfm(900e3), ("nfm", 3e3, 26))]
    return v


def fe_input(fs, vs, n, seed):
    t = np.arange(n, dtype=np.float64) / fs
    x = noise_iq(n, seed, 0.005).astype(np.complex128)
    for c, (kind, p, sd) in vs:
        if kind == "st":
            x = x + fm_stereo_iq(n, fs, p, sd, c.offset, 0.25)
        else:
            ph = 2 * np.pi * c.offset * t - (p / 1000.0) * np.cos(2 * np.pi * 1000.0 * t + sd)
            x = x + (0.25 if kind == "mono" else 0.05) * np.exp(1j * ph)
    return x.astype(np.complex64)


def _front_end(sb, fs, max_chunk, opts):
    fe = sb.FrontEnd(fs, max_chunk)
    for k, v in opts.items():
        fe.set_option(k, v)
    return fe


def run_front_end(sb, fs, cfgs, x, sched, opts=None, levels=None, reset_at=None):
    fe = _front_end(sb, fs, max(sched), opts or {})
    try:
        ids = [fe.add_vfo(c) for c in cfgs]
        got = {vid: [] for vid in ids}
        pos = 0
        for k, n in enumerate(sched):
            if reset_at is not None and k == reset_at:
                fe.reset()
                got = {vid: [] for vid in ids}
                pos = 0
            if levels is not None:
                for vid, c, lv in zip(ids, cfgs, levels):
                    if lv is not None:
                        c.squelch_level = float(lv[k])
                        fe.set_vfo_config(vid, c)
            outs, _ = fe.process(x[pos:pos + n])
            for vid in ids:
                got[vid].append(outs[vid])
            pos += n
        return [got[vid] for vid in ids], fe.stat("graph_hits")
    finally:
        fe.close()


V_OPTIONS = [{}, {"ft_regall": 0}, {"tails": 1, "ft_prereg": 0}, {"tails": 0, "ft_prereg": 0}, {"graph": 0}]
V_IDS = ["_".join("%s%d" % kv for kv in sorted(o.items())) or "default" for o in V_OPTIONS]


def gate_vfo(cfg, parts, ref):
    """one VFO of the front end against its float64 reference (y64, bound, ambiguous wraps, reach, info): every output of l
    and of r within its bound; a stereo VFO's M and S gains and edge ratios, a mono VFO's L == R and its gain and edge"""
    from sdrplusplus_b200 import lib as L
    y64, b, namb, reach, info = ref
    y = np.concatenate(parts)
    counts = [p.shape[0] for p in parts]
    assert y.shape[0] == y64.size, (y.shape, y64.size)
    yy = y.astype(np.float64)
    rl = _ratio_c(yy[:, 0], y64.real, b)
    rr = _ratio_c(yy[:, 1], y64.imag, b)
    res = {"offset": cfg.offset, "l_max_err_over_bound": float(rl.max()), "r_max_err_over_bound": float(rr.max()),
           "discriminator_ambiguous_wraps": namb}
    if cfg.demod == L.DEMOD_WFM_STEREO:
        res.update(ms_gate(y, y64, b, reach, counts))
        st = info["stereo"]
        res.update({k: st[k] for k in ("ambiguous_wraps", "ambiguous_clamps", "ill_steps", "last_clamped", "settled_from",
                                        "vacuous_from")})
        res["l_minus_r_rms"] = float(np.sqrt(np.mean((yy[:, 0] - yy[:, 1]) ** 2)))
    else:
        assert np.array_equal(y[:, 0].view(np.uint32), y[:, 1].view(np.uint32))
        clean = reach <= U * float(np.abs(y64).max(initial=0.0))
        g = _gate_clean(yy[:, 0], y64.real, clean, counts)
        res.update({"max_err_over_bound": max(res["l_max_err_over_bound"], res["r_max_err_over_bound"]),
                    "M": {k: g[k] for k in ("abs_g_minus_1", "edge_over_p999", "rel_rms", "gated_outputs")},
                    "S": {"abs_g_minus_1": 0.0, "edge_over_p999": 0.0}})
    res["max_err_over_bound"] = max(res["l_max_err_over_bound"], res["r_max_err_over_bound"])
    return res


def references(oracle, vs, x, sched, fs):
    xr = x.astype(np.complex128)
    out = []
    for c, _ in vs:
        info = {}
        out.append(vfo_audio_f64(oracle, xr, sched, fs, [c] * len(sched), info=info) + (info,))
    return out


@pytest.fixture(scope="module")
def v_case(oracle):
    vs = stereo_vfo_set()
    x = fe_input(FS_V, vs, sum(SCHED_V), 515)
    return vs, x, references(oracle, vs, x, SCHED_V, FS_V)


@pytest.mark.gpu
@pytest.mark.parametrize("opts", V_OPTIONS, ids=V_IDS)
def test_stereo_vfos_in_front_end_vs_float64(sb, oracle, v_case, report, opts):
    """three stereo VFOs in one batch (low-pass off; the AF chain with L != R through the resampler, the high-pass on
    l + j r and the two de-emphasis channels; a 200 kS/s IF) beside two mono WFM VFOs and one NFM VFO"""
    vs, x, refs = v_case
    cfgs = [c for c, _ in vs]
    parts, hits = run_front_end(sb, FS_V, cfgs, x, SCHED_V, opts)
    res = []
    for c, p, ref in zip(cfgs, parts, refs):
        assert [q.shape[0] for q in p] == vfo_counts(oracle, FS_V, c, SCHED_V)
        res.append(gate_vfo(c, p, ref))
    tag = V_IDS[V_OPTIONS.index(opts)]
    report["stereo_f64_in_situ_2p4msps_" + tag] = {"per_vfo": res, "graph_hits": int(hits)}
    for r in res:
        check_ms(r, r["offset"])
    assert res[1]["l_minus_r_rms"] > 0.01                 # the AF VFO carries L != R to its output
    if not opts:
        assert hits > 0
    # the stage sizes the schedule reaches at the stereo stage: 0, 1, fewer than delay, fewer than hist outputs
    st_counts = vfo_counts(oracle, FS_V, cfgs[0], SCHED_V)
    dl = stereo_delay(stereo_taps(250e3).size)
    assert 0 in st_counts and 1 in st_counts and any(1 < k < dl for k in st_counts) and any(dl < k < 2 * dl for k in st_counts)


@pytest.mark.gpu
def test_front_end_reset_gives_fresh_bits(sb, v_case):
    """reset() mid-stream, then the stream again from its start, gives the bits of a fresh front end (PLL phase and
    frequency, delay line and pilot history cleared)"""
    vs, x, _ = v_case
    cfgs = [c for c, _ in vs]
    k = 8
    fresh, _ = run_front_end(sb, FS_V, cfgs, x, SCHED_V[:k])
    again, _ = run_front_end(sb, FS_V, cfgs, x, SCHED_V[:6] + SCHED_V[:k], reset_at=6)
    for a, b in zip(fresh, again):
        assert np.array_equal(np.concatenate(a).view(np.uint32), np.concatenate(b).view(np.uint32))


@pytest.mark.gpu
def test_18_stereo_vfos_two_batches_10msps(sb, oracle, report):
    """18 stereo VFOs 500 kHz apart, each with its own programme and pilot offset: two stereo launch batches (16 + 2)"""
    from sdrplusplus_b200 import VfoConfig
    fs = 10e6
    sched = [0, 7, 41, 3001, 400003, 12000, 400000, 400000, 5, 250001]
    vs = []
    for k in range(18):
        c = VfoConfig.wfm_stereo(-4.25e6 + 500e3 * k + 37.0 * k)
        c.low_pass = k % 3 != 0
        vs.append((c, ("st", 19000.0 - 95.0 + 11.0 * k, 100 + k)))
    x = fe_input(fs, vs, sum(sched), 616)
    cfgs = [c for c, _ in vs]
    parts, _ = run_front_end(sb, fs, cfgs, x, sched)
    refs = references(oracle, vs, x, sched, fs)
    res = []
    for c, p, ref in zip(cfgs, parts, refs):
        assert [q.shape[0] for q in p] == vfo_counts(oracle, fs, c, sched)
        res.append(gate_vfo(c, p, ref))
    report["stereo_f64_in_situ_10msps_18vfos"] = {
        "per_vfo": res, "max_err_over_bound": max(r["max_err_over_bound"] for r in res),
        "max_abs_g_minus_1": max(max(r["M"]["abs_g_minus_1"], r["S"]["abs_g_minus_1"]) for r in res),
        "max_edge_over_p999": max(max(r["M"]["edge_over_p999"], r["S"]["edge_over_p999"]) for r in res)}
    for r in res:
        check_ms(r, r["offset"])


SQ_FE_CASES = {
    # RAW VFOs at 250 kS/s and 25 kS/s (one squelch batch, different n) and a WFM VFO behind the squelch
    "2p4msps": [0, 10, 1000, 24001, 96000, 96000, 96000, 131071, 7, 200001, 300000],
    # a RAW VFO at 1.2 MS/s whose IF chunks pass SQ_MAXPARTS * 4096 = 1,048,576 samples: the grid stops growing and
    # k_sq_sum's loop strides; beside it a RAW VFO at 250 kS/s
    "long": [5, 2400001, 3000000, 2097153, 1001],
}


def squelch_vfo_set(case):
    from sdrplusplus_b200 import VfoConfig
    if case == "long":
        return [(VfoConfig.raw(-500e3 + 3.5, 1.2e6, 1.2e6).with_squelch(-30.0), ("mono", 40e3, 4)),
                (VfoConfig.raw(300e3 - 12.5, 250e3, 200e3).with_squelch(-30.0), ("mono", 20e3, 5))]
    return [(VfoConfig.raw(-300e3 + 12.5, 250e3, 200e3).with_squelch(-30.0), ("mono", 20e3, 1)),
            (VfoConfig.raw(400e3 - 7.0, 25e3, 20e3).with_squelch(-30.0), ("mono", 3e3, 2)),
            (VfoConfig.wfm(100e3 + 321.0).with_squelch(-30.0), ("mono", 30e3, 3))]


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(SQ_FE_CASES))
def test_squelch_in_front_end_vs_float64(sb, oracle, report, case):
    """VFOs behind PowerSquelch; before every chunk each level is set to that chunk's float64 mean +- 4 bounds
    (alternating), so every decision is observable and none is ambiguous"""
    from dataclasses import replace
    from sdrplusplus_b200 import VfoConfig
    fs = FS_V
    sched = SQ_FE_CASES[case]
    vs = squelch_vfo_set(case)
    n = sum(sched)
    x = fe_input(fs, vs, n, 717)
    env = np.repeat(np.array([1.0, 0.05, 0.3, 0.01, 0.6, 0.02]), -(-n // 6))[:n]
    x = (x * env).astype(np.complex64)
    xr = x.astype(np.complex128)
    levels, ifref = [], []
    for c, _ in vs:
        # the IF stream the squelch sees: the same VFO as RAW without the squelch
        rc = replace(VfoConfig.raw(c.offset, c.out_samplerate, c.bandwidth))
        yc, bc, _, _ = vfo_audio_f64(oracle, xr, sched, fs, [rc] * len(sched))
        cnt = vfo_counts(oracle, fs, rc, sched)
        _, mar, bd, _ = squelch_f64(yc, bc, cnt, 0.0)
        db = np.where(np.isfinite(mar), mar, -200.0)
        with np.errstate(over="ignore"):             # a chunk of a few IF samples has a wide bound: its level rounds to -+inf
            levels.append([float(np.float32(db[k] + (-4.0 if k % 2 == 0 else 4.0) * max(bd[k], 1e-6))) for k in range(len(cnt))])
        ifref.append((yc, bc, cnt))
    cfgs = [c for c, _ in vs]
    parts, _ = run_front_end(sb, fs, cfgs, x, sched, levels=levels)
    res = []
    for k, (c, p) in enumerate(zip(cfgs, parts)):
        cs = [replace(c, squelch_level=lv) for lv in levels[k]]
        info = {}
        y64, b, namb, reach = vfo_audio_f64(oracle, xr, sched, fs, cs, info=info)
        sq = info["squelch"]
        assert not sq["ambiguous"].any(), sq
        live = [i for i, m in enumerate(sq["counts"]) if m > 0]
        assert [bool(sq["open"][i]) for i in live] == [i % 2 == 0 for i in live]
        y = np.concatenate(p)
        if y.dtype == np.complex64:
            ci = _chunk_index(sq["counts"])
            closed = ~sq["open"][ci]
            assert not np.any(y[closed].view(np.uint32)), "a closed chunk is exact zeros"
            rr = _ratio_c(y, y64, b)
            res.append({"offset": c.offset, "max_err_over_bound": float(rr.max()), "chunks": len(live),
                        "nparts": [squelch_nparts(m) for m in sq["counts"]]})
        else:
            rr = _ratio_c(y[:, 0] + 1j * y[:, 1], y64, b)
            res.append({"offset": c.offset, "max_err_over_bound": float(rr.max()), "chunks": len(live)})
        assert res[-1]["max_err_over_bound"] <= 1.0, res[-1]
    if case == "long":
        assert max(ifref[0][2]) > SQ_TILE_CAP and squelch_nparts(max(ifref[0][2])) == 256
    report["squelch_f64_in_situ_" + case] = res

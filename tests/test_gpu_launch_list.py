"""How the scheduler groups the stages behind stage 1 into launches: per-chunk launch counts and the final graph, stage-1
epilogue and fused-tail statistics for a fixed set of front-end scenarios, pinned as literals.  Batching (16 jobs per
launch), the flushes on a key change, the register-window and fused routes, graph replay and the input decimator all show
up in these numbers; a change to any of them changes a count here."""
import hashlib

import numpy as np
import pytest

from util import noise_iq, fm_carrier, am_carrier, ssb_tone, to_i16

pytestmark = pytest.mark.gpu
FS = 2.4e6
# a WFM VFO's plan is (32, 143) (4, 27) (2, 69), and offsets on the 4 MHz grid take the filter-bank stage 1: it runs the
# (4, 27) stage as its ÷4 epilogue
FS_256 = 64e6
STATS = ("graphs", "graph_hits", "graph_misses", "s1_f2_jobs", "fused_chains")


@pytest.fixture(scope="module")
def sb():
    import sdrplusplus_b200 as m
    from sdrplusplus_b200 import lib
    L = lib.load()
    assert L.b200_device_count() > 0
    assert L.b200_init(0) == 0
    return m


def _mix20(sb):
    """test_gpu_parity's 20 VFOs of four kinds: more than one 16-job batch per level, three stage-1 groups"""
    c = [sb.VfoConfig.wfm((k - 2.5) * 300e3) for k in range(6)]
    c += [sb.VfoConfig.nfm(-1.0e6 + k * 333e3) for k in range(6)]
    c += [sb.VfoConfig.am(120e3 + k * 210e3) for k in range(4)]
    c += [sb.VfoConfig.raw(-900e3 + k * 410e3, 250e3, 150e3) for k in range(4)]
    return c


def _radio(sb):
    """AM, USB and NFM behind noise blanker, squelch and FM IF noise reduction, with the AF chain and volume"""
    from sdrplusplus_b200 import lib as L
    return [sb.VfoConfig.am(-400e3).with_noise_blanker(10.0).with_squelch(-80.0).with_af(48000.0, True, 0.0).with_volume(0.8),
            sb.VfoConfig.ssb(600e3, L.DEMOD_USB).with_squelch(-80.0).with_af(48000.0, False, 0.0).with_volume(0.5),
            sb.VfoConfig.nfm(200e3).with_noise_blanker(8.0).with_squelch(-80.0).with_if_nr(32).with_af(48000.0, True, 50e-6)
            .with_volume(1.2),
            sb.VfoConfig.wfm(-800e3).with_af(48000.0, True, 50e-6).with_volume(0.7)]


def _signal(n, fs=FS):
    x = noise_iq(n, 23, 0.002).copy()
    for k, o in enumerate((-750e3, -450e3, -150e3, 150e3, 300e3, -800e3)):
        x += fm_carrier(n, fs, o, tones=((1000.0 * (k + 1), 0.5), (5000.0, 0.3)), amp=0.03)
    x += fm_carrier(n, fs, 200e3, dev=5000.0, tones=((1000.0, 0.7),), amp=0.03)
    x += am_carrier(n, fs, -400e3, amp=0.03)
    x += ssb_tone(n, fs, 600e3, amp=0.03)
    return x


def _drive(fe, x, chunk, fmt=None, between=None):
    """per-chunk launch count deltas, then the final statistics"""
    from sdrplusplus_b200 import lib as L
    fmt = L.FMT_CF32 if fmt is None else fmt
    a = to_i16(x) if fmt == L.FMT_CS16 else x
    per = 2 if fmt == L.FMT_CS16 else 1
    deltas = []
    for k, i in enumerate(range(0, x.size, chunk)):
        if between:
            between(fe, k)
        l0 = fe.launch_count()
        fe.process(a[i * per:(i + chunk) * per], fmt)
        deltas.append(fe.launch_count() - l0)
    return deltas, {s: fe.stat(s) for s in STATS}


def _front_end(sb, cfgs, opts, chunk, fs=FS):
    fe = sb.FrontEnd(fs, chunk)
    for k, v in opts:
        fe.set_option(k, v)
    ids = [fe.add_vfo(c) for c in cfgs]
    return fe, ids


def _scenario(sb, name):
    from sdrplusplus_b200 import lib as L
    base = [("tails", 2)]
    if name == "mix20":
        fe, _ = _front_end(sb, _mix20(sb), base, 12000)
        return _drive(fe, _signal(16 * 12000), 12000)
    if name == "mix20_regall0":
        fe, _ = _front_end(sb, _mix20(sb), base + [("ft_regall", 0)], 12000)
        return _drive(fe, _signal(16 * 12000), 12000)
    if name == "rds":
        fe, ids = _front_end(sb, [sb.VfoConfig.wfm_stereo(150e3), sb.VfoConfig.wfm_rds_bits(-450e3), sb.VfoConfig.wfm(300e3)], base, 12000)
        fe.bind_rds(ids[0])
        fe.bind_rds(ids[2])
        return _drive(fe, _signal(16 * 12000), 12000)
    if name.startswith("radio_tails"):           # radio_tails<t>: tails t with ft_regall 0, so tails 2 takes the fused route
        t = int(name[len("radio_tails"):])
        fe, _ = _front_end(sb, _radio(sb), [("tails", t), ("ft_regall", 0)], 12000)
        return _drive(fe, _signal(16 * 12000), 12000)
    if name.startswith("radio_g"):               # radio_g<graph>_o<overlap>
        g, o = name[len("radio_g"):].split("_o")
        fe, _ = _front_end(sb, _radio(sb), base + [("overlap", int(o)), ("graph", int(g))], 12000)
        return _drive(fe, _signal(16 * 12000), 12000)
    if name == "small_4096":
        fe, _ = _front_end(sb, _mix20(sb)[:8], base, 4096)
        return _drive(fe, _signal(24 * 4096), 4096)
    if name == "big_1m":
        cfgs = [sb.VfoConfig.wfm(o) for o in (-12e6, -4e6, 4e6, 12e6, 20e6)] + [sb.VfoConfig.raw(-20e6, 250e3, 150e3)]
        fe, _ = _front_end(sb, cfgs, base, 1 << 20, fs=FS_256)
        return _drive(fe, _signal(4 << 20, FS_256), 1 << 20)
    if name == "cs16":
        fe, _ = _front_end(sb, _mix20(sb)[:8], base, 12000)
        return _drive(fe, _signal(8 * 12000), 12000, fmt=L.FMT_CS16)
    if name == "retune":                      # the chunk behind a retune stores the stage-1 outputs (no ÷4 epilogue)
        cfgs = [sb.VfoConfig.wfm(4e6), sb.VfoConfig.wfm(-4e6), sb.VfoConfig.raw(12e6, 250e3, 150e3)]
        fe, ids = _front_end(sb, cfgs, base, 1 << 16, fs=FS_256)

        def retune(fe, k):
            if k in (3, 6):
                fe.set_vfo_offset(ids[0], 8e6 if k == 3 else 4e6)
        return _drive(fe, _signal(10 << 16, FS_256), 1 << 16, between=retune)
    if name == "vfo_config":
        cfgs = [sb.VfoConfig.nfm(200e3), sb.VfoConfig.am(-400e3), sb.VfoConfig.wfm(300e3)]
        fe, ids = _front_end(sb, cfgs, base, 12000)

        def switch(fe, k):
            if k == 3:
                fe.set_vfo_config(ids[0], sb.VfoConfig.nfm(200e3).with_squelch(-80.0).with_if_nr(32))
                fe.set_vfo_config(ids[1], sb.VfoConfig.am(-400e3).with_noise_blanker(10.0).with_volume(0.5))
            if k == 5:
                fe.set_vfo_config(ids[2], sb.VfoConfig.wfm(300e3).with_volume(0.6))
            if k == 7:
                fe.set_vfo_config(ids[0], sb.VfoConfig.nfm(200e3))
        return _drive(fe, _signal(10 * 12000), 12000, between=switch)
    if name == "decimation":
        fe, _ = _front_end(sb, [], base, 24000, fs=4.8e6)
        fe.set_decimation(2)
        for c in _mix20(sb)[:6]:
            fe.add_vfo(c)
        return _drive(fe, _signal(12 * 24000, 4.8e6), 24000)
    raise KeyError(name)


# per scenario: the launch count of every chunk, then the final statistics (measured on an H100)
EXPECTED = {
    "big_1m": ([7] * 4, {"graphs": 2, "graph_hits": 0, "graph_misses": 4, "s1_f2_jobs": 24, "fused_chains": 0}),
    "cs16": ([15] * 8, {"graphs": 2, "graph_hits": 4, "graph_misses": 4, "s1_f2_jobs": 0, "fused_chains": 0}),
    "decimation": ([11] * 12, {"graphs": 2, "graph_hits": 8, "graph_misses": 4, "s1_f2_jobs": 0, "fused_chains": 0}),
    "mix20": ([21] * 16, {"graphs": 4, "graph_hits": 8, "graph_misses": 8, "s1_f2_jobs": 0, "fused_chains": 0}),
    "mix20_regall0": ([14] * 16, {"graphs": 4, "graph_hits": 8, "graph_misses": 8, "s1_f2_jobs": 0, "fused_chains": 20}),
    "radio_g-1_o0": ([42] * 16, {"graphs": 4, "graph_hits": 8, "graph_misses": 8, "s1_f2_jobs": 0, "fused_chains": 0}),
    "radio_g-1_o1": ([42] * 16, {"graphs": 4, "graph_hits": 8, "graph_misses": 8, "s1_f2_jobs": 0, "fused_chains": 0}),
    "radio_g0_o0": ([42] * 16, {"graphs": 0, "graph_hits": 0, "graph_misses": 0, "s1_f2_jobs": 0, "fused_chains": 0}),
    "radio_g0_o1": ([42] * 16, {"graphs": 0, "graph_hits": 0, "graph_misses": 0, "s1_f2_jobs": 0, "fused_chains": 0}),
    "radio_g1_o0": ([42] * 16, {"graphs": 4, "graph_hits": 8, "graph_misses": 8, "s1_f2_jobs": 0, "fused_chains": 0}),
    "radio_g1_o1": ([42] * 16, {"graphs": 4, "graph_hits": 8, "graph_misses": 8, "s1_f2_jobs": 0, "fused_chains": 0}),
    "radio_tails0": ([42] * 16, {"graphs": 4, "graph_hits": 8, "graph_misses": 8, "s1_f2_jobs": 0, "fused_chains": 0}),
    "radio_tails1": ([42] * 16, {"graphs": 4, "graph_hits": 8, "graph_misses": 8, "s1_f2_jobs": 0, "fused_chains": 0}),
    "radio_tails2": ([33] * 16, {"graphs": 4, "graph_hits": 8, "graph_misses": 8, "s1_f2_jobs": 0, "fused_chains": 4}),
    "rds": ([24] * 16, {"graphs": 16, "graph_hits": 0, "graph_misses": 16, "s1_f2_jobs": 0, "fused_chains": 0}),
    "retune": ([7, 7, 7, 9, 8, 8, 9, 7, 7, 7], {"graphs": 5, "graph_hits": 2, "graph_misses": 8, "s1_f2_jobs": 20, "fused_chains": 0}),
    "small_4096": ([15] * 24, {"graphs": 6, "graph_hits": 12, "graph_misses": 12, "s1_f2_jobs": 0, "fused_chains": 0}),
    "vfo_config": ([19, 19, 19, 25, 25, 26, 26, 23, 23, 23], {"graphs": 10, "graph_hits": 0, "graph_misses": 10, "s1_f2_jobs": 0, "fused_chains": 0}),
}


@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_launch_counts_pinned(sb, name):
    deltas, stats = _scenario(sb, name)
    want_deltas, want_stats = EXPECTED[name]
    assert deltas == want_deltas, (name, deltas)
    assert stats == want_stats, (name, stats)


def test_fir_block_set_taps_output_pinned(sb):
    """A complex-data FIR block whose taps change mid-stream (b200_fir_cr_set_taps): its own scheduler replays graphs; the
    output bits are pinned."""
    from sdrplusplus_b200 import lib
    L = lib.load()
    x = noise_iq(9 * 5000, 5, 0.5)
    t0 = np.hanning(33).astype(np.float32) / 16.0
    t1 = np.hanning(57).astype(np.float32) / 28.0
    b = sb.Block.fir_cr(t0, 2)
    ys = []
    for k in range(9):
        if k == 4:
            lib.check(L.b200_fir_cr_set_taps(b._h, t1.ctypes.data, t1.size))
        ys.append(b.process(x[k * 5000:(k + 1) * 5000].view(np.float32)))
    b.close()
    y = np.concatenate(ys)
    assert y.size > 0
    assert hashlib.sha256(y.tobytes()).hexdigest() == FIR_BLOCK_SHA256


FIR_BLOCK_SHA256 = "7bd9a618d919d61d3c8c747a21832229c923a354ec07716ebeab7ceb78fe4751"

"""b200_fe_set_vfo_config: the radio module's setters on a running front-end VFO, each block keeping its state.

The GPU VFO and an oracle chain (vfo_settings_oracle.OracleVfo) get the same change at the same chunk boundary; they are
compared over the whole stream but its first chunk, so every change point lies in the compared part."""
import copy
import ctypes
import os
import subprocess

import numpy as np
import pytest

from util import rel_rms, noise_iq, fm_carrier, am_carrier, ssb_tone
from vfo_settings_oracle import OracleVfo

pytestmark = pytest.mark.gpu

TOL = 1e-5
FS = 2.4e6
CHUNK = 12000
EINVAL = -1                                       # B200_EINVAL


@pytest.fixture(scope="module")
def sb():
    import sdrplusplus_b200 as m
    from sdrplusplus_b200 import lib
    L = lib.load()
    assert L.b200_device_count() > 0
    assert L.b200_init(0) == 0
    return m


def _sig(n, seed, kind="wfm"):
    x = noise_iq(n, seed, 0.02).copy()
    if kind == "am":
        x += am_carrier(n, FS, 300e3)
    elif kind == "usb":
        x += ssb_tone(n, FS, 300e3, 1000.0)
    elif kind == "nfm":
        # a carrier that fades in and out, so a squelch level between the two opens and closes
        env = (0.2 + 0.8 * (np.sin(np.arange(n) * (2 * np.pi / 60000.0)) > 0)).astype(np.float32)
        x += fm_carrier(n, FS, 300e3, dev=5000.0, tones=((1000.0, 0.7),)) * env
    else:
        x += fm_carrier(n, FS, 300e3)
    x[::4099] *= np.float32(15.0)                 # impulses for the noise blanker
    return x


def _cfg(sb, kind):
    return {"wfm": sb.VfoConfig.wfm(300e3).with_af(48000.0, False, 50e-6).with_volume(0.7),
            "nfm": sb.VfoConfig.nfm(300e3).with_squelch(-60.0),
            "am": sb.VfoConfig.am(300e3),
            "usb": sb.VfoConfig.ssb(300e3)}[kind]


def _with(cfg, **kw):
    c = copy.copy(cfg)
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def _run(sb, oracle, x, cfg, changes, opts=(), with_oracle=True, resume=True):
    """GPU VFO and oracle chain, `changes` = {chunk index: VfoConfig} taken before that chunk; per-chunk outputs"""
    fe = sb.FrontEnd(FS, CHUNK)
    for k, v in opts:
        fe.set_option(k, v)
    vid = fe.add_vfo(cfg)
    ov = OracleVfo(oracle, FS, cfg, resume) if with_oracle else None
    xf = x.view(np.float32)
    yg, ya = [], []
    for k, i in enumerate(range(0, x.size, CHUNK)):
        if k in changes:
            fe.set_vfo_config(vid, changes[k])
            if ov is not None:
                ov.set(changes[k])
        outs, _ = fe.process(x[i:i + CHUNK])
        yg.append(outs[vid])
        if ov is not None:
            ya.append(ov.process(xf[2 * i: 2 * (i + CHUNK)]).reshape(-1, 2))
    fe.close()
    return yg, ya


def _oracle_only(oracle, x, cfg, changes, resume):
    ov = OracleVfo(oracle, FS, cfg, resume)
    xf = x.view(np.float32)
    ys = []
    for k, i in enumerate(range(0, x.size, CHUNK)):
        if k in changes:
            ov.set(changes[k])
        ys.append(ov.process(xf[2 * i: 2 * (i + CHUNK)]).reshape(-1, 2))
    return ys


def _tail(chunks, changes):
    """everything after the first chunk (the start-of-stream head), checked to hold the outputs of every change point"""
    assert changes and min(changes) >= 1
    head = chunks[0].shape[0]
    y = np.concatenate(chunks)
    for k in changes:
        assert sum(c.shape[0] for c in chunks[:k]) >= head and chunks[k].shape[0] > 0, k
    assert y.shape[0] > head
    return y[head:]


def _gate(report, name, yg, ya, changes):
    assert [a.shape for a in yg] == [b.shape for b in ya]
    g, a = _tail(yg, changes), _tail(ya, changes)
    e = rel_rms(g, a)
    report["vfo_settings_" + name] = {"rel_rms": e, "rows": int(g.shape[0])}
    assert e < TOL, (name, e)
    return g, a


# ------------------------------------------------------------------------------------------ coefficients, state kept
def _chunks(sb, x, cfg, changes):
    """the VFO's output chunk by chunk (a chunk's sample count varies with the resampler phases)"""
    fe = sb.FrontEnd(FS, CHUNK)
    vid = fe.add_vfo(cfg)
    ys = []
    for k, i in enumerate(range(0, x.size, CHUNK)):
        if k in changes:
            fe.set_vfo_config(vid, changes[k])
        ys.append(fe.process(x[i:i + CHUNK])[0][vid])
    fe.close()
    return ys


def test_volume_mute_bit_exact(sb):
    """each segment is the unchanged VFO's output times powf(volume, 2), or 0 while muted (volume.h:19-29,39-42)"""
    x = _sig(240000, 1)
    base = _cfg(sb, "wfm")
    yp = _chunks(sb, x, _with(base, af_volume_on=False), {})
    seq = {5: _with(base, af_volume=1.3), 10: _with(base, af_volume=1.3, af_muted=True), 15: _with(base, af_volume=1.3)}
    yv = _chunks(sb, x, base, seq)
    assert [a.shape for a in yp] == [b.shape for b in yv]
    for k, (a, b) in enumerate(zip(yp, yv)):
        v = 0.7 if k < 5 else (None if 10 <= k < 15 else 1.3)
        g = np.float32(0.0) if v is None else np.float32(np.float32(v) ** np.float32(2))
        assert np.array_equal((a * g).view(np.uint32), b.view(np.uint32)), k


COEF = {
    "squelch_level": ("nfm", lambda c: [(6, _with(c, squelch_level=-15.0)), (12, _with(c, squelch_level=-60.0))]),
    "nb_level": ("am", lambda c: [(0, _with(c, nb_on=True, nb_level=3.0)), (13, _with(c, nb_on=True, nb_level=1.5))]),
    "deemph_tau": ("wfm", lambda c: [(8, _with(c, af_deemph_tau=75e-6))]),
    "am_agc_dc": ("am", lambda c: [(6, _with(c, agc_attack=20 / 15e3, agc_decay=2 / 15e3)), (12, _with(c, agc_attack=20 / 15e3, agc_decay=2 / 15e3, dc_block_rate=30 / 15e3))]),
    "usb_agc": ("usb", lambda c: [(6, _with(c, agc_attack=10 / 24e3, agc_decay=1 / 24e3))]),
    "am_agc_mode": ("am", lambda c: [(7, _with(c, agc_mode=0)), (13, _with(c, agc_mode=1))]),
    "nr_bins": ("wfm", lambda c: [(0, _with(c, nr_on=True, nr_bins=32)), (6, _with(c, nr_on=True, nr_bins=9)), (12, _with(c, nr_on=True, nr_bins=15))]),
}


@pytest.mark.parametrize("name", sorted(COEF))
def test_coefficients_and_restarts(sb, oracle, report, name):
    kind, mk = COEF[name]
    # AM (15 kS/s) and SSB (24 kS/s) over 40 chunks of 5 ms: 3000 and 4800 audio rows
    x = _sig(480000 if kind in ("am", "usb") else 240000, 2, kind)
    cfg = _cfg(sb, kind)
    steps = mk(cfg)
    if steps[0][0] == 0:
        cfg = steps[0][1]
        steps = steps[1:]
    changes = dict(steps)
    yg, ya = _run(sb, oracle, x, cfg, changes)
    if name == "nr_bins":
        # FMIF keeps the strongest bin: where two bins tie to within the rounding of the stages in front of it, the GPU and the
        # CPU may keep different ones, and the audio low-pass spreads that sample.  As in tests/test_gpu_ifnr.py the rows with a
        # gross difference are set aside; the rest is gated at TOL or at the oracle's own floor -- the oracle against itself
        # with its input perturbed by 1e-7, the same gate applied -- whichever is larger.
        def gated(y, r):
            bad = np.any(np.abs(y - r) > 1e-3 * np.max(np.abs(r)), axis=1)
            return rel_rms(y[~bad], r[~bad]), int(bad.sum())
        g, a = _tail(yg, changes), _tail(ya, changes)
        xp = (x * (1 + np.float32(1e-7) * noise_iq(x.size, 77, 1.0).real)).astype(np.complex64)
        floor, floor_bad = gated(_tail(_oracle_only(oracle, xp, cfg, changes, True), changes), a)
        e, bad = gated(g, a)
        report["vfo_settings_nr_bins"] = {"rel_rms": e, "rows": int(g.shape[0]), "rows_behind_a_tied_bin": bad,
                                          "oracle_floor_rel_rms": floor, "oracle_floor_rows": floor_bad}
        assert e < max(TOL, 2 * floor) and bad <= max(10, 2 * floor_bad), report["vfo_settings_nr_bins"]
        return
    _gate(report, name, yg, ya, changes)
    if name == "squelch_level":
        zg = np.array([not np.any(c) for c in yg])
        za = np.array([not np.any(c) for c in ya])
        assert np.array_equal(zg, za) and zg.any() and not zg.all()


# ------------------------------------------------------------------------------------------ topology
OPTS = {"default": (), "tails1": (("tails", 1),), "regall0": (("ft_regall", 0),), "overlap0": (("overlap", 0),)}
TOGGLES = {
    "nb_on": dict(nb_on=True),
    "squelch_on": dict(squelch_on=True, squelch_level=-80.0),
    "nr_on": dict(nr_on=True, nr_bins=15),
    "af_high_pass": dict(af_high_pass=True),
    "deemph": dict(af_deemph_tau=75e-6),
    "af_volume_on": dict(af_volume_on=True, af_volume=0.8),
}


@pytest.mark.parametrize("opts", sorted(OPTS))
@pytest.mark.parametrize("toggle", sorted(TOGGLES))
def test_toggle_on_off_on(sb, oracle, report, toggle, opts):
    if toggle == "nb_on":
        # an FM demodulator ignores the amplitude the blanker works on: the blanker is toggled in front of AM
        x = _sig(480000, 3, "am")
        off = _with(sb.VfoConfig.am(300e3), nb_level=1.5)
        changes = {10: None, 20: None, 30: None}
    else:
        x = _sig(240000, 3)
        off = _with(sb.VfoConfig.wfm(300e3).with_af(48000.0, False, 0.0), squelch_level=-80.0, nr_bins=15, af_volume=0.8)
        changes = {5: None, 10: None, 15: None}
    on = _with(off, **TOGGLES[toggle])
    changes = dict(zip(sorted(changes), (on, off, on)))
    yg, ya = _run(sb, oracle, x, off, changes, OPTS[opts])
    g, a = _gate(report, "toggle_%s_%s" % (toggle, opts), yg, ya, changes)
    if toggle in ("nb_on", "nr_on", "af_high_pass", "deemph"):
        # these blocks carry state: a block that restarted when switched on again would be seen
        fresh = _tail(_oracle_only(oracle, x, off, changes, resume=False), changes)
        assert rel_rms(fresh, a) > 20 * TOL, rel_rms(fresh, a)
        assert rel_rms(g, fresh) > 10 * TOL


def test_toggles_on_rds_bits_if_chain(sb, oracle, report):
    """blanker and squelch switched on, off and on again in front of a WFM_RDS_BITS VFO's RDS branch: no bit differs from the
    oracle chain off threshold.  (The FM IF noise reduction is toggled on WFM audio above: in front of the RDS branch its bin
    choice makes bits a 1e-7 input change can flip -- the oracle against itself flips 108 of 1497 -- so no bit gate holds.)"""
    from test_gpu_rds import _gate as rds_gate
    from test_gpu_rds_frontend import _station, FS as RFS, OFF
    chunk = 40000
    x, bits = _station(1500, 3)
    x = x[: (x.size // chunk) * chunk]
    off = _with(sb.VfoConfig.wfm_rds_bits(OFF), nb_level=3.0, squelch_level=-80.0, nr_bins=31)
    on = _with(off, nb_on=True, squelch_on=True)
    nch = x.size // chunk
    changes = {nch // 4: on, nch // 2: off, 3 * nch // 4: on}
    fe = sb.FrontEnd(RFS, chunk)
    vid = fe.add_vfo(off)
    oracle.set_rotator_mode(1)
    try:
        ov = OracleVfo(oracle, RFS, off)
        soft, hard, ye = [], [], []
        for k in range(nch):
            if k in changes:
                fe.set_vfo_config(vid, changes[k])
                ov.set(changes[k])
            outs, _ = fe.process(x[k * chunk:(k + 1) * chunk])
            soft.append(outs[vid][0])
            hard.append(outs[vid][1])
            ye.append(ov.process(x[k * chunk:(k + 1) * chunk].view(np.float32)).view(np.complex64))
    finally:
        oracle.set_rotator_mode(0)
    fe.close()
    so, ho = oracle.rds_demod().process_chunks(np.concatenate(ye), 250)
    r = rds_gate(np.concatenate(soft), np.concatenate(hard), so, ho)
    report["vfo_settings_rds_bits_if_toggles"] = r
    assert r["bit_mismatches_off_threshold"] == 0, r


# ------------------------------------------------------------------------------------------ isolation, pipeline, errors
def test_isolation_and_same_config(sb):
    fs, chunk, nch = 100e6, 500000, 6
    n = chunk * nch
    offs = [5e6, -5e6, 15e6, -15e6, 25e6, -25e6, 35e6, -35e6]
    x = noise_iq(n, 12, 0.01).copy()
    for o in offs + [45e6]:
        x += fm_carrier(n, fs, o)
    res = []
    for changing in (False, True):
        fe = sb.FrontEnd(fs, chunk)
        ids = [fe.add_vfo(sb.VfoConfig.wfm(o).with_af(48000.0, False, 50e-6)) for o in offs]
        base = sb.VfoConfig.wfm(45e6).with_af(48000.0, False, 50e-6).with_volume(1.0)
        vc = fe.add_vfo(base)
        outs = {i: [] for i in ids}
        for k in range(nch):
            if changing:
                fe.set_vfo_config(vc, _with(base, af_volume=0.5 + 0.1 * k, nb_on=k % 2 == 1, af_high_pass=k % 3 == 1))
                fe.set_vfo_config(ids[0], sb.VfoConfig.wfm(offs[0]).with_af(48000.0, False, 50e-6))     # its own config
            o, _ = fe.process(x[k * chunk:(k + 1) * chunk])
            for i in ids:
                outs[i].append(o[i])
        res.append({i: np.concatenate(v) for i, v in outs.items()})
        fe.close()
    for i in res[0]:
        assert np.array_equal(res[0][i].view(np.uint32), res[1][i].view(np.uint32)), i


def _pipelined(sb, x, cfg, changes, opts, depth):
    """submit / wait with `depth` chunks in flight; changes[k] is set right after submit(k - 1), i.e. while chunks are in flight"""
    from sdrplusplus_b200 import lib as L
    fe = sb.FrontEnd(FS, CHUNK)
    for k, v in opts:
        fe.set_option(k, v)
    fe.set_option("inflight", depth)
    vid = fe.add_vfo(cfg)
    chunks = [np.ascontiguousarray(x[i:i + CHUNK]) for i in range(0, x.size, CHUNK)]
    pend, got = [], []
    for k, c in enumerate(chunks):
        if len(pend) == depth:
            o, b = pend.pop(0)
            fe.wait()
            got.append(b[vid][: 2 * o.vfo_count[vid]].copy())
        o, bufs, _ = fe._alloc_outputs(CHUNK)
        fe.submit_ptr(c.ctypes.data, CHUNK, L.FMT_CF32, L.MEM_HOST, o)
        pend.append((o, bufs))
        if k + 1 in changes:
            fe.set_vfo_config(vid, changes[k + 1])        # between submit(k) and wait(k): from chunk k + 1
    while pend:
        o, b = pend.pop(0)
        fe.wait()
        got.append(b[vid][: 2 * o.vfo_count[vid]].copy())
    fe.close()
    return np.concatenate(got)


def test_pipeline_same_outputs(sb):
    x = _sig(240000, 7)
    off = sb.VfoConfig.wfm(300e3).with_af(48000.0, False, 50e-6).with_volume(0.9)
    changes = {3: _with(off, nb_on=True, af_volume=1.2), 6: _with(off, nb_on=True, nr_on=True, af_high_pass=True),
               9: _with(off, af_deemph_tau=0.0), 12: off, 15: _with(off, squelch_on=True, squelch_level=-90.0, af_volume=0.4)}
    ref, _ = _run(sb, None, x, off, changes, with_oracle=False)
    ref = np.concatenate(ref).reshape(-1)
    for graph in (-1, 0):
        for depth in (2, 3, 4):
            y = _pipelined(sb, x, off, changes, (("graph", graph),), depth)
            assert np.array_equal(y.view(np.uint32), ref.view(np.uint32)), (graph, depth)


def test_rejections_leave_vfo_alone(sb):
    from sdrplusplus_b200 import lib as L
    x = _sig(120000, 8)
    cfg = sb.VfoConfig.wfm(300e3).with_af(48000.0, True, 50e-6).with_volume(0.7)
    ref, _ = _run(sb, None, x, cfg, {}, with_oracle=False)
    ref = np.concatenate(ref)
    fe = sb.FrontEnd(FS, CHUNK)
    vid = fe.add_vfo(cfg)
    bad = [_with(cfg, demod=L.DEMOD_NFM), _with(cfg, out_samplerate=200e3), _with(cfg, deviation=50e3), _with(cfg, low_pass=False),
           _with(cfg, af_samplerate=44100.0), _with(cfg, nr_on=True, nr_bins=65), _with(cfg, nr_on=True, nr_bins=1),
           _with(cfg, bandwidth=0.0)]
    max0 = fe.vfo_max_out(vid, CHUNK)
    ys = []
    for k, i in enumerate(range(0, x.size, CHUNK)):
        c, good = bad[k % len(bad)].to_c(), cfg.to_c()
        assert fe._l.b200_fe_set_vfo_config(fe._h, vid, ctypes.byref(c)) == EINVAL
        assert fe._l.b200_fe_set_vfo_config(fe._h, vid + 5, ctypes.byref(good)) == EINVAL
        outs, _ = fe.process(x[i:i + CHUNK])
        ys.append(outs[vid])
        assert fe.vfo_max_out(vid, CHUNK) == max0
    fe.close()
    y = np.concatenate(ys)
    assert np.array_equal(y.view(np.uint32), ref.view(np.uint32))


def test_reset_and_remove_with_parked_blocks(sb):
    """b200_fe_reset clears the parked blocks: switched on after it they give a fresh VFO's bits.  A VFO added in the slot of a
    removed one with parked blocks behaves as fresh too (that the parked stages' memory is released is not observed here)."""
    x = _sig(120000, 9)
    on = sb.VfoConfig.wfm(300e3).with_af(48000.0, True, 50e-6).with_if_nr(15)
    off = _with(on, nr_on=False, af_high_pass=False)
    # fresh front end, blocks on from the start  ==  blocks parked, reset, switched on again
    fresh = sb.FrontEnd(FS, CHUNK)
    vf = fresh.add_vfo(on)
    yf = fresh.process_chunks(x, CHUNK)[0][vf]
    fresh.close()
    fe = sb.FrontEnd(FS, CHUNK)
    vid = fe.add_vfo(on)
    fe.process_chunks(x[:60000], CHUNK)
    fe.set_vfo_config(vid, off)
    fe.process_chunks(x[60000:], CHUNK)                 # the parked blocks keep what they held ...
    fe.reset()                                          # ... until the reset clears them
    fe.set_vfo_config(vid, on)
    y = fe.process_chunks(x, CHUNK)[0][vid]
    assert np.array_equal(y.view(np.uint32), yf.view(np.uint32))
    fe.remove_vfo(vid)
    v2 = fe.add_vfo(on)
    fe.reset()
    y2 = fe.process_chunks(x, CHUNK)[0][v2]
    assert np.array_equal(y2.view(np.uint32), yf.view(np.uint32))
    fe.close()


def test_adapter_set_vfo_config_from_another_thread(sb, tmp_path):
    """dsp::b200::FrontEnd::setVFOConfig from a thread other than the running worker (tests/vfo_settings_adapter.cpp, built
    here): the audio is the Python run's with the same changes at the same chunks, bit for bit"""
    from sdrplusplus_b200 import lib as L
    here = os.path.dirname(os.path.abspath(__file__))
    host = os.path.join(os.path.dirname(here), "sdrplusplus_b200", "host")
    exe = tmp_path / "vfo_settings_adapter"
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-I", host, "-o", str(exe), os.path.join(here, "vfo_settings_adapter.cpp"),
                        "-L", os.path.dirname(L.LIB_PATH), "-lb200dsp", "-Wl,-rpath," + os.path.dirname(L.LIB_PATH), "-lpthread"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
    x = _sig(240000, 11)
    src, dst = tmp_path / "iq.f32", tmp_path / "audio.f32"
    x.tofile(src)
    r = subprocess.run([str(exe), str(src), str(dst)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
    got = np.fromfile(dst, np.float32).reshape(-1, 2)
    base = _with(sb.VfoConfig.wfm(300e3).with_af(48000.0, False, 50e-6).with_volume(0.7), nb_level=2.0, nr_bins=32)
    c5 = _with(base, af_volume=1.3, nb_on=True)
    c10 = _with(c5, af_high_pass=True)
    c15 = _with(c10, nb_on=False, af_muted=True)
    yg, _ = _run(sb, None, x, base, {5: c5, 10: c10, 15: c15}, with_oracle=False)
    want = np.concatenate(yg)
    assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert np.any(want[: want.shape[0] * 3 // 4]) and not np.any(yg[16])          # audio until chunk 15, then muted

"""GPU parity tests: every call goes through the C ABI of libb200dsp.so and is compared with the CPU oracle
(plain-C restatement of the reference path, oracle/) on the same seeded inputs.

Tolerances (north-star: 1e-5 relative, bit-exact for bin indexing / peak hold):
  * TOL = 1e-5  RMS-normalised relative error for FIR / resampler / demodulator outputs
  * FFT: linear power within 1e-5 of the line maximum; peak bin index exact
  * zoom / hold: bit-exact
  * the full-rate frequency translator is compared with the exact e^{jwn} (closed form, fp64) at 2e-6; its gap to
    the reference's fp32 phase recurrence is the reference's own rounding random walk and is reported, not gated
    (SURVEY.md section 7, "Rotator recurrence")
"""
import numpy as np
import pytest

from util import rel_rms, max_rel, noise_iq, fm_carrier, am_carrier, ssb_tone, to_i16

pytestmark = pytest.mark.gpu

TOL = 1e-5


@pytest.fixture(scope="module")
def sb():
    import sdrplusplus_b200 as m
    from sdrplusplus_b200 import lib
    L = lib.load()
    assert L.b200_device_count() > 0
    assert L.b200_init(0) == 0
    return m


# ---------------------------------------------------------------------------------------------- FFT branch
@pytest.mark.parametrize("N,nz", [(8, 8), (64, 64), (1024, 1024), (4096, 3000), (8192, 8192), (16384, 16384),
                                  (65536, 65536), (65536, 40000), (1 << 17, 1 << 17), (1 << 18, 200000), (1 << 19, 1 << 19),
                                  (1 << 20, 1 << 20), (1 << 21, 1 << 21)])
def test_fft_line_vs_oracle(sb, oracle, report, N, nz):
    x = noise_iq(nz, 11 + N, 1.0).copy()
    n = np.arange(nz)
    b = N // 2 + N // 8 + (3 if N >= 64 else 1)  # dsp bin of an injected tone (DC sits at N/2: (-1)^n pre-twist)
    x += (0.5 * np.exp(2j * np.pi * ((b - N // 2) / N) * n)).astype(np.complex64)
    h = sb.SpectrumHandler(N, nz, 2)
    raw = h.raw(x)
    ref_raw = oracle.fft_raw(N, nz, 2, x)
    e_raw = rel_rms(raw, ref_raw)
    line = h.frame(x)
    ref = oracle.fft_frame(N, nz, 2, x)
    p, pr = 10.0 ** (line.astype(np.float64) / 10), 10.0 ** (ref.astype(np.float64) / 10)
    e_pow = float(np.max(np.abs(p - pr)) / np.max(pr))
    report["fft_%d_%d" % (N, nz)] = {"raw_rel_rms": e_raw, "power_rel_max": e_pow}
    assert e_raw < 2e-6, e_raw
    assert e_pow < TOL, e_pow
    assert int(np.argmax(line)) == int(np.argmax(ref))
    if N >= 64:
        assert int(np.argmax(line)) == b          # the injected tone dominates the noise
    h.close()


def test_fft_matches_float64_dft(sb):
    N = 4096
    x = noise_iq(N, 5, 1.0)
    h = sb.SpectrumHandler(N, N, 0)
    raw = h.raw(x)
    w = np.where(np.arange(N) % 2, -1.0, 1.0)
    ref = np.fft.fft(x.astype(np.complex128) * w)
    assert rel_rms(raw, ref) < 1e-6
    h.close()


@pytest.mark.parametrize("offset,width,out_size", [(0, 65536, 1000), (1000, 60000, 1280), (60000, 8000, 777), (0, 65536, 4000)])
def test_zoom_hold_bit_exact(sb, oracle, offset, width, out_size):
    from sdrplusplus_b200 import frontend
    x = noise_iq(65536, 3, 1.0)
    line = oracle.fft_frame(65536, 65536, 2, x)
    hold0 = np.full(out_size, -200.0, np.float32)
    z, h = frontend.zoom_hold(line, offset, width, out_size, hold0, 0.5)
    zr = oracle.zoom(offset, width, out_size, line)
    hr = oracle.hold(hold0, zr, 0.5)
    assert np.array_equal(z.view(np.uint32), zr.view(np.uint32))
    assert np.array_equal(h.view(np.uint32), hr.view(np.uint32))
    z2, h2 = frontend.zoom_hold(line - 3.0, offset, width, out_size, h, 0.5)
    assert np.array_equal(h2.view(np.uint32), oracle.hold(hr, oracle.zoom(offset, width, out_size, line - 3.0), 0.5).view(np.uint32))


# ---------------------------------------------------------------------------------------------- blocks
FS = 2.4e6


def _sig(n, seed=1):
    x = noise_iq(n, seed, 0.02).copy()
    x += fm_carrier(n, FS, 300e3)
    x += fm_carrier(n, FS, -650e3, tones=((3000.0, 0.6),))
    return x


def test_xlator_closed_form(sb, oracle, report):
    n = 300000
    x = _sig(n)
    b = sb.Block.xlator(-300e3, FS)
    y = b.process_chunks(x.view(np.float32), 12000).view(np.complex64)
    o = oracle.xlator(-300e3, FS)
    yo = o.process_chunks(x.view(np.float32), 12000).view(np.complex64)
    ph, dl = oracle.xlator_phase(o)
    w = np.arctan2(np.float64(dl[1]), np.float64(dl[0]))       # angle of the fp32-rounded phaseDelta
    exact = x.astype(np.complex128) * np.exp(1j * w * np.arange(n))
    e_exact, e_ref = rel_rms(y, exact), rel_rms(y, yo)
    report["xlator"] = {"vs_exact_closed_form": e_exact, "vs_reference_recurrence": e_ref,
                        "reference_vs_exact": rel_rms(yo, exact)}
    assert e_exact < 2e-6, e_exact
    assert e_ref < 2e-4, e_ref        # bounded by the reference's own phase random walk, reported above


@pytest.mark.parametrize("ratio,chunk", [(2, 7777), (8, 12000), (16, 9999), (64, 12000), (256, 50000)])
def test_power_decimator(sb, oracle, report, ratio, chunk):
    n = 400000
    x = _sig(n, 2)
    y = sb.Block.decim(ratio).process_chunks(x.view(np.float32), chunk)
    yo = oracle.decim(ratio).process_chunks(x.view(np.float32), chunk)
    assert y.size == yo.size
    e = rel_rms(y, yo)
    report["decim_%d" % ratio] = e
    assert e < TOL, e


@pytest.mark.parametrize("rates,chunk", [((2.4e6, 250e3), 12000), ((250e3, 48e3), 1250), ((48e3, 250e3), 5000), ((300e3, 250e3), 1501),
                                         ((1e6, 1e6), 1000)])
def test_rational_resampler(sb, oracle, report, rates, chunk):
    n = 200000
    x = _sig(n, 3)
    y = sb.Block.resamp(*rates).process_chunks(x.view(np.float32), chunk)
    yo = oracle.resamp(*rates).process_chunks(x.view(np.float32), chunk)
    assert y.size == yo.size
    e = rel_rms(y, yo)
    report["resamp_%g_%g" % rates] = e
    assert e < TOL, e


def test_fir_blocks(sb, oracle, report):
    n = 100000
    x = _sig(n, 4)
    taps = oracle.lowpass(75e3, 7.5e3, 250e3)
    y = sb.Block.fir_cr(taps).process_chunks(x.view(np.float32), 1250)
    yo = oracle.fir_cr(taps).process_chunks(x.view(np.float32), 1250)
    e1 = rel_rms(y, yo)
    y = sb.Block.fir_cr(taps, 3).process_chunks(x.view(np.float32), 1000)
    yo = oracle.decfir_cr(taps, 3).process_chunks(x.view(np.float32), 1000)
    assert y.size == yo.size
    e2 = rel_rms(y, yo)
    r = x.real.copy()
    at = oracle.lowpass(15e3, 4e3, 250e3)
    y = sb.Block.fir_rr(at).process_chunks(r, 999)
    yo = oracle.fir_rr(at).process_chunks(r, 999)
    e3 = rel_rms(y, yo)
    report["fir"] = {"complex": e1, "decimating": e2, "real": e3}
    assert max(e1, e2, e3) < TOL
    # known answer: a unit impulse returns the tap table (time-reversed correlation form: taps are symmetric)
    imp = np.zeros(2 * 400, np.float32)
    imp[0] = 1.0
    y = sb.Block.fir_cr(taps).process(imp).view(np.complex64)
    assert np.allclose(y.real[: taps.size], taps[::-1], rtol=0, atol=1e-9)


def _vfo_out(oracle, x, chunk, offset=300e3, bw=150e3, out_sr=250e3):
    return oracle.rxvfo(FS, out_sr, bw, offset).process_chunks(x.view(np.float32), chunk)


def test_rxvfo_block(sb, oracle, report):
    n = 480000
    x = _sig(n, 5)
    y = sb.Block.rxvfo(FS, 250e3, 150e3, 300e3).process_chunks(x.view(np.float32), 12000).view(np.complex64)
    yo = _vfo_out(oracle, x, 12000).view(np.complex64)
    assert y.size == yo.size
    e = rel_rms(y, yo)
    # FM content is what the path preserves: compare the discriminator output of both
    d = np.angle(y[1:] * np.conj(y[:-1]))
    do = np.angle(yo[1:] * np.conj(yo[:-1]))
    e_fm = rel_rms(d[2000:], do[2000:])
    report["rxvfo"] = {"iq_rel_rms": e, "fm_rel_rms": e_fm}
    assert e < 2e-4, e            # carries the translator's phase random walk (reported by test_xlator_closed_form)
    assert e_fm < TOL, e_fm


@pytest.mark.parametrize("kind", ["quad", "wfm", "wfm_nolp", "nfm", "nfm_nolp", "am_audio", "am_carrier", "usb", "lsb", "dsb"])
def test_demodulator_blocks(sb, oracle, report, kind):
    n = 480000
    if kind.startswith("am"):
        x = noise_iq(n, 6, 0.002).copy() + am_carrier(n, FS, 300e3)
        osr, bw = 15e3, 10e3
    elif kind in ("usb", "lsb", "dsb"):
        x = noise_iq(n, 6, 0.002).copy() + ssb_tone(n, FS, 300e3, 1000.0 if kind != "lsb" else -1000.0)
        osr, bw = 24e3, 2800.0
    elif kind.startswith("nfm"):
        x = noise_iq(n, 6, 0.002).copy() + fm_carrier(n, FS, 300e3, dev=5000.0, tones=((1000.0, 0.7),))
        osr, bw = 50e3, 12500.0
    else:
        x = _sig(n, 6)
        osr, bw = 250e3, 150e3
    iq = _vfo_out(oracle, x, 12000, bw=bw, out_sr=osr)
    ch = max(1, int(12000 * osr / FS))
    mk = {
        "quad": (lambda: sb.Block.quad(75e3, osr), lambda: oracle.quad(75e3, osr)),
        "wfm": (lambda: sb.Block.wfm(75e3, osr), lambda: oracle.wfm(75e3, osr)),
        "wfm_nolp": (lambda: sb.Block.wfm(75e3, osr, False, False), lambda: oracle.wfm(75e3, osr, False, False)),
        "nfm": (lambda: sb.Block.nfm(osr, bw, True), lambda: oracle.nfm(osr, bw, True)),
        "nfm_nolp": (lambda: sb.Block.nfm(osr, bw, False), lambda: oracle.nfm(osr, bw, False)),
        "am_audio": (lambda: sb.Block.am(1, bw, 50 / osr, 5 / osr, 100 / osr, osr), lambda: oracle.am(1, bw, 50 / osr, 5 / osr, 100 / osr, osr)),
        "am_carrier": (lambda: sb.Block.am(0, bw, 50 / osr, 5 / osr, 100 / osr, osr), lambda: oracle.am(0, bw, 50 / osr, 5 / osr, 100 / osr, osr)),
        "usb": (lambda: sb.Block.ssb(0, bw, osr, 50 / osr, 5 / osr), lambda: oracle.ssb(0, bw, osr, 50 / osr, 5 / osr)),
        "lsb": (lambda: sb.Block.ssb(1, bw, osr, 50 / osr, 5 / osr), lambda: oracle.ssb(1, bw, osr, 50 / osr, 5 / osr)),
        "dsb": (lambda: sb.Block.ssb(2, 4600.0, osr, 50 / osr, 5 / osr), lambda: oracle.ssb(2, 4600.0, osr, 50 / osr, 5 / osr)),
    }[kind]
    y = mk[0]().process_chunks(iq, ch)
    yo = mk[1]().process_chunks(iq, ch)
    assert y.size == yo.size
    e = rel_rms(y, yo)
    report["demod_" + kind] = e
    assert e < TOL, e


# ---------------------------------------------------------------------------------------------- front end
def _oracle_chain(oracle, x, fs, chunk, cfg):
    """reference graph of one VFO: RxVFO -> demodulator (radio_module.h:80-125)."""
    from sdrplusplus_b200 import lib as L
    v = oracle.rxvfo(fs, cfg.out_samplerate, cfg.bandwidth, cfg.offset)
    sr = cfg.out_samplerate
    if cfg.demod == L.DEMOD_WFM:
        d = oracle.wfm(cfg.deviation, sr, False, cfg.low_pass)
    elif cfg.demod == L.DEMOD_NFM:
        d = oracle.nfm(sr, cfg.bandwidth, cfg.low_pass)
    elif cfg.demod == L.DEMOD_AM:
        d = oracle.am(cfg.agc_mode, cfg.bandwidth, cfg.agc_attack, cfg.agc_decay, cfg.dc_block_rate, sr)
    elif cfg.demod in (L.DEMOD_USB, L.DEMOD_LSB, L.DEMOD_DSB):
        d = oracle.ssb(cfg.demod - L.DEMOD_USB, cfg.bandwidth, sr, cfg.agc_attack, cfg.agc_decay)
    else:
        d = None
    outs = []
    xf = x.view(np.float32)
    for i in range(0, x.size, chunk):
        y = v.process(xf[2 * i: 2 * (i + chunk)])
        outs.append(d.process(y) if d is not None else y)
    return np.concatenate(outs)


def _oracle_lines(oracle, x, fs, size, rate):
    skip, nz = oracle.fft_params(fs, size, rate)
    lines = []
    f = 0
    while f + nz <= x.size:
        lines.append(oracle.fft_frame(size, nz, 2, x[f:f + nz]))
        f += nz + skip
    return np.array(lines)


@pytest.mark.parametrize("variant", [0, 5, 6, 7, 8])
def test_frontend_c1_geometry(sb, oracle, report, variant):
    """BASELINE config 1: 2.4 MS/s, chunk 12000, 65536-pt FFT @ 20 fps, one WFM VFO at +300 kHz."""
    n = 600000
    x = _sig(n, 7)
    fe = sb.FrontEnd(FS, 12000)
    fe.set_option("s1", variant)
    fe.set_fft(65536, 20.0, 2)
    cfg = sb.VfoConfig.wfm(300e3)
    vid = fe.add_vfo(cfg)
    outs, lines = fe.process_chunks(x, 12000)
    ya = _oracle_chain(oracle, x, FS, 12000, cfg)
    la = _oracle_lines(oracle, x, FS, 65536, 20.0)
    assert outs[vid].size == ya.size
    e = rel_rms(outs[vid][4000:], ya.reshape(-1, 2)[4000:])
    assert lines.shape == la.shape and lines.shape[0] == 5
    p, pr = 10.0 ** (lines.astype(np.float64) / 10), 10.0 ** (la.astype(np.float64) / 10)
    e_fft = float(np.max(np.abs(p - pr)) / np.max(pr))
    report["frontend_c1_variant%d" % variant] = {"wfm_audio_rel_rms": e, "fft_power_rel_max": e_fft}
    assert np.array_equal(np.argmax(lines, axis=1), np.argmax(la, axis=1))
    assert e_fft < TOL, e_fft
    assert e < TOL, e
    assert np.array_equal(outs[vid][:, 0], outs[vid][:, 1])       # mono: L == R
    fe.close()


def test_frontend_int16_ingest(sb, oracle, report):
    """file_source's native format: int16 IQ converted on the device (x/32768)."""
    n = 240000
    x = _sig(n, 8)
    xi = to_i16(x * 8.0)
    xf = oracle.i16_to_f32(xi).view(np.complex64)
    from sdrplusplus_b200 import lib as L
    fe = sb.FrontEnd(FS, 12000)
    fe.set_fft(65536, 20.0, 2)
    cfg = sb.VfoConfig.wfm(300e3)
    vid = fe.add_vfo(cfg)
    outs, lines = fe.process_chunks(xi, 12000, fmt=L.FMT_CS16)
    ya = _oracle_chain(oracle, xf, FS, 12000, cfg).reshape(-1, 2)
    la = _oracle_lines(oracle, xf, FS, 65536, 20.0)
    e = rel_rms(outs[vid][4000:], ya[4000:])
    p, pr = 10.0 ** (lines.astype(np.float64) / 10), 10.0 ** (la.astype(np.float64) / 10)
    e_fft = float(np.max(np.abs(p - pr)) / np.max(pr))
    report["frontend_int16"] = {"wfm_audio_rel_rms": e, "fft_power_rel_max": e_fft}
    assert e < TOL and e_fft < TOL
    fe.close()


def test_frontend_mixed_modes(sb, oracle, report):
    """AM / NFM / USB / LSB / DSB / RAW VFOs side by side on one stream (BASELINE config 4 mix)."""
    n = 480000
    x = noise_iq(n, 9, 0.002).copy()
    x += am_carrier(n, FS, -400e3)
    x += fm_carrier(n, FS, 200e3, dev=5000.0, tones=((1000.0, 0.7),))
    x += ssb_tone(n, FS, 600e3, 1000.0)
    x += ssb_tone(n, FS, -800e3, -700.0)
    x += fm_carrier(n, FS, 900e3)
    from sdrplusplus_b200 import lib as L
    cfgs = [sb.VfoConfig.am(-400e3), sb.VfoConfig.nfm(200e3), sb.VfoConfig.ssb(600e3, L.DEMOD_USB), sb.VfoConfig.ssb(-800e3, L.DEMOD_LSB),
            sb.VfoConfig.ssb(600e3, L.DEMOD_DSB, 4600.0), sb.VfoConfig.raw(900e3, 250e3, 150e3), sb.VfoConfig.am(-400e3, agc_mode=L.AGC_CARRIER)]
    fe = sb.FrontEnd(FS, 12000)
    ids = [fe.add_vfo(c) for c in cfgs]
    outs, _ = fe.process_chunks(x, 12000)
    res, floor = {}, {}
    for vid, c in zip(ids, cfgs):
        ssb = c.demod in (L.DEMOD_USB, L.DEMOD_LSB, L.DEMOD_DSB)
        ya = _oracle_chain(oracle, x, FS, 12000, c)
        y = outs[vid]
        if c.demod == L.DEMOD_RAW:
            ya = ya.view(np.complex64)
            d, do = np.angle(y[1:] * np.conj(y[:-1])), np.angle(ya[1:] * np.conj(ya[:-1]))
            e = rel_rms(d[2000:], do[2000:])
        else:
            ya = ya.reshape(-1, 2)
            assert y.shape == ya.shape
            skip = y.shape[0] // 4            # AGC / DC-block settling
            if ssb:
                # SSB/DSB audio = Re{x e^{j theta}} is first-order sensitive to the rounding walk of the reference's
                # fp32 phase recurrence (SURVEY.md section 7): gate against the exact-phase oracle mode and report
                # the faithful-vs-exact gap, which is the reference's own numerical floor for this offset
                oracle.set_rotator_mode(1)
                try:
                    yx = _oracle_chain(oracle, x, FS, 12000, c).reshape(-1, 2)
                finally:
                    oracle.set_rotator_mode(0)
                floor["vfo%d_demod%d" % (vid, c.demod)] = {"gpu_vs_faithful": rel_rms(y[skip:], ya[skip:]),
                                                          "faithful_vs_exact_phase": rel_rms(ya[skip:], yx[skip:])}
                ya = yx
            e = rel_rms(y[skip:], ya[skip:])
        res["vfo%d_demod%d" % (vid, c.demod)] = e
    report["frontend_mixed"] = res
    report["frontend_mixed_ssb_reference_floor"] = floor
    for k, e in res.items():
        assert e < TOL, (k, e)
    fe.close()


def test_frontend_many_vfos_batching(sb, oracle, report):
    """20 VFOs of four kinds on one stream: more than one 16-job launch batch per stage, three different first-stage
    decimations (stage-1 groups), conjugate pairs mixed with singles."""
    from sdrplusplus_b200 import lib as L
    n = 240000
    x = noise_iq(n, 17, 0.002).copy()
    cfgs = []
    for k in range(6):
        off = (k - 2.5) * 300e3
        x += fm_carrier(n, FS, off)
        cfgs.append(sb.VfoConfig.wfm(off))                       # +-150k, +-450k, +-750k: three conjugate pairs
    for k in range(6):
        off = -1.0e6 + k * 333e3
        x += fm_carrier(n, FS, off, dev=5000.0, tones=((1000.0, 0.7),), amp=0.03)
        cfgs.append(sb.VfoConfig.nfm(off))
    for k in range(4):
        off = 120e3 + k * 210e3
        x += am_carrier(n, FS, off, amp=0.03)
        cfgs.append(sb.VfoConfig.am(off))
    for k in range(4):
        off = -900e3 + k * 410e3
        x += fm_carrier(n, FS, off, amp=0.04)
        cfgs.append(sb.VfoConfig.raw(off, 250e3, 150e3))
    fe = sb.FrontEnd(FS, 12000)
    ids = [fe.add_vfo(c) for c in cfgs]
    assert len(ids) == 20
    outs, _ = fe.process_chunks(x, 12000)
    errs = []
    for vid, c in zip(ids, cfgs):
        ya = _oracle_chain(oracle, x, FS, 12000, c)
        y = outs[vid]
        if c.demod == L.DEMOD_RAW:
            ya = ya.view(np.complex64)
            d, do = np.angle(y[1:] * np.conj(y[:-1])), np.angle(ya[1:] * np.conj(ya[:-1]))
            errs.append(rel_rms(d[2000:], do[2000:]))
        else:
            ya = ya.reshape(-1, 2)
            assert y.shape == ya.shape
            sk = y.shape[0] // 4
            errs.append(rel_rms(y[sk:], ya[sk:]))
    report["frontend_20_vfos"] = errs
    assert max(errs) < TOL, errs
    # remove / re-add keeps the others running
    fe.remove_vfo(ids[3])
    vid = fe.add_vfo(sb.VfoConfig.wfm(0.0))
    outs, _ = fe.process(x[:12000])
    assert vid in outs and len(outs) == 20 and outs[vid].shape[0] > 0
    fe.close()


def test_compressed_stream_ingest_and_export(sb, oracle, report):
    """SURVEY section 8f data formats: a SampleStreamCompressor packet (int16 / int8 payload + scaler) fed to the front
    end gives what the reference's decompressor + cf32 path gives; the device-side compressor and the recorder sample
    conversions are bit-exact with the oracle."""
    from sdrplusplus_b200 import frontend, lib as L
    n, chunk = 120000, 12000
    x = _sig(n, 23)
    for pcm, fmt in ((1, L.FMT_CS16), (0, L.FMT_CS8)):
        fe_p, fe_f = sb.FrontEnd(FS, chunk), sb.FrontEnd(FS, chunk)
        for fe in (fe_p, fe_f):
            fe.set_fft(65536, 20.0, 2)
        cfg = sb.VfoConfig.wfm(300e3)
        vp, vf = fe_p.add_vfo(cfg), fe_f.add_vfo(cfg)
        yp, yf, lp, lf = [], [], [], []
        for c in range(0, n, chunk):
            pkt = oracle.pcm_compress(x[c:c + chunk], pcm)                   # what the server puts on the wire
            pf, sc, cnt, off = frontend.pcm_packet_info(pkt)
            assert pf == fmt and cnt == chunk and off == 8
            fe_p.set_ingest_scale(fmt, sc)
            payload = pkt[off:].view(np.int16 if pcm == 1 else np.int8)
            o1, l1 = fe_p.process(payload, fmt=fmt)
            o2, l2 = fe_f.process(oracle.pcm_decompress(pkt))                # reference: decompress, then the cf32 path
            yp.append(o1[vp]); yf.append(o2[vf]); lp.append(l1); lf.append(l2)
        yp, yf = np.concatenate(yp), np.concatenate(yf)
        e = rel_rms(yp[4000:], yf[4000:])
        lines_p, lines_f = np.concatenate([l for l in lp if l.size]), np.concatenate([l for l in lf if l.size])
        e_l = float(np.max(np.abs(lines_p - lines_f)))
        report["packet_ingest_pcm%d" % pcm] = {"wfm_audio_rel_rms": e, "fft_db_abs_max": e_l}
        assert e < 1e-6 and e_l < 1e-3
        fe_p.close(); fe_f.close()
    # device-side compressor: header and payload byte for byte
    for pcm, fmt in ((1, L.FMT_CS16), (0, L.FMT_CS8), (2, L.FMT_CF32)):
        assert np.array_equal(frontend.pcm_compress(x[:50001], fmt), oracle.pcm_compress(x[:50001], pcm))
    # recorder sample types
    a = np.concatenate([x.view(np.float32)[:100001] * 0.9, np.array([1.0, -1.0, 2.0, -2.0, 0.5, -0.5, 1.5e-5], np.float32)])
    for t, ot in ((frontend.EXPORT_I16, 1), (frontend.EXPORT_I32, 2)):
        assert np.array_equal(frontend.export_convert(a, t), oracle.export_convert(a, ot))
    a8 = np.clip(a, -1.0, 1.0)
    assert np.array_equal(frontend.export_convert(a8, frontend.EXPORT_U8), oracle.export_convert(a8, 0))


def test_deemphasis_block_bit_exact(sb, oracle):
    n = 20000
    x = noise_iq(n, 15, 0.5).view(np.float32)            # (l, r) pairs
    y = sb.Block.deemph(50e-6, 48e3).process_chunks(x, 480)
    yo = oracle.deemph(50e-6, 48e3).process_chunks(x, 480)
    assert np.array_equal(y.view(np.uint32), yo.view(np.uint32))


@pytest.mark.parametrize("high_pass", [False, True])
def test_frontend_af_chain(sb, oracle, report, high_pass):
    """SURVEY 8f rank 1: the radio module's AF chain behind the demodulator, fused into the same chunk pass:
    WFM (250 kS/s) -> RationalResampler<stereo_t> 48 kS/s -> [300 Hz high-pass] -> 50 us deemphasis."""
    n = 480000
    x = _sig(n, 16)
    fe = sb.FrontEnd(FS, 12000)
    cfg = sb.VfoConfig.wfm(300e3).with_af(48000.0, high_pass, 50e-6)
    vid = fe.add_vfo(cfg)
    outs, _ = fe.process_chunks(x, 12000)
    v, d = oracle.rxvfo(FS, 250e3, 150e3, 300e3), oracle.wfm(75e3, 250e3)
    r = oracle.resamp_stereo(250e3, 48e3)
    h = oracle.fir_cr(oracle.highpass(300.0, 100.0, 48000.0)) if high_pass else None
    de = oracle.deemph(50e-6, 48e3)
    ya = []
    xf = x.view(np.float32)
    for i in range(0, n, 12000):
        a = r.process(d.process(v.process(xf[2 * i: 2 * (i + 12000)])))
        if h is not None:
            a = h.process(a)
        ya.append(de.process(a).reshape(-1, 2))
    ya = np.concatenate(ya)
    assert outs[vid].shape == ya.shape
    e = rel_rms(outs[vid][3000:], ya[3000:])
    report["frontend_af_chain_hp%d" % int(high_pass)] = e
    assert e < TOL, e
    fe.close()


def test_af_volume_block_bit_exact(sb):
    """dsp::audio::Volume at the end of the AF chain (volume.h:13-17,39-42): out = in * powf(volume, 2), muted -> 0;
    one fp32 multiply per sample, so the check is bit for bit against the same chain without the block."""
    n = 120000
    x = _sig(n, 18)
    outs = {}
    for name, cfg in (("plain", sb.VfoConfig.wfm(300e3).with_af(48000.0, True, 50e-6)),
                      ("vol", sb.VfoConfig.wfm(300e3).with_af(48000.0, True, 50e-6).with_volume(0.7)),
                      ("muted", sb.VfoConfig.wfm(300e3).with_af(48000.0, True, 50e-6).with_volume(0.7, True)),
                      ("vol_noaf", sb.VfoConfig.nfm(200e3).with_volume(1.3))):
        fe = sb.FrontEnd(FS, 12000)
        vid = fe.add_vfo(cfg)
        outs[name] = fe.process_chunks(x, 12000)[0][vid]
        fe.close()
    g = np.float32(np.float32(0.7) ** np.float32(2))
    assert np.array_equal((outs["plain"] * g).view(np.uint32), outs["vol"].view(np.uint32))
    assert outs["muted"].shape == outs["plain"].shape and not np.any(outs["muted"])
    fe = sb.FrontEnd(FS, 12000)
    vid = fe.add_vfo(sb.VfoConfig.nfm(200e3))
    ref = fe.process_chunks(x, 12000)[0][vid]
    fe.close()
    assert np.array_equal((ref * np.float32(np.float32(1.3) ** np.float32(2))).view(np.uint32), outs["vol_noaf"].view(np.uint32))


def test_frontend_retune_and_bandwidth(sb, oracle, report):
    """RxVFO::setOffset / setBandwidth mid-stream, applied at a chunk boundary like the reference's ctrlMtx."""
    n = 480000
    x = _sig(n, 10)
    fe = sb.FrontEnd(FS, 12000)
    cfg = sb.VfoConfig.wfm(300e3)
    vid = fe.add_vfo(cfg)
    v = oracle.rxvfo(FS, 250e3, 150e3, 300e3)
    d = oracle.wfm(75e3, 250e3)
    ya, yg = [], []
    xf = x.view(np.float32)
    for k, i in enumerate(range(0, n, 12000)):
        if k == 10:
            fe.set_vfo_offset(vid, -650e3)
            v.set_offset(-650e3)
        if k == 20:
            fe.set_vfo_bandwidth(vid, 120e3)
            v.set_bandwidth(120e3)
        outs, _ = fe.process(x[i:i + 12000])
        yg.append(outs[vid])
        ya.append(d.process(v.process(xf[2 * i: 2 * (i + 12000)])).reshape(-1, 2))
    yg, ya = np.concatenate(yg), np.concatenate(ya)
    assert yg.shape == ya.shape
    e = rel_rms(yg[4000:], ya[4000:])
    report["frontend_retune"] = e
    assert e < TOL, e
    fe.close()


def test_frontend_multi_vfo_100msps(sb, oracle, report):
    """BASELINE config 2 geometry at reduced length: 100 MS/s, 1M-pt FFT @ 20 fps, 8 x WFM, chunk 500000."""
    fs, chunk, nch = 100e6, 500000, 5
    n = chunk * nch
    offs = [5e6, -5e6, 15e6, -15e6, 25e6, -25e6, 35e6, -35e6]
    x = noise_iq(n, 12, 0.01).copy()
    for o in offs:
        x += fm_carrier(n, fs, o)
    fe = sb.FrontEnd(fs, chunk)
    fe.set_fft(1 << 20, 20.0, 2)
    cfgs = [sb.VfoConfig.wfm(o) for o in offs]
    ids = [fe.add_vfo(c) for c in cfgs]
    outs, lines = fe.process_chunks(x, chunk)
    la = _oracle_lines(oracle, x, fs, 1 << 20, 20.0)
    assert lines.shape == la.shape == (1, 1 << 20)        # the frame spans three chunks
    p, pr = 10.0 ** (lines.astype(np.float64) / 10), 10.0 ** (la.astype(np.float64) / 10)
    e_fft = float(np.max(np.abs(p - pr)) / np.max(pr))
    errs = []
    for vid, c in zip(ids, cfgs):
        ya = _oracle_chain(oracle, x, fs, chunk, c).reshape(-1, 2)
        assert outs[vid].shape == ya.shape
        errs.append(rel_rms(outs[vid][1500:], ya[1500:]))
    report["frontend_c2_8vfo"] = {"wfm_audio_rel_rms": errs, "fft_power_rel_max": e_fft}
    assert e_fft < TOL, e_fft
    assert max(errs) < TOL, errs
    fe.close()


@pytest.mark.parametrize("variant,overlap,pair,tails", [
    (5, 1, 1, {}), (5, 0, 1, {"ft_regall": 0}), (0, 0, 0, {}), (5, 1, 0, {"tails": 1}), (5, 0, 1, {"tails": 0}),
    (6, 1, 1, {"tails": 1}), (6, 0, 0, {"ft_regall": 0}), (6, 1, 1, {"ft_regall": 0, "ft_threads": 256}),
    (6, 1, 1, {"ft_regall": 0, "ft_ob": 301}), (7, 1, 1, {}), (7, 0, 0, {"tails": 1}), (7, 0, 1, {"ft_regall": 0, "ft_direct": 0}),
    (6, 0, 1, {"ft_regall": 0, "ft_ob": 64, "ft_smem_kb": 48}), (6, 1, 1, {"ft_regall": 0, "ft_obmax": 2500, "ft_smem_kb": 200}),
    (8, 1, 1, {}), (8, 0, 0, {"tails": 1}), (8, 1, 1, {"ft_prereg": 0}), (7, 0, 1, {"tails": 1, "ft_prereg": 0}),
    (8, 1, 1, {"ft_regall": 0}), (8, 1, 1, {"ft_regall": 0, "ft_prereg": 1}), (8, 1, 1, {"s1_stages": 3})])
def test_frontend_variants_100msps(sb, oracle, report, variant, overlap, pair, tails):
    """kernel / scheduling A-B on the config-2 geometry (short): every stage-1 kernel (TMA filter bank, cp.async filter
    bank, per-VFO complex taps single / double buffered, one thread per output), tails on the main stream,
    conjugate-pair sharing off, register-window tails / fused tail (with forced slab sizes) / per-stage tails."""
    fs, chunk, nch = 100e6, 1000000, 4
    n = chunk * nch
    offs = [5e6, -5e6, 15e6, -25e6, 35e6, 25e6]
    x = noise_iq(n, 21, 0.01).copy()
    for o in offs:
        x += fm_carrier(n, fs, o)
    fe = sb.FrontEnd(fs, chunk)
    fe.set_option("overlap", overlap)
    fe.set_option("s1", variant)
    fe.set_option("pair", pair)
    for k, v in tails.items():
        fe.set_option(k, v)
    fe.set_fft(1 << 18, 200.0, 2)              # 500000-sample interval: frames inside chunks and across them
    cfgs = [sb.VfoConfig.wfm(o) for o in offs]
    ids = [fe.add_vfo(c) for c in cfgs]
    outs, lines = fe.process_chunks(x, chunk)
    la = _oracle_lines(oracle, x, fs, 1 << 18, 200.0)
    assert lines.shape == la.shape and lines.shape[0] == 8
    p, pr = 10.0 ** (lines.astype(np.float64) / 10), 10.0 ** (la.astype(np.float64) / 10)
    e_fft = float(np.max(np.abs(p - pr)) / np.max(pr))
    errs = []
    for vid, c in zip(ids, cfgs):
        ya = _oracle_chain(oracle, x, fs, chunk, c).reshape(-1, 2)
        assert outs[vid].shape == ya.shape
        errs.append(rel_rms(outs[vid][1500:], ya[1500:]))
    tag = "".join("_%s%d" % kv for kv in sorted(tails.items()))
    report["frontend_s1v%d_overlap%d_pair%d%s" % (variant, overlap, pair, tag)] = {"wfm_audio_rel_rms": errs, "fft_power_rel_max": e_fft}
    assert e_fft < TOL, e_fft
    assert max(errs) < TOL, errs
    fe.close()


def test_chunking_invariance_and_pipelining(sb, report):
    """Same stream, different chunk sizes -> same values (state is carried exactly); submit/wait == process."""
    n = 360000
    x = _sig(n, 13)
    res = []
    for chunk in (12000, 36000, 7001):
        fe = sb.FrontEnd(FS, 36000)
        fe.set_fft(65536, 20.0, 2)
        vid = fe.add_vfo(sb.VfoConfig.wfm(300e3))
        outs, lines = fe.process_chunks(x, chunk)
        res.append((outs[vid], lines))
        fe.close()
    for y, l in res[1:]:
        assert y.shape == res[0][0].shape and l.shape == res[0][1].shape
        assert rel_rms(y[4000:], res[0][0][4000:]) < 2e-6
        assert np.max(np.abs(l - res[0][1])) < 1e-3
    report["chunking_invariance"] = [rel_rms(r[0][4000:], res[0][0][4000:]) for r in res[1:]]


def test_ragged_and_empty_chunks(sb, oracle, report):
    """Edge cases of the chunked API: empty chunks, chunks shorter than a filter history, odd sizes."""
    n = 120000
    x = _sig(n, 14)
    sizes = [0, 1, 7, 300, 0, 12000, 1, 36000, 5, 11, 4099, 0, 20000, 39999]
    sizes.append(n - sum(sizes))
    assert 0 <= sizes[-1] <= 40000
    fe = sb.FrontEnd(FS, 40000)
    fe.set_fft(4096, 500.0, 2)                 # 4800-sample interval: many frames, some split over tiny chunks
    cfg = sb.VfoConfig.wfm(300e3)
    vid = fe.add_vfo(cfg)
    v, d = oracle.rxvfo(FS, 250e3, 150e3, 300e3), oracle.wfm(75e3, 250e3)
    pos, yg, ya, nl = 0, [], [], 0
    for sz in sizes:
        seg = x[pos:pos + sz]
        outs, lines = fe.process(seg)
        nl += lines.shape[0]
        yg.append(outs[vid])
        ya.append(d.process(v.process(seg.view(np.float32))).reshape(-1, 2))
        pos += sz
    yg, ya = np.concatenate(yg), np.concatenate(ya)
    assert yg.shape == ya.shape
    assert nl == len(_oracle_lines(oracle, x, FS, 4096, 500.0))
    e = rel_rms(yg[4000:], ya[4000:])
    report["ragged_chunks"] = e
    assert e < TOL, e
    fe.close()


# ---------------------------------------------------------------------------------------------- full-size properties
def test_full_size_known_answers(sb, report):
    """BASELINE config-2 sizes (one 4M-sample chunk at 100 MS/s, 8 VFOs, 1M-pt FFT): size-independent
    known answers instead of the oracle.  An unmodulated carrier 10 kHz above a WFM VFO demodulates to the
    constant 10k/75k; the FFT peak lands on the carrier's bin."""
    fs, n = 100e6, 1 << 22
    offs = [5e6, -5e6, 15e6, -15e6, 25e6, -25e6, 35e6, -35e6]
    t = np.arange(n, dtype=np.float64) / fs
    x = np.zeros(n, np.complex64)
    for o in offs:
        x += (0.05 * np.exp(2j * np.pi * (o + 10e3) * t)).astype(np.complex64)
    fe = sb.FrontEnd(fs, n)
    fe.set_fft(1 << 20, 20.0, 2)
    ids = [fe.add_vfo(sb.VfoConfig.wfm(o)) for o in offs]
    outs, lines = fe.process(x)
    assert lines.shape[0] == 1
    N = 1 << 20
    strongest = np.sort(np.argsort(lines[0])[-8:])
    want = np.sort([int(round((o + 10e3) / fs * N)) + N // 2 for o in offs])
    assert np.all(np.abs(strongest - want) <= 1), (strongest, want)
    dev = []
    for vid in ids:
        y = outs[vid][2000:, 0]
        dev.append(float(np.max(np.abs(y - 10e3 / 75e3))))
    report["full_size_const_fm"] = dev
    assert max(dev) < 2e-5, dev
    fe.close()

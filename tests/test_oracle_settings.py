"""The oracle side of b200_fe_set_vfo_config: the radio module's setters on the restatement's blocks (vfo_settings_oracle.py).

* the struct views read back what each block was created with (the layout they assume is the restatement's);
* a setter called at a chunk boundary changes only the coefficient: the output equals a block created with the new
  coefficient whose state was handed over from the old block at that boundary;
* a setter's coefficient arithmetic gives the bits of the reference-header build's block made with the new value.
A block switched off is skipped and kept (chain::setBlockEnabled); that it resumes from its state is checked on the GPU,
against the oracle chain, in tests/test_gpu_vfo_settings.py.
"""
import numpy as np
import pytest

from util import noise_iq, fm_carrier
import vfo_settings_oracle as S


def _iq(n, seed, amp=0.3):
    x = noise_iq(n, seed, 0.05).copy() + fm_carrier(n, 250e3, 20e3) * np.float32(amp)
    x[::613] *= np.float32(9.0)                 # impulses for the blanker
    return x.view(np.float32)


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_views_read_creation_values(oracle):
    blocks = [oracle.squelch(-27.5), oracle.noise_blanker(0.002, 3.5), oracle.deemph(50e-6, 48e3),
              oracle.am(1, 10e3, 50 / 15e3, 5 / 15e3, 100 / 15e3, 15e3), oracle.ssb(0, 2800.0, 24e3, 50 / 24e3, 5 / 24e3)]
    sq, nb, de, am, ssb = (S.view(b, t) for b, t in zip(blocks, (S.NSq, S.NNb, S.NDe, S.NAm, S.NSsb)))
    assert sq.level == np.float32(-27.5)
    assert (nb.rate, nb.inv_rate, nb.level, nb.amp) == (np.float32(0.002), np.float32(1.0) - np.float32(0.002), np.float32(3.5), 1.0)
    dt = np.float32(1.0 / 48e3)
    assert de.alpha == np.float32(dt / (50e-6 + dt)) and de.lastL == 0.0
    assert am.agcMode == 1 and am.dcRate == np.float32(100 / 15e3)
    for g in (am.carrier, am.audio):
        assert g.attack == np.float32(50 / 15e3) and g.decay == np.float32(5 / 15e3) and g.maxGain == np.float32(10e6)
    assert ssb.agc.attack == np.float32(50 / 24e3) and ssb.agc.maxOutputAmp == np.float32(10.0)


def _hand_over(mk_old, mk_new, setter, state, x, chunk, k):
    """old block with `setter` at chunk k  ==  old block up to k, then a block made with the new coefficient and the old state"""
    a = mk_old()
    ya = []
    for i, j in enumerate(range(0, x.size, chunk)):
        if i == k:
            setter(a)
        ya.append(a.process(x[j:j + chunk]))
    b, c = mk_old(), mk_new()
    yb = []
    for i, j in enumerate(range(0, x.size, chunk)):
        if i == k:
            state(b, c)
            b = c
        yb.append(b.process(x[j:j + chunk]))
    return np.concatenate(ya), np.concatenate(yb)


def _copy(struct, *fields):
    def f(old, new):
        vo, vn = S.view(old, struct), S.view(new, struct)
        for k in fields:
            setattr(vn, k, getattr(vo, k))
    return f


CASES = {
    "nb_level": (lambda o: o.noise_blanker(0.002, 3.0), lambda o: o.noise_blanker(0.002, 1.6),
                 lambda b: S.nb_set_level(b, 1.6), _copy(S.NNb, "amp")),
    "deemph_tau": (lambda o: o.deemph(50e-6, 48e3), lambda o: o.deemph(75e-6, 48e3),
                   lambda b: S.deemph_set_tau(b, 75e-6, 48e3), _copy(S.NDe, "lastL", "lastR")),
    "squelch_level": (lambda o: o.squelch(-30.0), lambda o: o.squelch(-5.0), lambda b: S.squelch_set_level(b, -5.0),
                      lambda old, new: None),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_setter_keeps_state(oracle, name):
    mk_old, mk_new, setter, state = CASES[name]
    x = _iq(30000, 3)
    ya, yb = _hand_over(lambda: mk_old(oracle), lambda: mk_new(oracle), setter, state, x, 2000, 7)
    assert _same(ya, yb)
    y0 = mk_old(oracle).process_chunks(x, 1000)
    assert not _same(ya, y0)                   # the new coefficient made a difference


@pytest.mark.parametrize("mode", [0, 1])
def test_am_setters_keep_state(oracle, mode):
    sr = 15e3
    x = np.ascontiguousarray(_iq(30000, 4))
    mk = lambda a, d, r: oracle.am(mode, 10e3, a / sr, d / sr, r / sr, sr)      # noqa: E731

    def setter(b):
        S.am_set_agc(b, 20 / sr, 2 / sr)
        S.am_set_dc_rate(b, 50 / sr)
    # same output up to the boundary, other output after it, and the new coefficients in place
    a = mk(50, 5, 100)
    ya = [a.process(x[j:j + 2000]) for j in range(0, 14000, 2000)]
    setter(a)
    ya += [a.process(x[j:j + 2000]) for j in range(14000, x.size, 2000)]
    v = S.view(a, S.NAm)
    assert v.carrier.attack == np.float32(20 / sr) and v.audio.decay == np.float32(2 / sr) and v.dcRate == np.float32(50 / sr)
    y0 = mk(50, 5, 100).process_chunks(x, 1000)
    n = sum(p.size for p in ya[:7])
    ya = np.concatenate(ya)
    assert _same(ya[:n], y0[:n]) and not _same(ya[n:], y0[n:])
    # setAGCMode -> reset: both AGCs and the DC blocker at their initial values, the mode switched
    S.am_set_agc_mode(a, 1 - mode)
    assert v.agcMode == 1 - mode and v.dcOffset == 0.0 and v.carrier.amp == 0.0 and v.audio.amp == 0.0


def test_ssb_setters(oracle):
    sr = 24e3
    x = _iq(24000, 5)
    a = oracle.ssb(0, 2800.0, sr, 50 / sr, 5 / sr)
    y1 = a.process(x[:12000])
    amp = S.view(a, S.NSsb).agc.amp
    S.ssb_set_agc(a, 10 / sr, 1 / sr)
    assert S.view(a, S.NSsb).agc.amp == amp                               # setAttack / setDecay leave the amplitude
    y2 = a.process(x[12000:])
    b = oracle.ssb(0, 2800.0, sr, 50 / sr, 5 / sr)
    assert _same(b.process(x[:12000]), y1) and not _same(b.process(x[12000:]), y2)


REF_CASES = {
    # name: (restatement block with the old value, setter to the new value, reference-header block made with the new value)
    "nb_level": (lambda o: o.noise_blanker(0.002, 3.0), lambda b: S.nb_set_level(b, 1.6), lambda r: r.noise_blanker(0.002, 1.6)),
    "squelch_level": (lambda o: o.squelch(-30.0), lambda b: S.squelch_set_level(b, -12.5), lambda r: r.squelch(-12.5)),
    "deemph_tau": (lambda o: o.deemph(50e-6, 48e3), lambda b: S.deemph_set_tau(b, 75e-6, 48e3), lambda r: r.deemph(75e-6, 48e3)),
    "am_agc_dc_audio": (lambda o: o.am(1, 10e3, 50 / 15e3, 5 / 15e3, 100 / 15e3, 15e3),
                        lambda b: (S.am_set_agc(b, 20 / 15e3, 2 / 15e3), S.am_set_dc_rate(b, 30 / 15e3)),
                        lambda r: r.am(1, 10e3, 20 / 15e3, 2 / 15e3, 30 / 15e3, 15e3)),
    "am_agc_dc_carrier": (lambda o: o.am(0, 10e3, 50 / 15e3, 5 / 15e3, 100 / 15e3, 15e3),
                          lambda b: (S.am_set_agc(b, 20 / 15e3, 2 / 15e3), S.am_set_dc_rate(b, 30 / 15e3)),
                          lambda r: r.am(0, 10e3, 20 / 15e3, 2 / 15e3, 30 / 15e3, 15e3)),
    "am_agc_mode": (lambda o: o.am(1, 10e3, 50 / 15e3, 5 / 15e3, 100 / 15e3, 15e3), lambda b: S.am_set_agc_mode(b, 0),
                    lambda r: r.am(0, 10e3, 50 / 15e3, 5 / 15e3, 100 / 15e3, 15e3)),
    "ssb_agc": (lambda o: o.ssb(0, 2800.0, 24e3, 50 / 24e3, 5 / 24e3), lambda b: S.ssb_set_agc(b, 10 / 24e3, 1 / 24e3),
                lambda r: r.ssb(0, 2800.0, 24e3, 10 / 24e3, 1 / 24e3)),
}


@pytest.mark.parametrize("name", sorted(REF_CASES))
def test_setter_values_match_the_reference(oracle, ref_oracle, name):
    """a setter's arithmetic against the reference's own: the restatement's block set to the new value before its first sample
    gives the bits of the reference-header build's block made with that value (init and setter share the member arithmetic:
    agc.h:13-24 / 32-44, deephasis.h:31-36,91-94, noise_blanker.h:26-30, power_squelch.h:27-31, am.h:49-56,69-87)"""
    mk, setter, mk_ref = REF_CASES[name]
    x = np.ascontiguousarray(_iq(30000, 8))
    b = mk(oracle)
    setter(b)
    assert _same(b.process_chunks(x, 1500), mk_ref(ref_oracle).process_chunks(x, 1500))


def test_squelch_level_mid_stream_matches_the_reference(oracle, ref_oracle):
    """PowerSquelch keeps no state: setLevel at a boundary is the reference's block with the new level from there on"""
    x = np.ascontiguousarray(_iq(30000, 9, amp=0.05))
    a = oracle.squelch(-30.0)
    ya = [a.process(x[j:j + 2000]) for j in range(0, 14000, 2000)]
    S.squelch_set_level(a, -18.0)
    ya += [a.process(x[j:j + 2000]) for j in range(14000, x.size, 2000)]
    r1, r2 = ref_oracle.squelch(-30.0), ref_oracle.squelch(-18.0)
    yr = [r1.process(x[j:j + 2000]) for j in range(0, 14000, 2000)] + [r2.process(x[j:j + 2000]) for j in range(14000, x.size, 2000)]
    assert _same(np.concatenate(ya), np.concatenate(yr))

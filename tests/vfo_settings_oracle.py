"""The radio module's setters on the oracle restatement's blocks, for the b200_fe_set_vfo_config tests.

Each setter writes the block's coefficient the way the reference's setter does and leaves its state alone:
PowerSquelch::setLevel, NoiseBlanker::setLevel, Deemphasis::setTau, AM::setAGCAttack / setAGCDecay / setDCBlockRate /
setAGCMode (-> reset), SSB's AGC setAttack / setDecay.  The restatement's blocks are plain C structs (oracle/sdrpp_oracle.c:
n_sq, n_nb, n_de, n_am, n_ssb); the views below mirror their layout.  A block switched off is skipped and kept, as
chain::setBlockEnabled does (core/src/dsp/chain.h:61-127).
"""
import ctypes as C

import numpy as np

_PTR3 = [("process", C.c_void_p), ("reset", C.c_void_p), ("destroy", C.c_void_p)]


class AgcT(C.Structure):
    _fields_ = [(k, C.c_float) for k in ("setPoint", "attack", "invAttack", "decay", "invDecay", "maxGain", "maxOutputAmp",
                                         "initGain", "amp")]


class NSq(C.Structure):
    _fields_ = _PTR3 + [("level", C.c_float)]


class NNb(C.Structure):
    _fields_ = _PTR3 + [("rate", C.c_float), ("inv_rate", C.c_float), ("level", C.c_float), ("amp", C.c_float)]


class NDe(C.Structure):
    _fields_ = _PTR3 + [("alpha", C.c_float), ("lastL", C.c_float), ("lastR", C.c_float)]


class NAm(C.Structure):
    _fields_ = _PTR3 + [("agcMode", C.c_int), ("carrier", AgcT), ("audio", AgcT), ("dcRate", C.c_float), ("dcOffset", C.c_float)]


class NSsb(C.Structure):
    _fields_ = _PTR3 + [("phase", C.c_float * 2), ("delta", C.c_float * 2), ("angle", C.c_double), ("agc", AgcT)]


def view(block, struct):
    """the restatement's C struct behind an oracle Block"""
    return struct.from_address(block._h)


def _f32(x):
    return float(np.float32(x))


def set_agc(agc, attack, decay):
    # loop::AGC::setAttack / setDecay (agc.h:32-44): float members, inv = 1.0f - member
    agc.attack = _f32(attack)
    agc.invAttack = _f32(np.float32(1.0) - np.float32(agc.attack))
    agc.decay = _f32(decay)
    agc.invDecay = _f32(np.float32(1.0) - np.float32(agc.decay))


def squelch_set_level(b, level):
    view(b, NSq).level = _f32(level)


def nb_set_level(b, level):
    view(b, NNb).level = _f32(level)


def deemph_set_tau(b, tau, sr):
    dt = _f32(1.0 / sr)                    # deephasis.h:91-94: float dt = 1.0f / samplerate, alpha = dt / (tau + dt)
    view(b, NDe).alpha = _f32(dt / (tau + dt))


def am_set_agc(b, attack, decay):
    a = view(b, NAm)
    set_agc(a.carrier, attack, decay)
    set_agc(a.audio, attack, decay)


def am_set_dc_rate(b, rate):
    view(b, NAm).dcRate = _f32(rate)


def am_set_agc_mode(b, mode):
    # AM::setAGCMode -> reset(): both AGCs and the DC blocker start over (am.h:49-56,90-98); the low-pass keeps its delay line
    a = view(b, NAm)
    a.agcMode = int(mode)
    for g in (a.carrier, a.audio):
        g.amp = _f32(np.float32(g.setPoint) / np.float32(g.initGain))
    a.dcOffset = 0.0


def ssb_set_agc(b, attack, decay):
    set_agc(view(b, NSsb).agc, attack, decay)


class OracleVfo:
    """One VFO of the radio module on the oracle: RxVFO -> [blanker] -> [squelch] -> [FM IF NR] -> demodulator ->
    [AF resampler -> [high-pass] -> [de-emphasis]] -> [volume], with every setter of b200_fe_set_vfo_config."""

    def __init__(self, oracle, fs, cfg, resume=True):
        """resume=False: a block switched off is dropped, so switching it on again starts a fresh one -- the semantics the
        tests must be able to tell apart from chain::setBlockEnabled's"""
        from sdrplusplus_b200 import lib as L
        self.o, self.L, self.cfg, self.resume = oracle, L, cfg, resume
        self.v = oracle.rxvfo(fs, cfg.out_samplerate, cfg.bandwidth, cfg.offset)
        sr = cfg.out_samplerate
        self.audio = cfg.demod not in (L.DEMOD_RAW, L.DEMOD_WFM_RDS, L.DEMOD_WFM_RDS_BITS)
        self.af = self.audio and cfg.af_samplerate > 0
        d = cfg.demod
        if d == L.DEMOD_WFM:
            self.d = oracle.wfm(cfg.deviation, sr, False, cfg.low_pass)
        elif d == L.DEMOD_NFM:
            self.d = oracle.nfm(sr, cfg.bandwidth, cfg.low_pass)
        elif d == L.DEMOD_AM:
            self.d = oracle.am(cfg.agc_mode, cfg.bandwidth, cfg.agc_attack, cfg.agc_decay, cfg.dc_block_rate, sr)
        elif d in (L.DEMOD_USB, L.DEMOD_LSB, L.DEMOD_DSB):
            self.d = oracle.ssb(d - L.DEMOD_USB, cfg.bandwidth, sr, cfg.agc_attack, cfg.agc_decay)
        elif d in (L.DEMOD_WFM_RDS, L.DEMOD_WFM_RDS_BITS):
            self.d = oracle.wfm_rds(cfg.deviation, sr)
        else:
            self.d = None
        self.r = oracle.resamp_stereo(sr, cfg.af_samplerate) if self.af else None
        self.nb = self.sq = self.nr = self.hp = self.de = None
        self.cur = None
        self.set(cfg)

    def set(self, c):
        """b200_fe_set_vfo_config's semantics, taken before the next process()"""
        o, sr = self.o, self.cfg.out_samplerate
        prev = self.cur
        if not self.resume:
            self.nb = self.nb if c.nb_on else None
            self.sq = self.sq if c.squelch_on else None
            self.nr = self.nr if c.nr_on else None
            self.hp = self.hp if c.af_high_pass else None
            self.de = self.de if c.af_deemph_tau > 0 else None
        if c.nb_on and self.nb is None:
            self.nb = o.noise_blanker(500.0 / sr, c.nb_level)
        if self.nb is not None:
            nb_set_level(self.nb, c.nb_level)
        if c.squelch_on and self.sq is None:
            self.sq = o.squelch(c.squelch_level)
        if self.sq is not None:
            squelch_set_level(self.sq, c.squelch_level)
        if prev is not None and c.nr_bins != prev.nr_bins:
            self.nr = None                                      # FMIF::setBins rebuilds the block
        if c.nr_on and self.nr is None:
            self.nr = o.fm_if(c.nr_bins)
        if self.af:
            if c.af_high_pass and self.hp is None:
                self.hp = o.fir_cr(o.highpass(300.0, 100.0, self.cfg.af_samplerate))
            if c.af_deemph_tau > 0 and self.de is None:
                self.de = o.deemph(c.af_deemph_tau, self.cfg.af_samplerate)
            if c.af_deemph_tau > 0:
                deemph_set_tau(self.de, c.af_deemph_tau, self.cfg.af_samplerate)
        if self.cfg.demod == self.L.DEMOD_AM:
            am_set_agc(self.d, c.agc_attack, c.agc_decay)
            am_set_dc_rate(self.d, c.dc_block_rate)
            if prev is not None and c.agc_mode != prev.agc_mode:
                am_set_agc_mode(self.d, c.agc_mode)
        elif self.cfg.demod in (self.L.DEMOD_USB, self.L.DEMOD_LSB, self.L.DEMOD_DSB):
            ssb_set_agc(self.d, c.agc_attack, c.agc_decay)
        if prev is not None and c.offset != prev.offset:
            self.v.set_offset(c.offset)
        if prev is not None and c.bandwidth != prev.bandwidth:
            self.v.set_bandwidth(c.bandwidth)
        self.cur = c

    def reset(self):
        for b in (self.v, self.nb, self.sq, self.nr, self.d, self.r, self.hp, self.de):
            if b is not None:
                b.reset()

    def process(self, xf):
        c = self.cur
        y = self.v.process(xf)
        if c.nb_on:
            y = self.nb.process(y)
        if c.squelch_on:
            y = self.sq.process(y)
        if c.nr_on:
            y = self.nr.process(y)
        if self.d is not None:
            y = self.d.process(y)
        if self.af:
            y = self.r.process(y)
            if c.af_high_pass:
                y = self.hp.process(y)
            if c.af_deemph_tau > 0:
                y = self.de.process(y)
        if self.audio and c.af_volume_on:
            y = y * np.float32(0.0 if c.af_muted else np.float32(np.float32(c.af_volume) ** np.float32(2)))
        return y

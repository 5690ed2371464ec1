"""Host-side mirrors of the reference interfaces on top of the C ABI.

FrontEnd          <-> IQFrontEnd (core/src/signal_path/iq_frontend.h:23-49) + the radio module's demodulator
                      behind each VFO (decoder_modules/radio/src/radio_module.h:80-125)
Block             <-> one dsp block: init(...) / process(count, in, out) -> out count (core/src/dsp/processor.h)
SpectrumHandler   <-> IQFrontEnd::handler on one framed block (iq_frontend.cpp:248-267)
"""
import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import lib as L


@dataclass
class VfoConfig:
    offset: float
    out_samplerate: float
    bandwidth: float
    demod: int = L.DEMOD_WFM
    deviation: float = 75000.0
    low_pass: bool = True
    agc_mode: int = L.AGC_AUDIO
    agc_attack: float = 0.0
    agc_decay: float = 0.0
    dc_block_rate: float = 0.0
    af_samplerate: float = 0.0       # radio AF chain: resample to this rate (0 = off) ...
    af_high_pass: bool = False       # ... 300 Hz high-pass ...
    af_deemph_tau: float = 0.0       # ... deemphasis time constant in seconds (0 = off)
    af_volume_on: bool = False       # dsp::audio::Volume at the end: out = in * (muted ? 0 : volume^2)
    af_muted: bool = False
    af_volume: float = 1.0
    squelch_on: bool = False         # noise_reduction::PowerSquelch in front of the demodulator (radio IF chain)
    squelch_level: float = -50.0
    nb_on: bool = False              # noise_reduction::NoiseBlanker in front of the squelch (rate 500 / out_samplerate)
    nb_level: float = 10.0
    nr_on: bool = False              # noise_reduction::FMIF behind the squelch
    nr_bins: int = 32

    def with_noise_blanker(self, level):
        self.nb_on, self.nb_level = True, level
        return self

    def with_if_nr(self, bins=32):
        self.nr_on, self.nr_bins = True, bins
        return self

    def with_volume(self, volume, muted=False):
        self.af_volume_on, self.af_volume, self.af_muted = True, volume, muted
        return self

    def with_squelch(self, level):
        self.squelch_on, self.squelch_level = True, level
        return self

    def with_af(self, audio_sr=48000.0, high_pass=False, deemph_tau=50e-6):
        self.af_samplerate, self.af_high_pass, self.af_deemph_tau = audio_sr, high_pass, deemph_tau
        return self

    @staticmethod
    def wfm(offset, bandwidth=150000.0):
        # decoder_modules/radio/src/demodulators/wfm.h:78,268-270: IF 250 kS/s, deviation = bandwidth/2
        return VfoConfig(offset, 250000.0, bandwidth, L.DEMOD_WFM, deviation=bandwidth / 2.0, low_pass=True)

    @staticmethod
    def wfm_stereo(offset, bandwidth=150000.0):
        return VfoConfig(offset, 250000.0, bandwidth, L.DEMOD_WFM_STEREO, deviation=bandwidth / 2.0, low_pass=True)

    @staticmethod
    def wfm_rds(offset, bandwidth=150000.0):
        # the RDS branch of BroadcastFM: complex baseband of the 57 kHz subcarrier at 5 kS/s (rds_demod.h's input)
        return VfoConfig(offset, 250000.0, bandwidth, L.DEMOD_WFM_RDS, deviation=bandwidth / 2.0)

    @staticmethod
    def wfm_rds_bits(offset, bandwidth=150000.0):
        # the same branch followed by RDSDemod: one (soft, bit) record per recovered symbol
        return VfoConfig(offset, 250000.0, bandwidth, L.DEMOD_WFM_RDS_BITS, deviation=bandwidth / 2.0)

    @staticmethod
    def nfm(offset, bandwidth=12500.0):
        return VfoConfig(offset, 50000.0, bandwidth, L.DEMOD_NFM, low_pass=True)          # nfm.h:29,56-58

    @staticmethod
    def am(offset, bandwidth=10000.0, agc_mode=L.AGC_AUDIO, attack=50.0, decay=5.0):
        sr = 15000.0                                                                       # am.h:34,76-78
        return VfoConfig(offset, sr, bandwidth, L.DEMOD_AM, agc_mode=agc_mode, agc_attack=attack / sr,
                         agc_decay=decay / sr, dc_block_rate=100.0 / sr)

    @staticmethod
    def ssb(offset, mode=L.DEMOD_USB, bandwidth=2800.0, attack=50.0, decay=5.0):
        sr = 24000.0                                                                       # usb.h:34,70-72
        return VfoConfig(offset, sr, bandwidth, mode, agc_attack=attack / sr, agc_decay=decay / sr)

    @staticmethod
    def raw(offset, out_samplerate, bandwidth):
        return VfoConfig(offset, out_samplerate, bandwidth, L.DEMOD_RAW)

    def to_c(self):
        return L.VfoCfg(self.offset, self.out_samplerate, self.bandwidth, self.demod, self.deviation, int(self.low_pass),
                        self.agc_mode, self.agc_attack, self.agc_decay, self.dc_block_rate, self.af_samplerate,
                        int(self.af_high_pass), self.af_deemph_tau, int(self.af_volume_on), int(self.af_muted), float(self.af_volume),
                        int(self.squelch_on), float(self.squelch_level), int(self.nb_on), float(self.nb_level),
                        int(self.nr_on), int(self.nr_bins))


_NP_FMT = {L.FMT_CF32: (np.complex64, 1), L.FMT_CS16: (np.int16, 2), L.FMT_CS8: (np.int8, 2)}
RDS_SYMBOL = np.dtype([("soft", np.float32), ("bit", np.uint32)])      # b200_rds_symbol


def rds_symbols(buf, n):
    """(soft float32, bit uint8) of the first n b200_rds_symbol records in a float32 output buffer"""
    r = np.ascontiguousarray(buf[: 2 * n]).view(RDS_SYMBOL)
    return r["soft"].copy(), r["bit"].astype(np.uint8)


def _as_input(iq, fmt):
    dt, per = _NP_FMT[fmt]
    a = np.ascontiguousarray(iq, dtype=dt).reshape(-1)
    return a, a.size // per


class FrontEnd:
    """One IQ stream -> FFT/waterfall lines + N VFO/demodulator outputs, one chunk per process()."""

    def __init__(self, samplerate, max_chunk=1000000, device=None):
        self._l = L.load()
        if device is not None:
            L.check(self._l.b200_init(device))
        self._h = L.check_ptr(self._l.b200_fe_create(float(samplerate), int(max_chunk)))
        self.samplerate = float(samplerate)
        self.max_chunk = int(max_chunk)
        self.fft_size = 0
        self.vfos = {}

    def close(self):
        if getattr(self, "_h", None):
            self._l.b200_fe_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # IQFrontEnd::setFFTSize / setFFTRate / setFFTWindow
    def set_fft(self, size, rate, window=L.WIN_NUTTALL):
        L.check(self._l.b200_fe_set_fft(self._h, int(size), float(rate), int(window)))
        self.fft_size = int(size)

    # IQFrontEnd::setDecimation / setDCBlocking / setInvertIQ
    def set_decimation(self, ratio):
        L.check(self._l.b200_fe_set_decimation(self._h, int(ratio)))

    def set_dc_blocking(self, on):
        L.check(self._l.b200_fe_set_dc_blocking(self._h, int(bool(on))))

    def set_invert_iq(self, on):
        L.check(self._l.b200_fe_set_invert_iq(self._h, int(bool(on))))

    def set_stream(self, cuda_stream):
        L.check(self._l.b200_fe_set_stream(self._h, C.c_void_p(cuda_stream)))

    def add_vfo(self, cfg):
        c = cfg.to_c()
        vid = L.check(self._l.b200_fe_add_vfo(self._h, C.byref(c)))
        self.vfos[vid] = cfg
        return vid

    def remove_vfo(self, vid):
        L.check(self._l.b200_fe_remove_vfo(self._h, vid))
        self.vfos.pop(vid, None)

    def set_vfo_offset(self, vid, offset):
        L.check(self._l.b200_fe_set_vfo_offset(self._h, vid, float(offset)))

    def set_vfo_bandwidth(self, vid, bw):
        L.check(self._l.b200_fe_set_vfo_bandwidth(self._h, vid, float(bw)))

    def set_ingest_scale(self, fmt, scale):
        """Conversion factor of the next int16 / int8 chunks (a compressed-stream packet's scaler); <= 0: default."""
        L.check(self._l.b200_fe_set_ingest_scale(self._h, int(fmt), float(scale)))

    def set_option(self, key, value):
        L.check(self._l.b200_fe_set_option(self._h, key.encode(), int(value)))

    def reset(self):
        L.check(self._l.b200_fe_reset(self._h))

    def s1_stats(self):
        ms, n = C.c_double(), C.c_int()
        L.check(self._l.b200_fe_s1_stats(self._h, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def group_stats(self, group):
        """(ms_total, launches) of a timed launch group since the last call: 0 stage 1, 1 behind stage 1, 2 spectrum branch"""
        ms, n = C.c_double(), C.c_int()
        L.check(self._l.b200_fe_group_stats(self._h, int(group), C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def launch_count(self):
        return self._l.b200_fe_launch_count(self._h)

    def stat(self, key):
        return self._l.b200_fe_stat(self._h, key.encode())

    def vfo_max_out(self, vid, count):
        return L.check(self._l.b200_fe_vfo_max_out(self._h, vid, count))

    def fft_max_lines(self, count):
        return self._l.b200_fe_fft_max_lines(self._h, count)

    def _alloc_outputs(self, count):
        o = L.Outputs()
        bufs = {}
        for vid, cfg in self.vfos.items():
            cap = self.vfo_max_out(vid, count)
            b = np.empty(cap * 2, np.float32)
            bufs[vid] = b
            o.vfo_out[vid] = b.ctypes.data
            o.vfo_cap[vid] = cap
        fft = None
        if self.fft_size:
            nl = self.fft_max_lines(count)
            fft = np.empty((nl, self.fft_size), np.float32)
            o.fft_out = fft.ctypes.data
            o.fft_cap_lines = nl
        o.out_mem = L.MEM_HOST
        return o, bufs, fft

    def process(self, iq, fmt=L.FMT_CF32):
        """Host numpy in, host numpy out.  Returns ({vfo_id: array}, fft_lines[n, N]); a DEMOD_WFM_RDS_BITS VFO gives the
        pair (soft float32, bit uint8)."""
        a, count = _as_input(iq, fmt)
        o, bufs, fft = self._alloc_outputs(count)
        L.check(self._l.b200_fe_process(self._h, a.ctypes.data, count, fmt, L.MEM_HOST, C.byref(o)))
        outs = {}
        for vid, cfg in self.vfos.items():
            n = o.vfo_count[vid]
            if cfg.demod == L.DEMOD_WFM_RDS_BITS:
                outs[vid] = rds_symbols(bufs[vid], n)
                continue
            y = bufs[vid][: 2 * n].copy()
            outs[vid] = y.view(np.complex64) if cfg.demod in (L.DEMOD_RAW, L.DEMOD_WFM_RDS) else y.reshape(-1, 2)
        lines = fft[: o.fft_lines].copy() if fft is not None else np.empty((0, 0), np.float32)
        return outs, lines

    def process_chunks(self, iq, chunk, fmt=L.FMT_CF32):
        a, count = _as_input(iq, fmt)
        per = _NP_FMT[fmt][1]
        acc = {vid: [] for vid in self.vfos}
        lines = []
        for i in range(0, count, chunk):
            outs, ln = self.process(a[i * per:(i + chunk) * per], fmt)
            for vid, y in outs.items():
                acc[vid].append(y)
            if ln.size:
                lines.append(ln)
        res = {}
        for vid, v in acc.items():
            if self.vfos[vid].demod == L.DEMOD_WFM_RDS_BITS:
                res[vid] = (np.concatenate([p[0] for p in v]) if v else np.empty(0, np.float32),
                            np.concatenate([p[1] for p in v]) if v else np.empty(0, np.uint8))
            else:
                res[vid] = np.concatenate(v) if v else np.empty(0, np.float32)
        return res, (np.concatenate(lines) if lines else np.empty((0, self.fft_size), np.float32))

    # raw-pointer variants used by bench.py (device-resident or pinned buffers, no numpy copies)
    def submit_ptr(self, ptr, count, fmt, mem, outputs):
        L.check(self._l.b200_fe_submit(self._h, C.c_void_p(ptr), count, fmt, mem, C.byref(outputs)))

    def process_ptr(self, ptr, count, fmt, mem, outputs):
        L.check(self._l.b200_fe_process(self._h, C.c_void_p(ptr), count, fmt, mem, C.byref(outputs)))

    def wait(self):
        L.check(self._l.b200_fe_wait(self._h))


class Block:
    """Stand-alone block with the reference's process(count, in, out) contract; state carried across calls."""

    def __init__(self, handle, in_floats, out_floats):
        self._l = L.load()
        self._h = L.check_ptr(handle)
        self._in_f, self._out_f = in_floats, out_floats

    @staticmethod
    def xlator(offset_hz, sr):
        return Block(L.load().b200_xlator_create(offset_hz, sr), 2, 2)

    @staticmethod
    def decim(ratio):
        return Block(L.load().b200_decim_create(ratio), 2, 2)

    @staticmethod
    def resamp(in_sr, out_sr):
        return Block(L.load().b200_resamp_create(in_sr, out_sr), 2, 2)

    @staticmethod
    def fir_cr(taps, decim=1):
        t = np.ascontiguousarray(taps, np.float32)
        return Block(L.load().b200_fir_cr_create(t.ctypes.data, t.size, decim), 2, 2)

    @staticmethod
    def fir_rr(taps):
        t = np.ascontiguousarray(taps, np.float32)
        return Block(L.load().b200_fir_rr_create(t.ctypes.data, t.size), 1, 1)

    @staticmethod
    def rxvfo(in_sr, out_sr, bw, offset):
        return Block(L.load().b200_rxvfo_create(in_sr, out_sr, bw, offset), 2, 2)

    @staticmethod
    def quad(dev, sr):
        return Block(L.load().b200_quad_create(dev, sr), 2, 1)

    @staticmethod
    def wfm(dev, sr, stereo=False, lowpass=True):
        return Block(L.load().b200_wfm_create(dev, sr, int(stereo), int(lowpass)), 2, 2)

    @staticmethod
    def wfm_rds(dev, sr):
        return Block(L.load().b200_wfm_rds_create(dev, sr), 2, 2)

    @staticmethod
    def nfm(sr, bw, lowpass=True):
        return Block(L.load().b200_nfm_create(sr, bw, int(lowpass)), 2, 2)

    @staticmethod
    def am(agc_mode, bw, attack, decay, dcrate, sr):
        return Block(L.load().b200_am_create(agc_mode, bw, attack, decay, dcrate, sr), 2, 2)

    @staticmethod
    def ssb(mode, bw, sr, attack, decay):
        return Block(L.load().b200_ssb_create(mode, bw, sr, attack, decay), 2, 2)

    @staticmethod
    def deemph(tau, sr):
        return Block(L.load().b200_deemph_create(tau, sr), 2, 2)

    @staticmethod
    def squelch(level):
        return Block(L.load().b200_squelch_create(level), 2, 2)

    @staticmethod
    def noise_blanker(rate, level):
        return Block(L.load().b200_noise_blanker_create(rate, level), 2, 2)

    @staticmethod
    def fm_if(bins):
        return Block(L.load().b200_fmif_create(bins), 2, 2)

    def set_offset(self, *a):
        if len(a) == 2:
            L.check(self._l.b200_xlator_set_offset(self._h, a[0], a[1]))
        else:
            L.check(self._l.b200_rxvfo_set_offset(self._h, a[0]))

    def set_bandwidth(self, bw):
        L.check(self._l.b200_rxvfo_set_bandwidth(self._h, bw))

    def process(self, x):
        x = np.ascontiguousarray(x, np.float32).reshape(-1)
        count = x.size // self._in_f
        cap = L.check(self._l.b200_block_max_out(self._h, count))
        out = np.empty(max(cap, 1) * self._out_f, np.float32)
        n = L.check(self._l.b200_block_process(self._h, count, x.ctypes.data, out.ctypes.data))
        return out[: n * self._out_f].copy()

    def process_chunks(self, x, chunk):
        x = np.ascontiguousarray(x, np.float32).reshape(-1)
        step = chunk * self._in_f
        outs = [self.process(x[i:i + step]) for i in range(0, x.size, step)]
        return np.concatenate(outs) if outs else np.empty(0, np.float32)

    def reset(self):
        L.check(self._l.b200_block_reset(self._h))

    def close(self):
        if getattr(self, "_h", None):
            self._l.b200_block_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class RdsDemod:
    """RDSDemod (decoder_modules/radio/src/rds_demod.h): complex at 5 kS/s in -> (soft float32, decoded bits uint8) per symbol."""

    def __init__(self):
        self._l = L.load()
        self._h = L.check_ptr(self._l.b200_rds_demod_create())

    def process(self, x):
        """x: complex64 numpy array, or a CUDA tensor of interleaved float32 (re, im) pairs (read in place)."""
        if hasattr(x, "data_ptr"):
            count, ptr = x.numel() // 2, x.data_ptr()
        else:
            x = np.ascontiguousarray(x, np.complex64).reshape(-1)
            count, ptr = x.size, x.ctypes.data
        cap = max(1, self._l.b200_rds_demod_max_out(count))
        soft, hard = np.empty(cap, np.float32), np.empty(cap, np.uint8)
        n = L.check(self._l.b200_rds_demod_process(self._h, count, ptr, soft.ctypes.data, hard.ctypes.data))
        return soft[:n].copy(), hard[:n].copy()

    def process_chunks(self, x, chunk):
        x = np.ascontiguousarray(x, np.complex64).reshape(-1)
        parts = [self.process(x[i:i + chunk]) for i in range(0, x.size, chunk)]
        if not parts:
            return np.empty(0, np.float32), np.empty(0, np.uint8)
        return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])

    def reset(self):
        L.check(self._l.b200_rds_demod_reset(self._h))

    def launch_count(self):
        return self._l.b200_rds_demod_launch_count(self._h)

    def close(self):
        if getattr(self, "_h", None):
            self._l.b200_rds_demod_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class SpectrumHandler:
    def __init__(self, size, nz, window=L.WIN_NUTTALL):
        self._l = L.load()
        self._h = L.check_ptr(self._l.b200_fft_create(size, nz, window))
        self.size, self.nz = size, nz

    def frame(self, iq):
        iq = np.ascontiguousarray(iq, np.complex64)
        assert iq.size == self.nz
        out = np.empty(self.size, np.float32)
        L.check(self._l.b200_fft_frame(self._h, iq.ctypes.data, out.ctypes.data))
        return out

    def raw(self, iq):
        iq = np.ascontiguousarray(iq, np.complex64)
        out = np.empty(self.size, np.complex64)
        L.check(self._l.b200_fft_raw(self._h, iq.ctypes.data, out.ctypes.data))
        return out

    def close(self):
        if getattr(self, "_h", None):
            self._l.b200_fft_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def zoom_hold(line, offset, width, out_size, hold=None, hold_speed=0.0):
    """doZoom + peak hold on the GPU (waterfall.cpp:65-90,935-939); returns (out, hold)."""
    l = L.load()
    line = np.ascontiguousarray(line, np.float32)
    out = np.empty(out_size, np.float32)
    h = None if hold is None else np.ascontiguousarray(hold, np.float32).copy()
    L.check(l.b200_fft_zoom_hold(line.ctypes.data, line.size, offset, width, out_size, out.ctypes.data,
                                 None if h is None else h.ctypes.data, hold_speed, L.MEM_HOST))
    return out, h


def taps_lowpass(cutoff, tw, sr, odd=False):
    l = L.load()
    n = l.b200_taps_lowpass(cutoff, tw, sr, int(odd), None, 0)
    out = np.empty(n, np.float32)
    l.b200_taps_lowpass(cutoff, tw, sr, int(odd), out.ctypes.data, n)
    return out


def taps_highpass(cutoff, tw, sr, odd=False):
    l = L.load()
    n = l.b200_taps_highpass(cutoff, tw, sr, int(odd), None, 0)
    out = np.empty(n, np.float32)
    l.b200_taps_highpass(cutoff, tw, sr, int(odd), out.ctypes.data, n)
    return out


def window(win, nz):
    l = L.load()
    out = np.empty(nz, np.float32)
    L.check(l.b200_window(win, nz, out.ctypes.data))
    return out


def resamp_plan(in_sr, out_sr):
    l = L.load()
    p = L.ResampPlan()
    L.check(l.b200_resamp_plan_get(in_sr, out_sr, C.byref(p)))
    return {"mode": p.mode, "predec_ratio": p.predec_ratio, "stages": [(p.stage_decim[i], p.stage_taps[i]) for i in range(p.nstages)],
            "interp": p.interp, "decim": p.decim, "ntaps": p.ntaps, "taps_per_phase": p.taps_per_phase}


def fft_frame_params(sr, size, rate):
    l = L.load()
    nz, skip = C.c_int(), C.c_int()
    L.check(l.b200_fft_frame_params(sr, size, rate, C.byref(nz), C.byref(skip)))
    return nz.value, skip.value


# ---------------------------------------------------------------------------------------------- data formats
EXPORT_U8, EXPORT_I16, EXPORT_I32 = 0, 1, 2


def pcm_packet_info(packet):
    """(fmt, scale, count, data_offset) of a SampleStreamCompressor packet (bytes / uint8 array)."""
    b = np.ascontiguousarray(np.frombuffer(packet, np.uint8) if isinstance(packet, (bytes, bytearray)) else packet, np.uint8)
    fmt, cnt, off = C.c_int(), C.c_int(), C.c_int()
    sc = C.c_float()
    L.check(L.load().b200_pcm_packet_info(b.ctypes.data, int(b.size), C.byref(fmt), C.byref(sc), C.byref(cnt), C.byref(off)))
    return fmt.value, sc.value, cnt.value, off.value


def pcm_compress(iq, pcm_fmt):
    """SampleStreamCompressor::process on the device: complex64 in, packet bytes (uint8 array) out."""
    x = np.ascontiguousarray(iq, np.complex64)
    out = np.empty(8 + x.size * 8, np.uint8)
    n = L.check(L.load().b200_pcm_compress(x.ctypes.data, int(x.size), int(pcm_fmt), out.ctypes.data, int(out.size), L.MEM_HOST))
    return out[:n].copy()


def export_convert(x, sample_type):
    """wav::Writer sample conversion on the device: float32 in, uint8 / int16 / int32 out."""
    a = np.ascontiguousarray(x, np.float32).reshape(-1)
    dt = {EXPORT_U8: np.uint8, EXPORT_I16: np.int16, EXPORT_I32: np.int32}[sample_type]
    out = np.empty(a.size, dt)
    L.check(L.load().b200_export_convert(a.ctypes.data, int(a.size), int(sample_type), out.ctypes.data, L.MEM_HOST))
    return out

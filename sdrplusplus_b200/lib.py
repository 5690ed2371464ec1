"""ctypes declaration of every entry point of include/b200dsp.h."""
import ctypes as C
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200dsp.so")
HEADER_PATH = os.path.join(_HERE, "..", "include", "b200dsp.h")

MAX_VFOS = 64
FMT_CF32, FMT_CS16, FMT_CS8 = 0, 1, 2
MEM_HOST, MEM_DEVICE = 0, 1
WIN_RECTANGULAR, WIN_BLACKMAN, WIN_NUTTALL = 0, 1, 2
DEMOD_RAW, DEMOD_WFM, DEMOD_NFM, DEMOD_AM, DEMOD_USB, DEMOD_LSB, DEMOD_DSB, DEMOD_WFM_STEREO, DEMOD_WFM_RDS = range(9)
DEMOD_WFM_RDS_BITS = 9
AGC_CARRIER, AGC_AUDIO = 0, 1
IQ_CF32, IQ_U8, IQ_I8, IQ_I16, IQ_I32 = range(5)        # b200_fe_bind_iq sample types
E = {0: "OK", -1: "EINVAL", -2: "ENODEV", -3: "ECUDA", -4: "ENOMEM", -5: "ECAP", -6: "ENOPLAN", -7: "ESTATE"}


class B200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("b200dsp error %s (%d): %s" % (E.get(code, "?"), code, msg))
        self.code = code


class VfoCfg(C.Structure):
    _fields_ = [("offset", C.c_double), ("out_samplerate", C.c_double), ("bandwidth", C.c_double), ("demod", C.c_int),
                ("deviation", C.c_double), ("low_pass", C.c_int), ("agc_mode", C.c_int), ("agc_attack", C.c_double),
                ("agc_decay", C.c_double), ("dc_block_rate", C.c_double), ("af_samplerate", C.c_double),
                ("af_high_pass", C.c_int), ("af_deemph_tau", C.c_double), ("af_volume_on", C.c_int), ("af_muted", C.c_int),
                ("af_volume", C.c_double), ("squelch_on", C.c_int), ("squelch_level", C.c_double),
                ("nb_on", C.c_int), ("nb_level", C.c_double), ("nr_on", C.c_int), ("nr_bins", C.c_int)]


class Outputs(C.Structure):
    _fields_ = [("vfo_out", C.c_void_p * MAX_VFOS), ("vfo_cap", C.c_int * MAX_VFOS), ("vfo_count", C.c_int * MAX_VFOS),
                ("fft_out", C.c_void_p), ("fft_cap_lines", C.c_int), ("fft_lines", C.c_int), ("out_mem", C.c_int)]


class RdsSymbol(C.Structure):
    """b200_rds_symbol: one record per recovered symbol of a DEMOD_WFM_RDS_BITS VFO"""
    _fields_ = [("soft", C.c_float), ("bit", C.c_uint32)]


class ResampPlan(C.Structure):
    _fields_ = [("mode", C.c_int), ("predec_ratio", C.c_int), ("nstages", C.c_int), ("stage_decim", C.c_int * 8),
                ("stage_taps", C.c_int * 8), ("interp", C.c_int), ("decim", C.c_int), ("ntaps", C.c_int),
                ("taps_per_phase", C.c_int)]


_vp, _d, _i, _ll = C.c_void_p, C.c_double, C.c_int, C.c_longlong
_ip = C.POINTER(C.c_int)
SIGNATURES = {
    "b200_init": (_i, [_i]),
    "b200_device_count": (_i, []),
    "b200_last_error": (C.c_char_p, []),
    "b200_version": (_i, []),
    "b200_register_decim_plan": (_i, [_i, _i, _ip, _ip, C.POINTER(C.POINTER(C.c_float))]),
    "b200_load_decim_plans": (_i, [C.c_char_p]),
    "b200_taps_lowpass": (_i, [_d, _d, _d, _i, _vp, _i]),
    "b200_taps_highpass": (_i, [_d, _d, _d, _i, _vp, _i]),
    "b200_taps_bandpass": (_i, [_d, _d, _d, _d, _i, _vp, _i]),
    "b200_window": (_i, [_i, _i, _vp]),
    "b200_fft_frame_params": (_i, [_d, _i, _d, _ip, _ip]),
    "b200_resamp_plan_get": (_i, [_d, _d, C.POINTER(ResampPlan)]),
    "b200_fe_create": (_vp, [_d, _i]),
    "b200_fe_destroy": (None, [_vp]),
    "b200_fe_set_stream": (_i, [_vp, _vp]),
    "b200_fe_set_fft": (_i, [_vp, _i, _d, _i]),
    "b200_fe_set_decimation": (_i, [_vp, _i]),
    "b200_fe_set_dc_blocking": (_i, [_vp, _i]),
    "b200_fe_set_invert_iq": (_i, [_vp, _i]),
    "b200_fe_add_vfo": (_i, [_vp, C.POINTER(VfoCfg)]),
    "b200_fe_remove_vfo": (_i, [_vp, _i]),
    "b200_fe_set_vfo_offset": (_i, [_vp, _i, _d]),
    "b200_fe_set_vfo_bandwidth": (_i, [_vp, _i, _d]),
    "b200_fe_set_vfo_config": (_i, [_vp, _i, C.POINTER(VfoCfg)]),
    "b200_fe_bind_iq": (_i, [_vp, _i, C.c_float]),
    "b200_fe_unbind_iq": (_i, [_vp, _i]),
    "b200_fe_bind_rds": (_i, [_vp, _i]),
    "b200_fe_unbind_rds": (_i, [_vp, _i]),
    "b200_fe_vfo_count": (_i, [_vp]),
    "b200_fe_vfo_max_out": (_i, [_vp, _i, _i]),
    "b200_fe_fft_max_lines": (_i, [_vp, _i]),
    "b200_fe_reset": (_i, [_vp]),
    "b200_fe_process": (_i, [_vp, _vp, _i, _i, _i, C.POINTER(Outputs)]),
    "b200_fe_submit": (_i, [_vp, _vp, _i, _i, _i, C.POINTER(Outputs)]),
    "b200_fe_wait": (_i, [_vp]),
    "b200_fe_launch_count": (_ll, [_vp]),
    "b200_fe_stat": (_ll, [_vp, C.c_char_p]),
    "b200_fe_set_option": (_i, [_vp, C.c_char_p, _i]),
    "b200_fe_s1_stats": (_i, [_vp, C.POINTER(C.c_double), _ip]),
    "b200_fe_group_stats": (_i, [_vp, _i, C.POINTER(C.c_double), _ip]),
    "b200_shard_unique_id": (_i, [_vp]),
    "b200_shard_create": (_vp, [_vp, _i, _i, _vp]),
    "b200_shard_submit": (_i, [_vp, _vp, _i, _i, _i, C.POINTER(Outputs)]),
    "b200_shard_wait": (_i, [_vp]),
    "b200_shard_bytes_broadcast": (_ll, [_vp]),
    "b200_shard_destroy": (None, [_vp]),
    "b200_fft_zoom_hold": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, C.c_float, _i]),
    "b200_xlator_create": (_vp, [_d, _d]),
    "b200_xlator_set_offset": (_i, [_vp, _d, _d]),
    "b200_decim_create": (_vp, [_i]),
    "b200_resamp_create": (_vp, [_d, _d]),
    "b200_fir_cr_create": (_vp, [_vp, _i, _i]),
    "b200_fir_cr_set_taps": (_i, [_vp, _vp, _i]),
    "b200_fir_rr_create": (_vp, [_vp, _i]),
    "b200_rxvfo_create": (_vp, [_d, _d, _d, _d]),
    "b200_rxvfo_set_offset": (_i, [_vp, _d]),
    "b200_rxvfo_set_bandwidth": (_i, [_vp, _d]),
    "b200_quad_create": (_vp, [_d, _d]),
    "b200_wfm_create": (_vp, [_d, _d, _i, _i]),
    "b200_nfm_create": (_vp, [_d, _d, _i]),
    "b200_am_create": (_vp, [_i, _d, _d, _d, _d, _d]),
    "b200_ssb_create": (_vp, [_i, _d, _d, _d, _d]),
    "b200_squelch_create": (_vp, [_d]),
    "b200_noise_blanker_create": (_vp, [_d, _d]),
    "b200_fmif_create": (_vp, [_i]),
    "b200_wfm_rds_create": (_vp, [_d, _d]),
    "b200_noise_blanker_set": (_i, [_vp, _d, _d]),
    "b200_deemph_create": (_vp, [_d, _d]),
    "b200_block_process": (_i, [_vp, _i, _vp, _vp]),
    "b200_block_max_out": (_i, [_vp, _i]),
    "b200_block_reset": (_i, [_vp]),
    "b200_block_destroy": (None, [_vp]),
    "b200_rds_demod_create": (_vp, []),
    "b200_rds_demod_process": (_i, [_vp, _i, _vp, _vp, _vp]),
    "b200_rds_demod_max_out": (_i, [_i]),
    "b200_rds_demod_reset": (_i, [_vp]),
    "b200_rds_demod_launch_count": (_ll, [_vp]),
    "b200_rds_demod_taps": (_i, [_vp, _i, _vp]),
    "b200_rds_demod_destroy": (None, [_vp]),
    "b200_fft_create": (_vp, [_i, _i, _i]),
    "b200_fft_frame": (_i, [_vp, _vp, _vp]),
    "b200_fft_raw": (_i, [_vp, _vp, _vp]),
    "b200_fft_destroy": (None, [_vp]),
    "b200_chan_create": (_vp, [_i, _i, _i]),
    "b200_chan_prototype": (_i, [_vp, _vp, _i]),
    "b200_chan_process": (_i, [_vp, _vp, _i, _i, _vp, _i]),
    "b200_chan_launch_count": (_ll, [_vp]),
    "b200_chan_destroy": (None, [_vp]),
    "b200_host_alloc": (_vp, [C.c_uint64]),
    "b200_host_free": (None, [_vp]),
    "b200_pcm_packet_info": (_i, [_vp, _i, _ip, C.POINTER(C.c_float), _ip, _ip]),
    "b200_fe_set_ingest_scale": (_i, [_vp, _i, C.c_float]),
    "b200_pcm_compress": (_i, [_vp, _i, _i, _vp, _i, _i]),
    "b200_export_convert": (_i, [_vp, C.c_longlong, _i, _vp, _i]),
}

_lib = None


def header_symbols():
    """Every function name include/b200dsp.h declares (used by the CPU-side export test)."""
    with open(HEADER_PATH) as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", text)))


def load():
    """dlopen libb200dsp.so and bind every declared symbol.  Makes no CUDA call."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FileNotFoundError("%s missing: run `python __graft_entry__.py` (there is no CPU fallback)" % LIB_PATH)
    L = C.CDLL(LIB_PATH, mode=C.RTLD_LOCAL)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(L, name)     # AttributeError if the library does not export a declared symbol
        fn.restype, fn.argtypes = res, args
    _lib = L
    return L


def check(code):
    if code is not None and code < 0:
        raise B200Error(code, load().b200_last_error().decode(errors="replace"))
    return code


def check_ptr(p):
    if not p:
        L = load()
        msg = L.b200_last_error().decode(errors="replace")
        raise B200Error(-2 if "no usable CUDA device" in msg else -1, msg)
    return p

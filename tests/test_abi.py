"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol that
include/b200dsp.h declares, refuses to compute without a device, and its host-side design helpers are
bit-identical to the reference's formulas (checked through the oracle)."""
import ctypes as C

import numpy as np
import pytest

from sdrplusplus_b200 import lib, frontend


def test_library_exports_every_declared_symbol():
    L = lib.load()
    declared = lib.header_symbols()
    assert len(declared) >= 50
    for name in declared:
        assert hasattr(L, name), "libb200dsp.so does not export %s" % name
        assert name in lib.SIGNATURES, "python binding lacks %s" % name
    assert L.b200_version() == 100


def test_no_device_fails_loudly():
    L = lib.load()
    if L.b200_device_count() > 0:
        pytest.skip("a CUDA device is present")
    assert L.b200_init(0) == -2
    assert b"no CPU fallback" in L.b200_last_error()
    assert not L.b200_fe_create(2.4e6, 1000)
    assert not L.b200_rxvfo_create(2.4e6, 250e3, 150e3, 0.0)
    assert not L.b200_fft_create(1024, 1024, 2)
    with pytest.raises(lib.B200Error):
        frontend.FrontEnd(2.4e6)


def test_bad_arguments_return_error_codes():
    L = lib.load()
    assert L.b200_register_decim_plan(3, 1, None, None, None) == -1
    assert L.b200_resamp_plan_get(1e6, 1e5, None) == -1
    assert L.b200_fft_frame_params(1e6, 1024, 0.0, None, None) == -1


@pytest.mark.parametrize("args", [(15000.0, 4000.0, 250000.0, False), (75000.0, 7500.0, 250000.0, False),
                                  (6250.0, 625.0, 50000.0, False), (1400.0, 140.0, 24000.0, True),
                                  (125000.0, 12500.0, 6250000.0, False)])
def test_lowpass_taps_bit_exact(oracle, args):
    a = frontend.taps_lowpass(*args)
    b = oracle.lowpass(*args)
    assert a.size == b.size
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_highpass_taps_bit_exact(oracle):
    a = frontend.taps_highpass(300.0, 100.0, 48000.0)
    b = oracle.highpass(300.0, 100.0, 48000.0)
    assert a.size == b.size == 1824
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


BANDPASS_SETS = [(18750.0, 19250.0, 3000.0, 250000.0, True), (18750.0, 19250.0, 3000.0, 200000.0, True),   # stereo pilot
                 (1000.0, 3000.0, 500.0, 48000.0, False), (1000.0, 3000.0, 500.0, 48000.0, True),          # even count
                 (0.0, 2375.0, 100.0, 5000.0, False)]                                                     # RDSDemod


@pytest.mark.parametrize("args", BANDPASS_SETS)
def test_bandpass_taps_bit_exact(oracle, args):
    """taps::bandPass<complex_t>: the pilot filter of BroadcastFM's stereo branch (odd count, centre off zero) at both IF
    rates, a set whose estimated count is even with and without the odd fix-up, and RDSDemod's zero-centred set"""
    a = frontend.taps_bandpass(*args)
    b = oracle.bandpass_c(*args)
    assert a.dtype == np.complex64 and a.size == b.size > 0
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    if args[2:4] == (500.0, 48000.0):
        assert a.size % 2 == int(args[4])                     # the estimate is even: odd=True adds the one tap
    if args[0] == 18750.0:
        assert a.size % 2 == 1 and np.abs(a.imag).max() > 0


def test_bandpass_taps_cap():
    L = lib.load()
    n = L.b200_taps_bandpass(18750.0, 19250.0, 3000.0, 250000.0, 1, None, 0)
    out = np.full(2 * n, 7.0, np.float32)
    assert L.b200_taps_bandpass(18750.0, 19250.0, 3000.0, 250000.0, 1, out.ctypes.data, 5) == n == 317
    full = frontend.taps_bandpass(18750.0, 19250.0, 3000.0, 250000.0, True)
    assert np.array_equal(out[:10].view(np.uint32), full[:5].view(np.float32).view(np.uint32))
    assert np.all(out[10:] == 7.0)


@pytest.mark.parametrize("win,nz", [(0, 1000), (1, 4097), (2, 65536), (2, 12000)])
def test_window_bit_exact(oracle, win, nz):
    assert np.array_equal(frontend.window(win, nz).view(np.uint32), oracle.window_buf(win, nz).view(np.uint32))


@pytest.mark.parametrize("rates", [(2.4e6, 250e3), (100e6, 250e3), (1.024e9, 250e3), (2.4e6, 50e3), (2.4e6, 15e3),
                                   (2.4e6, 24e3), (250e3, 48e3), (48e3, 250e3), (1e6, 1e6), (100e6, 50e3), (1.024e9, 24e3)])
def test_resampler_plan_matches(oracle, rates):
    p = frontend.resamp_plan(*rates)
    q = oracle.resamp_plan(*rates)
    for k in ("mode", "predec_ratio", "interp", "decim", "ntaps", "taps_per_phase"):
        assert p[k] == q[k], (k, p, q)
    if p["predec_ratio"] > 1:
        assert p["stages"] == oracle.decim_plan(p["predec_ratio"])


@pytest.mark.parametrize("cfg", [(2.4e6, 65536, 20.0), (100e6, 1 << 20, 20.0), (8e6, 1024, 20.0), (1e6, 65536, 60.0)])
def test_frame_params_match(oracle, cfg):
    nz, skip = frontend.fft_frame_params(*cfg)
    assert (skip, nz) == oracle.fft_params(*cfg)


def test_decim_plan_table_loads():
    L = lib.load()
    assert L.b200_load_decim_plans(None) == 0
    assert L.b200_load_decim_plans(b"/nonexistent/file") == -6


def test_fused_tail_range_arithmetic_invariants():
    """csrc/kernels.cuh ft_ranges / ft_need_in (shared by the CUDA kernel and the scheduler): slabs tile the outputs,
    every stage's needs are met by what the previous stage produces, the last slab hands over every history."""
    import os
    import subprocess
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build", "test_ft_ranges")
    assert os.path.exists(exe), "run python __graft_entry__.py first"
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "ok" in r.stdout


def test_pcm_packet_header_parsing_matches_reference_decompressor(oracle):
    """b200_pcm_packet_info is host-only: format, sample count and the conversion factor must be what
    SampleStreamDecompressor::process (sample_stream_decompressor.h:15-33) derives from the same header."""
    import numpy as np
    from sdrplusplus_b200 import frontend, lib as L
    rng = np.random.default_rng(5)
    x = (rng.standard_normal(777) + 1j * rng.standard_normal(777)).astype(np.complex64) * 0.2
    for pcm, fmt, dt in ((1, L.FMT_CS16, np.int16), (0, L.FMT_CS8, np.int8), (2, L.FMT_CF32, np.float32)):
        pkt = oracle.pcm_compress(x, pcm)
        f, sc, cnt, off = frontend.pcm_packet_info(pkt)
        assert (f, cnt, off) == (fmt, x.size, 8)
        ref = oracle.pcm_decompress(pkt).view(np.float32)
        payload = pkt[off:].view(dt)
        mine = payload.astype(np.float32) * np.float32(sc) if pcm != 2 else payload
        assert np.array_equal(mine.view(np.uint32), ref.view(np.uint32))      # (float)x * scale, bit for bit
    with pytest.raises(L.B200Error):
        frontend.pcm_packet_info(np.zeros(4, np.uint8))
    bad = oracle.pcm_compress(x, 1).copy()
    bad[2] = 9
    with pytest.raises(L.B200Error):
        frontend.pcm_packet_info(bad)


def test_rds_demod_tap_sets_bit_exact(oracle):
    """RDSDemod's two designed tap sets (band-pass of rds_demod.h:29, MM's 128 x 8 interpolator bank of mm.h:168-173) as the
    library's host side designs them, against the oracle (itself pinned to the reference build)."""
    L = lib.load()
    bp = np.zeros(2 * 256, np.float32)
    bank = np.zeros(128 * 8, np.float32)
    n = L.b200_rds_demod_taps(bp.ctypes.data, 256, bank.ctypes.data)
    obp, obank = oracle.rds_demod_taps()
    assert n == obp.size == 190
    assert np.array_equal(bp[: 2 * n].view(np.uint32), obp.view(np.float32).view(np.uint32))
    assert np.array_equal(bank.view(np.uint32), obank.reshape(-1).view(np.uint32))
    assert L.b200_rds_demod_max_out(0) == 2 and L.b200_rds_demod_max_out(5000) >= 1188 + 12


def test_shipped_library_carries_the_hopper_paths():
    """cuobjdump census of libb200dsp.so: sm_90a only; stage 1 is fed by the TMA engine under mbarriers (UTMALDG, SYNCS) and
    filters with fp32 FMAs (two per complex sample); the chain kernels behind it carry the programmatic
    dependent launch pair (PREEXIT = griddepcontrol.launch_dependents, ACQBULK = griddepcontrol.wait)."""
    import shutil
    import subprocess
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    try:
        elf = subprocess.run([exe, "-lelf", lib.LIB_PATH], capture_output=True, text=True, timeout=120)
        sass = subprocess.run([exe, "-sass", lib.LIB_PATH], capture_output=True, text=True, timeout=600)
    except (OSError, subprocess.TimeoutExpired):
        pytest.skip("cuobjdump not available")
    if elf.returncode != 0 or sass.returncode != 0:
        pytest.skip("cuobjdump cannot read the library here")
    archs = set(l.split(".")[-2] for l in elf.stdout.splitlines() if ".cubin" in l)
    assert archs == {"sm_90a"}, archs
    fun, census = None, {}
    for line in sass.stdout.splitlines():
        if "Function :" in line:
            fun = line.split("Function :")[1].strip()
            census[fun] = {"UTMALDG": 0, "SYNCS": 0, "FFMA": 0, "PREEXIT": 0, "ACQBULK": 0}
        elif fun:
            for k in census[fun]:
                if k in line:
                    census[fun][k] += 1
    s1 = [c for f, c in census.items() if "k_xd_tma" in f]
    assert len(s1) >= 8                                         # D = 32 / 64, PS = 8 / 10, ring of 2 / 3
    for c in s1:
        assert c["UTMALDG"] >= 4 and c["SYNCS"] >= 6 and c["FFMA"] >= 400, c
    for name in ("k_dfir_reg", "k_poly_reg", "k_fir_reg", "k_firr_reg", "k_quad", "k_carry"):
        ks = [c for f, c in census.items() if name in f]
        assert ks, name
        for c in ks:
            assert c["PREEXIT"] >= 1 and c["ACQBULK"] >= 1, (name, c)

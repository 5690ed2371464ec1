"""IQ taps of the front end (b200_fe_bind_iq / b200_fe_unbind_iq): IQFrontEnd::bindIQStream (core/src/signal_path/
iq_frontend.h:34-35, iq_frontend.cpp:132-139), the stream the recorder and the IQ exporter bind to in baseband mode, in their
sample types.  Exact cases where the effective stream is the chunk itself or its conjugate; the oracle's decimator and DC
blocker chained on the CPU otherwise (as tests/test_gpu_preproc.py does); every integer type against a CPU statement of its
rule applied to the CF32 tap of the same chunk; identical outputs of VFOs and FFT with and without taps; every delivery path;
the C++ adapter's bindIQStream behind a decimating, DC-blocking front end.  The CPU part checks the exports, the constants
and the rules themselves."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from util import rel_rms, noise_iq, fm_carrier

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "build", "test_adapter")
INT_MAX = 2147483647
TOL = 1e-5


# ------------------------------------------------------------------------------------------------ CPU statements of the rules
def rule(x, t, scalar=0.0):
    """The element rule of sample type t on float32 values x (interleaved I, Q), as the C ABI documents it."""
    from sdrplusplus_b200 import lib as L
    x = np.asarray(x, np.float32)
    if t == L.IQ_U8:       # wav.cpp: (uint8_t)((x * 127.0f) + 128.0f), truncated; defined for |x| <= 1
        v = x * np.float32(127.0) + np.float32(128.0)
        return np.trunc(v).astype(np.uint8)
    lo, hi, dt = {L.IQ_I8: (-128.0, 127.0, np.int8), L.IQ_I16: (-32768.0, 32767.0, np.int16),
                  L.IQ_I32: (-2147483648.0, 2147483647.0, np.int32)}[t]
    r = np.clip(x * np.float32(scalar), np.float32(lo), np.float32(hi))        # volk_32f_s32f_convert_*: clamp, then rintf
    r = np.rint(r).astype(np.float64)
    if t == L.IQ_I32:
        r = np.where(r >= 2147483648.0, INT_MAX, r)       # (float)INT_MAX is 2^31: the device saturates where the CPU overflows
    return r.astype(dt)


def test_library_exports_iq_tap_entry_points():
    from sdrplusplus_b200 import lib
    L = lib.load()
    for name in ("b200_fe_bind_iq", "b200_fe_unbind_iq"):
        assert hasattr(L, name) and name in lib.SIGNATURES and name in lib.header_symbols()


def test_sample_type_constants_match_header():
    from sdrplusplus_b200 import lib
    with open(lib.HEADER_PATH) as f:
        text = f.read()
    got = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define B200_IQ_(\w+)\s+(\d+)", text)}
    assert got == {"CF32": lib.IQ_CF32, "U8": lib.IQ_U8, "I8": lib.IQ_I8, "I16": lib.IQ_I16, "I32": lib.IQ_I32}


def test_rules_restated_on_cpu(oracle):
    """The CPU statements above against the oracle's recorder conversion (wav.cpp:150-183 over volk_32f_s32f_convert_*),
    with saturating values and exact .5 ties; int8 against the same rintf-of-clamp statement on known values."""
    from sdrplusplus_b200 import lib as L
    rng = np.random.default_rng(3)
    ties16 = (np.arange(-40, 40) + 0.5) / 32767.0
    a = np.concatenate([rng.uniform(-1.6, 1.6, 20000), ties16, [1.0, -1.0, 0.0, 2.0, -2.0, 0.5, -0.5]]).astype(np.float32)
    assert np.array_equal(rule(a, L.IQ_I16, 32767.0), oracle.export_convert(a, 1))
    ok = np.abs(a.astype(np.float64) * 2147483648.0) < 2147483520.0       # where the CPU conversion does not overflow
    assert np.array_equal(rule(a, L.IQ_I32, 2147483647.0)[ok], oracle.export_convert(a, 2)[ok])
    assert np.all(rule(a, L.IQ_I32, 2147483647.0)[a >= 1.0] == INT_MAX)
    u = np.clip(a, -1.0, 1.0)
    assert np.array_equal(rule(u, L.IQ_U8), oracle.export_convert(u, 0))
    v = np.array([0.5, 1.5, 2.5, -0.5, -1.5, 126.6, 127.5, 300.0, -128.5, -300.0], np.float32) / np.float32(128.0)
    assert list(rule(v, L.IQ_I8, 128.0)) == [0, 2, 2, 0, -2, 127, 127, 127, -128, -128]


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def sb():
    import sdrplusplus_b200 as m
    from sdrplusplus_b200 import lib
    L = lib.load()
    assert L.b200_device_count() > 0
    assert L.b200_init(0) == 0
    return m


def _feed(fe, x, sizes, fmt=0):
    """process() over the chunk schedule `sizes` (cycled); returns (per-chunk outputs, concatenated outputs)."""
    from sdrplusplus_b200.frontend import _NP_FMT
    per = _NP_FMT[fmt][1]
    flat = x.reshape(-1)
    n = flat.size // per
    parts, i, k = [], 0, 0
    while i < n:
        c = min(sizes[k % len(sizes)], n - i)
        outs, _ = fe.process(flat[i * per:(i + c) * per], fmt)
        parts.append(outs)
        i += c
        k += 1
    cat = {tid: np.concatenate([p[tid] for p in parts]) for tid in parts[0]}
    return parts, cat


def _same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


gpu = pytest.mark.gpu


@gpu
def test_cf32_tap_is_the_input(sb):
    """Nothing pre-processes: the CF32 tap is the chunk, bit for bit, at chunk sizes 1, 7001, 12000 and max_chunk."""
    L = sb.lib
    mc = 40000
    x = noise_iq(130000, 61, 0.7).copy()
    x.view(np.float32)[::97] = np.float32(-0.0)          # signed zeros come back as they went in
    fe = sb.FrontEnd(2.4e6, mc)
    tid = fe.bind_iq(L.IQ_CF32)
    assert fe.vfo_max_out(tid, 1234) == 1234 and L.load().b200_fe_vfo_count(fe._h) == 1
    parts, cat = _feed(fe, x, [1, 7001, 12000, mc])
    assert [p[tid].size for p in parts[:4]] == [1, 7001, 12000, mc]
    assert _same_bits(cat[tid], x)
    fe.close()


@gpu
@pytest.mark.parametrize("fmt", [1, 2])
def test_integer_ingest_tap_is_scaled_input(sb, fmt):
    """cs16 / cs8 ingest: the tap is (float)x * scale, bit for bit, with the default scale and with b200_fe_set_ingest_scale
    changing between chunks; an (I16, 32768) tap of default-scale cs16 returns the int16 input itself."""
    L = sb.lib
    dt, full = (np.int16, 32768.0) if fmt == 1 else (np.int8, 128.0)
    rng = np.random.default_rng(62 + fmt)
    info = np.iinfo(dt)
    n, chunk = 60000, 12000
    x = rng.integers(info.min, info.max + 1, 2 * n).astype(dt)
    x[:4] = [info.min, info.max, 0, -1]
    fe = sb.FrontEnd(2.4e6, chunk)
    tc = fe.bind_iq(L.IQ_CF32)
    ti = fe.bind_iq(L.IQ_I16, 32768.0) if fmt == 1 else None
    scales = [0.0, 0.37 / full, 3.0 / full, -1.0, 1.0 / 4096.0]        # <= 0: the default 1 / full
    got, want = [], []
    for k, s in enumerate(scales):
        fe.set_ingest_scale(fmt, s)
        seg = x[2 * k * chunk: 2 * (k + 1) * chunk]
        outs, _ = fe.process(seg, fmt)
        sc = np.float32(1.0 / full) if s <= 0 else np.float32(s)
        want.append((seg.astype(np.float32) * sc).view(np.complex64))
        got.append(outs[tc])
        if ti is not None and s <= 0:
            assert _same_bits(outs[ti].reshape(-1), seg)
    assert _same_bits(np.concatenate(got), np.concatenate(want))
    fe.close()


@gpu
def test_conjugate_only(sb):
    L = sb.lib
    x = noise_iq(50000, 63, 0.5).copy()
    fe = sb.FrontEnd(2.4e6, 12000)
    fe.set_invert_iq(True)
    tid = fe.bind_iq(L.IQ_CF32)
    _, cat = _feed(fe, x, [12000, 7001, 1])
    assert np.array_equal(cat[tid], np.conj(x))
    fe.close()


@gpu
@pytest.mark.parametrize("ratio", [4, 64])
def test_decimation_against_oracle(sb, oracle, report, ratio):
    """Decimation only: the tap reads the decimator's output; per-chunk counts are the oracle's, rel. RMS <= 1e-5."""
    L = sb.lib
    fs, n = 9.6e6, 960000
    x = noise_iq(n, 64, 0.02).copy() + fm_carrier(n, fs, 300e3 if ratio == 4 else 20e3)
    sizes = [48000, 7001, 12288, 1, 48000]
    fe = sb.FrontEnd(fs, 48000)
    fe.set_decimation(ratio)
    tid = fe.bind_iq(L.IQ_CF32)
    parts, cat = _feed(fe, x, sizes)
    dec = oracle.decim(ratio)
    ref, i, k = [], 0, 0
    while i < n:
        c = min(sizes[k % len(sizes)], n - i)
        ref.append(dec.process(x[i:i + c].view(np.float32)).view(np.complex64))
        i += c
        k += 1
    assert [p[tid].size for p in parts] == [r.size for r in ref]
    e = rel_rms(cat[tid], np.concatenate(ref))
    report["iq_tap_decim%d" % ratio] = {"rel_rms": e}
    assert e <= TOL, e
    fe.close()


@gpu
@pytest.mark.parametrize("ratio,conj", [(1, False), (4, False), (4, True)])
def test_dc_blocking_against_oracle(sb, oracle, report, ratio, conj):
    """DC blocking alone, behind decimation, and with the conjugate: rel. RMS within the measured floor of the reference's
    fp32 blocker against float64 plus 1e-5; the residual DC is gone."""
    from scipy.signal import lfilter
    L = sb.lib
    fs, n, chunk = 2.4e6 * ratio, 480000 * ratio, 12000 * ratio
    x = noise_iq(n, 65, 0.02).copy() + fm_carrier(n, fs, 300e3)
    x += np.complex64(0.05 - 0.03j)
    fe = sb.FrontEnd(fs, chunk)
    if ratio > 1:
        fe.set_decimation(ratio)
    fe.set_dc_blocking(True)
    fe.set_invert_iq(conj)
    tid = fe.bind_iq(L.IQ_CF32)
    _, cat = _feed(fe, x, [chunk, 7001])
    fe_eff = fs / ratio
    dec = oracle.decim(ratio) if ratio > 1 else None
    dcb = oracle.dcblock_c(50.0 / fe_eff)
    ref, pre, i, k = [], [], 0, 0
    while i < n:
        c = min([chunk, 7001][k % 2], n - i)
        seg = x[i:i + c].view(np.float32)
        if dec is not None:
            seg = dec.process(seg)
        pre.append(seg.view(np.complex64).copy())
        y = dcb.process(seg).view(np.complex64)
        ref.append(np.conj(y) if conj else y)
        i += c
        k += 1
    ref, pre = np.concatenate(ref), np.concatenate(pre).astype(np.complex128)
    r = float(np.float32(50.0 / fe_eff))
    y64 = pre - lfilter([0.0, r], [1.0, -(1.0 - r)], pre)
    y64 = np.conj(y64) if conj else y64
    floor = rel_rms(ref, y64)
    e = rel_rms(cat[tid], ref)
    report["iq_tap_dc_decim%d_conj%d" % (ratio, conj)] = {"rel_rms": e, "reference_fp32_blocker_vs_exact": floor}
    assert cat[tid].shape == ref.shape
    assert e <= floor + TOL, (e, floor)
    assert abs(np.mean(cat[tid][cat[tid].size // 4:])) < 2e-3
    fe.close()


def _conversion_input(n, seed):
    """Values across and beyond full scale, with exact .5 ties of every integer type's scalar."""
    rng = np.random.default_rng(seed)
    v = rng.uniform(-1.3, 1.3, 2 * n).astype(np.float32)
    k = np.arange(-64, 64)
    ties = np.concatenate([(k + 0.5) / 128.0, (k + 0.5) / 32768.0, (k + 0.5) / 32767.0, (2 * k + 1) / 2.0 ** 32,
                           [1.0, -1.0, 127.5 / 128.0, -128.5 / 128.0, 32767.5 / 32768.0, -1.5, 1.5, 0.0]]).astype(np.float32)
    v[: ties.size] = ties
    v[ties.size: 2 * ties.size] = -ties
    return v.view(np.complex64)


PRESETS = [("rec_u8", 1, 0.0), ("rec_i16", 3, 32767.0), ("rec_i32", 4, 2147483647.0),
           ("exp_i8", 2, 128.0), ("exp_i16", 3, 32768.0), ("exp_i32", 4, 2147483647.0), ("i16_half", 3, 1000.5)]


@gpu
@pytest.mark.parametrize("pre", ["none", "decim4_dc"])
def test_every_type_and_preset_equals_its_rule(sb, oracle, pre):
    """Every integer type and preset against its CPU rule applied to the CF32 tap of the same chunk, bit for bit:
    recorder presets against the oracle's export_convert, exporter presets against numpy rint(clip(x * scalar)); I32 where
    the CPU conversion overflows against the documented INT_MAX saturation; U8 where its rule is defined (|x| <= 1)."""
    L = sb.lib
    n, chunk = 96000, 24000
    x = _conversion_input(n, 66)
    fe = sb.FrontEnd(9.6e6, chunk)
    if pre != "none":
        x = (x * np.float32(0.4)).astype(np.complex64) + np.complex64(0.3 + 0.1j)
        fe.set_decimation(4)
        fe.set_dc_blocking(True)
    tc = fe.bind_iq(L.IQ_CF32)
    ids = {name: fe.bind_iq(t, s) for name, t, s in PRESETS}
    _, cat = _feed(fe, x, [chunk, 7001])
    f = cat[tc].view(np.float32)
    for name, t, s in PRESETS:
        got = cat[ids[name]].reshape(-1)
        if name == "rec_u8":
            ok = np.abs(f) <= 1.0
            assert np.array_equal(got[ok], oracle.export_convert(f[ok], 0)), name
            assert np.array_equal(got[ok], rule(f[ok], t)), name
        elif name == "rec_i16":
            assert np.array_equal(got, oracle.export_convert(f, 1)), name
        elif t == L.IQ_I32:
            ok = np.abs(f.astype(np.float64) * 2147483648.0) < 2147483520.0
            if name == "rec_i32":
                assert np.array_equal(got[ok], oracle.export_convert(f, 2)[ok]), name
            assert np.array_equal(got, rule(f, t, s)), name
            assert np.all(got[f >= 1.0] == INT_MAX) and np.all(got[f <= -1.0] == -2147483648), name
        else:
            assert np.array_equal(got, rule(f, t, s)), name
    if pre == "none":
        assert np.any(cat[ids["exp_i16"]].reshape(-1) == 32767) and np.any(cat[ids["exp_i8"]].reshape(-1) == -128)
    fe.close()


def _band_fe(sb, taps, chunk):
    fe = sb.FrontEnd(16e6, chunk)
    fe.set_fft(65536, 20.0, 2)
    vids = [fe.add_vfo(sb.VfoConfig.wfm(o)) for o in (-7e6, -5e6, -3e6, -1e6, 1e6, 3e6, 5e6, 7e6)]
    tids = [fe.bind_iq(t, s) for t, s in taps]
    return fe, vids, tids


@gpu
def test_taps_change_no_other_output(sb):
    """8 WFM VFOs and a 64 Ki-point FFT: audio and lines are bit-identical with and without CF32, I16 and U8 taps bound;
    each tap equals a run with that tap alone; the taps add one launch per chunk and nothing else."""
    L = sb.lib
    n, chunk = 1200000, 100000
    x = noise_iq(n, 67, 0.02).copy()
    for o in (-5e6, 1e6, 7e6):
        x += fm_carrier(n, 16e6, o)
    taps = [(L.IQ_CF32, 0.0), (L.IQ_I16, 32768.0), (L.IQ_U8, 0.0)]
    fe0, v0, _ = _band_fe(sb, [], chunk)
    o0, l0 = fe0.process_chunks(x, chunk)
    fe1, v1, t1 = _band_fe(sb, taps, chunk)
    o1, l1 = fe1.process_chunks(x, chunk)
    assert v0 == v1
    assert _same_bits(l0, l1) and l0.shape[0] >= 2
    for v in v0:
        assert _same_bits(o0[v], o1[v])
    assert fe1.launch_count() == fe0.launch_count() + n // chunk
    for k, t in enumerate(taps):
        fe, _, tid = _band_fe(sb, [t], chunk)
        o, _ = fe.process_chunks(x, chunk)
        assert _same_bits(o[tid[0]], o1[t1[k]])
        fe.close()
    assert _same_bits(o1[t1[0]], x)
    fe0.close()
    fe1.close()


def _path_run(sb, x, chunk, mode, inflight=2, graph=-1, host_direct=-1):
    """One WFM VFO + CF32 and I16 taps behind decimation 2 and DC blocking, fed by submit / wait with `inflight` chunks in
    flight; outputs in numpy buffers ("numpy"), b200_host_alloc buffers ("pinned") or device buffers ("device")."""
    import torch
    L = sb.lib
    lib = L.load()
    fe = sb.FrontEnd(4.8e6, chunk)
    fe.set_decimation(2)
    fe.set_dc_blocking(True)
    fe.set_option("inflight", inflight)
    fe.set_option("graph", graph)
    fe.set_option("host_direct", host_direct)
    vid = fe.add_vfo(sb.VfoConfig.wfm(300e3))
    tc, ti = fe.bind_iq(L.IQ_CF32), fe.bind_iq(L.IQ_I16, 32768.0)
    caps = {vid: (fe.vfo_max_out(vid, chunk), 8), tc: (fe.vfo_max_out(tc, chunk), 8), ti: (fe.vfo_max_out(ti, chunk), 4)}
    slots, keep, pinned = [], [], []
    for _ in range(inflight):
        o = L.Outputs()
        bufs = {}
        for i, (cap, b) in caps.items():
            if mode == "numpy":
                a = np.empty(cap * b, np.uint8)
                ptr = a.ctypes.data
            elif mode == "pinned":
                ptr = lib.b200_host_alloc(cap * b)
                pinned.append(ptr)
                a = (C.c_uint8 * (cap * b)).from_address(ptr)
            else:
                a = torch.empty(cap * b, dtype=torch.uint8, device="cuda")
                ptr = a.data_ptr()
            bufs[i] = a
            o.vfo_out[i], o.vfo_cap[i] = ptr, cap
        o.out_mem = L.MEM_DEVICE if mode == "device" else L.MEM_HOST
        slots.append((o, bufs))
        keep.append(bufs)
    res = {i: [] for i in caps}
    pend = []

    def drain():
        o, bufs = pend.pop(0)
        fe.wait()
        for i, (cap, b) in caps.items():
            nb = o.vfo_count[i] * b
            a = bufs[i]
            raw = a[:nb].cpu().numpy() if mode == "device" else np.frombuffer(a, np.uint8, count=nb).copy()
            res[i].append(raw)

    xs = np.ascontiguousarray(x)
    for k, i0 in enumerate(range(0, x.size, chunk)):
        if len(pend) == inflight:
            drain()
        o, bufs = slots[k % inflight]
        seg = xs[i0:i0 + chunk]
        if mode == "device":
            seg_t = torch.from_numpy(seg.view(np.float32).copy()).cuda()
            keep.append(seg_t)
            torch.cuda.synchronize()
            fe.submit_ptr(seg_t.data_ptr(), seg.size, L.FMT_CF32, L.MEM_DEVICE, o)
        else:
            keep.append(seg)
            fe.submit_ptr(seg.ctypes.data, seg.size, L.FMT_CF32, L.MEM_HOST, o)
        pend.append((o, bufs))
    while pend:
        drain()
    fe.close()
    for p in pinned:
        lib.b200_host_free(p)
    return [np.concatenate(res[i]).tobytes() for i in (vid, tc, ti)]


@gpu
def test_delivery_paths_agree(sb):
    """The same tap and VFO bytes from numpy, b200_host_alloc and device buffers, inflight 2 / 3 / 4, graph 0 / 1 and
    host_direct 0 / 1, and from process()."""
    x = noise_iq(240000, 68, 0.02).copy() + fm_carrier(240000, 4.8e6, 300e3) + np.complex64(0.02)
    chunk = 24000
    fe = sb.FrontEnd(4.8e6, chunk)
    fe.set_decimation(2)
    fe.set_dc_blocking(True)
    vid = fe.add_vfo(sb.VfoConfig.wfm(300e3))
    tc, ti = fe.bind_iq(sb.lib.IQ_CF32), fe.bind_iq(sb.lib.IQ_I16, 32768.0)
    o, _ = fe.process_chunks(x, chunk)
    fe.close()
    want = [o[vid].tobytes(), o[tc].tobytes(), o[ti].tobytes()]
    runs = {"numpy": dict(mode="numpy"), "pinned_hd1": dict(mode="pinned", host_direct=1), "pinned_hd0": dict(mode="pinned", host_direct=0),
            "device": dict(mode="device"), "inflight3": dict(mode="pinned", inflight=3), "inflight4": dict(mode="numpy", inflight=4),
            "graph0": dict(mode="pinned", graph=0), "graph1": dict(mode="device", graph=1)}
    for name, kw in runs.items():
        got = _path_run(sb, x, chunk, **kw)
        assert got == want, name


@gpu
def test_edge_cases_and_errors(sb):
    """A front end with only a tap; a 0-sample chunk; unbind then rebind; reset against a fresh front end; the EINVAL / ECAP /
    ESTATE cases, each leaving the front end usable."""
    L = sb.lib
    lib = L.load()
    x = noise_iq(48000, 69, 0.3).copy() + np.complex64(0.1)

    def fresh():
        fe = sb.FrontEnd(9.6e6, 12000)
        fe.set_decimation(4)
        fe.set_dc_blocking(True)
        return fe

    fe = fresh()
    tid = fe.bind_iq(L.IQ_I16, 32768.0)
    ref = fresh()
    rid = ref.bind_iq(L.IQ_I16, 32768.0)
    _, a = _feed(fe, x, [12000])
    outs, _ = fe.process(np.empty(0, np.complex64))
    assert outs[tid].shape == (0, 2)
    # reset: the decimator and the blocker the tap reads from start again
    fe.reset()
    _, b = _feed(fe, x, [12000])
    _, c = _feed(ref, x, [12000])
    assert _same_bits(a[tid], c[rid]) and _same_bits(b[tid], c[rid])
    # errors, each followed by a chunk that must still come out right
    with pytest.raises(L.B200Error) as e:
        fe.set_decimation(2)
    assert e.value.code == -7
    vid = fe.add_vfo(sb.VfoConfig.raw(0.0, 300e3, 300e3))
    for call in (lambda: fe.set_vfo_offset(tid, 1e3), lambda: fe.set_vfo_bandwidth(tid, 1e5),
                 lambda: fe.set_vfo_config(tid, sb.VfoConfig.raw(0.0, 300e3, 300e3)), lambda: fe.remove_vfo(tid),
                 lambda: fe.unbind_iq(vid), lambda: fe.bind_iq(7), lambda: fe.bind_iq(L.IQ_I16, float("nan"))):
        with pytest.raises(L.B200Error) as e:
            call()
        assert e.value.code == -1
    o = L.Outputs()
    small = np.empty((2999, 2), np.int16)
    vb = np.empty(2 * fe.vfo_max_out(vid, 12000), np.float32)
    o.vfo_out[tid], o.vfo_cap[tid] = small.ctypes.data, 2999
    o.vfo_out[vid], o.vfo_cap[vid] = vb.ctypes.data, fe.vfo_max_out(vid, 12000)
    xs = np.ascontiguousarray(x[:12000])
    assert lib.b200_fe_process(fe._h, xs.ctypes.data, 12000, L.FMT_CF32, L.MEM_HOST, C.byref(o)) == -5
    fe.remove_vfo(vid)
    fe.reset()
    ref.reset()
    _, b = _feed(fe, x, [12000])
    _, c = _feed(ref, x, [12000])
    assert _same_bits(b[tid], c[rid])
    # unbind then rebind: the id comes back, the output is the same
    fe.unbind_iq(tid)
    assert lib.b200_fe_vfo_count(fe._h) == 0
    outs, _ = fe.process(x[:12000])
    assert tid not in outs
    tid2 = fe.bind_iq(L.IQ_CF32)
    assert tid2 == tid
    fe.reset()
    ref2 = fresh()
    r2 = ref2.bind_iq(L.IQ_CF32)
    _, b = _feed(fe, x, [12000])
    _, c = _feed(ref2, x, [12000])
    assert _same_bits(b[tid2], c[r2])
    for f in (fe, ref, ref2):
        f.close()


@gpu
def test_adapter_bind_iq_stream(oracle, report, tmp_path):
    """dsp::b200::FrontEnd::bindIQStream: a sink::Handler<complex_t> worker behind a front end that decimates by 4 and
    blocks DC receives the oracle's decimator -> DC blocker stream, chunk for chunk."""
    from scipy.signal import lfilter
    if not os.path.exists(EXE):
        pytest.skip("build/test_adapter missing: run python __graft_entry__.py")
    fs, n, chunk = 2.4e6, 480000, 12000
    x = noise_iq(n, 70, 0.02).copy() + fm_carrier(n, fs, 300e3) + np.complex64(0.04 - 0.02j)
    src, dst = tmp_path / "iq.f32", tmp_path / "tap.f32"
    x.tofile(src)
    r = subprocess.run([EXE, str(src), str(dst), "iqtap"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
    got = np.fromfile(dst, np.complex64)
    dec, dcb = oracle.decim(4), oracle.dcblock_c(50.0 / (fs / 4))
    pre = [dec.process(x[i:i + chunk].view(np.float32)) for i in range(0, n, chunk)]
    ref = np.concatenate([dcb.process(p).view(np.complex64) for p in pre])
    p64 = np.concatenate(pre).view(np.complex64).astype(np.complex128)
    rr = float(np.float32(50.0 / (fs / 4)))
    floor = rel_rms(ref, p64 - lfilter([0.0, rr], [1.0, -(1.0 - rr)], p64))
    assert [int(v) for v in r.stdout.split()[:2]] == [ref.size, n // chunk]
    e = rel_rms(got, ref)
    report["iq_tap_adapter"] = {"rel_rms": e, "reference_fp32_blocker_vs_exact": floor}
    assert e <= floor + TOL, (e, floor)
    assert abs(np.mean(got[got.size // 4:])) < 2e-3

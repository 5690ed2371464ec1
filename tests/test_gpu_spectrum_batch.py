"""The spectrum branch's two ways of handling a frame that begins in one chunk and ends in a later one give the same lines, bit
for bit: "fft_v" 1 stages the frame's earlier part with copies in the input's own format and transforms the frame in its
chunk's batch, reading twiddles from shared memory; "fft_v" 0 converts the earlier part to cf32 and transforms the frame on its
own, twiddles from global memory.  Covers the bench geometry, frames that span three and more chunks, the C1 geometry, every
input format, the input decimator, an empty chunk, and format / scale changes while a frame is staged."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sb():
    import sdrplusplus_b200 as m
    from sdrplusplus_b200 import lib
    L = lib.load()
    assert L.b200_device_count() > 0
    assert L.b200_init(0) == 0
    return m


def _iq(n, seed, fmt):
    """n samples: complex64, or (n, 2) int16 / int8"""
    from sdrplusplus_b200 import lib
    rng = np.random.default_rng(seed)
    if fmt == lib.FMT_CF32:
        return (rng.standard_normal(2 * n, dtype=np.float32) * 0.3).view(np.complex64)
    if fmt == lib.FMT_CS16:
        return rng.integers(-20000, 20000, (n, 2), dtype=np.int16)
    return rng.integers(-100, 100, (n, 2), dtype=np.int8)


def _lines(sb, chunks, fs, size, rate, v, decim=1, scales=None, cta=None):
    """chunks: [(samples, fmt)]; returns the stacked lines and the launches of every chunk (size 0: no FFT)"""
    from sdrplusplus_b200 import lib
    fe = sb.FrontEnd(fs, max(max(len(c) for c, _ in chunks), 1))
    fe.set_option("fft_v", v)
    if cta:
        fe.set_option("fft_cta", cta)
    if decim > 1:
        fe.set_decimation(decim)
    if size:
        fe.set_fft(size, rate, 2)
    lines, launches = [], []
    for k, (x, fmt) in enumerate(chunks):
        if scales is not None and fmt != lib.FMT_CF32:
            fe.set_ingest_scale(fmt, scales[k])
        l0 = fe.launch_count()
        _, ln = fe.process(x, fmt)
        launches.append(fe.launch_count() - l0)
        if ln.size:
            lines.append(ln)
    fe.close()
    return (np.concatenate(lines) if lines else np.empty((0, size), np.float32)), launches


def _same(a, b):
    assert a.shape == b.shape and a.shape[0] > 0, (a.shape, b.shape)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _split(x, chunk, fmt):
    return [(x[i:i + chunk], fmt) for i in range(0, len(x), chunk)]


def test_bench_geometry_16mi_chunks(sb):
    """100 MS/s, 16 Mi-sample chunks, 1 Mi points at 20 fps: frames straddle chunk edges; the spectrum branch is one launch
    pair a chunk with fft_v 1"""
    from sdrplusplus_b200 import lib
    chunk = 1 << 24
    base = _iq(1 << 22, 1, lib.FMT_CF32)
    x = np.concatenate([np.roll(base, 1000 * k) for k in range(4 * 8)])          # 8 chunks of distinct samples
    chunks = _split(x, chunk, lib.FMT_CF32)
    a, la = _lines(sb, chunks, 100e6, 1 << 20, 20.0, 1)
    b, lb = _lines(sb, chunks, 100e6, 1 << 20, 20.0, 0)
    _, l0 = _lines(sb, chunks, 100e6, 0, 20.0, 1)                                   # what a chunk launches without the FFT
    _same(a, b)
    assert a.shape[0] == (8 * chunk - (1 << 20)) // 5_000_000 + 1
    fa, fb = [x - y for x, y in zip(la, l0)], [x - y for x, y in zip(lb, l0)]
    assert max(fa) <= 2, fa
    assert max(fb) > 2, fb                # the straddling frame costs fft_v 0 a convert launch and a launch pair of its own


@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_frames_spanning_three_chunks_every_format(sb, fmt):
    """500 k-sample chunks at 100 MS/s: each 1 Mi-point frame spans three chunks, its staged part grows chunk by chunk"""
    x = _iq(12_000_000, 2 + fmt, fmt)
    chunks = _split(x, 500_000, fmt)
    a, la = _lines(sb, chunks, 100e6, 1 << 20, 20.0, 1)
    b, _ = _lines(sb, chunks, 100e6, 1 << 20, 20.0, 0)
    _, l0 = _lines(sb, chunks, 100e6, 0, 20.0, 1)
    _same(a, b)
    assert a.shape[0] == 3 and max(x - y for x, y in zip(la, l0)) <= 2


@pytest.mark.parametrize("cta", [4, 8])
def test_c1_geometry(sb, cta):
    """2.4 MS/s, 65,536 points at 20 fps, 12,000-sample chunks: a frame spans six chunks"""
    from sdrplusplus_b200 import lib
    x = _iq(1_200_000, 5, lib.FMT_CS16)
    chunks = _split(x, 12_000, lib.FMT_CS16)
    a, _ = _lines(sb, chunks, 2.4e6, 65536, 20.0, 1, cta=cta)
    b, _ = _lines(sb, chunks, 2.4e6, 65536, 20.0, 0, cta=cta)
    _same(a, b)
    assert a.shape[0] == 10


def test_input_decimation(sb):
    from sdrplusplus_b200 import lib
    x = _iq(4_000_000, 6, lib.FMT_CS8)
    chunks = _split(x, 300_000, lib.FMT_CS8)
    a, _ = _lines(sb, chunks, 10e6, 65536, 20.0, 1, decim=4)
    b, _ = _lines(sb, chunks, 10e6, 65536, 20.0, 0, decim=4)
    _same(a, b)


def test_empty_chunk_while_a_frame_is_staged(sb):
    from sdrplusplus_b200 import lib
    x = _iq(1_000_000, 7, lib.FMT_CF32)
    chunks = _split(x, 100_000, lib.FMT_CF32)
    chunks = chunks[:3] + [(np.empty(0, np.complex64), lib.FMT_CF32)] + chunks[3:]
    a, la = _lines(sb, chunks, 2.4e6, 65536, 20.0, 1)
    b, _ = _lines(sb, chunks, 2.4e6, 65536, 20.0, 0)
    _same(a, b)
    assert a.shape[0] == 8


def test_format_and_scale_change_while_a_frame_is_staged(sb):
    """the staged part keeps the format and scale it arrived with: a chunk in another format or at another ingest scale
    carries the frame on in cf32"""
    from sdrplusplus_b200 import lib
    fmts = [lib.FMT_CS16, lib.FMT_CS16, lib.FMT_CF32, lib.FMT_CS8, lib.FMT_CS8, lib.FMT_CS16, lib.FMT_CS16, lib.FMT_CS16] * 4
    chunks = [(_iq(40_000, 10 + k, f), f) for k, f in enumerate(fmts)]
    scales = [1.0 / 32768 if k % 7 else 2.0 / 32768 for k in range(len(chunks))]
    scales = [s if f != lib.FMT_CS8 else 1.0 / 128 for s, (_, f) in zip(scales, chunks)]
    a, _ = _lines(sb, chunks, 2.4e6, 65536, 20.0, 1, scales=scales)
    b, _ = _lines(sb, chunks, 2.4e6, 65536, 20.0, 0, scales=scales)
    _same(a, b)
    assert a.shape[0] == 11

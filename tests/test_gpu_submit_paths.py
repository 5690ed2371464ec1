"""What b200_fe_submit does around the scheduler, pinned as literals: for a fixed set of front-end scenarios driven through
submit / wait, the launches of every chunk, every output's sample count and the number of FFT lines per chunk, and a
sha256 of every output stream (VFO audio, IQ tap samples, FFT lines, RDS records).  The scenarios cover the spectrum
framer (frames across chunk edges, a skip gap, the input format changing between chunks, fft_v 0 and 1), the input
decimator, DC blocker and IQ inversion with IQ taps of every sample type, outputs in numpy, b200_host_alloc and device
buffers with 2 to 4 chunks in flight, RDS records, overlap 0 and a one-rank shard."""
import ctypes as C
import hashlib

import numpy as np
import pytest

from util import noise_iq, fm_carrier, am_carrier

pytestmark = pytest.mark.gpu
FS = 2.4e6
TAP_BYTES = {0: 8, 1: 2, 2: 2, 3: 4, 4: 8}          # B200_IQ_CF32, U8, I8, I16, I32: bytes per complex sample


@pytest.fixture(scope="module")
def sb():
    import torch  # noqa: F401  (loads the process's libnccl.so.2 for the shard scenario)
    import sdrplusplus_b200 as m
    from sdrplusplus_b200 import lib
    L = lib.load()
    assert L.b200_device_count() > 0
    assert L.b200_init(0) == 0
    return m


def _signal(n, fs=FS):
    x = noise_iq(n, 31, 0.004).copy()
    for k, o in enumerate((-600e3, 300e3, 700e3)):
        x += fm_carrier(n, fs, o, tones=((1000.0 * (k + 1), 0.5), (5000.0, 0.3)), amp=0.04)
    x += fm_carrier(n, fs, -200e3, dev=5000.0, tones=((1000.0, 0.7),), amp=0.04)
    x += am_carrier(n, fs, 450e3, amp=0.04)
    return x


def _as_fmt(x, fmt):
    """a complex64 segment as the raw interleaved array of input format fmt"""
    from sdrplusplus_b200 import lib as L
    if fmt == L.FMT_CF32:
        return np.ascontiguousarray(x)
    f = np.ascontiguousarray(x).view(np.float32)
    if fmt == L.FMT_CS16:
        return np.clip(np.rint(f * 32767.0), -32768, 32767).astype(np.int16)
    return np.clip(np.rint(f * 127.0), -128, 127).astype(np.int8)


class _Outputs:
    """`n` output sets for the ids of a front end: numpy, b200_host_alloc ("pinned") or device buffers"""

    def __init__(self, fe, chunk, n, mode, ids):
        import torch
        from sdrplusplus_b200 import lib as L
        self.lib = L.load()
        self.mode, self.pinned, self.sets = mode, [], []
        self.ids = ids                              # id -> bytes per output element
        for _ in range(n):
            o = L.Outputs()
            bufs = {}
            for i, b in ids.items():
                cap = fe.vfo_max_out(i, chunk)
                bufs[i] = self._buf(max(cap, 1) * b, torch)
                o.vfo_out[i], o.vfo_cap[i] = self._ptr(bufs[i]), cap
            if fe.fft_size:
                nl = max(1, fe.fft_max_lines(chunk))
                bufs["fft"] = self._buf(nl * fe.fft_size * 4, torch)
                o.fft_out, o.fft_cap_lines = self._ptr(bufs["fft"]), nl
            o.out_mem = L.MEM_DEVICE if mode == "device" else L.MEM_HOST
            self.sets.append((o, bufs))

    def _buf(self, nb, torch):
        if self.mode == "numpy":
            return np.empty(nb, np.uint8)
        if self.mode == "pinned":
            p = self.lib.b200_host_alloc(nb)
            self.pinned.append(p)
            return (C.c_uint8 * nb).from_address(p)
        return torch.empty(nb, dtype=torch.uint8, device="cuda")

    def _ptr(self, a):
        if self.mode == "numpy":
            return a.ctypes.data
        if self.mode == "pinned":
            return C.addressof(a)
        return a.data_ptr()

    def read(self, k, fft_size):
        """(counts, fft lines, {name: bytes}) of output set k after its wait"""
        o, bufs = self.sets[k]
        counts = [o.vfo_count[i] for i in sorted(self.ids)]
        got = {i: self._bytes(bufs[i], o.vfo_count[i] * b) for i, b in self.ids.items()}
        if "fft" in bufs:
            got["fft"] = self._bytes(bufs["fft"], o.fft_lines * fft_size * 4)
        return counts, o.fft_lines, got

    def _bytes(self, a, nb):
        if self.mode == "device":
            return a[:nb].cpu().numpy().tobytes()
        return np.frombuffer(a, np.uint8, count=nb).tobytes()

    def free(self):
        for p in self.pinned:
            self.lib.b200_host_free(p)
        self.pinned = []


def _drive(fe, segs, ids, mode="numpy", inflight=2, submit=None, wait=None, between=None):
    """Feed (array, count, fmt) segments through submit / wait with `inflight` chunks in flight.  Returns the launches of
    every submit, the per-chunk output counts with the FFT line count last, and a sha256 per output stream."""
    import torch
    from sdrplusplus_b200 import lib as L
    chunk = max(n for _, n, _ in segs)
    outs = _Outputs(fe, chunk, inflight, mode, ids)
    submit = submit or fe.submit_ptr
    wait = wait or fe.wait
    sha = {str(i): hashlib.sha256() for i in ids}
    if fe.fft_size:
        sha["fft"] = hashlib.sha256()
    deltas, counts, pend, keep = [], [], [], []

    def drain():
        k = pend.pop(0)
        wait()
        c, nl, got = outs.read(k, fe.fft_size)
        counts.append(c + [nl])
        for name, b in got.items():
            sha[str(name)].update(b)

    for k, (a, n, fmt) in enumerate(segs):
        if len(pend) == inflight:
            drain()
        if between:
            between(fe, k)
        if mode == "device":
            t = torch.from_numpy(a.view(np.uint8).copy()).cuda()
            torch.cuda.synchronize()
            keep.append(t)
            ptr, mem = t.data_ptr(), L.MEM_DEVICE
        else:
            keep.append(a)
            ptr, mem = a.ctypes.data, L.MEM_HOST
        l0 = fe.launch_count()
        submit(ptr, n, fmt, mem, outs.sets[k % inflight][0])
        deltas.append(fe.launch_count() - l0)
        pend.append(k % inflight)
    while pend:
        drain()
    outs.free()
    return deltas, counts, {k: h.hexdigest() for k, h in sha.items()}


def _segs(x, sizes, fmts):
    out, i = [], 0
    for k, n in enumerate(sizes):
        fmt = fmts[k % len(fmts)]
        out.append((_as_fmt(x[i:i + n], fmt), n, fmt))
        i += n
    return out


def _vfo_ids(fe, cfgs):
    return {fe.add_vfo(c): 8 for c in cfgs}


def _scenario(sb, name):
    from sdrplusplus_b200 import lib as L
    cf, s16, s8 = L.FMT_CF32, L.FMT_CS16, L.FMT_CS8
    if name.startswith("spectrum_v"):
        # 8192-point frames at 200 lines/s: a 12000-sample interval, so a 3808-sample skip gap; chunks shorter and longer than
        # the interval, so frames begin in one chunk and complete in a later one, and a chunk can complete three
        sizes = [5000, 3000, 20000, 7001, 2000, 30000, 4096, 11000, 9000, 1500, 25000, 6000, 12000, 3333]
        fmts = [cf, cf, s16, s16, s8, cf, s8, s16, cf, s8, s8, s16, cf, cf]
        fe = sb.FrontEnd(FS, max(sizes))
        fe.set_option("fft_v", int(name[-1]))
        fe.set_fft(8192, 200.0, L.WIN_NUTTALL)
        ids = _vfo_ids(fe, [sb.VfoConfig.wfm(300e3), sb.VfoConfig.nfm(-200e3)])

        def scale(fe, k):             # cs16 from chunk 8 on at another ingest scale than the cs16 frame parts staged before
            if k == 8:
                fe.set_ingest_scale(s16, 1.0 / 16384.0)
        return _drive(fe, _segs(_signal(sum(sizes)), sizes, fmts), ids, between=scale)
    if name.startswith("preproc_d4"):
        fe = sb.FrontEnd(4 * FS, 48000)
        fe.set_decimation(4)
        if name.endswith("_dc_inv"):
            fe.set_dc_blocking(True)
            fe.set_invert_iq(True)
        fe.set_fft(4096, 100.0, L.WIN_NUTTALL)
        ids = _vfo_ids(fe, [sb.VfoConfig.wfm(300e3), sb.VfoConfig.am(450e3)])
        for t, sc in ((L.IQ_CF32, 0.0), (L.IQ_U8, 0.0), (L.IQ_I8, 100.0), (L.IQ_I16, 20000.0), (L.IQ_I32, 1e6)):
            ids[fe.bind_iq(t, sc)] = TAP_BYTES[t]
        x = _signal(12 * 48000, 4 * FS) + np.complex64(0.01 - 0.02j)
        return _drive(fe, _segs(x, [48000] * 12, [cf, s16]), ids)
    if name.startswith("out_"):                  # out_<mode>_<chunk>_if<inflight>
        mode, chunk, infl = name.split("_")[1:]
        chunk, infl = int(chunk), int(infl[2:])
        fe = sb.FrontEnd(FS, chunk)
        fe.set_option("inflight", infl)
        fe.set_fft(4096, 400.0, L.WIN_NUTTALL)
        ids = _vfo_ids(fe, [sb.VfoConfig.wfm(300e3), sb.VfoConfig.wfm_stereo(-600e3), sb.VfoConfig.nfm(-200e3),
                            sb.VfoConfig.am(450e3), sb.VfoConfig.raw(700e3, 250e3, 150e3)])
        for t, sc in ((L.IQ_CF32, 0.0), (L.IQ_U8, 0.0), (L.IQ_I16, 20000.0)):
            ids[fe.bind_iq(t, sc)] = TAP_BYTES[t]
        n = 16 * chunk
        return _drive(fe, _segs(_signal(n), [chunk] * 16, [cf]), ids, mode=mode, inflight=infl)
    if name.startswith("rds_"):
        fe = sb.FrontEnd(FS, 12000)
        v = fe.add_vfo(sb.VfoConfig.wfm(300e3))
        ids = {v: 8, fe.add_vfo(sb.VfoConfig.wfm_rds_bits(-600e3)): 8, fe.bind_rds(v): 8}
        return _drive(fe, _segs(_signal(16 * 12000), [12000] * 16, [cf]), ids, mode=name[4:])
    if name == "overlap0":
        fe = sb.FrontEnd(FS, 12000)
        fe.set_option("overlap", 0)
        fe.set_fft(8192, 200.0, L.WIN_NUTTALL)
        ids = _vfo_ids(fe, [sb.VfoConfig.wfm(300e3), sb.VfoConfig.nfm(-200e3), sb.VfoConfig.am(450e3)])
        ids[fe.bind_iq(L.IQ_I16, 20000.0)] = 4
        return _drive(fe, _segs(_signal(16 * 12000), [12000] * 16, [cf, s16]), ids)
    if name == "shard_world1":
        from sdrplusplus_b200.sharding import ShardedFrontEnd, make_unique_id
        fe = sb.FrontEnd(FS, 12000)
        fe.set_fft(8192, 200.0, L.WIN_NUTTALL)
        ids = _vfo_ids(fe, [sb.VfoConfig.wfm(300e3), sb.VfoConfig.nfm(-200e3)])
        sh = ShardedFrontEnd(fe, 0, 1, make_unique_id())
        try:
            return _drive(fe, _segs(_signal(12 * 12000), [12000] * 12, [cf, s16]), ids, submit=sh.submit_ptr, wait=sh.wait)
        finally:
            sh.close()
    raise KeyError(name)


# per scenario: the launches of every submit, the output counts of every chunk (ids in order, FFT lines last) and a sha256
# per output stream (measured on an H100)
EXPECTED = {
    "out_device_12000_if4": (
        [26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26],
        [[1250, 1250, 250, 76, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250,
         250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 74, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 76, 1250,
         12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250, 12000, 12000,
         12000, 2], [1250, 1250, 250, 74, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 76, 1250, 12000, 12000, 12000, 2],
         [1250, 1250, 250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250,
         250, 74, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 76, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250,
         12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 74, 1250, 12000, 12000,
         12000, 2]],
        {
            "0": "487ad7b11bebb43a8cf570d86efbd4781d6ffc4825188f2a5636e0f6441a4017",
            "1": "e6ee652db0e9c3ff9c29860853d3829fe3c3f33df98d0b4629d5252f151b7494",
            "2": "f575ef679488befa2f8e00cac4d11ec7c75c5a1669644ba338c45b86c4af9491",
            "3": "c88def91cb422e9e47d72fd948c34dcf3cdee75918d70636edba1b99d6e0cfa2",
            "4": "8da601ce4b38b5ba424a6acc5888e3e12423b334f458f542e82806f6f66eedf5",
            "5": "0d9e4e11c3c2c311574715eff6cabb9c65e439b64374b8a13444e9f07947d586",
            "6": "b808ff52393f55ba69bd890234e33a6a8ebe45632b0f5b5f28f39650b1981f10",
            "7": "3a83aa6396c18055e60bf127d39501711b5b1db6ede62bde25069a859df8efab",
            "fft": "c687d4cf03a900149f86ce8dfc778ce3e2aa51702025938a91e4f3ea43486198",
        }),
    "out_numpy_12000_if2": (
        [26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26],
        [[1250, 1250, 250, 76, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250,
         250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 74, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 76, 1250,
         12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250, 12000, 12000,
         12000, 2], [1250, 1250, 250, 74, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 76, 1250, 12000, 12000, 12000, 2],
         [1250, 1250, 250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250,
         250, 74, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 76, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250,
         12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 74, 1250, 12000, 12000,
         12000, 2]],
        {
            "0": "487ad7b11bebb43a8cf570d86efbd4781d6ffc4825188f2a5636e0f6441a4017",
            "1": "e6ee652db0e9c3ff9c29860853d3829fe3c3f33df98d0b4629d5252f151b7494",
            "2": "f575ef679488befa2f8e00cac4d11ec7c75c5a1669644ba338c45b86c4af9491",
            "3": "c88def91cb422e9e47d72fd948c34dcf3cdee75918d70636edba1b99d6e0cfa2",
            "4": "8da601ce4b38b5ba424a6acc5888e3e12423b334f458f542e82806f6f66eedf5",
            "5": "0d9e4e11c3c2c311574715eff6cabb9c65e439b64374b8a13444e9f07947d586",
            "6": "b808ff52393f55ba69bd890234e33a6a8ebe45632b0f5b5f28f39650b1981f10",
            "7": "3a83aa6396c18055e60bf127d39501711b5b1db6ede62bde25069a859df8efab",
            "fft": "c687d4cf03a900149f86ce8dfc778ce3e2aa51702025938a91e4f3ea43486198",
        }),
    "out_pinned_12000_if2": (
        [26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26, 26],
        [[1250, 1250, 250, 76, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250,
         250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 74, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 76, 1250,
         12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250, 12000, 12000,
         12000, 2], [1250, 1250, 250, 74, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 76, 1250, 12000, 12000, 12000, 2],
         [1250, 1250, 250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250,
         250, 74, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 76, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250,
         12000, 12000, 12000, 2], [1250, 1250, 250, 75, 1250, 12000, 12000, 12000, 2], [1250, 1250, 250, 74, 1250, 12000, 12000,
         12000, 2]],
        {
            "0": "487ad7b11bebb43a8cf570d86efbd4781d6ffc4825188f2a5636e0f6441a4017",
            "1": "e6ee652db0e9c3ff9c29860853d3829fe3c3f33df98d0b4629d5252f151b7494",
            "2": "f575ef679488befa2f8e00cac4d11ec7c75c5a1669644ba338c45b86c4af9491",
            "3": "c88def91cb422e9e47d72fd948c34dcf3cdee75918d70636edba1b99d6e0cfa2",
            "4": "8da601ce4b38b5ba424a6acc5888e3e12423b334f458f542e82806f6f66eedf5",
            "5": "0d9e4e11c3c2c311574715eff6cabb9c65e439b64374b8a13444e9f07947d586",
            "6": "b808ff52393f55ba69bd890234e33a6a8ebe45632b0f5b5f28f39650b1981f10",
            "7": "3a83aa6396c18055e60bf127d39501711b5b1db6ede62bde25069a859df8efab",
            "fft": "c687d4cf03a900149f86ce8dfc778ce3e2aa51702025938a91e4f3ea43486198",
        }),
    "out_pinned_4096_if3": (
        [26, 25, 26, 26, 25, 26, 26, 25, 26, 26, 25, 26, 26, 25, 26, 26],
        [[427, 427, 86, 26, 427, 4096, 4096, 4096, 1], [427, 427, 85, 26, 427, 4096, 4096, 4096, 0], [426, 426, 85, 25, 426,
         4096, 4096, 4096, 1], [427, 427, 86, 26, 427, 4096, 4096, 4096, 1], [427, 427, 85, 25, 427, 4096, 4096, 4096, 0], [426,
         426, 85, 26, 426, 4096, 4096, 4096, 1], [427, 427, 86, 26, 427, 4096, 4096, 4096, 1], [427, 427, 85, 25, 427, 4096,
         4096, 4096, 0], [426, 426, 85, 26, 426, 4096, 4096, 4096, 1], [427, 427, 86, 25, 427, 4096, 4096, 4096, 1], [427, 427,
         85, 26, 427, 4096, 4096, 4096, 0], [426, 426, 85, 26, 426, 4096, 4096, 4096, 1], [427, 427, 86, 25, 427, 4096, 4096,
         4096, 1], [427, 427, 85, 26, 427, 4096, 4096, 4096, 0], [426, 426, 85, 25, 426, 4096, 4096, 4096, 1], [427, 427, 86, 26,
         427, 4096, 4096, 4096, 1]],
        {
            "0": "62f5e021ac971b33cf068dcff7145b2953a3d256d8e6fd0139ea7820058352f8",
            "1": "766cbe41a38a72d8a956f18e422cb4c06505ab186864593b81a7a84dd35d833a",
            "2": "020a512497cfeeca309a06d0f085c02204f3e3e48d9aed078a5e747b3f816b7c",
            "3": "b6f1a1a441bfecce7bf0c382f42b35fcba70e5bdd251382ba154fbee37ea199c",
            "4": "9648235e6f318454ca97f06d6414e31fb46bd2ea002cdce6b842da074a23a882",
            "5": "53bbc0385408b9d555f9a95d29448aaa1c2446234ed9ade9abb932bf687a692a",
            "6": "d23f578de769a817b88f3deaea758f84ebd769dd239ff8891bda06a337f33a25",
            "7": "910d234c92d87c5b24e8a9bd3557b26e55a10672450461333a45d91e0b0c2cc1",
            "fft": "4df9d9c7b62ba6520c96d0169ec9d12eecdcbdec08d7b799dc1c097688bb7d9b",
        }),
    "overlap0": (
        [21, 21, 21, 21, 21, 21, 21, 21, 21, 21, 21, 21, 21, 21, 21, 21],
        [[1250, 250, 76, 12000, 1], [1250, 250, 75, 12000, 1], [1250, 250, 75, 12000, 1], [1250, 250, 74, 12000, 1], [1250, 250,
         76, 12000, 1], [1250, 250, 75, 12000, 1], [1250, 250, 75, 12000, 1], [1250, 250, 74, 12000, 1], [1250, 250, 76, 12000,
         1], [1250, 250, 75, 12000, 1], [1250, 250, 75, 12000, 1], [1250, 250, 74, 12000, 1], [1250, 250, 76, 12000, 1], [1250,
         250, 75, 12000, 1], [1250, 250, 75, 12000, 1], [1250, 250, 74, 12000, 1]],
        {
            "0": "fd001ed063f592d3411c93630999c428ce7c2a357e29f3cfea0ddae9939ab623",
            "1": "db1c653e1fe4701497f965bff0f7c0d9a3ac1f6d895c6b9f7e4773d16e85b718",
            "2": "e49b9d5cfd84165dd5b637698e788eb673514efd2f3544ba56ce0c7bdce2c2a2",
            "3": "c656f56f8fed6405d1bfa5da0cb59b03d7896c2fd30f2812db7ed386173039d4",
            "fft": "87573fb19df92d2ab1a4fdc90ce5c892e95a6cf6e4fbf926b1d96bcd5e854d8a",
        }),
    "preproc_d4": (
        [21, 20, 21, 20, 21, 20, 21, 20, 21, 20, 21, 20],
        [[1250, 76, 12000, 12000, 12000, 12000, 12000, 1], [1250, 75, 12000, 12000, 12000, 12000, 12000, 0], [1250, 75, 12000,
         12000, 12000, 12000, 12000, 1], [1250, 74, 12000, 12000, 12000, 12000, 12000, 0], [1250, 76, 12000, 12000, 12000, 12000,
         12000, 1], [1250, 75, 12000, 12000, 12000, 12000, 12000, 0], [1250, 75, 12000, 12000, 12000, 12000, 12000, 1], [1250,
         74, 12000, 12000, 12000, 12000, 12000, 0], [1250, 76, 12000, 12000, 12000, 12000, 12000, 1], [1250, 75, 12000, 12000,
         12000, 12000, 12000, 0], [1250, 75, 12000, 12000, 12000, 12000, 12000, 1], [1250, 74, 12000, 12000, 12000, 12000, 12000,
         0]],
        {
            "0": "985a996835381dc04ef9e6f41350bf78d919b6ee696bc141e5b8bd028412234d",
            "1": "5ead20e7fe2455db58d7665d297a7a7608522423a0442bf8ec450e2f31e781a5",
            "2": "4ec30e36a4ac659b5f0a468e0b4733d47b27bc2c051d5151332f515a8f9f1d1f",
            "3": "fc65ce7d7e9f89dc4d11d36068c00ed3b8dffa496d91be739c1d3ede09281c02",
            "4": "0a06c5f360add520bdccf8fd6c1a6d1096b07f2182a0226e12d94b42a8305c7e",
            "5": "01e0ffca8982eb7e0a21fa9834e918b11f02700406d267ffcaaf297b9a17f177",
            "6": "85302b97750871c5497c74c8798d919511699c326bbf73eae56619f5caea6bc7",
            "fft": "f3e4003533add4786709d6702ee5f87eeca2475625ed09f544334e92828c0956",
        }),
    "preproc_d4_dc_inv": (
        [24, 23, 24, 23, 24, 23, 24, 23, 24, 23, 24, 23],
        [[1250, 76, 12000, 12000, 12000, 12000, 12000, 1], [1250, 75, 12000, 12000, 12000, 12000, 12000, 0], [1250, 75, 12000,
         12000, 12000, 12000, 12000, 1], [1250, 74, 12000, 12000, 12000, 12000, 12000, 0], [1250, 76, 12000, 12000, 12000, 12000,
         12000, 1], [1250, 75, 12000, 12000, 12000, 12000, 12000, 0], [1250, 75, 12000, 12000, 12000, 12000, 12000, 1], [1250,
         74, 12000, 12000, 12000, 12000, 12000, 0], [1250, 76, 12000, 12000, 12000, 12000, 12000, 1], [1250, 75, 12000, 12000,
         12000, 12000, 12000, 0], [1250, 75, 12000, 12000, 12000, 12000, 12000, 1], [1250, 74, 12000, 12000, 12000, 12000, 12000,
         0]],
        {
            "0": "8afa9570e0e701757f6282d2bc47e533b7465d92c2afa7b696e2c81422c6646a",
            "1": "a0ca65dcebf0cb10d540cc4c240707bc3223cf2ebb0a3a828dfb0894626e0944",
            "2": "bc7627c10a8e44db19f16140a7dc93822381fd0a7c5befbf93fbdc35ba7bbae7",
            "3": "732104d78b5203477de097252ee6befb5cbf989d804c9791c96d38d6d9445989",
            "4": "71972967d7bfadfac7fd2352b80a404b662bbf3eba2dd0ea2a37f11b520f99e8",
            "5": "127dda7dbf6355303a329279f060db4822001d9448b9288ea9eafc13ff17cb07",
            "6": "6ec31899011b47f5810ef4682cd004d6f95cdd42ec82a2929afc8884d0f80469",
            "fft": "c5662baf90631bbacf09750ae0c7eb116409172d37298c085634a6eb5e41fafd",
        }),
    "rds_device": (
        [18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18],
        [[1250, 7, 7, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 5, 5, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0],
         [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0],
         [1250, 6, 6, 0], [1250, 6, 5, 0]],
        {
            "0": "f602ca3e0705d5481d18fbef7ccafef3779def02ff67f8c03b6c7bb93366872e",
            "1": "923ac99b1f41ea92d24909bac0a1cbfe058c4e02e3462efdf061a21df7dbf351",
            "2": "3d1d01d0b793c06447728c6329dcb48a839a964bdc5b850346d0905bd77ab5e8",
        }),
    "rds_numpy": (
        [18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18],
        [[1250, 7, 7, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 5, 5, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0],
         [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0],
         [1250, 6, 6, 0], [1250, 6, 5, 0]],
        {
            "0": "f602ca3e0705d5481d18fbef7ccafef3779def02ff67f8c03b6c7bb93366872e",
            "1": "923ac99b1f41ea92d24909bac0a1cbfe058c4e02e3462efdf061a21df7dbf351",
            "2": "3d1d01d0b793c06447728c6329dcb48a839a964bdc5b850346d0905bd77ab5e8",
        }),
    "rds_pinned": (
        [18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18, 18],
        [[1250, 7, 7, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 5, 5, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0],
         [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0], [1250, 6, 6, 0],
         [1250, 6, 6, 0], [1250, 6, 5, 0]],
        {
            "0": "f602ca3e0705d5481d18fbef7ccafef3779def02ff67f8c03b6c7bb93366872e",
            "1": "923ac99b1f41ea92d24909bac0a1cbfe058c4e02e3462efdf061a21df7dbf351",
            "2": "3d1d01d0b793c06447728c6329dcb48a839a964bdc5b850346d0905bd77ab5e8",
        }),
    "shard_world1": (
        [16, 16, 16, 16, 16, 16, 16, 16, 16, 16, 16, 16],
        [[1250, 250, 1], [1250, 250, 1], [1250, 250, 1], [1250, 250, 1], [1250, 250, 1], [1250, 250, 1], [1250, 250, 1], [1250,
         250, 1], [1250, 250, 1], [1250, 250, 1], [1250, 250, 1], [1250, 250, 1]],
        {
            "0": "dd05396a799146eaf7693b8d954b01e4a19d424bd7140daa531397f0374cbc1e",
            "1": "2a5b94747f95acc0b1712fb720c037d3ff349276adc49c8511887ee9f3768a2c",
            "fft": "1aedf92ed8a3ed6e88314966ae3e6a3f7385d967303a6cbb26faa71e10104287",
        }),
    "spectrum_v0": (
        [16, 16, 19, 17, 16, 19, 17, 16, 16, 17, 16, 16, 18, 16],
        [[521, 105, 0], [313, 62, 0], [2083, 417, 2], [730, 146, 1], [208, 42, 0], [3125, 624, 2], [427, 86, 1], [1146, 229, 1],
         [937, 187, 0], [156, 32, 1], [2604, 520, 2], [625, 126, 0], [1250, 250, 1], [348, 69, 0]],
        {
            "0": "ec19a0b3893c2a494f82c92fd31903cba4be5a4e3bf54b0aff335ef5da59d716",
            "1": "98b0c976aaf49a6a736f3ff250845ded584c8627c44b4063250d999dfe56208c",
            "fft": "940d4a7b99c7d7e9449161581f07230a71c071979c655d21a173c95ad1ff60c0",
        }),
    "spectrum_v1": (
        [15, 15, 18, 16, 15, 19, 17, 16, 15, 17, 16, 15, 18, 15],
        [[521, 105, 0], [313, 62, 0], [2083, 417, 2], [730, 146, 1], [208, 42, 0], [3125, 624, 2], [427, 86, 1], [1146, 229, 1],
         [937, 187, 0], [156, 32, 1], [2604, 520, 2], [625, 126, 0], [1250, 250, 1], [348, 69, 0]],
        {
            "0": "ec19a0b3893c2a494f82c92fd31903cba4be5a4e3bf54b0aff335ef5da59d716",
            "1": "98b0c976aaf49a6a736f3ff250845ded584c8627c44b4063250d999dfe56208c",
            "fft": "940d4a7b99c7d7e9449161581f07230a71c071979c655d21a173c95ad1ff60c0",
        }),
}


@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_submit_paths_pinned(sb, name):
    deltas, counts, sha = _scenario(sb, name)
    want_deltas, want_counts, want_sha = EXPECTED[name]
    assert deltas == want_deltas, (name, deltas)
    assert counts == want_counts, (name, counts)
    assert sha == want_sha, (name, sha)

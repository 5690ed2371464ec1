"""Kernel options belong to the front end they are set on.  Front end A sets every launch-time kernel choice away from its
default ("tails", "fft", "fft_cta", "s1_stages", "s1_mt", "s1_ctas", "pdl"); a front end B2 created beside it, and stand-alone
blocks and spectrum handles, run exactly as they do with no such front end in the process: the same kernels (names with their
template arguments, from torch.profiler), the same launches per chunk, the same stage-1 TMA launches and the same output bits.
A keeps its own choices after B2 was created.  The retired option "s1_cps" is refused like any unknown option."""
import hashlib
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from util import fm_carrier, noise_iq

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FS = 100e6
OFFSETS = [5e6, -5e6, 15e6, -15e6]          # on the 5 MHz grid: stage 1 runs k_xd_tma on cf32 chunks
SCHED = [1 << 20] * 4 + [300001]
PROFILED = 2                                 # a chunk after the launch list's first two sightings: a replayed graph
FFT_SIZE, FFT_RATE = 1 << 20, 200.0
A_OPTS = {"tails": 0, "ft_prereg": 0, "fft": 0, "fft_cta": 4, "s1_stages": 3, "s1_mt": 256, "s1_ctas": 8, "pdl": 0}


@pytest.fixture(scope="module")
def sb():
    import sdrplusplus_b200 as m
    from sdrplusplus_b200 import lib
    L = lib.load()
    assert L.b200_device_count() > 0
    assert L.b200_init(0) == 0
    return m


def signal():
    n = sum(SCHED)
    y = noise_iq(n, 77, 0.01).astype(np.complex128)
    for o in OFFSETS:
        y = y + fm_carrier(n, FS, o)
    return y.astype(np.complex64)


def _profile(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return list(prof.events())


def kernel_names(fn):
    """full names (template arguments included) of the library's kernels that fn() launches"""
    return {e.name for e in _profile(fn) if re.search(r"\bk_[a-z0-9_]+", e.name)}


def base_names(names):
    return {re.search(r"\bk_[a-z0-9_]+", n).group(0) for n in names}


def tma_stages(names):
    """the ring depth (template argument NST, the last one) of every k_xd_tma build that ran"""
    return {int(re.search(r"\bk_xd_tma<([^>]*)>", n).group(1).split(",")[-1]) for n in names if re.search(r"\bk_xd_tma<", n)}


def front_end(sb, opts):
    fe = sb.FrontEnd(FS, max(SCHED))
    for k, v in opts.items():
        fe.set_option(k, v)
    fe.set_fft(FFT_SIZE, FFT_RATE)
    ids = [fe.add_vfo(sb.VfoConfig.wfm(o)) for o in OFFSETS]
    return fe, ids


class Record:
    """what one front end did over the schedule: sha256 of every VFO's audio and of the lines, launches per chunk, its
    stage-1 TMA launches, and the kernels of the profiled chunk"""

    def __init__(self, fe, ids):
        self.fe, self.ids = fe, ids
        self.sha = {k: hashlib.sha256() for k in list(ids) + ["lines"]}
        self.launches, self.names, self.k, self.pos = [], None, 0, 0

    def step(self, x):
        n = SCHED[self.k]

        def run():
            outs, lines = self.fe.process(x[self.pos:self.pos + n])
            for vid in self.ids:
                self.sha[vid].update(np.ascontiguousarray(outs[vid]).tobytes())
            self.sha["lines"].update(lines.tobytes())
        l0 = self.fe.launch_count()
        if self.k == PROFILED:
            self.names = kernel_names(run)
        else:
            run()
        self.launches.append(self.fe.launch_count() - l0)
        self.k += 1
        self.pos += n

    def result(self):
        return {"sha": {k: h.hexdigest() for k, h in self.sha.items()}, "launches": self.launches,
                "tma": self.fe.stat("s1_tma_launches"), "names": sorted(self.names)}


def standalone(x):
    """a decimating FIR block (decimation 3: the shared-memory tiled k_fir_cd in the default tail build) and a 1M-point
    spectrum handle: output bits and kernel names"""
    from sdrplusplus_b200 import Block, SpectrumHandler
    taps = np.hanning(33).astype(np.float32)
    taps /= taps.sum()
    blk = Block.fir_cr(taps, 3)
    sp = SpectrumHandler(FFT_SIZE, FFT_SIZE)
    got = {}
    try:
        def run():
            got["block"] = blk.process(x[:300001].view(np.float32))
            got["fft"] = sp.frame(x[:FFT_SIZE])
        names = kernel_names(run)
    finally:
        blk.close()
        sp.close()
    return {k: hashlib.sha256(v.tobytes()).hexdigest() for k, v in got.items()}, sorted(names)


def scenario():
    """B alone, the stand-alone handles, then A and B2 side by side and the stand-alone handles again"""
    import sdrplusplus_b200 as sb
    from sdrplusplus_b200 import lib
    assert lib.load().b200_init(0) == 0
    x = signal()
    # the defaults: front end B alone, then the stand-alone handles with no other front end in the process
    fe, ids = front_end(sb, {})
    try:
        rec = Record(fe, ids)
        for _ in SCHED:
            rec.step(x)
        b = rec.result()
    finally:
        fe.close()
    alone = standalone(x)
    # A with every kernel choice away from its default; B2 created beside it, configured like B; chunks interleaved
    fa, ida = front_end(sb, A_OPTS)
    fb = None
    try:
        ra = Record(fa, ida)
        ra.step(x)
        a_before = sorted(kernel_names(lambda: fa.process(x[:SCHED[0]])))
        fb, idb = front_end(sb, {})
        rb = Record(fb, idb)
        for _ in SCHED:
            if ra.k < len(SCHED):
                ra.step(x)
            rb.step(x)
        a, b2 = ra.result(), rb.result()
        during = standalone(x)
    finally:
        fa.close()
        if fb is not None:
            fb.close()
    return {"b": b, "alone": alone, "a_before": a_before, "a": a, "b2": b2, "during": during}


def test_options_stay_with_their_front_end(sb):
    # The scenario runs in a process of its own.  Late in a long test process torch.profiler has come back with only some, or
    # none, of the GPU kernels of a window -- even of a torch kernel of its own -- after earlier modules' profiler sessions
    # and CUDA graphs launched outside torch; a fresh process records every kernel.
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__)]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600,
                       env=dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT] + sys.path)))
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    b, b2, a = res["b"], res["b2"], res["a"]
    (alone, alone_names), (during, during_names) = res["alone"], res["during"]
    assert b["tma"] > 0
    assert tma_stages(b["names"]) == {2} and "k_fftr_p1" in base_names(b["names"]), b["names"]
    assert {"k_fir_c", "k_fft_p1"}.isdisjoint(base_names(b["names"])), b["names"]
    assert {"k_fir_cd", "k_fft_p1"} <= base_names(alone_names), alone_names
    assert b2 == b
    assert during == alone and during_names == alone_names
    for names in (res["a_before"], a["names"]):
        base = base_names(names)
        assert tma_stages(names) == {3}, names                               # "s1_stages" 3
        assert {"k_fft_p1", "k_fft_p2"} <= base and "k_fftr_p1" not in base, names     # "fft" 0
        assert "k_fir_c" in base and "k_fir_cd" not in base, names           # "tails" 0 (with "ft_prereg" 0)
    assert a["tma"] > 0


def test_retired_option_is_refused(sb):
    from sdrplusplus_b200 import B200Error
    fe = sb.FrontEnd(FS, 1 << 16)
    try:
        with pytest.raises(B200Error) as e:
            fe.set_option("s1_cps", 1)
        assert e.value.code == -1                                            # EINVAL
    finally:
        fe.close()


if __name__ == "__main__":
    print(json.dumps(scenario()))

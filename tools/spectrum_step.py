"""Spectrum branch of BASELINE config 2 (100 MS/s, 16 Mi-sample chunks, 1,048,576-point Nuttall FFT at 20 fps), with the
front end's "fft_v" option at 1 (a frame begun in earlier chunks joins its chunk's batch, the register passes read their
twiddles from shared memory) and at 0 (the frame is converted and transformed on its own, twiddles from global memory).

Two legs per option value, each pipelined submit / wait with two chunks in flight on a device-resident input and
device-resident outputs:
  * alone: the FFT with no VFO.  Reports the spectrum branch's device time per chunk from the CUDA events the front end
    records around it (group 2), and the wall time per chunk.
  * c2:    the FFT beside 8 WFM VFOs, the bench's stream settings.  Reports the wall time per chunk and the in-situ time of
    each launch group (0 stage 1, 1 behind stage 1, 2 spectrum branch) from the same events.
The option values alternate for --reps repetitions, so that drift of a shared machine shows up as spread, not as a
difference.  Prints one JSON line with per-repetition numbers, their median and spread (max - min), and the card's name,
power limit and top SM clock read in the same run.

    python tools/spectrum_step.py [--chunks 64] [--warmup 8] [--reps 5] [--fft-cta 8]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

FS = 100e6
CHUNK = 1 << 24
FFT_SIZE, FFT_RATE = 1 << 20, 20.0
OFFSETS = [5e6, -5e6, 15e6, -15e6, 25e6, -25e6, 35e6, -35e6]


def card():
    import torch
    ident = {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_max_mhz": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        pl, mx = out.stdout.strip().splitlines()[0].split(",")
        ident.update(power_limit_w=float(pl), sm_max_mhz=float(mx))
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        pass
    return ident


def leg(sb, lib, torch, xin, nbuf, fft_v, vfos, chunks, warmup, fft_cta):
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        fe = sb.FrontEnd(FS, CHUNK)
        fe.set_stream(stream.cuda_stream)
        fe.set_option("fft_v", fft_v)
        fe.set_option("fft_cta", fft_cta)
        fe.set_option("overlap", 1)
        fe.set_option("pair", 1)
        fe.set_option("tails", 2)
        fe.set_fft(FFT_SIZE, FFT_RATE, lib.WIN_NUTTALL)
        ids = [fe.add_vfo(sb.VfoConfig.wfm(o)) for o in OFFSETS] if vfos else []
        nl = fe.fft_max_lines(CHUNK)
        outs, keep = [], []
        for _ in range(2):
            o = lib.Outputs()
            for v in ids:
                cap = fe.vfo_max_out(v, CHUNK)
                t = torch.empty(2 * cap, device="cuda", dtype=torch.float32)
                keep.append(t)
                o.vfo_out[v], o.vfo_cap[v] = t.data_ptr(), cap
            t = torch.empty(nl * FFT_SIZE, device="cuda", dtype=torch.float32)
            keep.append(t)
            o.fft_out, o.fft_cap_lines, o.out_mem = t.data_ptr(), nl, lib.MEM_DEVICE
            outs.append(o)

        def run(n, first):
            inflight = 0
            for i in range(first, first + n):
                fe.submit_ptr(xin[i % nbuf].data_ptr(), CHUNK, lib.FMT_CF32, lib.MEM_DEVICE, outs[i % 2])
                inflight += 1
                if inflight == 2:
                    fe.wait()
                    inflight -= 1
            while inflight:
                fe.wait()
                inflight -= 1
            torch.cuda.synchronize()

        run(warmup, 0)
        fe.set_option("time_s1", 1)
        l0 = fe.launch_count()
        t0 = time.perf_counter()
        run(chunks, warmup)
        wall_us = (time.perf_counter() - t0) * 1e6 / chunks
        launches = (fe.launch_count() - l0) / chunks
        groups = {}
        for g, name in ((0, "stage1"), (1, "behind_stage1"), (2, "spectrum")):
            ms, n = fe.group_stats(g)
            groups[name] = ms * 1e3 / n if n else None
        fe.set_option("time_s1", 0)
        fe.close()
    return wall_us, groups, launches


def summary(xs):
    xs = [x for x in xs if x is not None]
    if not xs:
        return {"median": None, "spread": None}
    return {"median": round(float(np.median(xs)), 2), "spread": round(float(max(xs) - min(xs)), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=64, help="timed chunks per leg")
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--fft-cta", type=int, default=8, help="transforms per CTA of the register passes (8 or 4)")
    ap.add_argument("--nbuf", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this measures the H100 and has nothing to fall back to")
    import sdrplusplus_b200 as sb
    from sdrplusplus_b200 import lib
    L = lib.load()
    lib.check(L.b200_init(0))
    ident = card()
    g = torch.Generator(device="cuda").manual_seed(0x5D12)
    xin = [torch.rand(2 * CHUNK, device="cuda", generator=g, dtype=torch.float32) * 2.0 - 1.0 for _ in range(a.nbuf)]
    res = {v: {"alone": {"spectrum_us": [], "wall_us": [], "launches_per_chunk": []},
               "c2": {"wall_us": [], "stage1_us": [], "behind_stage1_us": [], "spectrum_us": []}} for v in (1, 0)}
    for _ in range(a.reps):
        for v in (1, 0):
            w, gr, nlaunch = leg(sb, lib, torch, xin, a.nbuf, v, False, a.chunks, a.warmup, a.fft_cta)
            r = res[v]["alone"]
            r["spectrum_us"].append(gr["spectrum"])
            r["wall_us"].append(w)
            r["launches_per_chunk"].append(nlaunch)
            w, gr, _ = leg(sb, lib, torch, xin, a.nbuf, v, True, a.chunks, a.warmup, a.fft_cta)
            r = res[v]["c2"]
            r["wall_us"].append(w)
            for k in ("stage1", "behind_stage1", "spectrum"):
                r[k + "_us"].append(gr[k])
    out = {}
    for v, legs in res.items():
        out["fft_v=%d" % v] = {name: {k: {"runs": [round(x, 2) if x is not None else None for x in xs], **summary(xs)}
                                      for k, xs in m.items()} for name, m in legs.items()}
    print(json.dumps({"tool": "spectrum_step", "card": ident, "samplerate": FS, "chunk": CHUNK, "fft_size": FFT_SIZE,
                      "fft_rate": FFT_RATE, "fft_cta": a.fft_cta, "chunks": a.chunks, "warmup": a.warmup, "reps": a.reps,
                      "results": out}))


if __name__ == "__main__":
    main()

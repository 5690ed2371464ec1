"""Cost of an IQ tap (b200_fe_bind_iq) at the bench geometry: 100 MS/s cs16 input from pinned memory, 8 WFM VFOs and a
1M-point FFT at 20 fps, 2 chunks in flight, outputs in b200_host_alloc buffers.  Six legs, alternated for --reps
repetitions at 16 Mi- and 1 Mi-sample chunks, so that drift of a shared machine shows up as spread:
  * none:       no tap;
  * cf32:       a CF32 tap;
  * i16:        an (I16, 32768) tap;
  * i16_dec4dc: an (I16, 32768) tap behind decimation 4 with DC blocking (VFO offsets inside the decimated +-12.5 MHz band);
  * none_dec4dc: the same front end without the tap, which is what i16_dec4dc is to be compared with;
  * cf32_direct: the CF32 tap with option host_direct 1, so that k_iq_tap stores into the b200_host_alloc buffer itself
                instead of handing its output to the copy engine (the default above 64 KiB of tap output).
Prints one JSON line: per-repetition wall time per chunk (ms), median and spread (max - min) per leg, the tap bytes that leave
the device per chunk, k_iq_tap's device time per chunk from CUDA events (launch group 3, a separate run of the leg with the
events on; from the moment the tap stream may start, so time spent waiting for SMs counts) as a share of the 3.35 TB/s
HBM3 data-sheet bandwidth for the bytes it moves, and the card's name, power limit and
top SM clock read in the same run.

    python tools/iq_tap_step.py [--chunks 24] [--warmup 4] [--reps 5]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FS = 100e6
OFFSETS = [5e6, -5e6, 15e6, -15e6, 25e6, -25e6, 35e6, -35e6]
OFFSETS_DEC4 = [1.5e6, -1.5e6, 4.5e6, -4.5e6, 7.5e6, -7.5e6, 10.5e6, -10.5e6]
HBM_BPS = 3.35e12
LEGS = ("none", "cf32", "i16", "i16_dec4dc", "none_dec4dc", "cf32_direct")


def card():
    import torch
    ident = {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_max_mhz": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        p, c = [s.strip() for s in out.stdout.strip().split(",")]
        ident["power_limit_w"], ident["sm_max_mhz"] = float(p), float(c)
    except Exception:
        pass
    return ident


def leg(sb, L, lib, xin, chunk, mode, chunks, warmup, timed):
    """wall ms per chunk (or, timed, k_iq_tap ms per chunk), tap bytes leaving the device per chunk, tap kernel bytes per chunk"""
    fe = sb.FrontEnd(FS, chunk)
    dec = mode.endswith("_dec4dc")
    if dec:
        fe.set_decimation(4)
        fe.set_dc_blocking(True)
    fe.set_fft(1 << 20, 20.0, L.WIN_NUTTALL)
    ids = [fe.add_vfo(sb.VfoConfig.wfm(o)) for o in (OFFSETS_DEC4 if dec else OFFSETS)]
    tid, tbytes = None, 0
    if mode.startswith("cf32"):
        tid, tbytes = fe.bind_iq(L.IQ_CF32), 8
        if mode == "cf32_direct":
            fe.set_option("host_direct", 1)
    elif mode.startswith("i16"):
        tid, tbytes = fe.bind_iq(L.IQ_I16, 32768.0), 4
    if timed:
        fe.set_option("time_s1", 1)
    pinned, slots = [], []
    for _ in range(2):
        o = L.Outputs()
        for i, b in [(v, 8) for v in ids] + ([(tid, tbytes)] if tid is not None else []):
            cap = fe.vfo_max_out(i, chunk)
            p = lib.b200_host_alloc(cap * b)
            pinned.append(p)
            o.vfo_out[i], o.vfo_cap[i] = p, cap
        nl = fe.fft_max_lines(chunk)
        p = lib.b200_host_alloc(nl * (1 << 20) * 4)
        pinned.append(p)
        o.fft_out, o.fft_cap_lines, o.out_mem = p, nl, L.MEM_HOST
        slots.append(o)
    inflight, t0 = 0, None
    for k in range(warmup + chunks):
        if k == warmup:
            while inflight:
                fe.wait()
                inflight -= 1
            if timed:
                fe.group_stats(3)
            t0 = time.perf_counter()
        if inflight == 2:
            fe.wait()
            inflight -= 1
        fe.submit_ptr(xin, chunk, L.FMT_CS16, L.MEM_HOST, slots[k % 2])
        inflight += 1
    while inflight:
        fe.wait()
        inflight -= 1
    ms = (time.perf_counter() - t0) * 1e3 / chunks
    eff = slots[0].vfo_count[tid] if tid is not None else 0
    if timed:
        tap_ms, n = fe.group_stats(3)
        ms = tap_ms / max(n, 1)
    fe.close()
    for p in pinned:
        lib.b200_host_free(p)
    in_bytes = (8 if dec else 4) * eff         # what k_iq_tap reads: the decimated cf32 stream, or the cs16 chunk
    return ms, eff * tbytes, in_bytes + eff * tbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", default="16777216,1048576")
    a = ap.parse_args()
    import torch
    import sdrplusplus_b200 as sb
    from sdrplusplus_b200 import lib as L
    lib = L.load()
    torch.cuda.init()
    out = {"geometry": {"fs": FS, "vfos": len(OFFSETS), "fft": 1 << 20, "fft_rate": 20.0, "inflight": 2, "input": "cs16 pinned"},
           "card": card(), "sizes": {}}
    for chunk in [int(s) for s in a.sizes.split(",")]:
        xin = lib.b200_host_alloc(chunk * 4)
        x = np.frombuffer((C.c_int16 * (2 * chunk)).from_address(xin), np.int16)
        x[:] = np.random.default_rng(1).normal(0, 1600, 2 * chunk).clip(-32768, 32767).astype(np.int16)
        nch = max(8, a.chunks if chunk >= (1 << 23) else a.chunks * 8)
        for m in LEGS:                                              # warm every shape once
            leg(sb, L, lib, xin, chunk, m, 2, 2, False)
        res = {m: [] for m in LEGS}
        tb = {}
        for _ in range(a.reps):
            for m in LEGS:
                ms, tb[m], _ = leg(sb, L, lib, xin, chunk, m, nch, a.warmup, False)
                res[m].append(round(ms, 3))
        legs = {}
        for m, v in res.items():
            s = sorted(v)
            legs[m] = {"ms_per_chunk": v, "median": s[len(s) // 2], "spread": round(s[-1] - s[0], 3), "tap_bytes_out_per_chunk": tb[m]}
            if not m.startswith("none"):
                kms, _, kb = leg(sb, L, lib, xin, chunk, m, nch, a.warmup, True)
                legs[m]["k_iq_tap_ms_per_chunk"] = round(kms, 4)
                legs[m]["k_iq_tap_bytes_per_chunk"] = kb
                legs[m]["k_iq_tap_share_of_3_35_TBps"] = round(kb / HBM_BPS * 1e3 / kms, 3) if kms > 0 else None
        out["sizes"][str(chunk)] = legs
        lib.b200_host_free(xin)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

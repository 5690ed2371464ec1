"""RDS for every station of a band: step time of a 100 MS/s stream with 8 WFM VFOs and RDS symbols for the same 8 stations,
decoded either inside the front end (8 B200_DEMOD_WFM_RDS_BITS VFOs, one RDSDemod launch per chunk on the tail stream) or
by the two-piece path (8 B200_DEMOD_WFM_RDS VFOs whose 5 kS/s streams go to 8 stand-alone b200_rds_demod handles after every
wait).  A third leg, 8 WFM + 8 WFM_RDS with no symbol decoding at all, is the floor both are compared with.

Every leg pipelines submit / wait with two chunks in flight on a device-resident input, outputs in pinned b200_host_alloc
buffers, and the legs alternate (--rounds) so that drift of the shared machine shows up as spread, not as a difference.
Prints one JSON line: per leg the mean step time (ms) of each round, the symbols recovered per second of wall time and the
5 kS/s samples per second they came from, with the card's name and power limit read in the same run.

    python tools/rds_band_step.py --steps 40 --warmup 5 [--chunk 16777216] [--rounds 3]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

FS = 100e6
OFFS = [-42e6 + 12e6 * k for k in range(8)]


def card():
    import torch
    ident = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        ident["power_limit_w"] = float(out.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        pass
    return ident


def make_input(chunk, nbuf):
    """nbuf chunks of 8 FM carriers whose multiplex carries audio, the pilot and a 57 kHz biphase subcarrier, plus noise"""
    import torch
    n = chunk * nbuf
    g = torch.Generator(device="cuda").manual_seed(7)
    t = torch.arange(n, device="cuda", dtype=torch.float64) / FS
    x = torch.zeros(n, device="cuda", dtype=torch.complex64)
    for k, off in enumerate(OFFS):
        bits = (torch.randint(0, 2, (int(n / FS * 2375.0) + 2,), device="cuda", generator=g) * 2 - 1).to(torch.float64)
        base = bits[(t * 2375.0).long()]
        mpx = 0.4 * torch.sin(2 * np.pi * (1000.0 + 100 * k) * t) + 0.1 * torch.sin(2 * np.pi * 19000.0 * t) + \
            0.06 * base * torch.sin(2 * np.pi * 57000.0 * t)
        ph = 2 * np.pi * off * t + 2 * np.pi * 75000.0 * torch.cumsum(mpx, 0) / FS
        x += (0.05 * torch.exp(1j * ph)).to(torch.complex64)
        del bits, base, mpx, ph
    x += (0.002 * torch.complex(torch.rand(n, device="cuda", generator=g) - 0.5, torch.rand(n, device="cuda", generator=g) - 0.5)).to(torch.complex64)
    torch.cuda.synchronize()
    return torch.view_as_real(x).contiguous()


def leg(sb, lib, L, xin, chunk, nbuf, mode, steps, warmup):
    """mode: "bits" (RDSDemod in the front end), "two_piece" (stand-alone handles), "none" (5 kS/s streams, no decoding)"""
    fe = sb.FrontEnd(FS, chunk)
    wfm = [fe.add_vfo(sb.VfoConfig.wfm(o)) for o in OFFS]
    side = [fe.add_vfo(sb.VfoConfig.wfm_rds_bits(o) if mode == "bits" else sb.VfoConfig.wfm_rds(o)) for o in OFFS]
    demods = [sb.RdsDemod() for _ in OFFS] if mode == "two_piece" else []
    outs, bufs = [], []
    for _ in range(2):
        o = lib.Outputs()
        for v in wfm + side:
            cap = fe.vfo_max_out(v, chunk)
            p = L.b200_host_alloc(8 * cap)
            bufs.append(p)
            o.vfo_out[v], o.vfo_cap[v] = p, cap
        o.out_mem = lib.MEM_HOST
        outs.append(o)
    stats = {"symbols": 0, "rds_in": 0}

    def drain(o, timed):
        for j, v in enumerate(side):
            n = o.vfo_count[v]
            if mode == "two_piece":
                y = np.ctypeslib.as_array((C.c_float * (2 * n)).from_address(o.vfo_out[v])).view(np.complex64) if n else np.empty(0, np.complex64)
                nsym = demods[j].process(y)[0].size
            else:
                nsym = n if mode == "bits" else 0
            if timed:
                stats["symbols"] += nsym
                stats["rds_in"] += n if mode != "bits" else 0     # the 5 kS/s count of a bits VFO is not an output
    base = xin.data_ptr()
    total = steps + warmup
    pend, t0, timed = [], None, 0
    for i in range(total):
        if i == warmup:
            import torch
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        fe.submit_ptr(base + (i % nbuf) * chunk * 8, chunk, lib.FMT_CF32, lib.MEM_DEVICE, outs[i % 2])
        pend.append(i)
        if len(pend) == 2:
            k = pend.pop(0)
            fe.wait()
            drain(outs[k % 2], k >= warmup)
    while pend:
        k = pend.pop(0)
        fe.wait()
        drain(outs[k % 2], k >= warmup)
    dt = time.perf_counter() - t0
    fe.close()
    for d in demods:
        d.close()
    for p in bufs:
        L.b200_host_free(C.c_void_p(p))
    return dt / steps * 1e3, stats["symbols"] / dt, stats["rds_in"] / dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--chunk", type=int, default=1 << 24)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--nbuf", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this measures the H100 and has nothing to fall back to")
    import sdrplusplus_b200 as sb
    from sdrplusplus_b200 import lib
    L = lib.load()
    L.b200_host_alloc.restype = C.c_void_p
    L.b200_init(0)
    ident = card()
    xin = make_input(a.chunk, a.nbuf)
    res = {m: {"step_ms": [], "symbols_per_s": [], "rds_5ksps_per_s": []} for m in ("bits", "two_piece", "none")}
    for _ in range(a.rounds):
        for m in res:
            ms, sps, ins = leg(sb, lib, L, xin, a.chunk, a.nbuf, m, a.steps, a.warmup)
            res[m]["step_ms"].append(round(ms, 3))
            res[m]["symbols_per_s"].append(round(sps, 1))
            res[m]["rds_5ksps_per_s"].append(round(ins, 1))
    for m, r in res.items():
        r["step_ms_mean"] = round(float(np.mean(r["step_ms"])), 3)
        if m == "bits":
            del r["rds_5ksps_per_s"]          # the same chain as the other legs; its 5 kS/s stream never leaves the device
    print(json.dumps({"tool": "rds_band_step", "card": ident, "samplerate": FS, "chunk": a.chunk, "steps": a.steps,
                      "warmup": a.warmup, "rounds": a.rounds, "vfos": {"wfm": 8, "rds": 8}, "legs": res}))


if __name__ == "__main__":
    main()

"""Cost of b200_fe_set_vfo_config at the bench geometry (100 MS/s, 16 Mi-sample chunks, 8 WFM VFOs with the radio's AF chain
and volume, 2 chunks in flight on a device-resident input and device-resident outputs).  Three legs, alternated for --reps
repetitions so that drift of a shared machine shows up as spread:
  * still:  nothing changes;
  * slider: one VFO's volume changes before every chunk (a coefficient: a new launch list, so a graph miss, per chunk);
  * toggle: one VFO's noise blanker is switched on or off every 10 chunks (the device is drained, the chain re-planned).
Prints one JSON line: per-repetition wall time per chunk (ms), median and spread (max - min) per leg, the median host time per
chunk submit spent on checks and plans (where b200_fe_set_vfo_config's changes are applied), and the card's name, power limit
and top SM clock read in the same run.

    python tools/vfo_settings_step.py [--chunks 60] [--warmup 8] [--reps 5]
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FS = 100e6
CHUNK = 1 << 24
OFFSETS = [5e6, -5e6, 15e6, -15e6, 25e6, -25e6, 35e6, -35e6]


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


def leg(sb, L, torch, x, mode, chunks, warmup):
    fe = sb.FrontEnd(FS, CHUNK)
    cfgs = [sb.VfoConfig.wfm(o).with_af(48000.0, False, 50e-6).with_volume(0.8) for o in OFFSETS]
    ids = [fe.add_vfo(c) for c in cfgs]
    outs = []
    for _ in range(2):
        o = L.Outputs()
        for vid in ids:
            cap = fe.vfo_max_out(vid, CHUNK)
            b = torch.empty(2 * cap, dtype=torch.float32, device="cuda")
            o.vfo_out[vid], o.vfo_cap[vid] = b.data_ptr(), cap
            outs.append(b)
        o.out_mem = L.MEM_DEVICE
        outs.append(o)
    slots = [outs[len(ids)], outs[2 * len(ids) + 1]]
    inflight = 0
    t0 = None
    for k in range(warmup + chunks):
        if k == warmup:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        c = copy.copy(cfgs[0])
        if mode == "slider":
            c.af_volume = 0.5 + 0.01 * (k % 50)
            fe.set_vfo_config(ids[0], c)
        elif mode == "toggle" and k % 10 == 0:
            c.nb_on, c.nb_level = (k // 10) % 2 == 1, 3.0
            fe.set_vfo_config(ids[0], c)
        if inflight == 2:
            fe.wait()
            inflight -= 1
        fe.submit_ptr(x.data_ptr(), CHUNK, L.FMT_CF32, L.MEM_DEVICE, slots[k % 2])
        inflight += 1
    while inflight:
        fe.wait()
        inflight -= 1
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / chunks
    misses = fe.stat("graph_misses")
    host_ms = fe.stat("host_ns_plan") / 1e6 / (warmup + chunks)      # submit's checks and plans, b200_fe_set_vfo_config's work included
    fe.close()
    return ms, misses, host_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    import sdrplusplus_b200 as sb
    from sdrplusplus_b200 import lib as L
    L.load()
    g = torch.Generator(device="cuda").manual_seed(1)
    x = (torch.randn(2 * CHUNK, device="cuda", generator=g) * 0.05).contiguous()
    res = {m: [] for m in ("still", "slider", "toggle")}
    miss, host = {}, {m: [] for m in res}
    for _ in range(a.reps):
        for m in res:
            ms, miss[m], h = leg(sb, L, torch, x, m, a.chunks, a.warmup)
            res[m].append(round(ms, 3))
            host[m].append(round(h, 3))
    summary = {m: {"ms_per_chunk": v, "median": sorted(v)[len(v) // 2], "spread": round(max(v) - min(v), 3),
                   "host_plan_ms_per_chunk_median": sorted(host[m])[len(v) // 2], "graph_misses_last_rep": miss[m]}
               for m, v in res.items()}
    print(json.dumps({"geometry": {"fs": FS, "chunk": CHUNK, "vfos": len(OFFSETS)}, "card": card(), "legs": summary}))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""What bounds stage 1 (k_xd_tma) on the bench workload: the kernel alone (nothing else on the GPU), then with its two halves
switched off in turn -- tiles loaded by the TMA ring but not filtered (what the loads alone sustain), tiles filtered but never
loaded (what the four consumer warps per SM alone sustain) -- at both ring depths.  CUDA-event time per launch.
    python tools/s1_bounds.py > s1_bounds.json"""
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch                                                   # noqa: E402
import sdrplusplus_b200 as sb                                  # noqa: E402
from sdrplusplus_b200 import lib                               # noqa: E402
import bench                                                   # noqa: E402


def run(chunk, opts):
    fe = sb.FrontEnd(bench.FS, chunk)
    fe.set_option("overlap", 0)
    for k, v in opts.items():
        fe.set_option(k, v)
    ids = [fe.add_vfo(sb.VfoConfig.wfm(o)) for o in bench.OFFSETS]
    ins = [torch.rand(2 * chunk, device="cuda") * 2 - 1 for _ in range(3)]
    o, keep = lib.Outputs(), []
    for v in ids:
        cap = fe.vfo_max_out(v, chunk)
        t = torch.empty(2 * cap, device="cuda")
        keep.append(t)
        o.vfo_out[v] = t.data_ptr(); o.vfo_cap[v] = cap
    o.out_mem = lib.MEM_DEVICE
    for k in range(3):
        fe.submit_ptr(ins[k % 3].data_ptr(), chunk, lib.FMT_CF32, lib.MEM_DEVICE, o); fe.wait()
    fe.set_option("time_s1", 1)
    for k in range(12):
        fe.submit_ptr(ins[k % 3].data_ptr(), chunk, lib.FMT_CF32, lib.MEM_DEVICE, o); fe.wait()
    ms, n = fe.s1_stats()
    fe.close()
    return ms / max(n, 1) * 1e3


def main():
    torch.cuda.set_device(0)
    L = lib.load()
    lib.check(L.b200_init(0))
    chunk = 1 << 24
    algo = 9.0 * chunk
    res = []
    for stages in (2, 3):
        for diag, what in ((0, "whole kernel"), (1, "tiles loaded, not filtered"), (2, "tiles filtered, not loaded")):
            us = run(chunk, {"s1_stages": stages, "s1_diag": diag})
            res.append({"ring_slot": "tile", "stages": stages, "mode": what, "us_per_launch": us, "GBps_algorithmic": algo / us / 1e3})
            print(json.dumps(res[-1]), file=sys.stderr)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()

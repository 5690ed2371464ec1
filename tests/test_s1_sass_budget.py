"""Residency budget of stage 1 (k_xd_tma) in libb200dsp.so, from cuobjdump.  The kernel is persistent, one CTA per SM, and
shares every SM with the spectrum branch: beside a pass-1 FFT CTA of 8 (256 threads x 144 registers = 36,864) it may take at
most 65,536 - 36,864 = 28,672 registers as allocated.  A consumer lane owns one output, so a CTA runs MT / 32 consumer warps
(the thread count of their named barrier) and one producer warp: 9 warps at D = 32 (MT = 256), 5 at D = 64 (MT = 128).
Nothing spills to local memory."""
import re
import shutil
import subprocess

import pytest

from sdrplusplus_b200 import lib

S1 = re.compile(r"k_xd_tmaILi(\d)ELi(\d)ELi(\d+)ELi(\d+)ELi(\d)E")
REGS_PER_SM = 65536
FFT_P1_CTA = 256 * 144                      # k_fftr_p1<., 32, 32, 8> with its tables in shared memory
S1_MAX_REGS = REGS_PER_SM - FFT_P1_CTA      # 28,672


def _cuobjdump(*args):
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    try:
        r = subprocess.run([exe, *args, lib.LIB_PATH], capture_output=True, text=True, timeout=600)
    except (OSError, subprocess.TimeoutExpired):
        pytest.skip("cuobjdump not available")
    if r.returncode != 0:
        pytest.skip("cuobjdump cannot read the library here")
    return r.stdout


def _census():
    res, fun = {}, None
    for line in _cuobjdump("-res-usage").splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            fun = m.group(1)
        elif fun and "REG:" in line:
            res[fun] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
            fun = None
    sass, fun = {}, None
    for line in _cuobjdump("-sass").splitlines():
        if "Function :" in line:
            fun = line.split("Function :")[1].strip()
            sass[fun] = {"spill": 0, "bar1": set()}
        elif fun:
            op = line.split("*/")[1].strip() if "*/" in line else ""
            if re.match(r"(@!?U?P\w+\s+)?(LDL|STL)\b", op):
                sass[fun]["spill"] += 1
            m = re.match(r"(@!?U?P\w+\s+)?BAR\.SYNC\S*\s+0x1,\s*(0x[0-9a-f]+)", op)
            if m:
                sass[fun]["bar1"].add(int(m.group(2), 16))
    return {f: (res[f], sass[f]) for f in sass if S1.search(f) and f in res}


def test_stage1_fits_beside_a_pass1_fft_cta():
    census = _census()
    assert len(census) == 16, sorted(census)          # D = 32 / 64 (QC 5 / 5, 6, 7), PS = 8 / 10, ring of 2 / 3
    for f, (res, sass) in census.items():
        logd, qc, ps, mt, nst = map(int, S1.search(f).groups())
        assert res["LOCAL"] == 0 and res["STACK"] == 0 and sass["spill"] == 0, (f, res, sass)
        assert sass["bar1"] == {mt}, (f, sass["bar1"])               # MT / 32 consumer warps, one output per lane
        warps = mt // 32 + 1
        assert warps == (9 if logd == 5 else 5), (f, warps)
        allocated = -(-res["REG"] // 8) * 8 * warps * 32             # registers are allocated 8 per thread at a time
        assert allocated <= S1_MAX_REGS, (f, res["REG"], allocated)

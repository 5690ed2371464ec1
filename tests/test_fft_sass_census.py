"""cuobjdump census of the register FFT passes in libb200dsp.so.  With their twiddle tables in shared memory (the TAB = true
instances, the front end's default), a pass-1 thread issues global loads only for its RA samples, its window as RA/4 16-byte
vectors and the two table-staging loops; a pass-2 thread for its RA work values and one staging loop.  The gathers of the
global-table instances (step-1 twiddle, coarse and fine epilogue factors) are gone, and nothing spills to local memory."""
import re
import shutil
import subprocess

import pytest

from sdrplusplus_b200 import lib

P1 = re.compile(r"k_fftr_p1ILi(\d)ELi(\d+)ELi(\d+)ELi(\d+)ELb([01])E")
P2 = re.compile(r"k_fftr_p2ILi(\d+)ELi(\d+)ELi(\d+)ELb([01])E")


def _census():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    try:
        sass = subprocess.run([exe, "-sass", lib.LIB_PATH], capture_output=True, text=True, timeout=600)
    except (OSError, subprocess.TimeoutExpired):
        pytest.skip("cuobjdump not available")
    if sass.returncode != 0:
        pytest.skip("cuobjdump cannot read the library here")
    fun, census = None, {}
    for line in sass.stdout.splitlines():
        if "Function :" in line:
            fun = line.split("Function :")[1].strip()
            census[fun] = {"LDG": 0, "LDS": 0, "LDL": 0, "STL": 0}
        elif fun:
            op = line.split("*/")[1].strip() if "*/" in line else ""
            for k in census[fun]:
                if re.match(r"(@!?U?P\w+\s+)?" + k + r"\b", op):
                    census[fun][k] += 1
    return census


def test_register_fft_passes_load_only_their_data():
    census = _census()
    p1 = {tuple(map(int, P1.search(f).groups())): c for f, c in census.items() if P1.search(f)}
    p2 = {tuple(map(int, P2.search(f).groups())): c for f, c in census.items() if P2.search(f)}
    assert len(p1) == 3 * 3 * 2 * 2 and len(p2) == 3 * 2 * 2, (len(p1), len(p2))     # formats x (RA, RB) x widths x tables
    for (fmt, ra, rb, c, tab), k in p1.items():
        if tab:
            assert k["LDG"] <= ra + ra // 4 + 2, (fmt, ra, rb, c, k)
            assert k["LDS"] >= ra + rb, k                          # step-1 twiddles, exchange tile, epilogue factors
            assert k["LDL"] == 0 and k["STL"] == 0, (fmt, ra, rb, c, k)
        else:
            assert k["LDG"] >= 3 * ra + 2 * rb - 1, k        # the gathers the tables remove
    for (ra, rb, r, tab), k in p2.items():
        if tab:
            assert k["LDG"] <= ra + 1, (ra, rb, r, k)
            assert k["LDL"] == 0 and k["STL"] == 0, (ra, rb, r, k)
        else:
            assert k["LDG"] >= 2 * ra - 1, k

"""RDSDemod inside the front end (B200_DEMOD_WFM_RDS_BITS): the WFM_RDS chain of a VFO followed by k_rds_demod, one launch per
16 such VFOs per chunk, the symbol counts filled in by b200_fe_wait.  The records must be exactly what the two-piece path
(a WFM_RDS VFO handed to a stand-alone b200_rds_demod) produces, whatever the chunking, pipelining and output memory."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from util import noise_iq, rds_group_bits, rds_mpx_iq

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FS = 2.0e6
OFF = 250e3


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_header_and_binding_agree_on_the_mode():
    from sdrplusplus_b200 import lib
    with open(lib.HEADER_PATH) as f:
        text = f.read()
    m = re.search(r"#define\s+B200_DEMOD_WFM_RDS_BITS\s+(\d+)", text)
    assert m and int(m.group(1)) == lib.DEMOD_WFM_RDS_BITS == 9
    assert re.search(r"typedef struct \{\s*float\s+soft;\s*uint32_t\s+bit;\s*\} b200_rds_symbol;", text)


def test_symbol_record_is_eight_bytes():
    from sdrplusplus_b200 import lib, frontend
    assert C.sizeof(lib.RdsSymbol) == 8 and frontend.RDS_SYMBOL.itemsize == 8
    assert lib.RdsSymbol.soft.offset == 0 and lib.RdsSymbol.bit.offset == 4
    with open(os.path.join(ROOT, "sdrplusplus_b200", "csrc", "api.cpp")) as f:
        assert "static_assert(sizeof(b200_rds_symbol) == 8" in f.read()


def test_library_exports_only_the_declared_entry_points():
    from sdrplusplus_b200 import lib
    nm = shutil.which("nm")
    if not nm or not os.path.exists(lib.LIB_PATH):
        pytest.skip("nm or the library is not available")
    r = subprocess.run([nm, "-D", "--defined-only", lib.LIB_PATH], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0
    exported = set(re.findall(r"\sT\s+(b200_[a-z0-9_]+)$", r.stdout, flags=re.M))
    assert exported == set(lib.header_symbols())


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def sb():
    import sdrplusplus_b200 as m
    from sdrplusplus_b200 import lib
    L = lib.load()
    assert L.b200_device_count() > 0
    assert L.b200_init(0) == 0
    return m


def _station(nbits, seed, fs=FS, off=OFF, bits=None):
    x, b = rds_mpx_iq(nbits, seed, fs=fs, bits=bits)
    t = np.arange(x.size) / fs
    return (x * np.exp(2j * np.pi * off * t)).astype(np.complex64), b


def _same(a, b):
    """two (soft, bit) pairs, bit for bit"""
    return a[0].shape == b[0].shape and np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1])


def _two_piece(sb, y_chunks):
    """the WFM_RDS output of every chunk handed to a stand-alone RDSDemod, chunk by chunk"""
    d = sb.RdsDemod()
    parts = [d.process(y) for y in y_chunks]
    d.close()
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


def _run_pair(fe, x, chunk):
    """a WFM_RDS VFO and a WFM_RDS_BITS VFO at the same offset: per chunk the 5 kS/s stream and the records"""
    ys, recs = [], []
    for i in range(0, x.size, chunk):
        outs, _ = fe.process(x[i:i + chunk])
        ys.append(outs[0])
        recs.append(outs[1])
    return ys, (np.concatenate([r[0] for r in recs]), np.concatenate([r[1] for r in recs]))


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [40000, 12500, 300])       # 300: most chunks carry no 5 kS/s sample at all
def test_same_symbols_as_the_two_piece_path(sb, report, chunk):
    nbits = 700 if chunk >= 12500 else 120
    x, _ = _station(nbits, 11)
    fe = sb.FrontEnd(FS, chunk)
    assert fe.add_vfo(sb.VfoConfig.wfm_rds(OFF)) == 0 and fe.add_vfo(sb.VfoConfig.wfm_rds_bits(OFF)) == 1
    ys, got = _run_pair(fe, x, chunk)
    fe.close()
    if chunk == 300:
        assert any(y.size == 0 for y in ys) and any(y.size > 0 for y in ys)
    ref = _two_piece(sb, ys)
    report["rds_frontend_two_piece_chunk%d" % chunk] = {"symbols": int(got[0].size)}
    assert got[0].size > 0.9 * sum(y.size for y in ys) / (5000.0 / 1187.5)
    assert _same(got, ref)


@pytest.mark.gpu
def test_against_the_oracle(sb, oracle, report):
    from test_gpu_rds import _gate
    chunk = 40000
    x, bits = _station(1500, 3)
    fe = sb.FrontEnd(FS, chunk)
    v = fe.add_vfo(sb.VfoConfig.wfm_rds_bits(OFF))
    outs, _ = fe.process_chunks(x, chunk)
    soft, hard = outs[v]
    fe.close()
    oracle.set_rotator_mode(1)
    try:
        ov, od = oracle.rxvfo(FS, 250e3, 150e3, OFF), oracle.wfm_rds(75e3, 250e3)
        ye = np.concatenate([od.process(ov.process(x[i:i + chunk].view(np.float32))).view(np.complex64) for i in range(0, x.size, chunk)])
    finally:
        oracle.set_rotator_mode(0)
    so, ho = oracle.rds_demod().process_chunks(ye, 250)
    r = _gate(soft, hard, so, ho)
    report["rds_frontend_vs_oracle"] = r
    assert r["bit_mismatches_off_threshold"] == 0, r
    best = max(np.mean(hard[300:1300] == bits[k: k + 1000]) for k in range(200, 400))
    assert best == 1.0, best


@pytest.mark.gpu
def test_twenty_stations_in_one_pass(sb, ref_oracle, report):
    """20 stations (two batches of RDS jobs) at distinct offsets of a 10 MS/s stream, each with its own PI / PS"""
    fs, chunk, nst = 10e6, 1 << 20, 20
    offs = [-3.9e6 + 0.4e6 * k for k in range(nst)]
    names = [("ST%02d" % k).ljust(8, "*") for k in range(nst)]
    pis = [0xC000 + 17 * k for k in range(nst)]
    x = None
    for k in range(nst):
        s, _ = _station(0, 100 + k, fs=fs, off=offs[k], bits=rds_group_bits(pis[k], names[k], 3))
        x = s if x is None else x[: min(x.size, s.size)] + s[: min(x.size, s.size)]
    x = (x * np.float32(0.1) + noise_iq(x.size, 9, 0.002)).astype(np.complex64)
    fe = sb.FrontEnd(fs, chunk)
    ids = [fe.add_vfo(sb.VfoConfig.wfm_rds_bits(o)) for o in offs]
    first, _ = fe.process(x[:chunk])                        # first chunk: nothing to compare the launch count with yet
    l0 = fe.launch_count()
    fe2 = sb.FrontEnd(fs, chunk)
    for o in offs:
        fe2.add_vfo(sb.VfoConfig.wfm_rds(o))
    fe2.process(x[:chunk])
    m0 = fe2.launch_count()
    rest, _ = fe.process_chunks(x[chunk:], chunk)
    fe2.process_chunks(x[chunk:], chunk)
    nch = (x.size - chunk + chunk - 1) // chunk
    extra = (fe.launch_count() - l0) - (fe2.launch_count() - m0)
    fe.close(); fe2.close()
    report["rds_frontend_twenty_stations"] = {"chunks": nch, "rds_launches": int(extra)}
    assert nch <= extra <= 2 * nch, (extra, nch)           # ceil(20 / 16) launches per chunk
    for k, v in enumerate(ids):
        assert ref_oracle.rds_group_decode(np.concatenate([first[v][1], rest[v][1]])) == (pis[k], names[k]), k


def _pipelined(sb, x, chunk, opts, depth, mem):
    """submit / wait with `depth` chunks in flight; mem: "pinned" (b200_host_alloc) or "device" (torch) output buffers"""
    import torch
    from sdrplusplus_b200 import lib
    L = lib.load()
    L.b200_host_alloc.restype = C.c_void_p
    fe = sb.FrontEnd(FS, chunk)
    fe.set_option("inflight", depth)
    for k, v in opts.items():
        fe.set_option(k, v)
    va, vr = fe.add_vfo(sb.VfoConfig.wfm(OFF)), fe.add_vfo(sb.VfoConfig.wfm_rds_bits(OFF))
    hin = [L.b200_host_alloc(chunk * 8) for _ in range(depth)]
    outs, keep = [], []
    for _ in range(depth):
        o = lib.Outputs()
        for v in (va, vr):
            cap = fe.vfo_max_out(v, chunk)
            if mem == "device":
                t = torch.empty(2 * cap, dtype=torch.float32, device="cuda")
                keep.append(t)
                o.vfo_out[v] = t.data_ptr()
            else:
                o.vfo_out[v] = L.b200_host_alloc(8 * cap)
            o.vfo_cap[v] = cap
        o.out_mem = lib.MEM_DEVICE if mem == "device" else lib.MEM_HOST
        outs.append(o)
    torch.cuda.synchronize()
    audio, recs = [], []

    def collect(k):
        o = outs[k % depth]
        for v, acc in ((va, audio), (vr, recs)):
            n = o.vfo_count[v]
            if mem == "device":
                a = keep[(k % depth) * 2 + (0 if v == va else 1)][: 2 * n].cpu().numpy()
            else:
                a = np.ctypeslib.as_array((C.c_float * (2 * n)).from_address(o.vfo_out[v])).copy() if n else np.empty(0, np.float32)
            acc.append(a)
    nch, done = (x.size + chunk - 1) // chunk, 0
    for c in range(nch):
        part = x[c * chunk:(c + 1) * chunk]
        C.memmove(hin[c % depth], part.ctypes.data, part.size * 8)
        fe.submit_ptr(hin[c % depth], part.size, lib.FMT_CF32, lib.MEM_HOST, outs[c % depth])
        if c - done + 1 == depth:
            fe.wait(); collect(done); done += 1
    while done < nch:
        fe.wait(); collect(done); done += 1
    fe.close()
    for p in hin:
        L.b200_host_free(C.c_void_p(p))
    if mem != "device":
        for o in outs:
            for v in (va, vr):
                L.b200_host_free(C.c_void_p(o.vfo_out[v]))
    r = np.concatenate(recs).view(np.dtype([("soft", np.float32), ("bit", np.uint32)]))
    return np.concatenate(audio), (r["soft"].copy(), r["bit"].astype(np.uint8))


@pytest.mark.gpu
@pytest.mark.parametrize("case", [({}, 2, "pinned"), ({}, 4, "pinned"), ({"graph": 0}, 2, "pinned"), ({"graph": 1}, 2, "pinned"),
                                  ({"host_direct": 0}, 2, "pinned"), ({"host_direct": 1}, 3, "pinned"), ({}, 2, "device"),
                                  ({"graph": 1}, 4, "device")])
def test_pipelining_and_modes_give_identical_records(sb, case):
    opts, depth, mem = case
    chunk = 25000
    x, _ = _station(400, 5)
    fe = sb.FrontEnd(FS, chunk)
    va, vr = fe.add_vfo(sb.VfoConfig.wfm(OFF)), fe.add_vfo(sb.VfoConfig.wfm_rds_bits(OFF))
    ref, _ = fe.process_chunks(x, chunk)                     # b200_fe_process, one chunk at a time
    fe.close()
    audio, recs = _pipelined(sb, x, chunk, opts, depth, mem)
    assert recs[0].size > 100 and _same(recs, ref[vr])
    assert np.array_equal(audio.view(np.uint32), ref[va].reshape(-1).view(np.uint32))


@pytest.mark.gpu
def test_reset_and_removal(sb):
    chunk = 20000
    x, _ = _station(400, 8)
    fe = sb.FrontEnd(FS, chunk)
    va = fe.add_vfo(sb.VfoConfig.wfm(OFF))
    vq = fe.add_vfo(sb.VfoConfig.wfm_rds(OFF))
    vr = fe.add_vfo(sb.VfoConfig.wfm_rds_bits(OFF))
    d = sb.RdsDemod()
    first, _ = fe.process_chunks(x, chunk)
    d.process(first[vq])                                     # the stand-alone block gets the same history, and the same reset
    fe.reset()
    d.reset()
    per = [fe.process(x[i:i + chunk])[0] for i in range(0, x.size, chunk)]
    soft, hard = np.concatenate([o[vr][0] for o in per]), np.concatenate([o[vr][1] for o in per])
    # reset restores everything but the clock recovery's 7-sample tail, as RDSDemod::reset does
    assert soft.size == first[vr][0].size and np.array_equal(hard[8:], first[vr][1][8:])
    parts = [d.process(o[vq]) for o in per]
    assert _same((soft, hard), (np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])))
    d.close()
    # removing the RDS VFO leaves the others alone
    fe.reset()
    fe.remove_vfo(vr)
    third, _ = fe.process_chunks(x, chunk)
    assert vr not in third
    for v in (va, vq):
        assert np.array_equal(third[v].view(np.uint32), np.concatenate([o[v] for o in per]).view(np.uint32))
    fe.close()


@pytest.mark.gpu
def test_no_change_for_the_other_vfos(sb, report):
    """8 WFM VFOs: their audio is the same, id by id, with or without an RDS VFO beside them, and the only launches an RDS VFO
    adds over a WFM_RDS VFO are its RDSDemod launches"""
    fs, chunk = 10e6, 500000
    offs = [-3.5e6 + 1e6 * k for k in range(8)]
    x, _ = _station(300, 21, fs=fs, off=offs[2])
    x = (x + noise_iq(x.size, 4, 0.01)).astype(np.complex64)
    res = {}
    for extra in (None, "wfm_rds", "wfm_rds_bits"):
        fe = sb.FrontEnd(fs, chunk)
        ids = [fe.add_vfo(sb.VfoConfig.wfm(o)) for o in offs]
        if extra:
            fe.add_vfo(getattr(sb.VfoConfig, extra)(offs[2]))
        outs, _ = fe.process_chunks(x, chunk)
        res[extra] = ([outs[i] for i in ids], fe.launch_count())
        fe.close()
    base = res[None][0]
    for extra in ("wfm_rds", "wfm_rds_bits"):
        for a, b in zip(base, res[extra][0]):
            assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), extra
    nch = (x.size + chunk - 1) // chunk
    report["rds_frontend_launches"] = {k or "wfm_only": v[1] for k, v in res.items()}
    assert res["wfm_rds_bits"][1] - res["wfm_rds"][1] == nch       # one RDSDemod launch per chunk (each carries 5 kS/s samples)

"""RDS bound to a front-end WFM VFO (b200_fe_bind_rds): BroadcastFM's rdsOut branch hangs off the VFO's own discriminator, as the
radio's "Decode RDS" does.  The records must be exactly those of a B200_DEMOD_WFM_RDS_BITS VFO at the same offset and settings,
the parent's audio that of a WFM VFO without RDS, whatever the build, chunking, pipelining and output memory; the work in front
of the discriminator runs once."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from util import noise_iq, rds_group_bits, rds_mpx_iq

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FS = 2.0e6
OFF = 250e3


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_header_declares_bind_and_unbind():
    from sdrplusplus_b200 import lib
    with open(lib.HEADER_PATH) as f:
        text = f.read()
    assert re.search(r"int\s+b200_fe_bind_rds\(b200_fe\*\s*fe,\s*int\s+vfo_id\);", text)
    assert re.search(r"int\s+b200_fe_unbind_rds\(b200_fe\*\s*fe,\s*int\s+id\);", text)
    assert {"b200_fe_bind_rds", "b200_fe_unbind_rds"} <= set(lib.header_symbols())


def test_discriminators_share_the_branch_rule():
    """k_rxl and both discriminators that feed a bound branch (k_quad, k_tail_fused's FT_QUAD) store rds_xlate's value"""
    src = os.path.join(ROOT, "sdrplusplus_b200", "csrc")
    with open(os.path.join(src, "kernels.cu")) as f:
        k = f.read()
    with open(os.path.join(src, "fused_tail.cuh")) as f:
        ft = f.read()
    assert k.count("phasor_u64(phase0 + w * (unsigned long long)i)") == 1
    rxl = k[k.index("k_rxl(const"):]
    assert "rds_xlate(" in rxl[: rxl.index("\n}\n")]
    quad = k[k.index("k_quad(const"):]
    assert "rds_xlate(" in quad[: quad.index("\n}\n")]
    assert "rds_xlate(" in ft[ft.index("case FT_QUAD"):]


def test_adapter_program_compiles(tmp_path):
    from sdrplusplus_b200 import lib as L
    if not os.path.exists(L.LIB_PATH):
        pytest.skip("library not built")
    _adapter_exe(L, tmp_path)


def _adapter_exe(L, tmp_path):
    here = os.path.dirname(os.path.abspath(__file__))
    exe = os.path.join(str(tmp_path), "rds_bound_adapter")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "sdrplusplus_b200", "host"), "-o", exe,
                        os.path.join(here, "rds_bound_adapter.cpp"), "-L", os.path.dirname(L.LIB_PATH), "-lb200dsp",
                        "-Wl,-rpath," + os.path.dirname(L.LIB_PATH), "-lpthread"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
    return exe


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


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _cfgs(sb, stereo, low_pass, if_chain, off=OFF):
    """the parent (WFM or WFM stereo), and a WFM_RDS_BITS VFO at the same offset with the same IF chain"""
    par = (sb.VfoConfig.wfm_stereo if stereo else sb.VfoConfig.wfm)(off)
    par.low_pass = low_pass
    bits = sb.VfoConfig.wfm_rds_bits(off)
    for c in (par, bits):
        if if_chain:
            c.nb_on, c.nb_level = True, 3.0
            c.squelch_on, c.squelch_level = True, -100.0
            c.nr_on, c.nr_bins = True, 32
    return par, bits


# (stereo, low_pass, IF chain, chunk, options): every tail build; "ft_regall" 0 puts the discriminator of a parent without IF
# blocks into k_tail_fused (as its last stage for stereo, in the middle for mono)
BUILDS = [
    (False, True, False, 40000, {}), (False, False, True, 12500, {}), (True, True, False, 300, {}),
    (True, False, True, 40000, {"tails": 1}), (False, True, True, 12500, {"tails": 1}),
    (False, True, False, 12500, {"tails": 0}), (True, True, True, 40000, {"tails": 0}),
    (False, True, False, 40000, {"ft_regall": 0}), (True, True, False, 12500, {"ft_regall": 0}),
    (False, False, False, 300, {"ft_regall": 0}), (True, False, False, 12500, {"ft_regall": 0}),
]


@pytest.mark.gpu
@pytest.mark.parametrize("build", BUILDS, ids=lambda b: "%s-lp%d-if%d-c%d-%s" % ("st" if b[0] else "mono", b[1], b[2], b[3],
                                                                                ",".join("%s%d" % kv for kv in b[4].items()) or "default"))
def test_records_and_audio_equal_the_two_vfo_way(sb, report, build):
    stereo, low_pass, if_chain, chunk, opts = build
    x, _ = _station(700 if chunk >= 12500 else 150, 11)
    x = (x + noise_iq(x.size, 2, 0.002)).astype(np.complex64)
    fe = sb.FrontEnd(FS, chunk)
    for k, v in opts.items():
        fe.set_option(k, v)
    par, bits = _cfgs(sb, stereo, low_pass, if_chain)
    vp = fe.add_vfo(par)
    vr = fe.bind_rds(vp)                                      # before the first chunk: the audio is that of a VFO without RDS
    vb = fe.add_vfo(bits)
    va = fe.add_vfo(par)
    outs, _ = fe.process_chunks(x, chunk)
    fused = fe.stat("fused_chains")
    fe.close()
    if opts.get("ft_regall") == 0:
        assert fused >= 2                                     # the parent's discriminator ran inside k_tail_fused
    report["rds_bound_" + "_".join(str(b) for b in build[:4]) + "_" + str(sorted(opts.items()))] = {"symbols": int(outs[vr][0].size)}
    assert outs[vr][0].size > 20 and _same(outs[vr], outs[vb])
    assert outs[vp].size > 0 and _bits_equal(outs[vp], outs[va])


@pytest.mark.gpu
def test_other_vfos_and_fft_lines_do_not_change(sb):
    chunk = 40000
    x, _ = _station(400, 4)
    res = []
    for bind in (False, True):
        fe = sb.FrontEnd(FS, chunk)
        fe.set_fft(8192, 30.0)
        ids = [fe.add_vfo(sb.VfoConfig.wfm_stereo(OFF)), fe.add_vfo(sb.VfoConfig.nfm(-300e3)), fe.add_vfo(sb.VfoConfig.wfm(-600e3))]
        if bind:
            fe.bind_rds(ids[0])
        outs, lines = fe.process_chunks(x, chunk)
        res.append(([outs[i] for i in ids], lines))
        fe.close()
    for a, b in zip(res[0][0], res[1][0]):
        assert _bits_equal(a, b)
    assert res[0][1].shape[0] > 0 and _bits_equal(res[0][1], res[1][1])


def _pipelined(sb, x, chunk, opts, depth, mem):
    """submit / wait with `depth` chunks in flight; mem: "pinned" (b200_host_alloc) or "device" (torch) output buffers.
    Returns the parent's audio and the bound output's records."""
    import torch
    from sdrplusplus_b200 import lib
    L = lib.load()
    L.b200_host_alloc.restype = C.c_void_p
    fe = sb.FrontEnd(FS, chunk)
    fe.set_option("inflight", depth)
    for k, v in opts.items():
        fe.set_option(k, v)
    va = fe.add_vfo(sb.VfoConfig.wfm_stereo(OFF))
    vr = fe.bind_rds(va)
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
        for j, (v, acc) in enumerate(((va, audio), (vr, recs))):
            n = o.vfo_count[v]
            if mem == "device":
                a = keep[(k % depth) * 2 + j][: 2 * n].cpu().numpy()
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
@pytest.mark.parametrize("case", [({}, 2, "pinned"), ({}, 3, "pinned"), ({}, 4, "pinned"), ({"graph": 0}, 2, "pinned"),
                                  ({"graph": 1}, 2, "pinned"), ({"host_direct": 0}, 2, "pinned"), ({"host_direct": 1}, 3, "pinned"),
                                  ({}, 2, "device"), ({"graph": 1}, 4, "device")])
def test_pipelining_and_modes_give_identical_records(sb, case):
    opts, depth, mem = case
    chunk = 25000
    x, _ = _station(400, 5)
    fe = sb.FrontEnd(FS, chunk)
    va = fe.add_vfo(sb.VfoConfig.wfm_stereo(OFF))
    vb = fe.add_vfo(sb.VfoConfig.wfm_rds_bits(OFF))
    ref, _ = fe.process_chunks(x, chunk)                     # b200_fe_process, one chunk at a time, the two-VFO way
    fe.close()
    audio, recs = _pipelined(sb, x, chunk, opts, depth, mem)
    assert recs[0].size > 100 and _same(recs, ref[vb])
    assert np.array_equal(audio.view(np.uint32), ref[va].reshape(-1).view(np.uint32))


@pytest.mark.gpu
def test_against_the_oracle(sb, oracle, report):
    from test_gpu_rds import _gate
    chunk = 40000
    x, bits = _station(1500, 3)
    fe = sb.FrontEnd(FS, chunk)
    v = fe.add_vfo(sb.VfoConfig.wfm_stereo(OFF))
    r = fe.bind_rds(v)
    outs, _ = fe.process_chunks(x, chunk)
    soft, hard = outs[r]
    fe.close()
    oracle.set_rotator_mode(1)
    try:
        ov, od = oracle.rxvfo(FS, 250e3, 150e3, OFF), oracle.wfm_rds(75e3, 250e3)
        ye = np.concatenate([od.process(ov.process(x[i:i + chunk].view(np.float32))).view(np.complex64) for i in range(0, x.size, chunk)])
    finally:
        oracle.set_rotator_mode(0)
    so, ho = oracle.rds_demod().process_chunks(ye, 250)
    g = _gate(soft, hard, so, ho)
    report["rds_bound_vs_oracle"] = g
    assert g["bit_mismatches"] == 0, g
    best = max(np.mean(hard[300:1300] == bits[k: k + 1000]) for k in range(200, 400))
    assert best == 1.0, best


@pytest.mark.gpu
def test_twenty_stereo_stations_in_one_pass(sb, ref_oracle, report):
    """20 stereo stations of a 10 MS/s stream, one WFM VFO each with RDS bound: each decodes to its own PI / PS"""
    from sdrplusplus_b200 import lib
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
    vids = [fe.add_vfo(sb.VfoConfig.wfm_stereo(o)) for o in offs]
    rids = [fe.bind_rds(v) for v in vids]
    outs, _ = fe.process_chunks(x, chunk)
    nvfo = lib.load().b200_fe_vfo_count(fe._h)
    fe.close()
    # 20 VFOs go through stage 1 and the chain in front of the discriminator; each RDS output takes one more id
    report["rds_bound_twenty_stations"] = {"vfos": len(vids), "ids": int(nvfo)}
    assert nvfo == 2 * nst
    for k, r in enumerate(rids):
        assert outs[vids[k]].size > 0
        assert ref_oracle.rds_group_decode(outs[r][1]) == (pis[k], names[k]), k


@pytest.mark.gpu
def test_front_runs_once(sb, report):
    """100 MS/s cf32 chunks (TMA stage 1 with its ÷4 epilogue, plan (32, 143) (4, 27) (2, 69)): N WFM VFOs with RDS bound add N
    stage-1 ÷4 jobs per chunk where the two-VFO way adds 2N, and no more launches"""
    fs, chunk, n, nch = 100e6, 1 << 20, 4, 4
    x = noise_iq(chunk * nch, 3, 0.5)
    offs = [-20e6 + 10e6 * k for k in range(n)]
    res = {}
    for way in ("bound", "two"):
        fe = sb.FrontEnd(fs, chunk)
        for o in offs:
            v = fe.add_vfo(sb.VfoConfig.wfm_stereo(o))
            if way == "bound":
                fe.bind_rds(v)
            else:
                fe.add_vfo(sb.VfoConfig.wfm_rds_bits(o))
        fe.process(x[:chunk])
        j0, l0 = fe.stat("s1_f2_jobs"), fe.launch_count()
        for c in range(1, nch):
            fe.process(x[c * chunk:(c + 1) * chunk])
        res[way] = ((fe.stat("s1_f2_jobs") - j0) / (nch - 1), (fe.launch_count() - l0) / (nch - 1))
        fe.close()
    report["rds_bound_front_shared"] = {k: {"s1_f2_jobs_per_chunk": v[0], "launches_per_chunk": v[1]} for k, v in res.items()}
    assert res["bound"][0] == n and res["two"][0] == 2 * n
    assert res["bound"][1] <= res["two"][1]


def _oracle_audio(oracle, x, chunk, resets):
    """RxVFO -> BroadcastFM (mono, 15 kHz low-pass) in the reference, BroadcastFM::reset before the chunks in `resets`"""
    oracle.set_rotator_mode(1)
    try:
        ov, od = oracle.rxvfo(FS, 250e3, 150e3, OFF), oracle.wfm(75e3, 250e3, False, True)
        out = []
        for c, i in enumerate(range(0, x.size, chunk)):
            if c in resets:
                od.reset()
            out.append(od.process(ov.process(x[i:i + chunk].view(np.float32))))
    finally:
        oracle.set_rotator_mode(0)
    return np.concatenate(out).reshape(-1, 2)


@pytest.mark.gpu
def test_toggles_between_chunks(sb, oracle, report):
    """bind before chunk 4, unbind before 8, bind again before 12: the parent's BroadcastFM restarts at each toggle; the branch
    starts fresh, is parked by the unbind and resumes from there"""
    from test_gpu_rds import _gate
    chunk, nch = 40000, 16
    x, _ = _station(2000, 6)
    x = x[: chunk * nch]
    fe = sb.FrontEnd(FS, chunk)
    vp = fe.add_vfo(sb.VfoConfig.wfm(OFF))
    vq = fe.add_vfo(sb.VfoConfig.wfm(OFF))                     # the same VFO without RDS: never restarted
    audio, plain, recs = [], [], []
    rid = None
    for c in range(nch):
        if c in (4, 12):
            rid = fe.bind_rds(vp)
        if c == 8:
            fe.unbind_rds(rid)
            rid = None
        outs, _ = fe.process(x[c * chunk:(c + 1) * chunk])
        audio.append(outs[vp]); plain.append(outs[vq])
        if rid is not None:
            recs.append((c, outs[rid]))
    fe.close()
    audio, plain = np.concatenate(audio), np.concatenate(plain)
    per = audio.shape[0] // nch
    # before the first toggle the parent is the plain VFO; after it the restart shows
    assert _bits_equal(audio[: 4 * per], plain[: 4 * per])
    assert not np.array_equal(audio[4 * per: 4 * per + 200], plain[4 * per: 4 * per + 200])
    ref, ref_plain = _oracle_audio(oracle, x, chunk, {4, 8, 12}), _oracle_audio(oracle, x, chunk, set())
    scale = float(np.sqrt(np.mean(ref.astype(np.float64) ** 2)))
    errs = {}
    for b in (4, 8, 12):
        w = slice(b * per, b * per + 256)                      # the restart's transient: the delay lines refilling
        e = float(np.max(np.abs(audio[w] - ref[w]))) / scale
        e_plain = float(np.max(np.abs(ref_plain[w] - ref[w]))) / scale
        errs[b] = (e, e_plain)
        assert e < 1e-3 and e_plain > 100 * e, (b, e, e_plain)
    # the records: the reference's branch (RealToComplex -> xlator -> resampler -> RDSDemod) behind the same discriminator,
    # left alone while unbound
    oracle.set_rotator_mode(1)
    try:
        ov, q = oracle.rxvfo(FS, 250e3, 150e3, OFF), oracle.quad(75e3, 250e3)
        xl, rs, rd = oracle.xlator(-57000.0, 250e3), oracle.resamp(250e3, 5000.0), oracle.rds_demod()
        so, ho, bound_chunks = [], [], {c for c, _ in recs}
        for c in range(nch):
            if c in (4, 8, 12):
                q.reset()
            m = q.process(ov.process(x[c * chunk:(c + 1) * chunk].view(np.float32)))
            if c in bound_chunks:
                y = rs.process(xl.process(np.stack([m, np.zeros_like(m)], 1).reshape(-1))).view(np.complex64)
                s, h = rd.process(y)
                so.append(s); ho.append(h)
    finally:
        oracle.set_rotator_mode(0)
    soft = np.concatenate([r[1][0] for r in recs]); hard = np.concatenate([r[1][1] for r in recs])
    g = _gate(soft, hard, np.concatenate(so), np.concatenate(ho))
    report["rds_bound_toggles"] = {"audio_restart_err": errs, "records": g}
    assert g["bit_mismatches_off_threshold"] == 0, g
    assert abs(soft.size - np.concatenate(so).size) <= 1


@pytest.mark.gpu
def test_reset_clears_the_parked_branch(sb):
    """b200_fe_reset clears a parked branch: bound again after a reset, it gives what a first bind after the reset gives"""
    chunk = 40000
    x, _ = _station(800, 7)
    runs = []
    for park in (True, False):
        fe = sb.FrontEnd(FS, chunk)
        vp = fe.add_vfo(sb.VfoConfig.wfm(OFF))
        if park:
            r = fe.bind_rds(vp)
            fe.process_chunks(x[: 4 * chunk], chunk)
            fe.unbind_rds(r)
        fe.reset()
        r = fe.bind_rds(vp)
        outs, _ = fe.process_chunks(x, chunk)
        runs.append((outs[vp], outs[r]))
        fe.close()
    # as RDSDemod::reset: everything but the clock recovery's 7-sample work-buffer tail (tests/test_gpu_rds_frontend.py)
    assert runs[0][1][0].size == runs[1][1][0].size > 50 and np.array_equal(runs[0][1][1][8:], runs[1][1][1][8:])
    assert _bits_equal(runs[0][0], runs[1][0])


@pytest.mark.gpu
def test_rejections(sb):
    from sdrplusplus_b200 import lib
    L = lib.load()
    fe = sb.FrontEnd(FS, 10000)
    h = fe._h
    vw = fe.add_vfo(sb.VfoConfig.wfm(OFF))
    vn = fe.add_vfo(sb.VfoConfig.nfm(-300e3))
    vb = fe.add_vfo(sb.VfoConfig.wfm_rds_bits(-500e3))
    tap = fe.bind_iq(lib.IQ_CF32)
    for bad in (vn, vb, tap, 63, -1):
        assert L.b200_fe_bind_rds(h, bad) == -1             # B200_EINVAL: not a WFM / WFM stereo VFO
    n0 = L.b200_fe_vfo_count(h)
    r = fe.bind_rds(vw)
    assert L.b200_fe_vfo_count(h) == n0 + 1
    assert L.b200_fe_bind_rds(h, vw) == -1                   # one RDS output per VFO
    assert L.b200_fe_bind_rds(h, r) == -1                    # an RDS output is no WFM VFO
    cfg = sb.VfoConfig.wfm(OFF).to_c()
    assert L.b200_fe_set_vfo_offset(h, r, C.c_double(1.0)) == -1
    assert L.b200_fe_set_vfo_bandwidth(h, r, C.c_double(1e5)) == -1
    assert L.b200_fe_set_vfo_config(h, r, C.byref(cfg)) == -1
    assert L.b200_fe_remove_vfo(h, r) == -1
    assert L.b200_fe_unbind_iq(h, r) == -1
    assert L.b200_fe_unbind_rds(h, vw) == -1 and L.b200_fe_unbind_rds(h, tap) == -1
    assert L.b200_fe_remove_vfo(h, vw) == -7                 # B200_ESTATE: unbind first
    assert L.b200_fe_set_decimation(h, 2) == -7
    bound = fe.vfo_max_out(r, 10000)
    assert bound == fe.vfo_max_out(vb, 10000) > 0
    # the parent's settings go on working while bound: an IF-chain toggle re-plans it, the branch stays attached
    c2 = sb.VfoConfig.wfm(OFF)
    c2.nb_on, c2.nb_level = True, 3.0
    fe.set_vfo_config(vw, c2)
    x, _ = _station(200, 9)
    outs, _ = fe.process_chunks(x[:40000], 10000)
    assert outs[r][0].size > 0 and outs[vw].size > 0
    fe.unbind_rds(r)
    assert L.b200_fe_unbind_rds(h, r) == -1
    fe.remove_vfo(vw)
    fe.close()


@pytest.mark.gpu
def test_adapter_bind_rds_decodes(sb, ref_oracle, tmp_path):
    """dsp::b200::FrontEnd: a stereo WFM VFO with bindRDS on worker-thread blocks (tests/rds_bound_adapter.cpp); its records
    decode to the station's PI / PS through the reference's rds.cpp"""
    from sdrplusplus_b200 import lib as L
    exe = _adapter_exe(L, tmp_path)
    pi, name = 0xD123, "ADAPTER*"
    x, _ = _station(0, 31, bits=rds_group_bits(pi, name, 3))
    x = x[: (x.size // 40000) * 40000]
    src, dst = tmp_path / "iq.f32", tmp_path / "bits.u8"
    x.tofile(src)
    r = subprocess.run([exe, str(src), str(dst), str(FS), str(OFF)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
    nch, na, ns = (int(v) for v in r.stdout.split()[:3])
    got = np.fromfile(dst, np.uint8)
    assert nch == x.size // 40000 and na > 0 and ns == got.size > 0
    assert ref_oracle.rds_group_decode(got) == (pi, name)

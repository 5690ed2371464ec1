"""k_xd_tma's ÷4 epilogue: where a VFO's plan continues with the (4, 27) decimating FIR, stage 1 computes that stage's outputs
itself and the stage-1 outputs never reach memory (only the 26 the stage's history needs).  A chunk that needs the retune edge
kernel, any other input format, or a launch k_xd_tma declines stores the stage-1 outputs and runs k_dfir_reg<4,27> as before,
from the same history, so a VFO can switch between the two from one chunk to the next.

The GPU cases run RAW VFOs through test_gpu_stage1_f64.py's float64 reference and its a-priori bound, gain and edge checks,
from output 0: retunes every few chunks (fused and unfused chunks alternate), chunk lengths that move the ÷4 decimation phase,
and chunks too short to produce a ÷4 output between fused ones.  A profiler check holds the selection itself.
"""
import numpy as np
import pytest

from f64_ref import plan_of
from test_gpu_stage1_f64 import CASES, CF32, CS16, FS, PS10M, Run, _gate_parts, fir_offsets, sb  # noqa: F401

F2 = (4, 27)


def f2_chunks(r, variant=8):
    """Scheduler::run's choice of the ÷4 epilogue, per chunk and VFO of a Run (RAW VFOs, one prototype, default tail options:
    the (4, 27) stage runs in k_dfir_reg when not in stage 1, and every VFO of a chunk has the same taps): stage 1 takes
    k_xd_tma, the plan's second stage is the (4, 27) FIR with outputs this chunk, and no retune edge of the VFO reaches into
    the chunk (XdStage::plan: the newest boundary lies after the first output's window start)"""
    routes = r.routes(variant)
    if len(r.plan) < 3 or (r.plan[1][0], r.plan[1][1].size) != F2:
        return [[False] * len(co) for co in r.chunk_offs]
    offs1 = fir_offsets(r.sched, r.D)
    n1 = [(n - o + r.D - 1) // r.D if o < n else 0 for n, o in zip(r.sched, offs1)]
    offs2 = fir_offsets(n1, 4)
    nv = len(r.chunk_offs[0])
    bound = [None] * nv
    out, pos = [], 0
    for k, (route, n, a, b, o1, o2) in enumerate(zip(routes, r.sched, n1, n1, offs1, offs2)):
        for v in range(nv):
            if k > 0 and r.chunk_offs[k][v] != r.chunk_offs[k - 1][v]:
                bound[v] = pos
        n2 = (a - o2 + 3) // 4 if o2 < a else 0
        out.append([route == "tma" and n2 > 0 and not (bound[v] is not None and bound[v] > pos + o1 - (r.T - 1))
                    for v in range(nv)])
        pos += n
    return out


def test_f2_selection_mirror(oracle):
    """the bench plan at ratio 256, (32,143)(4,27)(2,69), runs fused on its TMA chunks; the TMA cases of the stage-1 suite whose
    plan continues with (4, 27) are the fused ones, and each case still reaches the build it is named after"""
    plan = plan_of(oracle, 256)
    assert [(D, h.size) for D, h in plan] == [(32, 143), (4, 27), (2, 69)]
    fused = set()
    for case in CASES:
        r = Run(oracle, case)
        routes = r.routes(case["opts"].get("s1", 8))
        assert case["build"] in routes
        f2 = f2_chunks(r, case["opts"].get("s1", 8))
        if any(any(c) for c in f2):
            fused.add(case["name"])
            assert all(rt == "tma" for rt, c in zip(routes, f2) if any(c))
    assert "tma_r256" in fused
    assert "retune_r256_two_short" in fused


def _custom_run(oracle, base, sched, chunk_offs, fmts=None):
    """a Run of test_gpu_stage1_f64.py with its own chunk schedule, per-chunk offsets and formats"""
    r = Run(oracle, next(c for c in CASES if c["name"] == base))
    r.case = dict(r.case, retune=None)
    r.sched = list(sched)
    r.chunk_offs = [list(o) for o in chunk_offs]
    r.fmts = list(fmts or [CF32] * len(sched))
    r.scales = [None] * len(sched)
    rng = np.random.default_rng(4242)
    r.chunks, vals = [], []
    for n, f in zip(r.sched, r.fmts):
        if f == CF32:
            c = rng.uniform(-1, 1, 2 * n).astype(np.float32)
            v = c.astype(np.float64)
        else:
            c = rng.integers(-32768, 32768, 2 * n).astype(np.int16)
            v = c.astype(np.float64) * float(np.float32(1.0 / 32768))
        r.chunks.append(c)
        vals.append(v)
    v = np.concatenate(vals)
    r.x = v[0::2] + 1j * v[1::2]
    return r


def _f2_case(oracle, name):
    if name == "retune_every_3":
        # one VFO retuned on the PS 10 grid every third chunk: the chunk after each retune runs the unfused path
        sched = [100003, 77777, 120001] * 5
        offs = [[(5e6, 15e6, -25e6)[k // 3 % 3]] for k in range(len(sched))]
        return _custom_run(oracle, "tma_r256", sched, offs)
    if name == "ragged_phase":
        # eight VFOs (+-5 ... +-35 MHz), lengths that are no multiple of 128 (the ÷4 phase moves), and a cs16 chunk between
        sched = [65537, 99999, 131075, 70001, 8 * 64 * 32 + 93, 123457, 100001]
        fmts = [CF32, CF32, CF32, CS16, CF32, CF32, CF32]
        return _custom_run(oracle, "tma_r256", sched, [PS10M] * len(sched), fmts)
    if name == "short_between":
        # chunks with no or one ÷4 output (no TMA launch) between fused ones: the next fused chunk's window starts in the
        # history the short ones carried
        sched = [150001, 40, 3, 0, 100, 150003, 33, 96, 150005, 60001]
        return _custom_run(oracle, "tma_r256", sched, [PS10M[:2]] * len(sched))
    raise KeyError(name)


F2_CASES = ["retune_every_3", "ragged_phase", "short_between"]


def test_f2_cases_route_both_ways(oracle):
    """each GPU case has fused chunks, and the retune and short cases also have chunks on the unfused path"""
    for name in F2_CASES:
        r = _f2_case(oracle, name)
        routes = r.routes(8)
        fused = [any(c) for c in f2_chunks(r)]
        assert any(fused), name
        # chunks with stage-1 outputs that take the unfused path: after the retunes, the cs16 chunk, the short chunks
        assert not all(f or rt is None for f, rt in zip(fused, routes)), name


def _run_chunks(sb, r):
    """test_gpu_stage1_f64.py's front-end run, with the TMA launches and the VFOs run fused counted per chunk"""
    fe = sb.FrontEnd(FS, max(max(r.sched), 1))
    try:
        outsr = FS / r.ratio
        nv = len(r.chunk_offs[0])
        ids = [fe.add_vfo(sb.VfoConfig.raw(r.chunk_offs[0][v], outsr, outsr)) for v in range(nv)]
        got = {vid: [] for vid in ids}
        tma, f2 = [], []
        prev = r.chunk_offs[0]
        for c, (n, f, co) in enumerate(zip(r.sched, r.fmts, r.chunk_offs)):
            for v, vid in enumerate(ids):
                if co[v] != prev[v]:
                    fe.set_vfo_offset(vid, co[v])
            prev = co
            if f != CF32:
                fe.set_ingest_scale(f, 0.0)
            t0, j0 = fe.stat("s1_tma_launches"), fe.stat("s1_f2_jobs")
            outs, _ = fe.process(r.chunks[c].view(np.complex64) if f == CF32 else r.chunks[c], f)
            tma.append(fe.stat("s1_tma_launches") - t0)
            f2.append(fe.stat("s1_f2_jobs") - j0)
            for vid in ids:
                got[vid].append(outs[vid])
    finally:
        fe.close()
    return [got[vid] for vid in ids], tma, f2


@pytest.mark.gpu
@pytest.mark.parametrize("name", F2_CASES)
def test_stage1_f2_vs_float64(sb, oracle, report, name):
    """the chunks run fused are the mirror's, and every output from output 0 is within the stage-1 suite's bound"""
    r = _f2_case(oracle, name)
    parts, tma, f2 = _run_chunks(sb, r)
    routes = r.routes(8)
    assert tma == [int(rt == "tma") for rt in routes], (tma, routes)
    assert f2 == [sum(c) for c in f2_chunks(r)], (f2, routes)
    worst, gains, gains_spec, edges = _gate_parts(oracle, r, parts, routes)
    report["stage1_f2_" + name] = {"max_err_over_bound": worst, "max_abs_g_minus_1": max(gains),
                                   "max_edge_over_p999": max(edges) if edges else None, "vfos": len(parts)}


def _kernel_launches(fn):
    """launches per kernel name while fn() runs (torch.profiler, CUDA activity: the library's kernels included)"""
    import collections
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return collections.Counter(e.name for e in prof.events())


@pytest.mark.gpu
def test_f2_replaces_dfir_4_27(sb):
    """the bench's VFO set (eight WFM VFOs at +-5 ... +-35 MHz, 100 MS/s, cf32): k_dfir_reg<4,27> runs once, for the retuned VFO
    on the retune chunk, and in no steady chunk before or after it"""
    fe = sb.FrontEnd(FS, 1 << 20)
    try:
        ids = [fe.add_vfo(sb.VfoConfig.wfm(o)) for o in PS10M]
        rng = np.random.default_rng(7)
        x = (rng.standard_normal(1 << 20) + 1j * rng.standard_normal(1 << 20)).astype(np.complex64) * np.float32(0.1)
        for _ in range(3):
            fe.process(x, CF32)

        tma, f2 = [], []

        def chunks():
            for k in range(6):
                if k == 3:
                    fe.set_vfo_offset(ids[0], 45e6)          # same PS 10 grid: the chunk still takes k_xd_tma
                t0, j0 = fe.stat("s1_tma_launches"), fe.stat("s1_f2_jobs")
                fe.process(x, CF32)
                tma.append(fe.stat("s1_tma_launches") - t0)
                f2.append(fe.stat("s1_f2_jobs") - j0)
        n = _kernel_launches(chunks)
        dfir = sum(v for k, v in n.items() if "k_dfir_reg<4, 27" in k)
        assert tma == [1] * 6, tma
        assert f2 == [8, 8, 8, 7, 8, 8], f2
        assert dfir == 1, (dfir, {k: v for k, v in n.items() if "k_" in k})
    finally:
        fe.close()

// sdrplusplus_b200/csrc/xd_tma.cuh -- stage 1 in filter-bank form (see xd_pfb.cuh for the identity) with the raw IQ
// tile brought in by the TMA engine ("s1" = 8, the default for cf32 chunks when the plan allows it; falls back to
// k_xd_pfb / k_xd_pipe).  Included by kernels.cu after xd_pfb.cuh.
//
// Replaces FrequencyXlator::process + the first DecimatingFIR of every VFO (frequency_xlator.h:43-50,
// decimating_fir.h:45-68) and the Splitter fan-out in front of them (splitter.h:46-61): the chunk is read from HBM once.
//
// Why a second filter-bank kernel: k_xd_pfb de-interleaves its tile by decimation phase with 8-byte cp.async copies,
// fills and computes in turn, and was latency-bound at a third of the HBM roof.  Here
//   * the chunk is described to the TMA engine as a 2-D tensor of "super-rows" (2*D samples = two decimation blocks);
//     one tile = NSEG*2 boxes of {16 samples, NR super-rows} with the 128-byte swizzle, issued by ONE thread, landing in
//     shared memory as [segment][block parity][row][128 B].  No thread touches the data on its way in.
//   * a persistent CTA per SM runs a ring of XT_STAGES tiles guarded by full / empty mbarriers: a producer warp keeps
//     the next tile in flight while MT/32 consumer warps (two per SM scheduler at D = 32) filter the one that landed.
//   * a lane owns ONE output and its window of QC blocks; a warp's 32 outputs are consecutive, lanes 0-15 take the even
//     ones and lanes 16-31 the odd ones (xt_lane_out), so that the eight lanes of a quarter warp read eight consecutive
//     rows of one parity region and every 16-byte window load is conflict-free through the hardware swizzle; a load feeds
//     two packed FMAs.  The real taps come from the kernel parameter block (constant bank), not from shared memory.
// Rows are cut at a 128-byte aligned origin org' <= org; the s = org - org' samples in front of a window are covered
// by s leading zero taps: the accumulator class of window position p is p mod PS, the tap it carries is k = p - s.
//
// ÷4 epilogue (XdJob::f2_out): when a VFO's next stage is the (4, 27) decimating FIR of the reference's plans, the kernel
// runs it too, so the stage-1 outputs (4x the bytes of the (4, 27) outputs) never make a round trip through memory.  The
// tile's stage-1 outputs are staged in the ring slot the tile arrived in (held until the epilogue has read it), behind
// the 26 outputs carried from the previous tile of the CTA's contiguous run; the first tile of a run recomputes them.
#pragma once
#include <cuda.h>

#define XT_STAGES NST        // ring depth, a template parameter of the kernel (2 or 3)
#define XT_MAXTAPS 512

struct XtGeom {
    float g[XT_MAXTAPS];      // signed real taps by window position p = q*D + r:  sigma^floor(k/PS) h[k], k = p - s
    long long jmin;           // block index (relative to the row origin) of the first tile's first output, even
    long long jend;           // one past the block index of the last output
    // CTA b owns the outputs of blocks [jmin + b*run, jmin + (b+1)*run) and walks them in consecutive tiles, so that the ÷4
    // epilogue carries its window from tile to tile.  With the epilogue, every CTA but the first starts `halo` outputs early
    // and only filters those: the ÷4 windows of its first outputs reach 26 stage-1 outputs back.  run, halo: multiples of 16,
    // so that every output keeps the coarse-phase grouping (PHW) it has in a launch without the epilogue.
    int run, halo;
    int f2;                   // some job has a ÷4 epilogue (XdJob::f2_out)
    int org;                  // sample index of row 0, phase 0 (chunk-relative; may be negative: history)
    int s;                    // leading zero taps
    int cj;                   // window of output m starts in block cj + m
    int rows_tma;             // super-rows the tensor map covers (all inside the chunk)
    int diag;                 // measurement only (option "s1_diag"): 1 = tiles are loaded but not filtered (what the TMA ring alone
                              // sustains), 2 = tiles are filtered but never loaded (what the consumer warps alone sustain); results are garbage
};

__device__ __forceinline__ void xt_mbar_init(unsigned bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void xt_mbar_wait(unsigned bar, unsigned parity) {
    asm volatile("{\n.reg .pred p;\nXT_WAIT_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@!p bra XT_WAIT_%=;\n}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void xt_mbar_arrive(unsigned bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void xt_mbar_expect(unsigned bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
// The raw chunk is read once and never again by this kernel: its lines are marked evict-first in L2, so that streaming 128 MiB
// through does not push out what the kernels of the other streams come back for (stage outputs, FFT work buffers).
__device__ __forceinline__ unsigned long long xt_policy_evict_first() {
    unsigned long long pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;\n" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void xt_tma_2d(unsigned dst, const CUtensorMap* tm, unsigned bar, int c0, int c1, unsigned long long pol) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;\n"
                 ::"r"(dst), "l"(reinterpret_cast<unsigned long long>(tm)), "r"(bar), "r"(c0), "r"(c1), "l"(pol) : "memory");
}

template <int LOGD, int QC, int MT>
struct XtLay {
    static constexpr int D = 1 << LOGD;
    static constexpr int NSEG = D / 16;                                  // 128-byte segments per decimation block
    static constexpr int NEED = (MT + QC + 2) / 2;                       // super-rows a tile reads
    static constexpr int NR = (NEED + 7) & ~7;                           // rows per region (whole swizzle atoms)
    static constexpr int REGION = NR * 128;
    static constexpr int STAGE = NSEG * 2 * REGION;
    static constexpr int NW = MT / 32;                                   // consumer warps, 32 outputs each
    static constexpr int NPH = MT / 16;                                  // coarse phases per job and tile (one per 16 outputs)
    // ÷4 epilogue: per job, the 26 carried stage-1 outputs and the MT of the tile, staged in the ring slot the tile came in,
    // one pad entry per 16 (a thread reads the 39-entry window of four ÷4 outputs; neighbouring threads are 16 apart)
    static constexpr int F2H = XD_F2_T - 1;
    static constexpr int F2P = (F2H + MT) + (F2H + MT) / 16 + 2;
    static_assert(B200_BATCH * F2P * 8 <= STAGE, "the epilogue's staging fits in one ring slot");
    static_assert(MT % 16 == 0, "whole groups of four ÷4 outputs per tile");
};
__device__ __forceinline__ int xt_f2_pad(int i) { return i + (i >> 4); }
// output of a consumer lane within its warp's 32: lanes 0-15 the even ones, lanes 16-31 the odd ones
__device__ __forceinline__ int xt_lane_out(int lane) { return ((lane & 15) << 1) | (lane >> 4); }

// decimation-phase pairs [RP0, RP1) of a tile -- they all lie in ONE 128-byte segment (8 pairs per segment), whose two parity
// regions start at sb -- into the PS class sums of a lane's output.  Every index is a compile-time constant: taps from the
// constant bank, accumulators in registers.  aoff[q]: the offset of the row of window block q in its parity region's segment.
template <int LOGD, int QC, int PS, int RP0, int RP1>
__device__ __forceinline__ void xt_accumulate(float2 (&S)[PS], const XtGeom& g, unsigned sb, const unsigned (&aoff)[QC]) {
    constexpr int D = 1 << LOGD;
    static_assert((RP0 >> 3) == ((RP1 - 1) >> 3), "one segment per call");
#pragma unroll
    for (int rp = RP0; rp < RP1; rp++) {
#pragma unroll
        for (int q = 0; q < QC; q++) {
            const unsigned addr = (sb + aoff[q]) ^ (unsigned)((rp & 7) << 4);    // sb: 1024-byte aligned
            float4 x;
            asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];\n" : "=f"(x.x), "=f"(x.y), "=f"(x.z), "=f"(x.w) : "r"(addr));
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int r = 2 * rp + e;
                const float2 xe = e ? make_float2(x.z, x.w) : make_float2(x.x, x.y);
                const float t = g.g[q * D + r];
                S[(q * D + r) % PS] = ffma2(make_float2(t, t), xe, S[(q * D + r) % PS]);
            }
        }
    }
}

// What bounds it is measured by switching the filter or the loads off (option "s1_diag", tools/s1_bounds.py).  Three
// restructurings of the consumer side are in the history (two groups of warps sharing a tile, ring slots of one 128-byte
// segment, filter warps handing their class sums to combine warps); none was faster on the GPU they were measured on.
// One output per lane (8 consumer warps instead of 4 at D = 32), on an H100 80GB HBM3 at 700 W: stage 1 alone 76.9 -> 68.7 us,
// bench `value` 109.3 -> 113.6 GS/s (medians of three alternated runs), same output bits.
// At most 96 registers per thread: at D = 32 the 288 threads take 27,648 of the SM's 65,536, which leaves room for a pass-1
// FFT CTA of 8 (36,864) beside it (tests/test_s1_sass_budget.py).
template <int LOGD, int QC, int PS, int MT, int NST>
__global__ void __maxnreg__(96)
k_xd_tma(const __grid_constant__ XdParams p, const __grid_constant__ XtGeom g, const __grid_constant__ CUtensorMap tm) {
    using Lay = XtLay<LOGD, QC, MT>;
    constexpr int D = Lay::D, NSEG = Lay::NSEG, NR = Lay::NR, REGION = Lay::REGION, STAGE = Lay::STAGE, NW = Lay::NW;
    constexpr int NSLOT = NST;                                           // ring depth: a slot is a whole tile (NSEG * 2 boxes)
    constexpr int SLOT = STAGE;
    extern __shared__ __align__(1024) unsigned char xt_smem[];
    // the dynamic window is 1024-byte aligned by the launch (checked on the host side: static shared memory is tiny)
    const unsigned sbase = ((unsigned)__cvta_generic_to_shared(xt_smem) + 1023u) & ~1023u;
    unsigned char* const gbase = xt_smem + (sbase - (unsigned)__cvta_generic_to_shared(xt_smem));
    float2* C = reinterpret_cast<float2*>(gbase + XT_STAGES * STAGE);    // [njobs][PS]  e^{j w_v ((b - s) mod PS)}
    float2* TL = C + (size_t)p.njobs * PS;                               // [njobs][16]  e^{j w_v D j}
    float2* PHW = TL + (size_t)p.njobs * 16;                             // [njobs][NPH] per tile: coarse phase of 16 outputs
    unsigned long long* bars = reinterpret_cast<unsigned long long*>(PHW + (size_t)p.njobs * Lay::NPH);
    const unsigned bar0 = (unsigned)__cvta_generic_to_shared(bars);     // full[s] = bar0 + 8 s, empty[s] = bar0 + 8 (NSLOT + s)
    float2* H = reinterpret_cast<float2*>(bars + 2 * NSLOT);              // [njobs][F2H] ÷4 epilogue: carried stage-1 outputs

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // this CTA's run of tiles (XtGeom::run)
    const long long own0 = g.jmin + (long long)blockIdx.x * g.run;
    const long long own1 = own0 + g.run < g.jend ? own0 + g.run : g.jend;
    const long long first = own0 - (blockIdx.x > 0 ? g.halo : 0);

    if (tid == 0) {
        for (int s = 0; s < NSLOT; s++) {
            xt_mbar_init(bar0 + 8 * s, 1);
            xt_mbar_init(bar0 + 8 * (NSLOT + s), NW);
        }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();
    // the producer starts the first tiles right away; the consumers build their tables under those loads
    if (warp < NW) {
        for (int idx = tid; idx < p.njobs * PS; idx += NW * 32) {
            const int v = idx / PS, b = idx - v * PS;
            int a = (b - g.s) % PS;
            if (a < 0) { a += PS; }
            C[idx] = phasor_u64(p.job[v].w * (unsigned long long)a);
        }
        for (int idx = tid; idx < p.njobs * 16; idx += NW * 32) {
            const int v = idx >> 4, j = idx & 15;
            TL[idx] = phasor_u64(p.job[v].w * (unsigned long long)((long long)j * D));
        }
        if (g.f2) {
            // the stage-1 outputs in front of the first tile: only the first CTA reads them (from the stage's history)
#pragma unroll 1
            for (int idx = tid; idx < p.njobs * Lay::F2H; idx += NW * 32) {
                const int v = idx / Lay::F2H, i = idx - v * Lay::F2H;
                const long long m = first - g.cj - Lay::F2H + i;
                H[idx] = (p.job[v].f2_out && m >= -Lay::F2H && m < 0) ? p.job[v].f2_hist[Lay::F2H + m] : make_float2(0.f, 0.f);
            }
        }
        asm volatile("bar.sync 1, %0;\n" ::"n"(NW * 32) : "memory");
    }

    // a tile is "fast" when every row it reads lies inside the tensor map; the few others (stream history in front of
    // the chunk, the ragged end) get their missing samples patched in by the consumer warps after the TMA boxes landed
    auto tile_fast = [&](long long J0) { return J0 >= 0 && (J0 >> 1) + Lay::NEED <= (long long)g.rows_tma; };

    if (warp == NW) {
        // ---------------- producer ----------------
        if (lane == 0 && !(g.diag & 2)) {
            const unsigned long long pol = xt_policy_evict_first();
            int it = 0;                                                  // slot steps issued so far
            for (long long J0 = first; J0 < own1; J0 += MT) {
                const int row0 = (int)(J0 >> 1);
                // every tile comes in through the TMA engine; rows outside the tensor (negative: stream history in front of
                // the chunk; past its last full super-row: the ragged end) arrive zero-filled and are patched by the consumers
                const int sl = it % NSLOT;
                const unsigned ph = (unsigned)((it / NSLOT) & 1);
                it++;
                xt_mbar_wait(bar0 + 8 * (NSLOT + sl), ph ^ 1u);
                const unsigned full = bar0 + 8 * sl;
                xt_mbar_expect(full, (unsigned)SLOT);
                const unsigned dst = sbase + (unsigned)(sl * SLOT);
#pragma unroll
                for (int sg = 0; sg < NSEG; sg++) {
#pragma unroll
                    for (int par = 0; par < 2; par++) {
                        xt_tma_2d(dst + (unsigned)((sg * 2 + par) * REGION), &tm, full, par * 2 * D + sg * 32, row0, pol);
                    }
                }
            }
        }
        return;
    }

    // ---------------- consumers ----------------
    const int jw = xt_lane_out(lane);
    const int jl = warp * 32 + jw;                  // this lane's output within the tile
    // window block jl + q: parity region (jl + q) & 1, row (jl + q) >> 1, its 16-byte chunks swizzled by row & 7
    unsigned aoff[QC];
#pragma unroll
    for (int q = 0; q < QC; q++) {
        const unsigned row = (unsigned)((jl + q) >> 1);
        aoff[q] = (unsigned)(((jl + q) & 1) * REGION) + row * 128u + ((row & 7u) << 4);
    }
    int it = 0;                                     // tiles consumed so far (the producer's sequence)
    for (long long J0 = first; J0 < own1; J0 += MT) {
        // coarse phases of this warp's 32 outputs: entry (job, 2 warp + i) = phase at output 32 warp + 16 i, drift-centred
        {
            for (int e = lane; e < p.njobs * 2; e += 32) {
                const int vv = e >> 1, i = e & 1;
                const XdJob& Jv = p.job[vv];
                const int a0 = Jv.offset - (Jv.T - 1);
                const long long im0 = (long long)a0 + (J0 + warp * 32 + i * 16 - (long long)g.cj) * D;
                unsigned long long dr = Jv.w * (unsigned long long)PS;
                if (p.pfb_sigma < 0) { dr -= 0x8000000000000000ULL; }
                const long long corr = (long long)dr * (long long)(Jv.T / (2 * PS));
                PHW[vv * Lay::NPH + 2 * warp + i] = phasor_u64(Jv.phase0 + Jv.w * (unsigned long long)im0 + (unsigned long long)corr);
            }
        }
        const bool fast = tile_fast(J0);

        // ---- accumulate: D/2 phase pairs x QC window blocks, PS classes per lane, segment by segment ----
        float2 S[PS];
#pragma unroll
        for (int a = 0; a < PS; a++) { S[a] = make_float2(0.f, 0.f); }
        const int sl = it % NSLOT;
        const unsigned ph = (unsigned)((it / NSLOT) & 1);
        it++;
        if (!(g.diag & 2)) { xt_mbar_wait(bar0 + 8 * sl, ph); }
        const unsigned sb = sbase + (unsigned)(sl * SLOT);
        if (!fast && !g.diag) {
            // patch what the tensor map does not cover: samples before the chunk (from the carried raw history) and the
            // samples of the last, partial super-row.  A few hundred at most, once or twice per launch.
            const long long ibase = J0 * D + g.org;
            unsigned char* stg = gbase + sl * SLOT;
            constexpr int NSAMP = (MT + QC + 1) * D;
            const long long tensor_end = (long long)g.org + (long long)g.rows_tma * (2 * D);
            // the tensor's row 0 starts at sample g.org: everything of this tile in front of it was zero-filled -- stream
            // history (index < 0) AND the first g.org samples of the chunk
            const long long front = (long long)g.org - ibase;
            const int head = (int)(front > 0 ? (front < NSAMP ? front : NSAMP) : 0);
            long long t0 = tensor_end - ibase, t1 = (long long)p.count - ibase;
            if (t0 < head) { t0 = head; }
            if (t1 > NSAMP) { t1 = NSAMP; }
            auto patch = [&](int idx) {
                const float2 v = load_x<FMT_CF32>(p, ibase + idx);
                const int j = idx >> LOGD, r = idx & (D - 1), row = j >> 1;
                const int off = ((r >> 4) * 2 + (j & 1)) * REGION + row * 128 + ((((r >> 1) & 7) ^ (row & 7)) << 4) + (r & 1) * 8;
                *reinterpret_cast<float2*>(stg + off) = v;
            };
            for (int idx = tid; idx < head; idx += NW * 32) { patch(idx); }
            for (long long idx = t0 + tid; idx < t1; idx += NW * 32) { patch((int)idx); }
            asm volatile("bar.sync 1, %0;\n" ::"n"(NW * 32) : "memory");
        }
        if (!(g.diag & 1)) {
            xt_accumulate<LOGD, QC, PS, 0, 8>(S, g, sb, aoff);
            xt_accumulate<LOGD, QC, PS, 8, 16>(S, g, sb + 2 * REGION, aoff);
            if constexpr (NSEG == 4) {
                xt_accumulate<LOGD, QC, PS, 16, 24>(S, g, sb + 4 * REGION, aoff);
                xt_accumulate<LOGD, QC, PS, 24, 32>(S, g, sb + 6 * REGION, aoff);
            }
        }
        static_assert(NSEG == 2 || NSEG == 4, "D = 32 or 64");
        __syncwarp();
        if (!g.f2) {
            // the tile is consumed: hand it back to the producer before the (register-only) combination.  Patched samples were
            // written through the generic proxy: order them before the TMA engine's next write into the slot
            if (!fast) { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); __syncwarp(); }
            if (lane == 0 && !(g.diag & 2)) { xt_mbar_arrive(bar0 + 8 * (NSLOT + sl)); }
            if (g.diag & 1) { continue; }
        }
        else {
            // the slot becomes the epilogue's staging once every warp has read its part of the tile
            asm volatile("bar.sync 1, %0;\n" ::"n"(NW * 32) : "memory");
        }
        float2* const stg = reinterpret_cast<float2*>(gbase + sl * SLOT);
        if (g.f2) {
#pragma unroll 1
            for (int idx = tid; idx < p.njobs * Lay::F2H; idx += NW * 32) {
                const int v = idx / Lay::F2H, i = idx - v * Lay::F2H;
                stg[v * Lay::F2P + xt_f2_pad(i)] = H[idx];
            }
        }

        // ---- combine per slot (a VFO, or a +f / -f pair sharing A = sum cos*S and B = sum sin*S), rotate, store ----
        const long long m0 = J0 + jl - (long long)g.cj;
        const int nout = p.job[0].n_out;                       // every job of a filter-bank launch has the same length
        // outputs of this CTA's run (the halo in front of it and the tail past its end belong to its neighbours)
        const bool ok = J0 + jl >= own0 && J0 + jl < own1 && m0 >= 0 && m0 < nout;
        const int ih = 2 * warp + (jw >> 4), il = jw & 15;
        // stage-1 output y of job v: to the ÷4 staging, and to `out` where the next stage's history needs it
        auto put = [&](int v, float2 y) {
            const XdJob& Jv = p.job[v];
            if (g.f2 && Jv.f2_out) {
                // m0 < 0 only in the first CTA's first tile, when the first output's block is odd: the value of the history
                stg[v * Lay::F2P + xt_f2_pad(Lay::F2H + jl)] = m0 >= 0 ? y : Jv.f2_hist[Lay::F2H + m0];
                if (ok && m0 >= nout - Lay::F2H) { Jv.out[m0] = y; }
            }
            else if (ok) { Jv.out[m0] = y; }
        };
        for (int sv = 0; sv < p.nslots; sv++) {
            const int ja = p.slot_a[sv], jb = p.slot_b[sv];
            float2 A = make_float2(0.f, 0.f), B = A;
            const float2* cv = C + ja * PS;
#pragma unroll
            for (int a = 0; a < PS; a++) {
                const float2 c = cv[a];
                A = ffma2(make_float2(c.x, c.x), S[a], A);
                B = ffma2(make_float2(c.y, c.y), S[a], B);
            }
            put(ja, cmulf(make_float2(A.x - B.y, A.y + B.x), cmulf(PHW[ja * Lay::NPH + ih], TL[ja * 16 + il])));
            if (jb >= 0) {                                     // conjugate coefficients
                put(jb, cmulf(make_float2(A.x + B.y, A.y - B.x), cmulf(PHW[jb * Lay::NPH + ih], TL[jb * 16 + il])));
            }
        }
        if (g.f2) {
            asm volatile("bar.sync 1, %0;\n" ::"n"(NW * 32) : "memory");
            // ---- ÷4 epilogue: a thread computes four consecutive outputs of one job from a 39-entry window in registers,
            //      with the tap order and arithmetic of k_dfir_reg ----
            constexpr int NG = MT / 16;                        // groups of four outputs per job and tile
            const long long t0 = J0 - g.cj;                    // stage-1 index of the tile's first output (staging entry F2H)
#pragma unroll 1
            for (int task = tid; task < p.njobs * NG; task += NW * 32) {
                const int v = task / NG, gi = task - v * NG;
                const XdJob& Jv = p.job[v];
                if (!Jv.f2_out) { continue; }
                // first output whose window ends inside the tile: f2_off + 4 j >= t0
                const long long d = t0 - Jv.f2_off;
                const long long jt0 = d >= 0 ? (d + 3) / 4 : -((-d) / 4);
                const int b = (int)(Jv.f2_off + 4 * jt0 - t0) + 16 * gi;
                const float2* w = stg + v * Lay::F2P;
                float2 x[3 * XD_F2_D + XD_F2_T];
#pragma unroll
                for (int i = 0; i < 3 * XD_F2_D + XD_F2_T; i++) { x[i] = w[xt_f2_pad(b + i)]; }
                float2 acc[4];
#pragma unroll
                for (int i = 0; i < 4; i++) { acc[i] = make_float2(0.0f, 0.0f); }
#pragma unroll
                for (int k = 0; k < XD_F2_T; k++) {
                    const float h = p.f2_taps[k];
#pragma unroll
                    for (int i = 0; i < 4; i++) { acc[i] = ffma2(make_float2(h, h), x[i * XD_F2_D + k], acc[i]); }
                }
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const long long j = jt0 + 4 * gi + i;
                    const long long J = Jv.f2_off + XD_F2_D * j + g.cj;   // block of the window's last stage-1 output
                    if (j >= 0 && j < Jv.f2_n && J >= own0 && J < own1) { Jv.f2_out[j] = acc[i]; }
                }
            }
            // the last F2H stage-1 outputs of the tile are the window's start in the next one
#pragma unroll 1
            for (int idx = tid; idx < p.njobs * Lay::F2H; idx += NW * 32) {
                const int v = idx / Lay::F2H, i = idx - v * Lay::F2H;
                H[idx] = stg[v * Lay::F2P + xt_f2_pad(MT + i)];
            }
            // the staging is read: the slot goes back to the producer, its generic-proxy writes ordered before the next TMA write
            asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
            __syncwarp();
            if (lane == 0) { xt_mbar_arrive(bar0 + 8 * (NSLOT + sl)); }
        }
        __syncwarp();                                          // PHW is rewritten for the next tile
    }
}

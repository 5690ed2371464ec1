// sdrplusplus_b200/csrc/dfir_reg.cuh -- the short decimating FIR stages behind stage 1 of a VFO (stages 2..k of
// PowerDecimator::process, power_decimator.h:58-65; DecimatingFIR<complex_t,float>::process, decimating_fir.h:45-68)
// with the whole input window of a thread in REGISTERS.  Included by kernels.cu.
//
// Every non-first stage of the reference's decimation plans is one of six (decimation, taps) pairs
// (decim/plans.h:24-140: (2,69) (2,12) (4,27) (8,54) (8,44) (8,36)), so the kernel is instantiated per pair: a thread
// produces R consecutive outputs, loads the (R-1)*D + T samples they read ONCE with 16-byte loads (staged once per CTA in shared memory by
// coalesced 16-byte loads -- the stage-1 output was just written: L2 hits -- in a padded layout that makes every thread's
// window loads conflict-free), and runs T*R fully unrolled complex-by-real FMA pairs whose tap
// operand comes from the kernel parameter block (constant bank -> uniform register): one barrier, no address arithmetic in the loop.  This replaces the fused tail's first stages, where the same work was LSU-bound.
//
// Index convention as in kernels.cuh (FirJob): out[m] = sum_k taps[k] * in[offset + m*D + k], `in` = oldest history sample.
#pragma once

template <int D, int T, int R>
struct DfrGeom {
    static constexpr int S = R * D / 2;                       // 16-byte pairs between the windows of neighbouring threads
    static constexpr int LS = (S == 1) ? 0 : (S == 2) ? 1 : (S == 4) ? 2 : (S == 8) ? 3 : (S == 16) ? 4 : (S == 32) ? 5 : 6;
    static_assert((1 << LS) == S, "R*D/2 must be a power of two");
    static constexpr int NS = (R - 1) * D + T;                // samples the R outputs of a thread read
    static constexpr int NV = (NS + 2) / 2;                   // pairs per thread (one spare for an odd start)
    static constexpr int NPT = (DFR_THREADS - 1) * S + NV;    // pairs per CTA tile
    static constexpr int SMEM = (NPT + (NPT >> LS) + 2) * 16; // one pad pair per S pairs: thread stride S + 1 (odd) -> conflict-free
};

template <int D, int T, int R>
__global__ void __launch_bounds__(DFR_THREADS) k_dfir_reg(const __grid_constant__ DfrParams p) {
    using G = DfrGeom<D, T, R>;
    extern __shared__ __align__(16) float4 dfr_sm[];
    const FirJob& J = p.job[blockIdx.y];
    pdl_trigger();
    const int mt = blockIdx.x * DFR_THREADS * R;              // first output of this CTA
    if (mt >= J.n_out) { return; }
    const long long first = (long long)J.offset + (long long)mt * D;
    const int sh = (int)(first & 1);                          // odd start: the tile begins at the even sample below
    // ---- the tile: coalesced 16-byte loads, padded layout ----
    {
        const float4* __restrict__ src = reinterpret_cast<const float4*>(J.in + (first - sh));
        // pairs past the data of the last tile stay inside the stage buffer (Scheduler::STAGE_SPARE) as long as they
        // belong to an output that exists; beyond that they are not read
        const long long last_out = (long long)J.n_out - 1 - mt;
        const int need = (int)((last_out < (long long)DFR_THREADS * R - 1 ? last_out : (long long)DFR_THREADS * R - 1) * D + T + 1 + sh + 1) / 2;
        // every load of the tile in flight at once (the fill is one round trip to L2 / HBM, not NPT / 128 of them)
        constexpr int NIT = (G::NPT + DFR_THREADS - 1) / DFR_THREADS;
        float4 t[NIT];
        pdl_wait();
#pragma unroll
        for (int u = 0; u < NIT; u++) {
            const int i = threadIdx.x + u * DFR_THREADS;
            t[u] = (i < G::NPT && i < need) ? __ldcg(src + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < NIT; u++) {
            const int i = threadIdx.x + u * DFR_THREADS;
            if (i < G::NPT) { dfr_sm[i + (i >> G::LS)] = t[u]; }
        }
    }
    __syncthreads();
    const int m0 = mt + threadIdx.x * R;
    if (m0 >= J.n_out) { return; }
    const float4* win = dfr_sm + threadIdx.x * (G::S + 1);
    float2 x[2 * G::NV];
#pragma unroll
    for (int v = 0; v < G::NV; v++) {
        const float4 t = win[v + (v >> G::LS)];
        x[2 * v] = make_float2(t.x, t.y);
        x[2 * v + 1] = make_float2(t.z, t.w);
    }
    float2 acc[R];
#pragma unroll
    for (int i = 0; i < R; i++) { acc[i] = make_float2(0.0f, 0.0f); }
    if (sh == 0) {
#pragma unroll
        for (int k = 0; k < T; k++) {
            const float h = p.taps[k];
#pragma unroll
            for (int i = 0; i < R; i++) { acc[i] = ffma2(make_float2(h, h), x[i * D + k], acc[i]); }
        }
    }
    else {
#pragma unroll
        for (int k = 0; k < T; k++) {
            const float h = p.taps[k];
#pragma unroll
            for (int i = 0; i < R; i++) { acc[i] = ffma2(make_float2(h, h), x[i * D + k + 1], acc[i]); }
        }
    }
#pragma unroll
    for (int i = 0; i < R; i++) {
        if (m0 + i < J.n_out) { J.out[m0 + i] = acc[i]; }
    }
}

template <int D, int T, int R>
static cudaError_t launch_dfir_reg_t(const DfrParams& p, const KernelOpts& o, cudaStream_t s) {
    dim3 grid((unsigned)((p.max_out + DFR_THREADS * R - 1) / (DFR_THREADS * R)), (unsigned)p.njobs);
    return launch_chain(k_dfir_reg<D, T, R>, grid, dim3(DFR_THREADS), DfrGeom<D, T, R>::SMEM, o, s, p);
}
// true when (D, T) is one of the plan stages the kernel is built for
bool dfir_reg_supported(int D, int T) {
    return (D == 2 && (T == 69 || T == 12)) || (D == 4 && T == 27) || (D == 8 && (T == 54 || T == 44 || T == 36));
}
// every job: same D and T (p.taps holds the common taps).  The reads run up to one sample past the last one an output
// needs (16-byte granularity): stage buffers carry 8 spare samples (Stage::alloc_in).
cudaError_t launch_dfir_reg(const DfrParams& p, int D, int T, const KernelOpts& o, cudaStream_t s) {
    if (p.njobs <= 0 || p.max_out <= 0) { return cudaSuccess; }
    if (D == 4 && T == 27) { return launch_dfir_reg_t<4, 27, 8>(p, o, s); }
    if (D == 2 && T == 69) { return launch_dfir_reg_t<2, 69, 4>(p, o, s); }
    if (D == 2 && T == 12) { return launch_dfir_reg_t<2, 12, 8>(p, o, s); }
    if (D == 8 && T == 54) { return launch_dfir_reg_t<8, 54, 4>(p, o, s); }
    if (D == 8 && T == 44) { return launch_dfir_reg_t<8, 44, 4>(p, o, s); }
    if (D == 8 && T == 36) { return launch_dfir_reg_t<8, 36, 4>(p, o, s); }
    return cudaErrorInvalidValue;
}

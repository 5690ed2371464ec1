// sdrplusplus_b200/csrc/rds.cuh -- RDSDemod, the symbol-rate half of the RDS path (decoder_modules/radio/src/rds_demod.h:64-73),
// behind BroadcastFM's rdsOut (complex at 5 kS/s).  Included by kernels.cu.
//
//   loop::FastAGC<complex_t>(1, 1e6, 0.1)        fast_agc.h:61-80          sequential (the gain is fed back every sample)
//   loop::Costas<2>(0.005)                       costas.h:18-24,28-33      sequential (phase control loop, phase_control_loop.h:58-85)
//   filter::FIR<complex_t,complex_t>             fir.h:74-76               190 complex taps (taps::bandPass<complex_t>(0, 2375, 100, 5000)): parallel
//   loop::Costas<2>(0.01, f = 2 pi 1187.5 / 5000 +/- 10 %)                 sequential
//   ComplexToReal -> clock_recovery::MM<float>   mm.h:94-147               sequential, data-dependent output count (128 x 8 interpolator)
//   BinarySlicer -> DifferentialDecoder(2)       binary_slicer.h:14-19, differential_decoder.h:39-44
//
// One CTA per RDS stream.  The stream is cut in tiles of RDS_TILE samples that live in shared memory from the AGC to the
// clock recovery: every block above is a streaming recurrence whose whole state is carried (gain, loop phases and
// frequencies, the band-pass delay line, MM's sample offset and 7-sample tail), so tiling is the reference's own chunking
// and changes nothing.  Thread 0 walks the three recurrences with the reference's fp32 statements (explicit roundings, no
// contraction: which interpolator phase and which sample the clock recovery picks are decisions of the fed-back value); all
// threads run the band-pass, two interleaved partial sums like the generic complex dot product of the oracle's leaf layer.
// 5 kS/s per stream: this is not a throughput kernel (a 16 Mi-sample chunk of a 100 MS/s stream carries 839 samples of it).
// Callers: the stand-alone b200_rds_demod (one job per call) and the front end's B200_DEMOD_WFM_RDS_BITS VFOs (up to B200_BATCH
// jobs per launch).  Each job writes b200_rds_symbol records and its symbol count to a count slot of its own.
#pragma once

#define RDS_TILE 1024
#define RDS_THREADS 256

__device__ __forceinline__ void rds_pcl_advance(float& phase, float& freq, float err, float alpha, float beta, float fmin, float fmax) {
    freq = __fadd_rn(freq, __fmul_rn(beta, err));                        // PhaseControlLoop::advance
    if (freq > fmax) { freq = fmax; }
    else if (freq < fmin) { freq = fmin; }
    phase = __fadd_rn(phase, __fadd_rn(freq, __fmul_rn(alpha, err)));
}
__device__ __forceinline__ void rds_clamp_phase(float& phase) {
    const float pi = FL_M_PI_REF, two_pi = __fsub_rn(FL_M_PI_REF, -FL_M_PI_REF);
    while (phase > pi) { phase = __fsub_rn(phase, two_pi); }
    while (phase < -pi) { phase = __fadd_rn(phase, two_pi); }
}
// Costas<2>::process on one sample: out = in * phasor(-phase); advance(clamp(out.re * out.im))
__device__ __forceinline__ float2 rds_costas(float2 v, float& phase, float& freq, float alpha, float beta, float fmin, float fmax) {
    float sn, cs;
    sincosf(-phase, &sn, &cs);
    float2 o;
    o.x = __fsub_rn(__fmul_rn(v.x, cs), __fmul_rn(v.y, sn));             // complex_t * complex_t (types.h:23-25)
    o.y = __fadd_rn(__fmul_rn(v.y, cs), __fmul_rn(v.x, sn));
    float err = __fmul_rn(o.x, o.y);
    if (err < -1.0f) { err = -1.0f; }
    if (err > 1.0f) { err = 1.0f; }
    rds_pcl_advance(phase, freq, err, alpha, beta, fmin, fmax);
    rds_clamp_phase(phase);
    return o;
}

__global__ void __launch_bounds__(RDS_THREADS) k_rds_demod(const __grid_constant__ RdsParams p) {
    const RdsJob& J = p.job[blockIdx.x];
    __shared__ float2 c1[RDS_MAXTAPS - 1 + RDS_TILE];     // [band-pass history | Costas 1 output of the tile]
    __shared__ float2 fb[RDS_TILE];                        // tile in, then band-pass output
    __shared__ float mb[RDS_MM_TAPS - 1 + RDS_TILE];       // [MM tail | real part behind Costas 2]
    __shared__ float2 taps[RDS_MAXTAPS];
    __shared__ float bank[RDS_MM_PHASES * RDS_MM_TAPS];
    const int tid = threadIdx.x, NT = J.ntaps, H = NT - 1;
    RdsState* S = J.state;
    for (int k = tid; k < NT; k += RDS_THREADS) { taps[k] = J.taps[k]; }
    for (int k = tid; k < RDS_MM_PHASES * RDS_MM_TAPS; k += RDS_THREADS) { bank[k] = J.bank[k]; }
    for (int k = tid; k < H; k += RDS_THREADS) { c1[k] = S->c1_hist[k]; }
    if (tid < RDS_MM_TAPS - 1) { mb[tid] = S->m_hist[tid]; }
    // thread 0 owns the scalar state
    float gain = 0.f, p1 = 0.f, f1 = 0.f, p2 = 0.f, f2 = 0.f, mph = 0.f, mfr = 0.f, last = 0.f;
    int offset = 0, dlast = 0, nout = 0;
    if (tid == 0) {
        gain = S->gain; p1 = S->c1_phase; f1 = S->c1_freq; p2 = S->c2_phase; f2 = S->c2_freq;
        mph = S->mm_phase; mfr = S->mm_freq; last = S->last_out; offset = S->offset; dlast = S->diff_last;
    }
    __syncthreads();
    for (int t0 = 0; t0 < J.n; t0 += RDS_TILE) {
        const int tn = min(RDS_TILE, J.n - t0);
        for (int i = tid; i < tn; i += RDS_THREADS) { fb[i] = J.in[t0 + i]; }
        __syncthreads();
        if (tid == 0) {
            for (int i = 0; i < tn; i++) {
                // FastAGC<complex_t>::process
                float2 v = fb[i];
                v.x = __fmul_rn(v.x, gain);
                v.y = __fmul_rn(v.y, gain);
                const float amp = __fsqrt_rn(__fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)));
                gain = __fadd_rn(gain, __fmul_rn(__fsub_rn(J.set_point, amp), J.rate));
                if (gain > J.max_gain) { gain = J.max_gain; }
                c1[H + i] = rds_costas(v, p1, f1, J.c1_alpha, J.c1_beta, J.c1_min, J.c1_max);
            }
        }
        __syncthreads();
        // band-pass: out[i] = sum_k taps[k] * c1[i + k]  (window ends at the sample itself: history in front)
        for (int i = tid; i < tn; i += RDS_THREADS) {
            float s0r = 0.f, s0i = 0.f, s1r = 0.f, s1i = 0.f;
            const int half = NT >> 1;
            for (int k = 0; k < half; k++) {
                const float2 a0 = c1[i + 2 * k], b0 = taps[2 * k], a1 = c1[i + 2 * k + 1], b1 = taps[2 * k + 1];
                s0r = __fadd_rn(s0r, __fsub_rn(__fmul_rn(a0.x, b0.x), __fmul_rn(a0.y, b0.y)));
                s0i = __fadd_rn(s0i, __fadd_rn(__fmul_rn(a0.x, b0.y), __fmul_rn(a0.y, b0.x)));
                s1r = __fadd_rn(s1r, __fsub_rn(__fmul_rn(a1.x, b1.x), __fmul_rn(a1.y, b1.y)));
                s1i = __fadd_rn(s1i, __fadd_rn(__fmul_rn(a1.x, b1.y), __fmul_rn(a1.y, b1.x)));
            }
            float rr = __fadd_rn(s0r, s1r), ri = __fadd_rn(s0i, s1i);
            if (NT & 1) {
                const float2 a = c1[i + NT - 1], b = taps[NT - 1];
                rr = __fadd_rn(rr, __fsub_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)));
                ri = __fadd_rn(ri, __fadd_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x)));
            }
            fb[i] = make_float2(rr, ri);
        }
        __syncthreads();
        if (tid == 0) {
            for (int i = 0; i < tn; i++) {
                mb[RDS_MM_TAPS - 1 + i] = rds_costas(fb[i], p2, f2, J.c2_alpha, J.c2_beta, J.c2_min, J.c2_max).x;     // ComplexToReal
            }
            // MM<float>::process on this tile (count = tn)
            // (a non-finite input would stall the reference's loop for good; here the symbol capacity ends it and the host
            // reports the overflow)
            while (offset < tn && nout <= J.out_cap) {
                int ph = (int)floorf(__fmul_rn(mph, (float)RDS_MM_PHASES));
                ph = ph < 0 ? 0 : (ph > RDS_MM_PHASES - 1 ? RDS_MM_PHASES - 1 : ph);
                float acc = 0.f;
#pragma unroll
                for (int k = 0; k < RDS_MM_TAPS; k++) { acc = __fadd_rn(acc, __fmul_rn(mb[offset + k], bank[ph * RDS_MM_TAPS + k])); }
                const int bit = acc > 0.0f ? 1 : 0;
                if (nout < J.out_cap) {
                    J.out[nout] = RdsSym{ acc, (unsigned int)((bit - dlast + 2) % 2) };    // slicer + differential decoder
                }
                dlast = bit;
                nout++;
                const float sl = last > 0.0f ? 1.0f : -1.0f, so = acc > 0.0f ? 1.0f : -1.0f;
                float err = __fsub_rn(__fmul_rn(sl, acc), __fmul_rn(last, so));
                last = acc;
                if (err > 1.0f) { err = 1.0f; }
                if (err < -1.0f) { err = -1.0f; }
                rds_pcl_advance(mph, mfr, err, J.mm_alpha, J.mm_beta, J.mm_min, J.mm_max);
                const float delta = floorf(mph);
                offset = (int)__fadd_rn((float)offset, delta);
                mph = __fsub_rn(mph, delta);
            }
            offset -= tn;
        }
        __syncthreads();
        // delay lines: the last H (7) samples of [history | tile] move to the front (memmove: read, barrier, write)
        float2 hv[(RDS_MAXTAPS - 1 + RDS_THREADS - 1) / RDS_THREADS];
#pragma unroll
        for (int r = 0; r < (RDS_MAXTAPS - 1 + RDS_THREADS - 1) / RDS_THREADS; r++) {
            const int k = tid + r * RDS_THREADS;
            if (k < H) { hv[r] = c1[tn + k]; }
        }
        float mv = 0.f;
        if (tid < RDS_MM_TAPS - 1) { mv = mb[tn + tid]; }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < (RDS_MAXTAPS - 1 + RDS_THREADS - 1) / RDS_THREADS; r++) {
            const int k = tid + r * RDS_THREADS;
            if (k < H) { c1[k] = hv[r]; }
        }
        if (tid < RDS_MM_TAPS - 1) { mb[tid] = mv; }
        __syncthreads();
    }
    for (int k = tid; k < H; k += RDS_THREADS) { S->c1_hist[k] = c1[k]; }
    if (tid < RDS_MM_TAPS - 1) { S->m_hist[tid] = mb[tid]; }
    if (tid == 0) {
        S->gain = gain; S->c1_phase = p1; S->c1_freq = f1; S->c2_phase = p2; S->c2_freq = f2;
        S->mm_phase = mph; S->mm_freq = mfr; S->last_out = last; S->offset = offset; S->diff_last = dlast;
        *J.count = nout;
    }
}

cudaError_t launch_rds_demod(const RdsParams& p, cudaStream_t s) {
    if (p.njobs <= 0) { return cudaSuccess; }
    k_rds_demod<<<p.njobs, RDS_THREADS, 0, s>>>(p);
    return cudaGetLastError();
}

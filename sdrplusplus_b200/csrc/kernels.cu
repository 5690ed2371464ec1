// sdrplusplus_b200/csrc/kernels.cu -- hand-written sm_90a kernels of the SDR++ streaming DSP hot path.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 (see __graft_entry__.build()).
// No cuFFT / cuBLAS / Thrust on any path; tensor cores are not used (no dense contraction here).
//
// Kernel inventory (reference call site each one replaces):
//   k_xd_tile / k_xd_simple   FrequencyXlator::process + first DecimatingFIR, all VFOs share one IQ tile
//                             (frequency_xlator.h:43-50, decimating_fir.h:45-68, splitter.h:46-61)
//   k_fir_c                   DecimatingFIR / FIR<complex_t,float>::process (decimating_fir.h:45-68, fir.h:62-83)
//   k_poly                    PolyphaseResampler::process (polyphase_resampler.h:69-99)
//   k_quad                    Quadrature::process (quadrature.h:39-46)
//   k_fir_r                   FIR<float,float>::process + LRToStereo/MonoToStereo (fir.h:69, l_r_to_stereo.h:21)
//   k_seq                     AM: AGC/magnitude/DCBlocker (am.h:101-133, agc.h:70-110, dc_blocker.h:54-60)
//                             SSB: second FrequencyXlator + ComplexToReal + AGC (ssb.h:77-92)
//   k_carry                   delay-line memmove at the end of process() (fir.h:80, decimating_fir.h:65)
//   k_fft_single / k_fft_p1 / k_fft_p2
//                             IQFrontEnd::handler: window multiply, forward FFT, 10log10(|X/N|^2)
//                             (iq_frontend.cpp:248-267)
//   k_zoom_hold               doZoom + peak hold (waterfall.cpp:65-90, 935-939)
#include "kernels.cuh"
#include <unordered_map>
#include <mutex>
#include <math.h>
#include <string.h>
#include <algorithm>

// ------------------------------------------------------------------------------------------------
// helpers
// ------------------------------------------------------------------------------------------------
// sc = 1 / scalar of volk_16i_s32f_convert_32f / volk_8i_s32f_convert_32f: 1/32768 for file_source's int16
// (file_source main.cpp:162), 1/128 for int8, scaler/32768 resp. scaler/128 for a compressed-stream packet
// (sample_stream_decompressor.h:24-33); unused for cf32
template <int FMT>
__device__ __forceinline__ float2 load_iq(const void* __restrict__ p, long long i, float sc) {
    if (FMT == FMT_CF32) {
        return __ldg(reinterpret_cast<const float2*>(p) + i);
    }
    else if (FMT == FMT_CS16) {
        short2 v = __ldg(reinterpret_cast<const short2*>(p) + i);
        return make_float2((float)v.x * sc, (float)v.y * sc);
    }
    else {
        char2 v = __ldg(reinterpret_cast<const char2*>(p) + i);
        return make_float2((float)v.x * sc, (float)v.y * sc);
    }
}

// sample at chunk-relative index i: history for i < 0, zero outside [-hist_len, count)
template <int FMT>
__device__ __forceinline__ float2 load_x(const XdParams& p, long long i) {
    if (i >= 0) {
        if (i < p.count) { return load_iq<FMT>(p.in, i, p.in_scale); }
        return make_float2(0.0f, 0.0f);
    }
    long long h = (long long)p.hist_len + i;
    if (h >= 0) { return __ldg(p.hist + h); }
    return make_float2(0.0f, 0.0f);
}

// e^{j*2*pi*phase/2^64}: phase is exact u64 "turns"; top 32 bits -> float in [-1,1) half-turns -> sincospi
__device__ __forceinline__ float2 phasor_u64(unsigned long long phase) {
    int hi = (int)(phase >> 32);
    float t = (float)hi * (1.0f / 2147483648.0f);
    float s, c;
    sincospif(t, &s, &c);
    return make_float2(c, s);
}

// RealToComplex + FrequencyXlator of BroadcastFM's RDS branch (broadcast_fm.h:165-170) for sample i of a chunk whose first
// sample has phase phase0: k_rxl, and the discriminators that feed a bound RDS output (k_quad, k_tail_fused), store exactly this
__device__ __forceinline__ float2 rds_xlate(float v, unsigned long long phase0, unsigned long long w, int i) {
    const float2 ph = phasor_u64(phase0 + w * (unsigned long long)i);
    return make_float2(v * ph.x, v * ph.y);
}

__device__ __forceinline__ float2 cmulf(float2 a, float2 b) {
    return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// d = a*b + c on both halves of a complex sample: two round-to-nearest fp32 FMAs (sm_90 has no packed fp32x2 FMA).
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// ---- programmatic dependent launch (PDL) for the chain of small dependent kernels behind stage 1 ----
// A chain kernel lets its successor be scheduled as soon as all of its own CTAs are running (pdl_trigger), and touches the
// stage buffers only after its predecessor has completed and its writes are visible (pdl_wait): the successor's launch
// latency, CTA scheduling and table loads (taps, banks: written at configure time) hide under the predecessor.  Both are
// no-ops in a kernel launched without the attribute.  Data a predecessor wrote is read with ld.global.cg (L2) after the
// wait, never with the non-coherent path: the CTA was resident before those lines were written.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
int kernels_pdl_default() {
    static const int mode = [] {
        const char* e = getenv("B200_PDL");
        const int m = e ? atoi(e) : PDL_DEFAULT;
        return (m < 0 || m > 2) ? PDL_DEFAULT : m;
    }();
    return mode;
}
static int num_sms();
// <<<>>> with the programmatic-serialization attribute (captured into graphs as programmatic edges).  Mode 2, the default,
// gives it to launches of at most two CTAs per SM: with the small grids of the reference's own chunk sizes (<= 1e6 samples)
// the early-resident successor costs nothing and the chain of seven dependent launches gets shorter; with the grids of a
// 16 Mi-sample chunk the successor's waiting CTAs take shared memory and registers from the spectrum branch on the other
// stream, which is what bounds the step there.
template <class P>
static cudaError_t launch_chain(void (*k)(const P), dim3 grid, dim3 block, size_t smem, const KernelOpts& o, cudaStream_t s, const P& p) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    if (o.pdl == 1 || (o.pdl == 2 && (long long)grid.x * grid.y * grid.z <= 2LL * num_sms())) {
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
    }
    return cudaLaunchKernelEx(&cfg, k, p);
}

// ------------------------------------------------------------------------------------------------
// stage 1, plain variant: one thread per (output, VFO); reads IQ through L1/L2.  Kept as the in-library
// cross-check of the tiled kernel (option "s1" = 0) and as the fallback for shapes the tile does not cover.
// ------------------------------------------------------------------------------------------------
template <int FMT>
__global__ void __launch_bounds__(128) k_xd_simple(const __grid_constant__ XdParams p) {
    const XdJob& J = p.job[blockIdx.y];
    int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= J.n_out) { return; }
    const int T = J.T;
    const long long i0 = (long long)J.offset + (long long)m * p.D - (T - 1);
    const float2* __restrict__ g = J.gpad + (p.D - 1);
    float ar = 0.0f, ai = 0.0f;
    for (int k = 0; k < T; k++) {
        float2 x = load_x<FMT>(p, i0 + k);
        float2 t = __ldg(g + k);
        ar += x.x * t.x - x.y * t.y;
        ai += x.x * t.y + x.y * t.x;
    }
    float2 ph = phasor_u64(J.phase0 + J.w * (unsigned long long)i0);
    J.out[m] = cmulf(make_float2(ar, ai), ph);
}

#define FL_M_PI_REF 3.1415926535f   // math::normalizePhase (normalize_phase.h:6-10)
#include "xd_pipe.cuh"
#include "xd_pfb.cuh"
#include "xd_tma.cuh"
#include "tails.cuh"
#include "dfir_reg.cuh"
#include "fused_tail.cuh"
#include "stereo.cuh"
#include "rds.cuh"

// ------------------------------------------------------------------------------------------------
// retune edge: outputs whose tap window starts before the newest retune boundary.  Explicit per-sample
// rotation (each history sample with the phase it was translated with, this chunk's with the current increment),
// real taps.
// ------------------------------------------------------------------------------------------------
template <int FMT>
__global__ void __launch_bounds__(128) k_xd_edge(const __grid_constant__ XdParams p) {
    const XdJob& J = p.job[blockIdx.y];
    if (!J.retuned) { return; }
    int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= J.n_out) { return; }
    const int T = J.T;
    const long long i0 = (long long)J.offset + (long long)m * p.D - (T - 1);
    if (i0 >= J.edge_start) { return; }
    float ar = 0.0f, ai = 0.0f;
    for (int k = 0; k < T; k++) {
        long long i = i0 + k;
        float2 x = load_x<FMT>(p, i);
        unsigned long long ph = (i < 0) ? J.hphase[T - 1 + i] : J.phase0 + J.w * (unsigned long long)i;
        float2 z = cmulf(x, phasor_u64(ph));
        float t = __ldg(J.h + k);
        ar = fmaf(z.x, t, ar);
        ai = fmaf(z.y, t, ai);
    }
    J.out[m] = make_float2(ar, ai);
}

// ------------------------------------------------------------------------------------------------
// generic decimating FIR, complex data x real taps
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_fir_c(const __grid_constant__ FirParams p) {
    const FirJob& J = p.job[blockIdx.y];
    int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= J.n_out) { return; }
    const float2* __restrict__ x = J.in + (size_t)J.offset + (size_t)m * J.decim;
    const float* __restrict__ h = J.taps;
    float ar = 0.0f, ai = 0.0f;
    for (int k = 0; k < J.ntaps; k++) {
        float2 v = __ldg(x + k);
        float t = __ldg(h + k);
        ar = fmaf(v.x, t, ar);
        ai = fmaf(v.y, t, ai);
    }
    J.out[m] = make_float2(ar, ai);
}

// ------------------------------------------------------------------------------------------------
// polyphase rational resampler
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_poly(const __grid_constant__ PolyParams p) {
    const PolyJob& J = p.job[blockIdx.y];
    int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= J.n_out) { return; }
    long long t = (long long)J.phase0 + (long long)m * J.decim;
    long long off = (long long)J.offset0 + t / J.interp;
    int ph = (int)(t % J.interp);
    const float2* __restrict__ x = J.in + off;
    const float* __restrict__ h = J.bank + (size_t)ph * J.tpp;
    float ar = 0.0f, ai = 0.0f;
    for (int k = 0; k < J.tpp; k++) {
        float2 v = __ldg(x + k);
        float c = __ldg(h + k);
        ar = fmaf(v.x, c, ar);
        ai = fmaf(v.y, c, ai);
    }
    J.out[m] = make_float2(ar, ai);
}

// ------------------------------------------------------------------------------------------------
// FM discriminator: out[i] = wrap(atan2f(x[i]) - atan2f(x[i-1])) * invDeviation
// wrap rule and the constant 3.1415926535f follow math::normalizePhase (normalize_phase.h:6-10)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_quad(const __grid_constant__ QuadParams p) {
    const QuadJob& J = p.job[blockIdx.y];
    pdl_trigger();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= J.n) { return; }
    pdl_wait();
    // J.in[0] is the last sample of the previous chunk (zero at start: atan2f(0,0) = 0 = Quadrature's initial phase)
    float2 c = __ldcg(J.in + i + 1);
    float2 q = __ldcg(J.in + i);
    float cur = atan2f(c.y, c.x);
    float prev = atan2f(q.y, q.x);
    float diff = __fsub_rn(cur, prev);
    if (diff > FL_M_PI_REF) { diff = __fsub_rn(diff, 2.0f * FL_M_PI_REF); }
    else if (diff <= -FL_M_PI_REF) { diff = __fadd_rn(diff, 2.0f * FL_M_PI_REF); }
    const float v = __fmul_rn(diff, J.inv_dev);
    J.out[i] = v;
    if (J.rds) { J.rds[i] = rds_xlate(v, J.rds_phase0, J.rds_w, i); }
}

// ------------------------------------------------------------------------------------------------
// real FIR with optional stereo duplication
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_fir_r(const __grid_constant__ FirRParams p) {
    const FirRJob& J = p.job[blockIdx.y];
    int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= J.n_out) { return; }
    const float* __restrict__ x = J.in + m;
    const float* __restrict__ h = J.taps;
    float acc = 0.0f;
    for (int k = 0; k < J.ntaps; k++) { acc = fmaf(__ldg(x + k), __ldg(h + k), acc); }
    if (J.stereo) { reinterpret_cast<float2*>(J.out)[m] = make_float2(acc, acc); }
    else { J.out[m] = acc; }
}

__global__ void __launch_bounds__(256) k_scale(const __grid_constant__ ScaleParams p) {
    const ScaleJob& J = p.job[blockIdx.y];
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= J.n) { return; }
    J.out[i] = __fmul_rn(__ldg(J.in + i), J.gain);
}

__global__ void __launch_bounds__(256) k_m2s(const __grid_constant__ M2SParams p) {
    const M2SJob& J = p.job[blockIdx.y];
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= J.n) { return; }
    float v = __ldg(J.in + i);
    reinterpret_cast<float2*>(J.out)[i] = make_float2(v, v);
}

__global__ void __launch_bounds__(256) k_rxl(const __grid_constant__ RxlParams p) {
    const RxlJob& J = p.job[blockIdx.y];
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= J.n) { return; }
    J.out[i] = rds_xlate(__ldg(J.in + i), J.phase0, J.w, i);
}

// ------------------------------------------------------------------------------------------------
// sequential audio-rate tails: one thread per VFO.  Arithmetic is written with explicit _rn intrinsics
// (no FMA contraction) because the AGC is branchy: the decisions must follow the reference's rounding.
// ------------------------------------------------------------------------------------------------
struct AgcCoef { float set_point, attack, inv_attack, decay, inv_decay, max_gain, max_out; };

__device__ __forceinline__ float agc_step(const AgcCoef& c, float& amp, float inAmp) {
    float gain;
    if (inAmp != 0.0f) {
        amp = (inAmp > amp) ? __fadd_rn(__fmul_rn(amp, c.inv_attack), __fmul_rn(inAmp, c.attack))
                            : __fadd_rn(__fmul_rn(amp, c.inv_decay), __fmul_rn(inAmp, c.decay));
        gain = fminf(__fdiv_rn(c.set_point, amp), c.max_gain);
    }
    else { gain = 1.0f; }
    return gain;
}
__device__ __forceinline__ float camp(float2 x) {
    return __fsqrt_rn(__fadd_rn(__fmul_rn(x.x, x.x), __fmul_rn(x.y, x.y)));
}

__global__ void k_seq(const __grid_constant__ SeqParams p) {
    const SeqJob& J = p.job[blockIdx.x];
    const int n = J.n;
    if (J.kind == 2) {
        // ---- Deemphasis<stereo_t>: y = alpha*x + (1-alpha)*y[-1] per channel  (deephasis.h:58-77) ----
        if (threadIdx.x >= 2) { return; }
        const int ch = threadIdx.x;
        const float* x = reinterpret_cast<const float*>(J.in);
        float y = J.state[5 + ch];
        const float a = J.alpha, b = __fsub_rn(1.0f, J.alpha);
        for (int i = 0; i < n; i++) {
            y = __fadd_rn(__fmul_rn(a, x[2 * i + ch]), __fmul_rn(b, y));
            J.out[2 * i + ch] = y;
        }
        J.state[5 + ch] = y;
        return;
    }
    if (threadIdx.x != 0) { return; }
    if (J.kind == 3) {
        // ---- NoiseBlanker: running mean amplitude, samples `level` times above it scaled back  (noise_blanker.h:38-57) ----
        float amp = J.state[7];
        float2* y = reinterpret_cast<float2*>(J.out);
        for (int i = 0; i < n; i++) {
            const float2 x = J.in[i];
            const float inAmp = camp(x);
            float gain = 1.0f;
            if (inAmp != 0.0f) {
                amp = __fadd_rn(__fmul_rn(amp, J.nb_inv_rate), __fmul_rn(inAmp, J.nb_rate));
                const float excess = __fdiv_rn(inAmp, amp);
                if (excess > J.nb_level) { gain = __fdiv_rn(1.0f, excess); }
            }
            y[i] = make_float2(__fmul_rn(x.x, gain), __fmul_rn(x.y, gain));
        }
        J.state[7] = amp;
        return;
    }
    AgcCoef c = { J.set_point, J.attack, J.inv_attack, J.decay, J.inv_decay, J.max_gain, J.max_out };
    float* st = J.state;
    if (J.kind == 0) {
        // ---- AM: [carrier AGC] -> magnitude -> DC block -> [audio AGC]   (am.h:101-133) ----
        float camp_state = st[0], aamp = st[1], dc = st[2];
        for (int i = 0; i < n; i++) {
            float2 x = J.in[i];
            if (J.agc_mode == 0) {
                float inAmp = camp(x);
                float gain = agc_step(c, camp_state, inAmp);
                if (__fmul_rn(inAmp, gain) > c.max_out) {
                    float maxAmp = 0.0f;
                    for (int j = i; j < n; j++) {
                        float a = camp(J.in[j]);
                        if (a > maxAmp) { maxAmp = a; }
                    }
                    camp_state = maxAmp;
                    gain = fminf(__fdiv_rn(c.set_point, camp_state), c.max_gain);
                }
                x = make_float2(__fmul_rn(x.x, gain), __fmul_rn(x.y, gain));
            }
            float mag = camp(x);                       // volk_32fc_magnitude_32f
            float y = __fsub_rn(mag, dc);              // DCBlocker (dc_blocker.h:54-60)
            dc = __fadd_rn(dc, __fmul_rn(y, J.dc_rate));
            J.out[i] = y;
        }
        if (J.agc_mode == 1) {
            for (int i = 0; i < n; i++) {
                float v = J.out[i];
                float inAmp = fabsf(v);
                float gain = agc_step(c, aamp, inAmp);
                if (__fmul_rn(inAmp, gain) > c.max_out) {
                    float maxAmp = 0.0f;
                    for (int j = i; j < n; j++) {
                        float a = fabsf(J.out[j]);
                        if (a > maxAmp) { maxAmp = a; }
                    }
                    aamp = maxAmp;
                    gain = fminf(__fdiv_rn(c.set_point, aamp), c.max_gain);
                }
                J.out[i] = __fmul_rn(v, gain);
            }
        }
        st[0] = camp_state; st[1] = aamp; st[2] = dc;
    }
    else {
        // ---- SSB: rotate by +-bw/2 (faithful fp32 recurrence, renormalised every 512 samples and at the
        //      end of the call: the VOLK rotator2 semantics) -> real part -> AGC   (ssb.h:77-92) ----
        float aamp = st[1];
        float pr = st[3], pi = st[4];
        const float dr = J.delta_re, di = J.delta_im;
        int since = 0;
        for (int i = 0; i < n; i++) {
            float2 x = J.in[i];
            float re = __fsub_rn(__fmul_rn(x.x, pr), __fmul_rn(x.y, pi));
            float nr = __fsub_rn(__fmul_rn(pr, dr), __fmul_rn(pi, di));
            float ni = __fadd_rn(__fmul_rn(pr, di), __fmul_rn(pi, dr));
            pr = nr; pi = ni;
            if (++since == 512) {
                float h = hypotf(pr, pi);
                pr = __fdiv_rn(pr, h); pi = __fdiv_rn(pi, h);
                since = 0;
            }
            J.out[i] = re;
        }
        if (since) {
            float h = hypotf(pr, pi);
            pr = __fdiv_rn(pr, h); pi = __fdiv_rn(pi, h);
        }
        for (int i = 0; i < n; i++) {
            float v = J.out[i];
            float inAmp = fabsf(v);
            float gain = agc_step(c, aamp, inAmp);
            if (__fmul_rn(inAmp, gain) > c.max_out) {
                float maxAmp = 0.0f;
                for (int j = i; j < n; j++) {
                    float a = fabsf(J.out[j]);
                    if (a > maxAmp) { maxAmp = a; }
                }
                aamp = maxAmp;
                gain = fminf(__fdiv_rn(c.set_point, aamp), c.max_gain);
            }
            J.out[i] = __fmul_rn(v, gain);
        }
        st[1] = aamp; st[3] = pr; st[4] = pi;
    }
}

// ------------------------------------------------------------------------------------------------
// end-of-chunk history carry (one CTA per delay line)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float carry_elem(const CarryJob& J, long long s, int comp) {
    if (s < J.la) { return J.a[s * J.esize + comp]; }
    long long b = s - J.la;
    if (J.bfmt < 0) { return reinterpret_cast<const float*>(J.b)[b * J.esize + comp]; }
    float2 v;
    if (J.bfmt == FMT_CF32) { v = load_iq<FMT_CF32>(J.b, b, 0.0f); }
    else if (J.bfmt == FMT_CS16) { v = load_iq<FMT_CS16>(J.b, b, J.scale); }
    else { v = load_iq<FMT_CS8>(J.b, b, J.scale); }
    return comp ? v.y : v.x;
}
__global__ void __launch_bounds__(256) k_carry(const __grid_constant__ CarryParams p) {
    const CarryJob& J = p.job[blockIdx.x];
    pdl_trigger();
    pdl_wait();
    const long long L = (long long)J.la + J.lb;
    const int hf = J.h * J.esize;                 // floats to produce
    for (int base = 0; base < hf; base += blockDim.x) {
        int f = base + threadIdx.x;
        float v = 0.0f;
        if (f < hf) {
            int e = f / J.esize, comp = f - e * J.esize;
            long long s = L - J.h + e;
            v = (s >= 0) ? carry_elem(J, s, comp) : 0.0f;
        }
        __syncthreads();
        if (f < hf) { J.dst[f] = v; }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------
// FFT branch: radix-2 DIF stages fused three at a time (radix-8 butterflies in registers) on a shared
// memory tile; output of the in-place DIF is bit-reversed, undone when the result is read back.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 mul_mj(float2 a) { return make_float2(a.y, -a.x); }   // a * (-j)
#define RSQRT2 0.70710678118654752440f
__device__ __forceinline__ float2 mul_w8_1(float2 a) { return make_float2((a.x + a.y) * RSQRT2, (a.y - a.x) * RSQRT2); }  // *(1-j)/sqrt2
__device__ __forceinline__ float2 mul_w8_3(float2 a) { return make_float2((a.y - a.x) * RSQRT2, -(a.x + a.y) * RSQRT2); } // *(-1-j)/sqrt2

// address of element r of transform c
// one pad slot every 16 elements: the late (small-stride) butterfly stages would otherwise hit a few banks only
__device__ __forceinline__ int padf(int a) { return a + (a >> 4); }
template <bool BATCH_INNER>
__device__ __forceinline__ int fft_addr(int r, int c, int C, int pitch) { return padf(BATCH_INNER ? (r * C + c) : (c * pitch + r)); }

// In-place forward DIF FFT of C transforms of length n = 2^logn living in shared memory.
template <bool BATCH_INNER>
__device__ void fft_dif_smem(float2* s, int logn, int C, int pitch, const float2* __restrict__ tw, int logTW) {
    const int n = 1 << logn;
    const int tid = threadIdx.x, nthr = blockDim.x;
    int logC = 0;
    while ((1 << logC) < C) { logC++; }
    int lognb = logn;
    while (lognb >= 3) {
        const int nb = 1 << lognb, e = nb >> 3;     // e = butterflies per sub-block
        const int per = n >> 3;                      // butterflies per transform
        const int logper = logn - 3;
        const int twsh = logTW - lognb;              // W_nb^j = tw[j << twsh]
        for (int t = tid; t < per * C; t += nthr) {
            int c, bi;
            if (BATCH_INNER) { c = t & (C - 1); bi = t >> logC; }
            else { bi = t & (per - 1); c = t >> logper; }
            const int blk = bi / e, j = bi - blk * e;
            const int base = blk * nb + j;
            float2 a[8];
#pragma unroll
            for (int i = 0; i < 8; i++) { a[i] = s[fft_addr<BATCH_INNER>(base + i * e, c, C, pitch)]; }
            const float2 w1 = __ldg(tw + ((size_t)j << twsh));
            const float2 w2 = __ldg(tw + ((size_t)(2 * j) << twsh));
            const float2 w4 = __ldg(tw + ((size_t)(4 * j) << twsh));
            // stage A: pairs (i, i+4), twiddle W_nb^(j + i*e) = w1 * W8^i
            float2 t0 = csub(a[0], a[4]); a[0] = cadd(a[0], a[4]);
            float2 t1 = csub(a[1], a[5]); a[1] = cadd(a[1], a[5]);
            float2 t2 = csub(a[2], a[6]); a[2] = cadd(a[2], a[6]);
            float2 t3 = csub(a[3], a[7]); a[3] = cadd(a[3], a[7]);
            a[4] = cmulf(t0, w1);
            a[5] = cmulf(mul_w8_1(t1), w1);
            a[6] = cmulf(mul_mj(t2), w1);
            a[7] = cmulf(mul_w8_3(t3), w1);
            // stage B: within each half, pairs (i, i+2), twiddle W_(nb/2)^(j + i*e) = w2 * W4^i
#pragma unroll
            for (int h = 0; h < 8; h += 4) {
                float2 u0 = csub(a[h + 0], a[h + 2]); a[h + 0] = cadd(a[h + 0], a[h + 2]);
                float2 u1 = csub(a[h + 1], a[h + 3]); a[h + 1] = cadd(a[h + 1], a[h + 3]);
                a[h + 2] = cmulf(u0, w2);
                a[h + 3] = cmulf(mul_mj(u1), w2);
            }
            // stage C: pairs (i, i+1), twiddle W_(nb/4)^j = w4
#pragma unroll
            for (int h = 0; h < 8; h += 2) {
                float2 u = csub(a[h], a[h + 1]); a[h] = cadd(a[h], a[h + 1]);
                a[h + 1] = cmulf(u, w4);
            }
#pragma unroll
            for (int i = 0; i < 8; i++) { s[fft_addr<BATCH_INNER>(base + i * e, c, C, pitch)] = a[i]; }
        }
        __syncthreads();
        lognb -= 3;
    }
    if (lognb == 2) {
        // radix-4: sub-blocks of 4, twiddles trivial (nb = 4: W_4^0 = 1, W_4^1 = -j; last stage W_2^0 = 1)
        const int per = n >> 2, logper = logn - 2;
        for (int t = tid; t < per * C; t += nthr) {
            int c, bi;
            if (BATCH_INNER) { c = t & (C - 1); bi = t >> logC; }
            else { bi = t & (per - 1); c = t >> logper; }
            const int base = bi * 4;
            float2 a0 = s[fft_addr<BATCH_INNER>(base + 0, c, C, pitch)];
            float2 a1 = s[fft_addr<BATCH_INNER>(base + 1, c, C, pitch)];
            float2 a2 = s[fft_addr<BATCH_INNER>(base + 2, c, C, pitch)];
            float2 a3 = s[fft_addr<BATCH_INNER>(base + 3, c, C, pitch)];
            float2 u0 = cadd(a0, a2), u1 = cadd(a1, a3);
            float2 v0 = csub(a0, a2), v1 = mul_mj(csub(a1, a3));
            s[fft_addr<BATCH_INNER>(base + 0, c, C, pitch)] = cadd(u0, u1);
            s[fft_addr<BATCH_INNER>(base + 1, c, C, pitch)] = csub(u0, u1);
            s[fft_addr<BATCH_INNER>(base + 2, c, C, pitch)] = cadd(v0, v1);
            s[fft_addr<BATCH_INNER>(base + 3, c, C, pitch)] = csub(v0, v1);
        }
        __syncthreads();
    }
    else if (lognb == 1) {
        const int per = n >> 1, logper = logn - 1;
        for (int t = tid; t < per * C; t += nthr) {
            int c, bi;
            if (BATCH_INNER) { c = t & (C - 1); bi = t >> logC; }
            else { bi = t & (per - 1); c = t >> logper; }
            const int base = bi * 2;
            float2 a0 = s[fft_addr<BATCH_INNER>(base + 0, c, C, pitch)];
            float2 a1 = s[fft_addr<BATCH_INNER>(base + 1, c, C, pitch)];
            s[fft_addr<BATCH_INNER>(base + 0, c, C, pitch)] = cadd(a0, a1);
            s[fft_addr<BATCH_INNER>(base + 1, c, C, pitch)] = csub(a0, a1);
        }
        __syncthreads();
    }
}

__device__ __forceinline__ int bitrev(int k, int bits) { return (int)(__brev((unsigned)k) >> (32 - bits)); }

// 10*log10(|X/N|^2) in VOLK's log2 formulation (volk_32fc_s32f_power_spectrum_32f, iq_frontend.cpp:262)
__device__ __forceinline__ float power_db(float2 X, float normFactSq) {
    float m2 = (X.x * X.x + X.y * X.y) * normFactSq;
    float l = log2f(m2);
    if (isinf(l)) { l = copysignf(127.0f, l); }
    return l * 3.01029995663981209120f;
}

// frame f of a batch (FftFrames) as two bases: its sample n is at lo[n] for n < lim (the staged part), at hi[n] from lim on
struct FrameSrc { const char* lo; const char* hi; int lim; };
template <int FMT>
__device__ __forceinline__ FrameSrc frame_src(const FftFrames& fr, int f) {
    constexpr int bps = FMT == FMT_CF32 ? 8 : (FMT == FMT_CS16 ? 4 : 2);
    return { reinterpret_cast<const char*>(fr.pre), reinterpret_cast<const char*>(fr.chunk) + ((long long)f * fr.stride - fr.split) * bps,
             f == 0 ? fr.split : 0 };
}
// sample n of a frame, zero from nz on; windowed: times window[n]
template <int FMT>
__device__ __forceinline__ float2 load_frame(const FftPlanDev& pl, const FrameSrc& fs, int n, bool windowed) {
    if (n >= pl.nz) { return make_float2(0.0f, 0.0f); }    // zero padding [nz, N)  (iq_frontend.cpp:301)
    const float2 x = load_iq<FMT>(n < fs.lim ? fs.lo : fs.hi, n, pl.in_scale);
    if (!windowed) { return x; }
    const float w = __ldg(pl.window + n);
    return make_float2(x.x * w, x.y * w);
}

// single-pass: the whole transform fits one CTA's shared memory
template <int FMT>
__global__ void __launch_bounds__(512) k_fft_single(const __grid_constant__ FftPlanDev pl, const __grid_constant__ FftFrames fr,
                                                      float* __restrict__ out_db0, float2* __restrict__ out_raw) {
    extern __shared__ __align__(16) float2 smem[];
    const int N = pl.N;
    float* out_db = out_db0 + (size_t)blockIdx.y * N;
    const FrameSrc fs = frame_src<FMT>(fr, blockIdx.y);
#pragma unroll 4
    for (int i = threadIdx.x; i < N; i += blockDim.x) { smem[padf(i)] = load_frame<FMT>(pl, fs, i, true); }
    __syncthreads();
    fft_dif_smem<false>(smem, pl.logN, 1, N, pl.tw, pl.logTW);
    const float nf = 1.0f / ((float)N * (float)N);
    for (int k = threadIdx.x; k < N; k += blockDim.x) {
        float2 X = smem[padf(bitrev(k, pl.logN))];
        out_db[k] = power_db(X, nf);
        if (out_raw) { out_raw[k] = X; }
    }
}

// pass 1 of the two-pass (four-step) transform: n = n1*N2 + n2, k = k1 + N1*k2.
// CTA = C adjacent columns n2, all rows n1: A[k1][n2] = W_N^(k1*n2) * sum_n1 x[n1*N2+n2] W_N1^(n1*k1)
template <int FMT>
__global__ void __launch_bounds__(512) k_fft_p1(const __grid_constant__ FftPlanDev pl, const __grid_constant__ FftFrames fr,
                                                  float2* __restrict__ work0, int C) {
    extern __shared__ __align__(16) float2 smem[];
    const int N1 = pl.N1, N2 = pl.N2;
    float2* work = work0 + (size_t)blockIdx.y * pl.N;
    const int c0 = blockIdx.x * C;
    const FrameSrc fs = frame_src<FMT>(fr, blockIdx.y);
#pragma unroll 4
    for (int t = threadIdx.x; t < N1 * C; t += blockDim.x) {
        int n1 = t / C, c = t - n1 * C;
        smem[padf(t)] = load_frame<FMT>(pl, fs, n1 * N2 + c0 + c, true);
    }
    __syncthreads();
    fft_dif_smem<true>(smem, pl.logN1, C, 0, pl.tw, pl.logTW);
    const float scale = -2.0f / (float)pl.N;
    for (int t = threadIdx.x; t < N1 * C; t += blockDim.x) {
        int k1 = t / C, c = t - k1 * C;
        float2 a = smem[padf(bitrev(k1, pl.logN1) * C + c)];
        int n2 = c0 + c;
        float sn, cs;
        sincospif((float)(k1 * n2) * scale, &sn, &cs);   // k1*n2 < N <= 2^22: exact in fp32
        work[(size_t)k1 * N2 + n2] = cmulf(a, make_float2(cs, sn));
    }
}

// pass 2: CTA = R adjacent rows k1; X[k1 + N1*k2] = sum_n2 A[k1][n2] W_N2^(n2*k2); fused dB epilogue
__global__ void __launch_bounds__(512) k_fft_p2(const __grid_constant__ FftPlanDev pl, const float2* __restrict__ work0,
                                                  float* __restrict__ out_db0, float2* __restrict__ out_raw, int R) {
    extern __shared__ __align__(16) float2 smem[];
    const int N1 = pl.N1, N2 = pl.N2;
    const float2* work = work0 + (size_t)blockIdx.y * pl.N;
    float* out_db = out_db0 + (size_t)blockIdx.y * pl.N;
    const int pitch = N2 + 1;
    const int r0 = blockIdx.x * R;
#pragma unroll 4
    for (int t = threadIdx.x; t < R * N2; t += blockDim.x) {
        int rl = t / N2, n2 = t - rl * N2;
        smem[padf(rl * pitch + n2)] = __ldg(work + (size_t)(r0 + rl) * N2 + n2);
    }
    __syncthreads();
    fft_dif_smem<false>(smem, pl.logN2, R, pitch, pl.tw, pl.logTW);
    const float nf = 1.0f / ((float)pl.N * (float)pl.N);
    for (int t = threadIdx.x; t < R * N2; t += blockDim.x) {
        int k2 = t / R, rl = t - k2 * R;
        float2 X = smem[padf(rl * pitch + bitrev(k2, pl.logN2))];
        size_t k = (size_t)(r0 + rl) + (size_t)N1 * k2;
        out_db[k] = power_db(X, nf);
        if (out_raw) { out_raw[k] = X; }
    }
}

#include "fft_reg.cuh"
#include "preproc.cuh"
#include "iqtap.cuh"

template <int FMT>
__global__ void __launch_bounds__(256) k_convert(const void* __restrict__ src, float2* __restrict__ dst, int n, float sc) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { dst[i] = load_iq<FMT>(src, i, sc); }
}

// doZoom + hold; start/len come from the host, which runs the reference's fp32 index loop verbatim so the
// bin selection is bit-exact (waterfall.cpp:65-90); the max-reduce and the hold update are exact in fp32.
__global__ void __launch_bounds__(256) k_zoom_hold(const float* __restrict__ line, const int* __restrict__ start,
                                                     const int* __restrict__ len, int out_size, float* __restrict__ out,
                                                     float* hold, float hold_speed) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= out_size) { return; }
    float maxVal = -INFINITY;
    const int s = start[i], l = len[i];
    for (int j = 0; j < l; j++) {
        float v = __ldg(line + s + j);
        if (v > maxVal) { maxVal = v; }
    }
    out[i] = maxVal;
    if (hold && i >= 1) {
        float d = __fsub_rn(hold[i], hold_speed);
        hold[i] = (maxVal < d) ? d : maxVal;
    }
}

// ------------------------------------------------------------------------------------------------
// launch wrappers
// ------------------------------------------------------------------------------------------------
static int g_smem_optin = -1;
int kernels_max_smem_optin() {
    if (g_smem_optin < 0) {
        int dev = 0, v = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        g_smem_optin = v;
    }
    return g_smem_optin;
}

// opt-in dynamic shared memory per kernel: grow-only and remembered, so the steady state costs no driver call per launch
template <typename K>
static cudaError_t set_smem(K kernel, size_t bytes) {
    static std::mutex mtx;
    static std::unordered_map<const void*, size_t> have;
    std::lock_guard<std::mutex> lk(mtx);
    size_t& cur = have[(const void*)kernel];
    if (bytes <= cur) { return cudaSuccess; }
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) { cur = bytes; }
    return e;
}

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

#include "chanpfb.cuh"
#include "ifnr.cuh"
#include "tails_reg.cuh"


static int g_num_sms = -1;
static int num_sms() {
    if (g_num_sms < 0) {
        int dev = 0, v = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
        g_num_sms = v > 0 ? v : 132;
    }
    return g_num_sms;
}

template <int FMT, int QC, int NT>
static cudaError_t launch_xd_pipe_t(const XdParams& p, const XpGeom& g, size_t smem, cudaStream_t s) {
    cudaError_t e = set_smem(k_xd_pipe<FMT, QC, NT>, smem);
    if (e != cudaSuccess) { return e; }
    // CTAs per SM by shared memory (1 KB reserved per CTA), threads and registers (<= 128/thread assumed above 1 CTA)
    int per_sm = (int)((size_t)233472 / (smem + 1024));
    if (per_sm > 2048 / NT) { per_sm = 2048 / NT; }
    if (per_sm > 512 / NT && NT >= 256) { per_sm = 512 / NT > 0 ? 512 / NT : 1; }
    if (NT == 128 && per_sm > 3) { per_sm = 3; }
    if (per_sm < 1) { per_sm = 1; }
    int grid = num_sms() * per_sm;
    if (grid > g.ntiles) { grid = g.ntiles; }
    k_xd_pipe<FMT, QC, NT><<<grid, NT, smem, s>>>(p, g);
    return cudaGetLastError();
}

// returns true when the pipelined kernel was launched
template <int FMT>
static bool try_xd_pipe(const XdParams& p, const KernelOpts& o, cudaStream_t s, cudaError_t* err, int nwarps, bool single = false) {
    const int D = p.D;
    if (D < 2 || (D & (D - 1))) { return false; }
    int logD = 0;
    while ((1 << logD) < D) { logD++; }
    // origin of the block grid: align it with job 0's window start so that the common case needs no tap shift
    int first = -1;
    for (int v = 0; v < p.njobs; v++) { if (p.job[v].n_out > 0) { first = v; break; } }
    if (first < 0) { return false; }
    const int a_first = p.job[first].offset - (p.job[first].T - 1);
    const int org = ((a_first % D) + D) % D;
    int QP = 1;
    long long jmin = (1LL << 60), jmax = -(1LL << 60);
    for (int v = 0; v < p.njobs; v++) {
        const int a = p.job[v].offset - (p.job[v].T - 1) - org;
        const int sft = ((a % D) + D) % D;
        const int qp = (p.job[v].T + sft + D - 1) / D;
        if (qp > QP) { QP = qp; }
        if (p.job[v].n_out <= 0) { continue; }
        const long long c = (a - sft) / D;
        if (c < jmin) { jmin = c; }
        if (c + p.job[v].n_out > jmax) { jmax = c + p.job[v].n_out; }
    }
    if (QP > p.QP) { return false; }              // the host sized gpad for p.QP blocks (+8 slack)
    int QC;
    if (QP <= 4) { QC = 4; }
    else if (QP <= 8) { QC = QP; }                // single chunk, odd sizes allowed
    else {
        QC = 6;
        int best = 1 << 30;
        const int qcs[3] = { 8, 6, 4 };           // several chunks: even sizes keep the LDS.128 window aligned
        for (int i = 0; i < 3; i++) {
            int pad = ((QP + qcs[i] - 1) / qcs[i]) * qcs[i] - QP;
            if (pad < best) { best = pad; QC = qcs[i]; }
        }
    }
    const int QPC = ((QP + QC - 1) / QC) * QC;
    if (jmin & 1) { jmin -= 1; }
    const int ngroups = (p.nslots + XP_VR - 1) / XP_VR;
    const int limit = kernels_max_smem_optin();
    // tile: about 8K raw samples (4K for the 4-warp configuration), a multiple of 128 outputs
    int MT = ((nwarps == 4 ? 4096 : 8192) / D) / 128 * 128;
    if (o.s1_mt > 0) { MT = o.s1_mt / 128 * 128; }
    if (MT < 128) { MT = 128; }
    if (MT > 1024) { MT = 1024; }
    XpGeom g;
    size_t smem = 0;
    for (;; MT -= 128) {
        if (MT < 128) { return false; }
        int jp = MT + QPC + 2;
        jp += (jp & 1);
        if ((jp & 3) == 0) { jp += 2; }
        const int nstrips_t = MT / 128;
        int rs = nwarps / (nstrips_t * ngroups);
        if (rs < 1) { rs = 1; }
        while (rs > 1 && (D % rs || (rs & (rs - 1)))) { rs--; }
        const int ntasks = nstrips_t * ngroups * rs;
        // the exchange buffer can live in the consumed tile buffer when all tasks run in one round
        const bool alias = ntasks <= nwarps && (size_t)D * jp >= (size_t)nwarps * 32 * 32;
        smem = ((size_t)(single ? 1 : 2) * D * jp + (size_t)ngroups * QPC * D * XP_VR + (size_t)p.njobs * MT + 3 * B200_BATCH +
                (!alias ? (size_t)nwarps * 32 * 32 : 0)) * sizeof(float2);
        if (smem <= (size_t)limit) { g.JP = jp; g.RS = rs; g.p_alias = alias ? 1 : 0; g.single = single ? 1 : 0; break; }
    }
    g.MT = MT; g.QPC = QPC; g.org = org; g.logD = logD; g.jmin = jmin;
    g.ntiles = cdiv(jmax - jmin, MT);
    cudaError_t e;
    (void)nwarps;
    switch (QC) {
    case 4: e = launch_xd_pipe_t<FMT, 4, 128>(p, g, smem, s); break;
    case 5: e = launch_xd_pipe_t<FMT, 5, 128>(p, g, smem, s); break;
    case 6: e = launch_xd_pipe_t<FMT, 6, 128>(p, g, smem, s); break;
    case 7: e = launch_xd_pipe_t<FMT, 7, 128>(p, g, smem, s); break;
    default: e = launch_xd_pipe_t<FMT, 8, 128>(p, g, smem, s); break;
    }
    *err = e;
    return true;
}


// ---- polyphase-filter-bank stage 1 (xd_pfb.cuh); returns true when it was launched ----
template <int LOGD, int QC, int PS>
static cudaError_t launch_xd_pfb_t(const XdParams& p, const XpGeom& g, int fmt, cudaStream_t s) {
    constexpr int D = 1 << LOGD, GQ = (QC + 3) & ~3;
    const size_t smem = ((size_t)D * g.JP + (size_t)B200_BATCH * (PS + PFB_MT / 16 + 16) + 3 * B200_BATCH) * sizeof(float2) +
                        (size_t)D * GQ * sizeof(float);
    if ((int)smem > kernels_max_smem_optin()) { return cudaErrorInvalidValue; }
    cudaError_t e = set_smem(k_xd_pfb<LOGD, QC, PS>, smem);
    if (e != cudaSuccess) { return e; }
    int per_sm = (int)((size_t)233472 / (smem + 1024));
    if (per_sm > 3) { per_sm = 3; }
    if (per_sm < 1) { per_sm = 1; }
    int grid = num_sms() * per_sm;
    if (grid > g.ntiles) { grid = g.ntiles; }
    k_xd_pfb<LOGD, QC, PS><<<grid, 128, smem, s>>>(p, g, fmt);
    return cudaGetLastError();
}
static bool try_xd_pfb(const XdParams& p, int fmt, cudaStream_t s, cudaError_t* err) {
    const int D = p.D, PS = p.pfb_ps;
    if ((PS != 8 && PS != 10) || D < 4 || (D & (D - 1))) { return false; }
    int logD = 0;
    while ((1 << logD) < D) { logD++; }
    const int T = p.job[0].T;
    const int org = (((p.job[0].offset - (T - 1)) % D) + D) % D;
    long long jmin = (1LL << 60), jmax = -(1LL << 60);
    for (int v = 0; v < p.njobs; v++) {
        const int a = p.job[v].offset - (p.job[v].T - 1) - org;
        if (p.job[v].T != T || (a % D) != 0 || p.job[v].n_out <= 0) { return false; }
        const long long c = a / D;
        if (c < jmin) { jmin = c; }
        if (c + p.job[v].n_out > jmax) { jmax = c + p.job[v].n_out; }
    }
    const int QC = (T + D - 1) / D;
    if (jmin & 1) { jmin -= 1; }
    XpGeom g;
    memset(&g, 0, sizeof(g));
    int jp = (PFB_MT + QC + 3) | 1;       // odd pitch: the 8-byte de-interleaving stores of a warp hit 32 distinct banks
    g.MT = PFB_MT; g.JP = jp; g.QPC = QC; g.org = org; g.logD = logD; g.jmin = jmin; g.RS = 1; g.single = 1;
    g.ntiles = cdiv(jmax - jmin, PFB_MT);
    cudaError_t e;
#define PFB_CASE(LD, Q)                                                                  \
    if (logD == LD && QC == Q) {                                                         \
        e = (PS == 10) ? launch_xd_pfb_t<LD, Q, 10>(p, g, fmt, s) : launch_xd_pfb_t<LD, Q, 8>(p, g, fmt, s); \
        *err = e;                                                                        \
        return true;                                                                     \
    }
    PFB_CASE(5, 5) PFB_CASE(6, 5) PFB_CASE(4, 5) PFB_CASE(3, 7) PFB_CASE(2, 7)
#undef PFB_CASE
    return false;
}


// ---- filter-bank stage 1 fed by the TMA engine (xd_tma.cuh); returns true when it was launched ----
typedef CUresult (*PFN_tmap_encode)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_tmap_encode tmap_encode_fn() {
    static PFN_tmap_encode fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) {
            fn = (PFN_tmap_encode)f;
        }
        else { cudaGetLastError(); }
    }
    return fn;
}
template <int LOGD, int QC, int PS, int MT, int NST>
static cudaError_t launch_xd_tma_n(const XdParams& p, const XtGeom& g, const CUtensorMap& tm, int grid, cudaStream_t s) {
    using Lay = XtLay<LOGD, QC, MT>;
    // ring + phasor tables of the launch's jobs + barriers + the ÷4 epilogue's carried window (F2H outputs per job, only with
    // the epilogue).  At config 2 (8 VFOs, PS 10) that is 141.3 KiB: with a pass-1 FFT CTA of 8 (82.1 KiB) and 2 x 1 KiB
    // reserved it stays within the SM's 228 KiB
    auto bytes = [&](int nj, bool f2) {
        return (size_t)NST * Lay::STAGE + ((size_t)nj * (PS + 16 + Lay::NPH) + (f2 ? (size_t)nj * Lay::F2H : 0)) * sizeof(float2) +
               2 * NST * sizeof(unsigned long long) + 1024;
    };
    const size_t smem = bytes(p.njobs, g.f2 != 0);
    if ((int)smem > kernels_max_smem_optin()) { return cudaErrorInvalidValue; }
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = set_smem(k_xd_tma<LOGD, QC, PS, MT, NST>, bytes(B200_BATCH, true));
        if (e != cudaSuccess) { return e; }
        attr_set = true;
    }
    k_xd_tma<LOGD, QC, PS, MT, NST><<<grid, (Lay::NW + 1) * 32, smem, s>>>(p, g, tm);
    return cudaGetLastError();
}
template <int LOGD, int QC, int PS, int MT>
static cudaError_t launch_xd_tma_t(const XdParams& p, const XtGeom& g, const CUtensorMap& tm, int grid, int stages, cudaStream_t s) {
    return stages == 3 ? launch_xd_tma_n<LOGD, QC, PS, MT, 3>(p, g, tm, grid, s) : launch_xd_tma_n<LOGD, QC, PS, MT, 2>(p, g, tm, grid, s);
}
static bool try_xd_tma(const XdParams& p, const KernelOpts& o, cudaStream_t s, cudaError_t* err, bool* f2) {
    const int D = p.D, PS = p.pfb_ps;
    if ((PS != 8 && PS != 10) || (D != 32 && D != 64) || !p.taps_host) { return false; }
    if (((uintptr_t)p.in & 15) != 0) { return false; }
    PFN_tmap_encode enc = tmap_encode_fn();
    if (!enc) { return false; }
    const int T = p.job[0].T;
    const int a0 = p.job[0].offset - (T - 1);
    const int org = ((a0 % D) + D) % D;
    for (int v = 0; v < p.njobs; v++) {
        const int a = p.job[v].offset - (p.job[v].T - 1);
        if (p.job[v].T != T || a != a0 || p.job[v].n_out != p.job[0].n_out || p.job[v].n_out <= 0) { return false; }
    }
    // row origin: 128-byte aligned when that costs no extra tap block, else 16-byte aligned (s leading zero taps)
    const int QC = (T + (org & 1) + D - 1) / D;
    int sh = org & 1;
    for (int al = 16; al >= 2; al >>= 1) {
        const int c = org & (al - 1);
        if ((T + c + D - 1) / D == QC) { sh = c; break; }
    }
    if (QC * D > XT_MAXTAPS) { return false; }
    XtGeom g;
    memset(&g, 0, sizeof(g));
    g.org = org - sh;
    g.s = sh;
    g.diag = o.s1_diag;
    g.cj = (a0 - org) / D;                        // exact: a0 - org is a multiple of D
    long long jmin = g.cj;
    if (jmin & 1) { jmin -= 1; }
    g.jmin = jmin;
    for (int q = 0; q < QC * D; q++) {
        const int k = q - sh;
        float t = (k >= 0 && k < T) ? p.taps_host[k] : 0.0f;
        if (p.pfb_sigma < 0 && k >= 0 && ((k / PS) & 1)) { t = -t; }
        g.g[q] = t;
    }
    const long long avail = (long long)p.count - g.org;
    g.rows_tma = avail > 0 ? (int)(avail / (2 * D)) : 0;
    const int MT = (D == 32) ? 256 : 128;
    g.jend = (long long)g.cj + p.job[0].n_out;
    if (g.rows_tma < 8) { return false; }
    // contiguous runs of whole tiles, one per persistent CTA (one per SM, or fewer: KernelOpts::s1_ctas leaves SMs free for
    // the kernels of the other streams).  With the ÷4 epilogue every CTA but the first also filters the 32 outputs in front of
    // its run; the run is then 32 short of its tiles, and no CTA does more tiles than without the epilogue plus the halo.
    for (int v = 0; v < p.njobs; v++) {
        if (p.job[v].f2_out && !g.diag) { g.f2 = 1; }
    }
    g.halo = g.f2 ? 32 : 0;
    int grid = num_sms();
    if (o.s1_ctas > 0 && o.s1_ctas < grid) { grid = o.s1_ctas; }
    const long long nblk = g.jend - jmin;
    const long long tiles_per_cta = cdiv(cdiv(nblk, grid) + g.halo, MT);
    g.run = (int)(tiles_per_cta * MT - g.halo);
    grid = (int)cdiv(nblk, g.run);
    CUtensorMap tm;
    const cuuint64_t gdim[2] = { (cuuint64_t)(4 * D), (cuuint64_t)g.rows_tma };
    const cuuint64_t gstr[1] = { (cuuint64_t)(4 * D) * sizeof(float) };
    const int NR = (((MT + QC + 2) / 2) + 7) & ~7;
    const cuuint32_t box[2] = { 32u, (cuuint32_t)NR };
    const cuuint32_t estr[2] = { 1u, 1u };
    void* base = (void*)((const float2*)p.in + g.org);
    CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { return false; }
#define XT_CASE(LD, Q, MTV)                                                                    \
    if (D == (1 << LD) && QC == Q) {                                                           \
        *err = (PS == 10) ? launch_xd_tma_t<LD, Q, 10, MTV>(p, g, tm, grid, o.s1_stages, s)                   \
                          : launch_xd_tma_t<LD, Q, 8, MTV>(p, g, tm, grid, o.s1_stages, s);                    \
        *f2 = g.f2 != 0;                                                                       \
        return true;                                                                           \
    }
    XT_CASE(5, 5, 256) XT_CASE(6, 5, 128) XT_CASE(6, 6, 128) XT_CASE(6, 7, 128)
#undef XT_CASE
    return false;
}

template <int FMT>
static cudaError_t launch_xd_fmt(const XdParams& p, int variant, const KernelOpts& o, cudaStream_t s, int* nlaunch, bool* tma, bool* f2) {
    int max_out = 0;
    for (int v = 0; v < p.njobs; v++) { max_out = p.job[v].n_out > max_out ? p.job[v].n_out : max_out; }
    if (max_out <= 0) { return cudaSuccess; }
    const int D = p.D;
    if (variant >= 7) {
        cudaError_t e = cudaSuccess;
        if (variant >= 8 && FMT == FMT_CF32 && p.pfb_ps > 0 && try_xd_tma(p, o, s, &e, f2)) {
            *tma = true;
            if (nlaunch) { (*nlaunch)++; }
            return e;
        }
        if (p.pfb_ps > 0 && try_xd_pfb(p, FMT, s, &e)) {
            if (nlaunch) { (*nlaunch)++; }
            return e;
        }
        variant = 6;
    }
    if (variant >= 1) {
        // per-VFO complex taps on cp.async tiles, 4-warp CTAs: 5 = double-buffered, one CTA per SM; anything else = one tile
        // buffer per CTA, three CTAs per SM (the retired 8- / 16-warp and single-buffer tile kernels map here)
        cudaError_t e = cudaSuccess;
        if (try_xd_pipe<FMT>(p, o, s, &e, 4, variant != 5)) {
            if (nlaunch) { (*nlaunch)++; }
            return e;
        }
    }
    // shapes the tile kernels do not cover (pure translate, D = 1): one thread per output
    dim3 grid(cdiv(max_out, 128), p.njobs);
    k_xd_simple<FMT><<<grid, 128, 0, s>>>(p);
    if (nlaunch) { (*nlaunch)++; }
    return cudaGetLastError();
}

cudaError_t launch_xlate_decim(const XdParams& p, int fmt, int variant, const KernelOpts& o, cudaStream_t s, int* nlaunch, bool* tma,
                               bool* f2) {
    *tma = false;
    *f2 = false;
    if (fmt == FMT_CF32) { return launch_xd_fmt<FMT_CF32>(p, variant, o, s, nlaunch, tma, f2); }
    if (fmt == FMT_CS16) { return launch_xd_fmt<FMT_CS16>(p, variant, o, s, nlaunch, tma, f2); }
    return launch_xd_fmt<FMT_CS8>(p, variant, o, s, nlaunch, tma, f2);
}


cudaError_t launch_xd_edge(const XdParams& p, int fmt, cudaStream_t s, int* nlaunch) {
    int medge = 0;
    bool any = false;
    for (int v = 0; v < p.njobs; v++) {
        if (!p.job[v].retuned || p.job[v].n_out <= 0) { continue; }
        any = true;
        int need = p.job[v].edge_start + p.job[v].T - 1 - p.job[v].offset;   // outputs with i_m < edge_start
        int me = need > 0 ? (need + p.D - 1) / p.D : 0;
        if (me > p.job[v].n_out) { me = p.job[v].n_out; }
        if (me > medge) { medge = me; }
    }
    if (!any || medge <= 0) { return cudaSuccess; }
    dim3 grid(cdiv(medge, 128), p.njobs);
    if (fmt == FMT_CF32) { k_xd_edge<FMT_CF32><<<grid, 128, 0, s>>>(p); }
    else if (fmt == FMT_CS16) { k_xd_edge<FMT_CS16><<<grid, 128, 0, s>>>(p); }
    else { k_xd_edge<FMT_CS8><<<grid, 128, 0, s>>>(p); }
    if (nlaunch) { (*nlaunch)++; }
    return cudaGetLastError();
}

cudaError_t launch_fir_c(const FirParams& p, const KernelOpts& o, cudaStream_t s) {
    if (p.max_out <= 0 || p.njobs <= 0) { return cudaSuccess; }
    if (o.tail_variant >= 1) {
        // all jobs of a batch share one kernel shape: pick by the first job, require the others to agree
        bool all_d1 = true, same_d = true;
        int maxT = 0, D0 = p.job[0].decim;
        for (int v = 0; v < p.njobs; v++) {
            all_d1 = all_d1 && p.job[v].decim == 1 && p.job[v].offset == 0;
            same_d = same_d && p.job[v].decim == D0;
            maxT = p.job[v].ntaps > maxT ? p.job[v].ntaps : maxT;
        }
        if (all_d1 && maxT <= TAIL_MAX_TAPS) {
            const int OB = FC2_THREADS * FC2_R;
            const int span = OB + maxT + FC2_R;
            size_t smem = ((size_t)((maxT + 1) >> 1) + (size_t)(span + (span >> 3) + 2)) * sizeof(float2);
            cudaError_t e = set_smem(k_fir_c2, smem);
            if (e != cudaSuccess) { return e; }
            dim3 grid(cdiv(p.max_out, OB), p.njobs);
            k_fir_c2<<<grid, FC2_THREADS, smem, s>>>(p);
            return cudaGetLastError();
        }
        if (same_d && D0 > 1 && D0 <= 64 && maxT <= TAIL_MAX_TAPS) {
            int lg = 30;
            if ((D0 & (D0 - 1)) == 0) { lg = 0; while ((1 << lg) < D0) { lg++; } }
            const int span = (FCD_THREADS - 1) * D0 + maxT;
            size_t smem = ((size_t)((maxT + 1) >> 1) + (size_t)(span + (lg < 30 ? (span >> lg) : 0) + 2)) * sizeof(float2);
            if (smem <= (size_t)kernels_max_smem_optin()) {
                cudaError_t e = set_smem(k_fir_cd, smem);
                if (e != cudaSuccess) { return e; }
                dim3 grid(cdiv(p.max_out, FCD_THREADS), p.njobs);
                k_fir_cd<<<grid, FCD_THREADS, smem, s>>>(p, lg);
                return cudaGetLastError();
            }
        }
    }
    dim3 grid(cdiv(p.max_out, 256), p.njobs);
    k_fir_c<<<grid, 256, 0, s>>>(p);
    return cudaGetLastError();
}
cudaError_t launch_poly(const PolyParams& p, const KernelOpts& o, cudaStream_t s) {
    if (p.max_out <= 0 || p.njobs <= 0) { return cudaSuccess; }
    if (o.tail_variant >= 1) {
        long long span_cap = 0, bank_floats = 0;
        for (int v = 0; v < p.njobs; v++) {
            long long sp = ((long long)PL2_THREADS * p.job[v].decim + p.job[v].interp - 1) / p.job[v].interp + p.job[v].tpp + 2;
            span_cap = sp > span_cap ? sp : span_cap;
            long long bf = (long long)p.job[v].interp * (p.job[v].tpp | 1);
            bank_floats = bf > bank_floats ? bf : bank_floats;
        }
        if (span_cap <= 8192) {
            const int in_smem = bank_floats <= 16384 ? 1 : 0;
            size_t smem = (size_t)span_cap * sizeof(float2) + (in_smem ? (size_t)bank_floats * sizeof(float) : 0);
            cudaError_t e = set_smem(k_poly2, smem);
            if (e != cudaSuccess) { return e; }
            dim3 grid(cdiv(p.max_out, PL2_THREADS), p.njobs);
            k_poly2<<<grid, PL2_THREADS, smem, s>>>(p, (int)span_cap, in_smem);
            return cudaGetLastError();
        }
    }
    dim3 grid(cdiv(p.max_out, 256), p.njobs);
    k_poly<<<grid, 256, 0, s>>>(p);
    return cudaGetLastError();
}
cudaError_t launch_quad(const QuadParams& p, const KernelOpts& o, cudaStream_t s) {
    if (p.max_n <= 0 || p.njobs <= 0) { return cudaSuccess; }
    dim3 grid(cdiv(p.max_n, 256), p.njobs);
    return launch_chain(k_quad, grid, dim3(256), 0, o, s, p);
}
// resident CTAs of the fused tail per SM for a thread count and dynamic shared-memory size (registers included)
// the opt-in shared-memory size of each k_tail_fused build only ever grows: the occupancy query and the launcher share it
static size_t g_ft_attr[3] = { 0, 0, 0 };
template <int NTV>
static cudaError_t ft_ensure_smem(int slot, size_t smem_bytes) {
    if (smem_bytes <= g_ft_attr[slot]) { return cudaSuccess; }
    cudaError_t e = cudaFuncSetAttribute(k_tail_fused<NTV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
    if (e == cudaSuccess) { g_ft_attr[slot] = smem_bytes; }
    return e;
}
int tail_fused_ctas_per_sm(int threads, size_t smem_bytes) {
    int n = 0;
    cudaError_t e;
    if ((int)smem_bytes > kernels_max_smem_optin()) { return 0; }
    if (threads == 512) {
        if ((e = ft_ensure_smem<512>(2, smem_bytes)) == cudaSuccess) { e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_tail_fused<512>, 512, smem_bytes); }
    }
    else if (threads == 256) {
        if ((e = ft_ensure_smem<256>(1, smem_bytes)) == cudaSuccess) { e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_tail_fused<256>, 256, smem_bytes); }
    }
    else {
        if ((e = ft_ensure_smem<128>(0, smem_bytes)) == cudaSuccess) { e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_tail_fused<128>, 128, smem_bytes); }
    }
    if (e != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}
cudaError_t launch_tail_fused(const FtParams& p, int max_slabs, int threads, size_t smem_bytes, cudaStream_t s) {
    if (p.njobs <= 0 || max_slabs <= 0) { return cudaSuccess; }
    if ((int)smem_bytes > kernels_max_smem_optin()) { return cudaErrorInvalidValue; }
    dim3 grid(max_slabs, p.njobs);
#define FT_LAUNCH(NTV, SLOT)                                                                                                   \
    do {                                                                                                                       \
        cudaError_t e = ft_ensure_smem<NTV>(SLOT, smem_bytes);                                                                 \
        if (e != cudaSuccess) { return e; }                                                                                    \
        k_tail_fused<NTV><<<grid, NTV, smem_bytes, s>>>(p);                                                                    \
    } while (0)
    if (threads == 512) { FT_LAUNCH(512, 2); }
    else if (threads == 256) { FT_LAUNCH(256, 1); }
    else { FT_LAUNCH(128, 0); }
#undef FT_LAUNCH
    return cudaGetLastError();
}
cudaError_t launch_fir_r(const FirRParams& p, const KernelOpts& o, cudaStream_t s) {
    if (p.max_out <= 0 || p.njobs <= 0) { return cudaSuccess; }
    if (o.tail_variant >= 1) {
        int maxT = 0;
        for (int v = 0; v < p.njobs; v++) { maxT = p.job[v].ntaps > maxT ? p.job[v].ntaps : maxT; }
        if (maxT <= TAIL_MAX_TAPS) {
            const int OB = FR2_THREADS * FR2_R;
            const int span = OB + maxT + FR2_R;
            size_t smem = ((size_t)maxT + (size_t)(span + (span >> 3) + 2)) * sizeof(float);
            cudaError_t e = set_smem(k_fir_r2, smem);
            if (e != cudaSuccess) { return e; }
            dim3 grid(cdiv(p.max_out, OB), p.njobs);
            k_fir_r2<<<grid, FR2_THREADS, smem, s>>>(p);
            return cudaGetLastError();
        }
    }
    dim3 grid(cdiv(p.max_out, 256), p.njobs);
    k_fir_r<<<grid, 256, 0, s>>>(p);
    return cudaGetLastError();
}
cudaError_t launch_seq(const SeqParams& p, cudaStream_t s) {
    if (p.njobs <= 0) { return cudaSuccess; }
    k_seq<<<p.njobs, 32, 0, s>>>(p);
    return cudaGetLastError();
}
cudaError_t launch_m2s(const M2SParams& p, cudaStream_t s) {
    if (p.max_n <= 0 || p.njobs <= 0) { return cudaSuccess; }
    dim3 grid(cdiv(p.max_n, 256), p.njobs);
    k_m2s<<<grid, 256, 0, s>>>(p);
    return cudaGetLastError();
}
cudaError_t launch_rxl(const RxlParams& p, cudaStream_t s) {
    if (p.max_n <= 0 || p.njobs <= 0) { return cudaSuccess; }
    dim3 grid(cdiv(p.max_n, 256), p.njobs);
    k_rxl<<<grid, 256, 0, s>>>(p);
    return cudaGetLastError();
}
cudaError_t launch_scale(const ScaleParams& p, cudaStream_t s) {
    if (p.max_n <= 0 || p.njobs <= 0) { return cudaSuccess; }
    dim3 grid(cdiv(p.max_n, 256), p.njobs);
    k_scale<<<grid, 256, 0, s>>>(p);
    return cudaGetLastError();
}
cudaError_t launch_carry(const CarryParams& p, const KernelOpts& o, cudaStream_t s) {
    if (p.njobs <= 0) { return cudaSuccess; }
    return launch_chain(k_carry, dim3((unsigned)p.njobs), dim3(256), 0, o, s, p);
}

bool fft_plan_uses_reg(const FftPlanDev& pl) {
    return pl.N2 > 1 && pl.logN1 >= 8 && pl.logN1 <= 10 && pl.logN2 >= 8 && pl.logN2 <= 10;
}

template <int FMT>
static cudaError_t launch_fft_fmt(const FftPlanDev& pl, const FftFrames& fr, float2* work, float* out_db, float2* out_raw,
                                  const KernelOpts& o, cudaStream_t s, int* nlaunch, bool tables) {
    cudaError_t e;
    const int nbatch = fr.nbatch;
    if (pl.N1 == pl.N) {
        size_t smem = ((size_t)pl.N + (pl.N >> 4) + 2) * sizeof(float2);
        e = set_smem(k_fft_single<FMT>, smem);
        if (e != cudaSuccess) { return e; }
        int thr = pl.N / 8 < 32 ? 32 : (pl.N / 8 > 512 ? 512 : pl.N / 8);
        k_fft_single<FMT><<<dim3(1, nbatch), thr, smem, s>>>(pl, fr, out_db, out_raw);
        if (nlaunch) { (*nlaunch)++; }
        return cudaGetLastError();
    }
    // two passes
    if (o.fft_variant >= 1 && !out_raw && pl.tw_fine && pl.window_p && fft_plan_uses_reg(pl)) {
        // register-resident column / row transforms (fft_reg.cuh)
        // transforms per CTA: 8 (256 threads) or 4 (128 threads) -- KernelOpts::fft_cta; DESIGN.md section 4 has the residency.
        // tables: + TW + N/TW float2 of twiddles in shared memory (pass 1), + TW (pass 2)
#define FR_P1(RA, RB, CC)                                                                                      \
        do {                                                                                                   \
            const size_t sm = (fr_smem_tiles<RA, RB>(CC) + (tables ? (size_t)pl.TW + (pl.N >> pl.logTW) : 0)) * sizeof(float2); \
            if (tables) {                                                                                      \
                e = set_smem(k_fftr_p1<FMT, RA, RB, CC, true>, sm);                                         \
                if (e != cudaSuccess) { return e; }                                                            \
                k_fftr_p1<FMT, RA, RB, CC, true><<<dim3(pl.N2 / CC, nbatch), CC * FrGeom<RA, RB>::TP, sm, s>>>(pl, fr, work); \
            }                                                                                                  \
            else {                                                                                             \
                e = set_smem(k_fftr_p1<FMT, RA, RB, CC, false>, sm);                                        \
                if (e != cudaSuccess) { return e; }                                                            \
                k_fftr_p1<FMT, RA, RB, CC, false><<<dim3(pl.N2 / CC, nbatch), CC * FrGeom<RA, RB>::TP, sm, s>>>(pl, fr, work); \
            }                                                                                                  \
        } while (0)
#define FR_P2(RA, RB, RR)                                                                                      \
        do {                                                                                                   \
            const size_t sm = (fr_smem_tiles<RA, RB>(RR) + (tables ? (size_t)pl.TW : 0)) * sizeof(float2);     \
            if (tables) {                                                                                      \
                e = set_smem(k_fftr_p2<RA, RB, RR, true>, sm);                                                 \
                if (e != cudaSuccess) { return e; }                                                            \
                k_fftr_p2<RA, RB, RR, true><<<dim3(pl.N1 / RR, nbatch), RR * FrGeom<RA, RB>::TP, sm, s>>>(pl, work, out_db); \
            }                                                                                                  \
            else {                                                                                             \
                e = set_smem(k_fftr_p2<RA, RB, RR, false>, sm);                                                \
                if (e != cudaSuccess) { return e; }                                                            \
                k_fftr_p2<RA, RB, RR, false><<<dim3(pl.N1 / RR, nbatch), RR * FrGeom<RA, RB>::TP, sm, s>>>(pl, work, out_db); \
            }                                                                                                  \
        } while (0)
        if (o.fft_cta == 4) {
            if (pl.logN1 == 10) { FR_P1(32, 32, 4); } else if (pl.logN1 == 9) { FR_P1(16, 32, 4); } else { FR_P1(16, 16, 4); }
        }
        else {
            if (pl.logN1 == 10) { FR_P1(32, 32, 8); } else if (pl.logN1 == 9) { FR_P1(16, 32, 8); } else { FR_P1(16, 16, 8); }
        }
        e = cudaGetLastError();
        if (e != cudaSuccess) { return e; }
        if (o.fft_cta == 4) {
            if (pl.logN2 == 10) { FR_P2(32, 32, 4); } else if (pl.logN2 == 9) { FR_P2(16, 32, 4); } else { FR_P2(16, 16, 4); }
        }
        else {
            if (pl.logN2 == 10) { FR_P2(32, 32, 8); } else if (pl.logN2 == 9) { FR_P2(16, 32, 8); } else { FR_P2(16, 16, 8); }
        }
#undef FR_P1
#undef FR_P2
        if (nlaunch) { (*nlaunch) += 2; }
        return cudaGetLastError();
    }
    // columns / rows per CTA: enough CTAs to fill the chip about twice, at least 4 (32-byte segments)
    int C = 16;
    while (C > 4 && (pl.N2 / C) * nbatch < 2 * num_sms()) { C >>= 1; }
    while ((size_t)pl.N1 * C * sizeof(float2) > 196608 && C > 1) { C >>= 1; }
    if (C > pl.N2) { C = pl.N2; }
    int R = 16;
    while (R > 4 && (pl.N1 / R) * nbatch < 2 * num_sms()) { R >>= 1; }
    while ((size_t)R * (pl.N2 + 1) * sizeof(float2) > 196608 && R > 1) { R >>= 1; }
    if (R > pl.N1) { R = pl.N1; }
    size_t smem1 = ((size_t)pl.N1 * C + ((size_t)pl.N1 * C >> 4) + 2) * sizeof(float2);
    size_t smem2 = ((size_t)R * (pl.N2 + 1) + ((size_t)R * (pl.N2 + 1) >> 4) + 2) * sizeof(float2);
    e = set_smem(k_fft_p1<FMT>, smem1);
    if (e != cudaSuccess) { return e; }
    e = set_smem(k_fft_p2, smem2);
    if (e != cudaSuccess) { return e; }
    const int thr1 = (pl.N1 / 8) * C >= 512 ? 512 : 256, thr2 = (pl.N2 / 8) * R >= 512 ? 512 : 256;
    k_fft_p1<FMT><<<dim3(pl.N2 / C, nbatch), thr1, smem1, s>>>(pl, fr, work, C);
    e = cudaGetLastError();
    if (e != cudaSuccess) { return e; }
    k_fft_p2<<<dim3(pl.N1 / R, nbatch), thr2, smem2, s>>>(pl, work, out_db, out_raw, R);
    if (nlaunch) { (*nlaunch) += 2; }
    return cudaGetLastError();
}

// gridDim.y holds a batch's frame index, so a batch of more frames is launched in slices of at most this many
#define FFT_MAX_GRID_Y 65535
cudaError_t launch_fft_frames(const FftPlanDev& pl, const FftFrames& fr, int fmt, float2* work, float* out_db,
                              float2* out_raw, const KernelOpts& o, cudaStream_t s, int* nlaunch, bool tables) {
    const int bps = fmt == FMT_CF32 ? 8 : (fmt == FMT_CS16 ? 4 : 2);
    for (int f0 = 0; f0 < fr.nbatch; f0 += FFT_MAX_GRID_Y) {
        // slice 0 keeps the staged part of its first frame; a later slice's first frame lies wholly in the chunk
        FftFrames sl = fr;
        sl.nbatch = std::min(fr.nbatch - f0, FFT_MAX_GRID_Y);
        if (f0 > 0) {
            sl.chunk = reinterpret_cast<const char*>(fr.chunk) + ((long long)f0 * fr.stride - fr.split) * bps;
            sl.pre = nullptr;
            sl.split = 0;
        }
        float2* const w = work + (size_t)f0 * pl.N;
        float* const db = out_db ? out_db + (size_t)f0 * pl.N : nullptr;
        float2* const raw = out_raw ? out_raw + (size_t)f0 * pl.N : nullptr;
        cudaError_t e;
        if (fmt == FMT_CF32) { e = launch_fft_fmt<FMT_CF32>(pl, sl, w, db, raw, o, s, nlaunch, tables); }
        else if (fmt == FMT_CS16) { e = launch_fft_fmt<FMT_CS16>(pl, sl, w, db, raw, o, s, nlaunch, tables); }
        else { e = launch_fft_fmt<FMT_CS8>(pl, sl, w, db, raw, o, s, nlaunch, tables); }
        if (e != cudaSuccess) { return e; }
    }
    return cudaSuccess;
}
cudaError_t launch_fft_frame(const FftPlanDev& pl, const void* src, int fmt, float2* work, float* out_db,
                             float2* out_raw, const KernelOpts& o, cudaStream_t s, int* nlaunch) {
    const FftFrames fr{ src, nullptr, 0, 0, 1 };
    return launch_fft_frames(pl, fr, fmt, work, out_db, out_raw, o, s, nlaunch, true);
}

cudaError_t launch_convert_cf32(const void* src, int fmt, float2* dst, int n, float scale, cudaStream_t s) {
    if (n <= 0) { return cudaSuccess; }
    int grid = cdiv(n, 256);
    if (fmt == FMT_CF32) { k_convert<FMT_CF32><<<grid, 256, 0, s>>>(src, dst, n, scale); }
    else if (fmt == FMT_CS16) { k_convert<FMT_CS16><<<grid, 256, 0, s>>>(src, dst, n, scale); }
    else { k_convert<FMT_CS8><<<grid, 256, 0, s>>>(src, dst, n, scale); }
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// export formats: recorder sample types (wav.cpp:150-183) and the compressed-stream packet payload
// (sample_stream_compressor.h:30-66).  r = x * scalar, clamped, rounded to nearest-even like rintf.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_export(const float* __restrict__ in, long long n, int type, float scalar, void* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) { return; }
    const float x = __ldg(in + i);
    // the element rules are iqtap.cuh's, shared with the front end's IQ taps
    if (type == EXP_U8) { reinterpret_cast<unsigned char*>(out)[i] = iq_rule_u8(x); }
    else if (type == EXP_I8) { reinterpret_cast<signed char*>(out)[i] = iq_rule_i8(x, scalar); }
    else if (type == EXP_I16) { reinterpret_cast<short*>(out)[i] = iq_rule_i16(x, scalar); }
    else { reinterpret_cast<int*>(out)[i] = iq_rule_i32(x, scalar); }
}
cudaError_t launch_export(const float* in, long long n, int type, float scalar, void* out, cudaStream_t s) {
    if (n <= 0) { return cudaSuccess; }
    k_export<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(in, n, type, scalar, out);
    return cudaGetLastError();
}
cudaError_t launch_iq_tap(const IqTapParams& p, cudaStream_t s) {
    if (p.n <= 0 || p.njobs <= 0) { return cudaSuccess; }
    const int grid = cdiv(cdiv(p.n, IQT_GROUP), IQT_THREADS);
    if (p.fmt == FMT_CF32) { k_iq_tap<FMT_CF32><<<grid, IQT_THREADS, 0, s>>>(p); }
    else if (p.fmt == FMT_CS16) { k_iq_tap<FMT_CS16><<<grid, IQT_THREADS, 0, s>>>(p); }
    else { k_iq_tap<FMT_CS8><<<grid, IQT_THREADS, 0, s>>>(p); }
    return cudaGetLastError();
}
// first index of the maximum VALUE (not magnitude) of n floats: volk_32f_index_max_32u.  One CTA; key = (value, -index).
__global__ void __launch_bounds__(1024) k_index_max(const float* __restrict__ in, long long n, float* __restrict__ out_val) {
    __shared__ float sv[32];
    __shared__ long long si[32];
    float best = -INFINITY;
    long long bi = 0x7fffffffffffffffLL;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const float v = __ldg(in + i);
        if (v > best || (v == best && i < bi)) { best = v; bi = i; }
    }
    for (int d = 16; d > 0; d >>= 1) {
        const float ov = __shfl_down_sync(0xffffffffu, best, d);
        const long long oi = __shfl_down_sync(0xffffffffu, bi, d);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x < 32) {
        best = (threadIdx.x < (blockDim.x >> 5)) ? sv[threadIdx.x] : -INFINITY;
        bi = (threadIdx.x < (blockDim.x >> 5)) ? si[threadIdx.x] : 0x7fffffffffffffffLL;
        for (int d = 16; d > 0; d >>= 1) {
            const float ov = __shfl_down_sync(0xffffffffu, best, d);
            const long long oi = __shfl_down_sync(0xffffffffu, bi, d);
            if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
        }
        if (threadIdx.x == 0) { *out_val = best; }
    }
}
cudaError_t launch_index_max(const float* in, long long n, float* out_val, cudaStream_t s) {
    k_index_max<<<1, 1024, 0, s>>>(in, n, out_val);
    return cudaGetLastError();
}

// start/len device arrays are supplied by the caller through `out`-adjacent scratch: see api.cpp
cudaError_t launch_zoom_hold_tbl(const float* line, const int* start, const int* len, int out_size, float* out,
                                 float* hold, float hold_speed, cudaStream_t s) {
    if (out_size <= 0) { return cudaSuccess; }
    k_zoom_hold<<<cdiv(out_size, 256), 256, 0, s>>>(line, start, len, out_size, out, hold, hold_speed);
    return cudaGetLastError();
}

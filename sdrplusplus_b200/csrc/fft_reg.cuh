// sdrplusplus_b200/csrc/fft_reg.cuh -- four-step FFT whose column / row transforms run in REGISTERS
// (included by kernels.cu after the shared-memory FFT; replaces it for N1, N2 in {256, 512, 1024}).
//
// A length-n transform, n = RA*RB (RA, RB in {16, 32}), is split once more:  x index = a*RB + b,  X index = c + RA*d
//   X[c + RA*d] = sum_b W_RB^(b d) * ( W_n^(b c) * sum_a x[a RB + b] W_RA^(a c) )
// step 1: thread b holds the RA samples x[a RB + b] and runs a radix-RA DIF in registers (constant twiddles, fully
//         unrolled), multiplies by W_n^(b c) and writes one shared-memory exchange tile;
// step 2: thread c reads its RB values back and runs the radix-RB transform.
// One shared-memory round trip and one barrier per transform instead of one per radix-8 pass; addresses are
// compile-time offsets.  The spectrum semantics (window * (-1)^n on load, 10 log10 |X/N|^2 in VOLK's log2 form on
// store: iq_frontend.cpp:248-266, 301) are those of k_fft_p1 / k_fft_p2.
#pragma once

__device__ constexpr float FR_COS[16] = { 1.000000000e+00f, 9.807852804e-01f, 9.238795325e-01f, 8.314696123e-01f, 7.071067812e-01f, 5.555702330e-01f,
                                          3.826834324e-01f, 1.950903220e-01f, 0.0f, -1.950903220e-01f, -3.826834324e-01f, -5.555702330e-01f,
                                          -7.071067812e-01f, -8.314696123e-01f, -9.238795325e-01f, -9.807852804e-01f };
__device__ constexpr float FR_SIN[16] = { 0.000000000e+00f, 1.950903220e-01f, 3.826834324e-01f, 5.555702330e-01f, 7.071067812e-01f, 8.314696123e-01f,
                                          9.238795325e-01f, 9.807852804e-01f, 1.0f, 9.807852804e-01f, 9.238795325e-01f, 8.314696123e-01f,
                                          7.071067812e-01f, 5.555702330e-01f, 3.826834324e-01f, 1.950903220e-01f };

// v * exp(-2 pi i K / R),  0 <= K < R/2,  R | 32
template <int R, int K>
__device__ __forceinline__ float2 fr_mul_w(float2 v) {
    constexpr int k32 = K * (32 / R);
    if constexpr (k32 == 0) { return v; }
    else if constexpr (k32 == 8) { return make_float2(v.y, -v.x); }
    else if constexpr (k32 == 4) { return make_float2((v.x + v.y) * RSQRT2, (v.y - v.x) * RSQRT2); }
    else if constexpr (k32 == 12) { return make_float2((v.y - v.x) * RSQRT2, -(v.x + v.y) * RSQRT2); }
    else {
        constexpr float c = FR_COS[k32], s = FR_SIN[k32];
        return make_float2(fmaf(v.y, s, v.x * c), fmaf(-v.x, s, v.y * c));
    }
}
// one radix-2 DIF stage of half-size H over a[0..R), butterfly I of R/2
template <int R, int H, int I>
__device__ __forceinline__ void fr_stage(float2 (&a)[R]) {
    constexpr int blk = I / H, j = I % H, i0 = blk * 2 * H + j;
    const float2 u = a[i0], v = a[i0 + H];
    a[i0] = make_float2(u.x + v.x, u.y + v.y);
    a[i0 + H] = fr_mul_w<2 * H, j>(make_float2(u.x - v.x, u.y - v.y));
    if constexpr (I + 1 < R / 2) { fr_stage<R, H, I + 1>(a); }
    else if constexpr (H > 1) { fr_stage<R, H / 2, 0>(a); }
}
// in-place forward DFT of R values; result index c is found at a[fr_brev<R>(c)]
template <int R>
__device__ __forceinline__ void fr_dft(float2 (&a)[R]) { fr_stage<R, R / 2, 0>(a); }
template <int R>
__host__ __device__ constexpr int fr_brev(int c) {
    int r = 0;
    for (int bit = 1; bit < R; bit <<= 1) { r = (r << 1) | ((c & bit) ? 1 : 0); }
    return r;
}
template <int RA, int RB> struct FrGeom {
    static constexpr int n = RA * RB;
    static constexpr int TP = RA > RB ? RA : RB;        // threads per transform
    static constexpr int crow = RB + 1;                  // exchange tile: element (c, b) at c*crow + b
    static constexpr int pitch = ((RA * crow + 13) / 16) * 16 + 2;   // == 2 (mod 16): adjacent transforms land 2 banks-pairs apart
};

// steps 1 + 2 of one length-n transform.  in: v[a] = x[a*RB + t] (threads t < RB); out: v[d'] with
// X[t + RA*d] = v[fr_brev<RB>(d)] (threads t < RA).  ex: this transform's exchange tile.
// twn[m] = exp(-2 pi i m / n) through the plan's table: tw[m << twsh], read from global memory (TAB = false) or from the
// CTA's shared-memory copy of the table (TAB = true)
template <int RA, int RB, bool TAB>
__device__ __forceinline__ void fr_transform(float2 (&v)[RA > RB ? RA : RB], float2* ex, int t, const float2* __restrict__ tw, int twsh) {
    using G = FrGeom<RA, RB>;
    if (t < RB) {
        float2 a[RA];
#pragma unroll
        for (int i = 0; i < RA; i++) { a[i] = v[i]; }
        fr_dft<RA>(a);
#pragma unroll
        for (int c = 0; c < RA; c++) {
            float2 y = a[fr_brev<RA>(c)];
            if (c > 0) { y = cmulf(y, TAB ? tw[(t * c) << twsh] : __ldg(tw + ((size_t)(t * c) << twsh))); }
            ex[c * G::crow + t] = y;
        }
    }
    __syncthreads();
    if (t < RA) {
        float2 b[RB];
#pragma unroll
        for (int i = 0; i < RB; i++) { b[i] = ex[t * G::crow + i]; }
        fr_dft<RB>(b);
#pragma unroll
        for (int i = 0; i < RB; i++) { v[i] = b[i]; }
    }
}

// copy n float2 (n even, both 16-byte aligned) from global into shared memory, the whole CTA
__device__ __forceinline__ void fr_stage_table(float2* dst, const float2* __restrict__ src, int n) {
    for (int i = threadIdx.x; i < n / 2; i += blockDim.x) {
        reinterpret_cast<float4*>(dst)[i] = __ldg(reinterpret_cast<const float4*>(src) + i);
    }
}
// shared memory of a register-FFT pass: the exchange tiles of its X transforms, then (TAB) the twiddle tables
template <int RA, int RB>
__host__ __device__ constexpr size_t fr_smem_tiles(int X) { return (size_t)X * FrGeom<RA, RB>::pitch; }

// pass 1: CTA = C adjacent columns n2, every row n1:  A[k1][n2] = W_N^(k1 n2) * sum_n1 x[n1 N2 + n2] W_N1^(n1 k1)
// TAB = false: twiddles and window straight from global memory (gathers).  TAB = true: the CTA first copies the coarse
// and fine twiddle tables (TW + N/TW float2, at most 16 KB) into shared memory -- the same fp32 values, so the same
// products -- and reads the window from the plan's per-thread layout (window_p) in 16-byte vectors.
// Registers: at most 144 with the tables (the least at which the 32 x 32 transform does not spill; DESIGN.md section 4 has
// what then fits on an SM); without them as before: 128 for a CTA of 8 transforms, unbounded for a CTA of 4.
template <int FMT, int RA, int RB, int C, bool TAB>
__global__ void __launch_bounds__(C * FrGeom<RA, RB>::TP) __maxnreg__(TAB ? 144 : (C == 8 ? 128 : 255)) k_fftr_p1(const __grid_constant__ FftPlanDev pl, const __grid_constant__ FftFrames fr,
                                                                    float2* __restrict__ work0) {
    using G = FrGeom<RA, RB>;
    extern __shared__ __align__(16) float2 smem[];
    const int N2 = pl.N2;
    const int f = blockIdx.y;
    float2* work = work0 + (size_t)f * pl.N;
    const int col = threadIdx.x % C, t = threadIdx.x / C;
    const int n2 = blockIdx.x * C + col;
    float2* const tws = smem + fr_smem_tiles<RA, RB>(C);      // [TW] coarse, then [N / TW] fine
    float2* const fine = tws + pl.TW;
    if (TAB) {
        fr_stage_table(tws, pl.tw, pl.TW);
        fr_stage_table(fine, pl.tw_fine, pl.N >> pl.logTW);
    }
    float2 v[G::TP];
    if (t < RB) {
        const FrameSrc fs = frame_src<FMT>(fr, f);
#pragma unroll
        for (int a = 0; a < RA; a++) { v[a] = load_frame<FMT>(pl, fs, (a * RB + t) * N2 + n2, !TAB); }
        if (TAB) {
            // window_p[(n2 RB + t) RA + a] = window[(a RB + t) N2 + n2], zero from nz on
            const float4* __restrict__ wp = reinterpret_cast<const float4*>(pl.window_p + ((size_t)n2 * RB + t) * RA);
#pragma unroll
            for (int q = 0; q < RA / 4; q++) {
                const float4 w = __ldg(wp + q);
                v[4 * q + 0] = make_float2(v[4 * q + 0].x * w.x, v[4 * q + 0].y * w.x);
                v[4 * q + 1] = make_float2(v[4 * q + 1].x * w.y, v[4 * q + 1].y * w.y);
                v[4 * q + 2] = make_float2(v[4 * q + 2].x * w.z, v[4 * q + 2].y * w.z);
                v[4 * q + 3] = make_float2(v[4 * q + 3].x * w.w, v[4 * q + 3].y * w.w);
            }
        }
    }
    if (TAB) { __syncthreads(); }
    fr_transform<RA, RB, TAB>(v, smem + col * G::pitch, t, TAB ? tws : pl.tw, pl.logTW - pl.logN1);
    if (t < RA) {
        // W_N^(k1 n2) = coarse[(k1 n2) >> s] * fine[(k1 n2) & (2^s - 1)],  coarse = tw (unit 1/TW), fine unit 1/N
        const int s = pl.logN - pl.logTW;
        const unsigned msk = (1u << s) - 1u;
#pragma unroll
        for (int d = 0; d < RB; d++) {
            const int k1 = t + RA * d;
            const unsigned e = (unsigned)k1 * (unsigned)n2;
            const float2 w = TAB ? cmulf(tws[e >> s], fine[e & msk]) : cmulf(__ldg(pl.tw + (e >> s)), __ldg(pl.tw_fine + (e & msk)));
            work[(size_t)k1 * N2 + n2] = cmulf(v[fr_brev<RB>(d)], w);
        }
    }
}

// pass 2: CTA = R adjacent rows k1:  X[k1 + N1 k2] = sum_n2 A[k1][n2] W_N2^(n2 k2); dB epilogue, transposed through
// shared memory so that the R rows' values of one k2 leave as one segment
// TAB: as in pass 1, the step-1 twiddles come from a shared-memory copy of tw
template <int RA, int RB, int R, bool TAB>
__global__ void __launch_bounds__(R * FrGeom<RA, RB>::TP) k_fftr_p2(const __grid_constant__ FftPlanDev pl, const float2* __restrict__ work0,
                                                                    float* __restrict__ out_db0) {
    using G = FrGeom<RA, RB>;
    extern __shared__ __align__(16) float2 smem[];
    const int N1 = pl.N1, N2 = pl.N2;
    const float2* work = work0 + (size_t)blockIdx.y * pl.N;
    float* out_db = out_db0 + (size_t)blockIdx.y * pl.N;
    const int t = threadIdx.x % G::TP, row = threadIdx.x / G::TP;
    const int r0 = blockIdx.x * R;
    float2* const tws = smem + fr_smem_tiles<RA, RB>(R);
    if (TAB) { fr_stage_table(tws, pl.tw, pl.TW); }
    float2 v[G::TP];
    if (t < RB) {
        const float2* __restrict__ p = work + (size_t)(r0 + row) * N2 + t;
#pragma unroll
        for (int a = 0; a < RA; a++) { v[a] = __ldg(p + a * RB); }
    }
    if (TAB) { __syncthreads(); }
    fr_transform<RA, RB, TAB>(v, smem + row * G::pitch, t, TAB ? tws : pl.tw, pl.logTW - pl.logN2);
    __syncthreads();                                    // every exchange tile has been read: reuse the space
    float* T = reinterpret_cast<float*>(smem);          // [k2][R + 1]
    const float nf = 1.0f / ((float)pl.N * (float)pl.N);
    if (t < RA) {
#pragma unroll
        for (int d = 0; d < RB; d++) { T[(t + RA * d) * (R + 1) + row] = power_db(v[fr_brev<RB>(d)], nf); }
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < G::n * R; idx += R * G::TP) {
        const int k2 = idx / R, rl = idx - k2 * R;
        out_db[(size_t)(r0 + rl) + (size_t)N1 * k2] = T[k2 * (R + 1) + rl];
    }
}

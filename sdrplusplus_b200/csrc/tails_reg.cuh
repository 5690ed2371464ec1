// sdrplusplus_b200/csrc/tails_reg.cuh -- the output-rate stages of a VFO with REGISTER windows (included by kernels.cu):
//   k_poly_reg<L,M>  multirate::PolyphaseResampler<complex_t>::process (polyphase_resampler.h:69-99) for the small L/M of the
//                    WFM / NFM plans: a thread produces one full period (L outputs from M inputs, every bank row once) while a
//                    register window slides one sample per tap -- 1 window load + L/4 tap loads per L packed FMAs
//   k_fir_reg        filter::FIR<complex_t,float>::process (fir.h:62-83; the RxVFO channel filter, rx_vfo.h:94-98): 8 consecutive
//                    outputs per thread, 8 taps per step: 4 window loads + 2 tap loads per 64 packed FMAs
//   k_firr_reg       filter::FIR<float,float>::process + LRToStereo (broadcast_fm.h:45,207-211; fm.h:84-93): two taps and two
//                    samples per packed FMA (even / odd tap sums, added at the end)
// All three stage their input ONCE per CTA with coalesced 16-byte loads into a padded shared-memory layout (groups of 32 or
// 64 bytes + 16 bytes of padding: the windows of neighbouring threads start an odd number of 16-byte slots apart, so every
// window load is conflict-free), keep the taps in shared memory as warp-wide broadcasts, and have no barrier after the fill.
// They replace the corresponding phases of k_tail_fused, whose ~14 barrier-separated phases per slab left the FMA pipe
// a quarter busy.
#pragma once

#define TR_THREADS 128

// ------------------------------------------------------------------------------------------------ polyphase resampler
template <int L, int M>
struct PolyGeom {
    static constexpr int W = ((L - 1) * M) / L + 1;          // window: samples the L outputs of a period reach at one tap
    __host__ __device__ static constexpr int off(int i) { return (i * M) / L; }  // input offset of output i of a period (period aligned to phase 0)
    __host__ __device__ static constexpr int ph(int i) { return (i * M) % L; }   // its bank row
};

// bank_kl: [tpp][L] (row k = tap k of every phase).  Output m of the chunk: t = phase0 + m M, row t % L, window at offset0 + t / L.
// The taps of a period are split over the PR_SPLIT warps of the CTA (warp q: taps [q KS, (q + 1) KS)), which quarters the serial
// chain of a thread (16 outputs x 119 taps in the WFM plan) and gives the kernel four times the warps; the partial sums meet in
// shared memory, warp q finishing outputs [q L/4, (q + 1) L/4) of each period, always in the same order.
#define PR_SPLIT 4
#define PR_PER 32                                                     // periods per CTA (one per lane)
template <int L, int M>
__global__ void __launch_bounds__(TR_THREADS) k_poly_reg(const __grid_constant__ PolyParams p) {
    using G = PolyGeom<L, M>;
    extern __shared__ __align__(16) float2 tr_sm[];
    const PolyJob& J = p.job[blockIdx.y];
    pdl_trigger();
    const int tpp = J.tpp;
    // periods are aligned to the outputs whose phase is 0: m_a = first such output index (0 <= m_a < L)
    int m_a = 0;
    while (((J.phase0 + m_a * M) % L) != 0) { m_a++; }
    const int g0 = blockIdx.x * PR_PER;                               // first period of this CTA (period g: outputs m_a - L + g L + i)
    const long long mfirst = (long long)m_a - L + (long long)g0 * L;
    if (mfirst >= J.n_out) { return; }
    // input index (into J.in) of the first sample of period g0
    const long long b0 = (long long)J.offset0 + ((long long)J.phase0 + mfirst * M) / L;    // exact: the numerator is a multiple of L
    float* bank = reinterpret_cast<float*>(tr_sm);                    // [tpp][L]
    const int bank_f = (tpp * L + 3) & ~3;
    float2* X = tr_sm + bank_f / 2;                                   // natural order, sample j of the tile at X[j]
    const int nx = (PR_PER - 1) * M + G::W + tpp;                     // samples the tile reads
    float2* red = X + ((nx + G::W + 9) & ~1);                         // [PR_SPLIT][L][PR_PER] partial sums
    for (int i = threadIdx.x; i < (tpp * L + 3) / 4; i += TR_THREADS) {
        reinterpret_cast<float4*>(bank)[i] = __ldg(reinterpret_cast<const float4*>(J.bank_kl) + i);
    }
    {
        // 8-byte elements at an arbitrary (possibly odd) start: plain coalesced loads; indices before the buffer (period 0 of
        // a chunk can start in front of the oldest history sample: those outputs are never stored) read as zero
        const long long lim = J.in_len;
        pdl_wait();
        for (int j = threadIdx.x; j < nx + G::W; j += TR_THREADS) {
            const long long s = b0 + j;
            X[j] = (j < nx && s >= 0 && s < lim) ? __ldcg(J.in + s) : make_float2(0.0f, 0.0f);
        }
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, q = threadIdx.x >> 5;
    const long long m0 = mfirst + (long long)lane * L;                // this lane's period
    float2 acc[L];
#pragma unroll
    for (int i = 0; i < L; i++) { acc[i] = make_float2(0.0f, 0.0f); }
    const int KS = (tpp + PR_SPLIT - 1) / PR_SPLIT;
    const int kbeg = q * KS, kend = min(tpp, kbeg + KS);              // this warp's taps
    if (m0 < J.n_out && kbeg < kend) {
        const float2* xw = X + lane * M + kbeg;                       // lane stride M samples: M odd -> conflict-free 8-byte loads
        float2 win[G::W];
#pragma unroll
        for (int j = 0; j < G::W; j++) { win[j] = xw[j]; }
        // tap kbeg + k: output i reads sample off(i) + k of xw = window slot (off(i) + k) % W after k slides
        const int nk = kend - kbeg;
        int k0 = 0;
        for (; k0 + G::W <= nk; k0 += G::W) {
#pragma unroll
            for (int kk = 0; kk < G::W; kk++) {
                const float* hk = bank + (kbeg + k0 + kk) * L;
                float h[L];
                if constexpr ((L & 3) == 0) {                         // rows of whole float4: broadcast 16-byte loads
#pragma unroll
                    for (int v = 0; v < L / 4; v++) {
                        const float4 t4 = reinterpret_cast<const float4*>(hk)[v];
                        h[4 * v] = t4.x; h[4 * v + 1] = t4.y; h[4 * v + 2] = t4.z; h[4 * v + 3] = t4.w;
                    }
                }
                else {
#pragma unroll
                    for (int v = 0; v < L; v++) { h[v] = hk[v]; }
                }
#pragma unroll
                for (int i = 0; i < L; i++) { acc[i] = ffma2(make_float2(h[G::ph(i)], h[G::ph(i)]), win[(G::off(i) + kk) % G::W], acc[i]); }
                win[kk] = xw[k0 + kk + G::W];                         // slot kk held sample k0 + kk: now the one W further on
            }
        }
#pragma unroll
        for (int kk = 0; kk < G::W; kk++) {
            if (k0 + kk < nk) {
                const float* hk = bank + (kbeg + k0 + kk) * L;
#pragma unroll
                for (int i = 0; i < L; i++) { acc[i] = ffma2(make_float2(hk[G::ph(i)], hk[G::ph(i)]), win[(G::off(i) + kk) % G::W], acc[i]); }
                win[kk] = xw[k0 + kk + G::W];
            }
        }
    }
#pragma unroll
    for (int i = 0; i < L; i++) { red[(q * L + i) * PR_PER + lane] = acc[i]; }
    __syncthreads();
    // warp q finishes outputs i = q, q + PR_SPLIT, ... of every period: ((p0 + p1) + (p2 + p3))
    for (int i = q; i < L; i += PR_SPLIT) {
        const long long m = m0 + i;
        if (m >= 0 && m < J.n_out) {
            const float2 a0 = red[(0 * L + i) * PR_PER + lane], a1 = red[(1 * L + i) * PR_PER + lane];
            const float2 a2 = red[(2 * L + i) * PR_PER + lane], a3 = red[(3 * L + i) * PR_PER + lane];
            J.out[m] = make_float2((a0.x + a1.x) + (a2.x + a3.x), (a0.y + a1.y) + (a2.y + a3.y));
        }
    }
}
template <int L, int M>
static cudaError_t launch_poly_reg_t(const PolyParams& p, int max_tpp, const KernelOpts& o, cudaStream_t s) {
    using G = PolyGeom<L, M>;
    static_assert(TR_THREADS == PR_SPLIT * 32, "one warp per tap range");
    const size_t nx = (size_t)(PR_PER - 1) * M + G::W + max_tpp;
    const size_t smem = ((size_t)((max_tpp * L + 3) & ~3) / 2 + ((nx + G::W + 9) & ~(size_t)1) + (size_t)PR_SPLIT * L * PR_PER + 8) * sizeof(float2);
    if ((int)smem > kernels_max_smem_optin()) { return cudaErrorInvalidValue; }
    cudaError_t e = set_smem(k_poly_reg<L, M>, smem);
    if (e != cudaSuccess) { return e; }
    const int periods = (p.max_out + L - 1) / L + 1;
    dim3 grid((unsigned)((periods + PR_PER - 1) / PR_PER), (unsigned)p.njobs);
    return launch_chain(k_poly_reg<L, M>, grid, dim3(TR_THREADS), smem, o, s, p);
}
bool poly_reg_supported(int L, int M) {
    return (L == 16 && M == 25) || (L == 5 && M == 6) || (L == 2 && M == 3) || (L == 4 && M == 5) || (L == 2 && M == 5);
}
// every job of p: the same (interp, decim)
cudaError_t launch_poly_reg(const PolyParams& p, const KernelOpts& o, cudaStream_t s) {
    if (p.njobs <= 0 || p.max_out <= 0) { return cudaSuccess; }
    const int L = p.job[0].interp, M = p.job[0].decim;
    int max_tpp = 0;
    for (int v = 0; v < p.njobs; v++) { max_tpp = p.job[v].tpp > max_tpp ? p.job[v].tpp : max_tpp; }
    if (L == 16 && M == 25) { return launch_poly_reg_t<16, 25>(p, max_tpp, o, s); }
    if (L == 5 && M == 6) { return launch_poly_reg_t<5, 6>(p, max_tpp, o, s); }
    if (L == 2 && M == 3) { return launch_poly_reg_t<2, 3>(p, max_tpp, o, s); }
    if (L == 4 && M == 5) { return launch_poly_reg_t<4, 5>(p, max_tpp, o, s); }
    if (L == 2 && M == 5) { return launch_poly_reg_t<2, 5>(p, max_tpp, o, s); }
    return cudaErrorInvalidValue;
}

// ------------------------------------------------------------------------------------------------ complex FIR, decimation 1
// out[m] = sum_k taps[k] in[offset + m + k].  Layout: groups of 8 samples (4 float4) + 1 float4 of padding.
#define FRG_R 8
__device__ __forceinline__ void frg_block(float2 (&acc)[FRG_R], const float2 (&lo)[8], float2 (&hi)[8], const float4* nxt, const float* taps) {
    const float4 t0 = *reinterpret_cast<const float4*>(taps), t1 = *reinterpret_cast<const float4*>(taps + 4);
    const float h[8] = { t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w };
#pragma unroll
    for (int v = 0; v < 4; v++) {
        const float4 q = nxt[v];
        hi[2 * v] = make_float2(q.x, q.y);
        hi[2 * v + 1] = make_float2(q.z, q.w);
    }
#pragma unroll
    for (int k = 0; k < 8; k++) {
#pragma unroll
        for (int i = 0; i < FRG_R; i++) {
            const int j = k + i;
            acc[i] = ffma2(make_float2(h[k], h[k]), j < 8 ? lo[j] : hi[j - 8], acc[i]);
        }
    }
}
// The 8-tap steps of a filter are split over the TS_SPLIT warps of the CTA (a lane = 8 consecutive outputs, a warp = a quarter of
// the taps): four times the warps and a quarter of the serial chain per thread; partial sums meet in shared memory.
#define TS_SPLIT 4
#define TS_TILE (32 * FRG_R)                                         // outputs per CTA
__global__ void __launch_bounds__(TR_THREADS) k_fir_reg(const __grid_constant__ FirParams p) {
    extern __shared__ __align__(16) float2 tr_sm[];
    const FirJob& J = p.job[blockIdx.y];
    pdl_trigger();
    const int mt = blockIdx.x * TS_TILE;
    if (mt >= J.n_out) { return; }
    const int T = J.ntaps;
    const long long first = (long long)J.offset + mt;
    const int sh = (int)(first & 1);                                  // odd start: begin one sample early, one leading zero tap
    const int Tp = (T + sh + 7) & ~7;                                 // taps incl. the shift, padded to whole steps of 8
    float* ts = reinterpret_cast<float*>(tr_sm);                      // [Tp + 8]
    float4* X4 = reinterpret_cast<float4*>(tr_sm + (Tp + 8) / 2);     // groups: 5 float4 per 8 samples
    const int npairs = (TS_TILE + Tp + 8) / 2;                        // pairs the windows can touch
    float2* red = reinterpret_cast<float2*>(X4 + ((npairs + 3) / 4 + 1) * 5);      // [TS_SPLIT][32 lanes][9]
    for (int k = threadIdx.x; k < Tp + 8; k += TR_THREADS) {
        const int kt = k - sh;
        ts[k] = (kt >= 0 && kt < T) ? __ldg(J.taps + kt) : 0.0f;
    }
    {
        const int nout = min(TS_TILE, J.n_out - mt);
        const int need = (nout + T - 1 + sh + 1) / 2;                 // pairs that hold data an output needs
        const float4* __restrict__ src = reinterpret_cast<const float4*>(J.in + (first - sh));
        pdl_wait();
        for (int i = threadIdx.x; i < npairs; i += TR_THREADS) {
            X4[(i >> 2) * 5 + (i & 3)] = (i < need) ? __ldcg(src + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, q = threadIdx.x >> 5;
    const int m0 = mt + lane * FRG_R;
    const int nb = Tp >> 3, nbq = (nb + TS_SPLIT - 1) / TS_SPLIT;
    const int kb0 = q * nbq, kb1 = min(nb, kb0 + nbq);                // this warp's steps
    float2 acc[FRG_R];
#pragma unroll
    for (int i = 0; i < FRG_R; i++) { acc[i] = make_float2(0.0f, 0.0f); }
    if (m0 < J.n_out && kb0 < kb1) {
        const float4* xg = X4 + (lane + kb0) * 5;                     // this thread's first group; step kb reads group kb + 1
        const float* tq = ts + kb0 * 8;
        float2 a[8], b[8];
#pragma unroll
        for (int v = 0; v < 4; v++) {
            const float4 t4 = xg[v];
            a[2 * v] = make_float2(t4.x, t4.y);
            a[2 * v + 1] = make_float2(t4.z, t4.w);
        }
        const int n = kb1 - kb0;
        int kb = 0;
        for (; kb + 1 < n; kb += 2) {
            frg_block(acc, a, b, xg + (kb + 1) * 5, tq + kb * 8);
            frg_block(acc, b, a, xg + (kb + 2) * 5, tq + kb * 8 + 8);
        }
        if (kb < n) { frg_block(acc, a, b, xg + (kb + 1) * 5, tq + kb * 8); }
    }
#pragma unroll
    for (int i = 0; i < FRG_R; i++) { red[(q * 32 + lane) * 9 + i] = acc[i]; }
    __syncthreads();
    // thread t finishes outputs t and t + 128 of the tile: ((p0 + p1) + (p2 + p3)), consecutive threads consecutive outputs
#pragma unroll
    for (int h = 0; h < TS_TILE / TR_THREADS; h++) {
        const int o = threadIdx.x + h * TR_THREADS;
        if (mt + o < J.n_out) {
            const int idx = (o >> 3) * 9 + (o & 7);
            const float2 a0 = red[idx], a1 = red[32 * 9 + idx], a2 = red[2 * 32 * 9 + idx], a3 = red[3 * 32 * 9 + idx];
            J.out[mt + o] = make_float2((a0.x + a1.x) + (a2.x + a3.x), (a0.y + a1.y) + (a2.y + a3.y));
        }
    }
}
// every job: decimation 1
cudaError_t launch_fir_reg(const FirParams& p, const KernelOpts& o, cudaStream_t s) {
    if (p.njobs <= 0 || p.max_out <= 0) { return cudaSuccess; }
    int maxT = 0;
    for (int v = 0; v < p.njobs; v++) { maxT = p.job[v].ntaps > maxT ? p.job[v].ntaps : maxT; }
    const int Tp = (maxT + 1 + 7) & ~7;
    const size_t smem = ((size_t)(Tp + 8) / 2 + ((size_t)(TS_TILE + Tp + 8) / 8 + 3) * 10 + (size_t)TS_SPLIT * 32 * 9 + 8) * sizeof(float2);
    if ((int)smem > kernels_max_smem_optin()) { return cudaErrorInvalidValue; }
    cudaError_t e = set_smem(k_fir_reg, smem);
    if (e != cudaSuccess) { return e; }
    dim3 grid((unsigned)((p.max_out + TS_TILE - 1) / TS_TILE), (unsigned)p.njobs);
    return launch_chain(k_fir_reg, grid, dim3(TR_THREADS), smem, o, s, p);
}

// ------------------------------------------------------------------------------------------------ real FIR (+ mono -> stereo)
// out[m] = sum_k taps[k] in[m + k].  A packed FMA takes the tap pair (h[2j], h[2j+1]) and the sample pair (x[m+2j], x[m+2j+1]):
// even-aligned pairs for even m, odd-aligned pairs (a second copy of the tile, shifted by one sample) for odd m; the two
// halves of the accumulator (even-tap sum, odd-tap sum) are added at the end.
// Layout of both copies: groups of 4 pairs (2 float4) + 1 float4 of padding.
__device__ __forceinline__ void frr_block(float2 (&acc)[8], const float2 (&elo)[4], float2 (&ehi)[4], const float2 (&olo)[4], float2 (&ohi)[4],
                                          const float4* enxt, const float4* onxt, const float* taps) {
    const float4 t0 = *reinterpret_cast<const float4*>(taps), t1 = *reinterpret_cast<const float4*>(taps + 4);
    const float2 h[4] = { make_float2(t0.x, t0.y), make_float2(t0.z, t0.w), make_float2(t1.x, t1.y), make_float2(t1.z, t1.w) };
#pragma unroll
    for (int v = 0; v < 2; v++) {
        const float4 q = enxt[v], r = onxt[v];
        ehi[2 * v] = make_float2(q.x, q.y); ehi[2 * v + 1] = make_float2(q.z, q.w);
        ohi[2 * v] = make_float2(r.x, r.y); ohi[2 * v + 1] = make_float2(r.z, r.w);
    }
#pragma unroll
    for (int j = 0; j < 4; j++) {                                     // tap pair j of this step
#pragma unroll
        for (int i = 0; i < 4; i++) {                                 // outputs m0 + 2 i (even copy) and m0 + 2 i + 1 (odd copy)
            const int w = j + i;
            acc[2 * i] = ffma2(h[j], w < 4 ? elo[w] : ehi[w - 4], acc[2 * i]);
            acc[2 * i + 1] = ffma2(h[j], w < 4 ? olo[w] : ohi[w - 4], acc[2 * i + 1]);
        }
    }
}
__global__ void __launch_bounds__(TR_THREADS) k_firr_reg(const __grid_constant__ FirRParams p) {
    extern __shared__ __align__(16) float2 tr_sm[];
    const FirRJob& J = p.job[blockIdx.y];
    pdl_trigger();
    const int mt = blockIdx.x * TS_TILE;
    if (mt >= J.n_out) { return; }
    const int T = J.ntaps;
    const int Tp = (T + 7) & ~7;
    float* ts = reinterpret_cast<float*>(tr_sm);                      // [Tp + 8]
    const int npairs = (TS_TILE + Tp + 8) / 2 + 4;                    // pairs per copy
    const int ngroups = (npairs + 3) / 4 + 1;
    float4* E4 = reinterpret_cast<float4*>(tr_sm + (Tp + 8) / 2);     // even copy: pair q = (x[2q], x[2q+1])
    float4* O4 = E4 + ngroups * 3;                                    // odd copy:  pair q = (x[2q+1], x[2q+2])
    float* red = reinterpret_cast<float*>(O4 + ngroups * 3);          // [TS_SPLIT][32 lanes][9]
    for (int k = threadIdx.x; k < Tp + 8; k += TR_THREADS) { ts[k] = (k < T) ? __ldg(J.taps + k) : 0.0f; }
    {
        const int nout = min(TS_TILE, J.n_out - mt);
        const int need = nout + T - 1;                                // samples that hold data
        const float* __restrict__ src = J.in + mt;                    // 4-byte elements, any alignment: scalar loads
        float* Ef = reinterpret_cast<float*>(E4);
        float* Of = reinterpret_cast<float*>(O4);
        pdl_wait();
        for (int n = threadIdx.x; n < 2 * npairs; n += TR_THREADS) {
            const float v = (n < need) ? __ldcg(src + n) : 0.0f;
            // pair q lives in group q >> 2 (12 floats per group), slot q & 3
            const int qe = n >> 1;
            Ef[(qe >> 2) * 12 + (qe & 3) * 2 + (n & 1)] = v;
            if (n >= 1) {
                const int qo = (n - 1) >> 1;
                Of[(qo >> 2) * 12 + (qo & 3) * 2 + ((n - 1) & 1)] = v;
            }
        }
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, q = threadIdx.x >> 5;
    const int m0 = mt + lane * 8;
    const int nb = Tp >> 3, nbq = (nb + TS_SPLIT - 1) / TS_SPLIT;
    const int kb0 = q * nbq, kb1 = min(nb, kb0 + nbq);                // this warp's steps of 8 taps
    float2 acc[8];
#pragma unroll
    for (int i = 0; i < 8; i++) { acc[i] = make_float2(0.0f, 0.0f); }
    if (m0 < J.n_out && kb0 < kb1) {
        const float4* eg = E4 + (lane + kb0) * 3;                     // thread stride: 4 pairs = one group (3 float4 incl. padding)
        const float4* og = O4 + (lane + kb0) * 3;
        const float* tq = ts + kb0 * 8;
        float2 ea[4], eb[4], oa[4], ob[4];
#pragma unroll
        for (int v = 0; v < 2; v++) {
            const float4 t4 = eg[v], r = og[v];
            ea[2 * v] = make_float2(t4.x, t4.y); ea[2 * v + 1] = make_float2(t4.z, t4.w);
            oa[2 * v] = make_float2(r.x, r.y); oa[2 * v + 1] = make_float2(r.z, r.w);
        }
        const int n = kb1 - kb0;
        int kb = 0;
        for (; kb + 1 < n; kb += 2) {
            frr_block(acc, ea, eb, oa, ob, eg + (kb + 1) * 3, og + (kb + 1) * 3, tq + kb * 8);
            frr_block(acc, eb, ea, ob, oa, eg + (kb + 2) * 3, og + (kb + 2) * 3, tq + kb * 8 + 8);
        }
        if (kb < n) { frr_block(acc, ea, eb, oa, ob, eg + (kb + 1) * 3, og + (kb + 1) * 3, tq + kb * 8); }
    }
#pragma unroll
    for (int i = 0; i < 8; i++) { red[(q * 32 + lane) * 9 + i] = acc[i].x + acc[i].y; }
    __syncthreads();
#pragma unroll
    for (int h = 0; h < TS_TILE / TR_THREADS; h++) {
        const int o = threadIdx.x + h * TR_THREADS;
        if (mt + o < J.n_out) {
            const int idx = (o >> 3) * 9 + (o & 7);
            const float v = (red[idx] + red[32 * 9 + idx]) + (red[2 * 32 * 9 + idx] + red[3 * 32 * 9 + idx]);
            if (J.stereo) { reinterpret_cast<float2*>(J.out)[mt + o] = make_float2(v, v); }
            else { J.out[mt + o] = v; }
        }
    }
}
cudaError_t launch_firr_reg(const FirRParams& p, const KernelOpts& o, cudaStream_t s) {
    if (p.njobs <= 0 || p.max_out <= 0) { return cudaSuccess; }
    int maxT = 0;
    for (int v = 0; v < p.njobs; v++) { maxT = p.job[v].ntaps > maxT ? p.job[v].ntaps : maxT; }
    const int Tp = (maxT + 7) & ~7;
    const int npairs = (TS_TILE + Tp + 8) / 2 + 4;
    const int ngroups = (npairs + 3) / 4 + 1;
    const size_t smem = ((size_t)(Tp + 8) / 2 + (size_t)ngroups * 3 * 2 * 2 + (size_t)TS_SPLIT * 32 * 9 / 2 + 8) * sizeof(float2);
    if ((int)smem > kernels_max_smem_optin()) { return cudaErrorInvalidValue; }
    cudaError_t e = set_smem(k_firr_reg, smem);
    if (e != cudaSuccess) { return e; }
    dim3 grid((unsigned)((p.max_out + TS_TILE - 1) / TS_TILE), (unsigned)p.njobs);
    return launch_chain(k_firr_reg, grid, dim3(TR_THREADS), smem, o, s, p);
}

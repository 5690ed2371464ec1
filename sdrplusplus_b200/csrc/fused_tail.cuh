// sdrplusplus_b200/csrc/fused_tail.cuh -- k_tail_fused: all FIR-like stages after stage 1 of a VFO in one launch
// (included by kernels.cu; descriptors and the shared host/device range arithmetic are in kernels.cuh).
//
// Replaces, for one VFO and one chunk, the per-stage launches of
//   DecimatingFIR stages 2..k        (power_decimator.h:58-65, decimating_fir.h:45-68)
//   PolyphaseResampler               (polyphase_resampler.h:69-99)
//   FIR<complex_t,float>             (rx_vfo.h:28-31 channel filter, fir.h:62-83)
//   Quadrature                       (quadrature.h:39-46)
//   FIR<float,float> + LRToStereo    (broadcast_fm.h:45, fm.h:123)
// Shared-memory arena: stage s's input lives at float offset st[s].buf in a PHASE-MAJOR layout -- sample i of the
// range sits in row (i - o) % D, column (i - o) / D, D the stage's decimation -- so that a thread producing FT_R
// consecutive outputs slides one register window along a row per tap phase: one LDS per FT_R packed FMAs.
// Taps are stored phase-major too (row r = taps[q*D + r]) and read as warp-wide broadcasts.
#pragma once

struct FtLay { int o, D, pitch, sh; };     // sh = log2(D) when D is a power of two, else -1

__device__ __forceinline__ FtLay ft_make_lay(const FtStage& S, int lo) {
    FtLay l;
    l.o = ft_origin(S, lo);
    l.D = ft_rows(S);
    l.pitch = S.pitch;
    l.sh = (l.D & (l.D - 1)) ? -1 : (31 - __clz(l.D));
    return l;
}
__device__ __forceinline__ int ft_lidx(const FtLay& l, int i) {
    const int rel = i - l.o;
    if (l.D == 1) { return rel; }
    if (l.sh >= 0) { return (rel & (l.D - 1)) * l.pitch + (rel >> l.sh); }
    const int j = rel / l.D;
    return (rel - j * l.D) * l.pitch + j;
}

__device__ __forceinline__ float2 ft_fma(float h, float2 x, float2 a) { return ffma2(make_float2(h, h), x, a); }
__device__ __forceinline__ float ft_fma(float h, float x, float a) { return fmaf(h, x, a); }
__device__ __forceinline__ void ft_zero(float2& a) { a = make_float2(0.0f, 0.0f); }
__device__ __forceinline__ void ft_zero(float& a) { a = 0.0f; }

// one block of N taps: all loads first (taps + the window refills), then N * R independent multiply-adds.
// The last block of a run needs only the refills its own later taps read (N - 1 of them).
template <typename T, int R, int N, bool LAST>
__device__ __forceinline__ void ft_blk(T (&acc)[R], T (&w)[R], const T* __restrict__ X, const float* __restrict__ taps) {
    constexpr int NR = LAST ? N - 1 : N;
    float h[N];
    T nw[NR > 0 ? NR : 1];
#pragma unroll
    for (int k = 0; k < N; k++) { h[k] = taps[k]; }
#pragma unroll
    for (int k = 0; k < NR; k++) { nw[k] = X[k + R]; }
#pragma unroll
    for (int k = 0; k < N; k++) {
#pragma unroll
        for (int i = 0; i < R; i++) { acc[i] = ft_fma(h[k], w[(k + i) % R], acc[i]); }
        if (k < NR) { w[k] = nw[k]; }
    }
}
template <typename T, int R, int N>
__device__ __forceinline__ void ft_tail_blk(T (&acc)[R], T (&w)[R], const T* __restrict__ X, const float* __restrict__ taps, int n) {
    if constexpr (N <= R) {
        if (n == N) { ft_blk<T, R, N, true>(acc, w, X, taps); }
        else { ft_tail_blk<T, R, N + 1>(acc, w, X, taps, n); }
    }
}
// acc[i] += sum_{q < Q} taps[q] * X[i + q],  Q >= 1
template <typename T, int R>
__device__ __forceinline__ void ft_firx(T (&acc)[R], const T* __restrict__ X, const float* __restrict__ taps, int Q) {
    T w[R];
#pragma unroll
    for (int i = 0; i < R; i++) { w[i] = X[i]; }
    int q0 = 0;
    for (; q0 + R < Q; q0 += R) { ft_blk<T, R, R, false>(acc, w, X + q0, taps + q0); }
    ft_tail_blk<T, R, 1>(acc, w, X + q0, taps + q0, Q - q0);
}

// where a stage's outputs go: the next stage's shared-memory buffer, or global memory for the last stage
struct FtDst {
    float* g;           // non-null: global
    float* sp;          // shared buffer base
    FtLay lay;
    int dup;
    __device__ __forceinline__ void put2(int m, float2 v) const {
        if (g) { reinterpret_cast<float2*>(g)[m] = v; }
        else { reinterpret_cast<float2*>(sp)[ft_lidx(lay, m)] = v; }
    }
    __device__ __forceinline__ void put1(int m, float v) const {
        if (dup) { put2(m, make_float2(v, v)); }
        else if (g) { g[m] = v; }
        else { sp[ft_lidx(lay, m)] = v; }
    }
    // R consecutive outputs m .. m+R-1 (those below mend): one division, then a (row, column) cursor
    template <int R>
    __device__ __forceinline__ void put2_run(int m, int mend, const float2 (&v)[R]) const {
        if (g) {
#pragma unroll
            for (int i = 0; i < R; i++) { if (m + i < mend) { reinterpret_cast<float2*>(g)[m + i] = v[i]; } }
            return;
        }
        float2* b = reinterpret_cast<float2*>(sp);
        if (lay.D == 1) {
#pragma unroll
            for (int i = 0; i < R; i++) { if (m + i < mend) { b[m - lay.o + i] = v[i]; } }
            return;
        }
        const int rel = m - lay.o;
        int j = rel / lay.D, r = rel - j * lay.D;
        int idx = r * lay.pitch + j;
#pragma unroll
        for (int i = 0; i < R; i++) {
            if (m + i < mend) { b[idx] = v[i]; }
            r++; idx += lay.pitch;
            if (r == lay.D) { r = 0; idx -= lay.D * lay.pitch - 1; }
        }
    }
};

// Outputs per thread of a phase: the phases of a slab run one after the other, so what a phase costs is
// rounds * (instructions of one unit); fewer outputs per thread give more units (all threads busy, fewer rounds)
// at more loads per multiply-add.  qtot = taps a unit walks through, rows = register-window restarts.
template <int MAXR>
__device__ __forceinline__ int ft_pick_r(int nout, int groups, int nthreads, int qtot, int rows) {
    int best = 5, best_cost = 0x7fffffff;
#pragma unroll
    for (int R = 5; R <= MAXR; R += 4) {
        const int units = groups * ((nout + R - 1) / R);
        const int rounds = (units + nthreads - 1) / nthreads;
        const int cost = rounds * (qtot * (R + 2) + rows * (R + 12) + 40);
        if (cost < best_cost) { best_cost = cost; best = R; }
    }
    return best;
}

template <int R, int NT>
__device__ __forceinline__ void ft_phase_firc(const FtStage& S, const FtLay& ls, const FtDst& dst, const float* sm, const float* xb, int t0, int t1) {
    const float2* X = reinterpret_cast<const float2*>(xb);
    const float* tp = sm + S.tap_off;
    const int D = S.D, T = S.T;
    const int m_o = (ls.o - (S.off - (T - 1))) / D;       // exact for D > 1; D == 1: o - c
    const int qf = T / D, rem = T - qf * D;
    const int units = (t1 - t0 + R - 1) / R;
    for (int u = threadIdx.x; u < units; u += NT) {
        const int m = t0 + u * R;
        const int pos = m - m_o;
        float2 acc[R];
#pragma unroll
        for (int i = 0; i < R; i++) { ft_zero(acc[i]); }
        for (int r = 0; r < D; r++) { ft_firx<float2, R>(acc, X + r * ls.pitch + pos, tp + r * S.qpitch, qf + (r < rem ? 1 : 0)); }
        dst.put2_run<R>(m, t1, acc);
    }
}
template <int R, int NT>
__device__ __forceinline__ void ft_phase_firr(const FtStage& S, const FtLay& ls, const FtDst& dst, const float* sm, const float* xb, int t0, int t1) {
    const float* tp = sm + S.tap_off;
    const int m_o = ls.o - (S.off - (S.T - 1));
    const int units = (t1 - t0 + R - 1) / R;
    for (int u = threadIdx.x; u < units; u += NT) {
        const int m = t0 + u * R;
        float acc[R];
#pragma unroll
        for (int i = 0; i < R; i++) { ft_zero(acc[i]); }
        ft_firx<float, R>(acc, xb + (m - m_o), tp, S.T);
#pragma unroll
        for (int i = 0; i < R; i++) {
            if (m + i < t1) { dst.put1(m + i, acc[i]); }
        }
    }
}
// per-class constants of the polyphase phase (class = output index mod L: same bank row, inputs M apart)
struct FtPolyClass { int m_c, cnt, ph, a, bb; };
template <int R, int NT>
__device__ __forceinline__ void ft_phase_poly(const FtStage& S, const FtLay& ls, const FtDst& dst, const float* sm, const float* xb,
                                              const FtPolyClass* cls, int t0, int t1) {
    const float2* X = reinterpret_cast<const float2*>(xb);
    const float* tp = sm + S.tap_off;
    const int L = S.L, M = S.D, tpp = S.T;
    const int qf = tpp / M, qrem = tpp - qf * M;
    const int per_class = (t1 - t0 + L - 1) / L;
    const int gmax = (per_class + R - 1) / R;
    for (int u = threadIdx.x; u < L * gmax; u += NT) {
        const int c = u / gmax, g = u - c * gmax;
        const FtPolyClass pc = cls[c];
        const int jj0 = g * R;
        if (jj0 >= pc.cnt) { continue; }
        float2 acc[R];
#pragma unroll
        for (int i = 0; i < R; i++) { ft_zero(acc[i]); }
        const float2* Xc = X + pc.a + jj0;
        const float* tc = tp + pc.ph * M * S.qpitch;
        // rows r >= bb read bank row r - bb at column offset 0; rows r < bb read bank row r - bb + M one column later
        for (int r = pc.bb; r < M; r++) {
            const int rp = r - pc.bb;
            const int Q = qf + (rp < qrem ? 1 : 0);
            if (Q > 0) { ft_firx<float2, R>(acc, Xc + r * ls.pitch, tc + rp * S.qpitch, Q); }
        }
        for (int r = 0; r < pc.bb; r++) {
            const int rp = r - pc.bb + M;
            const int Q = qf + (rp < qrem ? 1 : 0);
            if (Q > 0) { ft_firx<float2, R>(acc, Xc + r * ls.pitch + 1, tc + rp * S.qpitch, Q); }
        }
#pragma unroll
        for (int i = 0; i < R; i++) {
            if (jj0 + i < pc.cnt) { dst.put2(pc.m_c + (jj0 + i) * L, acc[i]); }
        }
    }
}
#define FT_MAX_L 64      // polyphase interpolation factors above this stay on the per-stage kernels

// ---- cp.async.bulk (TMA, one-dimensional) + mbarrier, for the direct first stage ----
__device__ __forceinline__ void ft_mbar_init(unsigned long long* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void ft_bulk_load(float* smem_dst, const void* gsrc, unsigned bytes, unsigned long long* bar) {
    const unsigned b = (unsigned)__cvta_generic_to_shared(bar), d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(b), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
                 ::"r"(d), "l"(gsrc), "r"(bytes), "r"(b) : "memory");
}
__device__ __forceinline__ void ft_mbar_wait(unsigned long long* bar, unsigned parity) {
    const unsigned b = (unsigned)__cvta_generic_to_shared(bar);
    asm volatile("{\n.reg .pred p;\nFT_WAIT_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@!p bra FT_WAIT_%=;\n}\n" ::"r"(b), "r"(parity) : "memory");
}
// outputs [t0, t1) of a decimating FIR (D = 2 or 4) from the raw sub-tile xs (natural order; xs[e0] is the first sample
// the tile reads).  Lanes own consecutive outputs: their 16-byte window loads sit D*8 bytes apart (conflict-free).
#define FT_RO 3
template <int NT>
__device__ __forceinline__ void ft_phase_direct(const FtStage& S, const FtDst& dst, const float* nat, const float2* xs, int e0, int t0, int t1) {
    const int D = S.D, T = S.T;
    for (int base = t0 + threadIdx.x; base < t1; base += NT * FT_RO) {
        float2 acc[FT_RO];
        const float2* px[FT_RO];
#pragma unroll
        for (int i = 0; i < FT_RO; i++) {
            ft_zero(acc[i]);
            const int m = min(base + i * NT, t1 - 1);            // clamp: idle slots recompute the last output
            px[i] = xs + e0 + (m - t0) * D;
        }
        int k = 0;
        if (e0) {                                                   // odd start: one tap alone, then 16-byte aligned pairs
            const float h = nat[0];
#pragma unroll
            for (int i = 0; i < FT_RO; i++) { acc[i] = ft_fma(h, px[i][0], acc[i]); }
            k = 1;
        }
#pragma unroll 2
        for (; k + 1 < T; k += 2) {
            const float h0 = nat[k], h1 = nat[k + 1];
#pragma unroll
            for (int i = 0; i < FT_RO; i++) {
                const float4 v = *reinterpret_cast<const float4*>(px[i] + k);
                acc[i] = ft_fma(h0, make_float2(v.x, v.y), acc[i]);
                acc[i] = ft_fma(h1, make_float2(v.z, v.w), acc[i]);
            }
        }
        if (k < T) {
            const float h = nat[k];
#pragma unroll
            for (int i = 0; i < FT_RO; i++) { acc[i] = ft_fma(h, px[i][k], acc[i]); }
        }
#pragma unroll
        for (int i = 0; i < FT_RO; i++) {
            const int m = base + i * NT;
            if (m < t1) { dst.put2(m, acc[i]); }
        }
    }
}

template <int NT>
__global__ void __launch_bounds__(NT, 2) k_tail_fused(const __grid_constant__ FtParams p) {
    extern __shared__ __align__(16) float sm[];
    __shared__ int s_lo[FT_MAXST + 1], s_hi[FT_MAXST + 1];
    __shared__ FtPolyClass s_cls[FT_MAX_L];
    __shared__ __align__(8) unsigned long long s_bar[3];
    const FtJob& J = p.job[blockIdx.y];
    const int slab = blockIdx.x;
    if (slab >= J.slabs) { return; }
    const int nst = J.nst;
    const int tid = threadIdx.x;
    const bool last = (slab == J.slabs - 1);
    if (tid == 0) {
        int lo[FT_MAXST + 1], hi[FT_MAXST + 1];
        ft_ranges(J, slab, lo, hi);
        for (int s = 0; s <= nst; s++) { s_lo[s] = lo[s]; s_hi[s] = hi[s]; }
    }
    if (tid == 0 && J.s0_direct) {
        for (int i = 0; i < 3; i++) { ft_mbar_init(&s_bar[i], 1); }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    if (J.s0_direct) {
        for (int k = tid; k < J.st[0].T; k += NT) { sm[J.nat_off + k] = __ldg(J.taps_nat + k); }
    }
    // ---- taps -> shared memory (already phase-major in global memory: Stage::taps_pm) ----
    for (int s = 0; s < nst; s++) {
        const FtStage& S = J.st[s];
        float4* tp = reinterpret_cast<float4*>(sm + S.tap_off);
        const float4* __restrict__ src = reinterpret_cast<const float4*>(S.taps);
        for (int k = tid; k < (S.ntap_f >> 2); k += NT) { tp[k] = __ldg(src + k); }
    }
    __syncthreads();

    for (int s = 0; s < nst; s++) {
        const FtStage& S = J.st[s];
        const bool fin = (s + 1 == nst);
        const int mlo = max(s_lo[s + 1], 0), mhi = s_hi[s + 1];
        FtDst dst;
        dst.g = fin ? J.out : nullptr;
        dst.dup = S.dup;
        dst.sp = sm;
        dst.lay.o = 0; dst.lay.D = 1; dst.lay.pitch = 0; dst.lay.sh = 0;
        if (!fin) {
            const FtStage& N = J.st[s + 1];
            dst.sp = sm + N.buf;
            dst.lay = ft_make_lay(N, s_lo[s + 1]);
            // history part of the next stage's input
            const int hend = min(0, s_hi[s + 1]);
            if (N.es == 2) {
                for (int i = s_lo[s + 1] + tid; i < hend; i += NT) {
                    reinterpret_cast<float2*>(dst.sp)[ft_lidx(dst.lay, i)] = __ldg(reinterpret_cast<const float2*>(N.hist_rd) + (i + N.hist));
                }
            }
            else {
                for (int i = s_lo[s + 1] + tid; i < hend; i += NT) { dst.sp[ft_lidx(dst.lay, i)] = __ldg(N.hist_rd + (i + N.hist)); }
            }
        }
        if (s == 0 && J.s0_direct) {
            // ring of three raw buffers filled by cp.async.bulk, two sub-tiles ahead of the one being filtered
            if (mhi > mlo) {
                const int nsub = (mhi - mlo + J.OT0 - 1) / J.OT0;
                const int tl = (mhi - mlo + nsub - 1) / nsub;
                auto ring = [&](int k) { return sm + (k % 3 == 0 ? S.buf : (k % 3 == 1 ? J.stg2 : J.stg3)); };
                auto g_first = [&](int k) { return S.off + (mlo + k * tl) * S.D - (S.T - 1) + S.hist; };   // index into J.src
                auto issue_bulk = [&](int k) {
                    const int t0 = mlo + k * tl, t1 = min(mhi, t0 + tl);
                    const int g0 = g_first(k), g0a = g0 & ~1;
                    const int g1 = S.off + (t1 - 1) * S.D + 1 + S.hist;                 // one past the last sample read
                    const unsigned bytes = (unsigned)(((g1 - g0a + 1) & ~1) * 8);
                    ft_bulk_load(ring(k), reinterpret_cast<const float2*>(J.src) + g0a, bytes, &s_bar[k % 3]);
                };
                if (tid == 0) {
                    issue_bulk(0);
                    if (nsub > 1) { issue_bulk(1); }
                }
                for (int k = 0; k < nsub; k++) {
                    const int t0 = mlo + k * tl, t1 = min(mhi, t0 + tl);
                    if (tid == 0 && k + 2 < nsub) { issue_bulk(k + 2); }
                    ft_mbar_wait(&s_bar[k % 3], (unsigned)((k / 3) & 1));
                    ft_phase_direct<NT>(S, dst, sm + J.nat_off, reinterpret_cast<const float2*>(ring(k)), g_first(k) & 1, t0, t1);
                    __syncthreads();
                }
            }
            __syncthreads();
            if (!fin && last) {
                const FtStage& N = J.st[s + 1];
                const int i0 = N.n_in - N.hist;
                for (int j = tid; j < N.hist; j += NT) {
                    reinterpret_cast<float2*>(N.hist_wr)[j] = reinterpret_cast<const float2*>(dst.sp)[ft_lidx(dst.lay, i0 + j)];
                }
            }
            continue;
        }
        // stage 0 streams its input from global memory through two staging buffers, sub-tile by sub-tile: the
        // cp.async copies of sub-tile k+1 are in flight while sub-tile k is computed
        int nsub = 1, tl = mhi - mlo;
        if (s == 0 && mhi > mlo) {
            nsub = (mhi - mlo + J.OT0 - 1) / J.OT0;
            tl = (mhi - mlo + nsub - 1) / nsub;
        }
        if (tl < 1) { tl = 1; }
        auto stage0_issue = [&](int k) {
            const int t0 = mlo + k * tl, t1 = min(mhi, t0 + tl);
            int ilo, ihi;
            ft_need_in(S, t0, t1, ilo, ihi);
            const FtLay l0 = ft_make_lay(S, ilo);
            const int n = ihi - l0.o;
            float* xk = sm + ((k & 1) ? J.stg2 : S.buf);
            // idx = i - o walks the rows round-robin: row = idx % D, column = idx / D, advanced without dividing
            const int D = l0.D;
            int col = tid / D, row = tid - col * D;
            const int dcol = NT / D, drow = NT - dcol * D;
            const int imin = -S.hist - l0.o;
            if (S.es == 2) {
                const float2* __restrict__ src = reinterpret_cast<const float2*>(J.src) + (l0.o + S.hist);
                // shared address advanced incrementally: +step per iteration, +wrap when the row index passes D
                unsigned sa = (unsigned)__cvta_generic_to_shared(reinterpret_cast<float2*>(xk) + (row * l0.pitch + col));
                const unsigned step = (unsigned)((drow * l0.pitch + dcol) * 8), wrap = (unsigned)((1 - D * l0.pitch) * 8);
                int idx = tid;
                for (; idx < n && idx < imin; idx += NT) {          // only the first slab of a stream start: before the history
                    asm volatile("st.shared.v2.f32 [%0], {%1, %1};\n" ::"r"(sa), "f"(0.0f) : "memory");
                    row += drow; sa += step;
                    if (row >= D) { row -= D; sa += wrap; }
                }
#pragma unroll 4
                for (; idx < n; idx += NT) {
                    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(sa), "l"(src + idx) : "memory");
                    row += drow; sa += step;
                    if (row >= D) { row -= D; sa += wrap; }
                }
            }
            else {
                const float* __restrict__ src = J.src + (l0.o + S.hist);
                for (int idx = tid; idx < n; idx += NT) {
                    xk[row * l0.pitch + col] = (idx >= imin) ? __ldg(src + idx) : 0.0f;
                    row += drow; col += dcol;
                    if (row >= D) { row -= D; col++; }
                }
            }
            cp_async_commit();
        };
        if (s == 0 && mhi > mlo) { stage0_issue(0); }
        for (int k = 0; k < nsub && mhi > mlo; k++) {
            const int t0 = mlo + k * tl, t1 = min(mhi, t0 + tl);
            const float* xb = sm + ((s == 0 && (k & 1)) ? J.stg2 : S.buf);
            FtLay ls;
            if (s == 0) {
                if (k + 1 < nsub) { stage0_issue(k + 1); cp_async_wait<1>(); }
                else { cp_async_wait<0>(); }
                int ilo, ihi;
                ft_need_in(S, t0, t1, ilo, ihi);
                ls = ft_make_lay(S, ilo);
                __syncthreads();
            }
            else { ls = ft_make_lay(S, s_lo[s]); }

            constexpr int MAXR = (NT >= 512) ? 5 : 9;
            switch (S.kind) {
            case FT_FIRC: {
                const int R = ft_pick_r<MAXR>(t1 - t0, 1, NT, S.T, S.D);
                if (R == 5) { ft_phase_firc<5, NT>(S, ls, dst, sm, xb, t0, t1); }
                else if constexpr (MAXR >= 9) { ft_phase_firc<9, NT>(S, ls, dst, sm, xb, t0, t1); }
                break;
            }
            case FT_FIRR: {
                const int R = ft_pick_r<MAXR>(t1 - t0, 1, NT, S.T, 1);
                if (R == 5) { ft_phase_firr<5, NT>(S, ls, dst, sm, xb, t0, t1); }
                else if constexpr (MAXR >= 9) { ft_phase_firr<9, NT>(S, ls, dst, sm, xb, t0, t1); }
                break;
            }
            case FT_POLY: {
                const int L = S.L, M = S.D, tpp = S.T;
                // class constants once per tile (the 64-bit divisions stay out of the unit loop)
                for (int c = tid; c < L; c += NT) {
                    FtPolyClass pc;
                    pc.m_c = t0 + ft_posmod((long long)c - t0, L);
                    pc.cnt = (pc.m_c < t1) ? (t1 - pc.m_c + L - 1) / L : 0;
                    const long long t = (long long)S.phase + (long long)pc.m_c * M;
                    pc.ph = (int)(t % L);
                    const int e = S.off + (int)(t / L) - (tpp - 1) - ls.o;     // >= 0 for every class with outputs
                    pc.a = e / M; pc.bb = e - pc.a * M;
                    s_cls[c] = pc;
                }
                __syncthreads();
                const int per_class = (t1 - t0 + L - 1) / L;
                const int R = ft_pick_r<MAXR>(per_class, L, NT, tpp, M);
                if (R == 5) { ft_phase_poly<5, NT>(S, ls, dst, sm, xb, s_cls, t0, t1); }
                else if constexpr (MAXR >= 9) { ft_phase_poly<9, NT>(S, ls, dst, sm, xb, s_cls, t0, t1); }
                break;
            }
            case FT_QUAD: {
                const float2* X = reinterpret_cast<const float2*>(xb);
                const int own_lo = J.rds ? ft_own_lo(J, slab, s) : 0, own_hi = J.rds ? ft_own_lo(J, slab + 1, s) : 0;
                for (int base = t0; base < t1; base += NT) {
                    const int m = base + tid;
                    const bool act = m < t1;
                    float2 cs = act ? X[m - ls.o] : make_float2(0.0f, 0.0f);
                    const float cur = atan2f(cs.y, cs.x);
                    float prev = __shfl_up_sync(0xffffffffu, cur, 1);
                    if ((tid & 31) == 0 && act) {
                        const float2 q = X[m - 1 - ls.o];
                        prev = atan2f(q.y, q.x);
                    }
                    if (act) {
                        float diff = __fsub_rn(cur, prev);
                        if (diff > FL_M_PI_REF) { diff = __fsub_rn(diff, 2.0f * FL_M_PI_REF); }
                        else if (diff <= -FL_M_PI_REF) { diff = __fadd_rn(diff, 2.0f * FL_M_PI_REF); }
                        const float v = __fmul_rn(diff, S.scale);
                        dst.put1(m, v);
                        if (m >= own_lo && m < own_hi) { J.rds[m] = rds_xlate(v, J.rds_phase0, J.rds_w, m); }
                    }
                }
                break;
            }
            default: {   // FT_M2S
                for (int m = t0 + tid; m < t1; m += NT) { dst.put1(m, xb[m - ls.o]); }
                break;
            }
            }
            if (s == 0) { __syncthreads(); }
        }
        __syncthreads();
        // ---- the last slab hands the next stage's final `hist` inputs to the next chunk ----
        if (!fin && last) {
            const FtStage& N = J.st[s + 1];
            const int i0 = N.n_in - N.hist;
            if (N.es == 2) {
                for (int j = tid; j < N.hist; j += NT) {
                    reinterpret_cast<float2*>(N.hist_wr)[j] = reinterpret_cast<const float2*>(dst.sp)[ft_lidx(dst.lay, i0 + j)];
                }
            }
            else {
                for (int j = tid; j < N.hist; j += NT) { N.hist_wr[j] = dst.sp[ft_lidx(dst.lay, i0 + j)]; }
            }
        }
    }
}

// sdrplusplus_b200/csrc/kernels.cuh -- job descriptors and launch wrappers of the sm_90a kernels.
// Plain structs passed BY VALUE as kernel parameters (one launch covers up to B200_BATCH jobs, i.e.
// the same stage of up to 16 VFOs); pointers are device pointers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define B200_BATCH 16

// ---- sample formats (must match include/b200dsp.h) ----
enum { FMT_CF32 = 0, FMT_CS16 = 1, FMT_CS8 = 2 };

// ---- stage 1: frequency translate + first decimating FIR, all VFOs of a group share the IQ tile ----
// y_v[m] = e^{j phi_v(i_m)} * sum_k x(i_m + k) * g_v[k],  i_m = offset_v + m*D - (T-1)  (chunk-relative),
// g_v[k] = h[k] e^{j w_v k} (host, fp64 -> fp32), phi_v(i) = 2*pi*(phase0_v + W_v*i)/2^64 (exact u64 turns).
// Replaces FrequencyXlator::process (frequency_xlator.h:43-50) + the first DecimatingFIR of
// PowerDecimator::process (power_decimator.h:58-65, decimating_fir.h:45-68) for every VFO at once.
struct XdJob {
    float2* out;            // stage output (data region of the next stage's [hist|data] buffer)
    const float2* gpad;     // complex taps, zero padded: (D-1) zeros | T taps | zeros up to (QP+1)*D total
    unsigned long long phase0;  // phase (turns * 2^64) at chunk-relative index 0
    unsigned long long w;       // phase increment per input sample (turns * 2^64)
    int offset;             // DecimatingFIR::offset for this chunk (decimating_fir.h:50), 0 <= offset
    int n_out;              // outputs this chunk
    int T;                  // tap count
    // retune at this chunk boundary (FrequencyXlator::setOffset keeps `phase`, frequency_xlator.h:25-29):
    // history samples (index < 0) were rotated with w_prev, new samples with w.  The edge kernel recomputes
    // the few outputs whose window straddles index 0 with the real taps h.
    const float* h;         // real taps (T)
    unsigned long long w_prev;
    int retuned;
};
struct XdParams {
    const void* in;         // chunk data (format FMT), chunk-relative index 0
    const float2* hist;     // last `hist_len` samples before the chunk (cf32), hist[hist_len + i] for i < 0
    int hist_len;
    int count;              // samples in this chunk
    int D;                  // decimation of the first stage (1 = pure translate)
    int QP;                 // taps are padded to QP*D entries after the (D-1) leading zeros (see gpad)
    int njobs;
    // "slots" of the pipelined kernel: a slot is one VFO, or two VFOs whose complex taps are exact conjugates
    // (offsets +f and -f through the same real prototype): both share the accumulators A = sum Re(g) x and
    // B = sum Im(g) x;  y(+f) = (A.x - B.y, A.y + B.x),  y(-f) = (A.x + B.y, A.y - B.x).  slot_b = -1: single.
    int nslots;
    signed char slot_a[B200_BATCH], slot_b[B200_BATCH];
    // polyphase-filter-bank form of stage 1 (xd_pfb.cuh): e^{j w_v PS} = sigma for every job, same taps and alignment.
    // pfb_ps = 0: not applicable
    int pfb_ps, pfb_sigma;
    float in_scale;         // integer formats: sample = (float)x * in_scale
    const float* taps_host; // HOST copy of the real prototype taps shared by the jobs of a filter-bank launch (launcher only)
    XdJob job[B200_BATCH];
};

// ---- generic decimating FIR, complex data x real taps (DecimatingFIR / FIR<complex_t,float>) ----
// out[m] = sum_k in[offset + m*decim + k] * taps[k];  `in` points at the oldest history sample.
struct FirJob {
    const float2* in;
    float2* out;
    const float* taps;
    int ntaps, decim, offset, n_out;
};
struct FirParams { int njobs; int max_out; FirJob job[B200_BATCH]; };

// ---- short decimating FIR stages with the input window in registers (dfir_reg.cuh) ----
#define DFR_THREADS 128
#define DFR_MAXT 72

struct DfrParams {
    int njobs;
    int max_out;
    float taps[DFR_MAXT];        // shared by every job of the launch (same plan stage)
    FirJob job[B200_BATCH];
};

bool dfir_reg_supported(int D, int T);
cudaError_t launch_dfir_reg(const DfrParams& p, int D, int T, cudaStream_t s);

// ---- polyphase rational resampler (PolyphaseResampler::process, polyphase_resampler.h:69-99) ----
// output m: t = phase0 + m*decim; off = offset0 + t/interp; ph = t%interp;
// out[m] = sum_k in[off + k] * bank[ph*tpp + k]
struct PolyJob {
    const float2* in;
    float2* out;
    const float* bank;      // [interp][tpp]
    int tpp, interp, decim, phase0, offset0, n_out;
    const float* bank_kl;   // the same bank as [tpp][interp] (k_poly_reg)
    long long in_len;       // samples in `in` that may be read (history + this chunk's input)
};
struct PolyParams { int njobs; int max_out; PolyJob job[B200_BATCH]; };
// register-window versions of the output-rate stages (tails_reg.cuh)
bool poly_reg_supported(int interp, int decim);
cudaError_t launch_poly_reg(const PolyParams& p, cudaStream_t s);           // every job: the same (interp, decim)

// ---- FM discriminator (Quadrature::process, quadrature.h:39-46) ----
struct QuadJob {
    const float2* in;       // [1 history sample | n samples]
    float* out;
    float inv_dev;
    int n;
};
struct QuadParams { int njobs; int max_n; QuadJob job[B200_BATCH]; };

// ---- real FIR (FIR<float,float>, fir.h:69) with optional mono->stereo duplication on store ----
struct FirRJob {
    const float* in;        // oldest history sample
    float* out;             // n floats, or n (l,r) pairs when stereo
    const float* taps;
    int ntaps, n_out, stereo;
};
struct FirRParams { int njobs; int max_out; FirRJob job[B200_BATCH]; };

// ---- fused tail: every FIR-like stage after stage 1 of one VFO in ONE launch ----
// A CTA owns a slab of `OB` final outputs of one VFO and walks the stage list forward; what one stage produces for
// the slab (plus the halo the next stage's taps need, recomputed per slab) stays in shared memory.  Each stage keeps
// the reference's [history | data] semantics: samples with a negative chunk-relative index come from a small
// per-stage history buffer (ping-pong: read `hist_rd`, the CTA of the last slab writes `hist_wr`).
// Index conventions (chunk-relative "data" coordinates, i < 0 = history):
//   FIRC/FIRR  out[m] = sum_k taps[k] * in[m*D + off - (T-1) + k]          (decimating_fir.h:45-68, fir.h:62-83)
//   POLY       t = phase + m*D; out[m] = sum_k bank[t%L][k] * in[off + t/L - (T-1) + k]   (polyphase_resampler.h:69-99)
//   QUAD       out[m] = wrap(arg(in[m]) - arg(in[m-1])) * scale              (quadrature.h:39-46)
//   M2S        out[m] = (in[m], in[m])
#define FT_MAXST 8
#define FT_R 9              // outputs per thread (odd: lanes R apart hit distinct banks without padding)
enum { FT_FIRC = 0, FT_POLY = 1, FT_QUAD = 2, FT_FIRR = 3, FT_M2S = 4 };
struct FtStage {
    int kind;
    int T;                  // taps (FIRC/FIRR) or taps per phase (POLY)
    int D;                  // decimation (FIRC), polyphase decimation (POLY), else 1
    int L;                  // POLY interpolation
    int off;                // FIRC: DecimatingFIR::offset of this chunk; POLY: offset
    int phase;              // POLY: phase
    int n_in, n_out;        // this chunk
    int hist;               // history samples in front of the input: T-1, QUAD 1, M2S 0
    int es;                 // floats per INPUT sample
    int buf;                // float offset of the input buffer in the shared-memory arena (stage 0: staging buffer)
    int pitch;              // row pitch (samples) of the phase-major layout (D rows)
    int tap_off, qpitch;    // taps in shared memory: row r holds taps[q*D + r] (POLY: row (ph*D + r)), qpitch = ceil(T/D)
    int ntap_f;             // floats of the phase-major tap array (multiple of 4)
    int dup;                // output is mono duplicated to (l, r)
    float scale;            // QUAD: 1/deviation
    const float* taps;      // global, phase-major as in shared memory (Stage::taps_pm)
    const float* hist_rd;   // stages 1..: hist*es floats
    float* hist_wr;
};
struct FtJob {
    int nst, slabs, OB, OT0;    // OT0: stage-0 outputs per staging sub-tile
    int stg2, pad;              // float offset of the second staging buffer (the first is st[0].buf)
    // "direct" first stage (decimating FIR with D in {2,4} fed from global memory): the raw input streams into a ring
    // of three shared-memory buffers with cp.async.bulk and is filtered in its natural (interleaved) order
    int s0_direct, stg3;        // third ring buffer (float offset)
    int nat_off, stg_floats;    // natural-order taps of stage 0 in the tap region; floats per ring buffer
    const float* taps_nat;
    const float* src;           // stage 0 input: [hist | data] in global memory
    float* out;                 // final output
    FtStage st[FT_MAXST];
};
struct FtParams { int njobs; int pad; long long* dbg; FtJob job[B200_BATCH]; };   // dbg: optional per-stage clock64() of CTA (1,0)

#if defined(__CUDACC__)
#define FT_HD __host__ __device__
#else
#define FT_HD
#endif
FT_HD inline int ft_posmod(long long a, int m) { long long r = a % m; return (int)(r < 0 ? r + m : r); }
// input range [ilo, ihi) (data coordinates) that outputs [mlo, mhi) of stage s read; mhi > mlo
FT_HD inline void ft_need_in(const FtStage& s, int mlo, int mhi, int& ilo, int& ihi) {
    switch (s.kind) {
    case FT_FIRC: case FT_FIRR:
        ilo = s.off + mlo * s.D - (s.T - 1);
        ihi = s.off + (mhi - 1) * s.D + 1;
        break;
    case FT_POLY:
        ilo = s.off + (int)(((long long)s.phase + (long long)mlo * s.D) / s.L) - (s.T - 1);
        ihi = s.off + (int)(((long long)s.phase + (long long)(mhi - 1) * s.D) / s.L) + 1;
        break;
    case FT_QUAD: ilo = mlo - 1; ihi = mhi; break;
    default: ilo = mlo; ihi = mhi; break;
    }
}
// origin of the phase-major shared-memory layout of stage s's input when the range starts at lo
FT_HD inline int ft_origin(const FtStage& s, int lo) {
    if (s.kind == FT_FIRC && s.D > 1) { return lo - ft_posmod((long long)lo - (s.off - (s.T - 1)), s.D); }
    return lo;
}
FT_HD inline int ft_rows(const FtStage& s) { return (s.kind == FT_FIRC || s.kind == FT_POLY) ? s.D : 1; }
// lo[s], hi[s]: input range of stage s for this slab (s = nst: the final output range)
FT_HD inline void ft_ranges(const FtJob& J, int slab, int* lo, int* hi) {
    const int nst = J.nst;
    const int n_last = J.st[nst - 1].n_out;
    int m0 = slab * J.OB, m1 = m0 + J.OB;
    if (m1 > n_last) { m1 = n_last; }
    if (m0 > m1) { m0 = m1; }
    lo[nst] = m0; hi[nst] = m1;
    const bool last = (slab == J.slabs - 1);
    for (int s = nst - 1; s >= 0; s--) {
        const FtStage& S = J.st[s];
        const int pl = lo[s + 1] > 0 ? lo[s + 1] : 0, ph = hi[s + 1];
        int ilo = 0, ihi = 0;
        if (ph > pl) { ft_need_in(S, pl, ph, ilo, ihi); }
        if (last && s > 0) {
            // the last slab also hands the next chunk its history: the final `hist` inputs of every stage
            const int hl = S.n_in - S.hist, hh = S.n_in;
            if (ihi <= ilo) { ilo = hl; ihi = hh; }
            else { if (hl < ilo) { ilo = hl; } if (hh > ihi) { ihi = hh; } }
        }
        lo[s] = ilo; hi[s] = ihi;
    }
}
cudaError_t launch_tail_fused(const FtParams& p, int max_slabs, int threads, size_t smem_bytes, cudaStream_t s);
int tail_fused_ctas_per_sm(int threads, size_t smem_bytes);

// ---- sequential audio-rate tails (one thread per job): AM envelope + DC block + AGC, SSB rotate + AGC ----
struct AgcState { float amp; };
struct SeqJob {
    const float2* in;       // n complex samples
    float* out;             // n mono floats
    float* state;           // device state block (see kernels.cu: SEQ_STATE_*)
    int n;
    int kind;               // 0 AM, 1 SSB, 2 stereo deemphasis (in/out are (l,r) pairs; threads 0/1 take one channel each),
                            // 3 noise blanker (complex in, complex out)
    int agc_mode;           // AM: 0 carrier, 1 audio
    float set_point, attack, inv_attack, decay, inv_decay, max_gain, max_out; // loop::AGC (agc.h:13-24)
    float dc_rate;          // AM
    float delta_re, delta_im; // SSB second rotator phaseDelta (ssb.h:29, frequency_xlator.h:17)
    float alpha;            // deemphasis: dt / (tau + dt)  (deephasis.h:91-94)
    float nb_rate, nb_inv_rate, nb_level;   // noise_reduction::NoiseBlanker (noise_blanker.h:12-17)
};
struct SeqParams { int njobs; SeqJob job[B200_BATCH]; };
#define SEQ_STATE_FLOATS 8   // [0] carrier amp [1] audio amp [2] dc offset [3] rot re [4] rot im [5] deemph last l [6] last r [7] blanker amp

// ---- FM IF noise reduction (ifnr.cuh): noise_reduction::FMIF (fm_if.h:44-77) ----
struct FmIfJob {
    const float2* in;       // [hist | data], hist = bins - 1
    float2* out;
    const float* win;       // window::nuttall(i, bins - 1)
    const float2* tw;       // exp(-2 pi i k / bins), k < bins
    int n, bins;
};
struct FmIfParams { int njobs; int max_n; FmIfJob job[B200_BATCH]; };
cudaError_t launch_fmif(const FmIfParams& p, cudaStream_t s);          // every job: the same bin count
bool fmif_supported(int bins);

// ---- stereo branch of BroadcastFM behind the discriminator (stereo.cuh) ----
struct StJob {
    const float* in;        // mono [hist | data], hist = ntaps - 1
    float2* out;            // (l, r) before the audio low-pass
    const float2* taps;     // pilot band-pass, complex
    float2* p;              // scratch: pilot filter output, n
    float2* vco;            // scratch: PLL output, n
    float* state;           // [0] phase [1] freq
    int ntaps, delay, n;
    float alpha, beta, min_freq, max_freq;
};
struct StParams { int njobs; int max_n; StJob job[B200_BATCH]; };
cudaError_t launch_stereo(const StParams& p, cudaStream_t s, int* nlaunch);

// ---- RDSDemod, the symbol-rate half of the RDS path (rds.cuh; decoder_modules/radio/src/rds_demod.h:64-73) ----
#define RDS_MAXTAPS 256
#define RDS_MM_PHASES 128
#define RDS_MM_TAPS 8
struct RdsState {
    float gain;                         // FastAGC::_gain
    float c1_phase, c1_freq;            // first Costas loop
    float c2_phase, c2_freq;            // second Costas loop
    float mm_phase, mm_freq, last_out;  // MM: pcl.phase (mu), pcl.freq (omega), lastOut
    int offset, diff_last;              // MM::offset, DifferentialDecoder::last
    float2 c1_hist[RDS_MAXTAPS];        // band-pass delay line (ntaps - 1 used)
    float m_hist[RDS_MM_TAPS];          // MM work-buffer tail (7 used)
};
// one recovered symbol: RDSDemod::soft and the differentially decoded bit of RDSDemod::out (b200_rds_symbol of b200dsp.h)
struct RdsSym { float soft; unsigned int bit; };
struct RdsJob {
    const float2* in;       // n complex samples at 5 kS/s
    RdsSym* out;            // out_cap records (device memory or mapped pinned host memory)
    int* count;             // symbols of this launch (out_cap + 1 when the capacity ran out); its own slot per launch
    RdsState* state;
    const float2* taps;     // band-pass, complex
    const float* bank;      // [RDS_MM_PHASES][RDS_MM_TAPS]
    int n, ntaps, out_cap, pad;
    float set_point, max_gain, rate;
    float c1_alpha, c1_beta, c1_min, c1_max;
    float c2_alpha, c2_beta, c2_min, c2_max;
    float mm_alpha, mm_beta, mm_min, mm_max;
};
struct RdsParams { int njobs; int pad; RdsJob job[B200_BATCH]; };
cudaError_t launch_rds_demod(const RdsParams& p, cudaStream_t s);

// programmatic dependent launch for the chain kernels behind stage 1 (kernels.cu: launch_chain); env B200_PDL, option "pdl"
int kernels_pdl();
void kernels_set_pdl(int on);

// ---- noise_reduction::PowerSquelch at the VFO output (stereo.cuh) ----
#define SQ_MAXPARTS 256
struct SqJob { const float2* in; float2* out; float* partial; int n; float level; };
struct SqParams { int njobs; int max_n; SqJob job[B200_BATCH]; };
cudaError_t launch_squelch(const SqParams& p, cudaStream_t s, int* nlaunch);

// ---- elementwise gain (dsp::audio::Volume, volume.h:39-42: volk_32f_s32f_multiply_32f) ----
struct ScaleJob { const float* in; float* out; int n; float gain; };      // n floats
struct ScaleParams { int njobs; int max_n; ScaleJob job[B200_BATCH]; };

// ---- mono -> stereo copy (convert::MonoToStereo) ----
struct M2SJob { const float* in; float* out; int n; };
struct M2SParams { int njobs; int max_n; M2SJob job[B200_BATCH]; };

// ---- real -> complex + frequency translation in one pass (RealToComplex + FrequencyXlator of the RDS branch,
//      broadcast_fm.h:165-170,196-202): out[i] = in[i] * e^{j 2 pi (phase0 + i w) / 2^64}, exact u64 phase ----
struct RxlJob { const float* in; float2* out; int n; int pad; unsigned long long phase0, w; };
struct RxlParams { int njobs; int max_n; RxlJob job[B200_BATCH]; };
cudaError_t launch_rxl(const RxlParams& p, cudaStream_t s);

// ---- end-of-chunk history carry: dst[0..h) = last h elements of concat(a[0..la), b[0..lb)) ----
// dst may alias a (memmove semantics of fir.h:80 / decimating_fir.h:65 / polyphase_resampler.h:96).
struct CarryJob {
    float* dst; const float* a; const void* b;
    int h, la, lb;          // element counts
    int esize;              // floats per element (1 or 2)
    int bfmt;               // format of b: -1 = float elements of esize, else FMT_* (IQ input -> cf32)
    float scale;            // integer formats: sample = (float)x * scale
};
#define CARRY_BATCH 64
struct CarryParams { int njobs; CarryJob job[CARRY_BATCH]; };

// ---- polyphase filter-bank channelizer, BASELINE config 3 (chanpfb.cuh) ----
struct ChanParams {
    const float2* in;        // [hist (P-1)*M | chunk]: sample (m + p) M + r of the window sits at in[(m + p) * M + r]
    float2* u;               // [n_out][M] branch outputs
    const float* h;          // taps re-ordered [M/32][P][32]: h[((r >> 5) * P + p) * 32 + (r & 31)] = h[p M + r]
    int M, P, n_out;
};
cudaError_t launch_channelizer(const ChanParams& p, float2* y, const float2* tw, cudaStream_t s, int* nlaunch);

// ---- FFT branch ----
struct FftPlanDev {
    int N, logN;            // transform size
    int N1, logN1;          // pass 1 (column) length; N1 == N -> single pass
    int N2, logN2;          // pass 2 (row) length
    const float2* tw;       // twiddle table exp(-2 pi i k / TW), k < TW
    int TW, logTW;
    const float2* tw_fine;  // exp(-2 pi i j / N), j < N / TW (two-pass plans; null otherwise)
    const float* window;    // nz floats: window(i,nz) * (-1)^i
    const float* window_p;  // register-FFT plans: window in pass 1's per-thread order (fft_reg.cuh), zero from nz on; else null
    float in_scale;         // integer input formats: sample = (float)x * in_scale
    int nz;
};

// launch wrappers (return cudaGetLastError())
cudaError_t launch_xlate_decim(const XdParams& p, int fmt, int variant, cudaStream_t s, int* nlaunch);
cudaError_t launch_xd_edge(const XdParams& p, int fmt, cudaStream_t s, int* nlaunch);
cudaError_t launch_fir_c(const FirParams& p, cudaStream_t s);
cudaError_t launch_fir_reg(const FirParams& p, cudaStream_t s);            // every job: decimation 1
cudaError_t launch_firr_reg(const FirRParams& p, cudaStream_t s);
cudaError_t launch_poly(const PolyParams& p, cudaStream_t s);
cudaError_t launch_quad(const QuadParams& p, cudaStream_t s);
cudaError_t launch_fir_r(const FirRParams& p, cudaStream_t s);
cudaError_t launch_seq(const SeqParams& p, cudaStream_t s);
cudaError_t launch_m2s(const M2SParams& p, cudaStream_t s);
cudaError_t launch_scale(const ScaleParams& p, cudaStream_t s);
cudaError_t launch_carry(const CarryParams& p, cudaStream_t s);
// Where a batch of frames comes from: frame f's sample n is chunk[f * stride + n - split] (format fmt, index in samples).
// split > 0 only for a frame that began in earlier chunks: its first split samples were staged, in the same format, at
// pre[0 .. split), and chunk points at the first sample of this chunk.
struct FftFrames {
    const void* chunk;
    const void* pre;
    long long stride;
    int split;
    int nbatch;
};
// src: nz samples of format fmt (chunk data), read directly; out_db: N floats; work: N float2 scratch
cudaError_t launch_fft_frame(const FftPlanDev& pl, const void* src, int fmt, float2* work, float* out_db,
                             float2* out_raw, cudaStream_t s, int* nlaunch);
// fr.nbatch frames in one launch pair; work: nbatch*N float2, out_db: nbatch*N.  tables: the register passes stage their
// twiddle tables in shared memory and read the window as vectors (same values, same output bits); false = global gathers
cudaError_t launch_fft_frames(const FftPlanDev& pl, const FftFrames& fr, int fmt, float2* work, float* out_db,
                              float2* out_raw, cudaStream_t s, int* nlaunch, bool tables);
// the register passes serve this plan (pass-1 window order: window_p)
bool fft_plan_uses_reg(const FftPlanDev& pl);
// IQFrontEnd pre-processing at the input rate: DC blocker + conjugate (preproc.cuh)
struct DcbParams {
    const void* in;          // chunk (format fmt)
    float2* out;             // cf32 chunk after the chain
    int fmt;
    int count;
    float in_scale;
    float rate;              // DCBlocker::_rate (float, dc_blocker.h:88)
    int dc_on, conj_on;
    float2* state;           // [0] offset carried across chunks
    float2* segB;            // [nseg] per-segment B, then rewritten by the scan to the offset at each segment start
    float* segA;             // [nseg] per-segment slope complement c
    int nseg;
};
cudaError_t launch_preproc(const DcbParams& p, cudaStream_t s, int* nlaunch);
cudaError_t launch_convert_cf32(const void* src, int fmt, float2* dst, int n, float scale, cudaStream_t s);
enum { EXP_U8 = 0, EXP_I8 = 1, EXP_I16 = 2, EXP_I32 = 3 };
cudaError_t launch_export(const float* in, long long n, int type, float scalar, void* out, cudaStream_t s);
cudaError_t launch_index_max(const float* in, long long n, float* out_val, cudaStream_t s);
// start/len: per-pixel bin ranges built on the host with the reference's fp32 index loop
cudaError_t launch_zoom_hold_tbl(const float* line, const int* start, const int* len, int out_size, float* out,
                                 float* hold, float hold_speed, cudaStream_t s);
int kernels_max_smem_optin();
void kernels_set_tail_variant(int v);
void kernels_set_fft_variant(int v);
void kernels_set_xd_tma_ctas(int v);      // persistent CTAs of the TMA stage 1 (0 = one per SM)
void kernels_set_fft_cta(int v);          // transforms per CTA of the register FFT passes (8 or 4)
void kernels_set_xd_tile(int mt);     // 0 = automatic
void kernels_set_xd_tma_diag(int v);      // measurement only: 1 = load the tiles, do not filter; 2 = filter, do not load
void kernels_set_xd_tma_stages(int n);   // ring depth of the TMA stage 1 (2 or 3)
void kernels_set_xd_cps(int v);       // cap on stage-1 CTAs per SM, 0 = automatic

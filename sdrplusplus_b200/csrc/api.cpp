// sdrplusplus_b200/csrc/api.cpp -- C ABI of libb200dsp.so (include/b200dsp.h) over engine.h.
#include "../../include/b200dsp.h"
#include "engine.h"
#include <chrono>
#include <map>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <algorithm>

using namespace b200;

// ------------------------------------------------------------------ device
static int g_device = -1;

static int ensure_device() {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        set_error("no usable CUDA device (%s): libb200dsp has no CPU fallback", e == cudaSuccess ? "0 devices" : cudaGetErrorString(e));
        cudaGetLastError();
        return B200_ENODEV;
    }
    if (g_device < 0) { g_device = 0; }
    B200_CK(cudaSetDevice(g_device));
    return 0;
}

extern "C" int b200_init(int device) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        set_error("no usable CUDA device (%s): libb200dsp has no CPU fallback", e == cudaSuccess ? "0 devices" : cudaGetErrorString(e));
        cudaGetLastError();
        return B200_ENODEV;
    }
    if (device < 0 || device >= n) { set_error("device %d out of range (0..%d)", device, n - 1); return B200_EINVAL; }
    g_device = device;
    B200_CK(cudaSetDevice(device));
    B200_CK(cudaFree(0));
    return 0;
}
extern "C" int b200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}
extern "C" const char* b200_last_error(void) { return last_error(); }
extern "C" int b200_version(void) { return B200_VERSION; }

extern "C" int b200_register_decim_plan(int ratio, int nstages, const int* d, const int* t, const float* const* taps) {
    if (!d || !t || !taps) { set_error("null argument"); return B200_EINVAL; }
    if (register_decim_plan(ratio, nstages, d, t, taps)) { set_error("invalid decimation plan for ratio %d", ratio); return B200_EINVAL; }
    return 0;
}
extern "C" int b200_load_decim_plans(const char* path) {
    if (load_decim_plans(path)) { set_error("cannot load decimation plans from %s", path ? path : "(default location)"); return B200_ENOPLAN; }
    return 0;
}

// ------------------------------------------------------------------ design helpers
extern "C" int b200_taps_lowpass(double cutoff, double tw, double sr, int odd, float* out, int cap) {
    std::vector<float> t = lowpass_taps(cutoff, tw, sr, odd != 0);
    if (out) { memcpy(out, t.data(), sizeof(float) * (size_t)std::min<int>((int)t.size(), cap)); }
    return (int)t.size();
}
extern "C" int b200_taps_highpass(double cutoff, double tw, double sr, int odd, float* out, int cap) {
    std::vector<float> t = highpass_taps(cutoff, tw, sr, odd != 0);
    if (out) { memcpy(out, t.data(), sizeof(float) * (size_t)std::min<int>((int)t.size(), cap)); }
    return (int)t.size();
}
extern "C" int b200_taps_bandpass(double b0, double b1, double tw, double sr, int odd, float* out_iq, int cap) {
    std::vector<float> t = bandpass_c_taps(b0, b1, tw, sr, odd != 0);                   // (re, im) pairs
    const int n = (int)(t.size() / 2);
    if (out_iq) { memcpy(out_iq, t.data(), 2 * sizeof(float) * (size_t)std::max(0, std::min(n, cap))); }
    return n;
}
extern "C" int b200_window(int window, int nz, float* out) {
    if (nz < 0 || !out) { set_error("bad window args"); return B200_EINVAL; }
    std::vector<float> w = fft_window(window, nz);
    memcpy(out, w.data(), sizeof(float) * (size_t)nz);
    return nz;
}
extern "C" int b200_fft_frame_params(double sr, int size, double rate, int* nz, int* skip) {
    if (!nz || !skip || rate <= 0) { set_error("bad args"); return B200_EINVAL; }
    fft_frame_params(sr, size, rate, *nz, *skip);
    return 0;
}
extern "C" int b200_resamp_plan_get(double inSR, double outSR, b200_resamp_plan* out) {
    if (!out) { set_error("null plan"); return B200_EINVAL; }
    ResampPlan pl = make_resamp_plan(inSR, outSR);
    memset(out, 0, sizeof(*out));
    out->mode = pl.mode;
    out->predec_ratio = pl.predec_ratio;
    out->interp = pl.interp;
    out->decim = pl.decim;
    out->ntaps = (int)pl.rtaps.size();
    out->taps_per_phase = pl.taps_per_phase;
    if (pl.use_decim) {
        const DecimPlan* dp = find_decim_plan(pl.predec_ratio);
        if (!dp) { set_error("no decimation plan for ratio %d", pl.predec_ratio); return B200_ENOPLAN; }
        out->nstages = (int)dp->stages.size();
        for (int i = 0; i < out->nstages && i < 8; i++) {
            out->stage_decim[i] = dp->stages[i].decim;
            out->stage_taps[i] = (int)dp->stages[i].taps.size();
        }
    }
    return 0;
}

// ------------------------------------------------------------------ FFT plan
static int bytes_per_sample(int fmt) { return fmt == B200_FMT_CF32 ? 8 : (fmt == B200_FMT_CS16 ? 4 : 2); }
static int ilog2(int n) { int l = 0; while ((1 << l) < n) { l++; } return l; }

struct FftCore {
    FftPlanDev plan;
    DevBuf tw, twf, win, winp, work;
    int size = 0, nz = 0, window = 0;
    int create(int size_, int nz_, int window_, int max_batch = 1) {
        if (size_ < 8 || size_ > (1 << 22) || (size_ & (size_ - 1))) { set_error("FFT size %d must be a power of two in [8, 4194304]", size_); return B200_EINVAL; }
        if (nz_ < 1 || nz_ > size_) { set_error("bad nz %d", nz_); return B200_EINVAL; }
        size = size_; nz = nz_; window = window_;
        memset(&plan, 0, sizeof(plan));
        plan.N = size; plan.logN = ilog2(size);
        if (size <= 8192) { plan.N1 = size; plan.logN1 = plan.logN; plan.N2 = 1; plan.logN2 = 0; }
        else {
            plan.logN1 = (plan.logN + 1) / 2; plan.N1 = 1 << plan.logN1;
            plan.logN2 = plan.logN - plan.logN1; plan.N2 = 1 << plan.logN2;
        }
        plan.TW = std::max(plan.N1, plan.N2); plan.logTW = ilog2(plan.TW);
        std::vector<float2> t((size_t)plan.TW);
        for (int k = 0; k < plan.TW; k++) {
            double a = -2.0 * 3.14159265358979323846 * (double)k / (double)plan.TW;
            t[k] = make_float2((float)std::cos(a), (float)std::sin(a));
        }
        int rc;
        if ((rc = tw.alloc(t.size() * sizeof(float2)))) { return rc; }
        B200_CK(cudaMemcpy(tw.p, t.data(), t.size() * sizeof(float2), cudaMemcpyHostToDevice));
        std::vector<float> w = fft_window(window, nz);
        if ((rc = win.alloc((size_t)nz * sizeof(float)))) { return rc; }
        B200_CK(cudaMemcpy(win.p, w.data(), (size_t)nz * sizeof(float), cudaMemcpyHostToDevice));
        if ((rc = work.alloc((size_t)size * sizeof(float2) * (size_t)(max_batch > 0 ? max_batch : 1)))) { return rc; }
        plan.tw = tw.as<float2>(); plan.window = win.as<float>(); plan.nz = nz;
        plan.tw_fine = nullptr;
        if (plan.N2 > 1) {
            // four-step twiddle W_N^e = tw[e >> s] * fine[e & (2^s - 1)], 2^s = N / TW
            const int nf = size / plan.TW;
            std::vector<float2> f((size_t)nf);
            for (int j = 0; j < nf; j++) {
                double a = -2.0 * 3.14159265358979323846 * (double)j / (double)size;
                f[j] = make_float2((float)std::cos(a), (float)std::sin(a));
            }
            if ((rc = twf.alloc(f.size() * sizeof(float2)))) { return rc; }
            B200_CK(cudaMemcpy(twf.p, f.data(), f.size() * sizeof(float2), cudaMemcpyHostToDevice));
            plan.tw_fine = twf.as<float2>();
        }
        plan.window_p = nullptr;
        if (fft_plan_uses_reg(plan)) {
            // pass 1 of the register FFT: thread t of column n2 multiplies x[(a RB + t) N2 + n2], a < RA, by the window.
            // Laid out as winp[(n2 RB + t) RA + a], those RA values are one contiguous run the thread reads in 16-byte vectors.
            const int RA = plan.logN1 == 8 ? 16 : (plan.logN1 == 9 ? 16 : 32), RB = plan.logN1 == 8 ? 16 : 32;
            std::vector<float> wp((size_t)size, 0.0f);
            for (int n2 = 0; n2 < plan.N2; n2++) {
                for (int t = 0; t < RB; t++) {
                    for (int a = 0; a < RA; a++) {
                        const long long n = (long long)(a * RB + t) * plan.N2 + n2;
                        if (n < nz) { wp[((size_t)n2 * RB + t) * RA + a] = w[(size_t)n]; }
                    }
                }
            }
            if ((rc = winp.alloc(wp.size() * sizeof(float)))) { return rc; }
            B200_CK(cudaMemcpy(winp.p, wp.data(), wp.size() * sizeof(float), cudaMemcpyHostToDevice));
            plan.window_p = winp.as<float>();
        }
        B200_CK(cudaDeviceSynchronize());       // tables uploaded on the legacy stream; the spectrum branch runs on a non-blocking one
        return 0;
    }
};

// ------------------------------------------------------------------ RDSDemod (decoder_modules/radio/src/rds_demod.h)
// One stream's carried state and tables, owned by a b200_rds_demod block or by a front-end VFO in B200_DEMOD_WFM_RDS_BITS mode.
static_assert(sizeof(b200_rds_symbol) == 8 && sizeof(RdsSym) == sizeof(b200_rds_symbol), "one RDS symbol record is 8 bytes");
struct RdsCore {
    DevBuf state, taps, bank;
    RdsState init;               // what reset() restores
    RdsJob proto;                // coefficients and tables; job() fills in the rest per launch
    int create(cudaStream_t s);
    int reset(cudaStream_t s);
    RdsJob job(const float2* in, int n, RdsSym* out, int out_cap, int* count) const {
        RdsJob J = proto;
        J.in = in; J.n = n; J.out = out; J.out_cap = out_cap; J.count = count;
        return J;
    }
};
int RdsCore::create(cudaStream_t s) {
    // init() of rds_demod.h:20-41
    const std::vector<float> bp = bandpass_c_taps(0.0, 2375.0, 100.0, 5000.0, false);      // (re, im) pairs
    const std::vector<float> bk = mm_interp_bank(RDS_MM_PHASES, RDS_MM_TAPS);
    const int nt = (int)bp.size() / 2;
    if (nt < 2 || nt > RDS_MAXTAPS) { set_error("RDS band-pass of %d taps", nt); return B200_EINVAL; }
    int rc;
    if ((rc = state.alloc(sizeof(RdsState), false)) || (rc = taps.alloc(bp.size() * sizeof(float), false)) ||
        (rc = bank.alloc(bk.size() * sizeof(float), false))) { return rc; }
    RdsJob& J = proto;
    memset(&J, 0, sizeof(J));
    J.state = state.as<RdsState>(); J.taps = taps.as<float2>(); J.bank = bank.as<float>();
    J.ntaps = nt;
    J.set_point = (float)1.0; J.max_gain = (float)1e6; J.rate = (float)0.1;               // agc.init(NULL, 1.0, 1e6, 0.1)
    pll_coefficients(0.005f, J.c1_alpha, J.c1_beta);                                       // costas.init(NULL, 0.005f)
    J.c1_min = -3.1415926535f; J.c1_max = 3.1415926535f;                                   // FL_M_PI (math/constants.h:4)
    const double baud = hz_to_rads(2375.0 / 2.0, 5000.0);
    pll_coefficients(0.01, J.c2_alpha, J.c2_beta);                                         // costas2.init(NULL, 0.01, 0, f, f - 10 %, f + 10 %)
    J.c2_min = (float)(baud - (baud * 0.1)); J.c2_max = (float)(baud + (baud * 0.1));
    const double omega = 5000.0 / (2375.0 / 2.0);                                          // recov.init(NULL, omega, 1e-6, 0.01, 0.01)
    J.mm_alpha = (float)0.01; J.mm_beta = (float)1e-6;
    J.mm_min = (float)(omega * (1.0 - 0.01)); J.mm_max = (float)(omega * (1.0 + 0.01));
    memset(&init, 0, sizeof(init));
    init.gain = (float)1.0;
    init.c2_freq = (float)baud;
    init.mm_freq = (float)omega;
    cudaError_t e = cudaMemcpyAsync(taps.p, bp.data(), bp.size() * sizeof(float), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) { e = cudaMemcpyAsync(bank.p, bk.data(), bk.size() * sizeof(float), cudaMemcpyHostToDevice, s); }
    if (e == cudaSuccess) { e = cudaMemcpyAsync(state.p, &init, sizeof(RdsState), cudaMemcpyHostToDevice, s); }
    if (e == cudaSuccess) { e = cudaStreamSynchronize(s); }
    if (e != cudaSuccess) { return cuda_fail(e, "RDS demodulator tables"); }
    return 0;
}
int RdsCore::reset(cudaStream_t s) {
    // RDSDemod::reset (rds_demod.h:52-62): gain, loop phases / frequencies, band-pass delay line, MM offset / phase / lastOut,
    // decoder memory.  MM::reset (mm.h:83-92) leaves its work-buffer tail alone: so does this.
    RdsState cur, st = init;
    B200_CK(cudaMemcpyAsync(&cur, state.p, sizeof(RdsState), cudaMemcpyDeviceToHost, s));
    B200_CK(cudaStreamSynchronize(s));
    memcpy(st.m_hist, cur.m_hist, sizeof(st.m_hist));
    B200_CK(cudaMemcpyAsync(state.p, &st, sizeof(RdsState), cudaMemcpyHostToDevice, s));
    B200_CK(cudaStreamSynchronize(s));
    return 0;
}

// ------------------------------------------------------------------ front end
// Stage::role of a VFO's stages: the radio blocks b200_fe_set_vfo_config switches on and off, in chain order (IF chain behind the
// channel filter, AF chain at the end), and the AM / SSB demodulator stage whose AGC it retunes
enum VfoRole { ROLE_NONE = 0, ROLE_NB, ROLE_SQUELCH, ROLE_NR, ROLE_HPF, ROLE_DEEMPH, ROLE_VOLUME, ROLE_DEMOD, ROLE_COUNT };
static bool role_in_if_chain(int r) { return r >= ROLE_NB && r <= ROLE_NR; }
static bool role_in_af_chain(int r) { return r >= ROLE_HPF && r <= ROLE_VOLUME; }

struct VfoSlot {
    bool used = false;
    b200_vfo_cfg cfg;
    Chain chain;
    bool pend_offset = false, pend_bw = false;
    double new_offset = 0, new_bw = 0;
    // b200_fe_set_vfo_config: the config taken at the next chunk boundary, and the blocks switched off by an earlier call,
    // parked with their state (chain::setBlockEnabled keeps a disabled block as it was)
    bool pend_cfg = false;
    b200_vfo_cfg new_cfg;
    std::unique_ptr<Stage> parked[ROLE_COUNT];
    bool hpf_at_add = false;     // b200_fe_vfo_max_out counts the high-pass FIR's spare output (FirCStage::max_out) when add built it
    // B200_DEMOD_WFM_RDS_BITS: RDSDemod behind the chain, and where its records wait for the copy to a host buffer
    std::unique_ptr<RdsCore> rds;
    DevBuf rds_rec;
    // an IQ tap (b200_fe_bind_iq) instead of a VFO: no chain, the chunk's effective stream in sample type tap_type (B200_IQ_*)
    int tap_type = -1;
    float tap_scalar = 0.0f;
    // an RDS output (b200_fe_bind_rds): `chain` is the branch behind the discriminator of VFO rds_parent, with rds / rds_rec as
    // for WFM_RDS_BITS.  On the parent: rds_child is its bound output, rds_parked the branch an unbind left, with its state.
    int rds_parent = -1;
    int rds_child = -1;
    std::unique_ptr<VfoSlot> rds_parked;
};
static bool is_tap(const VfoSlot* v) { return v->tap_type >= 0; }
static bool is_rds_out(const VfoSlot* v) { return v->rds_parent >= 0; }
// bytes per complex sample of an IQ tap's output (interleaved I, Q)
static size_t iq_tap_bytes(int type) {
    return type == B200_IQ_CF32 || type == B200_IQ_I32 ? 8 : (type == B200_IQ_I16 ? 4 : 2);
}

// input slots / event sets of a front end: a chunk uses slot (index % FE_SLOTS); up to FE_SLOTS chunks may be between submit and
// wait (default two, option "inflight": small chunks over PCIe want the copy engine fed a few chunks ahead)
#define FE_SLOTS 4

struct b200_fe {
    double fs = 0;
    int max_chunk = 0;
    KernelOpts opts;             // the kernel choices of this front end (b200_fe_set_option); sch and sch_pre launch with them
    Scheduler sch{opts};
    cudaStream_t own_stream = nullptr, copy_stream = nullptr, fft_stream = nullptr, tail_stream = nullptr, join_stream = nullptr;
    cudaEvent_t ev_tail_done[FE_SLOTS] = {};
    cudaEvent_t ev_fft_go = nullptr, ev_fft_done = nullptr, ev_lines_free = nullptr;
    bool lines_busy = false;
    std::vector<std::unique_ptr<VfoSlot>> vfos;
    std::mutex mtx;
    DevBuf in_dev[FE_SLOTS];
    // FFT branch
    bool fft_on = false;
    FftCore fft;
    int skip = 0;
    DevBuf frame, lines;
    int max_lines = 0;
    unsigned long long pos = 0, fstart = 0;
    // frame[0 .. pos - fstart) holds the part of the frame at fstart that earlier chunks carried, in format frame_fmt at
    // ingest scale frame_scale (cf32: already scaled)
    int frame_fmt = FMT_CF32;
    float frame_scale = 0.0f;
    // 1: a frame that began in earlier chunks joins its chunk's batch, staged by copies in the input's format; the register
    // passes read their twiddles from shared memory.  0: the frame is converted to cf32 and transformed on its own, twiddles
    // from global memory.  Same lines either way.
    int fft_v = 1;
    // pipelining
    cudaEvent_t ev_h2d[FE_SLOTS] = {}, ev_compute[FE_SLOTS] = {}, ev_out[FE_SLOTS] = {};
    bool slot_used[FE_SLOTS] = {};
    int max_inflight = 2;                    // chunks between submit and wait (option "inflight", up to FE_SLOTS)
    unsigned long long nsub = 0, nwait = 0;
    int host_direct = -1;                    // pinned host outputs written by the kernels themselves: -1 small chunks, 0 never, 1 always
    long long host_ns[4] = { 0, 0, 0, 0 };   // host time of submit(): [0] checks + plans, [1] spectrum branch, [2] Scheduler::run, [3] join + outputs
    float scale16 = 1.0f / 32768.0f, scale8 = 1.0f / 128.0f;
    // IQFrontEnd pre-processing chain (iq_frontend.cpp:32-39): PowerDecimator -> DCBlocker -> Conjugate, off by default
    int decim = 1;               // setDecimation: everything behind it runs at fs_eff = fs / decim
    double fs_eff = 0;
    bool dc_block = false, invert_iq = false;
    Chain pre;                   // the decimator (typed cf32 chain), built when decim > 1
    Scheduler sch_pre{opts};
    DevBuf pp[FE_SLOTS];         // chunk after DC blocker / conjugate (one per chunk in flight)
    DevBuf dc_state, dc_segA, dc_segB;
    int max_eff = 0;             // largest chunk behind the decimator
    // RDS symbol counts (B200_DEMOD_WFM_RDS_BITS VFOs): the device knows them only after the launch.  The kernel writes them
    // into the row of the chunk's slot in pinned memory, in stream order before ev_out; b200_fe_wait reads them after it.
    int* rds_count = nullptr;                // [FE_SLOTS][B200_MAX_VFOS], allocated with the first such VFO
    struct RdsPend { int id, n_in, bound; };
    std::vector<RdsPend> rds_pend[FE_SLOTS];
    b200_outputs* rds_out[FE_SLOTS] = {};    // whose vfo_count b200_fe_wait fills
    // IQ taps (b200_fe_bind_iq): k_iq_tap runs on a stream of its own, forked behind the pre-processing like the spectrum
    // branch and joined on join_stream; stream and events are made by the first bind
    cudaStream_t tap_stream = nullptr;
    cudaEvent_t ev_tap_go = nullptr, ev_tap_done = nullptr;
    bool tap_read_pre = false;               // the taps of the last chunk read pre.out, which the next chunk's decimator rewrites
    DevBuf tap_stage[FE_SLOTS];              // outputs that leave through a copy: one region per tap, 16-byte aligned
};

extern "C" b200_fe* b200_fe_create(double samplerate, int max_chunk) {
    if (ensure_device()) { return nullptr; }
    if (samplerate <= 0 || max_chunk < 1) { set_error("bad samplerate/max_chunk"); return nullptr; }
    b200_fe* fe = new b200_fe;
    fe->fs = samplerate;
    fe->fs_eff = samplerate;
    fe->max_chunk = max_chunk;
    fe->max_eff = max_chunk;
    // Stream priorities decide whose thread blocks the SMs take first when several kernels wait for room.  The chain behind
    // stage 1 is a sequence of short dependent launches and sets the pace of a step: it goes first; the spectrum branch (a few
    // frames per chunk, nobody waits for it before the outputs) goes last.  B200_STREAM_PRIO="tail,main,fft" (0 = lowest)
    // overrides the order for experiments.
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);                     // lo: numerically largest = least urgent
    int pt = 2, pm = 1, pf = 0;
    if (const char* e = getenv("B200_STREAM_PRIO")) { sscanf(e, "%d,%d,%d", &pt, &pm, &pf); }
    auto prio = [&](int level) { int p = lo - level; return p < hi ? hi : p; };
    bool ok = cudaStreamCreateWithPriority(&fe->own_stream, cudaStreamNonBlocking, prio(pm)) == cudaSuccess &&
              cudaStreamCreateWithFlags(&fe->copy_stream, cudaStreamNonBlocking) == cudaSuccess &&
              cudaStreamCreateWithPriority(&fe->fft_stream, cudaStreamNonBlocking, prio(pf)) == cudaSuccess &&
              cudaStreamCreateWithPriority(&fe->tail_stream, cudaStreamNonBlocking, prio(pt)) == cudaSuccess &&
              cudaStreamCreateWithFlags(&fe->join_stream, cudaStreamNonBlocking) == cudaSuccess &&
              cudaEventCreateWithFlags(&fe->ev_lines_free, cudaEventDisableTiming) == cudaSuccess &&
              cudaEventCreateWithFlags(&fe->ev_fft_go, cudaEventDisableTiming) == cudaSuccess &&
              cudaEventCreateWithFlags(&fe->ev_fft_done, cudaEventDisableTiming) == cudaSuccess;
    for (int i = 0; i < FE_SLOTS && ok; i++) {
        ok = cudaEventCreateWithFlags(&fe->ev_h2d[i], cudaEventDisableTiming) == cudaSuccess &&
             cudaEventCreateWithFlags(&fe->ev_compute[i], cudaEventDisableTiming) == cudaSuccess &&
             cudaEventCreateWithFlags(&fe->ev_tail_done[i], cudaEventDisableTiming) == cudaSuccess &&
             cudaEventCreateWithFlags(&fe->ev_out[i], cudaEventDisableTiming) == cudaSuccess;
    }
    if (!ok || fe->sch.init_raw()) {
        if (ok) {} else { cuda_fail(cudaGetLastError(), "stream/event creation"); }
        b200_fe_destroy(fe);
        return nullptr;
    }
    fe->sch.stream = fe->own_stream;
    fe->sch.fuse.on = true;
    {
        int dev = 0, sms = 0;
        if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && sms > 0) {
            fe->sch.sm_count = sms;
        }
    }
    if (fe->sch.enable_overlap(fe->tail_stream)) { b200_fe_destroy(fe); return nullptr; }
    return fe;
}

extern "C" void b200_fe_destroy(b200_fe* fe) {
    if (!fe) { return; }
    cudaDeviceSynchronize();
    for (int i = 0; i < FE_SLOTS; i++) {
        if (fe->ev_h2d[i]) { cudaEventDestroy(fe->ev_h2d[i]); }
        if (fe->ev_compute[i]) { cudaEventDestroy(fe->ev_compute[i]); }
        if (fe->ev_tail_done[i]) { cudaEventDestroy(fe->ev_tail_done[i]); }
        if (fe->ev_out[i]) { cudaEventDestroy(fe->ev_out[i]); }
    }
    if (fe->ev_lines_free) { cudaEventDestroy(fe->ev_lines_free); }
    if (fe->tail_stream) { cudaStreamDestroy(fe->tail_stream); }
    if (fe->join_stream) { cudaStreamDestroy(fe->join_stream); }
    if (fe->ev_fft_go) { cudaEventDestroy(fe->ev_fft_go); }
    if (fe->ev_fft_done) { cudaEventDestroy(fe->ev_fft_done); }
    if (fe->own_stream) { cudaStreamDestroy(fe->own_stream); }
    if (fe->copy_stream) { cudaStreamDestroy(fe->copy_stream); }
    if (fe->fft_stream) { cudaStreamDestroy(fe->fft_stream); }
    if (fe->tap_stream) { cudaStreamDestroy(fe->tap_stream); }
    if (fe->ev_tap_go) { cudaEventDestroy(fe->ev_tap_go); }
    if (fe->ev_tap_done) { cudaEventDestroy(fe->ev_tap_done); }
    if (fe->rds_count) { cudaFreeHost(fe->rds_count); }
    delete fe;
}

extern "C" int b200_fe_set_stream(b200_fe* fe, void* s) {
    if (!fe) { set_error("null fe"); return B200_EINVAL; }
    fe->sch.stream = s ? (cudaStream_t)s : fe->own_stream;
    return 0;
}

// IQFrontEnd::setDecimation / setDCBlocking / setInvertIQ (iq_frontend.cpp:100-119)
extern "C" int b200_fe_set_decimation(b200_fe* fe, int ratio) {
    if (!fe) { set_error("null fe"); return B200_EINVAL; }
    if (ratio < 1 || (ratio & (ratio - 1)) || ratio > 8192) { set_error("decimation must be a power of two <= 8192"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(fe->mtx);
    if (b200_fe_vfo_count(fe) > 0 || fe->fft_on || fe->nsub > 0) {
        set_error("the input decimation changes the effective sample rate: set it before the FFT and the VFOs are configured");
        return B200_ESTATE;
    }
    B200_CK(cudaDeviceSynchronize());
    fe->pre.st.clear();
    fe->decim = ratio;
    fe->fs_eff = fe->fs / (double)ratio;
    fe->max_eff = fe->max_chunk;
    if (ratio > 1) {
        int rc = fe->pre.add_power_decim(ratio);
        if (!rc) { rc = fe->pre.finalize(fe->max_chunk); }
        if (rc) { fe->pre.st.clear(); fe->decim = 1; fe->fs_eff = fe->fs; return rc; }
        fe->max_eff = fe->pre.max_out(fe->max_chunk);
        fe->sch_pre.stream = fe->sch.stream;
    }
    return 0;
}
extern "C" int b200_fe_set_dc_blocking(b200_fe* fe, int enabled) {
    if (!fe) { set_error("null fe"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(fe->mtx);
    fe->dc_block = enabled != 0;
    return 0;
}
extern "C" int b200_fe_set_invert_iq(b200_fe* fe, int enabled) {
    if (!fe) { set_error("null fe"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(fe->mtx);
    fe->invert_iq = enabled != 0;
    return 0;
}

extern "C" int b200_fe_set_fft(b200_fe* fe, int size, double rate, int window) {
    if (!fe) { set_error("null fe"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(fe->mtx);
    B200_CK(cudaDeviceSynchronize());
    if (size == 0) { fe->fft_on = false; return 0; }
    if (rate <= 0) { set_error("bad fft rate"); return B200_EINVAL; }
    int nz, skip;
    fft_frame_params(fe->fs_eff, size, rate, nz, skip);
    const int max_lines = (int)(fe->max_eff / ((long long)nz + skip)) + 2;
    int rc = fe->fft.create(size, nz, window, max_lines);
    if (rc) { return rc; }
    fe->skip = skip;
    fe->max_lines = max_lines;
    if ((rc = fe->frame.alloc((size_t)nz * sizeof(float2))) || (rc = fe->lines.alloc((size_t)max_lines * size * sizeof(float)))) { return rc; }
    // Reshaper restart (iq_frontend.cpp:269-279): framing restarts at the current stream position
    fe->fstart = fe->pos;
    fe->fft_on = true;
    return 0;
}

// the AF chain and the volume follow audio only
static bool vfo_has_audio(const b200_vfo_cfg& c) {
    return c.demod != B200_DEMOD_RAW && c.demod != B200_DEMOD_WFM_RDS && c.demod != B200_DEMOD_WFM_RDS_BITS;
}

// RDSDemod behind a chain that gives at most n_max 5 kS/s samples per chunk, and its record buffer
static int add_rds_demod(b200_fe* fe, VfoSlot* v, int n_max) {
    if (!fe->rds_count && cudaMallocHost((void**)&fe->rds_count, sizeof(int) * FE_SLOTS * B200_MAX_VFOS) != cudaSuccess) {
        fe->rds_count = nullptr;
        return cuda_fail(cudaGetLastError(), "cudaMallocHost");
    }
    v->rds = std::make_unique<RdsCore>();
    int rc = v->rds->create(nullptr);
    if (rc) { return rc; }
    return v->rds_rec.alloc((size_t)b200_rds_demod_max_out(n_max) * sizeof(RdsSym), false);
}

static int build_vfo_chain(b200_fe* fe, VfoSlot* v) {
    const b200_vfo_cfg& c = v->cfg;
    int rc = v->chain.add_rxvfo(fe->fs_eff, c.out_samplerate, c.bandwidth, c.offset);
    if (rc) { return rc; }
    // radio IF chain (radio_module.h:94-96): noise blanker -> power squelch -> FM IF noise reduction
    auto& st = v->chain.st;
    if (c.nb_on) {
        if ((rc = v->chain.add_noise_blanker(500.0 / c.out_samplerate, c.nb_level))) { return rc; }
        st.back()->role = ROLE_NB;
    }
    if (c.squelch_on) {
        if ((rc = v->chain.add_squelch(c.squelch_level))) { return rc; }
        st.back()->role = ROLE_SQUELCH;
    }
    if (c.nr_on) {
        if ((rc = v->chain.add_fmif(c.nr_bins))) { return rc; }
        st.back()->role = ROLE_NR;
    }
    switch (c.demod) {
    case B200_DEMOD_RAW: break;
    case B200_DEMOD_WFM: rc = v->chain.add_wfm(c.deviation, c.out_samplerate, c.low_pass != 0, false); break;
    case B200_DEMOD_WFM_STEREO: rc = v->chain.add_wfm(c.deviation, c.out_samplerate, c.low_pass != 0, true); break;
    case B200_DEMOD_WFM_RDS:
    case B200_DEMOD_WFM_RDS_BITS: rc = v->chain.add_wfm_rds(c.deviation, c.out_samplerate); break;
    case B200_DEMOD_NFM: rc = v->chain.add_nfm(c.out_samplerate, c.bandwidth, c.low_pass != 0); break;
    case B200_DEMOD_AM: rc = v->chain.add_am(c.agc_mode, c.bandwidth, c.agc_attack, c.agc_decay, c.dc_block_rate, c.out_samplerate); break;
    case B200_DEMOD_USB: rc = v->chain.add_ssb(0, c.bandwidth, c.out_samplerate, c.agc_attack, c.agc_decay); break;
    case B200_DEMOD_LSB: rc = v->chain.add_ssb(1, c.bandwidth, c.out_samplerate, c.agc_attack, c.agc_decay); break;
    case B200_DEMOD_DSB: rc = v->chain.add_ssb(2, c.bandwidth, c.out_samplerate, c.agc_attack, c.agc_decay); break;
    default: set_error("unknown demodulator %d", c.demod); return B200_EINVAL;
    }
    if (rc) { return rc; }
    if (c.demod >= B200_DEMOD_AM && c.demod <= B200_DEMOD_DSB) { st[st.size() - 2]->role = ROLE_DEMOD; }    // AGC stage, then low-pass / M2S
    const bool audio = vfo_has_audio(c);
    if (c.af_samplerate > 0 && audio) {
        if ((rc = v->chain.add_af_chain(c.out_samplerate, c.af_samplerate, c.af_high_pass != 0, c.af_deemph_tau))) { return rc; }
        size_t k = st.size();
        if (c.af_deemph_tau > 0.0) { st[--k]->role = ROLE_DEEMPH; }
        if (c.af_high_pass) { st[--k]->role = ROLE_HPF; v->hpf_at_add = true; }
    }
    if (c.af_volume_on && audio) {
        if ((rc = v->chain.add_volume(c.af_volume, c.af_muted != 0))) { return rc; }
        st.back()->role = ROLE_VOLUME;
    }
    const bool ov = fe->sch.tail_stream != nullptr;
    if (ov && v->chain.st.size() == 1) {
        // overlapped mode hands every chain's output to the tail stream: give a stage-1-only chain an exact copy stage
        if ((rc = v->chain.add_fir_c(std::vector<float>{ 1.0f }, 1))) { return rc; }
    }
    if ((rc = v->chain.finalize(fe->max_eff, ov, &fe->sch.fuse))) { return rc; }
    if (c.demod == B200_DEMOD_WFM_RDS_BITS) { return add_rds_demod(fe, v, v->chain.max_out(fe->max_eff)); }
    return 0;
}

// what one chunk of `count` samples can put into the output buffer of a VFO, an RDS output (8-byte elements) or an IQ tap
// (one sample per sample of the effective stream)
static int vfo_out_bound(const b200_fe* fe, const VfoSlot* v, int count) {
    if (is_tap(v)) { return std::max(count, 0); }
    if (is_rds_out(v)) {
        // the parent's stages up to its discriminator (the IF blocks are 1:1), then the branch
        const Chain& p = fe->vfos[v->rds_parent]->chain;
        int n = count;
        for (int i = 0; i <= p.quad_index(); i++) { n = p.st[i]->max_out(n); }
        return b200_rds_demod_max_out(v->chain.max_out(n));
    }
    int n = v->chain.max_out(count);
    // the high-pass FIR is 1:1 but its bound has a spare output: whether b200_fe_set_vfo_config switched it on or off since, the
    // bound stays the one b200_fe_add_vfo gave
    for (auto& s : v->chain.st) { n -= s->role == ROLE_HPF ? 1 : 0; }
    n += v->hpf_at_add ? 1 : 0;
    return v->rds ? b200_rds_demod_max_out(n) : n;
}

// the first unused id of the one id space of VFOs, IQ taps and RDS outputs (an unused slot is always a fresh VfoSlot: removing
// or unbinding an id replaces its slot), else a new one at the end; -1 when all B200_MAX_VFOS are taken
static int new_slot_id(b200_fe* fe) {
    for (size_t i = 0; i < fe->vfos.size(); i++) {
        if (!fe->vfos[i]->used) { return (int)i; }
    }
    if (fe->vfos.size() >= B200_MAX_VFOS) { return -1; }
    fe->vfos.push_back(std::make_unique<VfoSlot>());
    return (int)fe->vfos.size() - 1;
}

extern "C" int b200_fe_add_vfo(b200_fe* fe, const b200_vfo_cfg* cfg) {
    if (!fe || !cfg) { set_error("null argument"); return B200_EINVAL; }
    if (cfg->out_samplerate <= 0 || cfg->bandwidth <= 0) { set_error("bad VFO rates"); return B200_EINVAL; }
    if (cfg->demod == B200_DEMOD_AM && cfg->agc_mode != B200_AGC_CARRIER && cfg->agc_mode != B200_AGC_AUDIO) {
        set_error("bad AM agc_mode"); return B200_EINVAL;
    }
    std::lock_guard<std::mutex> lck(fe->mtx);
    const int id = new_slot_id(fe);
    if (id < 0) { set_error("too many VFOs"); return B200_ECAP; }
    VfoSlot* v = fe->vfos[id].get();
    v->cfg = *cfg;
    int rc = build_vfo_chain(fe, v);
    if (rc) { fe->vfos[id] = std::make_unique<VfoSlot>(); return rc; }
    v->used = true;
    return id;
}

// a VFO or an IQ tap
static VfoSlot* get_slot(b200_fe* fe, int id) {
    if (!fe || id < 0 || id >= (int)fe->vfos.size() || !fe->vfos[id]->used) { set_error("bad VFO id %d", id); return nullptr; }
    return fe->vfos[id].get();
}
static VfoSlot* get_vfo(b200_fe* fe, int id) {
    VfoSlot* v = get_slot(fe, id);
    if (v && is_tap(v)) { set_error("id %d is an IQ tap, not a VFO", id); return nullptr; }
    if (v && is_rds_out(v)) { set_error("id %d is the RDS output of VFO %d, not a VFO", id, v->rds_parent); return nullptr; }
    return v;
}

// BroadcastFM::setRDSOut calls reset() (broadcast_fm.h:121-142): the discriminator's previous sample, the stereo stage (pilot
// filter, PLL, delays) and the 15 kHz low-pass restart; RxVFO, the IF chain and the AF chain keep their state.  Device idle.
static void restart_broadcast_fm(VfoSlot* p) {
    Chain& ch = p->chain;
    const int q = ch.quad_index();
    const int n = (p->cfg.demod == B200_DEMOD_WFM_STEREO && p->cfg.low_pass) ? 3 : 2;     // QUAD, FIRR / M2S / STEREO [, FIRC]
    for (int i = q; i < q + n && i < (int)ch.st.size(); i++) { clear_stage_state(*ch.st[i]); }
    cudaDeviceSynchronize();          // legacy-stream memsets: done before the library's streams go on
}

// BroadcastFM's rdsOut (broadcast_fm.h:165-170,196-202) on a WFM VFO: the branch behind its own discriminator, RDSDemod behind it
extern "C" int b200_fe_bind_rds(b200_fe* fe, int vfo_id) {
    if (!fe) { set_error("null fe"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(fe->mtx);
    VfoSlot* p = get_vfo(fe, vfo_id);
    if (!p) { return B200_EINVAL; }
    if (p->cfg.demod != B200_DEMOD_WFM && p->cfg.demod != B200_DEMOD_WFM_STEREO) {
        set_error("VFO %d: RDS binds to a B200_DEMOD_WFM or B200_DEMOD_WFM_STEREO VFO", vfo_id);
        return B200_EINVAL;
    }
    if (p->rds_child >= 0) { set_error("VFO %d already has an RDS output (id %d)", vfo_id, p->rds_child); return B200_EINVAL; }
    B200_CK(cudaDeviceSynchronize());
    const int id = new_slot_id(fe);
    if (id < 0) { set_error("too many VFOs, IQ taps and RDS outputs"); return B200_ECAP; }
    QuadStage* q = (QuadStage*)p->chain.st[p->chain.quad_index()].get();
    if (p->rds_parked) {
        // the branch resumes where the unbind left it: the reference's xlator, rdsResamp and rdsDemod are not reset by the toggle
        fe->vfos[id] = std::move(p->rds_parked);
    }
    else {
        auto b = std::make_unique<VfoSlot>();
        int n_max = fe->max_eff;
        for (int i = 0; i <= p->chain.quad_index(); i++) { n_max = p->chain.st[i]->max_out(n_max); }
        int rc = b->chain.add_rds_branch(p->cfg.out_samplerate);
        if (!rc) { rc = b->chain.finalize(n_max); }
        if (!rc) { rc = add_rds_demod(fe, b.get(), b->chain.max_out(n_max)); }
        if (rc) { return rc; }
        b->chain.parent = &p->chain;
        b->rds_parent = vfo_id;
        b->used = true;
        fe->vfos[id] = std::move(b);
    }
    q->side = (RxlStage*)fe->vfos[id]->chain.st[0].get();
    p->rds_child = id;
    restart_broadcast_fm(p);
    return id;
}
extern "C" int b200_fe_unbind_rds(b200_fe* fe, int id) {
    if (!fe) { set_error("null fe"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(fe->mtx);
    VfoSlot* v = get_slot(fe, id);
    if (!v) { return B200_EINVAL; }
    if (!is_rds_out(v)) { set_error("id %d is not an RDS output", id); return B200_EINVAL; }
    B200_CK(cudaDeviceSynchronize());
    VfoSlot* p = fe->vfos[v->rds_parent].get();
    ((QuadStage*)p->chain.st[p->chain.quad_index()].get())->side = nullptr;
    p->rds_child = -1;
    p->rds_parked = std::move(fe->vfos[id]);          // parked with its state, as chain::setBlockEnabled keeps a disabled block
    fe->vfos[id] = std::make_unique<VfoSlot>();
    restart_broadcast_fm(p);
    return 0;
}

// IQFrontEnd::bindIQStream / unbindIQStream (iq_frontend.h:34-35): an id of the VFO id space, no state of its own
extern "C" int b200_fe_bind_iq(b200_fe* fe, int sample_type, float scalar) {
    if (!fe) { set_error("null fe"); return B200_EINVAL; }
    if (sample_type < B200_IQ_CF32 || sample_type > B200_IQ_I32) { set_error("bad IQ sample type %d", sample_type); return B200_EINVAL; }
    if (!std::isfinite(scalar)) { set_error("IQ tap scalar must be finite"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(fe->mtx);
    if (!fe->tap_stream) {
        // the most urgent priority: the chunk's outputs wait for this short, memory-bound launch, which at the least urgent
        // one queued behind stage 1 for up to 1.9 ms of a 3 ms step (DESIGN.md section 10)
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);
        if (cudaStreamCreateWithPriority(&fe->tap_stream, cudaStreamNonBlocking, hi) != cudaSuccess ||
            cudaEventCreateWithFlags(&fe->ev_tap_go, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&fe->ev_tap_done, cudaEventDisableTiming) != cudaSuccess) {
            return cuda_fail(cudaGetLastError(), "IQ tap stream/event creation");
        }
    }
    const int id = new_slot_id(fe);
    if (id < 0) { set_error("too many VFOs and IQ taps"); return B200_ECAP; }
    VfoSlot* v = fe->vfos[id].get();
    v->tap_type = sample_type;
    v->tap_scalar = (sample_type == B200_IQ_CF32 || sample_type == B200_IQ_U8) ? 0.0f : scalar;
    v->used = true;
    return id;
}
extern "C" int b200_fe_unbind_iq(b200_fe* fe, int id) {
    if (!fe) { set_error("null fe"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(fe->mtx);
    VfoSlot* v = get_slot(fe, id);
    if (!v) { return B200_EINVAL; }
    if (!is_tap(v)) { set_error("id %d is a VFO, not an IQ tap", id); return B200_EINVAL; }
    B200_CK(cudaDeviceSynchronize());
    fe->vfos[id] = std::make_unique<VfoSlot>();
    return 0;
}

extern "C" int b200_fe_remove_vfo(b200_fe* fe, int id) {
    if (!fe) { set_error("null fe"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(fe->mtx);
    VfoSlot* v = get_vfo(fe, id);
    if (!v) { return B200_EINVAL; }
    if (v->rds_child >= 0) { set_error("VFO %d has an RDS output (id %d): unbind it first", id, v->rds_child); return B200_ESTATE; }
    B200_CK(cudaDeviceSynchronize());
    fe->vfos[id] = std::make_unique<VfoSlot>();
    return 0;
}
extern "C" int b200_fe_set_vfo_offset(b200_fe* fe, int id, double offset) {
    if (!fe) { set_error("null fe"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(fe->mtx);
    VfoSlot* v = get_vfo(fe, id);
    if (!v) { return B200_EINVAL; }
    v->pend_offset = true;
    v->new_offset = offset;
    return 0;
}
extern "C" int b200_fe_set_vfo_bandwidth(b200_fe* fe, int id, double bw) {
    if (!fe) { set_error("null fe"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(fe->mtx);
    VfoSlot* v = get_vfo(fe, id);
    if (!v || bw <= 0) { set_error("bad bandwidth"); return B200_EINVAL; }
    v->pend_bw = true;
    v->new_bw = bw;
    return 0;
}
// the radio module's setters (radio_module.h:606-760) between chunks: checked here, taken whole by apply_pending
extern "C" int b200_fe_set_vfo_config(b200_fe* fe, int id, const b200_vfo_cfg* cfg) {
    if (!fe || !cfg) { set_error("null argument"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(fe->mtx);
    VfoSlot* v = get_vfo(fe, id);
    if (!v) { return B200_EINVAL; }
    const b200_vfo_cfg& o = v->cfg;
    const char* field = cfg->demod != o.demod ? "demod" : cfg->out_samplerate != o.out_samplerate ? "out_samplerate" :
                        cfg->deviation != o.deviation ? "deviation" : cfg->low_pass != o.low_pass ? "low_pass" :
                        cfg->af_samplerate != o.af_samplerate ? "af_samplerate" : nullptr;
    if (field) {
        set_error("VFO %d: %s needs a new demodulator or AF resampler: remove the VFO and add it again", id, field);
        return B200_EINVAL;
    }
    if (cfg->bandwidth <= 0) { set_error("bad bandwidth"); return B200_EINVAL; }
    if (o.demod == B200_DEMOD_AM && cfg->agc_mode != B200_AGC_CARRIER && cfg->agc_mode != B200_AGC_AUDIO) { set_error("bad AM agc_mode"); return B200_EINVAL; }
    if (cfg->nr_on && !fmif_supported(cfg->nr_bins)) {
        set_error("FM IF noise reduction: %d bins (supported: 2 ... %d)", cfg->nr_bins, 64);
        return B200_EINVAL;
    }
    // offset and bandwidth go the way of b200_fe_set_vfo_offset / _bandwidth; the last call before a chunk wins
    v->pend_offset = cfg->offset != o.offset;
    v->new_offset = cfg->offset;
    v->pend_bw = cfg->bandwidth != o.bandwidth;
    v->new_bw = cfg->bandwidth;
    v->new_cfg = *cfg;
    v->pend_cfg = true;
    return 0;
}
extern "C" int b200_fe_vfo_count(b200_fe* fe) {
    if (!fe) { return 0; }
    int n = 0;
    for (auto& v : fe->vfos) { n += v->used ? 1 : 0; }
    return n;
}
extern "C" int b200_fe_vfo_max_out(b200_fe* fe, int id, int count) {
    VfoSlot* v = get_slot(fe, id);
    return v ? vfo_out_bound(fe, v, count) : B200_EINVAL;
}
extern "C" int b200_fe_fft_max_lines(b200_fe* fe, int count) {
    if (!fe || !fe->fft_on) { return 0; }
    return (int)(count / ((long long)fe->fft.nz + fe->skip)) + 2;
}
extern "C" long long b200_fe_launch_count(b200_fe* fe) { return fe ? fe->sch.launches : 0; }
extern "C" long long b200_fe_stat(b200_fe* fe, const char* key) {
    if (!fe || !key) { return -1; }
    if (!strcmp(key, "launches")) { return fe->sch.launches; }
    if (!strcmp(key, "s1_tma_launches")) { return fe->sch.s1_tma_launches; }
    if (!strcmp(key, "s1_f2_jobs")) { return fe->sch.s1_f2_jobs; }
    if (!strcmp(key, "chunks")) { return (long long)fe->nsub; }
    // host time spent inside b200_fe_submit since creation, by section (ns)
    if (!strcmp(key, "host_ns_plan")) { return fe->host_ns[0]; }
    if (!strcmp(key, "host_ns_fft")) { return fe->host_ns[1]; }
    if (!strcmp(key, "host_ns_run")) { return fe->host_ns[2]; }
    if (!strcmp(key, "host_ns_join")) { return fe->host_ns[3]; }
    if (!strcmp(key, "graph_hits")) { return fe->sch.graph_hits; }
    if (!strcmp(key, "graph_misses")) { return fe->sch.graph_misses; }
    if (!strcmp(key, "graphs")) { return (long long)fe->sch.graphs.size(); }
    if (!strcmp(key, "host_ns_stage1")) { return fe->sch.host_ns[0]; }
    if (!strcmp(key, "host_ns_tail")) { return fe->sch.host_ns[1]; }
    if (!strcmp(key, "fused_chains")) {
        long long n = 0;
        for (auto& v : fe->vfos) { n += (v->used && v->chain.fp.active) ? 1 : 0; }
        return n;
    }
    return -1;
}
// the captured graphs of both schedulers hold launches made with the old kernel choices
static void fe_drop_graphs(b200_fe* fe) {
    fe->sch.drop_graphs();
    fe->sch_pre.drop_graphs();
}
extern "C" int b200_fe_set_option(b200_fe* fe, const char* key, int value) {
    if (!fe || !key) { set_error("null argument"); return B200_EINVAL; }
    if (!strcmp(key, "s1")) { fe->sch.s1_variant = value; return 0; }
    if (!strcmp(key, "overlap")) {
        if (b200_fe_vfo_count(fe) > 0) { set_error("'overlap' must be chosen before VFOs are added"); return B200_ESTATE; }
        if (cudaDeviceSynchronize() != cudaSuccess) { return cuda_fail(cudaGetLastError(), "sync"); }
        fe->sch.tail_stream = value ? fe->tail_stream : nullptr;
        return 0;
    }
    if (!strcmp(key, "pair")) { fe->sch.pair_conjugates = value != 0; return 0; }
    if (!strcmp(key, "s1_mt")) { fe->opts.s1_mt = value; return 0; }
    if (!strcmp(key, "s1_stages")) { fe->opts.s1_stages = value == 3 ? 3 : 2; return 0; }
    if (!strcmp(key, "s1_diag")) { fe->opts.s1_diag = value & 3; return 0; }                     // measurement only: outputs are garbage
    if (!strcmp(key, "s1_ctas")) { fe->opts.s1_ctas = value; return 0; }
    if (!strcmp(key, "tails") || !strncmp(key, "ft_", 3)) {
        // 0: one thread per output; 1: shared-memory tiled kernels, one launch per stage; 2: one fused launch per <= 16 VFOs
        if (b200_fe_vfo_count(fe) > 0) { set_error("'%s' must be chosen before VFOs are added", key); return B200_ESTATE; }
        if (!strcmp(key, "tails")) { fe->opts.tail_variant = value >= 1 ? 1 : 0; fe->sch.fuse.on = value >= 2; fe_drop_graphs(fe); return 0; }
        if (!strcmp(key, "ft_ob")) { fe->sch.fuse.ob_force = value; return 0; }
        if (!strcmp(key, "ft_obmax")) { fe->sch.fuse.ob_max = value; return 0; }
        if (!strcmp(key, "ft_smem_kb")) { fe->sch.fuse.smem_limit = value * 1024; return 0; }
        if (!strcmp(key, "ft_threads")) { fe->sch.fuse.threads = value; return 0; }
        if (!strcmp(key, "ft_direct")) { fe->sch.fuse.direct = value != 0; return 0; }
        if (!strcmp(key, "ft_prereg")) { fe->sch.fuse.pre_reg = value; return 0; }
        if (!strcmp(key, "ft_regall")) { fe->sch.fuse.reg_all = value != 0; return 0; }
    }
    if (!strcmp(key, "fft")) { fe->opts.fft_variant = value; return 0; }
    if (!strcmp(key, "fft_cta")) { fe->opts.fft_cta = value == 4 ? 4 : 8; return 0; }
    if (!strcmp(key, "host_direct")) { fe->host_direct = value; return 0; }
    if (!strcmp(key, "inflight")) {
        if (value < 1 || value > FE_SLOTS) { set_error("inflight: 1 ... %d", FE_SLOTS); return B200_EINVAL; }
        fe->max_inflight = value;
        return 0;
    }
    if (!strcmp(key, "fft_v")) {
        if (value != 0 && value != 1) { set_error("fft_v: 0 or 1"); return B200_EINVAL; }
        std::lock_guard<std::mutex> lck(fe->mtx);
        fe->fft_v = value;
        return 0;
    }
    if (!strcmp(key, "graph")) { fe->sch.graph_tails = value; if (value == 0) { fe->sch.drop_graphs(); } return 0; }
    if (!strcmp(key, "graph_max_count")) { fe->sch.graph_max_count = value; return 0; }
    if (!strcmp(key, "pdl")) { fe->opts.pdl = (value >= 0 && value <= 2) ? value : PDL_DEFAULT; fe_drop_graphs(fe); return 0; }
    if (!strcmp(key, "time_s1")) { fe->sch.time_s1 = value != 0; for (auto& t : fe->sch.timers) { t.used = 0; } return 0; }
    set_error("unknown option %s", key);
    return B200_EINVAL;
}

extern "C" int b200_fe_s1_stats(b200_fe* fe, double* ms_total, int* launches) {
    if (!fe || !ms_total || !launches) { set_error("null argument"); return B200_EINVAL; }
    return fe->sch.s1_stats(ms_total, launches);
}
extern "C" int b200_fe_group_stats(b200_fe* fe, int group, double* ms_total, int* launches) {
    if (!fe || !ms_total || !launches) { set_error("null argument"); return B200_EINVAL; }
    return fe->sch.group_stats(group, ms_total, launches);
}

extern "C" int b200_fe_reset(b200_fe* fe) {
    if (!fe) { set_error("null fe"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(fe->mtx);
    B200_CK(cudaDeviceSynchronize());
    for (auto& v : fe->vfos) {
        if (v->used && !is_tap(v.get())) { v->chain.reset_state(); }     // a tap has no state: it reads what the reset below clears
        if (v->used && v->rds) { int rcr = v->rds->reset(nullptr); if (rcr) { return rcr; } }
        for (auto& p : v->parked) { if (p) { clear_stage_state(*p); } }     // a block switched on later starts fresh
        if (v->rds_parked) {                                                 // so does an RDS branch bound again later
            v->rds_parked->chain.reset_state();
            int rcr = v->rds_parked->rds->reset(nullptr);
            if (rcr) { return rcr; }
        }
    }
    B200_CK(cudaDeviceSynchronize());
    int rc = fe->sch.reset_raw();
    if (!fe->pre.st.empty()) { fe->pre.reset_state(); }
    if (fe->dc_state.p) { B200_CK(cudaMemset(fe->dc_state.p, 0, 16)); B200_CK(cudaDeviceSynchronize()); }
    fe->pos = 0;
    fe->fstart = 0;
    return rc;
}

// pinned buffers handed out by b200_host_alloc: under unified addressing the device can store into them directly, which is
// how the audio of a small chunk leaves (no copy to enqueue).  Anything else goes through cudaMemcpyAsync.
static std::mutex g_host_mtx;
static std::map<uintptr_t, size_t> g_host_allocs;
static bool host_buffer_is_ours(const void* p, size_t bytes) {
    std::lock_guard<std::mutex> lk(g_host_mtx);
    auto it = g_host_allocs.upper_bound((uintptr_t)p);
    if (it == g_host_allocs.begin()) { return false; }
    --it;
    return (uintptr_t)p + bytes <= it->first + it->second;
}

static inline long long host_clock_ns() {
    return (long long)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// A VFO's stages with the IF / AF blocks in `order` and the switched-off blocks in `parked`.  Every stage comes from the chain,
// the parked slots or `pool`; what is left over goes to `pool`.
static void place_stages(VfoSlot* v, const std::vector<Stage*>& order, Stage* const* parked, std::vector<std::unique_ptr<Stage>>& pool) {
    for (auto& s : v->chain.st) { pool.push_back(std::move(s)); }
    for (auto& p : v->parked) { if (p) { pool.push_back(std::move(p)); } }
    v->chain.st.clear();
    auto take = [&](Stage* s) {
        std::unique_ptr<Stage> u;
        for (auto& q : pool) { if (q.get() == s) { u = std::move(q); break; } }
        return u;
    };
    for (Stage* s : order) { v->chain.st.push_back(take(s)); }
    for (int r = 0; r < ROLE_COUNT; r++) { if (parked[r]) { v->parked[r] = take(parked[r]); } }
    pool.erase(std::remove(pool.begin(), pool.end(), nullptr), pool.end());
}

// b200_fe_set_vfo_config at the chunk boundary.  Coefficients: the host-side parameters the next launch list carries (no device
// wait).  AGC mode (AM::setAGCMode -> reset, am.h:49-56) and bin count (FMIF::setBins, fm_if.h:26-34): that block restarts.
// Blocks switched on / off: chain::setBlockEnabled (chain.h:61-127) -- the other stages keep their buffers and state, a block
// switched off is parked as it is and carries on from there when switched on again.  On an error the VFO is left as it was.
static int apply_vfo_config(VfoSlot* v, const b200_vfo_cfg& n) {
    const b200_vfo_cfg& o = v->cfg;
    Chain& ch = v->chain;
    const bool audio = vfo_has_audio(o), af = audio && o.af_samplerate > 0;
    bool want[ROLE_COUNT] = {};
    want[ROLE_NB] = n.nb_on != 0;
    want[ROLE_SQUELCH] = n.squelch_on != 0;
    want[ROLE_NR] = n.nr_on != 0;
    want[ROLE_HPF] = af && n.af_high_pass;
    want[ROLE_DEEMPH] = af && n.af_deemph_tau > 0.0;
    want[ROLE_VOLUME] = audio && n.af_volume_on;
    Stage* live[ROLE_COUNT] = {};
    for (auto& s : ch.st) { if (s->role) { live[s->role] = s.get(); } }
    const bool new_bins = n.nr_bins != o.nr_bins;            // FMIF::setBins: the block restarts with the new bin count
    bool topo = new_bins && (live[ROLE_NR] || v->parked[ROLE_NR]);
    for (int r = ROLE_NB; r <= ROLE_VOLUME; r++) { topo = topo || want[r] != (live[r] != nullptr); }
    const bool am_restart = o.demod == B200_DEMOD_AM && n.agc_mode != o.agc_mode && live[ROLE_DEMOD];
    if (topo || am_restart) { B200_CK(cudaDeviceSynchronize()); }     // chunks in flight still read the stages
    if (topo) {
        // new stages first: nothing has changed when one of them fails
        std::unique_ptr<Stage> fresh[ROLE_COUNT];
        const size_t after_chan = (size_t)ch.chan_fir + 1;
        const int if_cap = after_chan < ch.st.size() ? ch.st[after_chan]->cap_in : ch.out_cap;    // every toggled block is 1:1
        for (int r = ROLE_NB; r <= ROLE_VOLUME; r++) {
            const bool reuse = (live[r] || v->parked[r]) && !(r == ROLE_NR && new_bins);
            if (!want[r] || reuse) { continue; }
            Chain tmp;
            int rc = 0;
            switch (r) {
            case ROLE_NB: rc = tmp.add_noise_blanker(500.0 / o.out_samplerate, n.nb_level); break;
            case ROLE_SQUELCH: rc = tmp.add_squelch(n.squelch_level); break;
            case ROLE_NR: rc = tmp.add_fmif(n.nr_bins); break;
            case ROLE_HPF: rc = tmp.add_af_highpass(o.af_samplerate); break;
            case ROLE_DEEMPH: rc = tmp.add_deemph(n.af_deemph_tau, o.af_samplerate); break;
            default: rc = tmp.add_volume(n.af_volume, n.af_muted != 0); break;
            }
            if (rc) { return rc; }
            fresh[r] = std::move(tmp.st[0]);
            fresh[r]->role = r;
            if (r == ROLE_VOLUME) { fresh[r]->in_es = fresh[r]->out_es = ch.out_es; }
            if ((rc = fresh[r]->alloc_in(role_in_if_chain(r) ? if_cap : ch.out_cap))) { return rc; }
        }
        auto pick = [&](int r) -> Stage* {
            if (!want[r]) { return nullptr; }
            if (fresh[r]) { return fresh[r].get(); }
            return live[r] ? live[r] : v->parked[r].get();
        };
        // the new order: IF blocks right behind the channel filter, AF blocks at the end, as build_vfo_chain places them
        std::vector<Stage*> order, old_order;
        Stage* parked[ROLE_COUNT] = {};
        Stage* old_parked[ROLE_COUNT] = {};
        for (size_t i = 0; i < ch.st.size(); i++) {
            Stage* s = ch.st[i].get();
            old_order.push_back(s);
            if (!role_in_if_chain(s->role) && !role_in_af_chain(s->role)) { order.push_back(s); }
            if ((int)i == ch.chan_fir) {
                for (int r = ROLE_NB; r <= ROLE_NR; r++) { if (pick(r)) { order.push_back(pick(r)); } }
            }
        }
        for (int r = ROLE_HPF; r <= ROLE_VOLUME; r++) { if (pick(r)) { order.push_back(pick(r)); } }
        for (int r = ROLE_NB; r <= ROLE_VOLUME; r++) {
            old_parked[r] = v->parked[r].get();
            if (!want[r] && !(r == ROLE_NR && new_bins)) { parked[r] = live[r] ? live[r] : v->parked[r].get(); }
        }
        std::vector<std::unique_ptr<Stage>> pool;
        for (auto& f : fresh) { if (f) { pool.push_back(std::move(f)); } }
        int rc = ch.unfuse_history();
        if (!rc) {
            place_stages(v, order, parked, pool);
            rc = ch.restage();
            if (rc) {
                place_stages(v, old_order, old_parked, pool);
                int rc2 = ch.restage();
                if (rc2) { return rc2; }
            }
        }
        if (rc) { return rc; }
    }
    // coefficients, on the running and on the parked stages
    auto coef = [&](Stage* s) {
        switch (s->role) {
        case ROLE_NB: ((SeqStage*)s)->proto.nb_level = (float)n.nb_level; break;                 // NoiseBlanker::setLevel
        case ROLE_SQUELCH: ((SquelchStage*)s)->level = (float)n.squelch_level; break;             // PowerSquelch::setLevel
        case ROLE_DEEMPH: if (n.af_deemph_tau > 0.0) { ((SeqStage*)s)->set_deemph_tau(n.af_deemph_tau, o.af_samplerate); } break;
        case ROLE_VOLUME: ((ScaleStage*)s)->gain = n.af_muted ? 0.0f : powf((float)n.af_volume, 2); break;   // Volume::setVolume / setMuted
        case ROLE_DEMOD: {
            SeqStage* q = (SeqStage*)s;
            q->set_agc(n.agc_attack, n.agc_decay);                                                   // AM / SSB setAGCAttack / setAGCDecay
            if (o.demod == B200_DEMOD_AM) { q->proto.dc_rate = (float)n.dc_block_rate; q->proto.agc_mode = n.agc_mode; }   // setDCBlockRate
            break;
        }
        default: break;
        }
    };
    for (auto& s : ch.st) { coef(s.get()); }
    for (auto& p : v->parked) { if (p) { coef(p.get()); } }
    if (am_restart) {
        // AM::reset: both AGCs and the DC blocker start over; the audio low-pass keeps its delay line
        SeqStage* q = nullptr;
        for (auto& s : ch.st) { if (s->role == ROLE_DEMOD) { q = (SeqStage*)s.get(); } }
        B200_CK(cudaMemcpy(q->state.p, q->init_state, sizeof(q->init_state), cudaMemcpyHostToDevice));
        B200_CK(cudaDeviceSynchronize());      // legacy-stream copy: done before the library's streams go on
    }
    const double off = v->cfg.offset, bw = v->cfg.bandwidth;      // routed through pend_offset / pend_bw
    v->cfg = n;
    v->cfg.offset = off;
    v->cfg.bandwidth = bw;
    return 0;
}

// apply RxVFO::setOffset / setBandwidth at the chunk boundary (rx_vfo.h:60-77), and b200_fe_set_vfo_config
static int apply_pending(b200_fe* fe) {
    for (auto& up : fe->vfos) {
        VfoSlot* v = up.get();
        if (!v->used || is_tap(v)) { continue; }
        if (v->pend_cfg) {
            v->pend_cfg = false;
            int rc = apply_vfo_config(v, v->new_cfg);
            if (rc) { return rc; }
        }
        if (v->pend_offset) {
            v->cfg.offset = v->new_offset;
            ((XdStage*)v->chain.st[0].get())->set_offset_rad(hz_to_rads(-v->cfg.offset, fe->fs_eff));
            v->pend_offset = false;
        }
        if (v->pend_bw) {
            // RxVFO::setBandwidth (rx_vfo.h:60-70): only the channel filter follows the bandwidth; bandwidth == outSR
            // bypasses it (identity tap here, Chain::add_rxvfo)
            FirCStage* f = v->chain.chan_fir >= 0 ? (FirCStage*)v->chain.st[v->chain.chan_fir].get() : nullptr;
            if (f) {
                double fw = v->new_bw / 2.0;
                f->pending = (v->new_bw != v->cfg.out_samplerate) ? lowpass_taps(fw, fw * 0.1, v->cfg.out_samplerate) : std::vector<float>{ 1.0f };
                v->cfg.bandwidth = v->new_bw;
            }
            v->pend_bw = false;
        }
    }
    return 0;
}

// One chunk on its way through b200_fe_submit: what its steps hand each other
struct FeChunk {
    int slot = 0;                            // input slot and event set: nsub % FE_SLOTS
    b200_outputs* out = nullptr;
    // the chunk as submitted (in: on the device once fe_upload has run), and the effective stream behind the pre-processing
    // that the spectrum branch, the IQ taps and the VFOs read.  scale: (float)x * scale for the integer formats
    const void* in = nullptr, *ein = nullptr;
    int fmt = 0, count = 0, efmt = 0, ecount = 0;
    float scale = 0.0f, escale = 0.0f;
    std::vector<Chain*> chains;              // every VFO's chain, a bound RDS branch right behind its parent's
    std::vector<int> ids;                    // the VFO id of chains[k]
    std::vector<int> taps;                   // IQ tap ids
    bool direct = false;                     // device outputs
    bool kernel_out[B200_MAX_VFOS] = {};     // by id: the output's last kernel writes the caller's buffer, no copy
    std::vector<size_t> tap_off;             // taps[k]'s region in tap_stage[slot] when it leaves by a copy
    bool fft_forked = false, tap_forked = false;
    int nlines = 0;                          // FFT lines the chunk completes
};

// the used slots: VFO chains, each bound RDS branch right behind the VFO whose discriminator feeds it (Chain::parent); IQ taps
static void fe_branches(b200_fe* fe, FeChunk& c) {
    for (size_t i = 0; i < fe->vfos.size(); i++) {
        const VfoSlot* v = fe->vfos[i].get();
        if (!v->used || is_rds_out(v)) { continue; }
        if (is_tap(v)) { c.taps.push_back((int)i); continue; }
        c.chains.push_back(&fe->vfos[i]->chain); c.ids.push_back((int)i);
        if (v->rds_child >= 0) { c.chains.push_back(&fe->vfos[v->rds_child]->chain); c.ids.push_back(v->rds_child); }
    }
}

// the spectrum frames that complete by stream position `end`: the frame at fstart and those behind it, nz + skip apart
static int fft_frames_by(const b200_fe* fe, unsigned long long end) {
    const unsigned long long nz = (unsigned long long)fe->fft.nz, interval = nz + (unsigned long long)fe->skip;
    return fe->fstart + nz <= end ? (int)((end - fe->fstart - nz) / interval) + 1 : 0;
}

// every capacity check against the exact counts, before anything is enqueued and before any state moves
static int fe_check_outputs(b200_fe* fe, FeChunk& c) {
    const b200_outputs* out = c.out;
    // samples that reach the FFT branch and the VFOs: the chunk itself, or what the input decimator makes of it
    c.ecount = (fe->decim > 1) ? fe->pre.peek(c.count) : c.count;
    if (c.ecount < 0) { set_error("input decimator is not a FIR cascade"); return B200_ESTATE; }
    for (const std::vector<int>* ids : { &c.ids, &c.taps }) {
        for (int id : *ids) {
            const VfoSlot* v = fe->vfos[id].get();
            const int bound = vfo_out_bound(fe, v, c.ecount);
            if (out->vfo_out[id] == nullptr || out->vfo_cap[id] < bound) {
                set_error("%s %d output buffer too small: need room for %d samples (b200_fe_vfo_max_out)", is_tap(v) ? "IQ tap" : "VFO", id, bound);
                return B200_ECAP;
            }
        }
    }
    if (fe->fft_on) {
        const int need = fft_frames_by(fe, fe->pos + (unsigned long long)c.ecount);
        if (need > fe->max_lines) { set_error("FFT line buffer overflow: %d lines complete in this chunk, room for %d", need, fe->max_lines); return B200_ECAP; }
        if (need > 0 && (out->fft_out == nullptr || out->fft_cap_lines < need)) {
            set_error("FFT output buffer too small: %d lines complete in this chunk", need);
            return B200_ECAP;
        }
    }
    return 0;
}

// a host chunk goes to in_dev[slot] on the copy stream, once the chunk that used the slot before is done with it; the main
// stream waits for the copy
static int fe_upload(b200_fe* fe, FeChunk& c, const void* iq, int in_mem) {
    c.in = iq;
    if (in_mem != B200_MEM_HOST || c.count == 0) { return 0; }
    const size_t in_bytes = (size_t)c.count * bytes_per_sample(c.fmt);
    DevBuf& buf = fe->in_dev[c.slot];
    if (buf.bytes < in_bytes) {
        B200_CK(cudaStreamSynchronize(fe->sch.stream));
        int rc = buf.alloc(std::max(in_bytes, (size_t)fe->max_chunk * bytes_per_sample(c.fmt)), false);
        if (rc) { return rc; }
    }
    if (fe->slot_used[c.slot]) { B200_CK(cudaStreamWaitEvent(fe->copy_stream, fe->ev_compute[c.slot], 0)); }
    trace_mark("h2d start", fe->copy_stream);
    B200_CK(cudaMemcpyAsync(buf.p, iq, in_bytes, cudaMemcpyHostToDevice, fe->copy_stream));
    trace_mark("h2d done", fe->copy_stream);
    B200_CK(cudaEventRecord(fe->ev_h2d[c.slot], fe->copy_stream));
    B200_CK(cudaStreamWaitEvent(fe->sch.stream, fe->ev_h2d[c.slot], 0));
    c.in = buf.p;
    return 0;
}

// The chains' deferred filter changes, then IQFrontEnd's pre-processing chain (iq_frontend.cpp:32-39): decimator -> DC
// blocker -> conjugate, on the main stream.  Then every chain plans the chunk.
static int fe_preprocess(b200_fe* fe, FeChunk& c) {
    int rc = fe->sch.apply_deferred(c.chains);
    if (rc) { return rc; }
    cudaStream_t s = fe->sch.stream;
    c.ein = c.in; c.efmt = c.fmt; c.escale = c.scale;
    const bool any = fe->decim > 1 || fe->dc_block || fe->invert_iq;
    if (any && fe->slot_used[c.slot]) { B200_CK(cudaStreamWaitEvent(s, fe->ev_compute[c.slot], 0)); }     // pp[slot] of two chunks ago
    if (fe->decim > 1) {
        // the decimator's output is one buffer: the last chunk's IQ taps may still be reading it
        if (fe->tap_read_pre) { B200_CK(cudaStreamWaitEvent(s, fe->ev_tap_done, 0)); }
        cudaError_t e = launch_convert_cf32(c.in, c.fmt, (float2*)fe->pre.st[0]->in_data(), c.count, c.scale, s);
        if (e != cudaSuccess) { return cuda_fail(e, "launch_convert_cf32"); }
        fe->sch.launches++;
        fe->pre.plan(c.count);
        std::vector<Chain*> pc{ &fe->pre };
        const long long l0 = fe->sch_pre.launches;
        fe->sch_pre.stream = s;
        if ((rc = fe->sch_pre.run(pc, nullptr, FMT_CF32, c.count, false))) { return rc; }
        fe->sch.launches += fe->sch_pre.launches - l0;
        c.ein = fe->pre.out.p; c.efmt = FMT_CF32; c.escale = 0.0f;
    }
    if (fe->dc_block || fe->invert_iq) {
        const size_t need = ((size_t)fe->max_eff + 8) * sizeof(float2);
        if (fe->pp[c.slot].bytes < need && (rc = fe->pp[c.slot].alloc(need, false))) { return rc; }
        const int nseg_max = fe->max_eff / 4096 + 2;
        if (!fe->dc_state.p && ((rc = fe->dc_state.alloc(16)) || (rc = fe->dc_segA.alloc((size_t)nseg_max * sizeof(float), false)) ||
                                (rc = fe->dc_segB.alloc((size_t)nseg_max * sizeof(float2), false)))) { return rc; }
        DcbParams dp;
        memset(&dp, 0, sizeof(dp));
        dp.in = c.ein; dp.out = fe->pp[c.slot].as<float2>(); dp.fmt = c.efmt; dp.count = c.ecount; dp.in_scale = c.escale;
        dp.rate = (float)(50.0 / fe->fs_eff);                      // genDCBlockRate (iq_frontend.h:55-57)
        dp.dc_on = fe->dc_block ? 1 : 0; dp.conj_on = fe->invert_iq ? 1 : 0;
        dp.state = fe->dc_state.as<float2>(); dp.segA = fe->dc_segA.as<float>(); dp.segB = fe->dc_segB.as<float2>();
        dp.nseg = (c.ecount + 4095) / 4096;
        int nl = 0;
        cudaError_t e = launch_preproc(dp, s, &nl);
        if (e != cudaSuccess) { return cuda_fail(e, "launch_preproc"); }
        fe->sch.launches += nl;
        c.ein = fe->pp[c.slot].p; c.efmt = FMT_CF32; c.escale = 0.0f;
    }
    for (Chain* ch : c.chains) { ch->plan(ch->parent ? ch->parent->st[ch->parent->quad_index()]->n_out : c.ecount); }
    return 0;
}

// Whether the last kernel of output `id` writes the caller's buffer itself, with no copy on the join stream: always for
// device outputs; a host buffer from b200_host_alloc (stored over PCIe) under "host_direct" 1, or under -1 for chunks up to
// 4 Mi samples whose output is at most max_bytes -- large ones keep the copy engine: a kernel's own stores moved a 1 Mi-sample
// CF32 IQ tap (8 MiB) at a third of its rate.
static bool kernel_writes_out(const b200_fe* fe, const FeChunk& c, int id, size_t elem_bytes, size_t max_bytes) {
    if (c.direct) { return true; }
    if (fe->host_direct == 0 || (fe->host_direct < 0 && (c.ecount > (1 << 22) || (size_t)c.ecount * elem_bytes > max_bytes))) { return false; }
    return host_buffer_is_ours(c.out->vfo_out[id], (size_t)c.out->vfo_cap[id] * elem_bytes);
}

static void fe_route_outputs(b200_fe* fe, FeChunk& c) {
    for (size_t k = 0; k < c.chains.size(); k++) {
        const int id = c.ids[k];
        c.kernel_out[id] = kernel_writes_out(fe, c, id, (size_t)c.chains[k]->out_es * sizeof(float), SIZE_MAX);
        // an RDS VFO's chain output stays in the chain: RDSDemod reads it there and writes the caller's buffer itself
        c.chains[k]->out_override = (c.kernel_out[id] && !fe->vfos[id]->rds) ? (float*)c.out->vfo_out[id] : nullptr;
    }
    for (int id : c.taps) { c.kernel_out[id] = kernel_writes_out(fe, c, id, iq_tap_bytes(fe->vfos[id]->tap_type), 64 << 10); }
}

// IQ taps: k_iq_tap reads the effective stream once and stores every tap, on its own stream so that neither the VFO branch
// nor the spectrum branch waits for it.  A tap whose kernel does not write the caller's buffer fills its region of
// tap_stage[slot], copied out on the join stream.  tap_stage[slot] was last read by the copies of chunk nsub - FE_SLOTS,
// which b200_fe_wait has seen complete.
static int fe_iq_taps(b200_fe* fe, FeChunk& c) {
    if (c.taps.empty() || c.ecount == 0) { fe->tap_read_pre = false; return 0; }
    c.tap_off.assign(c.taps.size(), 0);
    size_t need = 0, need_max = 0;
    for (size_t k = 0; k < c.taps.size(); k++) {
        if (c.kernel_out[c.taps[k]]) { continue; }
        const size_t b = iq_tap_bytes(fe->vfos[c.taps[k]]->tap_type);
        c.tap_off[k] = need;
        need += ((size_t)c.ecount * b + 15) & ~(size_t)15;
        need_max += ((size_t)fe->max_eff * b + 15) & ~(size_t)15;
    }
    int rc;
    if (fe->tap_stage[c.slot].bytes < need && (rc = fe->tap_stage[c.slot].alloc(need_max, false))) { return rc; }
    B200_CK(cudaEventRecord(fe->ev_tap_go, fe->sch.stream));
    B200_CK(cudaStreamWaitEvent(fe->tap_stream, fe->ev_tap_go, 0));
    cudaEvent_t t_tap = fe->sch.timer_begin(3, fe->tap_stream);
    IqTapParams tp;
    memset(&tp, 0, sizeof(tp));
    tp.in = c.ein; tp.fmt = c.efmt; tp.n = c.ecount; tp.in_scale = c.escale;
    auto aligned = [](const void* p) { return ((uintptr_t)p & 15) == 0; };
    for (size_t k0 = 0; k0 < c.taps.size(); k0 += IQT_MAX) {
        tp.njobs = 0;
        tp.vec = aligned(c.ein) ? 1 : 0;
        for (size_t k = k0; k < c.taps.size() && k < k0 + IQT_MAX; k++) {
            const VfoSlot* v = fe->vfos[c.taps[k]].get();
            void* dst = c.kernel_out[c.taps[k]] ? c.out->vfo_out[c.taps[k]] : (void*)((char*)fe->tap_stage[c.slot].p + c.tap_off[k]);
            tp.job[tp.njobs++] = IqTapJob{ dst, v->tap_type, v->tap_scalar };
            tp.vec &= aligned(dst) ? 1 : 0;
        }
        cudaError_t e = launch_iq_tap(tp, fe->tap_stream);
        if (e != cudaSuccess) { return cuda_fail(e, "launch_iq_tap"); }
        fe->sch.launches++;
    }
    if (t_tap) { B200_CK(cudaEventRecord(t_tap, fe->tap_stream)); }
    B200_CK(cudaEventRecord(fe->ev_tap_done, fe->tap_stream));
    c.tap_forked = true;
    fe->tap_read_pre = fe->decim > 1 && !fe->dc_block && !fe->invert_iq;
    return 0;
}

// The spectrum branch (IQFrontEnd's Reshaper -> FFT): the frames of the effective stream, nz samples every nz + skip, on
// fft_stream.  It only reads the chunk, so it forks from the main stream at its first enqueue, runs beside the VFO branch
// and joins before the outputs.
static int fe_fft_chunk(b200_fe* fe, FeChunk& c) {
    if (!fe->fft_on) { fe->pos += (unsigned long long)c.ecount; return 0; }
    const int bps = bytes_per_sample(c.efmt);
    const unsigned long long pos = fe->pos, end = pos + (unsigned long long)c.ecount;
    const unsigned long long nz = (unsigned long long)fe->fft.nz, interval = nz + (unsigned long long)fe->skip;
    fe->fft.plan.in_scale = c.escale;
    float* const lines_base = c.direct ? c.out->fft_out : fe->lines.as<float>();
    cudaStream_t s = fe->fft_stream;
    cudaEvent_t t_fft = nullptr;
    auto fork = [&]() -> int {
        if (c.fft_forked) { return 0; }
        B200_CK(cudaEventRecord(fe->ev_fft_go, fe->sch.stream));
        B200_CK(cudaStreamWaitEvent(s, fe->ev_fft_go, 0));
        // the line buffer of the previous chunk may still be on its way out (tail stream)
        if (fe->lines_busy) { B200_CK(cudaStreamWaitEvent(s, fe->ev_lines_free, 0)); }
        trace_mark("fft start", s);
        t_fft = fe->sch.timer_begin(2, s);
        c.fft_forked = true;
        return 0;
    };
    int rc = 0;
    char* const frame = (char*)fe->frame.p;
    const bool pending = fe->fstart < pos;
    const bool same_fmt = fe->frame_fmt == c.efmt && (c.efmt == FMT_CF32 || fe->frame_scale == c.escale);
    if (pending && (!fe->fft_v || !same_fmt)) {
        // a frame begun in earlier chunks whose staged part this chunk cannot extend in place (other format or scale, or the
        // cf32 staging of fft_v 0): convert that part to cf32 through the work buffer, and carry the frame on in cf32
        if (fe->frame_fmt != FMT_CF32) {
            if ((rc = fork())) { return rc; }
            const int len = (int)(pos - fe->fstart);
            cudaError_t e = launch_convert_cf32(frame, fe->frame_fmt, fe->fft.work.as<float2>(), len, fe->frame_scale, s);
            if (e != cudaSuccess) { return cuda_fail(e, "launch_convert_cf32"); }
            fe->sch.launches++;
            B200_CK(cudaMemcpyAsync(frame, fe->fft.work.p, (size_t)len * sizeof(float2), cudaMemcpyDeviceToDevice, s));
            fe->frame_fmt = FMT_CF32;
            fe->frame_scale = 0.0f;
        }
        // 1) this chunk's part of the frame, converted behind the staged cf32 part; transformed alone if it completes here
        const unsigned long long fend = fe->fstart + nz;
        const unsigned long long lo = pos, hi = std::min(fend, end);
        if (hi > lo) {
            if ((rc = fork())) { return rc; }
            cudaError_t e = launch_convert_cf32(c.ein, c.efmt, fe->frame.as<float2>() + (size_t)(lo - fe->fstart), (int)(hi - lo), c.escale, s);
            if (e != cudaSuccess) { return cuda_fail(e, "launch_convert_cf32"); }
            fe->sch.launches++;
        }
        if (fend <= end) {
            if ((rc = fork())) { return rc; }
            int nl = 0;
            const FftFrames fr{ fe->frame.p, nullptr, 0, 0, 1 };
            cudaError_t e = launch_fft_frames(fe->fft.plan, fr, FMT_CF32, fe->fft.work.as<float2>(), lines_base, nullptr, fe->opts, s, &nl,
                                              fe->fft_v != 0);
            if (e != cudaSuccess) { return cuda_fail(e, "launch_fft_frames"); }
            fe->sch.launches += nl;
            c.nlines++;
            fe->fstart += interval;
        }
    }
    else if (pending && fe->fstart + nz > end) {
        // a frame that spans this whole chunk: append the chunk to its staged part
        if (c.ecount > 0) {
            if ((rc = fork())) { return rc; }
            B200_CK(cudaMemcpyAsync(frame + (size_t)(pos - fe->fstart) * bps, c.ein, (size_t)c.ecount * bps, cudaMemcpyDeviceToDevice, s));
        }
    }
    // 2) the frames that complete in this chunk, one batched launch pair.  With fft_v 1 the first may have begun in earlier
    // chunks: its first `split` samples come from the staged part, the rest straight from the chunk.
    const unsigned long long split = fe->fstart < pos ? pos - fe->fstart : 0;
    const int nb = fft_frames_by(fe, end);
    if (nb > 0) {
        if ((rc = fork())) { return rc; }
        const FftFrames fr{ (const char*)c.ein + (size_t)(fe->fstart + split - pos) * bps, frame, (long long)interval, (int)split, nb };
        int nl = 0;
        cudaError_t e = launch_fft_frames(fe->fft.plan, fr, c.efmt, fe->fft.work.as<float2>(), lines_base + (size_t)c.nlines * fe->fft.size,
                                          nullptr, fe->opts, s, &nl, fe->fft_v != 0);
        if (e != cudaSuccess) { return cuda_fail(e, "launch_fft_frames"); }
        fe->sch.launches += nl;
        c.nlines += nb;
        fe->fstart += interval * (unsigned long long)nb;
    }
    // 3) the head of a frame that continues into the next chunk
    if (fe->fstart < end && fe->fstart >= pos) {
        const unsigned long long lo = fe->fstart, hi = end;
        if ((rc = fork())) { return rc; }
        const char* src = (const char*)c.ein + (size_t)(lo - pos) * bps;
        if (fe->fft_v) {
            B200_CK(cudaMemcpyAsync(frame, src, (size_t)(hi - lo) * bps, cudaMemcpyDeviceToDevice, s));
            fe->frame_fmt = c.efmt;
            fe->frame_scale = c.escale;
        }
        else {
            cudaError_t e = launch_convert_cf32(src, c.efmt, fe->frame.as<float2>(), (int)(hi - lo), c.escale, s);
            if (e != cudaSuccess) { return cuda_fail(e, "launch_convert_cf32"); }
            fe->sch.launches++;
            fe->frame_fmt = FMT_CF32;
            fe->frame_scale = 0.0f;
        }
    }
    if (c.fft_forked) {
        if (t_fft) { B200_CK(cudaEventRecord(t_fft, s)); }
        trace_mark("fft done", s);
        B200_CK(cudaEventRecord(fe->ev_fft_done, s));
    }
    fe->pos = end;
    return 0;
}

// RDSDemod behind the WFM_RDS_BITS VFOs and bound RDS outputs: one launch per B200_BATCH of those with 5 kS/s samples this
// chunk, on the stream of the tails, behind them and in front of the next chunk's (which overwrite the chain outputs and
// move the RDS states)
static int fe_rds(b200_fe* fe, FeChunk& c) {
    fe->rds_pend[c.slot].clear();
    fe->rds_out[c.slot] = c.out;
    if (!fe->rds_count) { return 0; }        // allocated with the first RDS demodulator: a handle that never had one skips all this
    RdsParams rp;
    memset(&rp, 0, sizeof(rp));
    auto flush = [&]() -> int {
        cudaError_t e = launch_rds_demod(rp, fe->sch.out_stream());
        if (e != cudaSuccess) { return cuda_fail(e, "launch_rds_demod"); }
        fe->sch.launches += rp.njobs > 0 ? 1 : 0;
        rp.njobs = 0;
        return 0;
    };
    int rc;
    for (size_t k = 0; k < c.chains.size(); k++) {
        const int id = c.ids[k];
        VfoSlot* v = fe->vfos[id].get();
        if (!v->rds) { continue; }
        const int n = c.chains[k]->n_out, bound = b200_rds_demod_max_out(n);
        fe->rds_pend[c.slot].push_back({ id, n, bound });
        if (n == 0) { continue; }
        RdsSym* dst = c.kernel_out[id] ? (RdsSym*)c.out->vfo_out[id] : v->rds_rec.as<RdsSym>();
        rp.job[rp.njobs++] = v->rds->job(c.chains[k]->out.as<float2>(), n, dst, bound, fe->rds_count + c.slot * B200_MAX_VFOS + id);
        if (rp.njobs == B200_BATCH && (rc = flush())) { return rc; }
    }
    return flush();
}

// The join on a stream of its own: the VFO branch (tail stream), the spectrum branch and the IQ taps (their streams) of this
// chunk meet here, and none waits for another -- the tail stream goes straight on to the next chunk.  Then every output that
// no kernel wrote into the caller's buffer is copied there.
static int fe_join_and_copy_out(b200_fe* fe, FeChunk& c) {
    b200_outputs* out = c.out;
    cudaStream_t os = fe->join_stream;
    B200_CK(cudaEventRecord(fe->ev_tail_done[c.slot], fe->sch.out_stream()));
    B200_CK(cudaStreamWaitEvent(os, fe->ev_tail_done[c.slot], 0));
    if (c.fft_forked) { B200_CK(cudaStreamWaitEvent(os, fe->ev_fft_done, 0)); }
    if (c.tap_forked) { B200_CK(cudaStreamWaitEvent(os, fe->ev_tap_done, 0)); }
    // the input chunk is no longer needed once stage 1, the raw carry (both in front of the tail on its stream) and the
    // spectrum branch are done
    B200_CK(cudaEventRecord(fe->ev_compute[c.slot], os));
    fe->slot_used[c.slot] = true;
    const cudaMemcpyKind kind = c.direct ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    for (size_t k = 0; k < c.chains.size(); k++) {
        const Chain* ch = c.chains[k];
        const int id = c.ids[k];
        if (fe->vfos[id]->rds) {
            // the symbol count is known after the launch: every record the bound allows leaves, b200_fe_wait sets the count
            const int bound = b200_rds_demod_max_out(ch->n_out);
            if (ch->n_out > 0 && !c.kernel_out[id]) {
                B200_CK(cudaMemcpyAsync(out->vfo_out[id], fe->vfos[id]->rds_rec.p, (size_t)bound * sizeof(RdsSym), kind, os));
            }
            continue;
        }
        out->vfo_count[id] = ch->n_out;
        if (ch->n_out > 0 && !c.kernel_out[id]) {
            B200_CK(cudaMemcpyAsync(out->vfo_out[id], ch->out.p, (size_t)ch->n_out * ch->out_es * sizeof(float), kind, os));
        }
    }
    for (size_t k = 0; k < c.taps.size(); k++) {
        const int id = c.taps[k];
        out->vfo_count[id] = c.ecount;
        if (c.ecount > 0 && !c.kernel_out[id]) {
            B200_CK(cudaMemcpyAsync(out->vfo_out[id], (const char*)fe->tap_stage[c.slot].p + c.tap_off[k],
                                    (size_t)c.ecount * iq_tap_bytes(fe->vfos[id]->tap_type), kind, os));
        }
    }
    out->fft_lines = c.nlines;
    if (c.nlines > 0 && !c.direct) {
        B200_CK(cudaMemcpyAsync(out->fft_out, fe->lines.p, (size_t)c.nlines * fe->fft.size * sizeof(float), kind, os));
        B200_CK(cudaEventRecord(fe->ev_lines_free, os));
        fe->lines_busy = true;
    }
    B200_CK(cudaEventRecord(fe->ev_out[c.slot], os));
    trace_mark("outputs done", os);
    return 0;
}

// what b200_fe_submit and b200_shard_submit check of a chunk before anything else
static int check_chunk_args(const b200_fe* fe, int count, int in_fmt, const b200_outputs* out) {
    if (!out) { set_error("null argument"); return B200_EINVAL; }
    if (count < 0 || count > fe->max_chunk) { set_error("count %d exceeds max_chunk %d", count, fe->max_chunk); return B200_ECAP; }
    if (in_fmt < 0 || in_fmt > 2) { set_error("bad input format"); return B200_EINVAL; }
    return 0;
}

extern "C" int b200_fe_submit(b200_fe* fe, const void* iq, int count, int in_fmt, int in_mem, b200_outputs* out) {
    if (!fe || (count > 0 && !iq)) { set_error("null argument"); return B200_EINVAL; }
    int rc = check_chunk_args(fe, count, in_fmt, out);
    if (rc) { return rc; }
    if (fe->nsub - fe->nwait >= (unsigned long long)fe->max_inflight) { set_error("%d chunks already in flight: call b200_fe_wait", fe->max_inflight); return B200_ESTATE; }
    std::lock_guard<std::mutex> lck(fe->mtx);
    const long long hp0 = host_clock_ns();
    if ((rc = apply_pending(fe))) { return rc; }
    FeChunk c;
    c.slot = (int)(fe->nsub % FE_SLOTS);
    c.out = out;
    c.fmt = in_fmt; c.count = count;
    // 1/32768 and 1/128 unless the caller set the scale of a compressed-stream packet (b200_fe_set_ingest_scale)
    c.scale = in_fmt == B200_FMT_CS16 ? fe->scale16 : (in_fmt == B200_FMT_CS8 ? fe->scale8 : 0.0f);
    c.direct = out->out_mem == B200_MEM_DEVICE;
    fe_branches(fe, c);
    if ((rc = fe_check_outputs(fe, c)) || (rc = fe_upload(fe, c, iq, in_mem)) || (rc = fe_preprocess(fe, c))) { return rc; }
    fe_route_outputs(fe, c);
    if ((rc = fe_iq_taps(fe, c))) { return rc; }
    // the spectrum branch forks first; its join comes after the VFO branch has been enqueued, so the two overlap on the device
    const long long hp1 = host_clock_ns();
    if ((rc = fe_fft_chunk(fe, c))) { return rc; }
    const long long hp2 = host_clock_ns();
    fe->sch.in_scale = c.escale;
    // host-side outputs leave through per-VFO device buffers that the copies of the previous chunk may still be reading
    if (!c.direct && fe->nsub > 0) { B200_CK(cudaStreamWaitEvent(fe->sch.out_stream(), fe->ev_out[(c.slot + FE_SLOTS - 1) % FE_SLOTS], 0)); }
    if ((rc = fe->sch.run(c.chains, c.ein, c.efmt, c.ecount, true)) || (rc = fe_rds(fe, c))) { return rc; }
    const long long hp3 = host_clock_ns();
    if ((rc = fe_join_and_copy_out(fe, c))) { return rc; }
    fe->nsub++;
    const long long hp4 = host_clock_ns();
    fe->host_ns[0] += hp1 - hp0; fe->host_ns[1] += hp2 - hp1; fe->host_ns[2] += hp3 - hp2; fe->host_ns[3] += hp4 - hp3;
    return 0;
}

extern "C" int b200_fe_wait(b200_fe* fe) {
    if (!fe) { set_error("null fe"); return B200_EINVAL; }
    if (fe->nwait >= fe->nsub) { set_error("nothing in flight"); return B200_ESTATE; }
    const int slot = (int)(fe->nwait % FE_SLOTS);
    B200_CK(cudaEventSynchronize(fe->ev_out[slot]));
    fe->nwait++;
    if (trace_on() && fe->nwait == fe->nsub && fe->nsub >= 8) { trace_dump("chunks in flight drained"); }
    int rc = 0;
    for (const auto& p : fe->rds_pend[slot]) {
        const int n = p.n_in > 0 ? fe->rds_count[slot * B200_MAX_VFOS + p.id] : 0;
        if (n < 0 || n > p.bound) {
            set_error("VFO %d: RDS clock recovery produced %d symbols from %d samples (bound %d)", p.id, n, p.n_in, p.bound);
            rc = B200_ECAP;
            continue;
        }
        fe->rds_out[slot]->vfo_count[p.id] = n;
    }
    fe->rds_pend[slot].clear();
    return rc;
}

extern "C" int b200_fe_process(b200_fe* fe, const void* iq, int count, int in_fmt, int in_mem, b200_outputs* out) {
    if (fe && fe->nsub != fe->nwait) { set_error("chunks in flight: drain with b200_fe_wait first"); return B200_ESTATE; }
    int rc = b200_fe_submit(fe, iq, count, in_fmt, in_mem, out);
    if (rc) { return rc; }
    return b200_fe_wait(fe);
}

// ------------------------------------------------------------------ zoom / hold
extern "C" int b200_fft_zoom_hold(const float* line, int fft_size, int offset, int width, int out_size, float* out,
                                  float* hold, float hold_speed, int mem) {
    if (ensure_device()) { return B200_ENODEV; }
    if (!line || !out || fft_size < 1 || out_size < 1) { set_error("bad zoom args"); return B200_EINVAL; }
    // index loop of doZoom (waterfall.cpp:65-90), fp32 accumulator and all
    std::vector<int> start(out_size), len(out_size);
    if (offset < 0) { offset = 0; }
    if (width > 524288) { width = 524288; }
    float factor = (float)width / (float)out_size;
    float sFactor = ceilf(factor);
    float id = (float)offset;
    for (int i = 0; i < out_size; i++) {
        int sId = (int)id;
        float uFactor = (sId + sFactor > fft_size) ? sFactor - ((sId + sFactor) - fft_size) : sFactor;
        int l = 0;
        for (int j = 0; j < uFactor; j++) { l++; }
        start[i] = sId;
        len[i] = l;
        if (l > 0 && (sId < 0 || sId + l > fft_size)) { set_error("zoom window outside the line"); return B200_EINVAL; }
        id += factor;
    }
    DevBuf tbl, dline, dout, dhold;
    int rc;
    if ((rc = tbl.alloc((size_t)out_size * 2 * sizeof(int), false))) { return rc; }
    B200_CK(cudaMemcpy(tbl.p, start.data(), (size_t)out_size * sizeof(int), cudaMemcpyHostToDevice));
    B200_CK(cudaMemcpy(tbl.as<int>() + out_size, len.data(), (size_t)out_size * sizeof(int), cudaMemcpyHostToDevice));
    const float* l = line;
    float* o = out;
    float* h = hold;
    if (mem == B200_MEM_HOST) {
        if ((rc = dline.alloc((size_t)fft_size * sizeof(float), false))) { return rc; }
        if ((rc = dout.alloc((size_t)out_size * sizeof(float), false))) { return rc; }
        B200_CK(cudaMemcpy(dline.p, line, (size_t)fft_size * sizeof(float), cudaMemcpyHostToDevice));
        l = dline.as<float>();
        o = dout.as<float>();
        if (hold) {
            if ((rc = dhold.alloc((size_t)out_size * sizeof(float), false))) { return rc; }
            B200_CK(cudaMemcpy(dhold.p, hold, (size_t)out_size * sizeof(float), cudaMemcpyHostToDevice));
            h = dhold.as<float>();
        }
    }
    cudaError_t e = launch_zoom_hold_tbl(l, tbl.as<int>(), tbl.as<int>() + out_size, out_size, o, h, hold_speed, 0);
    if (e != cudaSuccess) { return cuda_fail(e, "launch_zoom_hold_tbl"); }
    if (mem == B200_MEM_HOST) {
        B200_CK(cudaMemcpy(out, o, (size_t)out_size * sizeof(float), cudaMemcpyDeviceToHost));
        if (hold) { B200_CK(cudaMemcpy(hold, h, (size_t)out_size * sizeof(float), cudaMemcpyDeviceToHost)); }
    }
    else { B200_CK(cudaDeviceSynchronize()); }
    return 0;
}

// ------------------------------------------------------------------ stand-alone blocks
struct b200_block {
    Chain chain;
    KernelOpts opts;      // the defaults: a block has no kernel options
    Scheduler sch{opts};
    cudaStream_t stream = nullptr;
    DevBuf in_dev;        // raw chains: the chunk as uploaded
    int in_es = 2;
    int max_chunk = 1000000;   // STREAM_BUFFER_SIZE (core/src/dsp/stream.h:9)
    // rxvfo bookkeeping for the setters
    double inSR = 0, outSR = 0, bw = 0;
    bool is_rxvfo = false, is_xlator = false;
    // setters may come from another thread than the worker running b200_block_process (b200dsp.h conventions): they only
    // stage a value under `mtx`; process() applies it at its next chunk boundary, like the reference's ctrlMtx
    std::mutex mtx;
    bool pend_off = false, pend_bw = false;
    double new_off_rad = 0, new_bw = 0;
    bool is_fir_c = false;
    std::vector<float> pend_taps;   // FIR::setTaps of a stand-alone complex-data filter
    bool is_nb = false, pend_nb = false;
    double new_nb_rate = 0, new_nb_level = 0;   // NoiseBlanker::setRate / setLevel: the running amplitude is kept
};

static b200_block* block_new() {
    if (ensure_device()) { return nullptr; }
    b200_block* b = new b200_block;
    if (cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking) != cudaSuccess) {
        cuda_fail(cudaGetLastError(), "cudaStreamCreate");
        delete b;
        return nullptr;
    }
    b->sch.stream = b->stream;
    return b;
}
static b200_block* block_finish(b200_block* b, int rc) {
    if (!rc) {
        b->in_es = b->chain.st[0]->in_es;
        rc = b->chain.finalize(b->max_chunk);
    }
    if (!rc && b->chain.raw_input()) {
        rc = b->sch.init_raw();
        if (!rc) { rc = b->in_dev.alloc((size_t)b->max_chunk * sizeof(float2), false); }
    }
    if (rc) { b200_block_destroy(b); return nullptr; }
    return b;
}

extern "C" void b200_block_destroy(b200_block* b) {
    if (!b) { return; }
    if (b->stream) { cudaStreamSynchronize(b->stream); cudaStreamDestroy(b->stream); }
    delete b;
}

extern "C" b200_block* b200_xlator_create(double offsetHz, double sr) {
    b200_block* b = block_new();
    if (!b) { return nullptr; }
    b->is_xlator = true;
    return block_finish(b, b->chain.add_xlator(offsetHz, sr));
}
extern "C" int b200_xlator_set_offset(b200_block* b, double offsetHz, double sr) {
    if (!b || !b->is_xlator) { set_error("not an xlator block"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(b->mtx);
    b->pend_off = true;
    b->new_off_rad = hz_to_rads(offsetHz, sr);
    return 0;
}
extern "C" b200_block* b200_decim_create(int ratio) {
    if (ratio < 1 || (ratio & (ratio - 1)) || ratio > 8192) { set_error("ratio must be a power of two <= 8192"); return nullptr; }
    b200_block* b = block_new();
    if (!b) { return nullptr; }
    return block_finish(b, b->chain.add_power_decim(ratio));
}
extern "C" b200_block* b200_resamp_create(double inSR, double outSR) {
    if (inSR <= 0 || outSR <= 0) { set_error("bad rates"); return nullptr; }
    b200_block* b = block_new();
    if (!b) { return nullptr; }
    return block_finish(b, b->chain.add_resampler(inSR, outSR));
}
extern "C" b200_block* b200_fir_cr_create(const float* taps, int n, int decim) {
    if (!taps || n < 1 || decim < 1) { set_error("bad taps"); return nullptr; }
    b200_block* b = block_new();
    if (!b) { return nullptr; }
    b->is_fir_c = true;
    return block_finish(b, b->chain.add_fir_c(std::vector<float>(taps, taps + n), decim));
}
extern "C" int b200_fir_cr_set_taps(b200_block* b, const float* taps, int n) {
    if (!b || !b->is_fir_c || !taps || n < 1) { set_error("not a complex-data FIR block / bad taps"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(b->mtx);
    b->pend_taps.assign(taps, taps + n);
    return 0;
}
extern "C" b200_block* b200_fir_rr_create(const float* taps, int n) {
    if (!taps || n < 1) { set_error("bad taps"); return nullptr; }
    b200_block* b = block_new();
    if (!b) { return nullptr; }
    return block_finish(b, b->chain.add_fir_r(std::vector<float>(taps, taps + n), false));
}
extern "C" b200_block* b200_rxvfo_create(double inSR, double outSR, double bw, double offset) {
    if (inSR <= 0 || outSR <= 0 || bw <= 0) { set_error("bad rates"); return nullptr; }
    b200_block* b = block_new();
    if (!b) { return nullptr; }
    b->is_rxvfo = true; b->inSR = inSR; b->outSR = outSR; b->bw = bw;
    return block_finish(b, b->chain.add_rxvfo(inSR, outSR, bw, offset));
}
extern "C" int b200_rxvfo_set_offset(b200_block* b, double offset) {
    if (!b || !b->is_rxvfo) { set_error("not an RxVFO block"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(b->mtx);
    b->pend_off = true;
    b->new_off_rad = hz_to_rads(-offset, b->inSR);
    return 0;
}
extern "C" int b200_rxvfo_set_bandwidth(b200_block* b, double bw) {
    if (!b || !b->is_rxvfo || bw <= 0) { set_error("not an RxVFO block / bad bandwidth"); return B200_EINVAL; }
    if (b->chain.chan_fir < 0) { set_error("no channel filter"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(b->mtx);
    b->pend_bw = true;
    b->new_bw = bw;
    return 0;
}
// staged setter values -> stages; called by the worker at the top of process()
static void block_apply_pending(b200_block* b) {
    if (b->pend_nb) {
        SeqStage* q = (SeqStage*)b->chain.st[0].get();
        q->proto.nb_rate = (float)b->new_nb_rate;
        q->proto.nb_inv_rate = 1.0f - q->proto.nb_rate;
        q->proto.nb_level = (float)b->new_nb_level;
        b->pend_nb = false;
    }
    std::lock_guard<std::mutex> lck(b->mtx);
    if (b->pend_off) {
        ((XdStage*)b->chain.st[0].get())->set_offset_rad(b->new_off_rad);
        b->pend_off = false;
    }
    if (!b->pend_taps.empty()) {
        ((FirCStage*)b->chain.st[0].get())->pending.swap(b->pend_taps);
        b->pend_taps.clear();
    }
    if (b->pend_bw) {
        FirCStage* f = (FirCStage*)b->chain.st[b->chain.chan_fir].get();
        const double fw = b->new_bw / 2.0;
        f->pending = (b->new_bw != b->outSR) ? lowpass_taps(fw, fw * 0.1, b->outSR) : std::vector<float>{ 1.0f };
        b->bw = b->new_bw;
        b->pend_bw = false;
    }
}
extern "C" b200_block* b200_quad_create(double dev, double sr) {
    b200_block* b = block_new();
    if (!b) { return nullptr; }
    return block_finish(b, b->chain.add_quad(dev, sr));
}
extern "C" b200_block* b200_wfm_create(double dev, double sr, int stereo, int lowPass) {
    b200_block* b = block_new();
    if (!b) { return nullptr; }
    return block_finish(b, b->chain.add_wfm(dev, sr, lowPass != 0, stereo != 0));
}
extern "C" b200_block* b200_wfm_rds_create(double dev, double sr) {
    b200_block* b = block_new();
    if (!b) { return nullptr; }
    return block_finish(b, b->chain.add_wfm_rds(dev, sr));
}
extern "C" b200_block* b200_nfm_create(double sr, double bw, int lowPass) {
    b200_block* b = block_new();
    if (!b) { return nullptr; }
    return block_finish(b, b->chain.add_nfm(sr, bw, lowPass != 0));
}
extern "C" b200_block* b200_am_create(int agcMode, double bw, double att, double dec, double dcr, double sr) {
    if (agcMode != 0 && agcMode != 1) { set_error("bad agcMode"); return nullptr; }
    b200_block* b = block_new();
    if (!b) { return nullptr; }
    return block_finish(b, b->chain.add_am(agcMode, bw, att, dec, dcr, sr));
}
extern "C" b200_block* b200_noise_blanker_create(double rate, double level) {
    b200_block* b = block_new();
    if (!b) { return nullptr; }
    b->is_nb = true;
    b->new_nb_rate = rate; b->new_nb_level = level;
    return block_finish(b, b->chain.add_noise_blanker(rate, level));
}
extern "C" int b200_noise_blanker_set(b200_block* b, double rate, double level) {
    if (!b || !b->is_nb) { set_error("not a noise blanker block"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(b->mtx);
    b->new_nb_rate = rate; b->new_nb_level = level;
    b->pend_nb = true;
    return 0;
}
extern "C" b200_block* b200_fmif_create(int bins) {
    b200_block* b = block_new();
    if (!b) { return nullptr; }
    return block_finish(b, b->chain.add_fmif(bins));
}
extern "C" b200_block* b200_squelch_create(double level) {
    b200_block* b = block_new();
    if (!b) { return nullptr; }
    return block_finish(b, b->chain.add_squelch(level));
}
extern "C" b200_block* b200_deemph_create(double tau, double sr) {
    if (tau <= 0 || sr <= 0) { set_error("bad deemphasis parameters"); return nullptr; }
    b200_block* b = block_new();
    if (!b) { return nullptr; }
    return block_finish(b, b->chain.add_deemph(tau, sr));
}
extern "C" b200_block* b200_ssb_create(int mode, double bw, double sr, double att, double dec) {
    if (mode < 0 || mode > 2) { set_error("bad SSB mode"); return nullptr; }
    b200_block* b = block_new();
    if (!b) { return nullptr; }
    return block_finish(b, b->chain.add_ssb(mode, bw, sr, att, dec));
}

extern "C" int b200_block_max_out(b200_block* b, int count) {
    if (!b) { set_error("null block"); return B200_EINVAL; }
    return b->chain.max_out(count);
}

extern "C" int b200_block_process(b200_block* b, int count, const void* in, void* out) {
    if (!b || (count > 0 && (!in || !out))) { set_error("null argument"); return B200_EINVAL; }
    if (count < 0 || count > b->max_chunk) { set_error("count %d exceeds the block's chunk limit %d", count, b->max_chunk); return B200_ECAP; }
    block_apply_pending(b);
    std::vector<Chain*> chains{ &b->chain };
    { int rcd = b->sch.apply_deferred(chains); if (rcd) { return rcd; } }     // may move stage buffers: before the input copy
    cudaStream_t s = b->stream;
    const bool raw = b->chain.raw_input();
    const size_t in_bytes = (size_t)count * b->in_es * sizeof(float);
    if (count > 0) {
        void* dst = raw ? b->in_dev.p : (void*)b->chain.st[0]->in_data();
        B200_CK(cudaMemcpyAsync(dst, in, in_bytes, cudaMemcpyHostToDevice, s));
    }
    b->chain.plan(count);
    int rc = b->sch.run(chains, raw ? b->in_dev.p : nullptr, FMT_CF32, count, raw);
    if (rc) { return rc; }
    if (b->chain.n_out > 0) {
        B200_CK(cudaMemcpyAsync(out, b->chain.out.p, (size_t)b->chain.n_out * b->chain.out_es * sizeof(float), cudaMemcpyDeviceToHost, s));
    }
    B200_CK(cudaStreamSynchronize(s));
    return b->chain.n_out;
}

extern "C" int b200_block_reset(b200_block* b) {
    if (!b) { set_error("null block"); return B200_EINVAL; }
    B200_CK(cudaStreamSynchronize(b->stream));
    b->chain.reset_state();
    return b->sch.reset_raw();
}

// ------------------------------------------------------------------ RDSDemod as a stand-alone block (RdsCore above)
// The clock recovery's output count depends on the data: it comes back with the symbols (one small copy + one synchronisation
// per call at 5 kS/s).  A front-end VFO in B200_DEMOD_WFM_RDS_BITS mode runs the same kernel without that synchronisation.
struct b200_rds_demod {
    cudaStream_t stream = nullptr;
    RdsCore core;
    DevBuf in, rec;
    int max_chunk = 1000000;     // STREAM_BUFFER_SIZE (core/src/dsp/stream.h:9)
    int out_cap = 0;
    RdsSym* hrec = nullptr;      // pinned staging of the symbols
    int* hcount = nullptr;       // pinned: the symbol count of the last launch, written by the kernel
    long long launches = 0;
    std::mutex mtx;              // process() and reset() may come from different threads (worker / control), like the other blocks
};
extern "C" int b200_rds_demod_max_out(int count) {
    if (count < 0) { return 0; }
    // the recovered clock stays within 1 % of 5000 / 1187.5 samples per symbol (MM's omegaRelLimit, rds_demod.h:32)
    const double omega_min = (5000.0 / (2375.0 / 2.0)) * (1.0 - 0.01);
    return (int)((double)count / omega_min) + 2;
}
extern "C" void b200_rds_demod_destroy(b200_rds_demod* r) {
    if (!r) { return; }
    if (r->stream) { cudaStreamSynchronize(r->stream); cudaStreamDestroy(r->stream); }
    if (r->hrec) { cudaFreeHost(r->hrec); }
    if (r->hcount) { cudaFreeHost(r->hcount); }
    delete r;
}
extern "C" b200_rds_demod* b200_rds_demod_create(void) {
    if (ensure_device()) { return nullptr; }
    b200_rds_demod* r = new b200_rds_demod;
    int rc = 0;
    if (cudaStreamCreateWithFlags(&r->stream, cudaStreamNonBlocking) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "cudaStreamCreate"); r->stream = nullptr; }
    r->out_cap = b200_rds_demod_max_out(r->max_chunk);
    if (!rc) { rc = r->in.alloc((size_t)r->max_chunk * sizeof(float2), false); }
    if (!rc) { rc = r->rec.alloc((size_t)r->out_cap * sizeof(RdsSym), false); }
    if (!rc && cudaMallocHost((void**)&r->hrec, (size_t)r->out_cap * sizeof(RdsSym)) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "cudaMallocHost"); }
    if (!rc && cudaMallocHost((void**)&r->hcount, sizeof(int)) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "cudaMallocHost"); }
    if (!rc) { rc = r->core.create(r->stream); }
    if (rc) { b200_rds_demod_destroy(r); return nullptr; }
    return r;
}
extern "C" int b200_rds_demod_process(b200_rds_demod* r, int count, const void* in, float* soft, uint8_t* hard) {
    if (!r || (count > 0 && (!in || !soft || !hard))) { set_error("null argument"); return B200_EINVAL; }
    if (count < 0 || count > r->max_chunk) { set_error("count %d exceeds the block's chunk limit %d", count, r->max_chunk); return B200_ECAP; }
    if (count == 0) { return 0; }
    std::lock_guard<std::mutex> lk(r->mtx);
    cudaStream_t s = r->stream;
    B200_CK(cudaMemcpyAsync(r->in.p, in, (size_t)count * sizeof(float2), cudaMemcpyDefault, s));      // host or device memory
    RdsParams p;
    memset(&p, 0, sizeof(p));
    const int bound = std::min(r->out_cap, b200_rds_demod_max_out(count));
    p.njobs = 1;
    p.job[0] = r->core.job(r->in.as<float2>(), count, r->rec.as<RdsSym>(), bound, r->hcount);
    cudaError_t e = launch_rds_demod(p, s);
    if (e != cudaSuccess) { return cuda_fail(e, "launch_rds_demod"); }
    r->launches++;
    B200_CK(cudaMemcpyAsync(r->hrec, r->rec.p, (size_t)bound * sizeof(RdsSym), cudaMemcpyDeviceToHost, s));
    B200_CK(cudaStreamSynchronize(s));
    const int n = *r->hcount;
    if (n < 0 || n > bound) { set_error("RDS clock recovery produced %d symbols from %d samples (bound %d)", n, count, bound); return B200_ECAP; }
    for (int i = 0; i < n; i++) {
        soft[i] = r->hrec[i].soft;
        hard[i] = (uint8_t)r->hrec[i].bit;
    }
    return n;
}
extern "C" int b200_rds_demod_reset(b200_rds_demod* r) {
    if (!r) { set_error("null block"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lk(r->mtx);
    B200_CK(cudaStreamSynchronize(r->stream));
    return r->core.reset(r->stream);
}
extern "C" long long b200_rds_demod_launch_count(b200_rds_demod* r) { return r ? r->launches : 0; }
/* test hooks: the two tap sets of the block as the host designs them */
extern "C" int b200_rds_demod_taps(float* bandpass, int cap_bp, float* bank) {
    const std::vector<float> bp = bandpass_c_taps(0.0, 2375.0, 100.0, 5000.0, false);
    const int nt = (int)bp.size() / 2;
    if (bandpass) { memcpy(bandpass, bp.data(), sizeof(float) * 2 * (size_t)std::min(nt, cap_bp)); }
    if (bank) {
        const std::vector<float> b = mm_interp_bank(RDS_MM_PHASES, RDS_MM_TAPS);
        memcpy(bank, b.data(), b.size() * sizeof(float));
    }
    return nt;
}

// ------------------------------------------------------------------ stand-alone spectrum handler
struct b200_fft {
    FftCore core;
    DevBuf in, db, raw;
};
extern "C" b200_fft* b200_fft_create(int size, int nz, int window) {
    if (ensure_device()) { return nullptr; }
    b200_fft* f = new b200_fft;
    int rc = f->core.create(size, nz, window);
    if (!rc) { rc = f->in.alloc((size_t)nz * sizeof(float2), false); }
    if (!rc) { rc = f->db.alloc((size_t)size * sizeof(float), false); }
    if (!rc) { rc = f->raw.alloc((size_t)size * sizeof(float2), false); }
    if (rc) { delete f; return nullptr; }
    return f;
}
static int fft_run(b200_fft* f, const float* iq, float* out_db, float* out_c) {
    if (!f || !iq) { set_error("null argument"); return B200_EINVAL; }
    B200_CK(cudaMemcpy(f->in.p, iq, (size_t)f->core.nz * sizeof(float2), cudaMemcpyHostToDevice));
    cudaError_t e = launch_fft_frame(f->core.plan, f->in.p, FMT_CF32, f->core.work.as<float2>(), f->db.as<float>(),
                                     f->raw.as<float2>(), KernelOpts(), 0, nullptr);
    if (e != cudaSuccess) { return cuda_fail(e, "launch_fft_frame"); }
    if (out_db) { B200_CK(cudaMemcpy(out_db, f->db.p, (size_t)f->core.size * sizeof(float), cudaMemcpyDeviceToHost)); }
    if (out_c) { B200_CK(cudaMemcpy(out_c, f->raw.p, (size_t)f->core.size * sizeof(float2), cudaMemcpyDeviceToHost)); }
    B200_CK(cudaDeviceSynchronize());
    return f->core.size;
}
extern "C" int b200_fft_frame(b200_fft* f, const float* iq, float* out_db) { return fft_run(f, iq, out_db, nullptr); }
extern "C" int b200_fft_raw(b200_fft* f, const float* iq, float* out_c) { return fft_run(f, iq, nullptr, out_c); }
extern "C" void b200_fft_destroy(b200_fft* f) {
    if (f) { cudaDeviceSynchronize(); delete f; }
}

// ------------------------------------------------------------------ pinned host memory
extern "C" void* b200_host_alloc(uint64_t bytes) {
    if (ensure_device()) { return nullptr; }
    void* p = nullptr;
    cudaError_t e = cudaMallocHost(&p, bytes ? bytes : 16);
    if (e != cudaSuccess) { cuda_fail(e, "cudaMallocHost"); return nullptr; }
    {
        std::lock_guard<std::mutex> lk(g_host_mtx);
        g_host_allocs[(uintptr_t)p] = (size_t)(bytes ? bytes : 16);
    }
    return p;
}
extern "C" void b200_host_free(void* p) {
    if (p) {
        {
            std::lock_guard<std::mutex> lk(g_host_mtx);
            g_host_allocs.erase((uintptr_t)p);
        }
        cudaFreeHost(p);
    }
}


// ------------------------------------------------------------------ data formats either side of the path
extern "C" int b200_fe_set_ingest_scale(b200_fe* fe, int fmt, float scale) {
    if (!fe) { set_error("null fe"); return B200_EINVAL; }
    std::lock_guard<std::mutex> lck(fe->mtx);
    if (fmt == B200_FMT_CS16) { fe->scale16 = scale > 0.0f ? scale : 1.0f / 32768.0f; return 0; }
    if (fmt == B200_FMT_CS8) { fe->scale8 = scale > 0.0f ? scale : 1.0f / 128.0f; return 0; }
    set_error("ingest scale applies to B200_FMT_CS16 / B200_FMT_CS8");
    return B200_EINVAL;
}

// SampleStreamDecompressor::process header (sample_stream_decompressor.h:15-33)
extern "C" int b200_pcm_packet_info(const void* packet, int bytes, int* fmt, float* scale, int* count, int* data_offset) {
    if (!packet || bytes < 8 || !fmt || !scale || !count || !data_offset) { set_error("bad packet"); return B200_EINVAL; }
    const unsigned char* b = (const unsigned char*)packet;
    unsigned short sampleType;
    float scaler;
    memcpy(&sampleType, b + 2, 2);
    memcpy(&scaler, b + 4, 4);
    *data_offset = 8;
    if (sampleType == 2) { *fmt = B200_FMT_CF32; *scale = 0.0f; *count = (bytes - 8) / 8; return 0; }          // PCM_TYPE_F32
    if (sampleType == 1) { *fmt = B200_FMT_CS16; *scale = 1.0f / (32768.0f / scaler); *count = (bytes - 8) / 4; return 0; }
    if (sampleType == 0) { *fmt = B200_FMT_CS8; *scale = 1.0f / (128.0f / scaler); *count = (bytes - 8) / 2; return 0; }
    set_error("unknown PCM sample type %d", (int)sampleType);
    return B200_EINVAL;
}

static int export_scalar(int type, float* scalar) {
    switch (type) {
    case B200_EXPORT_U8: *scalar = 0.0f; return EXP_U8;
    case B200_EXPORT_I16: *scalar = 32767.0f; return EXP_I16;            // wav.cpp:168
    case B200_EXPORT_I32: *scalar = 2147483647.0f; return EXP_I32;       // wav.cpp:172
    default: return -1;
    }
}
static size_t export_bytes(int t) { return t == EXP_I32 ? 4 : (t == EXP_I16 ? 2 : 1); }

// wav::Writer::write sample conversion (core/src/utils/wav.cpp:150-183) on the device
extern "C" int b200_export_convert(const float* in, long long n, int sample_type, void* out, int mem) {
    if (!in || !out || n < 0) { set_error("null argument"); return B200_EINVAL; }
    float scalar;
    const int t = export_scalar(sample_type, &scalar);
    if (t < 0) { set_error("bad sample type %d", sample_type); return B200_EINVAL; }
    if (n == 0) { return 0; }
    if (mem == B200_MEM_DEVICE) {
        cudaError_t e = launch_export(in, n, t, scalar, out, nullptr);
        if (e != cudaSuccess) { return cuda_fail(e, "launch_export"); }
        B200_CK(cudaStreamSynchronize(nullptr));
        return 0;
    }
    DevBuf di, dout;
    int rc;
    if ((rc = di.alloc((size_t)n * sizeof(float), false)) || (rc = dout.alloc((size_t)n * export_bytes(t), false))) { return rc; }
    B200_CK(cudaMemcpy(di.p, in, (size_t)n * sizeof(float), cudaMemcpyHostToDevice));
    cudaError_t e = launch_export(di.as<float>(), n, t, scalar, dout.p, nullptr);
    if (e != cudaSuccess) { return cuda_fail(e, "launch_export"); }
    B200_CK(cudaMemcpy(out, dout.p, (size_t)n * export_bytes(t), cudaMemcpyDeviceToHost));
    return 0;
}

// SampleStreamCompressor::process (sample_stream_compressor.h:30-66): 8-byte header + PCM payload
// per-thread scratch of the packet builder: grow-only device buffers and a stream of its own, so that building a packet neither
// allocates nor synchronises the device (the compressor adapter calls this once per chunk from its worker thread)
namespace {
struct PcmScratch {
    DevBuf in, out, mx;
    cudaStream_t stream = nullptr;
    ~PcmScratch() { if (stream) { cudaStreamDestroy(stream); } }
    int ensure(DevBuf& b, size_t bytes) {
        if (b.bytes >= bytes) { return 0; }
        return b.alloc(bytes + bytes / 4 + 64, false);
    }
};
}
extern "C" int b200_pcm_compress(const float* iq, int count, int pcm_fmt, void* packet, int cap_bytes, int mem) {
    if (!iq || !packet || count < 0) { set_error("null argument"); return B200_EINVAL; }
    if (ensure_device()) { return B200_ENODEV; }
    const int bps = pcm_fmt == B200_FMT_CF32 ? 8 : (pcm_fmt == B200_FMT_CS16 ? 4 : (pcm_fmt == B200_FMT_CS8 ? 2 : 0));
    if (!bps) { set_error("bad pcm format %d", pcm_fmt); return B200_EINVAL; }
    const long long bytes64 = 8 + (long long)count * bps;
    if (bytes64 > 2147483647LL) { set_error("packet of %d samples does not fit an int byte count", count); return B200_ECAP; }
    const int bytes = (int)bytes64;
    if (cap_bytes < bytes) { set_error("packet buffer too small"); return B200_ECAP; }
    const unsigned short sampleType = pcm_fmt == B200_FMT_CF32 ? 2 : (pcm_fmt == B200_FMT_CS16 ? 1 : 0);
    const bool dev = mem == B200_MEM_DEVICE;
    static thread_local PcmScratch sc;
    if (!sc.stream && cudaStreamCreateWithFlags(&sc.stream, cudaStreamNonBlocking) != cudaSuccess) { return cuda_fail(cudaGetLastError(), "cudaStreamCreate"); }
    cudaStream_t st = sc.stream;
    int rc;
    const float* src = iq;
    // device buffers: whatever the caller queued on the default stream is finished first (work on other streams is the
    // caller's to synchronise, as for any device pointer handed to the library)
    if (dev) { B200_CK(cudaStreamSynchronize(nullptr)); }
    if (!dev) {
        if ((rc = sc.ensure(sc.in, (size_t)count * 8 + 16))) { return rc; }
        B200_CK(cudaMemcpyAsync(sc.in.p, iq, (size_t)count * 8, cudaMemcpyHostToDevice, st));
        src = sc.in.as<float>();
        if ((rc = sc.ensure(sc.out, (size_t)bytes + 16))) { return rc; }
    }
    unsigned char hdr[8] = { 0 };
    memcpy(hdr + 2, &sampleType, 2);
    unsigned char* dst = (unsigned char*)packet;
    unsigned char* dpk = dev ? dst : sc.out.as<unsigned char>();
    if (pcm_fmt == B200_FMT_CF32) {
        B200_CK(cudaMemcpyAsync(dpk + 8, src, (size_t)count * 8, cudaMemcpyDeviceToDevice, st));
    }
    else {
        if ((rc = sc.ensure(sc.mx, 16))) { return rc; }
        float maxVal = 0.0f;
        if (count > 0) {
            B200_CK(cudaMemsetAsync(sc.mx.p, 0, 16, st));
            cudaError_t e = launch_index_max(src, (long long)count * 2, sc.mx.as<float>(), st);
            if (e != cudaSuccess) { return cuda_fail(e, "launch_index_max"); }
            B200_CK(cudaMemcpyAsync(&maxVal, sc.mx.p, sizeof(float), cudaMemcpyDeviceToHost, st));
            B200_CK(cudaStreamSynchronize(st));            // the scale of the packet depends on it
        }
        memcpy(hdr + 4, &maxVal, 4);
        const float scalar = (pcm_fmt == B200_FMT_CS16 ? 32768.0f : 128.0f) / maxVal;
        cudaError_t e = launch_export(src, (long long)count * 2, pcm_fmt == B200_FMT_CS16 ? EXP_I16 : EXP_I8, scalar, dpk + 8, st);
        if (e != cudaSuccess) { return cuda_fail(e, "launch_export"); }
    }
    B200_CK(cudaMemcpyAsync(dpk, hdr, 8, cudaMemcpyHostToDevice, st));
    if (!dev) { B200_CK(cudaMemcpyAsync(dst, dpk, (size_t)bytes, cudaMemcpyDeviceToHost, st)); }
    B200_CK(cudaStreamSynchronize(st));
    return bytes;
}

// ------------------------------------------------------------------ one stream, VFO groups on several GPUs (BASELINE config 4)
// The path has no exchange step (SURVEY.md section 8e): every VFO consumes the same raw IQ -- the reference's Splitter
// memcpy fan-out (core/src/dsp/routing/splitter.h:46-61).  Across GPUs the fan-out is one ncclBroadcast of each raw chunk
// from the ingest rank, on a communication stream, one chunk ahead of the compute (two chunk buffers per rank).
// NCCL is bound at run time (dlopen "libnccl.so.2": the process's own copy when a framework already loaded one).
#include <dlfcn.h>
namespace {
struct NcclId { char internal[128]; };
typedef void* NcclComm;
struct NcclApi {
    int (*GetUniqueId)(NcclId*) = nullptr;
    int (*CommInitRank)(NcclComm*, int, NcclId, int) = nullptr;
    int (*CommDestroy)(NcclComm) = nullptr;
    int (*Broadcast)(const void*, void*, size_t, int, int, NcclComm, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool ok = false;
};
NcclApi& nccl() {
    static NcclApi a;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_LOCAL);
        if (!h) { h = dlopen("libnccl.so", RTLD_NOW | RTLD_LOCAL); }
        if (h) {
            a.GetUniqueId = (int (*)(NcclId*))dlsym(h, "ncclGetUniqueId");
            a.CommInitRank = (int (*)(NcclComm*, int, NcclId, int))dlsym(h, "ncclCommInitRank");
            a.CommDestroy = (int (*)(NcclComm))dlsym(h, "ncclCommDestroy");
            a.Broadcast = (int (*)(const void*, void*, size_t, int, int, NcclComm, cudaStream_t))dlsym(h, "ncclBroadcast");
            a.GetErrorString = (const char* (*)(int))dlsym(h, "ncclGetErrorString");
            a.ok = a.GetUniqueId && a.CommInitRank && a.CommDestroy && a.Broadcast;
        }
    }
    return a;
}
int nccl_fail(int r, const char* what) {
    set_error("NCCL error %d (%s) in %s", r, nccl().GetErrorString ? nccl().GetErrorString(r) : "?", what);
    return B200_ECUDA;
}
}

struct b200_shard {
    b200_fe* fe = nullptr;
    int rank = 0, world = 1;
    NcclComm comm = nullptr;
    cudaStream_t comm_stream = nullptr;
    DevBuf buf[FE_SLOTS];                // the raw chunk on this rank (root: staged host input or the caller's device chunk)
    cudaEvent_t ev_bcast[FE_SLOTS] = {}, ev_src[FE_SLOTS] = {};
    unsigned long long nsub = 0;
    long long bytes_broadcast = 0;
};

extern "C" int b200_shard_unique_id(void* id128) {
    if (!id128) { set_error("null id"); return B200_EINVAL; }
    if (!nccl().ok) { set_error("libnccl.so.2 not found: the sharded front end needs NCCL"); return B200_ENODEV; }
    NcclId id;
    int r = nccl().GetUniqueId(&id);
    if (r) { return nccl_fail(r, "ncclGetUniqueId"); }
    memcpy(id128, &id, sizeof(id));
    return 0;
}

extern "C" void b200_shard_destroy(b200_shard* sh) {
    if (!sh) { return; }
    cudaDeviceSynchronize();
    if (sh->comm) { nccl().CommDestroy(sh->comm); }
    for (int i = 0; i < FE_SLOTS; i++) {
        if (sh->ev_bcast[i]) { cudaEventDestroy(sh->ev_bcast[i]); }
        if (sh->ev_src[i]) { cudaEventDestroy(sh->ev_src[i]); }
    }
    if (sh->comm_stream) { cudaStreamDestroy(sh->comm_stream); }
    delete sh;
}

extern "C" b200_shard* b200_shard_create(b200_fe* fe, int rank, int world, const void* id128) {
    if (!fe || !id128 || world < 1 || rank < 0 || rank >= world) { set_error("bad shard arguments"); return nullptr; }
    if (!nccl().ok) { set_error("libnccl.so.2 not found: the sharded front end needs NCCL"); return nullptr; }
    b200_shard* sh = new b200_shard;
    sh->fe = fe; sh->rank = rank; sh->world = world;
    bool ok = cudaStreamCreateWithFlags(&sh->comm_stream, cudaStreamNonBlocking) == cudaSuccess;
    for (int i = 0; i < FE_SLOTS && ok; i++) {
        ok = cudaEventCreateWithFlags(&sh->ev_bcast[i], cudaEventDisableTiming) == cudaSuccess &&
             cudaEventCreateWithFlags(&sh->ev_src[i], cudaEventDisableTiming) == cudaSuccess;
    }
    if (!ok) { cuda_fail(cudaGetLastError(), "shard stream/event creation"); b200_shard_destroy(sh); return nullptr; }
    NcclId id;
    memcpy(&id, id128, sizeof(id));
    int r = nccl().CommInitRank(&sh->comm, world, id, rank);
    if (r) { nccl_fail(r, "ncclCommInitRank"); sh->comm = nullptr; b200_shard_destroy(sh); return nullptr; }
    return sh;
}

// Every rank calls submit with the same count and format; `iq` is read on rank 0 only.  Values and counts per VFO are
// those of b200_fe_submit on the rank that owns the VFO.
extern "C" int b200_shard_submit(b200_shard* sh, const void* iq, int count, int in_fmt, int in_mem, b200_outputs* out) {
    if (!sh) { set_error("null argument"); return B200_EINVAL; }
    b200_fe* fe = sh->fe;
    int rc = check_chunk_args(fe, count, in_fmt, out);
    if (rc) { return rc; }
    if (sh->rank == 0 && count > 0 && !iq) { set_error("rank 0 needs the chunk"); return B200_EINVAL; }
    if (fe->nsub - fe->nwait >= 2) { set_error("two chunks already in flight: call b200_shard_wait"); return B200_ESTATE; }
    if (sh->world == 1) {                                   // nothing to fan out: the plain front end
        if (!(rc = b200_fe_submit(fe, iq, count, in_fmt, in_mem, out))) { sh->nsub++; }
        return rc;
    }
    const int slot = (int)(fe->nsub % FE_SLOTS);            // the front end's own input slot of this chunk
    const size_t bytes = (size_t)count * bytes_per_sample(in_fmt);
    cudaStream_t cs = sh->comm_stream, ms = fe->sch.stream;
    if (sh->buf[slot].bytes < bytes) {
        B200_CK(cudaDeviceSynchronize());
        if ((rc = sh->buf[slot].alloc(std::max(bytes, (size_t)fe->max_chunk * bytes_per_sample(in_fmt)), false))) { return rc; }
    }
    // buf[slot] was the input of the chunk two submissions ago: its compute has to be over before it is overwritten
    if (fe->slot_used[slot]) { B200_CK(cudaStreamWaitEvent(cs, fe->ev_compute[slot], 0)); }
    if (count > 0) {
        if (sh->rank == 0) {
            if (in_mem == B200_MEM_HOST) {
                B200_CK(cudaMemcpyAsync(sh->buf[slot].p, iq, bytes, cudaMemcpyHostToDevice, cs));
            }
            else {
                // the caller's device chunk is valid on the stream it submits on
                B200_CK(cudaEventRecord(sh->ev_src[slot], ms));
                B200_CK(cudaStreamWaitEvent(cs, sh->ev_src[slot], 0));
                B200_CK(cudaMemcpyAsync(sh->buf[slot].p, iq, bytes, cudaMemcpyDeviceToDevice, cs));
            }
        }
        int r = nccl().Broadcast(sh->buf[slot].p, sh->buf[slot].p, bytes, 1 /* ncclUint8 */, 0, sh->comm, cs);
        if (r) { return nccl_fail(r, "ncclBroadcast"); }
        sh->bytes_broadcast += (long long)bytes;
    }
    B200_CK(cudaEventRecord(sh->ev_bcast[slot], cs));
    B200_CK(cudaStreamWaitEvent(ms, sh->ev_bcast[slot], 0));
    if ((rc = b200_fe_submit(fe, sh->buf[slot].p, count, in_fmt, B200_MEM_DEVICE, out))) { return rc; }
    sh->nsub++;
    return 0;
}
extern "C" int b200_shard_wait(b200_shard* sh) {
    if (!sh) { set_error("null shard"); return B200_EINVAL; }
    return b200_fe_wait(sh->fe);
}
extern "C" long long b200_shard_bytes_broadcast(b200_shard* sh) { return sh ? sh->bytes_broadcast : 0; }


// ------------------------------------------------------------------ BASELINE config 3: polyphase filter-bank channelizer
struct b200_chan {
    int M = 256, P = 127, max_chunk = 0;
    cudaStream_t stream = nullptr;
    DevBuf inbuf, u, y, h, tw;
    std::vector<float> proto;
    long long launches = 0;
};
extern "C" void b200_chan_destroy(b200_chan* c) {
    if (!c) { return; }
    if (c->stream) { cudaStreamSynchronize(c->stream); cudaStreamDestroy(c->stream); }
    delete c;
}
extern "C" b200_chan* b200_chan_create(int channels, int taps_per_branch, int max_chunk) {
    if (ensure_device()) { return nullptr; }
    if (channels != 256 || taps_per_branch < 1 || taps_per_branch > 255 || max_chunk < channels || (max_chunk % channels)) {
        set_error("channelizer: 256 channels, 1..255 taps per branch, max_chunk a multiple of 256");
        return nullptr;
    }
    b200_chan* c = new b200_chan;
    c->M = channels; c->P = taps_per_branch; c->max_chunk = max_chunk;
    const int M = c->M, P = c->P, T = M * P;
    // prototype: taps::windowedSinc<float>(T, cutoff = fs / (2 M), fs, nuttall)  ->  omega = 2 pi / (2 M)
    c->proto = windowed_sinc_taps(T, 3.14159265358979323846 / (double)M);
    std::vector<float> hr((size_t)T);
    for (int pI = 0; pI < P; pI++) {
        for (int r = 0; r < M; r++) { hr[((size_t)(r >> 5) * P + pI) * 32 + (r & 31)] = c->proto[(size_t)pI * M + r]; }
    }
    std::vector<float2> tw((size_t)M);
    for (int k = 0; k < M; k++) {
        const double a = -2.0 * 3.14159265358979323846 * (double)k / (double)M;
        tw[k] = make_float2((float)std::cos(a), (float)std::sin(a));
    }
    const size_t hist = (size_t)(P - 1) * M;
    int rc = 0;
    if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) { cuda_fail(cudaGetLastError(), "cudaStreamCreate"); rc = B200_ECUDA; }
    if (!rc) { rc = c->inbuf.alloc((hist + (size_t)max_chunk + 64) * sizeof(float2)); }
    if (!rc) { rc = c->u.alloc((size_t)max_chunk * sizeof(float2), false); }
    if (!rc) { rc = c->y.alloc((size_t)max_chunk * sizeof(float2), false); }
    if (!rc) { rc = c->h.alloc(hr.size() * sizeof(float), false); }
    if (!rc) { rc = c->tw.alloc(tw.size() * sizeof(float2), false); }
    if (!rc && (cudaMemcpy(c->h.p, hr.data(), hr.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess ||
                cudaMemcpy(c->tw.p, tw.data(), tw.size() * sizeof(float2), cudaMemcpyHostToDevice) != cudaSuccess ||
                cudaDeviceSynchronize() != cudaSuccess)) { cuda_fail(cudaGetLastError(), "channelizer tables"); rc = B200_ECUDA; }
    if (rc) { b200_chan_destroy(c); return nullptr; }
    return c;
}
extern "C" int b200_chan_prototype(b200_chan* c, float* out, int cap) {
    if (!c) { set_error("null channelizer"); return B200_EINVAL; }
    if (out) { memcpy(out, c->proto.data(), sizeof(float) * (size_t)std::min<int>((int)c->proto.size(), cap)); }
    return (int)c->proto.size();
}
// count: complex input samples, a multiple of the channel count; out: [count / M][M] complex (channel k of output time m at
// out[m * M + k]).  in_mem / out_mem: B200_MEM_*.  Returns the number of output times (count / M).
extern "C" int b200_chan_process(b200_chan* c, const void* iq, int count, int in_mem, void* out, int out_mem) {
    if (!c || (count > 0 && (!iq || !out))) { set_error("null argument"); return B200_EINVAL; }
    if (count < 0 || count > c->max_chunk || (count % c->M)) { set_error("channelizer: count must be a multiple of %d, at most %d", c->M, c->max_chunk); return B200_ECAP; }
    if (count == 0) { return 0; }
    const int M = c->M, P = c->P, n_out = count / M;
    const size_t hist = (size_t)(P - 1) * M;
    cudaStream_t s = c->stream;
    float2* data = c->inbuf.as<float2>() + hist;
    B200_CK(cudaMemcpyAsync(data, iq, (size_t)count * sizeof(float2), in_mem == B200_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s));
    ChanParams p;
    p.in = c->inbuf.as<float2>(); p.u = c->u.as<float2>(); p.h = c->h.as<float>(); p.M = M; p.P = P; p.n_out = n_out;
    float2* y = (out_mem == B200_MEM_DEVICE) ? (float2*)out : c->y.as<float2>();
    int nl = 0;
    cudaError_t e = launch_channelizer(p, y, c->tw.as<float2>(), s, &nl);
    if (e != cudaSuccess) { return cuda_fail(e, "launch_channelizer"); }
    // history for the next chunk: the last (P - 1) M samples of [hist | chunk] (memmove semantics: alias-safe kernel)
    if ((size_t)count >= hist) {
        // the tail of the chunk does not overlap the history slot: a plain device copy
        B200_CK(cudaMemcpyAsync(c->inbuf.p, c->inbuf.as<float2>() + count, hist * sizeof(float2), cudaMemcpyDeviceToDevice, s));
    }
    else {
        CarryParams cp;
        cp.njobs = 1;
        CarryJob& j = cp.job[0];
        j.dst = c->inbuf.as<float>(); j.a = c->inbuf.as<float>(); j.b = data;
        j.h = (int)hist; j.la = (int)hist; j.lb = count; j.esize = 2; j.bfmt = -1; j.scale = 0.0f;
        e = launch_carry(cp, KernelOpts(), s);
        if (e != cudaSuccess) { return cuda_fail(e, "launch_carry"); }
        nl++;
    }
    c->launches += nl;
    if (out_mem != B200_MEM_DEVICE) { B200_CK(cudaMemcpyAsync(out, c->y.p, (size_t)count * sizeof(float2), cudaMemcpyDeviceToHost, s)); }
    B200_CK(cudaStreamSynchronize(s));
    return n_out;
}
extern "C" long long b200_chan_launch_count(b200_chan* c) { return c ? c->launches : 0; }

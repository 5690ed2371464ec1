// sdrplusplus_b200/csrc/engine.cpp -- see engine.h
#include "engine.h"
#include <chrono>
#include "../../include/b200dsp.h"
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <map>
#include <functional>
#include <cstdlib>

namespace b200 {

// ------------------------------------------------------------------ errors
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
const char* last_error() { return g_err; }
int cuda_fail(cudaError_t e, const char* what) {
    set_error("CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
    if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) { return B200_ENODEV; }
    return B200_ECUDA;
}

// ------------------------------------------------------------------ trace
struct TraceRec { const char* label; cudaEvent_t ev; };
static std::vector<TraceRec> g_trace;
static int g_trace_on = -1;
bool trace_on() {
    if (g_trace_on < 0) { const char* e = getenv("B200_TRACE"); g_trace_on = (e && *e && *e != '0') ? 1 : 0; }
    return g_trace_on == 1;
}
void trace_mark(const char* label, cudaStream_t s) {
    if (!trace_on()) { return; }
    cudaEvent_t e;
    if (cudaEventCreate(&e) != cudaSuccess) { return; }
    cudaEventRecord(e, s);
    g_trace.push_back({ label, e });
}
void trace_dump(const char* title) {
    if (!trace_on() || g_trace.empty()) { return; }
    cudaDeviceSynchronize();
    fprintf(stderr, "[b200 trace] %s\n", title);
    for (size_t i = 0; i < g_trace.size(); i++) {
        float ms = 0.0f;
        cudaEventElapsedTime(&ms, g_trace[0].ev, g_trace[i].ev);
        fprintf(stderr, "[b200 trace]   %9.1f us  %s\n", ms * 1e3, g_trace[i].label);
    }
    for (auto& r : g_trace) { cudaEventDestroy(r.ev); }
    g_trace.clear();
}

// ------------------------------------------------------------------ DevBuf
int DevBuf::alloc(size_t n, bool zero) {
    release();
    if (n == 0) { n = 16; }
    cudaError_t e = cudaMalloc(&p, n);
    if (e != cudaSuccess) { p = nullptr; return cuda_fail(e, "cudaMalloc"); }
    bytes = n;
    if (zero) {
        // cudaMemset is asynchronous on the legacy default stream, which the library's non-blocking streams do not
        // wait for: without the synchronisation a later cudaMemcpyAsync / kernel on those streams can be overtaken by
        // the zero fill (seen as an intermittent all-zero tap table)
        e = cudaMemset(p, 0, n);
        if (e == cudaSuccess) { e = cudaDeviceSynchronize(); }
        if (e != cudaSuccess) { return cuda_fail(e, "cudaMemset"); }
    }
    return 0;
}
void DevBuf::release() {
    if (p) { cudaFree(p); }
    p = nullptr;
    bytes = 0;
}

int Stage::alloc_in(int cap) {
    cap_in = cap;
    const size_t bytes = ((size_t)hist + (size_t)cap + Scheduler::STAGE_SPARE) * in_es * sizeof(float);
    int rc = inbuf.alloc(bytes);
    if (!rc && dbl) { rc = inbuf_alt.alloc(bytes); }
    return rc;
}

// t = `sets` tap sets of equal length T laid end to end; each set becomes D rows of pitch ceil(T/D), row r = t[q*D + r]
int Stage::upload_pm(const std::vector<float>& t, int D, int sets) {
    const int T = (int)(t.size() / (size_t)sets);
    const int qp = (T + D - 1) / D;
    pm_floats = (sets * D * qp + 3) & ~3;
    std::vector<float> pm((size_t)pm_floats, 0.0f);
    for (int s = 0; s < sets; s++) {
        for (int k = 0; k < T; k++) { pm[((size_t)s * D + (k % D)) * qp + k / D] = t[(size_t)s * T + k]; }
    }
    int rc = taps_pm.alloc(pm.size() * sizeof(float));
    if (rc) { return rc; }
    B200_CK(cudaMemcpy(taps_pm.p, pm.data(), pm.size() * sizeof(float), cudaMemcpyHostToDevice));
    return 0;
}

// ------------------------------------------------------------------ XdStage
void XdStage::configure(int D_, const std::vector<float>& taps) {
    D = D_;
    h = taps;
    T = (int)taps.size();
    QP = (T + D - 1 + D - 1) / D;                 // blocks of D covering the taps shifted by up to D-1
    gpad_len = (D - 1) + (QP + 8) * D;            // room for the launcher's QC in {4,6,8} round-up
    hist = T - 1;
    taps_dirty = true;
}

static const long double kTwoPiL = 6.283185307179586476925286766559L;

// The reference rotates by phaseDelta = ((float)cos(w), (float)sin(w)) (frequency_xlator.h:17,28): the
// angle actually applied per sample is the angle of that fp32-rounded phasor, not w itself.
static long double effective_omega(double rad) {
    float dre = (float)std::cos(rad), dim = (float)std::sin(rad);
    return atan2l((long double)dim, (long double)dre);
}

void XdStage::set_offset_rad(double rad) {
    offset_rad = rad;
    long double turns = effective_omega(rad) / kTwoPiL;           // (-0.5, 0.5]
    long double scaled = turns * 18446744073709551616.0L;         // * 2^64
    if (scaled >= 9223372036854775807.0L) { scaled = 9223372036854775807.0L; }
    if (scaled <= -9223372036854775807.0L) { scaled = -9223372036854775807.0L; }
    w = (unsigned long long)(long long)llroundl(scaled);
    // a retune after samples were translated with the current increment starts a segment; before that it replaces it
    if (segs.empty() || segs.back().start < pos) { segs.push_back(Seg{ pos, phase, w }); }
    else { segs.back().w = w; }
    taps_dirty = true;
}

void RxlStage::set_offset_rad(double rad) {
    long double turns = effective_omega(rad) / kTwoPiL;
    long double scaled = turns * 18446744073709551616.0L;
    if (scaled >= 9223372036854775807.0L) { scaled = 9223372036854775807.0L; }
    if (scaled <= -9223372036854775807.0L) { scaled = -9223372036854775807.0L; }
    w = (unsigned long long)(long long)llroundl(scaled);
}

int XdStage::upload_taps(cudaStream_t s) {
    if (!gpad.p || gpad.bytes < (size_t)gpad_len * sizeof(float2)) {
        int rc = gpad.alloc((size_t)gpad_len * sizeof(float2));
        if (rc) { return rc; }
    }
    std::vector<float2> g((size_t)gpad_len, make_float2(0.0f, 0.0f));
    const long double om = effective_omega(offset_rad);
    for (int k = 0; k < T; k++) {
        long double a = om * (long double)k;
        g[(size_t)(D - 1) + k] = make_float2((float)((long double)h[k] * cosl(a)), (float)((long double)h[k] * sinl(a)));
    }
    B200_CK(cudaMemcpyAsync(gpad.p, g.data(), g.size() * sizeof(float2), cudaMemcpyHostToDevice, s));
    if (!hdev.p) {
        int rc = hdev.alloc((size_t)T * sizeof(float));
        if (rc) { return rc; }
        B200_CK(cudaMemcpyAsync(hdev.p, h.data(), (size_t)T * sizeof(float), cudaMemcpyHostToDevice, s));
    }
    taps_dirty = false;
    return 0;
}

int XdStage::plan(int n) {
    n_in = n;
    chunk_offset = offset;
    chunk_phase0 = phase;
    n_out = (offset < n) ? (n - offset + D - 1) / D : 0;
    if (segs.empty()) { segs.push_back(Seg{ pos, phase, w }); }
    // Every stage-1 build rotates the history with the current increment.  The outputs whose window starts before the
    // newest boundary are recomputed by the edge kernel, which takes the history's phases from edge_tab.
    // (the first segment is the stream start, not a boundary: before it lie no samples translated with another increment)
    const long long b = segs.back().start - pos;                     // newest boundary, chunk-relative, <= 0
    chunk_retuned = segs.size() > 1 && n_out > 0 && b > (long long)offset - (T - 1);
    if (chunk_retuned) {
        chunk_edge_start = (int)b;
        edge_tab.resize((size_t)(T - 1));
        size_t s = 0;
        for (int j = 0; j < T - 1; j++) {
            const long long a = pos + j - (T - 1);                   // absolute index of history sample j - (T-1)
            while (s + 1 < segs.size() && segs[s + 1].start <= a) { s++; }
            edge_tab[(size_t)j] = segs[s].phase + segs[s].w * (unsigned long long)(a - segs[s].start);
        }
    }
    offset = offset + n_out * D - n;
    phase += w * (unsigned long long)(long long)n;
    pos += n;
    size_t drop = 0;
    while (drop + 1 < segs.size() && segs[drop + 1].start <= pos - (T - 1)) { drop++; }
    if (drop) { segs.erase(segs.begin(), segs.begin() + (long)drop); }
    return n_out;
}

// ------------------------------------------------------------------ FirCStage
int FirCStage::configure(const std::vector<float>& t, int decim_) {
    ntaps = (int)t.size();
    decim = decim_;
    hist = ntaps - 1;
    htaps = t;
    int rc = taps.alloc((size_t)ntaps * sizeof(float));
    if (rc) { return rc; }
    B200_CK(cudaMemcpy(taps.p, t.data(), (size_t)ntaps * sizeof(float), cudaMemcpyHostToDevice));
    return upload_pm(t, decim, 1);
}
int FirCStage::plan(int n) {
    prev_n_in = n_in;
    n_in = n;
    chunk_offset = offset;
    n_out = (offset < n) ? (n - offset + decim - 1) / decim : 0;
    offset = offset + n_out * decim - n;
    return n_out;
}

// ------------------------------------------------------------------ PolyStage
int PolyStage::configure(int interp_, int decim_, const std::vector<float>& t) {
    interp = interp_;
    decim = decim_;
    std::vector<float> b = build_polyphase_bank(interp, t, tpp);
    hist = tpp - 1;
    int rc = bank.alloc(b.size() * sizeof(float));
    if (rc) { return rc; }
    B200_CK(cudaMemcpy(bank.p, b.data(), b.size() * sizeof(float), cudaMemcpyHostToDevice));
    {
        std::vector<float> kl(((size_t)tpp * interp + 3) & ~(size_t)3, 0.0f);
        for (int ph = 0; ph < interp; ph++) {
            for (int k = 0; k < tpp; k++) { kl[(size_t)k * interp + ph] = b[(size_t)ph * tpp + k]; }
        }
        if ((rc = bank_kl.alloc(kl.size() * sizeof(float)))) { return rc; }
        B200_CK(cudaMemcpy(bank_kl.p, kl.data(), kl.size() * sizeof(float), cudaMemcpyHostToDevice));
    }
    return upload_pm(b, decim, interp);
}
int PolyStage::plan(int n) {
    n_in = n;
    chunk_phase = phase;
    chunk_offset = offset;
    long long avail = ((long long)n - offset) * interp - phase;
    long long no = avail > 0 ? (avail + decim - 1) / decim : 0;
    n_out = (int)no;
    long long tend = (long long)phase + no * decim;
    offset = (int)((long long)offset + tend / interp - n);
    phase = (int)(tend % interp);
    return n_out;
}

// ------------------------------------------------------------------ QuadStage
int QuadStage::configure(double deviationHz, double samplerate) {
    inv_dev = (float)(1.0 / hz_to_rads(deviationHz, samplerate));    // quadrature.h:19-26
    return 0;
}

// ------------------------------------------------------------------ FirRStage
int FirRStage::configure(const std::vector<float>& t, bool stereo_) {
    ntaps = (int)t.size();
    stereo = stereo_ ? 1 : 0;
    out_es = stereo ? 2 : 1;
    hist = ntaps - 1;
    int rc = taps.alloc((size_t)ntaps * sizeof(float));
    if (rc) { return rc; }
    B200_CK(cudaMemcpy(taps.p, t.data(), (size_t)ntaps * sizeof(float), cudaMemcpyHostToDevice));
    return upload_pm(t, 1, 1);
}

// ------------------------------------------------------------------ StereoStage
int StereoStage::configure(double samplerate) {
    std::vector<float> t = bandpass_c_taps(18750.0, 19250.0, 3000.0, samplerate, true);     // broadcast_fm.h:44
    ntaps = (int)(t.size() / 2);
    hist = ntaps - 1;
    delay = ((ntaps - 1) / 2) + 1;                                                           // broadcast_fm.h:48-49
    pll_coefficients(25000.0 / samplerate, alpha, beta);                                     // broadcast_fm.h:47, pll.h:17-21
    init_freq = (float)hz_to_rads(19000.0, samplerate);
    min_freq = (float)hz_to_rads(18750.0, samplerate);
    max_freq = (float)hz_to_rads(19250.0, samplerate);
    int rc = taps.alloc(t.size() * sizeof(float));
    if (rc) { return rc; }
    B200_CK(cudaMemcpy(taps.p, t.data(), t.size() * sizeof(float), cudaMemcpyHostToDevice));
    if ((rc = state.alloc(16))) { return rc; }
    reset_state();
    return 0;
}
void StereoStage::reset_state() {
    const float st[2] = { 0.0f, init_freq };                                                 // PLL initPhase 0, initFreq 19 kHz
    if (state.p) { cudaMemcpy(state.p, st, sizeof(st), cudaMemcpyHostToDevice); }
}

// ------------------------------------------------------------------ SeqStage
static void agc_coefs(SeqJob& j, double setPoint, double attack, double decay, double maxGain, double maxOut) {
    // loop::AGC::init (agc.h:13-24): doubles narrowed to float members
    j.set_point = (float)setPoint;
    j.attack = (float)attack;
    j.inv_attack = 1.0f - j.attack;
    j.decay = (float)decay;
    j.inv_decay = 1.0f - j.decay;
    j.max_gain = (float)maxGain;
    j.max_out = (float)maxOut;
}
int SeqStage::configure_am(int agcMode, double attack, double decay, double dcRate) {
    memset(&proto, 0, sizeof(proto));
    proto.kind = 0;
    proto.agc_mode = agcMode;
    agc_coefs(proto, 1.0, attack, decay, 10e6, 10.0);            // am.h:33-34
    proto.dc_rate = (float)dcRate;
    memset(init_state, 0, sizeof(init_state));
    // amp = setPoint / initGain with initGain = INFINITY -> 0  (agc.h:22, am.h:33)
    init_state[0] = 0.0f;
    init_state[1] = 0.0f;
    int rc = state.alloc(sizeof(init_state));
    if (rc) { return rc; }
    B200_CK(cudaMemcpy(state.p, init_state, sizeof(init_state), cudaMemcpyHostToDevice));
    return 0;
}
int SeqStage::configure_ssb(int mode, double bandwidth, double samplerate, double attack, double decay) {
    memset(&proto, 0, sizeof(proto));
    proto.kind = 1;
    agc_coefs(proto, 1.0, attack, decay, 10e6, 10.0);            // ssb.h:29
    double tr = (mode == 0) ? bandwidth / 2.0 : ((mode == 1) ? -bandwidth / 2.0 : 0.0);   // ssb.h:106-116
    double rad = hz_to_rads(tr, samplerate);
    proto.delta_re = (float)std::cos(rad);
    proto.delta_im = (float)std::sin(rad);
    memset(init_state, 0, sizeof(init_state));
    init_state[3] = 1.0f;                                          // rotator phase (1, 0)
    int rc = state.alloc(sizeof(init_state));
    if (rc) { return rc; }
    B200_CK(cudaMemcpy(state.p, init_state, sizeof(init_state), cudaMemcpyHostToDevice));
    return 0;
}

void SeqStage::set_agc(double attack, double decay) {
    proto.attack = (float)attack;
    proto.inv_attack = 1.0f - proto.attack;
    proto.decay = (float)decay;
    proto.inv_decay = 1.0f - proto.decay;
}
void SeqStage::set_deemph_tau(double tau, double samplerate) {
    float dt = 1.0f / samplerate;                       // deephasis.h:91-94: dt is a float
    proto.alpha = dt / (tau + dt);
}

int SeqStage::configure_deemph(double tau, double samplerate) {
    memset(&proto, 0, sizeof(proto));
    proto.kind = 2;
    set_deemph_tau(tau, samplerate);
    in_es = 2;
    out_es = 2;
    memset(init_state, 0, sizeof(init_state));
    int rc = state.alloc(sizeof(init_state));
    if (rc) { return rc; }
    B200_CK(cudaMemcpy(state.p, init_state, sizeof(init_state), cudaMemcpyHostToDevice));
    return 0;
}

int SeqStage::configure_noise_blanker(double rate, double level) {
    memset(&proto, 0, sizeof(proto));
    proto.kind = 3;
    proto.nb_rate = (float)rate;                        // noise_blanker.h:13-15: _rate, _invRate = 1.0f - _rate, _level are floats
    proto.nb_inv_rate = 1.0f - proto.nb_rate;
    proto.nb_level = (float)level;
    in_es = 2;
    out_es = 2;
    memset(init_state, 0, sizeof(init_state));
    init_state[7] = 1.0f;                               // amp = 1.0 (noise_blanker.h:74; reset() restores it)
    int rc = state.alloc(sizeof(init_state));
    if (rc) { return rc; }
    B200_CK(cudaMemcpy(state.p, init_state, sizeof(init_state), cudaMemcpyHostToDevice));
    return 0;
}
int FmIfStage::configure(int nbins) {
    if (!fmif_supported(nbins)) { set_error("FM IF noise reduction: %d bins (supported: 2 ... %d)", nbins, 64); return B200_EINVAL; }
    bins = nbins;
    hist = bins - 1;
    const std::vector<float> w = fmif_window(bins), t = dft_twiddles(bins);
    int rc;
    if ((rc = win.alloc(w.size() * sizeof(float), false)) || (rc = tw.alloc(t.size() * sizeof(float), false))) { return rc; }
    B200_CK(cudaMemcpy(win.p, w.data(), w.size() * sizeof(float), cudaMemcpyHostToDevice));
    B200_CK(cudaMemcpy(tw.p, t.data(), t.size() * sizeof(float), cudaMemcpyHostToDevice));
    return 0;
}

// ------------------------------------------------------------------ Chain
// the decimating FIR that k_xd_tma can run as its ÷4 epilogue (kernels.cuh: XdJob::f2_out)
static bool s1_f2_stage(const Stage* s) {
    return s->kind == K_FIRC && s->in_es == 2 && ((const FirCStage*)s)->decim == XD_F2_D && ((const FirCStage*)s)->ntaps == XD_F2_T;
}
int Chain::finalize(int max_in, bool dbl_first, const FuseCfg* fuse) {
    if (st.empty()) { set_error("empty chain"); return B200_EINVAL; }
    int cap = max_in;
    if (dbl_first && st.size() >= 2 && st[0]->kind == K_XD) {
        st[1]->dbl = true;
        // stage 1 may produce the (4, 27) stage's outputs itself (Scheduler::run), where k_dfir_reg would run that stage: the
        // stage after it is then fed by stage 1
        if (st.size() >= 3 && s1_f2_stage(st[1].get()) && (fuse ? fuse->pre_reg : fcfg.pre_reg) > 0) { st[2]->dbl = true; }
    }
    for (auto& s : st) {
        if (s->kind != K_XD) {
            int rc = s->alloc_in(cap);
            if (rc) { return rc; }
        }
        else { s->cap_in = cap; }
        cap = s->max_out(cap);
    }
    {
        int c2 = max_in;
        for (auto& s : st) {
            if (s->kind == K_STEREO) {
                StereoStage* q = (StereoStage*)s.get();
                int rc2;
                if ((rc2 = q->p.alloc(((size_t)c2 + 8) * sizeof(float2), false)) || (rc2 = q->vco.alloc(((size_t)c2 + 8) * sizeof(float2), false))) { return rc2; }
            }
            c2 = s->max_out(c2);
        }
    }
    out_es = st.back()->out_es;
    out_cap = cap;
    int rc = out.alloc(((size_t)cap + 8) * out_es * sizeof(float));
    if (rc) { return rc; }
    if (fuse) { fcfg = *fuse; }
    rc = plan_fused();
    if (rc) { return rc; }
    // every table was uploaded with legacy-stream copies / memsets; the data path runs on non-blocking streams
    B200_CK(cudaDeviceSynchronize());
    return 0;
}

// ---- fused tail: static plan ----
static bool ft_fusable(const Stage* s) {
    switch (s->kind) {
    case K_FIRC: return s->in_es == 2;
    case K_POLY: return s->in_es == 2 && ((const PolyStage*)s)->interp <= 64;    // FT_MAX_L (fused_tail.cuh)
    case K_QUAD: case K_FIRR: case K_M2S: return true;
    default: return false;
    }
}
// fills the static fields of an FtStage from a Stage (the per-chunk fields are set by the scheduler)
static void ft_describe(const Stage* s, FtStage& d) {
    memset(&d, 0, sizeof(d));
    d.D = 1; d.L = 1; d.T = 1;
    d.hist = s->hist;
    d.es = s->in_es;
    switch (s->kind) {
    case K_FIRC: { const FirCStage* f = (const FirCStage*)s; d.kind = FT_FIRC; d.T = f->ntaps; d.D = f->decim; break; }
    case K_POLY: { const PolyStage* f = (const PolyStage*)s; d.kind = FT_POLY; d.T = f->tpp; d.D = f->decim; d.L = f->interp; break; }
    case K_QUAD: { const QuadStage* f = (const QuadStage*)s; d.kind = FT_QUAD; d.scale = f->inv_dev; break; }
    case K_FIRR: { const FirRStage* f = (const FirRStage*)s; d.kind = FT_FIRR; d.T = f->ntaps; d.dup = f->stereo; break; }
    default: d.kind = FT_M2S; d.dup = 1; break;
    }
    d.taps = s->taps_pm.as<float>();
    d.ntap_f = s->pm_floats;
}
static long long ft_need_len(const FtStage& d, long long len) {
    switch (d.kind) {
    case FT_FIRC: case FT_FIRR: return (len - 1) * d.D + d.T;
    case FT_POLY: return ((len - 1) * d.D + d.L - 1) / d.L + d.T + 1;
    case FT_QUAD: return len + 1;
    default: return len;
    }
}
static int ft_slack(const FtStage& d) {
    if (d.kind == FT_FIRC || d.kind == FT_FIRR) { return d.D; }
    if (d.kind == FT_POLY) { return d.D / d.L + 2; }
    return 0;
}
static int round4(int x) { return (x + 3) & ~3; }

int Chain::plan_fused() {
    fp.active = false;
    for (auto& s : st) { s->fmid = false; }
    fp.beg = 1;
    if (!fcfg.on || st.size() < 3 || st[0]->kind != K_XD) { return 0; }
    // the short decimating FIRs right behind stage 1 run in registers (k_dfir_reg), one launch each, in front of the fused
    // launch -- as long as at least two stages are left to fuse
    int beg = 1;
    if (fcfg.pre_reg > 0) {
        while (beg - 1 < fcfg.pre_reg && beg < (int)st.size() && st[beg]->kind == K_FIRC && st[beg]->in_es == 2 && ((FirCStage*)st[beg].get())->decim > 1 &&
               dfir_reg_supported(((FirCStage*)st[beg].get())->decim, ((FirCStage*)st[beg].get())->ntaps)) { beg++; }
    }
    int end = beg;
    for (;;) {
        end = beg;
        while (end < (int)st.size() && end - beg < FT_MAXST && ft_fusable(st[end].get())) { end++; }
        if (end - beg >= 2 || beg == 1) { break; }
        beg--;                                   // too little left behind the register stages: give one back
    }
    const int nst = end - beg;
    if (nst < 2) { return 0; }
    if (fcfg.reg_all && fcfg.pre_reg > 0) {
        // every stage behind stage 1 has a register-window kernel of its own: no fused launch for this chain
        bool all = true;
        for (int i = 1; i < end && all; i++) {
            const Stage* s = st[i].get();
            switch (s->kind) {
            case K_FIRC: {
                const FirCStage* f = (const FirCStage*)s;
                all = s->in_es == 2 && ((f->decim == 1 && f->ntaps <= 2000) || (f->decim > 1 && dfir_reg_supported(f->decim, f->ntaps)));
                break;
            }
            case K_POLY: all = s->in_es == 2 && poly_reg_supported(((const PolyStage*)s)->interp, ((const PolyStage*)s)->decim) && ((const PolyStage*)s)->tpp <= 512; break;
            case K_FIRR: all = ((const FirRStage*)s)->ntaps <= 2000; break;
            case K_QUAD: case K_M2S: break;
            default: all = false; break;
            }
        }
        if (all) { return 0; }
    }
    fp.beg = beg;
    FtStage d[FT_MAXST];
    for (int i = 0; i < nst; i++) { ft_describe(st[beg + i].get(), d[i]); }
    // taps region
    int toff = 0;
    for (int i = 0; i < nst; i++) {
        fp.tap_off[i] = toff;
        fp.qpitch[i] = 0;
        if (d[i].kind == FT_FIRC || d[i].kind == FT_FIRR || d[i].kind == FT_POLY) {
            fp.qpitch[i] = (d[i].T + d[i].D - 1) / d[i].D;
            toff += d[i].ntap_f;
        }
    }
    // direct first stage: decimating FIR by 2 or 4 on the complex stream
    fp.s0_direct = fcfg.direct && d[0].kind == FT_FIRC && (d[0].D == 2 || d[0].D == 4) && d[0].T <= 512;
    fp.nat_off = toff;
    if (fp.s0_direct) { toff += round4(d[0].T); }
    const int limit_f = fcfg.smem_limit / 4;
    int ob = fcfg.ob_force > 0 ? fcfg.ob_force : fcfg.ob_max;
    for (; ob >= 4 * FT_R; ob = (ob * 3 / 4) / FT_R * FT_R) {
        // bounds on the per-slab input range of every stage (see DESIGN.md: fused tail)
        long long lb[FT_MAXST + 1];
        lb[nst] = ob;
        for (int i = nst - 1; i >= 0; i--) {
            long long need = ft_need_len(d[i], lb[i + 1]) + ft_slack(d[i]);
            lb[i] = std::max<long long>(need, d[i].hist);
        }
        int region[2] = { 0, 0 };
        bool ok = true;
        for (int i = 1; i < nst; i++) {
            const int rows = ft_rows(d[i]);
            const long long cols = (lb[i] + rows + rows - 1) / rows + FT_R + 2;
            if (cols * rows * d[i].es > limit_f) { ok = false; break; }
            fp.pitch[i] = (int)cols;
            region[i & 1] = std::max(region[i & 1], round4((int)(cols * rows * d[i].es)));
        }
        if (!ok) { continue; }
        const int fixed = toff + region[1];
        // stage 0 streams through what is left of the budget, at most what one pass over the slab needs
        const int rows0 = ft_rows(d[0]);
        int ot0 = (int)((lb[1] + FT_R - 1) / FT_R) * FT_R;
        std::function<long long(int)> stage0_floats = [&](int ot) {
            long long cols = (ft_need_len(d[0], ot) + rows0 + rows0 - 1) / rows0 + FT_R + 2;
            return cols * rows0 * d[0].es;
        };
        // two staging buffers (double-buffered cp.async); sub-tiles that give every thread of the CTA a 5-output unit.
        // direct first stage: three raw ring buffers, 3 outputs per thread and sub-tile.
        const int nbuf = fp.s0_direct ? 3 : 2;
        if (fp.s0_direct) {
            stage0_floats = [&](int ot) { return (long long)((((long long)(ot - 1) * d[0].D + d[0].T + 3) & ~1LL) * 2); };
        }
        const int want = fcfg.threads * (fp.s0_direct ? 3 : 5);
        if (ot0 > want) { ot0 = want; }
        while (ot0 >= FT_R && std::max<long long>(nbuf * (long long)round4((int)stage0_floats(ot0)), region[0]) > (long long)limit_f - fixed - 64) { ot0 -= FT_R; }
        if (ot0 < FT_R) { continue; }
        {
            long long cols = (ft_need_len(d[0], ot0) + rows0 + rows0 - 1) / rows0 + FT_R + 2;
            fp.pitch[0] = (int)cols;
            fp.stg2_rel = round4((int)stage0_floats(ot0));
            region[0] = std::max(region[0], nbuf * fp.stg2_rel);
        }
        // arena: [taps | odd stages | even stages (incl. staging)]
        for (int i = 0; i < nst; i++) { fp.buf[i] = (i & 1) ? toff : toff + region[1]; }
        fp.smem = (size_t)(toff + region[0] + region[1] + 64) * sizeof(float);
        fp.ob_max = ob;
        fp.ot0 = ot0;
        fp.end = end;
        fp.active = true;
        break;
    }
    if (!fp.active) { return 0; }
    for (int i = 1; i < nst; i++) {
        Stage* s = st[fp.beg + i].get();
        s->fmid = true;
        for (int b = 0; b < 2; b++) {
            const size_t need = ((size_t)s->hist + 8) * s->in_es * sizeof(float);
            if (!s->fh[b].p || s->fh[b].bytes < need) {
                int rc = s->fh[b].alloc(need);
                if (rc) { return rc; }
            }
        }
    }
    return 0;
}
int Chain::plan(int n) {
    for (auto& s : st) { n = s->plan(n); }
    n_out = n;
    return n;
}
int Chain::quad_index() const {
    for (size_t i = 0; i < st.size(); i++) { if (st[i]->kind == K_QUAD) { return (int)i; } }
    return -1;
}
int Chain::max_out(int n) const {
    for (auto& s : st) { n = s->max_out(n); }
    return n;
}
int Chain::peek(int n) const {
    for (auto& s : st) {
        if (s->kind != K_FIRC) { return -1; }
        const FirCStage* f = (const FirCStage*)s.get();
        n = (f->offset < n) ? (n - f->offset + f->decim - 1) / f->decim : 0;
    }
    return n;
}
void clear_stage_state(Stage& s) {
    s.reset_state();
    if (s.inbuf.p && s.hist > 0) { cudaMemset(s.inbuf.p, 0, (size_t)s.hist * s.in_es * sizeof(float)); }
    if (s.inbuf_alt.p && s.hist > 0) { cudaMemset(s.inbuf_alt.p, 0, (size_t)s.hist * s.in_es * sizeof(float)); }
    for (int i = 0; i < 2; i++) {
        if (s.fh[i].p) { cudaMemset(s.fh[i].p, 0, s.fh[i].bytes); }
    }
    s.fpar = 0;
    if (s.kind == K_SEQ) {
        SeqStage* q = (SeqStage*)&s;
        // AM::reset / AGC::reset (am.h:90-98, agc.h:64-68), Deemphasis::reset; the SSB demodulator has no reset
        cudaMemcpy(q->state.p, q->init_state, sizeof(q->init_state), cudaMemcpyHostToDevice);
    }
}
void Chain::reset_state() {
    for (auto& s : st) { clear_stage_state(*s); }
    cudaDeviceSynchronize();      // the memsets above run on the legacy stream: finish them before the library's streams go on
}

int Chain::unfuse_history() {
    for (auto& s : st) {
        if (s->fmid && s->hist > 0) {
            // its plain history is the head of the buffer the next chunk uses (of a double-buffered stage: not this chunk's)
            B200_CK(cudaMemcpy(s->dbl ? s->other_base() : s->inbuf.as<float>(), s->fh[s->fpar].p, (size_t)s->hist * s->in_es * sizeof(float),
                               cudaMemcpyDeviceToDevice));
        }
        s->fmid = false;
    }
    B200_CK(cudaDeviceSynchronize());
    return 0;
}
int Chain::restage() {
    int rc = plan_fused();
    if (rc) { return rc; }
    for (auto& s : st) {
        if (s->fmid && s->hist > 0) {
            B200_CK(cudaMemcpy(s->fh[s->fpar].p, s->dbl ? s->other_base() : s->inbuf.as<float>(), (size_t)s->hist * s->in_es * sizeof(float),
                               cudaMemcpyDeviceToDevice));
        }
    }
    B200_CK(cudaDeviceSynchronize());      // device-to-device copies on the legacy stream
    return 0;
}

int Chain::add_xlator(double offsetHz, double samplerate) {
    auto x = std::make_unique<XdStage>();
    x->configure(1, std::vector<float>{ 1.0f });
    x->set_offset_rad(hz_to_rads(offsetHz, samplerate));
    st.push_back(std::move(x));
    return 0;
}

int Chain::add_power_decim(int ratio) {
    if (ratio == 1) { return add_fir_c(std::vector<float>{ 1.0f }, 1); }   // memcpy path (power_decimator.h:53-56)
    const DecimPlan* p = find_decim_plan(ratio);
    if (!p) { set_error("no decimation plan for ratio %d (decim_plans.bin not found?)", ratio); return B200_ENOPLAN; }
    for (auto& s : p->stages) {
        int rc = add_fir_c(s.taps, s.decim);
        if (rc) { return rc; }
    }
    return 0;
}

int Chain::add_fir_c(const std::vector<float>& taps, int decim) {
    auto f = std::make_unique<FirCStage>();
    int rc = f->configure(taps, decim);
    if (rc) { return rc; }
    st.push_back(std::move(f));
    return 0;
}
int Chain::add_fir_r(const std::vector<float>& taps, bool stereo) {
    auto f = std::make_unique<FirRStage>();
    int rc = f->configure(taps, stereo);
    if (rc) { return rc; }
    st.push_back(std::move(f));
    return 0;
}

int Chain::add_resampler(double inSR, double outSR) {
    ResampPlan pl = make_resamp_plan(inSR, outSR);
    if (pl.use_decim) {
        int rc = add_power_decim(pl.predec_ratio);
        if (rc) { return rc; }
    }
    if (!pl.rtaps.empty()) {
        auto r = std::make_unique<PolyStage>();
        int rc = r->configure(pl.interp, pl.decim, pl.rtaps);
        if (rc) { return rc; }
        st.push_back(std::move(r));
    }
    if (!pl.use_decim && pl.rtaps.empty()) { return add_fir_c(std::vector<float>{ 1.0f }, 1); }  // Mode::NONE memcpy
    return 0;
}

// channel::RxVFO::init (rx_vfo.h:17-31): xlator(-offset) -> RationalResampler -> [FIR lowPass(bw/2, 0.1*bw/2, outSR)]
int Chain::add_rxvfo(double inSR, double outSR, double bw, double offset) {
    ResampPlan pl = make_resamp_plan(inSR, outSR);
    auto x = std::make_unique<XdStage>();
    size_t first_other = 0;
    const DecimPlan* dp = nullptr;
    if (pl.use_decim) {
        dp = find_decim_plan(pl.predec_ratio);
        if (!dp) { set_error("no decimation plan for ratio %d (decim_plans.bin not found?)", pl.predec_ratio); return B200_ENOPLAN; }
        if ((int)dp->stages[0].taps.size() - 1 > Scheduler::RAW_HIST) {
            set_error("first decimation stage of ratio %d has %d taps: more than the %d samples of raw history kept", pl.predec_ratio,
                      (int)dp->stages[0].taps.size(), Scheduler::RAW_HIST + 1);
            return B200_ECAP;
        }
        x->configure(dp->stages[0].decim, dp->stages[0].taps);     // xlator fused with the first DecimatingFIR
        first_other = 1;
    }
    else {
        x->configure(1, std::vector<float>{ 1.0f });
    }
    x->set_offset_rad(hz_to_rads(-offset, inSR));
    st.push_back(std::move(x));
    if (dp) {
        for (size_t i = first_other; i < dp->stages.size(); i++) {
            int rc = add_fir_c(dp->stages[i].taps, dp->stages[i].decim);
            if (rc) { return rc; }
        }
    }
    if (!pl.rtaps.empty()) {
        auto r = std::make_unique<PolyStage>();
        int rc = r->configure(pl.interp, pl.decim, pl.rtaps);
        if (rc) { return rc; }
        st.push_back(std::move(r));
    }
    // The reference always owns the channel filter and bypasses it while bandwidth == outSamplerate (rx_vfo.h:24,60-70,
    // 91-93).  Here the stage always exists; bypass = the exact identity tap {1.0f}, so setBandwidth can switch between
    // the two at a chunk boundary.  (The reference's bypassed filter keeps a stale delay line; after identity -> low-pass
    // this one starts from the cleared history a fresh block has.)
    {
        double fw = bw / 2.0;
        int rc = add_fir_c(bw != outSR ? lowpass_taps(fw, fw * 0.1, outSR) : std::vector<float>{ 1.0f }, 1);
        if (rc) { return rc; }
        chan_fir = (int)st.size() - 1;
    }
    return 0;
}

int Chain::add_quad(double deviationHz, double samplerate) {
    auto q = std::make_unique<QuadStage>();
    int rc = q->configure(deviationHz, samplerate);
    if (rc) { return rc; }
    st.push_back(std::move(q));
    return 0;
}
int Chain::add_wfm(double deviationHz, double samplerate, bool lowPass, bool stereo) {
    int rc = add_quad(deviationHz, samplerate);
    if (rc) { return rc; }
    if (stereo) {
        // pilot filter -> PLL -> L-R recovery -> (l, r); alFir / arFir are one real-tap FIR over the (l, r) pairs
        auto sst = std::make_unique<StereoStage>();
        if ((rc = sst->configure(samplerate))) { return rc; }
        st.push_back(std::move(sst));
        if (lowPass) { return add_fir_c(lowpass_taps(15000.0, 4000.0, samplerate), 1); }
        return 0;
    }
    if (lowPass) { return add_fir_r(lowpass_taps(15000.0, 4000.0, samplerate), true); }   // broadcast_fm.h:45
    st.push_back(std::make_unique<M2SStage>());
    return 0;
}
int Chain::add_wfm_rds(double deviationHz, double samplerate) {
    int rc = add_quad(deviationHz, samplerate);
    if (rc) { return rc; }
    return add_rds_branch(samplerate);
}
int Chain::add_rds_branch(double samplerate) {
    auto x = std::make_unique<RxlStage>();
    x->set_offset_rad(hz_to_rads(-57000.0, samplerate));                 // xlator.init(NULL, -57000.0, samplerate)
    st.push_back(std::move(x));
    return add_resampler(samplerate, 5000.0);                              // rdsResamp.init(NULL, samplerate, 5000.0)
}
int Chain::add_nfm(double samplerate, double bandwidth, bool lowPass) {
    int rc = add_quad(bandwidth / 2.0, samplerate);                                         // fm.h:28
    if (rc) { return rc; }
    if (lowPass) { return add_fir_r(lowpass_taps(bandwidth / 2.0, (bandwidth / 2.0) * 0.1, samplerate), true); } // fm.h:123
    st.push_back(std::make_unique<M2SStage>());
    return 0;
}
int Chain::add_am(int agcMode, double bandwidth, double attack, double decay, double dcRate, double samplerate) {
    auto s = std::make_unique<SeqStage>();
    int rc = s->configure_am(agcMode, attack, decay, dcRate);
    if (rc) { return rc; }
    st.push_back(std::move(s));
    return add_fir_r(lowpass_taps(bandwidth / 2.0, (bandwidth / 2.0) * 0.1, samplerate), true);   // am.h:36-37
}
int Chain::add_ssb(int mode, double bandwidth, double samplerate, double attack, double decay) {
    auto s = std::make_unique<SeqStage>();
    int rc = s->configure_ssb(mode, bandwidth, samplerate, attack, decay);
    if (rc) { return rc; }
    st.push_back(std::move(s));
    st.push_back(std::make_unique<M2SStage>());
    return 0;
}

int Chain::add_deemph(double tau, double samplerate) {
    auto s = std::make_unique<SeqStage>();
    int rc = s->configure_deemph(tau, samplerate);
    if (rc) { return rc; }
    st.push_back(std::move(s));
    return 0;
}
int Chain::add_af_chain(double afSR, double audioSR, bool highPass, double deemphTau) {
    int rc = add_resampler(afSR, audioSR);                                   // stereo_t == two packed floats: same kernels
    if (rc) { return rc; }
    if (highPass && (rc = add_af_highpass(audioSR))) { return rc; }
    if (deemphTau > 0.0 && (rc = add_deemph(deemphTau, audioSR))) { return rc; }
    return 0;
}
int Chain::add_af_highpass(double audioSR) {
    return add_fir_c(highpass_taps(300.0, 100.0, audioSR), 1);              // radio_module.h:597-598
}

int Chain::add_noise_blanker(double rate, double level) {
    auto s = std::make_unique<SeqStage>();
    int rc = s->configure_noise_blanker(rate, level);
    if (rc) { return rc; }
    st.push_back(std::move(s));
    return 0;
}
int Chain::add_fmif(int bins) {
    auto s = std::make_unique<FmIfStage>();
    int rc = s->configure(bins);
    if (rc) { return rc; }
    st.push_back(std::move(s));
    return 0;
}
int Chain::add_squelch(double level) {
    auto q = std::make_unique<SquelchStage>();
    q->level = (float)level;
    int rc = q->partial.alloc(SQ_MAXPARTS * sizeof(float));
    if (rc) { return rc; }
    st.push_back(std::move(q));
    return 0;
}
int Chain::add_volume(double volume, bool muted) {
    const float v = powf((float)volume, 2);                                  // volume.h:14: _volume = powf(volume, 2)
    st.push_back(std::make_unique<ScaleStage>(st.empty() ? 2 : st.back()->out_es, muted ? 0.0f : v));
    return 0;
}

// ------------------------------------------------------------------ Scheduler
int Scheduler::init_raw() {
    if (raw_hist.p) { return 0; }
    return raw_hist.alloc((size_t)RAW_HIST * sizeof(float2));
}
Scheduler::~Scheduler() {
    drop_graphs();
    for (Timer& t : timers) { for (cudaEvent_t e : t.ev) { cudaEventDestroy(e); } }
    for (int i = 0; i < 2; i++) {
        if (ev_stage1[i]) { cudaEventDestroy(ev_stage1[i]); }
        if (ev_tail[i]) { cudaEventDestroy(ev_tail[i]); }
    }
}
cudaEvent_t Scheduler::timer_begin(int group, cudaStream_t s) {
    if (!time_s1) { return nullptr; }
    Timer& t = timers[group];
    if (t.used + 2 > 2 * TIMER_MAX) { return nullptr; }
    if (t.used + 2 > t.ev.size()) {
        cudaEvent_t a, b;
        if (cudaEventCreate(&a) != cudaSuccess || cudaEventCreate(&b) != cudaSuccess) { return nullptr; }
        t.ev.push_back(a);
        t.ev.push_back(b);
    }
    cudaEvent_t t0 = t.ev[t.used], t1 = t.ev[t.used + 1];
    t.used += 2;
    cudaEventRecord(t0, s);
    return t1;
}
int Scheduler::group_stats(int group, double* ms_total, int* n) {
    if (group < 0 || group > 3) { set_error("bad timer group"); return B200_EINVAL; }
    Timer& t = timers[group];
    double tot = 0.0;
    for (size_t i = 0; i + 1 < t.used; i += 2) {
        B200_CK(cudaEventSynchronize(t.ev[i + 1]));
        float ms = 0.0f;
        B200_CK(cudaEventElapsedTime(&ms, t.ev[i], t.ev[i + 1]));
        tot += ms;
    }
    *ms_total = tot;
    *n = (int)(t.used / 2);
    t.used = 0;
    return 0;
}
int Scheduler::reset_raw() {
    if (raw_hist.p) { B200_CK(cudaMemset(raw_hist.p, 0, raw_hist.bytes)); B200_CK(cudaDeviceSynchronize()); }
    return 0;
}

// FIR::setTaps (fir.h:31-52): new taps, keep the most recent history
static int apply_pending_taps(FirCStage* f, cudaStream_t s) {
    if (f->pending.empty()) { return 0; }
    (void)s;
    B200_CK(cudaDeviceSynchronize());
    const int newT = (int)f->pending.size(), oldT = f->ntaps;
    const int newH = newT - 1, oldH = oldT - 1;
    const size_t bytes = ((size_t)newH + f->cap_in + Scheduler::STAGE_SPARE) * f->in_es * sizeof(float);
    DevBuf nb, nb2;
    int rc = nb.alloc(bytes);
    if (rc) { return rc; }
    if (f->dbl && (rc = nb2.alloc(bytes))) { return rc; }
    int keep = std::min(newH, oldH);
    // the live history sits in the buffer the NEXT chunk will use (the carry wrote it there)
    const float* live = f->dbl ? ((f->par ? f->inbuf.as<float>() : f->inbuf_alt.as<float>())) : f->inbuf.as<float>();
    float* live_new = f->dbl ? ((f->par ? nb.as<float>() : nb2.as<float>())) : nb.as<float>();
    if (keep > 0) {
        B200_CK(cudaMemcpy(live_new + (size_t)(newH - keep) * f->in_es, live + (size_t)(oldH - keep) * f->in_es,
                           (size_t)keep * f->in_es * sizeof(float), cudaMemcpyDeviceToDevice));
    }
    if (f->dbl && keep > 0) {
        // and in front of the previous chunk's (empty) data in the other buffer, where stage 1's ÷4 epilogue looks for it
        float* other_new = f->par ? nb2.as<float>() : nb.as<float>();
        B200_CK(cudaMemcpy(other_new + (size_t)(newH - keep) * f->in_es, live + (size_t)(oldH - keep) * f->in_es,
                           (size_t)keep * f->in_es * sizeof(float), cudaMemcpyDeviceToDevice));
    }
    f->n_in = 0;
    std::swap(f->inbuf.p, nb.p);
    std::swap(f->inbuf.bytes, nb.bytes);
    if (f->dbl) {
        std::swap(f->inbuf_alt.p, nb2.p);
        std::swap(f->inbuf_alt.bytes, nb2.bytes);
    }
    if (f->fmid) {
        // fused tail: the stage's history lives in fh[fpar]
        DevBuf h0, h1;
        const size_t hb = ((size_t)newH + 8) * f->in_es * sizeof(float);
        if ((rc = h0.alloc(hb)) || (rc = h1.alloc(hb))) { return rc; }
        if (keep > 0) {
            B200_CK(cudaMemcpy(h0.as<float>() + (size_t)(newH - keep) * f->in_es, f->fh[f->fpar].as<float>() + (size_t)(oldH - keep) * f->in_es,
                               (size_t)keep * f->in_es * sizeof(float), cudaMemcpyDeviceToDevice));
        }
        std::swap(f->fh[f->fpar].p, h0.p); std::swap(f->fh[f->fpar].bytes, h0.bytes);
        std::swap(f->fh[f->fpar ^ 1].p, h1.p); std::swap(f->fh[f->fpar ^ 1].bytes, h1.bytes);
    }
    rc = f->taps.alloc((size_t)newT * sizeof(float));
    if (rc) { return rc; }
    B200_CK(cudaMemcpy(f->taps.p, f->pending.data(), (size_t)newT * sizeof(float), cudaMemcpyHostToDevice));
    if ((rc = f->upload_pm(f->pending, f->decim, 1))) { return rc; }
    f->htaps = f->pending;
    f->ntaps = newT;
    f->hist = newH;
    if (f->decim != 1) { f->offset = 0; }          // DecimatingFIR::setTaps (decimating_fir.h:18-25)
    f->pending.clear();
    B200_CK(cudaDeviceSynchronize());              // the device-to-device copies above ran on the legacy stream
    return 0;
}

// ---- launch list of everything behind stage 1 of a chunk (engine.h: LaunchRec) ----
void LaunchRec::add(Launch fn, const void* p, size_t size, int a, size_t b) {
    const size_t off = (bytes.size() + 15) & ~(size_t)15;
    bytes.resize(off + size, 0);
    memcpy(bytes.data() + off, p, size);
    items.push_back(Item{ fn, off, size, a, b });
}
unsigned long long LaunchRec::hash() const {
    // 64-bit multiply-xorshift over the launchers, the launch arguments and the parameter bytes
    unsigned long long h = 0x9E3779B97F4A7C15ULL ^ (unsigned long long)items.size();
    auto mix = [&](unsigned long long v) { h ^= v; h *= 0xD6E8FEB86659FD93ULL; h ^= h >> 32; };
    for (const Item& it : items) {
        mix((unsigned long long)(uintptr_t)it.fn); mix((unsigned long long)it.size);
        mix((unsigned long long)(unsigned)it.a); mix((unsigned long long)it.b);
    }
    const size_t n8 = bytes.size() / 8;
    const unsigned char* b = bytes.data();
    for (size_t i = 0; i < n8; i++) { unsigned long long v; memcpy(&v, b + 8 * i, 8); mix(v); }
    for (size_t i = n8 * 8; i < bytes.size(); i++) { mix(b[i]); }
    return h;
}
int LaunchRec::replay(const KernelOpts& o, cudaStream_t s, long long* nlaunch) const {
    for (const Item& it : items) {
        int nl = 0;
        cudaError_t e = it.fn(bytes.data() + it.off, it, o, s, &nl);
        if (e != cudaSuccess) { return cuda_fail(e, "kernel launch (tail list)"); }
        if (nlaunch) { *nlaunch += nl; }
    }
    return 0;
}

// the launchers of the list: one per typed launch function, with or without kernel choices
template <class P, cudaError_t (*L)(const P&, const KernelOpts&, cudaStream_t)>
static cudaError_t launch_of(const void* p, const LaunchRec::Item&, const KernelOpts& o, cudaStream_t s, int* nl) {
    *nl = 1;
    return L(*(const P*)p, o, s);
}
template <class P, cudaError_t (*L)(const P&, cudaStream_t)>
static cudaError_t launch_of(const void* p, const LaunchRec::Item&, const KernelOpts&, cudaStream_t s, int* nl) {
    *nl = 1;
    return L(*(const P*)p, s);
}
template <class P, cudaError_t (*L)(const P&, cudaStream_t, int*)>        // launch_stereo, launch_squelch: more than one kernel
static cudaError_t launch_of_n(const void* p, const LaunchRec::Item&, const KernelOpts&, cudaStream_t s, int* nl) {
    return L(*(const P*)p, s, nl);
}
static cudaError_t launch_of_dfr(const void* q, const LaunchRec::Item&, const KernelOpts& o, cudaStream_t s, int* nl) {
    const DfrParams& p = *(const DfrParams*)q;                              // every job of a batch: the same D and T
    *nl = 1;
    return launch_dfir_reg(p, p.job[0].decim, p.job[0].ntaps, o, s);
}
static cudaError_t launch_of_ft(const void* q, const LaunchRec::Item& it, const KernelOpts&, cudaStream_t s, int* nl) {
    const FtParams& p = *(const FtParams*)q;
    int max_slabs = 0;
    for (int i = 0; i < p.njobs; i++) { max_slabs = std::max(max_slabs, p.job[i].slabs); }
    *nl = 1;
    return launch_tail_fused(p, max_slabs, it.a, it.b, s);                  // a, b: threads, shared memory
}

// One parameter block of the launch list: jobs go in one at a time, and the block goes into the list when it is full, when
// the caller's key (what every job of one launch must share) changes, and at the end of a level.  `mx`: the block's largest
// job count, if it keeps one.  Blocks start zero-filled: the list is hashed and compared as bytes.
template <class P>
struct Batch {
    static const int CAP = (int)(sizeof(P::job) / sizeof(P::job[0]));
    P p;
    LaunchRec::Launch fn;
    int P::*mx;
    int a = 0;
    size_t b = 0;                // launch arguments outside the block (LaunchRec::Item)
    explicit Batch(LaunchRec::Launch f, int P::*m = nullptr) : fn(f), mx(m) { memset(&p, 0, sizeof(P)); }
    void flush(LaunchRec& rec) {
        if (p.njobs == 0) { return; }
        rec.add(fn, &p, sizeof(P), a, b);
        p.njobs = 0;
        if (mx) { p.*mx = 0; }
    }
    // the slot of the next job; a full block, or one holding jobs under another key, goes into the list first
    auto& next(LaunchRec& rec, bool key_changed = false) {
        if (p.njobs > 0 && (key_changed || p.njobs == CAP)) { flush(rec); }
        return p.job[p.njobs++];
    }
    // after the job is filled in: its count, and a block that is now full goes into the list (unless `eager` is false, where
    // it waits for the next job)
    void done(LaunchRec& rec, int n, bool eager = true) {
        if (mx) { p.*mx = std::max(p.*mx, n); }
        if (eager && p.njobs == CAP) { flush(rec); }
    }
};

void Scheduler::drop_graphs() {
    for (auto& kv : graphs) { if (kv.second.exec) { cudaGraphExecDestroy(kv.second.exec); } }
    graphs.clear();
}

int Scheduler::enable_overlap(cudaStream_t tail) {
    tail_stream = tail;
    for (int i = 0; i < 2; i++) {
        if (!ev_stage1[i]) { B200_CK(cudaEventCreateWithFlags(&ev_stage1[i], cudaEventDisableTiming)); }
        if (!ev_tail[i]) { B200_CK(cudaEventCreateWithFlags(&ev_tail[i], cudaEventDisableTiming)); }
    }
    return 0;
}

// deferred parameter changes (FIR::setTaps at a chunk boundary); fallible, so callers run it BEFORE Chain::plan()
int Scheduler::apply_deferred(std::vector<Chain*>& chains) {
    for (Chain* c : chains) {
        bool changed = false;
        for (auto& sp : c->st) {
            if (sp->kind == K_FIRC && !((FirCStage*)sp.get())->pending.empty()) {
                int rc = apply_pending_taps((FirCStage*)sp.get(), stream);
                if (rc) { return rc; }
                changed = true;
            }
        }
        if (changed && c->fp.active) {
            int rc = c->plan_fused();
            if (rc) { return rc; }
            if (!c->fp.active) { set_error("new filter does not fit the fused tail (set option tails=1 before adding VFOs)"); return B200_ECAP; }
        }
    }
    return 0;
}

// the recorded launch list of this chunk: first sight -> plain launches; second sight -> capture into a graph; then replay
int Scheduler::launch_recorded(cudaStream_t ts, bool may_graph) {
    if (rec.items.empty()) { return 0; }
    if (!may_graph) { return rec.replay(opts, ts, &launches); }
    const unsigned long long h = rec.hash();
    auto it = graphs.find(h);
    if (it != graphs.end() && it->second.key.size() == rec.bytes.size() && memcmp(it->second.key.data(), rec.bytes.data(), rec.bytes.size()) == 0) {
        GraphEntry& g = it->second;
        if (g.exec) {
            B200_CK(cudaGraphLaunch(g.exec, ts));
            launches += g.launches;
            graph_hits++;
            return 0;
        }
        // second sight: capture
        if (cudaStreamBeginCapture(ts, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
            long long nl = 0;
            int rc = rec.replay(opts, ts, &nl);
            cudaGraph_t graph = nullptr;
            cudaError_t e = cudaStreamEndCapture(ts, &graph);
            cudaGraphExec_t exec = nullptr;
            if (rc == 0 && e == cudaSuccess && graph && cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess) {
                cudaGraphDestroy(graph);
                g.exec = exec;
                g.launches = nl;
                B200_CK(cudaGraphLaunch(exec, ts));
                launches += nl;
                graph_misses++;
                return 0;
            }
            if (graph) { cudaGraphDestroy(graph); }
            cudaGetLastError();
            graph_tails = 0;                       // capture is not possible here: plain launches from now on
        }
        return rec.replay(opts, ts, &launches);
    }
    if (graphs.size() >= 256) { drop_graphs(); }
    GraphEntry& g = graphs[h];
    if (g.exec) { cudaGraphExecDestroy(g.exec); g.exec = nullptr; }      // (hash collision with other bytes: start over)
    g.key = rec.bytes;
    g.launches = 0;
    graph_misses++;
    return rec.replay(opts, ts, &launches);
}

static inline long long host_now_ns() {
    return (long long)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// level of a chain's first stage in the level-by-level section: an RDS branch starts at its parent's discriminator
static size_t first_level(const Chain* c) { return c->parent ? (size_t)std::max(0, c->parent->quad_index()) : 0; }

int Scheduler::wire(std::vector<Chain*>& chains, int parity) {
    int rc = apply_deferred(chains);          // no-op when the caller already did it
    if (rc) { return rc; }
    for (Chain* c : chains) {
        for (auto& sp : c->st) { sp->par = parity; }
    }
    if (tail_stream && chunk_idx >= 2) {
        // stage 1 of this chunk overwrites the stage-2 input buffers that the tails of chunk-2 were reading
        B200_CK(cudaStreamWaitEvent(stream, ev_tail[parity], 0));
    }
    trace_mark("stage1 start", stream);
    for (Chain* c : chains) {
        for (size_t i = 0; i < c->st.size(); i++) {
            Stage* s = c->st[i].get();
            s->out_ptr = (i + 1 < c->st.size()) ? c->st[i + 1]->in_data() : (c->out_override ? c->out_override : c->out.as<float>());
            if (s->kind == K_XD && ((XdStage*)s)->taps_dirty && (rc = ((XdStage*)s)->upload_taps(stream))) { return rc; }
        }
    }
    return 0;
}

// slots of a stage-1 batch: pair VFOs whose complex taps are exact conjugates (offsets +f / -f, same real prototype, same
// decimation phase): they share every multiply-accumulate of stage 1 (kernels.cuh: XdParams)
static void pair_slots(XdParams& p, XdStage* const* g, bool pair) {
    bool used[B200_BATCH] = { false };
    p.nslots = 0;
    for (int v = 0; v < p.njobs; v++) {
        if (used[v]) { continue; }
        used[v] = true;
        int partner = -1;
        XdStage* a = g[v];
        if (pair && a->w != 0) {
            for (int u = v + 1; u < p.njobs; u++) {
                XdStage* c = g[u];
                if (!used[u] && c->w == (0ULL - a->w) && c->T == a->T && c->chunk_offset == a->chunk_offset &&
                    c->n_out == a->n_out && c->h == a->h) {
                    partner = u;
                    used[u] = true;
                    break;
                }
            }
        }
        p.slot_a[p.nslots] = (signed char)v;
        p.slot_b[p.nslots] = (signed char)partner;
        p.nslots++;
    }
}

// polyphase-filter-bank form (xd_pfb.cuh): every job on a common frequency grid fs / (2 PS), same prototype, same alignment.
// Accept when e^{j w_v PS} is within a few 1e-6 rad (over one tap window) of the same sign.
static void pfb_grid(XdParams& p, XdStage* const* g) {
    XdStage* x0 = g[0];
    for (int v = 1; v < p.njobs; v++) {
        XdStage* xv = g[v];
        if (xv->T != x0->T || xv->chunk_offset != x0->chunk_offset || xv->n_out != x0->n_out || xv->h != x0->h) { return; }
    }
    if (x0->n_out <= 0) { return; }
    p.taps_host = x0->h.data();
    for (int P = 1; P <= 10 && !p.pfb_ps; P++) {
        // drift allowed per P samples so that it stays below 8e-6 rad over the T-tap window
        const double tol_turns = (8e-6 / 6.283185307179586) * (double)P / (double)x0->T;
        const double tol = tol_turns * 18446744073709551616.0;
        int sg = 0;
        bool ok = true;
        for (int v = 0; v < p.njobs && ok; v++) {
            const unsigned long long r = g[v]->w * (unsigned long long)P;
            const double d0 = (double)(long long)r;                                    // distance to 0 (signed)
            const double d1 = (double)(long long)(r - 0x8000000000000000ULL);            // distance to 1/2 turn
            int sv = 0;
            if (std::fabs(d0) <= tol) { sv = 1; } else if (std::fabs(d1) <= tol) { sv = -1; }
            if (sv == 0 || (sg != 0 && sv != sg)) { ok = false; }
            sg = sv;
        }
        if (!ok) { continue; }
        // run the kernel's PS = 8 or 10 instantiation: sigma' = sigma^(PS / P)
        for (int PS : { 8, 10 }) {
            if (PS % P == 0) {
                p.pfb_ps = PS;
                p.pfb_sigma = (sg < 0 && ((PS / P) & 1)) ? -1 : 1;
                break;
            }
        }
    }
}

// The (4, 27) stage behind stage 1 is computed by k_xd_tma's ÷4 epilogue where it would otherwise run in k_dfir_reg (the
// epilogue has its arithmetic), the stage after it is double-buffered like the one stage 1 feeds, and the chunk needs no
// k_xd_edge patch of the stage-1 outputs.  Every other chunk -- a retune inside the tap window, another input format, a
// launch k_xd_tma declines -- stores the stage-1 outputs and runs k_dfir_reg, reading and writing the same history.
static FirCStage* f2_stage(const Scheduler& S, const Chain* c, const XdStage* x, int fmt) {
    if (fmt != FMT_CF32 || S.s1_variant < 8 || S.fuse.pre_reg <= 0 || x->chunk_retuned || c->st.size() < 3) { return nullptr; }
    if (!s1_f2_stage(c->st[1].get()) || (S.tail_stream && !c->st[2]->dbl) || (c->fp.active && c->fp.beg <= 1)) { return nullptr; }
    return (FirCStage*)c->st[1].get();
}

// every raw-input chain, grouped by first-stage decimation so they share the IQ tile
int Scheduler::stage1(std::vector<Chain*>& chains, const void* raw, int fmt, int count) {
    std::map<int, std::vector<XdStage*>> groups;
    std::map<XdStage*, Chain*> chain_of;
    for (Chain* c : chains) {
        if (c->raw_input()) {
            XdStage* x = (XdStage*)c->st[0].get();
            groups[x->D].push_back(x);
            chain_of[x] = c;
        }
    }
    for (auto& kv : groups) {
        std::vector<XdStage*>& g = kv.second;
        for (size_t b = 0; b < g.size(); b += B200_BATCH) {
            XdParams p;
            memset(&p, 0, sizeof(p));
            p.in = raw;
            p.hist = raw_hist.as<float2>();
            p.hist_len = RAW_HIST;
            p.count = count;
            p.D = kv.first;
            p.in_scale = in_scale;
            p.QP = 1;
            p.njobs = (int)std::min<size_t>(B200_BATCH, g.size() - b);
            const std::vector<float>* f2_taps = nullptr;
            for (int v = 0; v < p.njobs; v++) {
                XdStage* x = g[b + v];
                p.job[v].out = (float2*)x->out_ptr;
                p.job[v].gpad = x->gpad.as<float2>();
                p.job[v].phase0 = x->chunk_phase0;
                p.job[v].w = x->w;
                p.job[v].offset = x->chunk_offset;
                p.job[v].n_out = x->n_out;
                p.job[v].T = x->T;
                p.job[v].h = x->hdev.as<float>();
                p.job[v].retuned = x->chunk_retuned ? 1 : 0;
                if (x->chunk_retuned) {
                    const size_t bytes = x->edge_tab.size() * sizeof(unsigned long long);
                    if (!x->edge_ph.p || x->edge_ph.bytes < bytes) {
                        int rc = x->edge_ph.alloc((size_t)RAW_HIST * sizeof(unsigned long long));
                        if (rc) { return rc; }
                    }
                    B200_CK(cudaMemcpyAsync(x->edge_ph.p, x->edge_tab.data(), bytes, cudaMemcpyHostToDevice, stream));
                    p.job[v].hphase = x->edge_ph.as<unsigned long long>();
                    p.job[v].edge_start = x->chunk_edge_start;
                }
                p.QP = std::max(p.QP, x->QP);
                FirCStage* f = f2_stage(*this, chain_of[x], x, fmt);
                if (f && f->n_out > 0 && (!f2_taps || *f2_taps == f->htaps)) {       // one tap set per launch
                    f2_taps = &f->htaps;
                    memcpy(p.f2_taps, f->htaps.data(), sizeof(p.f2_taps));
                    p.job[v].f2_out = (float2*)f->out_ptr;
                    // the F2H stage-1 outputs in front of this chunk: the carry of the previous chunk's tail puts them at the
                    // head of this chunk's buffer and may not have run yet; they are the last ones of the previous chunk's
                    // [history | data], in the other buffer of a double-buffered stage
                    p.job[v].f2_hist = (const float2*)(f->dbl ? f->other_base() + (size_t)2 * f->prev_n_in : f->base());
                    p.job[v].f2_off = f->chunk_offset;
                    p.job[v].f2_n = f->n_out;
                }
            }
            pair_slots(p, &g[b], pair_conjugates);
            p.pfb_ps = 0; p.pfb_sigma = 1; p.taps_host = nullptr;
            if (s1_variant >= 7 && p.njobs >= 1) { pfb_grid(p, &g[b]); }
            // the tiled kernel pads every job to the group's QP: all jobs of a batch must have room for it
            int variant = s1_variant;
            for (int v = 0; v < p.njobs; v++) {
                if (g[b + v]->gpad_len < (p.D - 1) + (p.QP + 8) * p.D) { variant = 0; }
            }
            int nl = 0;
            bool tma = false, f2 = false;
            cudaEvent_t t1 = timer_begin(0, stream);
            cudaError_t e = launch_xlate_decim(p, fmt, variant, opts, stream, &nl, &tma, &f2);
            if (e != cudaSuccess) { return cuda_fail(e, "launch_xlate_decim"); }
            if (tma) { s1_tma_launches++; }
            // ÷4-epilogue bookkeeping: which (4, 27) stages stage 1 computed this chunk
            for (int v = 0; v < p.njobs; v++) {
                Chain* c = chain_of[g[b + v]];
                if (c->st.size() >= 2 && c->st[1]->kind == K_FIRC) { ((FirCStage*)c->st[1].get())->s1_fused = f2 && p.job[v].f2_out; }
                if (f2 && p.job[v].f2_out) { s1_f2_jobs++; }
            }
            if (t1) { B200_CK(cudaEventRecord(t1, stream)); }
            trace_mark("stage1 done", stream);
            e = launch_xd_edge(p, fmt, stream, &nl);
            if (e != cudaSuccess) { return cuda_fail(e, "launch_xd_edge"); }
            launches += nl;
        }
    }
    return 0;
}

// raw-IQ history for the next chunk's stage 1 (same stream as stage 1)
int Scheduler::carry_raw_hist(const void* raw, int fmt, int count) {
    CarryParams rc1;
    rc1.njobs = 1;
    CarryJob& j = rc1.job[0];
    j.dst = raw_hist.as<float>(); j.a = raw_hist.as<float>(); j.b = raw;
    j.h = RAW_HIST; j.la = RAW_HIST; j.lb = count; j.esize = 2; j.bfmt = fmt; j.scale = in_scale;
    cudaError_t e = launch_carry(rc1, opts, stream);
    if (e != cudaSuccess) { return cuda_fail(e, "launch_carry"); }
    launches++;
    return 0;
}

// ---- the launch list behind stage 1 ----
// k_dfir_reg: the short decimating FIRs with the window in registers; one batch shares D, T and the taps
static bool dfr_ok(const Stage* s, int pre_reg) {
    if (pre_reg <= 0 || s->kind != K_FIRC || s->in_es != 2) { return false; }
    const FirCStage* f = (const FirCStage*)s;
    return f->decim > 1 && f->ntaps <= DFR_MAXT && dfir_reg_supported(f->decim, f->ntaps);
}
static void dfr_push(LaunchRec& rec, Batch<DfrParams>& dfr, const FirCStage* f) {
    const FirJob& j0 = dfr.p.job[0];
    FirJob& j = dfr.next(rec, j0.decim != f->decim || j0.ntaps != f->ntaps || !std::equal(f->htaps.begin(), f->htaps.end(), dfr.p.taps));
    if (dfr.p.njobs == 1) { memcpy(dfr.p.taps, f->htaps.data(), (size_t)f->ntaps * sizeof(float)); }
    j.in = (const float2*)f->base(); j.out = (float2*)f->out_ptr; j.taps = f->taps.as<float>();
    j.ntaps = f->ntaps; j.decim = f->decim; j.offset = f->chunk_offset; j.n_out = f->n_out;
    dfr.done(rec, f->n_out, false);
}

// the register FIRs in front of fused chains: one launch per level and plan stage
static void rec_reg_firs(LaunchRec& rec, std::vector<Chain*>& chains, Batch<DfrParams>& dfr) {
    int max_beg = 1;
    for (Chain* c : chains) { if (c->fp.active) { max_beg = std::max(max_beg, c->fp.beg); } }
    for (int lvl = 1; lvl < max_beg; lvl++) {
        for (Chain* c : chains) {
            if (!c->fp.active || lvl >= c->fp.beg) { continue; }
            FirCStage* f = (FirCStage*)c->st[lvl].get();
            if (f->n_out <= 0 || f->s1_fused) { continue; }
            dfr_push(rec, dfr, f);
        }
        dfr.flush(rec);
    }
}

// fused tails: every FIR-like stage after stage 1 of a VFO in one launch (kernels.cuh: FtJob)
static void rec_fused_tails(LaunchRec& rec, std::vector<Chain*>& chains, const FuseCfg& fuse, int sm_count) {
    std::vector<Chain*> fc;
    for (Chain* c : chains) {
        if (c->fp.active && c->st[c->fp.beg]->n_in > 0) { fc.push_back(c); }
    }
    if (fc.empty()) { return; }
    // slab size: the fewest waves the largest slabs allow, then the smallest slab that keeps that wave count
    // (less halo-free work per CTA; the halo a slab recomputes is a fixed cost)
    const int threads = (fuse.threads == 512 || fuse.threads == 256) ? fuse.threads : 128;
    size_t smem = 0;
    int ob_cap = 1 << 30;
    for (Chain* c : fc) { smem = std::max(smem, c->fp.smem); ob_cap = std::min(ob_cap, c->fp.ob_max); }
    // resident CTAs per SM as the device will actually place them (registers bound the 256-thread build at two)
    static std::map<std::pair<int, size_t>, int> occ_cache;
    int cps;
    {
        auto key = std::make_pair(threads, smem);
        auto it = occ_cache.find(key);
        if (it == occ_cache.end()) { it = occ_cache.emplace(key, tail_fused_ctas_per_sm(threads, smem)).first; }
        cps = it->second;
    }
    if (cps < 1) { cps = std::max(1, std::min((int)((227 * 1024) / (smem + 1024)), 2048 / threads)); }
    const long long slots = (long long)sm_count * cps;
    auto total_slabs = [&](int ob) {
        long long t = 0;
        for (Chain* c : fc) { t += std::max(1, (c->st[c->fp.end - 1]->n_out + ob - 1) / ob); }
        return t;
    };
    int ob = ob_cap;
    if (fuse.ob_force <= 0) {
        const long long waves = (total_slabs(ob_cap) + slots - 1) / slots;
        int lo_ob = 4 * FT_R, hi_ob = ob_cap;           // smallest ob with total_slabs(ob) <= waves * slots
        while (lo_ob < hi_ob) {
            int mid = (lo_ob + hi_ob) / 2;
            if (total_slabs(mid) <= waves * slots) { hi_ob = mid; } else { lo_ob = mid + 1; }
        }
        ob = hi_ob;
    }
    Batch<FtParams> ft(launch_of_ft);
    ft.a = threads;
    ft.b = smem;
    for (Chain* c : fc) {
        FtJob& J = ft.next(rec);
        const int nst = c->fp.end - c->fp.beg;
        J.nst = nst;
        J.OB = ob;
        J.OT0 = c->fp.ot0;
        J.stg2 = c->fp.buf[0] + c->fp.stg2_rel; J.pad = 0;
        J.s0_direct = c->fp.s0_direct ? 1 : 0;
        J.stg3 = c->fp.buf[0] + 2 * c->fp.stg2_rel;
        J.nat_off = c->fp.nat_off;
        J.stg_floats = c->fp.stg2_rel;
        J.taps_nat = c->fp.s0_direct ? ((FirCStage*)c->st[c->fp.beg].get())->taps.as<float>() : nullptr;
        J.rds = nullptr; J.rds_phase0 = 0; J.rds_w = 0;
        for (int i = 0; i < nst; i++) {
            Stage* sg = c->st[c->fp.beg + i].get();
            FtStage& d = J.st[i];
            ft_describe(sg, d);
            d.n_in = sg->n_in; d.n_out = sg->n_out;
            d.buf = c->fp.buf[i]; d.pitch = c->fp.pitch[i]; d.tap_off = c->fp.tap_off[i]; d.qpitch = c->fp.qpitch[i];
            if (sg->kind == K_FIRC) { d.off = ((FirCStage*)sg)->chunk_offset; }
            if (sg->kind == K_POLY) { d.off = ((PolyStage*)sg)->chunk_offset; d.phase = ((PolyStage*)sg)->chunk_phase; }
            if (sg->kind == K_QUAD && ((QuadStage*)sg)->side) {
                const RxlStage* x = ((QuadStage*)sg)->side;
                J.rds = (float2*)x->out_ptr; J.rds_phase0 = x->chunk_phase0; J.rds_w = x->w;
            }
            if (i > 0) {
                d.hist_rd = sg->fh[sg->fpar].as<float>();
                d.hist_wr = sg->fh[sg->fpar ^ 1].as<float>();
                sg->fpar ^= 1;
            }
        }
        J.src = c->st[c->fp.beg]->base();
        J.out = c->st[c->fp.end - 1]->out_ptr;
        J.slabs = std::max(1, (J.st[nst - 1].n_out + ob - 1) / ob);
        ft.done(rec, 0);
    }
    ft.flush(rec);
}

// the remaining stages level by level: one launch per stage kind per level (batches of 16 VFOs)
static void rec_levels(LaunchRec& rec, std::vector<Chain*>& chains, int pre_reg, Batch<DfrParams>& dfr) {
    size_t depth = 0;
    for (Chain* c : chains) { depth = std::max(depth, first_level(c) + c->st.size()); }
    for (size_t lvl = 0; lvl < depth; lvl++) {
        Batch<FirParams> fpr(launch_of<FirParams, launch_fir_reg>, &FirParams::max_out);        // decimation-1 filters with register windows
        Batch<PolyParams> ppr(launch_of<PolyParams, launch_poly_reg>, &PolyParams::max_out);    // polyphase resamplers with register windows: one (L, M) per batch
        Batch<FirRParams> rpr(launch_of<FirRParams, launch_firr_reg>, &FirRParams::max_out);
        Batch<FirParams> fp(launch_of<FirParams, launch_fir_c>, &FirParams::max_out);
        Batch<PolyParams> pp(launch_of<PolyParams, launch_poly>, &PolyParams::max_out);
        Batch<QuadParams> qp(launch_of<QuadParams, launch_quad>, &QuadParams::max_n);
        Batch<FirRParams> rp(launch_of<FirRParams, launch_fir_r>, &FirRParams::max_out);
        Batch<SeqParams> sp(launch_of<SeqParams, launch_seq>);
        Batch<M2SParams> mp(launch_of<M2SParams, launch_m2s>, &M2SParams::max_n);
        Batch<ScaleParams> cp(launch_of<ScaleParams, launch_scale>, &ScaleParams::max_n);
        Batch<FmIfParams> fmp(launch_of<FmIfParams, launch_fmif>, &FmIfParams::max_n);         // one bin count per batch
        Batch<RxlParams> xlp(launch_of<RxlParams, launch_rxl>, &RxlParams::max_n);
        Batch<StParams> stp(launch_of_n<StParams, launch_stereo>, &StParams::max_n);
        Batch<SqParams> sqp(launch_of_n<SqParams, launch_squelch>, &SqParams::max_n);
        for (Chain* c : chains) {
            const size_t l0 = first_level(c);
            if (lvl < l0 || lvl - l0 >= c->st.size()) { continue; }
            if (c->fp.active && lvl >= 1 && (int)lvl < c->fp.end) { continue; }     // done by the fused launch
            Stage* s = c->st[lvl - l0].get();
            if (s->n_out <= 0) { continue; }
            switch (s->kind) {
            case K_XD: break;
            case K_FIRC: {
                FirCStage* f = (FirCStage*)s;
                if (f->s1_fused) { break; }
                if (dfr_ok(f, pre_reg)) { dfr_push(rec, dfr, f); break; }
                Batch<FirParams>& b = (pre_reg > 0 && f->decim == 1 && f->in_es == 2 && f->ntaps <= 2000 && f->chunk_offset == 0) ? fpr : fp;
                FirJob& j = b.next(rec);
                j.in = (const float2*)f->base(); j.out = (float2*)f->out_ptr; j.taps = f->taps.as<float>();
                j.ntaps = f->ntaps; j.decim = f->decim; j.offset = f->chunk_offset; j.n_out = f->n_out;
                b.done(rec, f->n_out);
                break;
            }
            case K_POLY: {
                PolyStage* f = (PolyStage*)s;
                const bool regp = pre_reg > 0 && f->in_es == 2 && f->tpp <= 512 && poly_reg_supported(f->interp, f->decim);
                Batch<PolyParams>& b = regp ? ppr : pp;
                PolyJob& j = b.next(rec, regp && (ppr.p.job[0].interp != f->interp || ppr.p.job[0].decim != f->decim));
                j.in = (const float2*)f->base(); j.out = (float2*)f->out_ptr; j.bank = f->bank.as<float>();
                j.tpp = f->tpp; j.interp = f->interp; j.decim = f->decim; j.phase0 = f->chunk_phase; j.offset0 = f->chunk_offset;
                j.n_out = f->n_out;
                j.bank_kl = f->bank_kl.as<float>(); j.in_len = (long long)f->hist + f->n_in;
                b.done(rec, f->n_out);
                break;
            }
            case K_QUAD: {
                QuadStage* f = (QuadStage*)s;
                QuadJob& j = qp.next(rec);
                j.in = (const float2*)f->base(); j.out = f->out_ptr;
                j.inv_dev = f->inv_dev; j.n = f->n_out;
                j.rds = f->side ? (float2*)f->side->out_ptr : nullptr;
                j.rds_phase0 = f->side ? f->side->chunk_phase0 : 0; j.rds_w = f->side ? f->side->w : 0;
                qp.done(rec, f->n_out);
                break;
            }
            case K_FIRR: {
                FirRStage* f = (FirRStage*)s;
                Batch<FirRParams>& b = (pre_reg > 0 && f->ntaps <= 2000) ? rpr : rp;
                FirRJob& j = b.next(rec);
                j.in = f->base(); j.out = f->out_ptr; j.taps = f->taps.as<float>();
                j.ntaps = f->ntaps; j.n_out = f->n_out; j.stereo = f->stereo;
                b.done(rec, f->n_out);
                break;
            }
            case K_SEQ: {
                SeqStage* f = (SeqStage*)s;
                SeqJob& j = sp.next(rec);
                j = f->proto;
                j.in = (const float2*)f->in_data(); j.out = f->out_ptr; j.state = f->state.as<float>(); j.n = f->n_out;
                sp.done(rec, f->n_out);
                break;
            }
            case K_SCALE: {
                ScaleJob& j = cp.next(rec);
                j.in = s->in_data(); j.out = s->out_ptr; j.n = s->n_out * s->in_es; j.gain = ((ScaleStage*)s)->gain;
                cp.done(rec, j.n);
                break;
            }
            case K_STEREO: {
                StereoStage* f = (StereoStage*)s;
                StJob& j = stp.next(rec);
                j.in = f->base(); j.out = (float2*)f->out_ptr; j.taps = f->taps.as<float2>(); j.p = f->p.as<float2>(); j.vco = f->vco.as<float2>();
                j.state = f->state.as<float>(); j.ntaps = f->ntaps; j.delay = f->delay; j.n = f->n_out;
                j.alpha = f->alpha; j.beta = f->beta; j.min_freq = f->min_freq; j.max_freq = f->max_freq;
                stp.done(rec, f->n_out);
                break;
            }
            case K_RXL: {
                RxlStage* f = (RxlStage*)s;
                if (c->parent && lvl == l0) { break; }      // an RDS branch's: its parent's discriminator stored it
                RxlJob& j = xlp.next(rec);
                j.in = f->in_data(); j.out = (float2*)f->out_ptr; j.n = f->n_out; j.phase0 = f->chunk_phase0; j.w = f->w;
                xlp.done(rec, f->n_out);
                break;
            }
            case K_FMIF: {
                FmIfStage* f = (FmIfStage*)s;
                FmIfJob& j = fmp.next(rec, fmp.p.job[0].bins != f->bins);
                j.in = (const float2*)f->base(); j.out = (float2*)f->out_ptr; j.win = f->win.as<float>(); j.tw = f->tw.as<float2>();
                j.n = f->n_out; j.bins = f->bins;
                fmp.done(rec, f->n_out);
                break;
            }
            case K_SQUELCH: {
                SquelchStage* f = (SquelchStage*)s;
                SqJob& j = sqp.next(rec);
                j.in = (const float2*)f->in_data(); j.out = (float2*)f->out_ptr; j.partial = f->partial.as<float>(); j.n = f->n_out; j.level = f->level;
                sqp.done(rec, f->n_out);
                break;
            }
            case K_M2S: {
                M2SJob& j = mp.next(rec);
                j.in = s->in_data(); j.out = s->out_ptr; j.n = s->n_out;
                mp.done(rec, s->n_out);
                break;
            }
            }
        }
        // the order of these launches is part of the plan: programmatic dependent launch overlaps each with the one before
        dfr.flush(rec); fpr.flush(rec); ppr.flush(rec); rpr.flush(rec); fp.flush(rec); pp.flush(rec); qp.flush(rec);
        rp.flush(rec); sp.flush(rec); mp.flush(rec); cp.flush(rec); fmp.flush(rec); xlp.flush(rec); stp.flush(rec); sqp.flush(rec);
    }
}

// history carry (the memmove at the end of every reference process())
static void rec_history_carry(LaunchRec& rec, std::vector<Chain*>& chains) {
    Batch<CarryParams> cp(launch_of<CarryParams, launch_carry>);
    for (Chain* c : chains) {
        for (auto& sp : c->st) {
            Stage* s = sp.get();
            if (s->kind == K_XD || s->hist <= 0 || s->fmid) { continue; }
            if (s->n_in <= 0 && !s->dbl) { continue; }      // a double-buffered stage always hands its history over
            CarryJob& j = cp.next(rec);
            memset(&j, 0, sizeof(j));
            j.dst = s->other_base(); j.a = s->base(); j.b = s->in_data();
            j.h = s->hist; j.la = s->hist; j.lb = s->n_in; j.esize = s->in_es; j.bfmt = -1; j.scale = 0.0f;
            cp.done(rec, 0);
        }
    }
    cp.flush(rec);
}

int Scheduler::run(std::vector<Chain*>& chains, const void* raw, int fmt, int count, bool carry_raw) {
    const long long hp0 = host_now_ns();
    const int parity = (int)(chunk_idx & 1);
    cudaStream_t ts = out_stream();
    int rc;
    if ((rc = wire(chains, parity)) || (rc = stage1(chains, raw, fmt, count))) { return rc; }
    if (carry_raw && count > 0 && (rc = carry_raw_hist(raw, fmt, count))) { return rc; }
    if (tail_stream) {
        B200_CK(cudaEventRecord(ev_stage1[parity], stream));
        B200_CK(cudaStreamWaitEvent(ts, ev_stage1[parity], 0));
    }
    trace_mark("tails start", ts);
    const long long hp1 = host_now_ns();
    host_ns[0] += hp1 - hp0;
    cudaEvent_t t_tail = timer_begin(1, ts);
    // Everything behind stage 1 goes into one launch list, then replays: as a captured CUDA graph when the same list was
    // seen before (one cudaGraphLaunch instead of seven to ten launches), else as plain launches.
    rec.clear();
    Batch<DfrParams> dfr(launch_of_dfr, &DfrParams::max_out);     // k_dfir_reg, in front of fused chains and in the levels
    rec_reg_firs(rec, chains, dfr);
    rec_fused_tails(rec, chains, fuse, sm_count);
    rec_levels(rec, chains, fuse.pre_reg, dfr);
    rec_history_carry(rec, chains);
    if ((rc = launch_recorded(ts, graph_tails > 0 || (graph_tails < 0 && count <= graph_max_count)))) { return rc; }
    if (t_tail) { B200_CK(cudaEventRecord(t_tail, ts)); }
    trace_mark("tails+carry done", ts);
    if (tail_stream) { B200_CK(cudaEventRecord(ev_tail[parity], ts)); }
    host_ns[1] += host_now_ns() - hp1;
    chunk_idx++;
    return 0;
}

}

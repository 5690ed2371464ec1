// sdrplusplus_b200/csrc/engine.h -- host runtime of libb200dsp: stages with carried state, chains,
// the per-chunk scheduler that batches the same stage of every VFO into one launch, and the FFT framer.
// The integer state (decimation offsets, polyphase phase, frame cursor) is mirrored on the host so every
// per-chunk output count is known without a device round trip.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <memory>
#include <mutex>
#include <string>
#include <vector>
#include <unordered_map>
#include "kernels.cuh"
#include "design.h"

namespace b200 {

// optional launch timeline (env B200_TRACE=1): an event after every launch group, dumped by trace_dump()
void trace_mark(const char* label, cudaStream_t s);
void trace_dump(const char* title);
bool trace_on();

void set_error(const char* fmt, ...);
const char* last_error();
int cuda_fail(cudaError_t e, const char* what);   // records message, returns B200_ECUDA
#define B200_CK(call)                                                     \
    do {                                                                  \
        cudaError_t _e = (call);                                          \
        if (_e != cudaSuccess) { return b200::cuda_fail(_e, #call); }     \
    } while (0)

struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    DevBuf() {}
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    int alloc(size_t n, bool zero = true);
    void release();
    template <class T> T* as() const { return (T*)p; }
};

enum StageKind { K_XD, K_FIRC, K_POLY, K_QUAD, K_FIRR, K_SEQ, K_M2S, K_SCALE, K_STEREO, K_SQUELCH, K_FMIF, K_RXL };

struct Stage {
    StageKind kind;
    int in_es = 2, out_es = 2;   // floats per input / output sample
    int hist = 0;                // history samples kept in front of the data in inbuf
    int cap_in = 0;              // max input samples per chunk
    DevBuf inbuf;                // [hist | data]; unused by K_XD (reads the shared raw IQ)
    DevBuf inbuf_alt;            // second buffer of the stage fed by stage 1 when tails overlap the next chunk
    bool dbl = false;
    int par = 0;                 // which buffer this chunk uses (dbl only)
    int n_in = 0, n_out = 0;     // this chunk
    float* out_ptr = nullptr;    // where this chunk's output goes (set by the scheduler)
    // fused tail (kernels.cuh: FtStage): an intermediate stage keeps only its history, ping-pong between chunks
    DevBuf fh[2];
    int fpar = 0;                // read fh[fpar], write fh[fpar ^ 1]
    bool fmid = false;
    int role = 0;                // which radio block a front-end VFO built this stage for (api.cpp: VfoRole); 0 = none
    DevBuf taps_pm;              // taps in the fused kernel's phase-major order: row r = taps[q*D + r], pitch ceil(T/D)
    int pm_floats = 0;           // multiple of 4
    int upload_pm(const std::vector<float>& t, int rows_per_set, int sets);
    virtual ~Stage() {}
    virtual int plan(int n) = 0;             // host: output count for n inputs, advances the mirrored state
    virtual int max_out(int n) const = 0;    // upper bound
    virtual void reset_state() {}
    float* base() const { return (dbl && par) ? inbuf_alt.as<float>() : inbuf.as<float>(); }
    float* other_base() const { return (dbl && !par) ? inbuf_alt.as<float>() : inbuf.as<float>(); }
    float* in_data() const { return base() + (size_t)hist * in_es; }
    int alloc_in(int cap);
};

struct XdStage : Stage {
    int D = 1, T = 1;
    std::vector<float> h;        // real taps of the first decimation stage ({1} for a pure translate)
    double offset_rad = 0.0;     // hzToRads(-vfoOffset, fs) as the reference passes it to the xlator
    unsigned long long phase = 0, w = 0;
    long long pos = 0;           // input samples consumed since the stream (or the last reset) began
    // Retunes still inside a tap window.  A sample keeps the rotation it was translated with: segment s covers the
    // samples from segs[s].start up to the next segment's start, with phase(i) = segs[s].phase + segs[s].w * (i - start).
    // The last segment is the current increment; a segment is dropped once T-1 samples lie past its successor's start.
    struct Seg { long long start; unsigned long long phase, w; };
    std::vector<Seg> segs;
    bool chunk_retuned = false;  // this chunk has outputs whose window starts before the newest boundary
    int chunk_edge_start = 0;    // newest boundary, chunk-relative (<= 0)
    std::vector<unsigned long long> edge_tab;   // phase of chunk-relative samples -(T-1) .. -1 (when chunk_retuned)
    DevBuf edge_ph;              // edge_tab on the device
    DevBuf hdev;                 // real taps on the device (retune edge kernel)
    int offset = 0;              // DecimatingFIR::offset
    DevBuf gpad;                 // complex taps, padded
    int gpad_len = 0;
    int QP = 1;
    bool taps_dirty = true;
    XdStage() { kind = K_XD; }
    void configure(int D_, const std::vector<float>& taps);
    void set_offset_rad(double rad);       // FrequencyXlator::setOffset: phase-continuous
    int upload_taps(cudaStream_t s);
    int plan(int n) override;
    int max_out(int n) const override { return (n + D - 1) / D + 1; }
    void reset_state() override { phase = 0; offset = 0; pos = 0; segs.assign(1, Seg{ 0, 0, w }); chunk_retuned = false; }
    unsigned long long chunk_phase0 = 0; int chunk_offset = 0;   // snapshot used by this chunk's launch
};

struct FirCStage : Stage {
    int ntaps = 1, decim = 1, offset = 0, chunk_offset = 0;
    int prev_n_in = 0;           // n_in of the previous chunk (where its last ntaps-1 inputs lie in the other buffer of a dbl stage)
    bool s1_fused = false;       // this chunk: stage 1 computed this stage's outputs (k_xd_tma's ÷4 epilogue)
    DevBuf taps;
    std::vector<float> htaps;    // host copy of the taps in use
    std::vector<float> pending;  // FIR::setTaps applied at the next chunk boundary
    FirCStage() { kind = K_FIRC; }
    int configure(const std::vector<float>& t, int decim_);
    int plan(int n) override;
    // one output more than plan() can give: with decim 1 the stage is 1:1 (the radio's 300 Hz high-pass), and the front end keeps a
    // VFO's bound the same when that filter is switched on or off (api.cpp: vfo_out_bound)
    int max_out(int n) const override { return (n + decim - 1) / decim + 1; }
    void reset_state() override { offset = 0; n_in = 0; prev_n_in = 0; }
};

struct PolyStage : Stage {
    int interp = 1, decim = 1, tpp = 1, phase = 0, offset = 0, chunk_phase = 0, chunk_offset = 0;
    DevBuf bank, bank_kl;        // [interp][tpp] and [tpp][interp]
    PolyStage() { kind = K_POLY; }
    int configure(int interp_, int decim_, const std::vector<float>& taps);
    int plan(int n) override;
    int max_out(int n) const override { return (int)(((long long)n * interp + decim - 1) / decim) + 2; }
    void reset_state() override { phase = 0; offset = 0; }
};

struct RxlStage;
struct QuadStage : Stage {
    float inv_dev = 1.0f;
    RxlStage* side = nullptr;    // first stage of a bound RDS branch (b200_fe_bind_rds): this discriminator computes its output
    QuadStage() { kind = K_QUAD; out_es = 1; hist = 1; }   // history = the previous chunk's last sample (Quadrature::phase)
    int configure(double deviationHz, double samplerate);
    int plan(int n) override { n_in = n; n_out = n; return n; }
    int max_out(int n) const override { return n; }
};

struct FirRStage : Stage {
    int ntaps = 1, stereo = 0;
    DevBuf taps;
    FirRStage() { kind = K_FIRR; in_es = 1; out_es = 1; }
    int configure(const std::vector<float>& t, bool stereo_);
    int plan(int n) override { n_in = n; n_out = n; return n; }
    int max_out(int n) const override { return n; }
};

struct SeqStage : Stage {
    SeqJob proto;                // coefficients; pointers filled per chunk
    DevBuf state;
    float init_state[SEQ_STATE_FLOATS];
    SeqStage() { kind = K_SEQ; out_es = 1; }
    int configure_am(int agcMode, double attack, double decay, double dcRate);
    int configure_ssb(int mode, double bandwidth, double samplerate, double attack, double decay);
    int configure_deemph(double tau, double samplerate);
    int configure_noise_blanker(double rate, double level);               // complex in, complex out
    // the reference's coefficient setters: the device state (AGC amplitude, DC offset, de-emphasis output, blanker amplitude)
    // is left alone, the next launch carries the new coefficient
    void set_agc(double attack, double decay);                            // AGC::setAttack / setDecay (agc.h:32-44)
    void set_deemph_tau(double tau, double samplerate);                   // Deemphasis::setTau (deephasis.h:31-36,91-94)
    int plan(int n) override { n_in = n; n_out = n; return n; }
    int max_out(int n) const override { return n; }
};

struct M2SStage : Stage {
    M2SStage() { kind = K_M2S; in_es = 1; out_es = 2; }
    int plan(int n) override { n_in = n; n_out = n; return n; }
    int max_out(int n) const override { return n; }
};

// Static part of a chain's fused-tail launch: which stages, the shared-memory arena, the slab size limit.
struct FusedPlan {
    bool active = false;
    int beg = 1;                 // stages [1, beg): short decimating FIRs run by k_dfir_reg in front of the fused launch
    int end = 0;                 // stages [beg, end) run in k_tail_fused
    int ob_max = 0, ot0 = 0, stg2_rel = 0;
    bool s0_direct = false;      // first fused stage filters the raw stream from a cp.async.bulk ring (kernels.cuh: FtJob)
    int nat_off = 0;
    size_t smem = 0;
    int buf[FT_MAXST], pitch[FT_MAXST], tap_off[FT_MAXST], qpitch[FT_MAXST];
};
struct FuseCfg { bool on = false; int ob_max = 1280; int smem_limit = 110 * 1024; int threads = 256; int ob_force = 0; bool direct = true; int pre_reg = 8; bool reg_all = true; };   // pre_reg: how many short decimating FIR stages may run in registers in front of the fused launch; reg_all: chains whose every stage has a register-window kernel are not fused at all

// stereo branch of BroadcastFM behind the discriminator (broadcast_fm.h:147-177): mono multiplex in, (l, r) out
struct StereoStage : Stage {
    int ntaps = 1, delay = 0;
    float alpha = 0, beta = 0, min_freq = 0, max_freq = 0, init_freq = 0;
    DevBuf taps, p, vco, state;
    StereoStage() { kind = K_STEREO; in_es = 1; out_es = 2; }
    int configure(double samplerate);
    int plan(int n) override { n_in = n; n_out = n; return n; }
    int max_out(int n) const override { return n; }
    void reset_state() override;
};

// noise_reduction::PowerSquelch (power_squelch.h:33-50) between the VFO and the demodulator (radio IF chain)
struct SquelchStage : Stage {
    float level = -50.0f;
    DevBuf partial;
    SquelchStage() { kind = K_SQUELCH; in_es = 2; out_es = 2; }
    int plan(int n) override { n_in = n; n_out = n; return n; }
    int max_out(int n) const override { return n; }
};

// RealToComplex + FrequencyXlator in one pass (the RDS branch of BroadcastFM, broadcast_fm.h:165-170): real in, complex out,
// closed-form phase like stage 1 (the angle of the reference's fp32-rounded phaseDelta, exact u64 accumulation)
struct RxlStage : Stage {
    unsigned long long w = 0, phase = 0, chunk_phase0 = 0;
    RxlStage() { kind = K_RXL; in_es = 1; out_es = 2; }
    void set_offset_rad(double rad);
    int plan(int n) override { n_in = n; n_out = n; chunk_phase0 = phase; phase += w * (unsigned long long)(long long)n; return n; }
    int max_out(int n) const override { return n; }
    void reset_state() override { phase = 0; }
};

// noise_reduction::FMIF (fm_if.h:44-77): history = bins - 1 samples, one transform per output sample (ifnr.cuh)
struct FmIfStage : Stage {
    int bins = 32;
    DevBuf win, tw;
    FmIfStage() { kind = K_FMIF; in_es = 2; out_es = 2; }
    int configure(int nbins);
    int plan(int n) override { n_in = n; n_out = n; return n; }
    int max_out(int n) const override { return n; }
};

struct ScaleStage : Stage {
    float gain = 1.0f;
    ScaleStage(int es, float g) { kind = K_SCALE; in_es = es; out_es = es; gain = g; }
    int plan(int n) override { n_in = n; n_out = n; return n; }
    int max_out(int n) const override { return n; }
};

// A chain = one VFO (+ demodulator) or one stand-alone block.
struct Chain {
    std::vector<std::unique_ptr<Stage>> st;
    DevBuf out;                  // final output of the chain
    int out_es = 2;
    int out_cap = 0;
    int n_out = 0;               // this chunk
    float* out_override = nullptr;   // this chunk: final stage writes straight into the caller's device buffer
    bool raw_input() const { return !st.empty() && st[0]->kind == K_XD; }
    // an RDS branch bound to a WFM VFO (b200_fe_bind_rds): `parent`'s discriminator writes what st[0] (RxlStage) would, so
    // st[0] launches nothing and st[i] runs at level quad_index() + i of the parent.  The scheduler takes the branch right
    // behind its parent in the chain list.
    const Chain* parent = nullptr;
    int quad_index() const;      // index of the discriminator stage, -1 when there is none
    int chan_fir = -1;           // stage index of RxVFO's channel filter (rx_vfo.h:28-31), set by add_rxvfo
    FusedPlan fp;
    FuseCfg fcfg;
    int plan_fused();            // (re)builds fp from the stage list; clears fp.active when the chain cannot be fused
    int finalize(int max_in, bool dbl_first = false, const FuseCfg* fuse = nullptr);    // allocates stage buffers for chunks of up to max_in samples
    int plan(int n);             // all stages; returns final count
    int max_out(int n) const;
    int peek(int n) const;       // output count Chain::plan(n) would return, without moving any state (FIR-only chains; else -1)
    void reset_state();
    // Blocks switched on or off between chunks (chain::setBlockEnabled): with the device idle the caller calls unfuse_history(),
    // edits `st` in place (a 1:1 stage of the same sample size in or out; a stage that stays keeps its buffers), then
    // restage().  A fused-middle stage keeps its history in fh[fpar], every other stage in front of its inbuf data:
    // unfuse_history() copies the former into the latter for every stage, restage() rebuilds the fused plan and copies it back
    // for the stages the new plan fuses.
    int unfuse_history();
    int restage();
    // builders (reference block -> stage list)
    int add_rxvfo(double inSR, double outSR, double bw, double offset);     // rx_vfo.h:17-31
    int add_xlator(double offsetHz, double samplerate);
    int add_power_decim(int ratio);                                         // power_decimator.h:92-110
    int add_resampler(double inSR, double outSR);                           // rational_resampler.h:120-165
    int add_fir_c(const std::vector<float>& taps, int decim);
    int add_fir_r(const std::vector<float>& taps, bool stereo);
    int add_quad(double deviationHz, double samplerate);
    int add_wfm(double deviationHz, double samplerate, bool lowPass, bool stereo = false);   // broadcast_fm.h:36-52,144-212
    int add_nfm(double samplerate, double bandwidth, bool lowPass);         // fm.h:24-40
    int add_am(int agcMode, double bandwidth, double attack, double decay, double dcRate, double samplerate); // am.h:28-45
    int add_ssb(int mode, double bandwidth, double samplerate, double attack, double decay); // ssb.h:22-35
    int add_deemph(double tau, double samplerate);                          // filter::Deemphasis<stereo_t> (deephasis.h:14-28)
    // radio AF chain: RationalResampler<stereo_t> -> [300 Hz high-pass FIR] -> [Deemphasis]  (radio_module.h:99-110,546-553)
    int add_af_chain(double afSamplerate, double audioSamplerate, bool highPass, double deemphTau);
    int add_af_highpass(double audioSamplerate);                            // taps::highPass(300, 100, audioSR) (radio_module.h:597-598)
    int add_wfm_rds(double deviationHz, double samplerate);                 // BroadcastFM's RDS branch: discriminator -> -57 kHz -> 5 kS/s (broadcast_fm.h:52-53,165-170)
    int add_rds_branch(double samplerate);                                  // the part behind the discriminator: -57 kHz -> 5 kS/s
    int add_noise_blanker(double rate, double level);                       // noise_reduction::NoiseBlanker (noise_blanker.h:12-17)
    int add_fmif(int bins);                                                 // noise_reduction::FMIF (fm_if.h:20-24)
    int add_squelch(double level);                                          // noise_reduction::PowerSquelch (power_squelch.h:16-20)
    int add_volume(double volume, bool muted);                              // dsp::audio::Volume (volume.h:13-17,39-42)
};

// block::reset of one stage: delay lines, fused history, mirrored counters and device state back to a fresh block's.  Memsets on
// the legacy stream: the caller synchronises the device before the library's streams go on.
void clear_stage_state(Stage& s);

// Launch list of everything behind stage 1 of one chunk (parameter blocks by value).  Small chunks are launch-bound: the
// list is hashed, and a chunk whose list was seen before replays a captured CUDA graph (one cudaGraphLaunch instead of
// seven to ten kernel launches).  Decimation offsets / resampler phases / buffer parities make the list periodic over a few
// chunks for any fixed chunk size, so a handful of graphs covers a stream.
struct LaunchRec {
    struct Item;
    // a typed launch function behind a type-erased pointer (engine.cpp: launch_of); *nl = the kernels it enqueued
    typedef cudaError_t (*Launch)(const void* params, const Item& it, const KernelOpts& o, cudaStream_t s, int* nl);
    struct Item { Launch fn; size_t off, size; int a; size_t b; };    // a, b: launch arguments outside the parameter block
    std::vector<Item> items;
    std::vector<unsigned char> bytes;
    void clear() { items.clear(); bytes.clear(); }
    void add(Launch fn, const void* p, size_t size, int a = 0, size_t b = 0);
    unsigned long long hash() const;
    int replay(const KernelOpts& o, cudaStream_t s, long long* nlaunch) const;     // the real launches, in order
};

// Runs a set of chains over one chunk: stage-1 launches grouped by decimation, then level by level one
// launch per stage kind, then the history carry.
struct Scheduler {
    // the kernel choices of the handle that owns this scheduler (a front end's two schedulers share its one instance)
    const KernelOpts& opts;
    explicit Scheduler(const KernelOpts& o) : opts(o) {}
    cudaStream_t stream = nullptr;
    // overlapped mode: stage 1 (+ raw history carry) runs on `stream`, every later stage on `tail_stream`, so the
    // tails of chunk k overlap stage 1 of chunk k+1.  The stage fed by stage 1 is double-buffered (Stage::dbl).
    cudaStream_t tail_stream = nullptr;
    cudaEvent_t ev_stage1[2] = { nullptr, nullptr }, ev_tail[2] = { nullptr, nullptr };
    unsigned long long chunk_idx = 0;
    cudaStream_t out_stream() const { return tail_stream ? tail_stream : stream; }
    int enable_overlap(cudaStream_t tail);
    long long launches = 0;
    long long s1_f2_jobs = 0;    // VFO-chunks whose (4, 27) stage stage 1 computed (k_xd_tma's ÷4 epilogue; b200_fe_stat "s1_f2_jobs")
    long long s1_tma_launches = 0;   // stage-1 launches that ran k_xd_tma (b200_fe_stat "s1_tma_launches")
    // CUDA graphs of the launch list (LaunchRec): -1 = for chunks up to graph_max_count samples, 0 = never (plain replay), 1 = always
    int graph_tails = -1;
    int graph_max_count = 1 << 30;
    struct GraphEntry { cudaGraphExec_t exec = nullptr; long long launches = 0; std::vector<unsigned char> key; };
    std::unordered_map<unsigned long long, GraphEntry> graphs;
    LaunchRec rec;
    long long graph_hits = 0, graph_misses = 0;
    void drop_graphs();
    int launch_recorded(cudaStream_t ts, bool may_graph);
    long long host_ns[4] = { 0, 0, 0, 0 };   // host time of run(): [0] wiring + stage 1, [1] everything behind it (b200_fe_stat)
    int s1_variant = 8;          // 8: filter-bank stage 1 fed by the TMA engine (cf32 chunks), 7: cp.async filter bank, when the VFO plan allows it; else 6
    FuseCfg fuse;                // tails: one fused launch per <= 16 VFOs instead of one launch per stage kind
    int sm_count = 132;
    float in_scale = 1.0f / 32768.0f;   // integer raw formats of this chunk: sample = (float)x * in_scale (set by the caller)
    bool pair_conjugates = true;   // stage 1: VFOs at +f / -f share their multiply-accumulates (exact identity)
    // optional device-side timing (bench.py's roofline legs): CUDA events around a launch group on the stream it runs on.
    // group 0 = stage 1 (stream), 1 = everything behind stage 1 of a chunk: register FIRs, fused tail, carries (tail stream),
    // 2 = the spectrum branch of a chunk (its own stream; recorded by the front end), 3 = the IQ taps of a chunk (their own
    // stream; recorded by the front end).  At most TIMER_MAX samples per group.
    bool time_s1 = false;
    static const size_t TIMER_MAX = 512;
    struct Timer { std::vector<cudaEvent_t> ev; size_t used = 0; };
    Timer timers[4];
    cudaEvent_t timer_begin(int group, cudaStream_t s);      // returns the stop event to record, nullptr when off / full
    int group_stats(int group, double* ms_total, int* launches);   // synchronises the recorded events, then clears them
    int s1_stats(double* ms_total, int* launches) { return group_stats(0, ms_total, launches); }
    ~Scheduler();
    DevBuf raw_hist;             // last RAW_HIST samples of the raw IQ stream (cf32)
    static const int RAW_HIST = 1024;
    static const int STAGE_SPARE = 72;  // samples past the data of a stage buffer that vector loads may touch (k_dfir_reg)
    int init_raw();
    // raw: device pointer to the chunk (format fmt) for chains with raw_input(); typed chains were fed by
    // copying into st[0]->in_data() beforehand.  counts were planned already (Chain::plan).
    int run(std::vector<Chain*>& chains, const void* raw, int fmt, int count, bool carry_raw);
    // the steps of run() in front of the launch list: output pointers and tap uploads, stage 1, the raw-IQ history carry
    int wire(std::vector<Chain*>& chains, int parity);
    int stage1(std::vector<Chain*>& chains, const void* raw, int fmt, int count);
    int carry_raw_hist(const void* raw, int fmt, int count);
    int apply_deferred(std::vector<Chain*>& chains);   // pending FIR taps; call before Chain::plan()
    int reset_raw();
};

}

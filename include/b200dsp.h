/*
 * include/b200dsp.h -- C ABI of libb200dsp.so: SDR++'s per-block streaming DSP hot path
 * (windowed FFT -> dB line; multi-VFO xlate -> decimate -> resample -> FIR -> demodulate)
 * as hand-written sm_90a (H100) CUDA kernels.
 *
 * The reference has no binary boundary at block level: dsp blocks are header-only C++
 * templates whose contract is `int process(int count, const I* in, O* out)` / `run()` /
 * `dsp::stream<T>` (core/src/dsp/processor.h:7-73, core/src/dsp/stream.h:25-141).  This
 * library sits UNDER that contract: the adapter headers in sdrplusplus_b200/host/dsp/ keep
 * the reference's class names and signatures and forward process() to the entry points
 * below (INTEGRATION.md shows the binding a maintainer adds to core/CMakeLists.txt).
 * Each entry point cites the reference interface it replaces.
 *
 * Conventions: plain pointers and sizes only; complex samples are interleaved (re, im)
 * float pairs == dsp::complex_t, audio is (l, r) == dsp::stereo_t (core/src/dsp/types.h).
 * Every function returns >= 0 on success and a negative B200_E* code on failure, never
 * throws, and records a message retrievable with b200_last_error().  There is NO CPU
 * fallback: without a usable CUDA device every compute call fails with B200_ENODEV.
 * Handles are thread-confined (one worker thread per block, like the reference,
 * core/src/dsp/block.h:71-73); setters may be called from another thread and take effect
 * at the next chunk boundary (the reference applies them under ctrlMtx between run()
 * iterations, core/src/dsp/channel/rx_vfo.h:72-77).
 */
#ifndef B200DSP_H
#define B200DSP_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_VERSION 100

/* error codes */
#define B200_OK        0
#define B200_EINVAL   (-1)   /* bad argument */
#define B200_ENODEV   (-2)   /* no CUDA device / driver: the product path refuses to run */
#define B200_ECUDA    (-3)   /* CUDA runtime error (message in b200_last_error) */
#define B200_ENOMEM   (-4)
#define B200_ECAP     (-5)   /* caller buffer too small / chunk larger than configured maximum */
#define B200_ENOPLAN  (-6)   /* decimation plan table not loaded / ratio unsupported */
#define B200_ESTATE   (-7)   /* call sequence error (e.g. wait without submit) */

/* sample formats of the IQ input */
#define B200_FMT_CF32  0     /* dsp::complex_t, 8 B/sample */
#define B200_FMT_CS16  1     /* int16 I,Q; x/32768 (file_source, source_modules/file_source/src/main.cpp:158-162) */
#define B200_FMT_CS8   2     /* int8 I,Q; x/128 (dsp/compression/sample_stream_decompressor.h PCM_TYPE_I8) */

/* where a caller buffer lives */
#define B200_MEM_HOST   0
#define B200_MEM_DEVICE 1

/* FFT windows: IQFrontEnd::FFTWindow (core/src/signal_path/iq_frontend.h:13-17) */
#define B200_WIN_RECTANGULAR 0
#define B200_WIN_BLACKMAN    1
#define B200_WIN_NUTTALL     2

/* demodulators: decoder_modules/radio/src/demodulators/{raw,wfm,nfm,am,usb,lsb,dsb}.h */
#define B200_DEMOD_RAW  0    /* VFO output itself (complex_t)            -- channel::RxVFO          */
#define B200_DEMOD_WFM  1    /* demod::BroadcastFM (mono branch)         -- broadcast_fm.h:192-212  */
#define B200_DEMOD_NFM  2    /* demod::FM<stereo_t>                      -- fm.h:79-96              */
#define B200_DEMOD_AM   3    /* demod::AM<stereo_t>                      -- am.h:101-133            */
#define B200_DEMOD_USB  4    /* demod::SSB<stereo_t> Mode::USB           -- ssb.h:77-92             */
#define B200_DEMOD_LSB  5
#define B200_DEMOD_DSB  6
#define B200_DEMOD_WFM_RDS    8  /* the RDS branch of demod::BroadcastFM instead of audio: discriminator -> RealToComplex -> FrequencyXlator(-57 kHz) ->
                                  * RationalResampler to 5 kS/s (broadcast_fm.h:52-53,165-170,196-202); output = complex_t at 5 kS/s, what
                                  * decoder_modules/radio/src/rds_demod.h consumes */
#define B200_DEMOD_WFM_STEREO 7  /* demod::BroadcastFM stereo branch: pilot filter + PLL + L-R recovery -- broadcast_fm.h:147-190 */
#define B200_DEMOD_WFM_RDS_BITS 9  /* the B200_DEMOD_WFM_RDS chain followed by RDSDemod (decoder_modules/radio/src/rds_demod.h:64-73, the
                                    * b200_rds_demod_* block below) inside the front end: output = one b200_rds_symbol per recovered
                                    * symbol.  The symbol count depends on the recovered clock: vfo_count of such a VFO is filled by
                                    * b200_fe_wait (b200_fe_process, b200_shard_wait), valid when it returns like the data, so the
                                    * b200_outputs given to b200_fe_submit must stay alive until that wait.  vfo_cap counts records and
                                    * b200_fe_vfo_max_out bounds them (b200_rds_demod_max_out of the 5 kS/s samples); records past
                                    * vfo_count are unspecified.  AF chain, volume and audio fields are ignored as for mode 8; the IF
                                    * chain (blanker, squelch, FM IF noise reduction) applies as for mode 8. */

/* one recovered RDS symbol: RDSDemod::soft and the differentially decoded bit of RDSDemod::out (0 or 1); 8 bytes, the element
 * size of every other VFO output (complex_t, stereo_t) */
typedef struct {
    float    soft;
    uint32_t bit;
} b200_rds_symbol;

#define B200_AGC_CARRIER 0   /* demod::AM::AGCMode (am.h:14-17) */
#define B200_AGC_AUDIO   1

#define B200_MAX_VFOS 64

/* ------------------------------------------------------------------------------------------
 * Library / device
 * ------------------------------------------------------------------------------------------ */

/* Select the CUDA device for the calling thread's handles.  B200_ENODEV when no device. */
int b200_init(int device);
int b200_device_count(void);
const char* b200_last_error(void);
int b200_version(void);

/* Power-of-two pre-decimation plans (stage decimations + FIR coefficient tables).  The
 * reference keeps them in dsp::multirate::decim::plans (core/src/dsp/multirate/decim/plans.h:124-139);
 * an adapter built against the reference headers registers them verbatim with
 * b200_register_decim_plan(); standalone users load the flat table shipped in
 * sdrplusplus_b200/data/decim_plans.bin (default location resolved next to the library,
 * or $B200_DECIM_PLANS) -- done lazily on first use. */
int b200_register_decim_plan(int ratio, int nstages, const int* decimations, const int* tapcounts,
                             const float* const* taps);
int b200_load_decim_plans(const char* path /* NULL = default */);

/* ------------------------------------------------------------------------------------------
 * Host-side design helpers (fp64 -> fp32, identical formulas to the reference; exposed so that
 * the parity tests can compare them bit-for-bit and so that adapters need not duplicate them)
 * ------------------------------------------------------------------------------------------ */
/* dsp::taps::lowPass (core/src/dsp/taps/low_pass.h:7-11): returns tap count, writes min(count,cap) */
int b200_taps_lowpass(double cutoff, double transWidth, double samplerate, int oddTapCount, float* out, int cap);
/* dsp::taps::highPass (core/src/dsp/taps/high_pass.h:7-14) */
int b200_taps_highpass(double cutoff, double transWidth, double samplerate, int oddTapCount, float* out, int cap);
/* dsp::taps::bandPass<complex_t> (core/src/dsp/taps/band_pass.h:11-26): returns the tap count, writes min(count,cap) taps as
 * interleaved (re, im) pairs */
int b200_taps_bandpass(double bandStart, double bandStop, double transWidth, double samplerate, int oddTapCount,
                       float* out_iq, int cap);
/* IQFrontEnd::updateFFTPath window (core/src/signal_path/iq_frontend.cpp:281-291): w(i,nz)*(-1)^i */
int b200_window(int window, int nz, float* out);
/* IQFrontEnd::genReshapeParams (core/src/signal_path/iq_frontend.h:59-63) */
int b200_fft_frame_params(double samplerate, int fftSize, double fftRate, int* nz, int* skip);

typedef struct {
    int mode;            /* 0 BOTH, 1 DECIM_ONLY, 2 RESAMP_ONLY, 3 NONE (rational_resampler.h:112-117) */
    int predec_ratio;    /* 1 when the power decimator is bypassed */
    int nstages;         /* pre-decimation stages */
    int stage_decim[8];
    int stage_taps[8];
    int interp, decim;   /* polyphase L / M */
    int ntaps;           /* prototype taps */
    int taps_per_phase;
} b200_resamp_plan;
/* dsp::multirate::RationalResampler::reconfigure (rational_resampler.h:120-165) */
int b200_resamp_plan_get(double inSamplerate, double outSamplerate, b200_resamp_plan* plan);

/* ------------------------------------------------------------------------------------------
 * Front end: one IQ stream -> { FFT/waterfall branch, N x (RxVFO + demodulator) }
 * Replaces IQFrontEnd's Splitter fan-out + Reshaper/handler FFT branch + per-VFO RxVFO blocks
 * (core/src/signal_path/iq_frontend.h:23-49, iq_frontend.cpp:248-309) and the radio module's
 * demodulator block behind each VFO (decoder_modules/radio/src/radio_module.h:80-125).
 * One b200_fe_process() call == one IQ chunk == what the reference moves with one
 * stream<complex_t>::swap(count); the raw IQ is read from HBM once for all consumers.
 * ------------------------------------------------------------------------------------------ */
typedef struct b200_fe b200_fe;

typedef struct {
    double offset;            /* Hz, VFO centre relative to the stream centre (RxVFO::init offset)       */
    double out_samplerate;    /* RxVFO output rate == demodulator IF rate (e.g. WFM 250000)              */
    double bandwidth;         /* channel filter bandwidth (RxVFO::init bandwidth)                        */
    int    demod;             /* B200_DEMOD_*                                                            */
    /* demodulator parameters (unused ones ignored) */
    double deviation;         /* WFM: Hz (wfm.h:78 passes bandwidth/2); NFM uses bandwidth/2 (fm.h:28)  */
    int    low_pass;          /* WFM/NFM post-demod audio low-pass enabled (wfm.h:364, nfm.h)            */
    int    agc_mode;          /* AM: B200_AGC_*                                                          */
    double agc_attack;        /* AM/SSB: per-sample coefficient (radio passes attack/IFrate)             */
    double agc_decay;
    double dc_block_rate;     /* AM: per-sample rate (radio passes 100/IFrate, demodulators/am.h:34)     */
    /* optional radio AF chain behind the demodulator (decoder_modules/radio/src/radio_module.h:99-110,546-553):
     * RationalResampler<stereo_t> out_samplerate -> af_samplerate, 300 Hz high-pass FIR, Deemphasis.          */
    double af_samplerate;     /* 0 = no AF chain (output at out_samplerate); e.g. 48000                      */
    int    af_high_pass;      /* taps::highPass(300, 100, af_samplerate)                                     */
    double af_deemph_tau;     /* seconds, 0 = off (50e-6 EU / 75e-6 US, radio_module.h deempTaus)            */
    /* dsp::audio::Volume at the very end (core/src/dsp/audio/volume.h:13-17,39-42): out = in * (muted ? 0 : powf(volume, 2)) */
    int    af_volume_on;      /* 0 = no volume block                                                         */
    int    af_muted;
    double af_volume;
    /* radio IF chain between the VFO and the demodulator (decoder_modules/radio/src/radio_module.h:88-96): power squelch,
     * noise_reduction::PowerSquelch (core/src/dsp/noise_reduction/power_squelch.h:33-50): a chunk whose mean amplitude is
     * below squelch_level dB is zeroed before it reaches the demodulator */
    int    squelch_on;
    double squelch_level;
    /* the other two blocks of that IF chain, in the reference's order noise blanker -> squelch -> FM IF noise reduction:
     * noise_reduction::NoiseBlanker (core/src/dsp/noise_reduction/noise_blanker.h:12-17,38-57) with the radio's rate
     * 500 / out_samplerate (radio_module.h:526), and noise_reduction::FMIF (fm_if.h:20-24,44-77) with nr_bins bins
     * (the radio's presets: 9, 15, 31, 32; radio_module.h:31-36; 2 ... 64 accepted) */
    int    nb_on;
    double nb_level;
    int    nr_on;
    int    nr_bins;
} b200_vfo_cfg;

typedef struct {
    /* per VFO: caller buffer for this chunk's output (stereo_t pairs, complex_t for RAW / WFM_RDS, b200_rds_symbol for WFM_RDS_BITS) */
    void* vfo_out[B200_MAX_VFOS];
    int   vfo_cap[B200_MAX_VFOS];     /* capacity in output samples                               */
    int   vfo_count[B200_MAX_VFOS];   /* OUT: samples produced this chunk (WFM_RDS_BITS: set by b200_fe_wait) */
    /* FFT branch: dB lines completed during this chunk, fft_size floats each                     */
    float* fft_out;
    int   fft_cap_lines;
    int   fft_lines;                  /* OUT                                                       */
    int   out_mem;                    /* B200_MEM_HOST (pinned preferred) or B200_MEM_DEVICE       */
} b200_outputs;

/* samplerate: effective IQ rate; max_chunk: largest count ever passed to process (the reference caps a
 * chunk at STREAM_BUFFER_SIZE = 1e6 samples, core/src/dsp/stream.h:9; stream<T>::setBufferSize raises it) */
b200_fe* b200_fe_create(double samplerate, int max_chunk);
void     b200_fe_destroy(b200_fe* fe);
/* run on the caller's CUDA stream (cudaStream_t passed as void*), e.g. torch's current stream; NULL = own */
int b200_fe_set_stream(b200_fe* fe, void* cuda_stream);

/* IQFrontEnd::setFFTSize/Rate/Window (iq_frontend.h:37-39); size 0 disables the branch. size must be a
 * power of two in [8, 4194304]. */
int b200_fe_set_fft(b200_fe* fe, int size, double rate, int window);
/* IQFrontEnd's pre-processing chain in front of the FFT branch and every VFO (core/src/signal_path/iq_frontend.cpp:32-39):
 * PowerDecimator -> correction::DCBlocker<complex_t> (rate 50 / effective samplerate, iq_frontend.h:55-57) -> math::Conjugate;
 * all off by default like the reference's.  setDecimation (iq_frontend.cpp:100-115): ratio = power of two <= 8192; it
 * changes the effective sample rate (samplerate / ratio) every later setting is interpreted with, so it must come before
 * b200_fe_set_fft / b200_fe_add_vfo.  setDCBlocking / setInvertIQ (:117-123) may change between chunks. */
int b200_fe_set_decimation(b200_fe* fe, int ratio);
int b200_fe_set_dc_blocking(b200_fe* fe, int enabled);
int b200_fe_set_invert_iq(b200_fe* fe, int enabled);
/* IQFrontEnd::addVFO / removeVFO (iq_frontend.h:32-33) + radio demodulator selection: returns vfo id */
int b200_fe_add_vfo(b200_fe* fe, const b200_vfo_cfg* cfg);
int b200_fe_remove_vfo(b200_fe* fe, int id);
/* RxVFO::setOffset / setBandwidth (core/src/dsp/channel/rx_vfo.h:60-77): phase-continuous, next chunk */
int b200_fe_set_vfo_offset(b200_fe* fe, int id, double offset);
int b200_fe_set_vfo_bandwidth(b200_fe* fe, int id, double bandwidth);
/* radio_module.h setters: the VFO takes cfg at the next chunk boundary, keeping state as the reference's setters do.
 * Checked whole at the call (B200_EINVAL leaves the VFO as it was), stored, and applied by the first submit / process after
 * it; of several calls before one chunk the last wins.  offset / bandwidth: as b200_fe_set_vfo_offset / _bandwidth -- and, the
 * last call winning, a cfg.offset / cfg.bandwidth equal to the VFO's applied value cancels an earlier set_vfo_offset / _bandwidth.
 * Coefficients keep the block's state: af_volume, af_muted, squelch_level, nb_level, agc_attack, agc_decay, dc_block_rate
 * (AM), af_deemph_tau non-zero -> non-zero.  agc_mode (AM) restarts the AM demodulator's AGCs and DC blocker, nr_bins the
 * FM IF noise reduction.  nb_on, squelch_on, nr_on, af_high_pass, af_deemph_tau 0 <-> non-zero and af_volume_on switch a
 * block on or off (chain::setBlockEnabled): the other blocks keep their state, a block switched off keeps its own and goes
 * on from it when switched on again (b200_fe_reset clears it).  demod, out_samplerate, deviation, low_pass and
 * af_samplerate need a new demodulator: B200_EINVAL (remove the VFO and add it again).  Output counts never change. */
int b200_fe_set_vfo_config(b200_fe* fe, int id, const b200_vfo_cfg* cfg);
/* IQFrontEnd::bindIQStream / unbindIQStream (core/src/signal_path/iq_frontend.h:34-35, iq_frontend.cpp:132-139): an IQ tap
 * delivers the effective stream -- the chunk behind the pre-processing chain (decimator -> DC blocker -> conjugate), what the
 * FFT branch and the VFOs read -- in one of the sample types below, interleaved I, Q.  Bytes per complex sample: CF32 8,
 * U8 2, I8 2, I16 4, I32 8.  A tap takes an id of the VFO id space: its output travels in b200_outputs.vfo_out[id], vfo_cap[id]
 * counts complex samples, vfo_count[id] is the number of samples of the effective stream in the chunk (the chunk's count,
 * or what the decimator makes of it) and b200_fe_vfo_max_out(fe, id, count) returns `count`.  b200_fe_vfo_count counts taps.
 * Bind and unbind follow the rules of add / remove VFO (b200_fe_set_decimation fails with B200_ESTATE after either); a tap id
 * passed to the VFO setters or to b200_fe_remove_vfo, and a VFO id passed to b200_fe_unbind_iq, fail with B200_EINVAL.  A tap
 * has no state of its own (b200_fe_reset resets the decimator and the DC blocker it reads from).  Every path that delivers
 * VFO outputs delivers taps: b200_fe_process, submit / wait, B200_MEM_DEVICE outputs, b200_shard_*.
 * Consumers' settings -- recorder (misc_modules/recorder, wav::Writer) WAV uint8 / int16 / int32 / float32: U8 / (I16, 32767) /
 * (I32, 2147483647) / CF32; IQ exporter (misc_modules/iq_exporter) int8 / int16 / int32 / float32: (I8, 128) / (I16, 32768) /
 * (I32, 2147483647) / CF32. */
#define B200_IQ_CF32 0   /* complex_t: the stream bindIQStream hands out; scalar ignored                                  */
#define B200_IQ_U8   1   /* wav.cpp uint8 rule: (unsigned char)(x * 127 + 128), truncated; scalar ignored                */
#define B200_IQ_I8   2   /* rintf(clamp(x * scalar)) -- volk_32f_s32f_convert_8i / _16i / _32i; I32 saturates at INT_MAX */
#define B200_IQ_I16  3   /*   exactly as b200_export_convert does                                                         */
#define B200_IQ_I32  4
int b200_fe_bind_iq(b200_fe* fe, int sample_type, float scalar);   /* returns an id */
int b200_fe_unbind_iq(b200_fe* fe, int id);
/* BroadcastFM's rdsOut on a front-end VFO, the radio's "Decode RDS" (decoder_modules/radio/src/demodulators/wfm.h:118-119,
 * broadcast_fm.h:121-142,165-170,196-202): the RDS branch hangs off the discriminator of VFO vfo_id (B200_DEMOD_WFM or
 * B200_DEMOD_WFM_STEREO, at most one RDS output each), whose audio goes on.  Returns an id of the VFO id space: its records
 * travel in b200_outputs.vfo_out[id] exactly as those of a B200_DEMOD_WFM_RDS_BITS VFO at the same offset and settings --
 * vfo_cap[id] counts records, vfo_count[id] is filled by b200_fe_wait (b200_fe_process, b200_shard_wait), b200_fe_vfo_max_out
 * bounds them (b200_rds_demod_max_out of the branch's 5 kS/s samples); b200_fe_vfo_count counts RDS outputs.  The work in
 * front of the discriminator runs once for both, and the branch's stages join the chunk's batched launches.
 * As setRDSOut's reset(): at the first chunk after a bind or an unbind the parent's discriminator history, stereo stage and
 * 15 kHz low-pass restart; RxVFO, IF chain and AF chain keep their state (a bind before the first chunk changes nothing of the
 * audio).  The branch starts fresh at its first bind; an unbind parks it with its state (translator phase, resampler
 * histories, RDSDemod), a later bind resumes it, b200_fe_reset clears it.
 * B200_EINVAL: a parent of another mode, a second output, an RDS id passed to the VFO setters, b200_fe_remove_vfo or
 * b200_fe_unbind_iq; B200_ESTATE: b200_fe_remove_vfo on a VFO that has an RDS output, b200_fe_set_decimation after a bind. */
int b200_fe_bind_rds(b200_fe* fe, int vfo_id);        /* returns an id */
int b200_fe_unbind_rds(b200_fe* fe, int id);
int b200_fe_vfo_count(b200_fe* fe);
/* upper bound of output samples one chunk of `count` input samples can produce for VFO id */
int b200_fe_vfo_max_out(b200_fe* fe, int id, int count);
int b200_fe_fft_max_lines(b200_fe* fe, int count);
/* clears every delay line / phase / counter (block::reset semantics) */
int b200_fe_reset(b200_fe* fe);

/* Synchronous chunk: returns when all outputs are in the caller's buffers (process() semantics of the
 * reference: data available on return).  in_fmt: B200_FMT_*, in_mem: B200_MEM_* */
int b200_fe_process(b200_fe* fe, const void* iq, int count, int in_fmt, int in_mem, b200_outputs* out);
/* Pipelined pair: submit() enqueues chunk k (H2D on a side stream + kernels + D2H) and returns
 * immediately; wait() blocks until the OLDEST submitted chunk's outputs are complete and fills its
 * counts.  Up to 2 chunks in flight (option "inflight": up to 4 -- each needs its own b200_outputs buffers).  Values are
 * identical to b200_fe_process; only timing changes. */
int b200_fe_submit(b200_fe* fe, const void* iq, int count, int in_fmt, int in_mem, b200_outputs* out);
int b200_fe_wait(b200_fe* fe);
/* number of kernels this handle has launched so far (bench.py's gpu_launches) */
long long b200_fe_launch_count(b200_fe* fe);
/* counters by name: "launches", "chunks", "s1_tma_launches" (stage-1 launches of this handle that ran the TMA-fed
 * filter-bank kernel), "s1_f2_jobs" (VFO-chunks of this handle whose (4, 27) decimating FIR ran inside that kernel), "graphs" / "graph_hits" / "graph_misses" (launch lists captured / replayed / launched plainly),
 * "host_ns_plan" / "host_ns_fft" / "host_ns_run" / "host_ns_join" / "host_ns_stage1" / "host_ns_tail" (host time spent inside
 * b200_fe_submit since creation, by section, in ns), "fused_chains" (VFOs whose stages behind stage 1 are planned into one
 * k_tail_fused launch per chunk); -1 for an unknown key */
long long b200_fe_stat(b200_fe* fe, const char* key);
/* Tuning / A-B switches (defaults are the fast paths; every variant is held to the same parity tests).  Every option applies
 * to the front end it is set on and to no other handle; stand-alone handles (b200_block, b200_fft, b200_chan) use the defaults.
 *  "s1"      stage-1 kernel: 8 (default) filter-bank form fed by the TMA engine (cf32 chunks, VFO offsets on a common
 *            frequency grid, first decimation 32 or 64); 7 the same form on cp.async tiles; 6 per-VFO complex taps on
 *            cp.async tiles, one tile buffer per CTA, three 4-warp CTAs per SM; 5 the same double-buffered, one CTA per SM;
 *            0 one thread per output.  Each falls through to the next when a plan does not fit it.
 *            "s1_stages" ring depth of the TMA kernel (2 default, 3); "s1_mt" tile of the per-VFO cp.async kernel in outputs,
 *            rounded down to a multiple of 128 (0 = automatic); "pair" 1 = VFOs at +f / -f share their stage-1 sums
 *  "tails"   2 (default): every stage behind stage 1 that has a register-window kernel runs in it (k_dfir_reg, k_poly_reg,
 *            k_fir_reg, k_firr_reg; "ft_prereg" caps how many leading decimating FIRs may, "ft_regall" 0 keeps the others in
 *            the fused launch k_tail_fused, tuned by "ft_threads", "ft_obmax", "ft_ob", "ft_smem_kb", "ft_direct");
 *            1 = one tiled kernel per stage, 0 = one thread per output.  Before VFOs are added.
 *  "overlap" 1 = tails of chunk k overlap stage 1 of chunk k+1 on a second stream (default).  Before VFOs are added.
 *  "fft"     1 = register-resident four-step passes (default), 0 = shared-memory radix-8 passes; "fft_cta" 8 (default)
 *            or 4 transforms per CTA;
 *            "fft_v" 1 (default) = a frame begun in earlier chunks is staged by copies and joins its chunk's batch, twiddles
 *            from shared memory; 0 = the frame is converted to cf32 and transformed alone, twiddles from global memory
 *            (same lines either way)
 *  "graph"   -1 (default) / 1: the launches behind stage 1 of a chunk are recorded; a chunk whose list was seen before
 *            replays a captured CUDA graph (decimation offsets, resampler phases and buffer parities repeat after a few
 *            chunks of any fixed size); 0 = plain launches.
 *  "host_direct" -1 (default): VFO outputs in b200_host_alloc buffers are stored by the kernels themselves for chunks up to
 *            4 Mi samples (no copy to enqueue), 1 always, 0 never (copy engine); IQ taps (b200_fe_bind_iq) under -1 only
 *            when their output is at most 64 KiB, since the kernel's own stores over PCIe are slower than the copy engine
 *  "inflight" chunks between b200_fe_submit and b200_fe_wait: 2 (default) ... 4
 *  "s1_ctas" persistent CTAs of the TMA stage 1 (0 = one per SM)
 *  "pdl"     programmatic dependent launch for the chain kernels behind stage 1 (a successor is scheduled and loads its tables
 *            under its predecessor, and touches the stage buffers behind griddepcontrol.wait): 2 (default) launches of at most
 *            two CTAs per SM -- the small grids of chunks up to about 1e6 samples --, 1 every launch, 0 never.  The environment
 *            variable B200_PDL, read once per process, sets the default
 *  "s1_diag" measurement only (outputs are garbage): 1 = the TMA stage 1 loads its tiles but does not filter them, 2 = it
 *            filters whatever its tile buffers hold and loads nothing -- what the ring alone and the consumer warps alone
 *            sustain (tools/s1_bounds.py)
 *  "time_s1" 1 = bracket the launch groups of every chunk with CUDA events (b200_fe_s1_stats / b200_fe_group_stats) */
int b200_fe_set_option(b200_fe* fe, const char* key, int value);
/* device time spent in the stage-1 (translate + first decimation) launches since the last call, and their count;
 * synchronises on the recorded events ("time_s1" must be on).  bench.py's roofline leg reads this. */
int b200_fe_s1_stats(b200_fe* fe, double* ms_total, int* launches);
/* the same for a launch group: 0 = stage 1, 1 = everything behind stage 1 of a chunk (register FIRs, fused tail, carries),
 * 2 = the spectrum branch of a chunk, 3 = the IQ taps of a chunk (k_iq_tap).  At most 512 samples per group are kept between
 * two calls. */
int b200_fe_group_stats(b200_fe* fe, int group, double* ms_total, int* launches);

/* ------------------------------------------------------------------------------------------
 * One IQ stream, VFO groups on several GPUs (BASELINE config 4).  Replaces the Splitter fan-out
 * (core/src/dsp/routing/splitter.h:46-61: every bound consumer gets a memcpy of every chunk) ACROSS devices: one process per
 * GPU, each with its own b200_fe holding its VFO group (rank 0 also keeps the FFT branch); rank 0 ingests the chunk and
 * ncclBroadcasts the raw IQ on a communication stream, one chunk ahead of the compute.  There is no other exchange.
 * b200_shard_unique_id: rank 0 makes the 128-byte NCCL id, the caller hands it to the other ranks (any side channel);
 * every rank then calls b200_shard_create, and b200_shard_submit / b200_shard_wait with the SAME count and format per
 * chunk (iq is read on rank 0 only).  NCCL is bound at run time (libnccl.so.2).
 * ------------------------------------------------------------------------------------------ */
typedef struct b200_shard b200_shard;
int         b200_shard_unique_id(void* id128);
b200_shard* b200_shard_create(b200_fe* fe, int rank, int world, const void* id128);
int         b200_shard_submit(b200_shard* sh, const void* iq, int count, int in_fmt, int in_mem, b200_outputs* out);
int         b200_shard_wait(b200_shard* sh);
long long   b200_shard_bytes_broadcast(b200_shard* sh);      /* bytes this rank has put through ncclBroadcast so far */
void        b200_shard_destroy(b200_shard* sh);

/* waterfall zoom (max-decimate) + peak hold on the device line, bit-exact with
 * doZoom / pushFFT hold loop (core/src/gui/widgets/waterfall.cpp:65-90, 935-939).
 * line: fft_size dB values (mem), out/hold: out_size floats (same mem). hold may be NULL. */
int b200_fft_zoom_hold(const float* line, int fft_size, int offset, int width, int out_size,
                       float* out, float* hold, float hold_speed, int mem);

/* ------------------------------------------------------------------------------------------
 * Stand-alone blocks (un-fused graphs keep working): each mirrors one reference block's
 * init(...) / process(count, in, out) -> out count.  Host buffers in, host buffers out,
 * synchronous, state carried across calls exactly like the reference block.
 * ------------------------------------------------------------------------------------------ */
typedef struct b200_block b200_block;

b200_block* b200_xlator_create(double offsetHz, double samplerate);             /* channel::FrequencyXlator (frequency_xlator.h:15-50) */
int         b200_xlator_set_offset(b200_block* b, double offsetHz, double samplerate);
b200_block* b200_decim_create(int ratio);                                       /* multirate::PowerDecimator<complex_t> (power_decimator.h:51-67) */
b200_block* b200_resamp_create(double inSamplerate, double outSamplerate);      /* multirate::RationalResampler<complex_t|stereo_t> (rational_resampler.h:82-96) */
b200_block* b200_fir_cr_create(const float* taps, int ntaps, int decimation);   /* filter::FIR / DecimatingFIR<complex_t,float> (fir.h:62-83, decimating_fir.h:45-68) */
/* FIR::setTaps (fir.h:31-52) of a block made by b200_fir_cr_create: new coefficients at the next chunk boundary, the
 * most recent delay-line samples are kept (a decimating filter restarts its decimation phase, decimating_fir.h:18-25) */
int         b200_fir_cr_set_taps(b200_block* b, const float* taps, int ntaps);
b200_block* b200_fir_rr_create(const float* taps, int ntaps);                   /* filter::FIR<float,float> */
b200_block* b200_rxvfo_create(double inSamplerate, double outSamplerate, double bandwidth, double offset); /* channel::RxVFO (rx_vfo.h:89-100) */
int         b200_rxvfo_set_offset(b200_block* b, double offset);
int         b200_rxvfo_set_bandwidth(b200_block* b, double bandwidth);
b200_block* b200_quad_create(double deviationHz, double samplerate);            /* demod::Quadrature (quadrature.h:39-46): complex -> float */
b200_block* b200_wfm_create(double deviationHz, double samplerate, int stereo, int lowPass); /* demod::BroadcastFM (mono or stereo branch, broadcast_fm.h:144-212): complex -> stereo */
b200_block* b200_wfm_rds_create(double deviationHz, double samplerate);             /* its RDS branch (rdsOut, broadcast_fm.h:165-170,196-202): complex IF -> complex at 5 kS/s */
b200_block* b200_nfm_create(double samplerate, double bandwidth, int lowPass);  /* demod::FM<stereo_t> */
b200_block* b200_am_create(int agcMode, double bandwidth, double agcAttack, double agcDecay, double dcBlockRate, double samplerate); /* demod::AM<stereo_t> */
b200_block* b200_noise_blanker_create(double rate, double level);                     /* noise_reduction::NoiseBlanker (noise_blanker.h:12-17): complex -> complex */
int         b200_noise_blanker_set(b200_block* b, double rate, double level);         /* setRate / setLevel (noise_blanker.h:19-30): next chunk, the running amplitude is kept */
b200_block* b200_fmif_create(int bins);                                              /* noise_reduction::FMIF (fm_if.h:20-24): complex -> complex */
b200_block* b200_squelch_create(double level);                                       /* noise_reduction::PowerSquelch (power_squelch.h:33-50): complex -> complex */
b200_block* b200_deemph_create(double tau, double samplerate);                       /* filter::Deemphasis<stereo_t> (deephasis.h:58-77): stereo -> stereo */
b200_block* b200_ssb_create(int mode /*0 USB,1 LSB,2 DSB*/, double bandwidth, double samplerate, double agcAttack, double agcDecay); /* demod::SSB<stereo_t> */
/* returns the output sample count; in/out are host pointers of the block's sample types */
int  b200_block_process(b200_block* b, int count, const void* in, void* out);
int  b200_block_max_out(b200_block* b, int count);
int  b200_block_reset(b200_block* b);
void b200_block_destroy(b200_block* b);

/* RDSDemod, the symbol-rate half of the RDS path (decoder_modules/radio/src/rds_demod.h:20-73): FastAGC -> Costas loop ->
 * complex band-pass -> second Costas loop at the symbol frequency -> real part -> Mueller & Mueller clock recovery (128 x 8
 * polyphase interpolator) -> slicer -> differential decoder.  Input: the complex 5 kS/s stream BroadcastFM's rdsOut carries
 * (b200_wfm_rds_create, or a front-end VFO in B200_DEMOD_WFM_RDS mode); `in` may be a host or a device pointer.  Per recovered
 * symbol one soft value (RDSDemod::soft) and one decoded bit (RDSDemod::out), written to HOST buffers of at least
 * b200_rds_demod_max_out(count) entries; returns the number of symbols of this call (it depends on the recovered clock, so this
 * call waits for its launch; a front-end VFO in B200_DEMOD_WFM_RDS_BITS mode runs the same kernel inside the submit / wait
 * pipeline instead).
 * The three feedback loops run on one thread of the device in the reference's fp32 statement order; the band-pass in parallel. */
typedef struct b200_rds_demod b200_rds_demod;
b200_rds_demod* b200_rds_demod_create(void);
int        b200_rds_demod_process(b200_rds_demod* r, int count, const void* in_iq, float* soft, uint8_t* hard);
int        b200_rds_demod_max_out(int count);
int        b200_rds_demod_reset(b200_rds_demod* r);                        /* RDSDemod::reset (rds_demod.h:52-62) */
long long  b200_rds_demod_launch_count(b200_rds_demod* r);
int        b200_rds_demod_taps(float* bandpass_iq, int cap_taps, float* bank_128x8);   /* test hook: tap count; the two designed tap sets */
void       b200_rds_demod_destroy(b200_rds_demod* r);

/* Stand-alone spectrum handler == IQFrontEnd::handler on one already-framed block of nz samples:
 * window*(-1)^n -> FFT -> 10log10(|X/N|^2)  (iq_frontend.cpp:248-267).  Host in, host out. */
typedef struct b200_fft b200_fft;
b200_fft* b200_fft_create(int size, int nz, int window);
int       b200_fft_frame(b200_fft* f, const float* iq_nz, float* out_db);
int       b200_fft_raw(b200_fft* f, const float* iq_nz, float* out_complex);    /* test hook: complex spectrum */
void      b200_fft_destroy(b200_fft* f);

/* BASELINE config 3 (not a reference block: SURVEY.md section 0 fact 9, section 8d): a 256-channel critically sampled polyphase
 * filter-bank channelizer, `taps_per_branch` (127) taps per branch; prototype = the reference's
 * taps::windowedSinc<float>(256 * 127, fs / 512, fs, window::nuttall) (core/src/dsp/taps/windowed_sinc.h:31-34).
 * Channel k of output time m:  y_k[m] = sum_t h[t] x[n0 + t] e^{-j 2 pi k (n0 + t) / 256},  n0 = 256 m + 255 - (T - 1), T = 256 * 127
 * (translate by -k fs/256, T-tap FIR, keep every 256th sample); the stream history is carried across calls.
 * count: a multiple of 256; out[m * 256 + k]; returns the number of output times. */
typedef struct b200_chan b200_chan;
b200_chan* b200_chan_create(int channels, int taps_per_branch, int max_chunk);
int        b200_chan_prototype(b200_chan* c, float* out, int cap);          /* the prototype taps (tests) */
int        b200_chan_process(b200_chan* c, const void* iq, int count, int in_mem, void* out, int out_mem);
long long  b200_chan_launch_count(b200_chan* c);
void       b200_chan_destroy(b200_chan* c);

/* pinned host memory for stream buffers (replaces buffer::alloc/volk_malloc, core/src/dsp/buffer/buffer.h:7-18) */
void* b200_host_alloc(uint64_t bytes);
void  b200_host_free(void* p);

/* ------------------------------------------------------------------------------------------
 * Data formats either side of the path (SURVEY.md section 8f)
 * ------------------------------------------------------------------------------------------ */
/* Compressed-stream ingest: dsp::compression::SampleStreamDecompressor::process
 * (core/src/dsp/compression/sample_stream_decompressor.h:15-37).  A packet is an 8-byte header
 * {u16 compression, u16 PCMType, f32 scaler} + int8 / int16 / float32 I,Q pairs.  b200_pcm_packet_info reads
 * the header (host memory) and returns the B200_FMT_* of the payload, the conversion factor
 * 1 / (32768/scaler) resp. 1 / (128/scaler) the reference hands to volk_16i/8i_s32f_convert_32f, the sample
 * count and the payload offset; b200_fe_set_ingest_scale makes the front end convert the next integer chunks
 * with that factor (scale <= 0 restores 1/32768, 1/128).  The payload then goes to b200_fe_process as is. */
int b200_pcm_packet_info(const void* packet, int bytes, int* fmt, float* scale, int* count, int* data_offset);
int b200_fe_set_ingest_scale(b200_fe* fe, int fmt, float scale);
/* IQ export: dsp::compression::SampleStreamCompressor::process (sample_stream_compressor.h:30-66): finds the
 * maximum VALUE of the 2*count floats (volk_32f_index_max_32u), writes header + payload scaled by 32768/max
 * (int16) or 128/max (int8), rounded like rintf and saturated; B200_FMT_CF32 copies.  Returns the packet size.
 * Runs on a stream of the calling thread with grow-only scratch buffers (no allocation, no device-wide synchronisation per
 * packet); with device buffers, work the caller queued on other streams than the default one must be finished. */
int b200_pcm_compress(const float* iq, int count, int pcm_fmt, void* packet, int cap_bytes, int mem);
/* Recorder sample types: wav::Writer::write (core/src/utils/wav.cpp:150-183): uint8 = x*127 + 128 (truncated),
 * int16 = rint(x*32767) saturated, int32 = rint(x*2147483647) saturated (the device saturates at INT_MAX where the
 * CPU conversion overflows).  in/out are n floats / n samples in `mem`. */
#define B200_EXPORT_U8  0
#define B200_EXPORT_I16 1
#define B200_EXPORT_I32 2
int b200_export_convert(const float* in, long long n, int sample_type, void* out, int mem);

#ifdef __cplusplus
}
#endif
#endif

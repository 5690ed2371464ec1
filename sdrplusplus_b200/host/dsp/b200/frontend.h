// host/dsp/b200/frontend.h -- the fused front end as a block: one input stream, every VFO's demodulated audio and
// the FFT lines per chunk in ONE device pass (IQ read from HBM once).  This is what replaces the reference's
// Splitter + Reshaper/Handler + N x (RxVFO + demodulator) worker threads inside IQFrontEnd
// (core/src/signal_path/iq_frontend.cpp:30-72) when a maintainer opts into the GPU path (INTEGRATION.md).
#pragma once
#include <cstring>
#include <vector>
#include "../block.h"

namespace dsp::b200 {
    class FrontEnd : public block {
    public:
        // acquire/release: the reference's FFT line callbacks (iq_frontend.h:23), unchanged
        // decimRatio / dcBlocking: IQFrontEnd::init's arguments of the same name (iq_frontend.h:23); the decimation has to be
        // known before the FFT branch and the VFOs are configured, which is why it is an init argument here too
        void init(stream<complex_t>* in, double samplerate, int fftSize, double fftRate, int fftWindow,
                  float* (*acquireFFTBuffer)(void*), void (*releaseFFTBuffer)(void*), void* fftCtx,
                  int decimRatio = 1, bool dcBlocking = false) {
            _in = in;
            acquire = acquireFFTBuffer; release = releaseFFTBuffer; ctx = fftCtx;
            fe = b200_fe_create(samplerate, in->bufferSize());
            _samplerate = samplerate; _decim = decimRatio; _rate = fftRate; _window = fftWindow;
            if (fe && decimRatio > 1) { b200_fe_set_decimation(fe, decimRatio); }
            if (fe && dcBlocking) { b200_fe_set_dc_blocking(fe, 1); }
            registerInput(_in);
            inited = true;
            setFFTSize(fftSize);
        }
        ~FrontEnd() override {
            if (inited) { stop(); }
            for (auto* s : outs_) { delete s; }
            b200_host_free(lines);
            b200_fe_destroy(fe);
        }
        // returns the VFO id; its audio arrives on vfoOut(id)
        int addVFO(const b200_vfo_cfg& cfg) {
            std::lock_guard<std::recursive_mutex> lk(ctrlMtx);
            tempStop();
            int id = b200_fe_add_vfo(fe, &cfg);
            if (id >= 0) {
                if ((int)outs_.size() <= id) { outs_.resize(id + 1, nullptr); }
                outs_[id] = new stream<stereo_t>(b200_fe_vfo_max_out(fe, id, _in->bufferSize()));
                registerOutput(outs_[id]);
            }
            tempStart();
            return id;
        }
        void removeVFO(int id) {
            std::lock_guard<std::recursive_mutex> lk(ctrlMtx);
            tempStop();
            for (size_t i = 0; i < rds_.size(); i++) {
                if (rds_[i].vfo == id) { unbindRDS(rds_[i].id); break; }
            }
            if (b200_fe_remove_vfo(fe, id) == 0) { dropOut(id); }
            tempStart();
        }
        // the radio's "Decode RDS" (BroadcastFM::setRDSOut, demodulators/wfm.h:118-119) on a WFM VFO: returns an id whose
        // stream, vfoOut(id), carries one b200_rds_symbol per recovered symbol (read them with rdsSymbols), decoded from that
        // VFO's own discriminator beside its audio (b200_fe_bind_rds)
        int bindRDS(int vfoId) {
            std::lock_guard<std::recursive_mutex> lk(ctrlMtx);
            tempStop();
            int id = b200_fe_bind_rds(fe, vfoId);
            if (id >= 0) {
                if ((int)outs_.size() <= id) { outs_.resize(id + 1, nullptr); }
                outs_[id] = new stream<stereo_t>(b200_fe_vfo_max_out(fe, id, _in->bufferSize()));
                registerOutput(outs_[id]);
                rds_.push_back({ vfoId, id });
            }
            tempStart();
            return id;
        }
        void unbindRDS(int id) {
            std::lock_guard<std::recursive_mutex> lk(ctrlMtx);
            tempStop();
            if (b200_fe_unbind_rds(fe, id) == 0) {
                dropOut(id);
                for (size_t i = 0; i < rds_.size(); i++) {
                    if (rds_[i].id == id) { rds_.erase(rds_.begin() + i); break; }
                }
            }
            tempStart();
        }
        // IQFrontEnd::bindIQStream / unbindIQStream (iq_frontend.h:34-35): the effective stream (behind the decimation and DC
        // blocking given to init, and setInvertIQ) goes to every bound stream, whose buffer must hold a whole input chunk;
        // each is a CF32 tap of the front end (b200_fe_bind_iq).  Any number of streams, up to the VFO id space.
        void bindIQStream(stream<complex_t>* s) {
            std::lock_guard<std::recursive_mutex> lk(ctrlMtx);
            tempStop();
            int id = b200_fe_bind_iq(fe, B200_IQ_CF32, 0.0f);
            if (id >= 0) {
                iqs_.push_back({ s, id });
                registerOutput(s);
            }
            tempStart();
        }
        void unbindIQStream(stream<complex_t>* s) {
            std::lock_guard<std::recursive_mutex> lk(ctrlMtx);
            tempStop();
            for (size_t i = 0; i < iqs_.size(); i++) {
                if (iqs_[i].s != s) { continue; }
                b200_fe_unbind_iq(fe, iqs_[i].id);
                unregisterOutput(s);
                iqs_.erase(iqs_.begin() + i);
                break;
            }
            tempStart();
        }
        void setVFOOffset(int id, double offset) { b200_fe_set_vfo_offset(fe, id, offset); }
        void setVFOBandwidth(int id, double bandwidth) { b200_fe_set_vfo_bandwidth(fe, id, bandwidth); }
        // the radio module's volume / squelch / blanker / noise-reduction / de-emphasis / AGC setters: taken at the next chunk,
        // every block keeps its state, the worker keeps running (b200_fe_set_vfo_config); returns B200_EINVAL for a change
        // that needs a new demodulator (removeVFO + addVFO)
        int setVFOConfig(int id, const b200_vfo_cfg& cfg) { return b200_fe_set_vfo_config(fe, id, &cfg); }
        // IQFrontEnd::setDCBlocking / setInvertIQ (iq_frontend.cpp:117-123): take effect at the next chunk
        void setDCBlocking(bool enabled) { b200_fe_set_dc_blocking(fe, enabled); }
        void setInvertIQ(bool enabled) { b200_fe_set_invert_iq(fe, enabled); }
        // IQFrontEnd::getEffectiveSamplerate (iq_frontend.cpp:214-216)
        double getEffectiveSamplerate() const { return _samplerate / _decim; }
        // IQFrontEnd::setFFTSize / setFFTRate / setFFTWindow (iq_frontend.cpp:185-201)
        void setFFTSize(int fftSize) { size = fftSize; updateFFTPath(); }
        void setFFTRate(double rate) { _rate = rate; updateFFTPath(); }
        void setFFTWindow(int window) { _window = window; updateFFTPath(); }
        // every VFO's output stream has 8-byte elements: stereo_t audio, complex_t for B200_DEMOD_RAW / B200_DEMOD_WFM_RDS, and
        // one b200_rds_symbol per recovered symbol for B200_DEMOD_WFM_RDS_BITS (read them with rdsSymbols)
        stream<stereo_t>* vfoOut(int id) { return outs_[id]; }
        static const b200_rds_symbol* rdsSymbols(const stream<stereo_t>* s) { return (const b200_rds_symbol*)s->readBuf; }

        int run() override {
            int count = _in->read();
            if (count < 0) { return -1; }
            b200_outputs o = {};
            for (size_t i = 0; i < outs_.size(); i++) {
                if (!outs_[i]) { continue; }
                o.vfo_out[i] = outs_[i]->writeBuf;
                o.vfo_cap[i] = outs_[i]->bufferSize();
            }
            for (auto& t : iqs_) {
                o.vfo_out[t.id] = t.s->writeBuf;
                o.vfo_cap[t.id] = t.s->bufferSize();
            }
            o.fft_out = lines;
            o.fft_cap_lines = b200_fe_fft_max_lines(fe, count);
            o.out_mem = B200_MEM_HOST;
            int rc = b200_fe_process(fe, _in->readBuf, count, B200_FMT_CF32, B200_MEM_HOST, &o);
            _in->flush();
            if (rc < 0) { return -1; }
            for (int l = 0; l < o.fft_lines && acquire; l++) {
                float* dst = acquire(ctx);
                if (dst) { memcpy(dst, lines + (size_t)l * size, (size_t)size * sizeof(float)); }
                release(ctx);
            }
            for (size_t i = 0; i < outs_.size(); i++) {
                if (outs_[i] && o.vfo_count[i] > 0 && !outs_[i]->swap(o.vfo_count[i])) { return -1; }
            }
            // every bound stream gets every chunk, as IQFrontEnd's splitter hands it out (splitter.h:46-61)
            for (auto& t : iqs_) {
                if (!t.s->swap(o.vfo_count[t.id])) { return -1; }
            }
            return count;
        }
    private:
        void dropOut(int id) {
            if (id < (int)outs_.size() && outs_[id]) {
                unregisterOutput(outs_[id]);
                delete outs_[id];
                outs_[id] = nullptr;
            }
        }
        void updateFFTPath() {
            std::lock_guard<std::recursive_mutex> lk(ctrlMtx);
            tempStop();
            if (fe) { b200_fe_set_fft(fe, size, _rate, _window); }
            b200_host_free(lines);
            lines = (float*)b200_host_alloc((uint64_t)(fe && size ? b200_fe_fft_max_lines(fe, _in->bufferSize()) : 1) * (size ? size : 1) * sizeof(float));
            tempStart();
        }
        double _samplerate = 0, _rate = 20.0;
        int _decim = 1, _window = 2;
        stream<complex_t>* _in = nullptr;
        b200_fe* fe = nullptr;
        std::vector<stream<stereo_t>*> outs_;
        struct BoundIQ { stream<complex_t>* s; int id; };
        std::vector<BoundIQ> iqs_;
        struct BoundRDS { int vfo, id; };
        std::vector<BoundRDS> rds_;
        float* lines = nullptr;
        int size = 0;
        float* (*acquire)(void*) = nullptr;
        void (*release)(void*) = nullptr;
        void* ctx = nullptr;
    };
}

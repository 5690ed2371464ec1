// host/test_adapter.cpp -- the reference's graph idiom on the adapter headers: a writer thread swap()s IQ chunks into
// a stream, RxVFO -> BroadcastFM run as worker-thread blocks, the main thread reads stereo audio.  Prints one line
// "<samples_out> <checksum>"; tests/test_host_adapter.py compares it with the oracle on the same seeded input.
#include <cmath>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>
#include "dsp/channel/rx_vfo.h"
#include "dsp/demod/broadcast_fm.h"
#include "dsp/b200/frontend.h"
#include "dsp/sink/handler_sink.h"
#include "radio/rds_demod.h"
#include "dsp/compression/sample_stream_compressor.h"   // compiled here; exercised through the C ABI in tests/test_gpu_parity.py

static std::vector<float> g_line(65536);
static int g_lines = 0;
static float* acquireLine(void*) { return g_line.data(); }
static void releaseLine(void*) { g_lines++; }

int main(int argc, char** argv) {
    if (argc < 3) { fprintf(stderr, "usage: %s iq.f32 audio_out.f32\n", argv[0]); return 2; }
    if (b200_init(0) != 0) { fprintf(stderr, "%s\n", b200_last_error()); return 3; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { return 2; }
    fseek(f, 0, SEEK_END);
    long bytes = ftell(f);
    fseek(f, 0, SEEK_SET);
    std::vector<dsp::complex_t> iq(bytes / sizeof(dsp::complex_t));
    if (fread(iq.data(), sizeof(dsp::complex_t), iq.size(), f) != iq.size()) { return 2; }
    fclose(f);

    const double fs = 2.4e6;
    const int chunk = 12000;                       // file_source: fs / 200
    dsp::stream<dsp::complex_t> input(chunk);
    if (argc > 3 && !strcmp(argv[3], "fused")) {
        // the fused front end block: FFT lines through the reference's acquire/release callbacks + one WFM VFO
        dsp::b200::FrontEnd fe;
        fe.init(&input, fs, 65536, 20.0, B200_WIN_NUTTALL, acquireLine, releaseLine, nullptr);
        b200_vfo_cfg cfg = {};
        cfg.offset = 300000.0; cfg.out_samplerate = 250000.0; cfg.bandwidth = 150000.0; cfg.demod = B200_DEMOD_WFM;
        cfg.deviation = 75000.0; cfg.low_pass = 1;
        int id = fe.addVFO(cfg);
        if (id < 0) { fprintf(stderr, "%s\n", b200_last_error()); return 3; }
        fe.start();
        std::thread w([&] {
            for (size_t i = 0; i + chunk <= iq.size(); i += chunk) {
                memcpy(input.writeBuf, &iq[i], chunk * sizeof(dsp::complex_t));
                if (!input.swap(chunk)) { return; }
            }
        });
        std::vector<dsp::stereo_t> audio;
        for (size_t c = 0; c < iq.size() / chunk; c++) {
            int n = fe.vfoOut(id)->read();
            if (n < 0) { break; }
            audio.insert(audio.end(), fe.vfoOut(id)->readBuf, fe.vfoOut(id)->readBuf + n);
            fe.vfoOut(id)->flush();
        }
        w.join();
        fe.stop();
        FILE* o = fopen(argv[2], "wb");
        fwrite(audio.data(), sizeof(dsp::stereo_t), audio.size(), o);
        fclose(o);
        printf("%zu %d\n", audio.size(), g_lines);
        return 0;
    }
    if (argc > 3 && !strcmp(argv[3], "iqtap")) {
        // a baseband recorder's wiring: a sink::Handler<complex_t> worker on a stream bound with bindIQStream behind a
        // front end that decimates by 4 and blocks DC (IQFrontEnd::init's decimRatio / dcBlocking); no FFT, no VFO
        dsp::b200::FrontEnd fe;
        fe.init(&input, fs, 0, 20.0, B200_WIN_NUTTALL, nullptr, nullptr, nullptr, 4, true);
        dsp::stream<dsp::complex_t> iqs(chunk);
        fe.bindIQStream(&iqs);
        struct Rec { std::vector<dsp::complex_t> x; std::mutex m; std::condition_variable cv; size_t chunks = 0; } rec;
        dsp::sink::Handler<dsp::complex_t> sink(&iqs, [](dsp::complex_t* d, int n, void* ctx) {
            Rec* r = (Rec*)ctx;
            std::lock_guard<std::mutex> lk(r->m);
            r->x.insert(r->x.end(), d, d + n);
            r->chunks++;
            r->cv.notify_all();
        }, &rec);
        sink.start();
        fe.start();
        const size_t nch = iq.size() / chunk;
        for (size_t i = 0; i < nch; i++) {
            memcpy(input.writeBuf, &iq[i * chunk], chunk * sizeof(dsp::complex_t));
            if (!input.swap(chunk)) { return 4; }
        }
        {
            std::unique_lock<std::mutex> lk(rec.m);
            rec.cv.wait(lk, [&] { return rec.chunks == nch; });
        }
        fe.stop();
        sink.stop();
        fe.unbindIQStream(&iqs);
        FILE* o = fopen(argv[2], "wb");
        fwrite(rec.x.data(), sizeof(dsp::complex_t), rec.x.size(), o);
        fclose(o);
        printf("%zu %zu\n", rec.x.size(), rec.chunks);
        return 0;
    }
    if (argc > 3 && !strcmp(argv[3], "rds")) {
        // the radio module's RDS wiring (demodulators/wfm.h:78-81): BroadcastFM(rdsOut = true) -> RDSDemod; input at the 250 kS/s IF
        const int ifchunk = 12500;
        dsp::stream<dsp::complex_t> ifin(ifchunk);
        dsp::demod::BroadcastFM wfm(&ifin, 75000.0, 250000.0, false, true, true);
        RDSDemod rds(&wfm.rdsOut, true);
        if (!wfm.ok() || !rds.ok()) { fprintf(stderr, "%s\n", b200_last_error()); return 3; }
        rds.start();
        wfm.start();
        const size_t nch = iq.size() / ifchunk;
        std::thread w([&] {
            for (size_t i = 0; i < nch; i++) {
                memcpy(ifin.writeBuf, &iq[i * ifchunk], ifchunk * sizeof(dsp::complex_t));
                if (!ifin.swap(ifchunk)) { return; }
            }
        });
        std::thread audio([&] {                       // the audio output has to be drained like the radio's sink does
            for (size_t c = 0; c < nch; c++) {
                if (wfm.out.read() < 0) { return; }
                wfm.out.flush();
            }
        });
        std::vector<uint8_t> bits;
        std::vector<float> softs;
        for (size_t c = 0; c < nch; c++) {            // one RDS chunk (250 samples at 5 kS/s) per IF chunk
            int n = rds.out.read();
            if (n < 0) { break; }
            bits.insert(bits.end(), rds.out.readBuf, rds.out.readBuf + n);
            rds.out.flush();
            int m = rds.soft.read();
            if (m < 0) { break; }
            softs.insert(softs.end(), rds.soft.readBuf, rds.soft.readBuf + m);
            rds.soft.flush();
        }
        w.join();
        audio.join();
        wfm.stop();
        rds.stop();
        FILE* o = fopen(argv[2], "wb");
        fwrite(bits.data(), 1, bits.size(), o);
        fclose(o);
        printf("%zu %zu\n", bits.size(), softs.size());
        return 0;
    }
    dsp::channel::RxVFO vfo(&input, fs, 250000.0, 150000.0, 300000.0);
    dsp::demod::BroadcastFM wfm(&vfo.out, 75000.0, 250000.0, false, true, false);
    if (!vfo.ok() || !wfm.ok()) { fprintf(stderr, "%s\n", b200_last_error()); return 3; }
    wfm.start();
    vfo.start();
    std::thread writer([&] {
        for (size_t i = 0; i + chunk <= iq.size(); i += chunk) {
            memcpy(input.writeBuf, &iq[i], chunk * sizeof(dsp::complex_t));
            if (!input.swap(chunk)) { return; }
        }
    });
    const size_t nchunks = iq.size() / chunk;
    std::vector<dsp::stereo_t> audio;
    for (size_t c = 0; c < nchunks; c++) {
        int n = wfm.out.read();
        if (n < 0) { break; }
        audio.insert(audio.end(), wfm.out.readBuf, wfm.out.readBuf + n);
        wfm.out.flush();
    }
    writer.join();
    vfo.stop();
    wfm.stop();
    FILE* o = fopen(argv[2], "wb");
    fwrite(audio.data(), sizeof(dsp::stereo_t), audio.size(), o);
    fclose(o);
    double cs = 0;
    for (auto& s : audio) { cs += std::fabs(s.l) + std::fabs(s.r); }
    printf("%zu %.9e\n", audio.size(), cs);
    return 0;
}

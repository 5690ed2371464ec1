// tests/vfo_settings_adapter.cpp -- dsp::b200::FrontEnd::setVFOConfig called from a thread other than the block's worker while
// the worker runs: a WFM VFO with the radio's AF chain and volume, settings changed before chunks 5, 10 and 15 (volume + noise
// blanker on, high-pass on, blanker off + muted).  The writer thread makes each change once the audio of the chunk before it
// has been read, so the change lands at that chunk boundary whatever the thread timing.  Writes the stereo audio; the test
// compares it with FrontEnd.set_vfo_config on the Python side.  Built and run by tests/test_gpu_vfo_settings.py.
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <thread>
#include <vector>
#include "dsp/b200/frontend.h"

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
    const int chunk = 12000;
    const size_t nch = iq.size() / chunk;
    dsp::stream<dsp::complex_t> input(chunk);
    dsp::b200::FrontEnd fe;
    fe.init(&input, fs, 0, 20.0, B200_WIN_NUTTALL, nullptr, nullptr, nullptr);
    b200_vfo_cfg cfg = {};
    cfg.offset = 300000.0; cfg.out_samplerate = 250000.0; cfg.bandwidth = 150000.0; cfg.demod = B200_DEMOD_WFM;
    cfg.deviation = 75000.0; cfg.low_pass = 1;
    cfg.af_samplerate = 48000.0; cfg.af_deemph_tau = 50e-6;
    cfg.af_volume_on = 1; cfg.af_volume = 0.7;
    cfg.nb_level = 2.0; cfg.nr_bins = 32; cfg.squelch_level = -50.0;
    int id = fe.addVFO(cfg);
    if (id < 0) { fprintf(stderr, "%s\n", b200_last_error()); return 3; }
    b200_vfo_cfg c5 = cfg, c10, c15;
    c5.af_volume = 1.3; c5.nb_on = 1;
    c10 = c5; c10.af_high_pass = 1;
    c15 = c10; c15.nb_on = 0; c15.af_muted = 1;
    fe.start();
    std::atomic<size_t> delivered{ 0 };
    std::atomic<int> failed{ 0 };
    std::thread writer([&] {
        for (size_t k = 0; k < nch; k++) {
            const b200_vfo_cfg* c = k == 5 ? &c5 : k == 10 ? &c10 : k == 15 ? &c15 : nullptr;
            if (c) {
                while (delivered.load() < k) { std::this_thread::sleep_for(std::chrono::microseconds(50)); }
                if (fe.setVFOConfig(id, *c) != 0) { failed = 1; }
            }
            memcpy(input.writeBuf, &iq[k * chunk], chunk * sizeof(dsp::complex_t));
            if (!input.swap(chunk)) { return; }
        }
    });
    std::vector<dsp::stereo_t> audio;
    for (size_t k = 0; k < nch; k++) {
        int n = fe.vfoOut(id)->read();
        if (n < 0) { break; }
        audio.insert(audio.end(), fe.vfoOut(id)->readBuf, fe.vfoOut(id)->readBuf + n);
        fe.vfoOut(id)->flush();
        delivered = k + 1;
    }
    writer.join();
    fe.stop();
    if (failed) { fprintf(stderr, "setVFOConfig: %s\n", b200_last_error()); return 4; }
    FILE* o = fopen(argv[2], "wb");
    fwrite(audio.data(), sizeof(dsp::stereo_t), audio.size(), o);
    fclose(o);
    printf("%zu\n", audio.size());
    return 0;
}
